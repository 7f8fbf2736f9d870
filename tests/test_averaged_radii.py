"""Per-particle radii of the averaged-position surface (Zhu & Bridson's r_bar; reconstruct_surface(particle_radii=...), DESIGN.md
section 12.2).

* the plain-C restatement (so_reconstruct_averaged_radii in tests/averaged_radii_oracle.c) against a float64 numpy restatement, within
  a per-point rounding bound, plain and with the Jacobian correction;
* radii all equal to particle_radius reduce to the single radius bit for bit (oracle and CPU executor);
* one particle, the edge-of-support particle, two distant particles and a bidisperse pair of balls, measured on the oracle;
* refusals, context reuse and the command line;
* the device pipeline on the CPU executor of the CUDA sources against the oracle, bit for bit.
The GPU-marked counterpart of the device cases is tests/test_zzz_gpu_averaged_radii.py."""
import ctypes as C
import os

import numpy as np
import pytest

import c_oracle
from test_anisotropic import KW, R, _aniso_params, _cube, _sphere
from test_averaged_correction import T_LOW, T_HIGH, _params_hrc, numpy_corrected, oracle_reconstruct_corrected
from test_averaged_surface import (CASES, ORACLE_CLOUDS, SHELL_KW, _busiest_tile, _edge_shell_particle, _shell_point, _tile_points,
                                   mesh_topology, numpy_averaged, oracle_reconstruct_averaged)
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

EPS = 2.0 ** -24               # unit roundoff of f32


# ------------------------------------------------------------------ the radii oracle (tests/averaged_radii_oracle.c) ----
def _rad_lib():
    """tests/averaged_radii_oracle.c (it includes tests/averaged_correction_oracle.c, tests/averaged_oracle.c and the pinned oracle
    unchanged) with its entry point bound."""
    from oracle import _Params, _Result
    return c_oracle.build("averaged_radii_oracle.c", {
        "so_reconstruct_averaged_radii": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_void_p, C.c_int, C.c_float,
                                                    C.c_float, C.POINTER(C.POINTER(_Result)), C.c_int64, C.c_void_p]),
        "so_free": (None, [C.POINTER(_Result)])})


def oracle_reconstruct_radii(particles, radii, *, particle_radius, smoothing_length, cube_size, rest_density=1000.0, iso_surface_threshold=0.6,
                             aabb_min=None, aabb_max=None, subdomain_grid=True, subdomain_num_cubes_per_dim=64, radius_factor=1.0,
                             corrected=False, t_low=T_LOW, t_high=T_HIGH, tile_of_subdomain=None, **_ignored):
    """C-oracle reconstruction with per-particle radii (plain or corrected): the dict of oracle_reconstruct_averaged, or {"rc": code}
    on a refusal."""
    from oracle import _Result, _grid_dict
    L = _rad_lib()
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    rr = np.ascontiguousarray(radii, dtype=np.float32)
    assert rr.shape == (len(xyz),)
    p = _aniso_params(particle_radius, smoothing_length, cube_size, rest_density, iso_surface_threshold, aabb_min, aabb_max,
                      subdomain_grid, subdomain_num_cubes_per_dim)
    S = int(subdomain_num_cubes_per_dim)
    tile = np.zeros((S + 1,) * 3, dtype=np.float32) if tile_of_subdomain is not None else None
    out = C.POINTER(_Result)()
    rc = L.so_reconstruct_averaged_radii(xyz.ctypes.data, len(xyz), C.byref(p), float(np.float32(radius_factor)), rr.ctypes.data if len(rr) else None,
                                         int(bool(corrected)), float(np.float32(t_low)), float(np.float32(t_high)), C.byref(out),
                                         -1 if tile_of_subdomain is None else int(tile_of_subdomain), None if tile is None else tile.ctypes.data)
    try:
        if rc != 0:
            return {"rc": rc}
        res = out.contents
        n, nv, nt, ns = res.n_filtered, res.nv, res.nt, res.n_subdomains
        d = {"rc": rc, "grid": _grid_dict(res.grid), "subdomain_grid": _grid_dict(res.subdomain_grid)}
        d["particle_densities"] = np.ctypeslib.as_array(res.densities, (n,)).copy() if n else np.zeros(0, np.float32)
        d["vertices"] = np.ctypeslib.as_array(res.vertices, (nv, 3)).copy() if nv else np.zeros((0, 3), np.float32)
        d["triangles"] = np.ctypeslib.as_array(res.triangles, (nt, 3)).copy() if nt else np.zeros((0, 3), np.uint64)
        d["vertex_keys"] = np.ctypeslib.as_array(res.vertex_keys, (nv, 4)).copy() if nv else np.zeros((0, 4), np.int64)
        d["subdomain_flat"] = np.ctypeslib.as_array(res.subdomain_flat, (ns,)).copy() if ns else np.zeros(0, np.int64)
        d["subdomain_count"] = np.ctypeslib.as_array(res.subdomain_count, (ns,)).copy() if ns else np.zeros(0, np.uint64)
        d["tile"] = tile
        return d
    finally:
        L.so_free(out)


def seeded_radii(n, seed, r, lo=0.6, hi=1.4):
    """Radii uniform in [lo, hi] r (float32)."""
    return (np.random.default_rng(seed).uniform(lo, hi, n) * r).astype(np.float32)


# ------------------------------------------------------------------ float64 restatement ----
def numpy_radii(p, radii, pts, h, rs, radius_factor=1.0, corrected=False, t_low=T_LOW, t_high=T_HIGH):
    """The value of DESIGN.md section 12.2 in float64 at the points `pts`, the candidate count and a bound on |f32 oracle - value|.

    b = sum w_j delta_j / S with delta_j the f32 deviations R_j - R_s (exact inputs of the f32 sum).  The bound extends the bound of
    numpy_averaged (plain) or numpy_corrected (corrected) by the error of b:
    * weight errors: with relative errors e_j of the weights (e3 of numpy_corrected: the base's 9 u q + u b, cubed, two roundings),
      b moves by sum w_j e_j |delta_j - b| / S', S' >= S - dS the perturbed sum (dS = sum w_j e_j + n u S; the rounding of S is a
      common relative error of the denominator, n u |b|); a candidate whose f32 membership can flip (|q - 1| < 20 u) adds
      (10 u)^3 |delta_j - b| / S';
    * the rounding of Q: each product one u, the n additions n u, on sum w_j |delta_j|, over S'; the division one u |b|;
    * plain: the addition (h - |m|) + b one u (h + |b|);
    * corrected: v = (plain + b) - (R_s + b)(1 - f): numpy_corrected's bound scaled by (R_s + |b|) / R_s covers the error of f times
      the larger radius, plus the error of b twice (through plain + b and R_s + b) and four more roundings on R_s + |b| + h.
    Where dS >= S the bound of b is |delta|_max + |b| (two averages of the deviations)."""
    from scipy.spatial import cKDTree
    u = EPS
    x = p.astype(np.float64)
    g = pts.astype(np.float64)
    dlt = (np.float32(radius_factor) * np.asarray(radii, np.float32) - np.float32(rs)).astype(np.float64)
    if corrected:
        _, _, fv, plain, n, bbase = numpy_corrected(p, pts, h, rs, t_low, t_high)
    else:
        plain, n, bbase = numpy_averaged(p, pts, h)
        fv = np.ones(len(pts))
    val, bound = np.zeros(len(g)), np.zeros(len(g))
    if not len(x):
        return val, n, bound
    tree = cKDTree(x)
    for k, nb in enumerate(tree.query_ball_point(g, h * (1 + 1e-6))):
        if not nb:
            continue
        d = x[nb] - g[k]
        qq = (d * d).sum(1) / (h * h)
        bb = np.where(qq < 1.0, 1.0 - qq, 0.0)
        w = bb ** 3
        S = w.sum()
        dj = dlt[nb]
        if not S > 0:
            bound[k] = bbase[k] + np.abs(dj).max()
            continue
        b = (w * dj).sum() / S
        val[k] = (plain[k] + b) - (rs + b) * (1.0 - fv[k]) if corrected else plain[k] + b
        nn = len(nb)
        rho = np.where(bb > 0, (9 * u * qq + u * bb) / np.where(bb > 0, bb, 1.0), 0.0)
        e3 = (1 + rho) ** 3 * (1 + u) ** 2 - 1
        dS = (w * e3).sum() + nn * u * S
        edge = np.where(np.abs(qq - 1.0) < 20 * u, (10.0 * u) ** 3, 0.0)
        if dS >= S:
            db = np.abs(dj).max() + abs(b)
        else:
            low = S - dS
            db = (((w * e3 + edge) * np.abs(dj - b)).sum() + (nn + 1) * u * (w * np.abs(dj)).sum()) / low + nn * u * abs(b) + u * abs(b)
        if corrected:
            bound[k] = bbase[k] * (rs + abs(b)) / rs + 1.25 * (2 * db + 4 * u * (rs + abs(b) + h))
        else:
            bound[k] = bbase[k] + 1.25 * (db + u * (h + abs(b)))
    return val, n, bound


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_oracle_matches_float64_restatement(name, corrected):
    """The oracle's tile of one subdomain against the value of §12.2 in float64 with radii uniform in [0.6, 1.4] r, point by point
    within numpy_radii's bound; prints the largest error as a fraction of its bound."""
    p = ORACLE_CLOUDS[name]()
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    r, h, c = _params_hrc(kw)
    radii = seeded_radii(len(p), 801, r)
    o = oracle_reconstruct_radii(p, radii, corrected=corrected, **kw)
    flat = _busiest_tile(o)
    o = oracle_reconstruct_radii(p, radii, corrected=corrected, tile_of_subdomain=flat, **kw)
    pts = _tile_points(o, flat, S)
    val, n, bound = numpy_radii(p, radii, pts, h, float(np.float32(r)), corrected=corrected)
    tile = o["tile"].reshape(-1).astype(np.float64)
    assert np.all(tile[n == 0] == 0.0)
    m = n > 0
    assert m.sum() > 100
    err = np.abs(tile[m] - val[m])
    frac = err / bound[m]
    assert np.all(err <= bound[m]), (err.max(), frac.max())
    print(f"{name} {'corrected' if corrected else 'plain'}: {m.sum()} points, median bound {np.median(bound[m]) / h:.2e} h, "
          f"max err/bound {frac.max():.3f}")
    assert np.median(bound[m]) < 1e-4 * h
    # the radii matter: the tile differs from the single radius's
    single = (oracle_reconstruct_corrected(p, tile_of_subdomain=flat, **kw) if corrected
              else oracle_reconstruct_averaged(p, tile_of_subdomain=flat, **kw))
    assert not np.array_equal(o["tile"], single["tile"])


# ------------------------------------------------------------------ equal radii reduce to the single radius ----
def _single(p, corrected, tile_of_subdomain=None, **kw):
    if corrected:
        return oracle_reconstruct_corrected(p, tile_of_subdomain=tile_of_subdomain, **kw)
    return oracle_reconstruct_averaged(p, tile_of_subdomain=tile_of_subdomain, **kw)


@pytest.mark.parametrize("radius_factor", [1.0, 0.8])
@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_equal_radii_reduce_to_single_radius_oracle(name, corrected, radius_factor):
    """Every r_j = particle_radius: delta_j = +0, Q = b = +0, and tiles and meshes bit-identical to AveragedSurface() (§12.2)."""
    p = ORACLE_CLOUDS[name]()
    kw = dict(KW, subdomain_num_cubes_per_dim=16, radius_factor=radius_factor)
    r, h, c = _params_hrc(kw)
    radii = np.full(len(p), np.float32(r), np.float32)
    flat = _busiest_tile(_single(p, corrected, **kw))
    a = _single(p, corrected, tile_of_subdomain=flat, **kw)
    b = oracle_reconstruct_radii(p, radii, corrected=corrected, tile_of_subdomain=flat, **kw)
    for k in ("vertices", "triangles", "vertex_keys", "particle_densities", "tile"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
def test_equal_radii_reduce_to_single_radius_emulated(emu, corrected):  # noqa: F811
    p = _cube(9, 811)
    for rf in (1.0, 0.8):
        kw = dict(KW, subdomain_num_cubes_per_dim=16)
        r, h, c = _params_hrc(kw)
        av = emu.AveragedSurface(rf, emu.JacobianCorrection() if corrected else None)
        a = emu.reconstruct_surface(p, averaged_surface=av, with_debug=True, **kw)
        flat = int(a.subdomains["flat"][int(np.argmax(a.subdomains["count"]))])
        a = emu.reconstruct_surface(p, averaged_surface=av, keep_levelset_tile_of=flat, **kw)
        b = emu.reconstruct_surface(p, averaged_surface=av, keep_levelset_tile_of=flat, particle_radii=np.full(len(p), r), **kw)
        assert np.array_equal(a.levelset_tile, b.levelset_tile)
        assert np.array_equal(a.mesh.vertices, b.mesh.vertices) and np.array_equal(a.mesh.triangles, b.mesh.triangles)


# ------------------------------------------------------------------ single particles ----
def test_one_particle_is_a_sphere_of_its_own_radius():
    """One particle of radius rho != particle_radius: b = delta to two roundings, so v = (h - |g - p|) + delta and the surface is the
    sphere of radius radius_factor * rho.  Every vertex lies within c^2 / R (+ rounding) inside it, radially (§12's bound with R for
    R_s, c <= R / sqrt(2))."""
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    r, h, c = _params_hrc(kw)
    for rho, rf in ((1.3 * r, 1.0), (0.8 * r, 1.25), (1.9 * r, 1.5)):
        R_ = float(np.float32(rf) * np.float32(rho))
        assert c <= R_ / np.sqrt(2.0)
        for corrected in (False, True):
            o = oracle_reconstruct_radii(p, [rho], radius_factor=rf, corrected=corrected, **kw)
            assert mesh_topology(o["triangles"]) == (1, True, [2])
            v = o["vertices"].astype(np.float64)
            rad = np.linalg.norm(v - p[0].astype(np.float64), axis=1)
            slack = 32 * float(np.spacing(np.float32(h))) + 8 * float(np.spacing(np.float32(np.abs(v).max())))
            assert np.all(rad <= R_ + slack) and np.all(rad >= R_ - c * c / R_ - slack), (rad.min(), rad.max(), R_)


def test_edge_of_support_particle_with_its_own_radius():
    """§12's particle with a grid point in the outermost f32 shell of its support (weight 2^-72), radius 1.3 r: w delta stays normal
    (the scale window of §12.2), the shell points stay outside, and the mesh is one closed sphere of radius 1.3 r."""
    p = _edge_shell_particle()
    kw = SHELL_KW
    r, h, c = _params_hrc(kw)
    rho = np.float32(1.3 * r)
    o = oracle_reconstruct_averaged(p[None], **kw)
    flat, hit, g = _shell_point(o, p)
    assert len(hit)
    for corrected in (False, True):
        o = oracle_reconstruct_radii(p[None], [rho], corrected=corrected, tile_of_subdomain=flat, **kw)
        assert mesh_topology(o["triangles"]) == (1, True, [2])
        tile = o["tile"].reshape(-1)
        val, n, bound = numpy_radii(p[None], [rho], g[hit], h, float(np.float32(r)), corrected=corrected)
        assert np.all(n == 1) and np.all(np.abs(tile[hit].astype(np.float64) - val) <= bound)
        assert np.all(tile[hit] < np.float32(h) - np.float32(r))               # outside
        rad = np.linalg.norm(o["vertices"].astype(np.float64) - p.astype(np.float64), axis=1)
        assert rad.max() <= float(rho) * (1 + 1e-4) and rad.min() >= float(rho) - c * c / float(rho)


def test_two_distant_particles_each_at_its_own_radius():
    """Radii 0.5 r and 1.5 r, farther apart than 2 (h + c): two closed components, each a sphere of its own radius."""
    kw = dict(KW, subdomain_num_cubes_per_dim=16, cube_size=0.25)
    r, h, c = _params_hrc(kw)
    p = np.array([[0.0, 0.0, 0.0], [2 * (h + c) * 1.05, 0.01, 0.0]], np.float32)
    radii = np.array([0.5 * r, 1.5 * r], np.float32)
    for corrected in (False, True):
        o = oracle_reconstruct_radii(p, radii, corrected=corrected, **kw)
        assert mesh_topology(o["triangles"]) == (2, True, [2, 2])
        v = o["vertices"].astype(np.float64)
        for k in range(2):
            rad = np.linalg.norm(v - p[k].astype(np.float64), axis=1)
            mine = rad < h
            R_ = float(radii[k])
            assert mine.sum() > 20
            assert np.all(rad[mine] <= R_ * (1 + 1e-4)) and np.all(rad[mine] >= R_ - c * c / R_), (k, rad[mine].min(), rad[mine].max())


# ------------------------------------------------------------------ surface quality (oracle) ----
def _bidisperse():
    """Two jittered balls 8 h apart: A at lattice spacing 2 r (radius 6 spacings), B at spacing 3 r (radius 4 spacings), jitter +-0.1
    spacing; per-particle radii r on A and 1.5 r on B.  Returns particles, radii, centres, lattice extents (largest particle
    distance from its centre) and the own radius of each ball."""
    a = _sphere(6, 821, jitter=0.1).astype(np.float64)
    b = _sphere(4, 822, jitter=0.1).astype(np.float64) * 1.5
    h = 4 * R
    cb = np.array([np.linalg.norm(a, axis=1).max() + np.linalg.norm(b, axis=1).max() + 8 * h, 0.0, 0.0])
    p = np.concatenate([a, b + cb]).astype(np.float32)
    radii = np.concatenate([np.full(len(a), R), np.full(len(b), 1.5 * R)]).astype(np.float32)
    ext = [np.linalg.norm(a, axis=1).max(), np.linalg.norm(b, axis=1).max()]
    return p, radii, [np.zeros(3), cb], ext, [R, 1.5 * R], len(a)


def _ball_errors(o, centres, ext, own):
    """Per ball: (mean vertex distance from its centre) - (lattice extent + own radius)."""
    v = o["vertices"].astype(np.float64)
    out = []
    for cen, e, rr in zip(centres, ext, own):
        d = np.linalg.norm(v - cen, axis=1)
        mine = d < e + 4 * R * 2
        out.append(float(d[mine].mean() - (e + rr)))
    return out


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
def test_quality_bidisperse_balls(corrected):
    """Each ball's mean vertex distance from its centre against its lattice extent plus its own radius (S = 32), with per-particle
    radii and with the single radius r.  Measured on the oracle (DESIGN.md §12.2), error in units of r:
      plain:      radii A -1.149, B -1.403;  single radius A -1.149, B -2.034
      corrected:  radii A -1.164, B -1.504;  single radius A -1.164, B -2.088
    The averaged surface sits inside the outermost particles on both balls (the average is pulled inwards at a free surface), more so
    on the coarser ball B.  Ball A (radius r) is the same either way (no particle of B within h of it); on ball B the radii move the
    surface out by 0.63 r (plain) and 0.58 r (corrected) of the 0.5 r by which its radius grew.  Thresholds: A equal within 1e-3 r;
    B improved by more than 0.45 r, within 1.6 r with the radii and beyond 1.9 r without; two closed spheres."""
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    p, radii, centres, ext, own, na = _bidisperse()
    o_r = oracle_reconstruct_radii(p, radii, corrected=corrected, **kw)
    o_s = _single(p, corrected, **kw)
    er, es = _ball_errors(o_r, centres, ext, own), _ball_errors(o_s, centres, ext, own)
    print(f"{'corrected' if corrected else 'plain'}: radii A {er[0] / R:+.3f} r, B {er[1] / R:+.3f} r; "
          f"single radius A {es[0] / R:+.3f} r, B {es[1] / R:+.3f} r")
    assert mesh_topology(o_r["triangles"]) == (2, True, [2, 2])
    assert abs(er[0] - es[0]) < 1e-3 * R
    assert abs(es[1]) - abs(er[1]) > 0.45 * R
    assert abs(er[1]) < 1.6 * R and abs(es[1]) > 1.9 * R


# ------------------------------------------------------------------ refusals ----
def _bad_radii(r, h, rf):
    """Each entry: radii that must be refused at index 3 (factor rf, compact support radius h)."""
    edge = np.float32(np.float32(h) / np.float32(rf))
    while np.float32(rf) * edge < np.float32(h):          # the smallest f32 with radius_factor * r >= h
        edge = np.nextafter(edge, np.float32(np.inf))
    return [np.nan, np.inf, -np.inf, 0.0, -r, edge, 2 * h / rf]


def test_oracle_refusals():
    p = _cube(5, 831)
    r, h, c = _params_hrc(KW)
    for rf in (1.0, 1.5):
        for bad in _bad_radii(r, h, rf):
            radii = np.full(len(p), r, np.float32)
            radii[3] = bad
            for corrected in (False, True):
                assert oracle_reconstruct_radii(p, radii, radius_factor=rf, corrected=corrected, **KW)["rc"] == 6, (rf, bad)
    ok = np.full(len(p), r, np.float32)
    assert oracle_reconstruct_radii(p, ok, subdomain_grid=False, **KW)["rc"] == 7
    # every input radius is checked, also those the particle-AABB filter drops
    radii = ok.copy()
    outside = np.nonzero(p[:, 0] >= 0.05)[0][0]
    radii[outside] = np.nan
    assert oracle_reconstruct_radii(p, radii, aabb_min=[-1.0, -1.0, -1.0], aabb_max=[0.05, 1.0, 1.0], **KW)["rc"] == 6


def test_emulated_refusals(emu):  # noqa: F811
    p = _cube(6, 832)
    r, h, c = _params_hrc(KW)
    ctx = emu.Context()
    L = ctx._L
    av = emu.AveragedSurface()
    try:
        params = emu.make_params(**KW)
        out = C.c_void_p()
        for rf in (1.0, 1.5):
            for bad in _bad_radii(r, h, rf):
                radii = np.full(len(p), r, np.float32)
                radii[3] = bad
                with pytest.raises(emu.SplashsurfError) as e:
                    emu.reconstruct_surface(p, context=ctx, averaged_surface=emu.AveragedSurface(rf), particle_radii=radii, **KW)
                assert e.value.code == 6 and "index 3" in str(e.value), (rf, bad, str(e.value))
        assert L.ss_context_set_averaged_radii_f32(None, None, 0) == 6
        ok = np.full(len(p), r, np.float32)
        # wrong length
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, C.byref(av._abi())))
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, ok.ctypes.data, len(p) - 1))
        assert L.ss_reconstruct_surface_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(out)) == 6 and not out
        # spatial_decomposition = None: the averaged surface's refusal
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, ok.ctypes.data, len(p)))
        p_none = emu.make_params(**KW, subdomain_grid=False)
        assert L.ss_reconstruct_surface_f32(ctx._h, p.ctypes.data, len(p), C.byref(p_none), C.byref(out)) == 7 and not out
        # partitioned entries: unsupported with the averaged surface on ...
        grid = emu._Grid()
        emu._check(L, L.ss_grid_for_reconstruction_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid)))
        rc = L.ss_reconstruct_partition_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid), 0, 0, 100, 1, 0, 0, C.byref(out))
        assert rc == 7 and not out
        # ... and radii without the averaged surface: invalid on both entries
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, None))
        assert L.ss_reconstruct_surface_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(out)) == 6 and not out
        rc = L.ss_reconstruct_partition_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid), 0, 0, 100, 1, 0, 0, C.byref(out))
        assert rc == 6 and not out
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, None, 0))
        # the Python front end
        with pytest.raises(ValueError, match="averaged_surface"):
            emu.reconstruct_surface(p, context=ctx, particle_radii=ok, **KW)
        with pytest.raises(ValueError, match="shape"):
            emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=ok[:-1], **KW)
        with pytest.raises(ValueError, match="shape"):
            emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=ok[:, None], **KW)
        with pytest.raises(TypeError):
            emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=np.ones(len(p), np.int32), **KW)
        with pytest.raises(ValueError, match="averaged_surface"):
            emu.reconstruction_pipeline(p, context=ctx, particle_radii=ok, **KW)
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=ok, subdomain_grid=False, **KW)
        assert e.value.code == 7
        # float64 radii are converted
        a = emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=ok.astype(np.float64) * 1.1, **KW)
        b = emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=(ok.astype(np.float64) * 1.1).astype(np.float32), **KW)
        assert np.array_equal(a.mesh.vertices, b.mesh.vertices)
        # a refused call leaves the context on the standard level set
        base = emu.reconstruct_surface(p, context=ctx, subdomain_grid_auto_disable=False, with_debug=True, **KW)
        assert base.mesh.nvertices > 0 and base.levelset_paths["avg_512"] == 0
    finally:
        ctx.close()


def test_runner_refuses_radii_on_several_gpus():
    from splashsurf_b200 import distributed as ssd
    import splashsurf_b200 as ss
    rn = ssd.Runner.__new__(ssd.Runner)
    rn.world, rn.particle_radii = 2, np.ones(4, np.float32)
    with pytest.raises(ValueError, match="multi-GPU"):
        rn.step(None)
    assert "particle_radii" in ss.reconstruct_surface.__code__.co_varnames
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "splashsurf_b200.h")).read()
    assert "int ss_context_set_averaged_radii_f32(ss_context *ctx, const float *radii /* NULL = off */, uint64_t n);" in hdr


# ------------------------------------------------------------------ context reuse ----
def test_emulated_context_reuse(emu):  # noqa: F811
    """Radii persist on the context until reset: set, reconstruct twice (both with radii), reset, reconstruct -- the last result equals
    a fresh context's plain averaged result."""
    p = _cube(8, 841)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    r, h, c = _params_hrc(kw)
    radii = seeded_radii(len(p), 842, r)
    av = emu.AveragedSurface()
    ctx = emu.Context()
    L = ctx._L
    try:
        with_r = emu.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=radii, **kw)
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, radii.ctypes.data, len(radii)))
        tmp = radii.copy()
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, tmp.ctypes.data, len(tmp)))
        tmp[:] = np.nan                                     # the context holds its own copy
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, C.byref(av._abi())))
        params = emu.make_params(**kw)
        for _ in range(2):
            s = ctx.reconstruct_raw(p.ctypes.data, len(p), params)
            v = np.empty((L.ss_surface_num_vertices(s), 3), np.float32)
            emu._check(L, L.ss_surface_copy_vertices(s, v.ctypes.data))
            L.ss_surface_free(s)
            assert np.array_equal(v, with_r.mesh.vertices)
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, None))
        emu._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, None, 0))
        again = emu.reconstruct_surface(p, context=ctx, averaged_surface=av, **kw)
    finally:
        ctx.close()
    fresh = emu.reconstruct_surface(p, averaged_surface=av, **kw)
    assert np.array_equal(again.mesh.vertices, fresh.mesh.vertices) and np.array_equal(again.mesh.triangles, fresh.mesh.triangles)
    assert not np.array_equal(with_r.mesh.vertices, fresh.mesh.vertices)


# ------------------------------------------------------------------ command line ----
def _write_vtk(path, p, point_data):
    """Legacy ASCII VTK particle file: one VERTEX cell per particle and the given POINT_DATA arrays (1-D: SCALARS, (n, 3): VECTORS)."""
    n = len(p)
    with open(path, "w") as f:
        f.write("# vtk DataFile Version 4.2\nparticles\nASCII\nDATASET UNSTRUCTURED_GRID\n")
        f.write(f"POINTS {n} float\n" + "\n".join(" ".join(repr(float(v)) for v in row) for row in p) + "\n")
        f.write(f"CELLS {n} {2 * n}\n" + "\n".join(f"1 {i}" for i in range(n)) + "\n")
        f.write(f"CELL_TYPES {n}\n" + "\n".join("1" for _ in range(n)) + "\n")
        f.write(f"POINT_DATA {n}\n")
        for name, a in point_data.items():
            if a.ndim == 1:
                f.write(f"SCALARS {name} float 1\nLOOKUP_TABLE default\n" + "\n".join(repr(float(v)) for v in a) + "\n")
            else:
                f.write(f"VECTORS {name} float\n" + "\n".join(" ".join(repr(float(v)) for v in row) for row in a) + "\n")


def test_emulated_cli(emu, tmp_path):  # noqa: F811
    """`reconstruct --averaged-surface=on --averaged-radius-attribute radius` reads the scalar point attribute of the frame and writes
    the mesh of reconstruct_surface(particle_radii=...), plain and corrected; refused without --averaged-surface=on, for a missing
    attribute and for one that is not a float scalar per particle."""
    from splashsurf_b200 import __main__ as cli
    p = _cube(8, 851)
    r = R
    radii = seeded_radii(len(p), 852, r)
    src = str(tmp_path / "cloud.vtk")
    _write_vtk(src, p, {"radius": radii, "vel": np.zeros((len(p), 3), np.float32)})
    args = ["reconstruct", src, "-r", str(r), "-l", "2.0", "-c", "0.5", "-q", "--averaged-surface=on", "--averaged-radius-attribute", "radius"]
    kw = dict(particle_radius=r, smoothing_length=2.0, cube_size=0.5, subdomain_grid_auto_disable=False)
    assert cli.main(args + ["-o", str(tmp_path / "a.npz")]) == 0
    got = np.load(tmp_path / "a.npz")
    want = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(), particle_radii=radii, **kw)
    assert np.array_equal(got["vertices"], want.mesh.vertices) and np.array_equal(got["triangles"], want.mesh.triangles)
    plain = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(), **kw)
    assert not np.array_equal(got["vertices"], plain.mesh.vertices)
    assert cli.main(args + ["--averaged-correction=on", "-o", str(tmp_path / "b.npz")]) == 0
    want = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(correction=emu.JacobianCorrection()), particle_radii=radii, **kw)
    assert np.array_equal(np.load(tmp_path / "b.npz")["vertices"], want.mesh.vertices)
    bad = [(args[:-3] + ["--averaged-radius-attribute", "radius"], "--averaged-surface=on"),
           (args[:-1] + ["nope"], "Missing attribute"),
           (args[:-1] + ["vel"], "not a float scalar per particle")]
    for a, msg in bad:
        with pytest.raises(ValueError, match=msg):
            cli.main(a + ["-o", str(tmp_path / "d.npz")])
        assert not os.path.exists(tmp_path / "d.npz")


# ------------------------------------------------------------------ device on the CPU executor ----
def case_radii(name, p, kw):
    """Seeded radii of a device case: uniform in [0.6, 1.4] r; for particle_aabb, [0.8, 1.2] r on the kept particles and 0.5 r on the
    ones the filter drops (an index mix-up in the compaction then reads radii of a different size)."""
    r, h, c = _params_hrc(kw)
    radii = seeded_radii(len(p), 860 + len(name), r)
    if name == "particle_aabb":
        inside = np.all(p >= np.asarray(kw["aabb_min"], np.float32), axis=1) & np.all(p < np.asarray(kw["aabb_max"], np.float32), axis=1)
        radii = np.where(inside, seeded_radii(len(p), 869, r, 0.8, 1.2), np.float32(0.5 * r)).astype(np.float32)
    return radii


def check_device_case(ss, oracle_mod, name, corrected, radii_on_device=False):
    """Device (or CPU executor) vs the radii oracle, bit for bit (mesh, densities, the kept tile); densities vs the standard run; two
    runs identical.  Returns the level-set path counters of the first run."""
    gen, kw, opts = CASES[name]
    p = gen()
    radii = case_radii(name, p, kw)
    rf = opts.get("radius_factor", 1.0)
    av = ss.AveragedSurface(rf, ss.JacobianCorrection() if corrected else None)
    o = oracle_reconstruct_radii(p, radii, radius_factor=rf, corrected=corrected, **kw)
    assert o["rc"] == 0
    flat = _busiest_tile(o)
    if flat is not None:
        o = oracle_reconstruct_radii(p, radii, radius_factor=rf, corrected=corrected, tile_of_subdomain=flat, **kw)
    ctx = ss.Context()
    try:
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        g = ss.reconstruct_surface(p, context=ctx, with_debug=True, averaged_surface=av, particle_radii=radii, keep_levelset_tile_of=flat, **kw)
        g2 = ss.reconstruct_surface(p, context=ctx, with_debug=True, averaged_surface=av, particle_radii=radii, **kw)
        std = ss.reconstruct_surface(p, context=ctx, subdomain_grid_auto_disable=False, **kw)
    finally:
        ctx.close()
    assert np.array_equal(g.particle_densities, o["particle_densities"])
    assert np.array_equal(g.particle_densities, std.particle_densities)
    assert np.array_equal(g.subdomains["flat"], o["subdomain_flat"]) and np.array_equal(g.subdomains["count"], o["subdomain_count"])
    if flat is not None:
        assert np.array_equal(g.levelset_tile, o["tile"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                               kw.get("subdomain_num_cubes_per_dim", 64))
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, m
    assert np.array_equal(g.mesh.vertices, g2.mesh.vertices) and np.array_equal(g.mesh.triangles, g2.mesh.triangles)
    if name == "particle_aabb":
        # the case guards the compaction: radii read by unfiltered index give a different mesh
        inside = np.all(p >= np.asarray(kw["aabb_min"], np.float32), axis=1) & np.all(p < np.asarray(kw["aabb_max"], np.float32), axis=1)
        mixed = radii.copy()
        mixed[inside] = radii[:inside.sum()]
        w = oracle_reconstruct_radii(p, mixed, radius_factor=rf, corrected=corrected, **kw)
        assert not np.array_equal(w["vertices"], o["vertices"]) or len(w["vertices"]) != len(o["vertices"])
    lp = g.levelset_paths
    assert all(lp[k] == 0 for k in ("aniso_512", "aniso_4096", "aniso_select", "exact_512", "cert_fused", "cert_warp_384", "cert_warp_576"))
    if opts.get("tier"):
        assert lp[opts["tier"]] > 0, lp
    if len(p) > 100:
        assert g.mesh.nvertices > 0 and lp["avg_512"] > 0
    return lp


_TIERS = {}


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_matches_oracle(emu, oracle_mod, name, corrected):  # noqa: F811
    lp = check_device_case(emu, oracle_mod, name, corrected)
    _TIERS[(name, corrected)] = {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")}
    if name == "clustered_overflow":
        assert _TIERS[(name, corrected)]["avg_select"] > 0


def test_emulated_every_tier_reached():
    """Runs after the cases above (same module, file order): each tier of the cascade was reached, plain and corrected."""
    if len(_TIERS) < 2 * len(CASES):
        pytest.skip("needs every device case of this module")
    for corrected in (False, True):
        for k in ("avg_512", "avg_4096", "avg_select"):
            assert any(t[k] > 0 for (n, cc), t in _TIERS.items() if cc == corrected), (k, corrected, _TIERS)
