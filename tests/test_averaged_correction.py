"""Jacobian correction of the averaged-position surface (Solenthaler et al. 2007; splashsurf_b200.JacobianCorrection, DESIGN.md
section 12.1).

* the plain-C restatement (so_reconstruct_averaged_corrected in tests/averaged_correction_oracle.c) against an independent float64 numpy
  restatement, within a per-point rounding bound derived below;
* the correction reduces to the plain averaged surface: bit for bit where f == 1, and everywhere with thresholds above every EV;
* surface quality measured on the oracle against the plain averaged surface;
* refusals and the command line;
* the device pipeline on the CPU executor of the CUDA sources against the oracle, bit for bit.
The GPU-marked counterpart of the device cases is tests/test_zzz_gpu_averaged_correction.py."""
import ctypes as C
import os

import numpy as np
import pytest

import c_oracle
from test_anisotropic import KW, R, _aniso_params, _sphere
from test_averaged_surface import (CASES, ORACLE_CLOUDS, SHELL_KW, _busiest_tile, _edge_shell_particle, _shell_point,
                                   _tile_points, mesh_topology, numpy_averaged, oracle_reconstruct_averaged)
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

EPS = 2.0 ** -24               # unit roundoff of f32
T_LOW, T_HIGH = 0.4, 3.5       # the paper's thresholds (JacobianCorrection())


# ------------------------------------------------------------------ the corrected oracle (tests/averaged_correction_oracle.c) ----
def _corr_lib():
    """tests/averaged_correction_oracle.c (it includes tests/averaged_oracle.c and the pinned oracle unchanged) with its entry points
    bound."""
    from oracle import _Params, _Result
    return c_oracle.build("averaged_correction_oracle.c", {
        "so_reconstruct_averaged_corrected": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_float, C.c_float,
                                                        C.POINTER(C.POINTER(_Result)), C.c_int64, C.c_void_p]),
        "so_free": (None, [C.POINTER(_Result)])})


def oracle_reconstruct_corrected(particles, *, particle_radius, smoothing_length, cube_size, rest_density=1000.0, iso_surface_threshold=0.6,
                                 aabb_min=None, aabb_max=None, subdomain_grid=True, subdomain_num_cubes_per_dim=64, radius_factor=1.0,
                                 t_low=T_LOW, t_high=T_HIGH, tile_of_subdomain=None, **_ignored):
    """C-oracle reconstruction with the corrected averaged-position surface: the dict of oracle_reconstruct_averaged, or {"rc": code}
    on a refusal."""
    from oracle import _Result, _grid_dict
    L = _corr_lib()
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    p = _aniso_params(particle_radius, smoothing_length, cube_size, rest_density, iso_surface_threshold, aabb_min, aabb_max,
                      subdomain_grid, subdomain_num_cubes_per_dim)
    S = int(subdomain_num_cubes_per_dim)
    tile = np.zeros((S + 1,) * 3, dtype=np.float32) if tile_of_subdomain is not None else None
    out = C.POINTER(_Result)()
    rc = L.so_reconstruct_averaged_corrected(xyz.ctypes.data, len(xyz), C.byref(p), float(np.float32(radius_factor)), float(np.float32(t_low)),
                                             float(np.float32(t_high)), C.byref(out), -1 if tile_of_subdomain is None else int(tile_of_subdomain),
                                             None if tile is None else tile.ctypes.data)
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


def _params_hrc(kw):
    from oracle import absolute_params
    r, h, c = (float(v) for v in absolute_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"]))
    return r, h, c


# ------------------------------------------------------------------ float64 restatement ----
def _f_of_gamma(g):
    return 1.0 - (1.0 - g) ** 3


def numpy_corrected(p, pts, h, rs, t_low=T_LOW, t_high=T_HIGH):
    """The corrected value of DESIGN.md section 12.1 in float64 at the points `pts`, EV, f, the plain value, the candidate count and
    a bound on |f32 oracle - value| per point.

    The bound adds to numpy_averaged's bound on the plain value h - |m| the effect of the rounding on the correction R_s (1 - f):
    * every candidate's base b = 1 - q carries at most 9 u q + u b (numpy_averaged); relative to b that is rho, and the f32 weight
      w = b^3 and factor b^2 carry (1 + rho)^3 (1 + u)^2 - 1 and (1 + rho)^2 (1 + u) - 1, each product with d one u per factor;
    * a quotient N / S of sums of n terms a_j with relative errors e_j: |d(N / S)| <= (sum |a_j| (e_j + n u) + |N / S| dS) / (S - dS)
      + u |N / S|, dS = sum w_j e_j + n u S; this gives the errors of m = X / S, t = T / S and q = M / S;
    * J' = q - m t^T and its symmetric part A: first-order products plus one u per operation on the magnitudes; the Jacobi sweeps
      cost at most 200 u |A|_F; Weyl's inequality turns |dA|_F into the error of lambda_max, and 6 / h^2 scales it (two roundings);
    * gamma and f: the subtractions and the division in gamma move EV by at most 4 u (t_high + |EV| + t_low); f is monotone in gamma,
      so its error is the larger step of F(gamma) = 1 - (1 - gamma)^3 from the float64 gamma to the ends of the gamma interval that
      the EV error allows (near t_low and t_high the slope of F decides, no point is excluded), plus 16 u for its four roundings;
    * the value: R_s |df| plus 3 u (R_s + h).
    Where a candidate's f32 membership is ambiguous (|q - 1| < 20 u) or dS >= S, only |df| <= 1 is claimed.  The sum is enlarged by
    a quarter for the second-order terms, as in numpy_averaged."""
    from scipy.spatial import cKDTree
    u = EPS
    plain, n, bplain = numpy_averaged(p, pts, h)
    x = p.astype(np.float64)
    g = pts.astype(np.float64)
    npt = len(g)
    val, ev, fv, bound = np.zeros(npt), np.full(npt, np.nan), np.ones(npt), np.zeros(npt)
    if not len(x):
        return val, ev, fv, plain, n, bound
    tree = cKDTree(x)
    h2 = h * h
    for k, nb in enumerate(tree.query_ball_point(g, h * (1 + 1e-6))):
        if not nb:
            continue
        d = x[nb] - g[k]
        qq = (d * d).sum(1) / h2
        inside = qq < 1.0
        b = np.where(inside, 1.0 - qq, 0.0)
        w, uu = b ** 3, b ** 2
        S = w.sum()
        if not S > 0:
            bound[k] = bplain[k] + rs
            continue
        m = (w[:, None] * d).sum(0) / S
        t = (uu[:, None] * d).sum(0) / S
        q = (uu[:, None, None] * d[:, :, None] * d[:, None, :]).sum(0) / S
        J = q - np.outer(m, t)
        A = 0.5 * (J + J.T)
        e = 6.0 / h2 * np.linalg.eigvalsh(A)[-1]
        gam = min(max((t_high - e) / (t_high - t_low), 0.0), 1.0)
        f = _f_of_gamma(gam)
        ev[k], fv[k] = e, f
        val[k] = plain[k] - rs * (1.0 - f)
        # ---- the bound
        nn = len(nb)
        ambiguous = np.any(np.abs(qq - 1.0) < 20 * u)
        rho = np.where(b > 0, (9 * u * qq + u * b) / np.where(b > 0, b, 1.0), 0.0)
        e3 = (1 + rho) ** 3 * (1 + u) ** 2 - 1
        e2 = (1 + rho) ** 2 * (1 + u) - 1
        dS = (w * e3).sum() + nn * u * S
        if ambiguous or dS >= S:
            bound[k] = 1.25 * (bplain[k] + rs + 3 * u * (rs + h))
            continue
        low = S - dS

        def quot(a, ej, Q):
            return ((np.abs(a) * (ej[:, None] + nn * u)).sum(0) + np.abs(Q) * dS) / low + u * np.abs(Q)
        dm = quot(w[:, None] * d, e3 + 2 * u, m)
        dt = quot(uu[:, None] * d, e2 + 2 * u, t)
        aq = (uu[:, None, None] * d[:, :, None] * d[:, None, :]).reshape(nn, 9)
        dq = quot(aq, e2 + 4 * u, q.reshape(9)).reshape(3, 3)
        mt = np.abs(np.outer(m, t))
        dmt = np.outer(dm, np.abs(t)) + np.outer(np.abs(m), dt) + np.outer(dm, dt) + u * mt
        dJ = dq + dmt + u * (np.abs(q) + mt)
        dA = 0.5 * (dJ + dJ.T) + u * np.abs(A) + u * 0.5 * (np.abs(J) + np.abs(J.T))
        dl = np.linalg.norm(dA) + 200 * u * np.linalg.norm(A)
        de = 6.0 / h2 * dl + 2 * u * abs(e)
        de += 4 * u * (t_high + abs(e) + t_low)
        g_hi = min(max((t_high - (e - de)) / (t_high - t_low), 0.0), 1.0)
        g_lo = min(max((t_high - (e + de)) / (t_high - t_low), 0.0), 1.0)
        df = max(_f_of_gamma(g_hi) - f, f - _f_of_gamma(g_lo)) + 16 * u
        bound[k] = 1.25 * (bplain[k] + rs * min(df, 1.0) + 3 * u * (rs + h))
    return val, ev, fv, plain, n, bound


def _tile_of(o, p, kw, **corr):
    flat = _busiest_tile(o)
    return flat, oracle_reconstruct_corrected(p, tile_of_subdomain=flat, **kw, **corr)


@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_oracle_matches_float64_restatement(name):
    """The oracle's tile of one subdomain against the corrected value in float64, point by point within numpy_corrected's bound; the
    bound is tight at most points and the correction is active at some (f < 1)."""
    p = ORACLE_CLOUDS[name]()
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    r, h, c = _params_hrc(kw)
    flat, o = _tile_of(oracle_reconstruct_corrected(p, **kw), p, kw)
    pts = _tile_points(o, flat, S)
    val, ev, fv, plain, n, bound = numpy_corrected(p, pts, h, float(np.float32(r)))
    tile = o["tile"].reshape(-1).astype(np.float64)
    assert np.all(tile[n == 0] == 0.0)
    m = n > 0
    assert m.sum() > 100
    err = np.abs(tile[m] - val[m])
    assert np.all(err <= bound[m]), (err.max(), bound[m][np.argmax(err / bound[m])])
    print(f"{name}: {m.sum()} points, f < 1 at {(fv[m] < 1).sum()}, median bound {np.median(bound[m]) / h:.2e} h, "
          f"loose (bound > 1e-3 h) at {(bound[m] > 1e-3 * h).sum()}, max err/bound {(err / bound[m]).max():.3f}")
    assert np.median(bound[m]) < 1e-4 * h


def test_jacobian_is_identity_inside_a_regular_lattice():
    """The derivation of J in float64: deep inside an unbounded regular lattice x_bar moves with g, J -> I (here: a lattice of spacing
    h / 8, far from its boundary, J within 2 % of I), so EV is about 1."""
    h = 1.0
    a = np.arange(-24, 25) * (h / 8)
    p = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(1)
    for g in rng.uniform(-0.2, 0.2, (5, 3)):
        d = p - g
        b = np.clip(1 - (d * d).sum(1) / h ** 2, 0, None)
        w, uu = b ** 3, b ** 2
        S = w.sum()
        m, t = (w[:, None] * d).sum(0) / S, (uu[:, None] * d).sum(0) / S
        q = (uu[:, None, None] * d[:, :, None] * d[:, None, :]).sum(0) / S
        J = 6 / h ** 2 * (q - np.outer(m, t))
        assert np.abs(J - np.eye(3)).max() < 0.02, J


# ------------------------------------------------------------------ reduces to the plain mode ----
@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_reduces_to_plain_mode(name):
    """Thresholds above every EV (f == 1 everywhere): tiles and mesh bit-identical to AveragedSurface().  With the paper's
    thresholds: bit-identical at every point with f == 1 and never above the plain value."""
    p = ORACLE_CLOUDS[name]()
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    a0 = oracle_reconstruct_averaged(p, **kw)
    flat = _busiest_tile(a0)
    a = oracle_reconstruct_averaged(p, tile_of_subdomain=flat, **kw)
    off = oracle_reconstruct_corrected(p, t_low=1e30, t_high=2e30, tile_of_subdomain=flat, **kw)
    for k in ("vertices", "triangles", "vertex_keys", "particle_densities", "tile"):
        assert np.array_equal(off[k], a[k]), k
    on = oracle_reconstruct_corrected(p, tile_of_subdomain=flat, **kw)
    r, h, c = _params_hrc(kw)
    _, _, fv, _, n, _ = numpy_corrected(p, _tile_points(a, flat, S), h, float(np.float32(r)))
    t_on, t_a = on["tile"].reshape(-1), a["tile"].reshape(-1)
    assert np.all(t_on <= t_a)
    full = fv > 0.999999                                  # f == 1 in float64 well inside the f32 rounding of gamma
    lower = t_on < t_a
    assert np.array_equal(t_on[~lower], t_a[~lower])
    print(f"{name}: {lower.sum()} of {(n > 0).sum()} reached points lowered, {(lower & full).sum()} of them where float64 f == 1")


def _edge_points_lowered(p, kw, rs):
    """Per tile point of the busiest tile: (lowered by the correction, float64 f, reached)."""
    flat = _busiest_tile(oracle_reconstruct_averaged(p, **kw))
    a = oracle_reconstruct_averaged(p, tile_of_subdomain=flat, **kw)
    on = oracle_reconstruct_corrected(p, tile_of_subdomain=flat, **kw)
    r, h, c = _params_hrc(kw)
    _, ev, fv, _, n, _ = numpy_corrected(p, _tile_points(a, flat, kw["subdomain_num_cubes_per_dim"]), h, rs)
    return on["tile"].reshape(-1) < a["tile"].reshape(-1), fv, n > 0, on, a


def test_one_particle_is_the_plain_sphere():
    """One particle: J = 0 in exact arithmetic (EV = 0, f = 1 everywhere), so the mesh is the plain mode's sphere.  Rounding leaves an
    EV of order 1 only where the two terms of J cancel at the edge of the support; those points lie about h from the particle, far
    outside R_s, and the correction only lowers them: the mesh is bit-identical to the plain mode's."""
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    r, h, c = _params_hrc(kw)
    lowered, fv, reached, on, a = _edge_points_lowered(p, kw, float(np.float32(r)))
    assert np.all(fv[reached] == 1.0)
    assert np.array_equal(on["vertices"], a["vertices"]) and np.array_equal(on["triangles"], a["triangles"])
    pts = _tile_points(a, _busiest_tile(a), 16).astype(np.float64)
    dist = np.linalg.norm(pts - p[0].astype(np.float64), axis=1)
    if lowered.any():
        assert dist[lowered].min() > r + c
    print(f"one particle: {lowered.sum()} of {reached.sum()} reached points lowered by edge-of-support cancellation, "
          f"nearest {dist[lowered].min() / h if lowered.any() else float('nan'):.4f} h from the particle")


def test_edge_of_support_particle_stays_one_sphere():
    """§12's particle with a grid point in the outermost f32 shell of its support (u = 2^-24, u^2 = 2^-48): the cancellation in J is
    largest there.  Still one closed sphere, bit-identical to the plain mode's mesh, and every lowered point lies beyond R_s + c."""
    p = _edge_shell_particle()
    kw = SHELL_KW
    o = oracle_reconstruct_averaged(p[None], **kw)
    flat, hit, g = _shell_point(o, p)
    assert len(hit)
    a = oracle_reconstruct_averaged(p[None], tile_of_subdomain=flat, **kw)
    on = oracle_reconstruct_corrected(p[None], tile_of_subdomain=flat, **kw)
    r, h, c = _params_hrc(kw)
    assert (mesh_topology(on["triangles"])) == (1, True, [2])
    assert np.array_equal(on["vertices"], a["vertices"]) and np.array_equal(on["triangles"], a["triangles"])
    t_on, t_a = on["tile"].reshape(-1), a["tile"].reshape(-1)
    lowered = t_on < t_a
    assert np.all(t_on <= t_a)
    dist = np.linalg.norm(g.astype(np.float64) - p.astype(np.float64), axis=1)
    if lowered.any():
        assert dist[lowered].min() > r + c
    val, ev, fv, plain, n, bound = numpy_corrected(p[None], g[hit], h, float(np.float32(r)))
    assert np.all(np.abs(t_on[hit].astype(np.float64) - val) <= bound)
    print(f"edge-of-support particle: {lowered.sum()} lowered points (cancellation only: float64 f == 1 everywhere), "
          f"nearest {dist[lowered].min() / h if lowered.any() else float('nan'):.4f} h; shell points {t_on[hit]} vs plain {t_a[hit]}")


def test_isolated_particles_give_the_plain_spheres():
    """4096 isolated particles (§12's lattice): 4096 closed spheres, bit-identical to the plain mode's mesh."""
    rng = np.random.default_rng(709)
    g = np.stack(np.meshgrid(*[np.arange(16)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.12
    p = (g + rng.uniform(-0.005, 0.005, g.shape)).astype(np.float32)
    a = oracle_reconstruct_averaged(p, **SHELL_KW)
    on = oracle_reconstruct_corrected(p, **SHELL_KW)
    ncomp, closed, chi = mesh_topology(on["triangles"])
    assert ncomp == len(p) and closed and set(chi) == {2}
    assert np.array_equal(on["vertices"], a["vertices"]) and np.array_equal(on["triangles"], a["triangles"])


# ------------------------------------------------------------------ surface quality (oracle) ----
def _two_balls(gap_d):
    """Two jittered balls (radius 6 d, +-0.1 d) whose lattices are `gap_d` lattice spacings d = 2 r apart along x, and the x of the
    middle plane between them."""
    d = 2 * R
    b1 = _sphere(6, 801, jitter=0.1).astype(np.float64)
    b2 = _sphere(6, 802, jitter=0.1).astype(np.float64)
    off = (2 * 6 + 1 + gap_d) * d
    b2[:, 0] += off
    return np.concatenate([b1, b2]).astype(np.float32), off / 2


def test_quality_two_balls_do_not_bridge():
    """Two jittered balls 1.5 d apart (concave region between them).  Measured on the oracle (S = 32): the plain averaged surface puts
    46 vertices within d / 2 of the middle plane and has 3 components (a blob between the balls); the corrected one puts none there
    and gives exactly the two balls, closed, Euler characteristic 2 each."""
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    p, xm = _two_balls(1.5)
    a = oracle_reconstruct_averaged(p, **kw)
    c = oracle_reconstruct_corrected(p, **kw)
    band = lambda o: int((np.abs(o["vertices"][:, 0].astype(np.float64) - xm) < R).sum())   # noqa: E731
    assert band(a) >= 20, band(a)
    assert band(c) == 0
    assert mesh_topology(c["triangles"]) == (2, True, [2, 2])
    assert mesh_topology(a["triangles"])[0] > 2


def test_quality_sphere_radii_spread():
    """Particle sphere of radius 9 d jittered by +-0.1 d: the spread of the vertex radii stays within 5 % of the plain averaged
    surface's.  Measured on the oracle: 0.00620 corrected against 0.00612 plain (ratio 1.014)."""
    p = _sphere(9, 609, jitter=0.1)
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    a = oracle_reconstruct_averaged(p, **kw)
    c = oracle_reconstruct_corrected(p, **kw)
    sa = np.linalg.norm(a["vertices"].astype(np.float64), axis=1).std()
    sc = np.linalg.norm(c["vertices"].astype(np.float64), axis=1).std()
    assert sc < 1.05 * sa, (sc, sa)


@pytest.mark.parametrize("jitter", [0.1, 0.25])
def test_jittered_ball_is_one_closed_sphere(jitter):
    p = _sphere(9, 706, jitter=jitter)
    o = oracle_reconstruct_corrected(p, **dict(KW, subdomain_num_cubes_per_dim=32))
    assert mesh_topology(o["triangles"]) == (1, True, [2])


# ------------------------------------------------------------------ refusals and the command line ----
BAD_THRESHOLDS = [(-0.1, 3.5), (1.0, 1.0), (2.0, 1.0), (float("nan"), 3.5), (0.4, float("nan")), (0.4, float("inf")), (float("-inf"), 1.0)]


def test_oracle_refusals():
    from test_anisotropic import _cube
    p = _cube(5, 707)
    for lo, hi in BAD_THRESHOLDS:
        assert oracle_reconstruct_corrected(p, t_low=lo, t_high=hi, **KW)["rc"] == 6, (lo, hi)
    for rf in (0.0, 4.0, float("nan")):
        assert oracle_reconstruct_corrected(p, radius_factor=rf, **KW)["rc"] == 6, rf
    assert oracle_reconstruct_corrected(p, subdomain_grid=False, **KW)["rc"] == 7
    assert oracle_reconstruct_corrected(p, t_low=0.0, t_high=1e-30, **KW)["rc"] == 0


def test_emulated_refusals(emu):  # noqa: F811
    from test_anisotropic import _cube
    p = _cube(6, 708)
    ctx = emu.Context()
    L = ctx._L
    try:
        for lo, hi in BAD_THRESHOLDS:
            rc = L.ss_context_set_averaged_correction_f32(ctx._h, C.byref(emu.JacobianCorrection(lo, hi)._abi()))
            assert rc == 6, (lo, hi)
            with pytest.raises(emu.SplashsurfError) as e:
                emu.reconstruct_surface(p, context=ctx, averaged_surface=emu.AveragedSurface(correction=emu.JacobianCorrection(lo, hi)), **KW)
            assert e.value.code == 6
        assert L.ss_context_set_averaged_correction_f32(None, None) == 6
        # the correction without the averaged surface, on both reconstruction entries
        emu._check(L, L.ss_context_set_averaged_correction_f32(ctx._h, C.byref(emu.JacobianCorrection()._abi())))
        out = C.c_void_p()
        params = emu.make_params(**KW)
        rc = L.ss_reconstruct_surface_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(out))
        assert rc == 6 and not out
        grid = emu._Grid()
        emu._check(L, L.ss_grid_for_reconstruction_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid)))
        rc = L.ss_reconstruct_partition_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid), 0, 0, 100, 1, 0, 0, C.byref(out))
        assert rc == 6 and not out
        emu._check(L, L.ss_context_set_averaged_correction_f32(ctx._h, None))
        # with the averaged surface, the existing refusals hold
        corr = emu.AveragedSurface(correction=emu.JacobianCorrection())
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, averaged_surface=corr, subdomain_grid=False, **KW)
        assert e.value.code == 7
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, averaged_surface=corr, anisotropy=emu.Anisotropy(), **KW)
        assert e.value.code == 6
        # a refused call leaves the context on the standard level set
        base = emu.reconstruct_surface(p, context=ctx, subdomain_grid_auto_disable=False, with_debug=True, **KW)
        assert base.mesh.nvertices > 0 and base.levelset_paths["avg_512"] == 0
    finally:
        ctx.close()


def test_defaults_and_abi():
    import splashsurf_b200 as ss
    assert "JacobianCorrection" in ss.__all__
    assert ss.JacobianCorrection() == ss.JacobianCorrection(0.4, 3.5)
    assert ss.AveragedSurface(1.0) == ss.AveragedSurface(1.0, None) and ss.AveragedSurface(1.0).correction is None
    with pytest.raises(Exception):
        ss.JacobianCorrection().t_low = 1.0
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "splashsurf_b200.h")).read()
    assert "ss_context_set_averaged_correction_f32" in hdr and "float t_low, t_high;" in hdr


def test_emulated_cli(emu, tmp_path):  # noqa: F811
    """`reconstruct --averaged-surface=on --averaged-correction=on` writes the mesh of reconstruct_surface with
    AveragedSurface(correction=JacobianCorrection()); the thresholds reach the library; the switches are refused without
    --averaged-surface=on, and the thresholds without --averaged-correction=on."""
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "--averaged-surface=on"]
    p = io.read_particles(src)
    kw = dict(particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False)
    assert cli.main(args + ["--averaged-correction=on", "-o", str(tmp_path / "a.npz")]) == 0
    got = np.load(tmp_path / "a.npz")
    want = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(correction=emu.JacobianCorrection()), **kw)
    assert np.array_equal(got["vertices"], want.mesh.vertices) and np.array_equal(got["triangles"], want.mesh.triangles)
    plain = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(), **kw)
    assert not np.array_equal(got["vertices"], plain.mesh.vertices)
    assert cli.main(args + ["--averaged-correction=on", "--averaged-correction-low", "0.2", "--averaged-correction-high", "2.5",
                            "-o", str(tmp_path / "b.npz")]) == 0
    want = emu.reconstruct_surface(p, averaged_surface=emu.AveragedSurface(correction=emu.JacobianCorrection(0.2, 2.5)), **kw)
    assert np.array_equal(np.load(tmp_path / "b.npz")["vertices"], want.mesh.vertices)
    assert cli.main(args + ["--averaged-correction=off", "-o", str(tmp_path / "c.npz")]) == 0
    assert np.array_equal(np.load(tmp_path / "c.npz")["vertices"], plain.mesh.vertices)
    bad = [(["--averaged-correction=on"], "--averaged-surface=on", True),
           (["--averaged-correction-low", "0.2"], "--averaged-correction=on", False),
           (["--averaged-correction-high", "2.0"], "--averaged-correction=on", False),
           (["--averaged-correction=off", "--averaged-correction-low", "0.2"], "--averaged-correction=on", False)]
    for extra, msg, drop_avg in bad:
        a = (args[:-1] if drop_avg else args) + extra + ["-o", str(tmp_path / "d.npz")]
        with pytest.raises(ValueError, match=msg):
            cli.main(a)
        assert not os.path.exists(tmp_path / "d.npz")


# ------------------------------------------------------------------ device on the CPU executor ----
# §12's device cases with non-default thresholds (the paper's for the one-particle and edge cases, where J vanishes)
THRESHOLDS = {"cube_S16": (0.3, 2.5), "splash_S24": (0.5, 4.0), "cube_S64": (0.2, 3.0), "droplets_sparse": (0.6, 2.0),
              "tile_batch_1": (0.3, 2.5), "particle_aabb": (0.4, 1.8), "clustered_overflow": (0.25, 3.0), "radius_factor": (0.1, 5.0),
              "cfg1_fixture": (0.35, 2.2), "empty": (0.4, 3.5), "one_particle": (0.4, 3.5), "edge_of_support": (0.4, 3.5)}


def check_device_case(ss, oracle_mod, name):
    """Device (or CPU executor) vs the corrected oracle, bit for bit (mesh, densities, the kept tile); densities vs the standard
    run; two runs identical.  Returns the level-set path counters of the first run."""
    gen, kw, opts = CASES[name]
    p = gen()
    lo, hi = THRESHOLDS[name]
    av = ss.AveragedSurface(opts.get("radius_factor", 1.0), ss.JacobianCorrection(lo, hi))
    ok = dict(radius_factor=av.radius_factor, t_low=lo, t_high=hi)
    o = oracle_reconstruct_corrected(p, **ok, **kw)
    assert o["rc"] == 0
    flat = _busiest_tile(o)
    if flat is not None:
        o = oracle_reconstruct_corrected(p, tile_of_subdomain=flat, **ok, **kw)
    ctx = ss.Context()
    try:
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        g = ss.reconstruct_surface(p, context=ctx, with_debug=True, averaged_surface=av, keep_levelset_tile_of=flat, **kw)
        g2 = ss.reconstruct_surface(p, context=ctx, with_debug=True, averaged_surface=av, **kw)
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
    lp = g.levelset_paths
    assert all(lp[k] == 0 for k in ("aniso_512", "aniso_4096", "aniso_select", "exact_512", "cert_fused", "cert_warp_384", "cert_warp_576"))
    if opts.get("tier"):
        assert lp[opts["tier"]] > 0, lp
    if len(p) > 100:
        assert g.mesh.nvertices > 0 and lp["avg_512"] > 0
    return lp


_TIERS = {}


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_matches_oracle(emu, oracle_mod, name):  # noqa: F811
    lp = check_device_case(emu, oracle_mod, name)
    _TIERS[name] = {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")}
    if name == "clustered_overflow":
        assert _TIERS[name]["avg_select"] > 0


def test_emulated_every_tier_reached():
    """Runs after the cases above (same module, file order): each tier of the cascade was reached by some case."""
    if len(_TIERS) < len(CASES):
        pytest.skip("needs every device case of this module")
    for k in ("avg_512", "avg_4096", "avg_select"):
        assert any(t[k] > 0 for t in _TIERS.values()), (k, _TIERS)
