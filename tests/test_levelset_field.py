"""The level set at arbitrary points (LevelSetField / ss_levelset_field_*_f32, DESIGN.md section 13), on the CPU executor of the CUDA
sources (also run with SS_EMUL_GUARD=1):

* the point-scan oracle (tests/levelset_field_oracle.c) at points that are not grid points, against the float64 restatements of the
  averaged and corrected surfaces within their per-point bounds;
* the device equals the oracle bit for bit at random points, at points on tile, brick and bin faces and in the last cell of a brick
  for R = 1, 6, 7, 8, 9, 17, at 0.9 / 0.97 / 0.995 h from a lone particle in 26 directions, outside the grid and in empty
  subdomains (exactly 0), for m = 0 and n = 0, and in the clustered case that reaches the selection walk;
* the device equals the reconstruction's level-set tile bit for bit at the tile's own f32 grid coordinates (the standard level set
  with simd = False), and the densities are the reconstruction's;
* the two grid points of every mesh vertex's edge lie on opposite sides of the threshold;
* refusals, NaN points, a stale handle and one context reused across handles and reconstructions.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_field.py."""
import ctypes as C
import os

import numpy as np
import pytest

from test_anisotropic import KW, R, _aniso_params, _clustered, _cube
from test_averaged_correction import numpy_corrected
from test_averaged_surface import CASES, ORACLE_CLOUDS, numpy_averaged
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

MODES = ["sph", "aniso", "avg", "corr", "rad", "corr_rad"]
MODE_ID = {m: i for i, m in enumerate(MODES)}            # the fold numbers of so_field_scan
T_LOW, T_HIGH = 0.4, 3.5                                  # JacobianCorrection() defaults

# ------------------------------------------------------------------ the point-scan oracle ----
_LIBS = {}


def _field_lib(aniso: bool):
    """Compiles tests/levelset_field_oracle.c (with SO_FIELD_ANISO: on top of tests/anisotropic_oracle.c, otherwise on top of
    tests/averaged_radii_oracle.c) into a temporary directory with the oracle's compiler flags."""
    if aniso not in _LIBS:
        import subprocess
        import tempfile
        from oracle import _Params
        so = os.path.join(tempfile.mkdtemp(prefix="levelset_field_oracle_"), "liblevelset_field_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
                               "-mfma", "-mavx2", *(["-DSO_FIELD_ANISO"] if aniso else []), "-o", so,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "levelset_field_oracle.c"), "-lm", "-lpthread"])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.so_field_scan.restype = None
        L.so_field_scan.argtypes = [C.c_int, vp, vp, vp, vp, C.c_uint64, C.c_float, C.c_float, C.c_float, C.c_float, vp, C.c_uint64, vp]
        if aniso:
            L.so_field_aniso_records.restype = C.c_int64
            L.so_field_aniso_records.argtypes = [vp, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_float, C.c_uint32, vp, vp, vp, vp]
        _LIBS[aniso] = L
    return _LIBS[aniso]


def _kw_abs(kw):
    from oracle import absolute_params
    r, h, c = (np.float32(v) for v in absolute_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"]))
    return r, h, c


def _filtered(p, kw, extra=None):
    if "aabb_min" not in kw:
        return p, extra
    keep = np.all(p >= np.asarray(kw["aabb_min"], np.float32), axis=1) & np.all(p < np.asarray(kw["aabb_max"], np.float32), axis=1)
    return np.ascontiguousarray(p[keep]), (None if extra is None else np.ascontiguousarray(extra[keep]))


def oracle_field(p, kw, mode, pts, radii=None, radius_factor=1.0):
    """The field at `pts` by the point-scan oracle; the densities come from the oracles of tests/ (the anisotropic one for x_bar,
    G and V det G)."""
    from test_averaged_surface import oracle_reconstruct_averaged
    r, h, c = _kw_abs(kw)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    out = np.zeros(len(pts), np.float32)
    rs = np.float32(np.float32(radius_factor) * r)
    if mode == "aniso":
        L = _field_lib(True)
        xyz = np.ascontiguousarray(p, np.float32)
        prm = _aniso_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"], kw.get("rest_density", 1000.0), 0.6,
                            kw.get("aabb_min"), kw.get("aabb_max"), True, kw.get("subdomain_num_cubes_per_dim", 64))
        n = max(len(xyz), 1)
        xbar, g, vdet, rho = np.zeros((n, 3), np.float32), np.zeros((n, 6), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        nf = L.so_field_aniso_records(xyz.ctypes.data if len(xyz) else None, len(xyz), C.byref(prm), 0.9, 4.0, 10,
                                      xbar.ctypes.data, g.ctypes.data, vdet.ctypes.data, rho.ctypes.data)
        assert nf >= 0
        if len(pts):
            L.so_field_scan(1, xbar.ctypes.data, vdet.ctypes.data, g.ctypes.data, None, nf, h, rs, T_LOW, T_HIGH, pts.ctypes.data, len(pts), out.ctypes.data)
        return out, rho[:nf]
    L = _field_lib(False)
    o = oracle_reconstruct_averaged(p, **kw)
    rho = o["particle_densities"]
    xyz, rr = _filtered(np.ascontiguousarray(p, np.float32), kw, radii)
    r2 = np.float32(r + r)
    vol = (np.float32(r2 * r2 * r2 * np.float32(kw.get("rest_density", 1000.0))) / rho).astype(np.float32)
    delta = None
    if mode in ("rad", "corr_rad"):
        delta = np.ascontiguousarray((np.float32(radius_factor) * rr).astype(np.float32) - rs, np.float32)
    if len(pts) and len(xyz):
        L.so_field_scan(MODE_ID[mode], xyz.ctypes.data, vol.ctypes.data, None, None if delta is None else delta.ctypes.data, len(xyz), h, rs,
                        T_LOW, T_HIGH, pts.ctypes.data, len(pts), out.ctypes.data)
    return out, rho


def mode_kwargs(ss, mode, p, kw):
    """LevelSetField / reconstruct_surface keywords of a mode (the radii: seeded, uniform in [0.6, 1.4] r)."""
    if mode == "sph":
        return {}
    if mode == "aniso":
        return dict(anisotropy=ss.Anisotropy())
    corr = ss.JacobianCorrection() if mode in ("corr", "corr_rad") else None
    d = dict(averaged_surface=ss.AveragedSurface(1.0, corr))
    if mode in ("rad", "corr_rad"):
        r = float(_kw_abs(kw)[0])
        d["particle_radii"] = np.random.default_rng(880 + len(p)).uniform(0.6 * r, 1.4 * r, len(p)).astype(np.float32)
    return d


# ------------------------------------------------------------------ point sets ----
def random_points(grid, m, seed, pad=0.0):
    lo, hi = np.asarray(grid.aabb.min, np.float64), np.asarray(grid.aabb.max, np.float64)
    ext = hi - lo
    return np.random.default_rng(seed).uniform(lo - pad * ext, hi + pad * ext, (m, 3)).astype(np.float32)


def face_points(grid, S, seed):
    """Points on tile, brick and bin faces (cells 0 and 8 mod 8 of a tile, with both rounding neighbours) and in the last cell of a
    brick (7.5 and 7.999 cells into a brick), mixed with random coordinates on the other axes."""
    rng = np.random.default_rng(seed)
    c = np.float32(grid.cell_size)
    lo = np.asarray(grid.aabb.min, np.float32)
    nc = np.asarray(grid.ncells_per_dim)
    offs = []
    for base in range(0, int(nc.max()) + 1, 8):
        for f in (0.0, 7.5, 7.999, 8.0):
            offs.append(base + f)
    offs = np.asarray(offs, np.float64)
    pts = []
    for axis in range(3):
        for o in offs:
            q = rng.uniform(0, nc, (6, 3))
            q[:, axis] = o
            x = (lo + q.astype(np.float32) * c).astype(np.float32)
            pts += [x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))]
    return np.concatenate(pts).astype(np.float32)


def shell_points(center, h):
    """26 directions at 0.9, 0.97 and 0.995 h from a point."""
    d = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)], np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([np.asarray(center, np.float64) + f * float(h) * d for f in (0.9, 0.97, 0.995)]).astype(np.float32)


# ------------------------------------------------------------------ oracle vs float64 ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_oracle_within_float64_bounds_off_grid(cloud):
    """At random points that are not grid points the point-scan oracle lies within the float64 per-point bounds of DESIGN.md
    sections 12 (averaged) and 12.1 (corrected)."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, c = _kw_abs(KW)
    lo, hi = p.min(0) - float(h), p.max(0) + float(h)
    pts = np.random.default_rng(31).uniform(lo, hi, (3000, 3)).astype(np.float32)
    v, _ = oracle_field(p, KW, "avg", pts)
    f, n, bound = numpy_averaged(p, pts, float(h))
    m = n > 0
    assert np.all(v[~m] == 0.0) and m.sum() > 300
    assert np.all(np.abs(v[m] - f[m]) <= bound[m])
    v, _ = oracle_field(p, KW, "corr", pts)
    val, _ev, _fv, _plain, n, bound = numpy_corrected(p, pts, float(h), float(r))
    m = n > 0
    assert np.all(np.abs(v[m] - val[m]) <= bound[m])


# ------------------------------------------------------------------ device (CPU executor) ----
def _tile_coords(g, flat, S):
    """f32 coordinates of the grid points of subdomain `flat` of a reconstruction, min + index * cell as the tile kernel computes
    them (ss_grid_xy, and ss_grid_z of sparse subdomains)."""
    nsd = g.subdomain_grid.ncells_per_dim
    ijk = np.array([flat // (nsd[1] * nsd[2]), (flat // nsd[2]) % nsd[1], flat % nsd[2]])
    idx = np.stack(np.meshgrid(*[np.arange(S + 1)] * 3, indexing="ij"), -1).reshape(-1, 3) + ijk * S
    return (np.asarray(g.grid.aabb.min, np.float32) + idx.astype(np.float32) * np.float32(g.grid.cell_size)).astype(np.float32)


def check_field_vs_reconstruction(ss, name, mode):
    """Field at the busiest tile's grid points == the reconstruction's level-set tile, densities equal, and the two grid points of
    every vertex's edge on opposite sides of the threshold.  Returns (field values at the tile, reconstruction)."""
    gen, kw, opts = CASES[name]
    p = gen()
    kw = {k: v for k, v in kw.items()}
    S = kw.get("subdomain_num_cubes_per_dim", 64)
    mk = mode_kwargs(ss, mode, p, kw)
    ctx = ss.Context()
    try:
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        base = dict(kw, context=ctx, with_debug=True, simd=False, subdomain_grid_auto_disable=False, **mk)
        g = ss.reconstruct_surface(p, **base)
        flat = int(g.subdomains["flat"][np.argmax(g.subdomains["count"])]) if len(g.subdomains["flat"]) else None
        if flat is not None:
            g = ss.reconstruct_surface(p, keep_levelset_tile_of=flat, **base)
        f = ss.LevelSetField(p, context=ctx, **kw, **mk)
        assert np.array_equal(f.particle_densities, g.particle_densities)
        assert f.grid.aabb.min.tolist() == g.grid.aabb.min.tolist() and f.grid.ncells_per_dim == g.grid.ncells_per_dim
        if flat is not None:
            pts = _tile_coords(g, flat, S)
            v = f.evaluate(pts)
            assert np.array_equal(v.view(np.uint32), np.asarray(g.levelset_tile, np.float32).reshape(-1).view(np.uint32)), mode
        # mesh consistency: the end points of each vertex's edge straddle the threshold
        if g.mesh.nvertices:
            keys = np.asarray(g.vertex_edge_keys, np.int64).reshape(-1, 4)
            a = keys[:, :3].astype(np.float32)
            b = a.copy()
            b[np.arange(len(b)), keys[:, 3]] += 1
            lo, c = np.asarray(g.grid.aabb.min, np.float32), np.float32(g.grid.cell_size)
            va, vb = f.evaluate((lo + a * c).astype(np.float32)), f.evaluate((lo + b * c).astype(np.float32))
            assert np.all((va > f.threshold) != (vb > f.threshold)), mode
        f.close()
        return g
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64", "tile_batch_1", "particle_aabb"])
def test_emulated_field_equals_reconstruction(emu, name, mode):  # noqa: F811
    check_field_vs_reconstruction(emu, name, mode)


def check_field_vs_oracle(ss, p, kw, mode, pts, expect_tier=None):
    """Device field == point-scan oracle bit for bit at `pts`; densities == the oracle's.  Returns the tier counters."""
    mk = mode_kwargs(ss, mode, p, kw)
    f = ss.LevelSetField(p, **kw, **mk)
    try:
        v = f.evaluate(pts)
        o, rho = oracle_field(p, kw, mode, pts, radii=mk.get("particle_radii"))
        assert np.array_equal(f.particle_densities, rho)
        bad = np.flatnonzero(v.view(np.uint32) != o.view(np.uint32))
        assert len(bad) == 0, (mode, len(bad), pts[bad[:3]], v[bad[:3]], o[bad[:3]])
        if expect_tier:
            assert f.paths[expect_tier] > 0, f.paths
        return f.paths
    finally:
        f.close()


@pytest.mark.parametrize("mode", MODES)
def test_emulated_random_points_equal_oracle(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = emu.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 3000, 41), random_points(f.grid, 300, 42, pad=0.3)])
    f.close()
    paths = check_field_vs_oracle(emu, p, kw, mode, pts)
    assert paths["512"] > 0


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_emulated_faces_and_last_cells_equal_oracle(emu, Rc):  # noqa: F811
    """Points on tile, brick and bin faces and in the last cell of a brick at R = ceil(h / c) = Rc: the group's candidate bins
    must reach one cell past the brick's grid points."""
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = emu.LevelSetField(p, **kw)
    assert int(np.ceil(np.float32(4 * R) / np.float32(f.grid.cell_size))) == Rc
    pts = face_points(f.grid, 16, 77 + Rc)
    f.close()
    for mode in ("sph", "avg"):
        check_field_vs_oracle(emu, p, kw, mode, pts)


@pytest.mark.parametrize("mode", MODES)
def test_emulated_lone_particle_shells(emu, mode):  # noqa: F811
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    _, h, _ = _kw_abs(KW)
    pts = np.concatenate([shell_points(p[0], h), p])
    check_field_vs_oracle(emu, p, KW, mode, pts)


@pytest.mark.parametrize("mode", MODES)
def test_emulated_outside_and_empty_subdomains_are_zero(emu, mode):  # noqa: F811
    """Points outside the grid, far away, and in subdomains without members (the droplets' gaps) are exactly 0."""
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    mk = mode_kwargs(emu, mode, p, kw)
    f = emu.LevelSetField(p, **kw, **mk)
    try:
        far = np.array([[1e6, 0, 0], [-1e6, 5, 5], [0, 0, 3e38]], np.float32)
        outside = random_points(f.grid, 500, 51, pad=2.0)
        lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
        outside = outside[np.any((outside < lo) | (outside > hi), axis=1)]
        assert np.all(f.evaluate(far) == 0.0) and np.all(f.evaluate(outside) == 0.0)
        inside = random_points(f.grid, 4000, 52)
        v = f.evaluate(inside)
        o, _ = oracle_field(p, kw, mode, inside, radii=mk.get("particle_radii"))
        assert np.array_equal(v.view(np.uint32), o.view(np.uint32))
        assert (v == 0).sum() > 100
    finally:
        f.close()


@pytest.mark.parametrize("mode", ["sph", "avg", "corr"])
def test_emulated_clustered_reaches_select(emu, mode):  # noqa: F811
    """4400 particles in a ball of 0.6 h: the groups inside it exceed the 4096-slot slice and go to the selection walk."""
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(61).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    check_field_vs_oracle(emu, p, kw, mode, pts, expect_tier="select")


def test_emulated_empty_inputs(emu):  # noqa: F811
    f = emu.LevelSetField(np.zeros((0, 3), np.float32), **KW)
    try:
        assert f.evaluate(np.zeros((0, 3), np.float32)).shape == (0,)
        assert np.all(f.evaluate(np.array([[0, 0, 0], [1, 1, 1]], np.float32)) == 0.0)
        assert len(f.particle_densities) == 0
    finally:
        f.close()
    f = emu.LevelSetField(_cube(5, 3), **KW)
    try:
        assert f.evaluate(np.zeros((0, 3), np.float32)).shape == (0,) and f.paths == {"512": 0, "4096": 0, "select": 0}
    finally:
        f.close()


def test_emulated_refusals_and_reuse(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    with pytest.raises(TypeError):
        ss.LevelSetField(p.astype(np.float64), **KW)
    with pytest.raises(ss.SplashsurfError, match="error 1"):
        ss.LevelSetField(p, **dict(KW, cube_size=0.0))
    with pytest.raises(ss.SplashsurfError, match="radius_factor"):
        ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(100.0), **KW)
    with pytest.raises(ss.SplashsurfError, match="exclusive"):
        ss.LevelSetField(p, anisotropy=ss.Anisotropy(), averaged_surface=ss.AveragedSurface(), **KW)
    bad = np.full(len(p), np.float32(KW["particle_radius"]))
    bad[3] = np.nan
    with pytest.raises(ss.SplashsurfError, match="index 3"):
        ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(), particle_radii=bad, **KW)
    with pytest.raises(ValueError):
        ss.LevelSetField(p, particle_radii=bad, **KW)
    ctx = ss.Context()
    try:
        f1 = ss.LevelSetField(p, context=ctx, **KW)
        pts = random_points(f1.grid, 100, 71)
        v1 = f1.evaluate(pts)
        nan = pts.copy()
        nan[17, 1] = np.nan
        nan[40, 0] = np.inf
        with pytest.raises(ss.SplashsurfError, match="point 17"):
            f1.evaluate(nan)
        with pytest.raises(TypeError):
            f1.evaluate(pts.astype(np.float64))
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f1.evaluate(pts)
        f2 = ss.LevelSetField(p, context=ctx, averaged_surface=ss.AveragedSurface(), **KW)
        f3 = ss.LevelSetField(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f2.evaluate(pts)
        assert np.array_equal(f3.evaluate(pts), v1)
        for f in (f1, f2, f3):
            f.close()
        # the context's own settings are untouched: a reconstruction afterwards is the standard one
        g = ss.reconstruct_surface(p, context=ctx, **KW)
        assert np.array_equal(g.mesh.vertices, ss.reconstruct_surface(p, **KW).mesh.vertices)
    finally:
        ctx.close()
