"""What the level-set field's tests share (DESIGN.md sections 13, 13.1, 13.2 and 14): the modes, their keywords and records, the point
sets, the point-scan oracle (tests/levelset_field_oracle.c) and the brute-force SDF oracle (tests/levelset_sdf_oracle.c, one library
for both), the device-versus-oracle checks, and the float64 restatement of the field and its gradient.  Not a test module: the
device-versus-oracle cases live in tests/test_levelset_field.py and tests/test_zzz_gpu_levelset_field.py."""
import ctypes as C

import numpy as np

import c_oracle
from test_anisotropic import _aniso_lib, _aniso_params, _sphere, numpy_anisotropy
from test_averaged_surface import CASES, oracle_reconstruct_averaged

MODES = ["sph", "aniso", "avg", "corr", "rad", "corr_rad"]
MODE_ID = {m: i for i, m in enumerate(MODES)}            # the fold numbers of so_field_scan
GRAD_MODES = ["sph", "aniso", "avg", "rad"]               # the modes with a gradient, Hessian and curvature
SDF_MODES = ["sph", "sph_simd", "aniso", "avg", "corr", "rad"]
T_LOW, T_HIGH = 0.4, 3.5                                  # JacobianCorrection() defaults


def _kw_abs(kw):
    from oracle import absolute_params
    r, h, c = (np.float32(v) for v in absolute_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"]))
    return r, h, c


def _filtered(p, kw, extra=None):
    if "aabb_min" not in kw:
        return p, extra
    keep = np.all(p >= np.asarray(kw["aabb_min"], np.float32), axis=1) & np.all(p < np.asarray(kw["aabb_max"], np.float32), axis=1)
    return np.ascontiguousarray(p[keep]), (None if extra is None else np.ascontiguousarray(extra[keep]))


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


def _ball(jitter, seed):
    """A ball of radius 12 r.  With jitter 0.25 the anisotropic mesh has a few small interior voids, at whose vertices the
    area-weighted normals of the few triangles disagree with the level set's (8 of 11324 vertices); 0.1 keeps the ball one surface."""
    return _sphere(6, seed, jitter)


# ------------------------------------------------------------------ the oracles ----
def _ptr(a):
    return None if a is None or a.size == 0 else a.ctypes.data


def _field_lib():
    """tests/levelset_sdf_oracle.c, which includes tests/levelset_field_oracle.c: the point scan and the SDF grid."""
    vp = C.c_void_p
    return c_oracle.build("levelset_sdf_oracle.c", {
        "so_field_scan": (None, [C.c_int, vp, vp, vp, vp, C.c_uint64, C.c_float, C.c_float, C.c_float, C.c_float, vp, C.c_uint64,
                                 vp, vp, vp, vp]),
        "so_sdf_distance": (None, [vp, vp, C.c_uint64, vp, C.c_uint64, vp]),
        "so_sdf_grid": (C.c_int64, [C.c_int, vp, vp, vp, vp, C.c_uint64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                    vp, vp, C.c_uint64, vp, C.c_float, vp, C.c_uint32, vp, vp, vp])})


def records(p, kw, mode, radii=None):
    """The f32 records of a mode as the device folds read them: centres (n, 3), weights V_j (standard) or V_j det G_j
    (anisotropic), G (n, 6; anisotropic), delta_j (radii modes), and the densities.  The anisotropic ones come from the anisotropic
    oracle (tests/anisotropic_oracle.c), the densities of the others from the averaged oracle."""
    r, h, c = _kw_abs(kw)
    if mode == "aniso":
        xyz = np.ascontiguousarray(p, np.float32)
        prm = _aniso_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"], kw.get("rest_density", 1000.0), 0.6,
                            kw.get("aabb_min"), kw.get("aabb_max"), True, kw.get("subdomain_num_cubes_per_dim", 64))
        n = max(len(xyz), 1)
        xbar, g, vdet, rho = np.zeros((n, 3), np.float32), np.zeros((n, 6), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        nf = _aniso_lib().so_aniso_records(_ptr(xyz), len(xyz), C.byref(prm), 0.9, 4.0, 10, xbar.ctypes.data, g.ctypes.data,
                                           vdet.ctypes.data, rho.ctypes.data)
        assert nf >= 0
        return xbar[:nf], vdet[:nf], g[:nf], None, rho[:nf]
    rho = oracle_reconstruct_averaged(p, **kw)["particle_densities"]
    xyz, rr = _filtered(np.ascontiguousarray(p, np.float32), kw, radii)
    r2 = np.float32(r + r)
    vol = (np.float32(r2 * r2 * r2 * np.float32(kw.get("rest_density", 1000.0))) / rho).astype(np.float32)
    delta = np.ascontiguousarray(rr.astype(np.float32) - r, np.float32) if mode in ("rad", "corr_rad") else None
    return xyz, vol, None, delta, rho


def oracle_field(p, kw, mode, pts, radii=None):
    """(values, gradients (m, 3), Hessians (m, 6), curvatures (m, 2), densities) at `pts` by one so_field_scan; the corrected modes have
    no derivatives and leave them 0 (curvatures NaN)."""
    r, h, _ = _kw_abs(kw)
    ctr, w, g6, dlt, rho = records(p, kw, mode, radii)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    m = len(pts)
    val, grad, hess, curv = np.zeros(m, np.float32), np.zeros((m, 3), np.float32), np.zeros((m, 6), np.float32), np.full((m, 2), np.nan, np.float32)
    if m and len(ctr):
        arr = [np.ascontiguousarray(a) if a is not None else None for a in (ctr, w, g6, dlt)]
        _field_lib().so_field_scan(MODE_ID[mode], *[_ptr(a) for a in arr], len(ctr), h, r, T_LOW, T_HIGH, pts.ctypes.data, m, val.ctypes.data,
                                   grad.ctypes.data, hess.ctypes.data, curv.ctypes.data)
    return val, grad, hess, curv, rho


def oracle_distance(verts, tris, pts):
    """f32 unsigned distance of section 14 at `pts` by a scan over the given triangles."""
    verts, tris = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(tris, np.uint32)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    d = np.empty(len(pts), np.float32)
    if len(pts):
        _field_lib().so_sdf_distance(_ptr(verts), _ptr(tris), len(tris), _ptr(pts), len(pts), d.ctypes.data)
    return d


def oracle_sdf(p, kw, mode, verts, tris, band, grid, thr, radii=None):
    """(brick_coords, values, brick_inside) of section 14 by the oracle, with the field records of `records`."""
    r, h, c = _kw_abs(kw)
    fmode = "sph" if mode == "sph_simd" else mode
    ctr, w, g, delta, _ = records(p, kw, fmode, radii)
    npd = np.asarray(grid.npoints_per_dim, np.int64)
    nb = (npd + 7) // 8
    nbt = int(np.prod(nb))
    coords, values, inside = np.zeros((nbt, 3), np.int32), np.zeros((nbt, 8, 8, 8), np.float32), np.zeros(nb, np.uint8)
    verts, tris = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(tris, np.uint32)
    gmin = np.asarray(grid.aabb.min, np.float32)
    arr = [np.ascontiguousarray(a) if a is not None else None for a in (ctr, w, g, delta)]
    nl = _field_lib().so_sdf_grid(MODE_ID[fmode], *[_ptr(a) for a in arr], len(ctr), h, r, T_LOW, T_HIGH, np.float32(thr), _ptr(verts),
                                  _ptr(tris), len(tris), gmin.ctypes.data, np.float32(grid.cell_size), npd.ctypes.data, band, coords.ctypes.data,
                                  values.ctypes.data, inside.ctypes.data)
    return coords[:nl], values[:nl], inside.astype(bool)


# ------------------------------------------------------------------ device vs oracle ----
def _same(a, b):
    """Bit equality, with every NaN equal to every NaN (device and host NaN payloads differ)."""
    a, b = np.asarray(a), np.asarray(b)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.where(np.isnan(a), 0, a).view(np.uint32),
                                                                        np.where(np.isnan(b), 0, b).view(np.uint32))


def check_field_vs_oracle(ss, p, kw, mode, pts, expect_tier=None):
    """Every query the mode supports against the point-scan oracle at `pts`: evaluate(), and in the modes with derivatives
    gradient(), hessian() and curvature().  Values, gradients, Hessians and curvatures equal the oracle bit for bit (NaN equal to NaN);
    each query's values equal evaluate() and its gradients gradient() bit for bit; the curvature is NaN where the gradient is 0; the
    densities are the oracle's; shapes are right.  Returns the tier counters of each query ({query: paths})."""
    mk = mode_kwargs(ss, mode, p, kw)
    f = ss.LevelSetField(p, **kw, **mk)
    m = len(pts)
    try:
        ov, og, oh, oc, rho = oracle_field(p, kw, mode, pts, radii=mk.get("particle_radii"))
        assert np.array_equal(f.particle_densities, rho)
        v = f.evaluate(pts)
        tiers = {"evaluate": f.paths}
        assert v.shape == (m,)
        bad = np.flatnonzero(v.view(np.uint32) != ov.view(np.uint32))
        assert len(bad) == 0, (mode, len(bad), pts[bad[:3]], v[bad[:3]], ov[bad[:3]])
        if mode in GRAD_MODES:
            gv, g = f.gradient(pts)
            tiers["gradient"] = f.paths
            hv, hg, H = f.hessian(pts)
            tiers["hessian"] = f.paths
            kh, kg = f.curvature(pts)
            tiers["curvature"] = f.paths
            assert g.shape == (m, 3) and H.shape == (m, 6) and kh.shape == (m,) and kg.shape == (m,) and kh.dtype == np.float32
            for x in (gv, hv):
                assert np.array_equal(x.view(np.uint32), v.view(np.uint32)), mode
            assert np.array_equal(hg.view(np.uint32), g.view(np.uint32)), mode
            bad = np.flatnonzero(np.any(g.view(np.uint32) != og.view(np.uint32), axis=1))
            assert len(bad) == 0, (mode, len(bad), pts[bad[:3]], g[bad[:3]], og[bad[:3]])
            bad = np.flatnonzero(np.any(H.view(np.uint32) != oh.view(np.uint32), axis=1))
            assert len(bad) == 0, (mode, len(bad), pts[bad[:3]], H[bad[:3]], oh[bad[:3]])
            assert _same(kh, oc[:, 0]) and _same(kg, oc[:, 1]), mode
            assert np.all(np.isnan(kh[np.all(g == 0, axis=1)]))
        if expect_tier:
            for q, paths in tiers.items():
                assert paths[expect_tier] > 0, (q, paths)
        return tiers
    finally:
        f.close()


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


def assert_sdf_equal(got, coords, values, inside, what=""):
    assert np.array_equal(np.asarray(got.brick_coords), coords), (what, len(got.brick_coords), len(coords))
    bad = np.flatnonzero(np.asarray(got.values).view(np.uint32).ravel() != values.view(np.uint32).ravel())
    assert len(bad) == 0, (what, len(bad), np.asarray(got.values).ravel()[bad[:4]], values.ravel()[bad[:4]])
    assert np.array_equal(np.asarray(got.brick_inside), inside), what


def raw_case(ss, p, kw, mode, ctx=None):
    """(field, raw mesh, reconstruction keywords) of a mode: the standard mode reconstructs with simd off except in sph_simd."""
    mk = mode_kwargs(ss, "sph" if mode == "sph_simd" else mode, p, kw)
    rec = ss.reconstruct_surface(p, simd=(mode == "sph_simd"), subdomain_grid_auto_disable=False, context=ctx, **kw, **mk)
    f = ss.LevelSetField(p, **kw, **mk)
    return f, rec, mk


def check_sdf_vs_oracle(ss, p, kw, mode, band):
    f, rec, mk = raw_case(ss, p, kw, mode)
    try:
        got = f.signed_distance(rec.mesh, band=band)
        o = oracle_sdf(p, kw, mode, rec.mesh.vertices, rec.mesh.triangles, band, f.grid, f.threshold, radii=mk.get("particle_radii"))
        assert_sdf_equal(got, *o, what=(mode, band))
        assert got.background == np.float32(band) * np.float32(f.grid.cell_size)
        return f, rec, got
    except Exception:
        f.close()
        raise


def check_properties(ss, f, rec, got):
    """Sign bit = field.inside at listed points; adjacent listed unclamped values within a cell; every vertex's edge listed with opposite
    signs and |s| <= cell; to_dense() has the field's sign everywhere."""
    c = np.float32(f.grid.cell_size)
    B = np.float32(got.background)
    n = np.asarray(f.grid.npoints_per_dim)
    lo = np.asarray(f.grid.aabb.min, np.float32)
    dense = got.to_dense()
    assert dense.shape == tuple(n)
    idx = np.stack(np.meshgrid(*[np.arange(k) for k in n], indexing="ij"), -1).reshape(-1, 3)
    pts = (lo + idx.astype(np.float32) * c).astype(np.float32)
    inside = f.inside(pts).reshape(tuple(n))
    assert np.array_equal(np.signbit(dense), inside)                # -0.0: an inside point on the mesh
    listed = np.zeros(tuple((n + 7) // 8 * 8), bool)
    for b in np.asarray(got.brick_coords):
        listed[8 * b[0]:8 * b[0] + 8, 8 * b[1]:8 * b[1] + 8, 8 * b[2]:8 * b[2] + 8] = True
    listed = listed[:n[0], :n[1], :n[2]]
    unclamped = listed & (np.abs(dense) < B)
    # the distances are 1-Lipschitz; the f32 coordinates of points and vertices round relative to their magnitude, not to the cell
    tol = float(c) * (1 + 1e-5) + 8 * float(np.spacing(np.float32(np.abs(np.concatenate([pts[[0, -1]].ravel(), lo])).max())))
    for ax in range(3):
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[ax], b[ax] = slice(0, -1), slice(1, None)
        both = unclamped[tuple(a)] & unclamped[tuple(b)]
        diff = np.abs(dense[tuple(a)].astype(np.float64) - dense[tuple(b)])
        assert np.all(diff[both] <= tol), (ax, float(diff[both].max()), tol)
    if rec.mesh.nvertices:
        keys = np.asarray(rec.vertex_edge_keys, np.int64).reshape(-1, 4) if rec.vertex_edge_keys is not None else None
        if keys is not None:
            i0 = keys[:, :3]
            i1 = i0.copy()
            i1[np.arange(len(i1)), keys[:, 3]] += 1
            s0, s1 = dense[tuple(i0.T)], dense[tuple(i1.T)]
            assert np.all(listed[tuple(i0.T)] & listed[tuple(i1.T)])
            assert np.all(np.signbit(s0) != np.signbit(s1))
            assert np.all((np.abs(s0) <= tol) & (np.abs(s1) <= tol))


# ------------------------------------------------------------------ float64 restatement ----
U = 2.0 ** -24


def _w(r, h):
    q = 2.0 * r / h
    f = np.where(q < 1.0, 1.5 / np.pi * (2.0 / 3.0 - q * q + 0.5 * q ** 3), np.where(q < 2.0, 0.25 / np.pi * (2.0 - q) ** 3, 0.0))
    return 8.0 / h ** 3 * f


def _dw(r, h):
    """W'(r) and W''(r) of the cubic spline in float64."""
    q = 2.0 * r / h
    s = 8.0 / h ** 3 * 2.0 / h
    d1 = np.where(q < 1.0, 1.5 / np.pi * (1.5 * q * q - 2.0 * q), np.where(q < 2.0, -0.75 / np.pi * (2.0 - q) ** 2, 0.0))
    d2 = np.where(q < 1.0, 1.5 / np.pi * (3.0 * q - 2.0), np.where(q < 2.0, 1.5 / np.pi * (2.0 - q), 0.0))
    return s * d1, s * d2 * 2.0 / h


def f64_field(mode, ctr, w, g6, dlt, h, rs, pts, bound=False):
    """Value, analytic gradient and (bound=True) a per-point bound on |f32 fold gradient - gradient| in float64.  The bound
    propagates the rounding of every operation of the fold to first order (each f32 operation one relative u on its result, the
    inputs -- records, radii, points -- exact), the magnitudes taken in float64, and enlarges the sum by a quarter for the
    second-order terms:
    * standard / anisotropic: per term the offset (u |d|), u = G d (four roundings on |G| |d|), |u|^2, its root, q = 2 r / h, W'
      (its slope |W''| times the error of r plus eight roundings with the constants), the quotient by r and the products; n u on the
      sum of the terms' magnitudes;
    * averaged: the sums S, X, T, M (and Q, U) with the weight errors of numpy_corrected (the base's 9 u q + u b cubed or squared),
      their n additions, a candidate whose membership can flip (|q - 1| < 20 u) adding (10 u)^3 to S and (10 u)^2 h^k to the others;
      then m = X / S, M m, |m|^2 T, the difference, the product with 6 / h^2, the quotients by S and |m|.  Where every candidate sits
      near the edge of the support the weights carry u^3 and the second moments u^2, so the error of the quotient grows like 1/u:
      the bound follows it, it is not capped.  The one case claimed without a bound is S - dS <= 0 (the f32 sum of the weights may
      vanish); it is counted and reported."""
    from scipy.spatial import cKDTree
    x = ctr.astype(np.float64)
    g = pts.astype(np.float64)
    npt = len(g)
    val, grad, bnd = np.zeros(npt), np.zeros((npt, 3)), np.zeros(npt)
    nobound = 0
    if not len(x):
        return val, grad, bnd, nobound
    G = None
    if mode == "aniso":
        G = g6.astype(np.float64)[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
    tree = cKDTree(x)
    h2 = h * h
    k6 = 6.0 / h2
    for q, nb in enumerate(tree.query_ball_point(g, h * 1.006)):
        if not nb:
            continue
        nb = np.asarray(nb)
        d = x[nb] - g[q]
        n = len(nb)
        if mode in ("sph", "aniso"):
            V = w[nb].astype(np.float64)
            if mode == "aniso":
                Gj = G[nb]
                uv = np.einsum("jab,jb->ja", Gj, d)
                ga = np.abs(Gj)
                a = np.einsum("jab,jb->ja", ga, np.abs(d))
            else:
                uv, ga, a = d, None, np.abs(d)
            r = np.linalg.norm(uv, axis=1)
            inside = (r < h) & (r > 0)
            val[q] = (V * _w(r, h) * (r < h)).sum()
            W1, W2 = _dw(r, h)
            t = np.where(inside, V * W1 / np.where(r > 0, r, 1.0), 0.0)
            v = np.einsum("jab,jb->ja", Gj, uv) if mode == "aniso" else uv
            grad[q] = -(t[:, None] * v).sum(0)
            if bound:
                du = 4.0 * U * a if mode == "aniso" else U * a
                duu = 2.0 * (np.abs(uv) * du).sum(1) + 5.0 * U * r * r
                rr = np.where(r > 0, r, 1.0)
                dr = duu / (2.0 * rr) + U * r
                dW = np.abs(W2) * (dr + 2.0 * U * r) + 8.0 * U * np.abs(W1)
                dt = np.abs(V) * dW / rr + np.abs(t) * (dr / rr + 2.0 * U)
                if mode == "aniso":
                    dv = np.einsum("jab,jb->ja", ga, du) + 3.0 * U * np.einsum("jab,jb->ja", ga, np.abs(uv))
                else:
                    dv = du
                term = np.where(inside[:, None], dt[:, None] * np.abs(v) + np.abs(t)[:, None] * dv + U * np.abs(t[:, None] * v), 0.0)
                mag = np.abs(t[:, None] * v).sum(0)
                bnd[q] = 1.25 * float(np.linalg.norm(term.sum(0) + (n + 1) * U * mag))
            continue
        qq = (d * d).sum(1) / h2
        inside = qq < 1.0
        b = np.where(inside, 1.0 - qq, 0.0)
        wt, uu = b ** 3, b ** 2
        S = wt.sum()
        if not S > 0:
            continue
        X = (wt[:, None] * d).sum(0)
        T = (uu[:, None] * d).sum(0)
        M = (uu[:, None, None] * d[:, :, None] * d[:, None, :]).sum(0)
        m = X / S
        nm = np.linalg.norm(m)
        val[q] = h - nm
        gf = (m - k6 * (M @ m - nm * nm * T) / S) / nm if nm > 0 else np.zeros(3)
        if mode == "rad":
            dj = dlt[nb].astype(np.float64)
            bq = (wt * dj).sum() / S
            Uv = (uu[:, None] * dj[:, None] * d).sum(0)
            val[q] += bq
            gf = gf + k6 * (Uv - bq * T) / S
        grad[q] = gf
        if not bound:
            continue
        rho = np.where(b > 0, (9 * U * qq + U * b) / np.where(b > 0, b, 1.0), 0.0)
        e3 = (1 + rho) ** 3 * (1 + U) ** 2 - 1
        e2 = (1 + rho) ** 2 * (1 + U) - 1
        edge = np.abs(qq - 1.0) < 20 * U
        dS = (wt * e3).sum() + n * U * S + edge.sum() * (10 * U) ** 3
        low = S - dS
        if low <= 0:
            nobound += 1
            bnd[q] = np.inf
            continue
        ad = np.abs(d)
        eX = ((wt * (e3 + 2 * U))[:, None] * ad).sum(0) + n * U * (wt[:, None] * ad).sum(0) + edge.sum() * (10 * U) ** 3 * h
        eT = ((uu * (e2 + 2 * U))[:, None] * ad).sum(0) + n * U * (uu[:, None] * ad).sum(0) + edge.sum() * (10 * U) ** 2 * h
        aM = uu[:, None, None] * ad[:, :, None] * ad[:, None, :]
        eM = ((e2 + 4 * U)[:, None, None] * aM).sum(0) + n * U * aM.sum(0) + edge.sum() * (10 * U) ** 2 * h2
        dm = (eX + np.abs(m) * dS) / low + U * np.abs(m)
        dm2 = 2.0 * (np.abs(m) * dm).sum() + 5 * U * nm * nm
        Mm = M @ m
        dMm = np.abs(M) @ dm + eM @ np.abs(m) + 3 * U * (np.abs(M) @ np.abs(m))
        diff = Mm - nm * nm * T
        ddiff = dMm + dm2 * np.abs(T) + nm * nm * eT + U * nm * nm * np.abs(T) + U * np.abs(diff)
        jm = k6 * diff / S
        djm = k6 * ddiff / low + np.abs(jm) * (dS / low + 3 * U)
        if nm > 0:
            dnm = dm2 / (2 * nm) + U * nm
            num = m - jm
            dg = (dm + djm + U * np.abs(num)) / nm + np.abs(num) / nm * (dnm / nm + U)
        else:
            dg = np.zeros(3)
        if mode == "rad":
            adj = np.abs(dj)
            eQ = (wt * (e3 + 2 * U) * adj).sum() + n * U * (wt * adj).sum()
            db = (eQ + abs(bq) * dS) / low + U * abs(bq)
            eU = ((uu * (e2 + 3 * U) * adj)[:, None] * ad).sum(0) + n * U * ((uu * adj)[:, None] * ad).sum(0)
            res = Uv - bq * T
            dres = eU + db * np.abs(T) + abs(bq) * eT + U * abs(bq) * np.abs(T) + U * np.abs(res)
            add = k6 * res / S
            dg = dg + k6 * dres / low + np.abs(add) * (dS / low + 3 * U) + U * (np.abs(gf))
        bnd[q] = 1.25 * float(np.linalg.norm(dg))
    return val, grad, bnd, nobound


def f64_records(p, kw, mode, radii=None):
    """The float64 records of a mode: the f32 oracle's densities, and for the anisotropic mode numpy_anisotropy's x_bar, G and det G
    (the f32 records of the other modes are exact float64 inputs)."""
    ctr, w, g6, dlt, rho = records(p, kw, mode, radii)
    if mode != "aniso":
        return ctr, w, g6, dlt
    r, h, _ = _kw_abs(kw)
    xb, G, det, _, _ = numpy_anisotropy(p, float(h))
    vol = (2 * float(r)) ** 3 * kw.get("rest_density", 1000.0) / rho.astype(np.float64) * det
    return xb, vol, G.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]], None
