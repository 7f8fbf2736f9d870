"""The gradient of the level set at arbitrary points (LevelSetField.gradient / .normals, ss_levelset_field_gradient_at_f32,
DESIGN.md section 13.1), on the CPU executor of the CUDA sources (also run with SS_EMUL_GUARD=1):

* the float64 analytic gradient of every supported mode is the derivative of the float64 field (central differences);
* the f32 point-scan oracle (tests/levelset_gradient_oracle.c) lies within a per-point float64 bound at every point, including the
  1/u amplification at the edge of the support of the averaged modes, and in the narrow band around the surface its normal lies
  within a small angle of the float64 normal;
* the device equals the oracle bit for bit, and its values equal evaluate() bit for bit, on the point sets of
  tests/test_levelset_field.py;
* properties (radial normals of one particle, the standard mode against SphInterpolator.interpolate_normals, equal radii), refusals,
  and reconstruction_pipeline(levelset_normals=True) / reconstruct --levelset-normals=on.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_gradient.py."""
import ctypes as C
import os

import numpy as np
import pytest

from test_anisotropic import KW, R, _aniso_params, _clustered, _cube, _sphere, numpy_anisotropy
from test_averaged_surface import CASES, ORACLE_CLOUDS
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)
from test_levelset_field import _filtered, _kw_abs, face_points, mode_kwargs, random_points, shell_points

MODES = ["sph", "aniso", "avg", "rad"]                    # the modes with a gradient
MODE_ID = {"sph": 0, "aniso": 1, "avg": 2, "rad": 4}      # the fold numbers of so_gradient_scan
U = 2.0 ** -24

# ------------------------------------------------------------------ the point-scan oracle ----
_LIBS = {}


def _grad_lib(aniso: bool):
    """Compiles tests/levelset_gradient_oracle.c (on top of tests/levelset_field_oracle.c, with or without SO_FIELD_ANISO) into a
    temporary directory with the oracle's compiler flags."""
    if aniso not in _LIBS:
        import subprocess
        import tempfile
        from oracle import _Params
        so = os.path.join(tempfile.mkdtemp(prefix="levelset_gradient_oracle_"), "liblevelset_gradient_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
                               "-mfma", "-mavx2", *(["-DSO_FIELD_ANISO"] if aniso else []), "-o", so,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "levelset_gradient_oracle.c"), "-lm", "-lpthread"])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.so_gradient_scan.restype = None
        L.so_gradient_scan.argtypes = [C.c_int, vp, vp, vp, vp, C.c_uint64, C.c_float, C.c_float, vp, C.c_uint64, vp, vp]
        if aniso:
            L.so_field_aniso_records.restype = C.c_int64
            L.so_field_aniso_records.argtypes = [vp, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_float, C.c_uint32, vp, vp, vp, vp]
        _LIBS[aniso] = L
    return _LIBS[aniso]


def records(p, kw, mode, radii=None):
    """The f32 records of a mode as the device folds read them: centres (n, 3), weights V_j (standard) or V_j det G_j
    (anisotropic), G (n, 6; anisotropic), delta_j (radii mode), and the densities."""
    from test_averaged_surface import oracle_reconstruct_averaged
    r, h, c = _kw_abs(kw)
    if mode == "aniso":
        L = _grad_lib(True)
        xyz = np.ascontiguousarray(p, np.float32)
        prm = _aniso_params(kw["particle_radius"], kw["smoothing_length"], kw["cube_size"], kw.get("rest_density", 1000.0), 0.6,
                            kw.get("aabb_min"), kw.get("aabb_max"), True, kw.get("subdomain_num_cubes_per_dim", 64))
        n = max(len(xyz), 1)
        xbar, g, vdet, rho = np.zeros((n, 3), np.float32), np.zeros((n, 6), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        nf = L.so_field_aniso_records(xyz.ctypes.data if len(xyz) else None, len(xyz), C.byref(prm), 0.9, 4.0, 10,
                                      xbar.ctypes.data, g.ctypes.data, vdet.ctypes.data, rho.ctypes.data)
        assert nf >= 0
        return xbar[:nf], vdet[:nf], g[:nf], None, rho[:nf]
    rho = oracle_reconstruct_averaged(p, **kw)["particle_densities"]
    xyz, rr = _filtered(np.ascontiguousarray(p, np.float32), kw, radii)
    r2 = np.float32(r + r)
    vol = (np.float32(r2 * r2 * r2 * np.float32(kw.get("rest_density", 1000.0))) / rho).astype(np.float32)
    delta = (rr.astype(np.float32) - r).astype(np.float32) if mode == "rad" else None
    return xyz, vol, None, delta, rho


def oracle_gradient(p, kw, mode, pts, radii=None):
    """(values, gradients, densities) at `pts` by the point-scan oracle."""
    r, h, _ = _kw_abs(kw)
    ctr, w, g6, dlt, rho = records(p, kw, mode, radii)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    val, grad = np.zeros(len(pts), np.float32), np.zeros((len(pts), 3), np.float32)
    if len(pts) and len(ctr):
        L = _grad_lib(mode == "aniso")
        arr = [np.ascontiguousarray(a) if a is not None else None for a in (ctr, w, g6, dlt)]
        L.so_gradient_scan(MODE_ID[mode], *[a.ctypes.data if a is not None else None for a in arr], len(ctr), h, r,
                           pts.ctypes.data, len(pts), val.ctypes.data, grad.ctypes.data)
    return val, grad, rho


# ------------------------------------------------------------------ float64 restatement ----
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


def _cloud_radii(p, kw):
    r = float(_kw_abs(kw)[0])
    return np.random.default_rng(880 + len(p)).uniform(0.6 * r, 1.4 * r, len(p)).astype(np.float32)


# ------------------------------------------------------------------ 1. the formula is the derivative ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_formula_is_the_derivative(cloud):
    """The float64 analytic gradient of every supported mode against central differences of the float64 field (step 1e-5 h) at
    random off-grid points; only points with |m| < 1e-3 h (the kink of the norm, averaged modes) are left out."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    h = float(h)
    lo, hi = p.min(0) - h, p.max(0) + h
    pts = np.random.default_rng(91).uniform(lo, hi, (400, 3))
    for mode in MODES:
        radii = _cloud_radii(p, KW) if mode == "rad" else None
        ctr, w, g6, dlt = f64_records(p, KW, mode, radii)
        v, g, _, _ = f64_field(mode, ctr, w, g6, dlt, h, float(r), pts)
        step = 1e-5 * h
        fd = np.zeros_like(g)
        for a in range(3):
            e = np.zeros(3)
            e[a] = step
            fd[:, a] = (f64_field(mode, ctr, w, g6, dlt, h, float(r), pts + e)[0] - f64_field(mode, ctr, w, g6, dlt, h, float(r), pts - e)[0]) / (2 * step)
        keep = v != 0
        if mode in ("avg", "rad"):                             # |m| = h - the plain averaged value
            va = f64_field("avg", ctr, w, g6, dlt, h, float(r), pts)[0]
            keep &= (va != 0) & (h - va > 1e-3 * h)
        scale = np.linalg.norm(g[keep], axis=1).max()
        err = np.abs(g[keep] - fd[keep]).max()
        assert keep.sum() > 50 and err <= 1e-6 * scale, (mode, err, scale)


# ------------------------------------------------------------------ 2. f32 oracle within float64 bounds ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_oracle_within_float64_bounds(cloud):
    """At every random point (none excluded) the f32 oracle's gradient lies within f64_field's per-point bound; prints the largest
    error / bound ratio of each mode."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    lo, hi = p.min(0) - float(h), p.max(0) + float(h)
    pts = np.random.default_rng(93).uniform(lo, hi, (1500, 3)).astype(np.float32)
    for mode in ("sph", "avg", "rad"):                       # the f32 records of these modes are the float64 inputs
        radii = _cloud_radii(p, KW) if mode == "rad" else None
        ctr, w, g6, dlt, _ = records(p, KW, mode, radii)
        _, og, _ = oracle_gradient(p, KW, mode, pts, radii)
        _, g, bnd, nobound = f64_field(mode, ctr, w, g6, dlt, float(h), float(r), pts, bound=True)
        assert nobound == 0, (mode, nobound)
        err = np.linalg.norm(og.astype(np.float64) - g, axis=1)
        reach = bnd > 0
        assert np.all(og[~reach] == 0.0)
        ratio = err[reach] / bnd[reach]
        print(cloud, mode, "largest error / bound", float(ratio.max()), "points", int(reach.sum()))
        assert np.all(err <= bnd), (mode, float(ratio.max()))
    # the anisotropic records: the f32 oracle's own x_bar, G and V det G as exact inputs of the float64 restatement
    ctr, w, g6, dlt, _ = records(p, KW, "aniso")
    _, og, _ = oracle_gradient(p, KW, "aniso", pts)
    _, g, bnd, _ = f64_field("aniso", ctr, w, g6, dlt, float(h), float(r), pts, bound=True)
    err = np.linalg.norm(og.astype(np.float64) - g, axis=1)
    reach = bnd > 0
    print(cloud, "aniso", "largest error / bound", float((err[reach] / bnd[reach]).max()))
    assert np.all(err <= bnd)


# ------------------------------------------------------------------ 3. narrow band ----
NARROW_BAND_DEG = 0.1            # largest angle measured on the oracle 0.029 degrees (DESIGN.md section 13.1)


@pytest.mark.parametrize("mode", MODES)
def test_narrow_band_normal_angle(emu, mode):  # noqa: F811
    """At the mesh vertices and at vertices moved by up to half a cell, the f32 oracle's normal lies within NARROW_BAND_DEG of the
    float64 normal; prints the largest angle."""
    p = ORACLE_CLOUDS["sphere"]()
    r, h, c = _kw_abs(KW)
    mk = mode_kwargs(emu, mode, p, KW)
    g = emu.reconstruct_surface(p, subdomain_grid_auto_disable=False, **KW, **mk)
    v = g.mesh.vertices
    rng = np.random.default_rng(95)
    pts = np.concatenate([v, v + rng.uniform(-0.5, 0.5, v.shape) * float(c)]).astype(np.float32)
    radii = mk.get("particle_radii")
    ctr, w, g6, dlt, _ = records(p, KW, mode, radii)
    _, og, _ = oracle_gradient(p, KW, mode, pts, radii)
    _, fg, _, _ = f64_field(mode, ctr, w, g6, dlt, float(h), float(r), pts)
    cos = (og.astype(np.float64) * fg).sum(1) / (np.linalg.norm(og, axis=1) * np.linalg.norm(fg, axis=1))
    ang = np.degrees(np.arccos(np.clip(cos, -1.0, 1.0)))
    print(mode, "largest narrow-band angle (deg)", float(ang.max()), len(pts))
    assert np.all(ang <= NARROW_BAND_DEG), float(ang.max())


# ------------------------------------------------------------------ 4. device == oracle, values == evaluate ----
def check_gradient_vs_oracle(ss, p, kw, mode, pts, expect_tier=None):
    """Device values and gradients == the point-scan oracle bit for bit, values == evaluate() bit for bit.  Returns the tier
    counters of the gradient query."""
    mk = mode_kwargs(ss, mode, p, kw)
    f = ss.LevelSetField(p, **kw, **mk)
    try:
        v, g = f.gradient(pts)
        paths = f.paths
        assert v.shape == (len(pts),) and g.shape == (len(pts), 3)
        assert np.array_equal(v.view(np.uint32), f.evaluate(pts).view(np.uint32)), mode
        ov, og, rho = oracle_gradient(p, kw, mode, pts, radii=mk.get("particle_radii"))
        assert np.array_equal(f.particle_densities, rho)
        assert np.array_equal(v.view(np.uint32), ov.view(np.uint32)), mode
        bad = np.flatnonzero(np.any(g.view(np.uint32) != og.view(np.uint32), axis=1))
        assert len(bad) == 0, (mode, len(bad), pts[bad[:3]], g[bad[:3]], og[bad[:3]])
        if expect_tier:
            assert paths[expect_tier] > 0, paths
        return paths
    finally:
        f.close()


@pytest.mark.parametrize("mode", MODES)
def test_emulated_random_points_equal_oracle(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = emu.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 2000, 41), random_points(f.grid, 200, 42, pad=0.3)])
    f.close()
    assert check_gradient_vs_oracle(emu, p, kw, mode, pts)["512"] > 0


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_emulated_faces_and_last_cells_equal_oracle(emu, Rc):  # noqa: F811
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = emu.LevelSetField(p, **kw)
    pts = face_points(f.grid, 16, 77 + Rc)
    f.close()
    for mode in ("sph", "avg"):
        check_gradient_vs_oracle(emu, p, kw, mode, pts)


@pytest.mark.parametrize("mode", MODES)
def test_emulated_lone_particle_shells(emu, mode):  # noqa: F811
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    _, h, _ = _kw_abs(KW)
    check_gradient_vs_oracle(emu, p, KW, mode, np.concatenate([shell_points(p[0], h), p]))


@pytest.mark.parametrize("mode", MODES)
def test_emulated_outside_and_empty_subdomains_are_zero(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    mk = mode_kwargs(emu, mode, p, kw)
    f = emu.LevelSetField(p, **kw, **mk)
    try:
        far = np.array([[1e6, 0, 0], [-1e6, 5, 5], [0, 0, 3e38]], np.float32)
        outside = random_points(f.grid, 500, 51, pad=2.0)
        lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
        outside = np.concatenate([far, outside[np.any((outside < lo) | (outside > hi), axis=1)]])
        v, g = f.gradient(outside)
        assert np.all(v == 0.0) and np.all(g == 0.0)
        inside = random_points(f.grid, 3000, 52)
        v, g = f.gradient(inside)
        assert ((v == 0) & np.all(g == 0, axis=1)).sum() > 100
    finally:
        f.close()
    check_gradient_vs_oracle(emu, p, kw, mode, inside)


@pytest.mark.parametrize("mode", ["sph", "avg"])
def test_emulated_clustered_reaches_select(emu, mode):  # noqa: F811
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(61).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    check_gradient_vs_oracle(emu, p, kw, mode, pts, expect_tier="select")


def test_emulated_empty_inputs(emu):  # noqa: F811
    f = emu.LevelSetField(np.zeros((0, 3), np.float32), **KW)
    try:
        v, g = f.gradient(np.zeros((0, 3), np.float32))
        assert v.shape == (0,) and g.shape == (0, 3)
        v, g = f.gradient(np.array([[0, 0, 0], [1, 1, 1]], np.float32))
        assert np.all(v == 0.0) and np.all(g == 0.0)
        assert np.all(np.isnan(f.normals(np.array([[0, 0, 0]], np.float32))))
    finally:
        f.close()


# ------------------------------------------------------------------ 5. properties ----
@pytest.mark.parametrize("mode", MODES)
def test_emulated_one_particle_normals_are_radial(emu, mode):  # noqa: F811
    """One particle: the outward normal at every vertex of its mesh points away from the particle (for the averaged modes within the
    1/u-free bound of a single candidate: offsets of about h / 2 carry a few u; the standard and anisotropic modes are radial by
    symmetry of each term)."""
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    mk = mode_kwargs(emu, mode, p, KW)
    g = emu.reconstruct_surface(p, subdomain_grid_auto_disable=False, **KW, **mk)
    f = emu.LevelSetField(p, **KW, **mk)
    try:
        v = g.mesh.vertices
        assert len(v) > 10
        n = f.normals(v)
        radial = (v - p[0]).astype(np.float64)
        radial /= np.linalg.norm(radial, axis=1, keepdims=True)
        # a single term: n = fl(d) / |fl(d)| up to the roundings of the fold; the averaged modes' M m - |m|^2 T cancels, and at the
        # surface (|d| = R_s = h / 4, b = 15 / 16) its rounding reaches the direction scaled by 6 |d|^2 / (h^2 b) < 1: tens of u
        assert np.abs(n - radial).max() <= 512 * U, np.abs(n - radial).max()
    finally:
        f.close()


def test_emulated_standard_normals_match_sph_interpolator(emu):  # noqa: F811
    """Standard mode: normals() equals SphInterpolator(...).interpolate_normals() up to summation order where the gradient is not
    negligible."""
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    r, h, _ = _kw_abs(kw)
    f = emu.LevelSetField(p, **kw)
    try:
        pts = random_points(f.grid, 3000, 97)
        _, g = f.gradient(pts)
        n = f.normals(pts)
        rest_mass = float(np.float32(np.float32(r + r) ** 3 * np.float32(kw.get("rest_density", 1000.0))))
        si = emu.SphInterpolator(p, f.particle_densities, rest_mass, float(h))
        ref = si.interpolate_normals(pts)
        si.close()
        gn = np.linalg.norm(g, axis=1)
        big = gn > 1e-3 * gn.max()
        assert big.sum() > 200
        assert np.abs(n[big] - ref[big]).max() <= 1e-4, np.abs(n[big] - ref[big]).max()
    finally:
        f.close()


def test_emulated_equal_radii_equal_plain_averaged(emu):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    rad = np.full(len(p), np.float32(_kw_abs(kw)[0]))
    a = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), **kw)
    b = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), particle_radii=rad, **kw)
    try:
        pts = random_points(a.grid, 2000, 98, pad=0.1)
        va, ga = a.gradient(pts)
        vb, gb = b.gradient(pts)
        assert np.array_equal(va.view(np.uint32), vb.view(np.uint32)) and np.array_equal(ga.view(np.uint32), gb.view(np.uint32))
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ 6. refusals ----
def test_emulated_refusals(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    for corr_rad in (False, True):
        mk = dict(averaged_surface=ss.AveragedSurface(1.0, ss.JacobianCorrection()))
        if corr_rad:
            mk["particle_radii"] = _cloud_radii(p, KW)
        f = ss.LevelSetField(p, **KW, **mk)
        try:
            pts = random_points(f.grid, 10, 3)
            with pytest.raises(ss.SplashsurfError, match="no gradient") as e:
                f.gradient(pts)
            assert e.value.code == 7                          # SS_ERR_UNSUPPORTED through the C entry
            with pytest.raises(ss.SplashsurfError, match="no gradient"):
                f.normals(pts)
            assert f.evaluate(pts).shape == (10,)              # the value query stays available
        finally:
            f.close()
    ctx = ss.Context()
    try:
        f = ss.LevelSetField(p, context=ctx, **KW)
        pts = random_points(f.grid, 50, 4)
        with pytest.raises(TypeError):
            f.gradient(pts.astype(np.float64))
        with pytest.raises(ValueError):
            f.gradient(pts[:, :2])
        nan = pts.copy()
        nan[7, 2] = np.nan
        with pytest.raises(ss.SplashsurfError, match="point 7"):
            f.gradient(nan)
        L = ctx._L
        out = np.empty(50, np.float32)
        assert L.ss_levelset_field_gradient_at_f32(f._s, pts.ctypes.data, 50, out.ctypes.data, None) == 6
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f.gradient(pts)
        f.close()
    finally:
        ctx.close()


def test_emulated_pipeline_and_cli_refusals(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli
    p = _cube(6, 5)
    with pytest.raises(ValueError, match="compute_normals"):
        emu.reconstruction_pipeline(p, levelset_normals=True, **KW)
    with pytest.raises(ValueError, match="exclusive"):
        emu.reconstruction_pipeline(p, compute_normals=True, sph_normals=True, levelset_normals=True, **KW)
    with pytest.raises(ValueError, match="Jacobian-corrected"):
        emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True,
                                    averaged_surface=emu.AveragedSurface(1.0, emu.JacobianCorrection()), **KW)
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "-o", str(tmp_path / "x.vtk")]
    for extra, msg in ((["--levelset-normals=on"], "--normals=on"),
                       (["--levelset-normals=on", "--normals=on", "--sph-normals=on"], "exclusive"),
                       (["--levelset-normals=on", "--normals=on", "--averaged-surface=on", "--averaged-correction=on"], "no gradient"),
                       (["--levelset-normals=on", "--normals=on", "--partition=on"], "--partition=on")):
        with pytest.raises(ValueError, match=msg):
            cli.main(args + extra)
        assert not os.path.exists(tmp_path / "x.vtk")


# ------------------------------------------------------------------ 7. pipeline and CLI ----
def _ball(jitter, seed):
    """A ball of radius 12 r.  With jitter 0.25 the anisotropic mesh has a few small interior voids, at whose vertices the
    area-weighted normals of the few triangles disagree with the level set's (8 of 11324 vertices); 0.1 keeps the ball one surface."""
    return _sphere(6, seed, jitter)


@pytest.mark.parametrize("mode", ["aniso", "avg"])
def test_emulated_pipeline_levelset_normals(emu, mode):  # noqa: F811
    """On a jittered ball: level-set normals are unit vectors whose dot product with the area-weighted normal is positive at every
    vertex, and normals_smoothing_iters is applied to them."""
    p = _ball(0.1, 111)
    mk = mode_kwargs(emu, mode, p, KW)
    mesh, rec = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, **KW, **mk)
    area, _ = emu.reconstruction_pipeline(p, compute_normals=True, **KW, **mk)
    n, a = mesh.point_attributes["normals"], area.point_attributes["normals"]
    assert len(n) > 100 and np.abs(np.linalg.norm(n, axis=1) - 1.0).max() < 1e-5
    assert np.all((n * a).sum(1) > 0)
    f = emu.LevelSetField(p, **KW, **mk)
    assert np.array_equal(n, f.normals(mesh.mesh.vertices))
    f.close()
    sm, _ = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, normals_smoothing_iters=3, output_raw_normals=True,
                                        **KW, **mk)
    assert np.array_equal(sm.point_attributes["raw_normals"], n)
    assert not np.array_equal(sm.point_attributes["normals"], n)
    assert np.all((sm.point_attributes["normals"] * a).sum(1) > 0)


def test_emulated_cli_levelset_normals(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    out = tmp_path / "n.vtk"
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "--averaged-surface=on"]
    assert cli.main(args + ["--normals=on", "--levelset-normals=on", "-o", str(out)]) == 0
    p = io.read_particles(src)
    mesh, _ = emu.reconstruction_pipeline(p, particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False,
                                          compute_normals=True, levelset_normals=True, averaged_surface=emu.AveragedSurface())
    _, _, _, point, _ = io.read_vtk_mesh(str(out))
    assert np.array_equal(np.asarray(point["normals"], np.float32), mesh.point_attributes["normals"])
