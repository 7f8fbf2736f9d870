"""The Hessian and curvature of the level set at arbitrary points (LevelSetField.hessian / .curvature,
ss_levelset_field_hessian_at_f32 / ss_levelset_field_curvature_at_f32, DESIGN.md section 13.2), on the CPU executor of the CUDA
sources (also run with SS_EMUL_GUARD=1):

* the float64 analytic Hessian of every supported mode is the derivative of the float64 analytic gradient of
  tests/levelset_field_harness.py (central differences);
* the f32 point-scan oracle (tests/levelset_field_oracle.c) lies within a per-point float64 bound at every point: a first-order
  propagation of every rounding of the fold, including the 1/b^2 growth at the edge of the support of the averaged modes;
* the device equals the oracle bit for bit (Hessian and curvature), and its values and gradients equal evaluate() and gradient()
  bit for bit: the device-versus-oracle cases of every query live in tests/test_levelset_field.py;
* properties (one particle: kappa_H = 1 / rho and kappa_G = 1 / rho^2; a jittered ball and a flat slab; equal radii), refusals, and
  reconstruction_pipeline(levelset_curvature=True) / reconstruct --levelset-curvature=on.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_curvature.py."""
import os

import numpy as np
import pytest

import splashsurf_b200
from levelset_field_harness import (GRAD_MODES as MODES, _ball, _kw_abs, _same, f64_field, f64_records, mode_kwargs, oracle_field,
                                    random_points, records)
from test_anisotropic import KW, _cube, _lattice
from test_averaged_surface import CASES, ORACLE_CLOUDS
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

U = 2.0 ** -24
HIJ = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]       # the six entries xx xy xz yy yz zz


# ------------------------------------------------------------------ float64 restatement with a rounding bound ----
class E:
    """A float64 value of the real-arithmetic fold and a first-order bound on the error of its f32 counterpart: every operation adds
    one relative rounding u of its result and propagates its operands' errors through its derivatives."""
    __slots__ = ("v", "e")
    __array_ufunc__ = None                                   # numpy arrays defer to E's operators

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()

    def __add__(a, b):
        b = _e(b)
        v = a.v + b.v
        return E(v, a.e + b.e + U * np.abs(v))

    def __sub__(a, b):
        b = _e(b)
        v = a.v - b.v
        return E(v, a.e + b.e + U * np.abs(v))

    def __rsub__(a, b):
        return _e(b) - a

    def __mul__(a, b):
        b = _e(b)
        v = a.v * b.v
        return E(v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + U * np.abs(v))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = _e(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = np.where(b.v != 0, a.v / np.where(b.v != 0, b.v, 1.0), 0.0)
            low = np.abs(b.v) - b.e
            e = np.where(low > 0, (a.e + np.abs(v) * b.e) / np.where(low > 0, low, 1.0), np.inf) + U * np.abs(v)
        return E(v, e)

    def __neg__(a):
        return E(-a.v, a.e)


def _e(x):
    return x if isinstance(x, E) else E(x)


def _sqrt(a):
    v = np.sqrt(a.v)
    lo = np.sqrt(np.maximum(a.v - a.e, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(v + lo > 0, a.e / np.where(v + lo > 0, v + lo, 1.0), np.sqrt(a.e))
    return E(v, e + U * v)


def _sel(cond, a, b):
    a, b = _e(a), _e(b)
    return E(np.where(cond, a.v, b.v), np.where(cond, a.e, b.e))


def _acc(t, mask, edge=None):
    """The f32 running sum of the terms t over the candidates (axis 1) where mask is set, in order: the terms' errors plus u times
    every partial sum; `edge` adds the magnitude of terms whose membership may flip."""
    tv = np.where(mask, t.v, 0.0)
    e = np.where(mask, t.e, 0.0).sum(1) + U * np.abs(np.cumsum(tv, axis=1)).sum(1)
    return E(tv.sum(1), e + (0.0 if edge is None else edge))


def _kernel_d2(r, h, inside):
    """W'/r and W'' of ss_kernel_scalar_d2 as E values; the f32 constants sigma, c_inner, c_outer carry 3 u."""
    sigma, cin, cout = E(8.0 / h ** 3, 3 * U * 8.0 / h ** 3), E(1.5 / np.pi, 3 * U * 1.5 / np.pi), E(0.25 / np.pi, 3 * U * 0.25 / np.pi)
    q = (r + r) / h
    t = E(2.0) / h
    s2 = t * t
    x = 2.0 - q
    f1q = _sel(q.v < 1.0, cin * (1.5 * q - 2.0), _sel(q.v < 2.0, ((-3.0 * cout) * x) * x / q, 0.0))
    f2 = _sel(q.v < 1.0, cin * (3.0 * q - 2.0), _sel(q.v < 2.0, (6.0 * cout) * x, 0.0))
    f1q, f2 = _sel(inside, f1q, 0.0), _sel(inside, f2, 0.0)
    return (sigma * f1q) * s2, (sigma * f2) * s2


def f64_hessian(mode, ctr, w, g6, dlt, h, pts):
    """Values, gradients (averaged modes: of the plain part, for curvature use f64_field's) and Hessians (m, 6) of the fold in real
    arithmetic, with per-entry first-order bounds on the f32 fold's error (E.e of each entry, enlarged by a quarter for the
    second-order terms by the caller).  Candidates are padded per point (axis 1).  Where every candidate sits near the edge of the
    support the averaged sums carry b^3 (S) against b (N, O) and the bound grows like 1/b^2: it is not capped."""
    with np.errstate(all="ignore"):
        return _f64_hessian(mode, ctr, w, g6, dlt, float(h), pts)


def _f64_hessian(mode, ctr, w, g6, dlt, h, pts):
    from scipy.spatial import cKDTree
    x = ctr.astype(np.float64)
    g = pts.astype(np.float64)
    m = len(g)
    H = [E(np.zeros(m)) for _ in range(6)]
    if not len(x) or not m:
        return H, np.zeros(m, bool)
    nbl = cKDTree(x).query_ball_point(g, h * 1.006)
    K = max(1, max(len(a) for a in nbl))
    idx = np.zeros((m, K), np.int64)
    has = np.zeros((m, K), bool)
    for i, a in enumerate(nbl):
        a = sorted(a)
        idx[i, :len(a)] = a
        has[i, :len(a)] = True
    d = [E(x[idx, a] - g[:, a, None]) for a in range(3)]
    for a in range(3):
        d[a].e = U * np.abs(d[a].v)
    if mode in ("sph", "aniso"):
        V = E(w.astype(np.float64)[idx])
        if mode == "aniso":
            G6 = g6.astype(np.float64)[idx]
            Gm = [[G6[..., k] for k in row] for row in ((0, 1, 2), (1, 3, 4), (2, 4, 5))]
            u = [(Gm[i][0] * d[0] + Gm[i][1] * d[1]) + Gm[i][2] * d[2] for i in range(3)]
            uu = (u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]
            inside = has & (uu.v < h * h)
            v = [(E(Gm[i][0]) * u[0] + E(Gm[i][1]) * u[1]) + E(Gm[i][2]) * u[2] for i in range(3)]
            Kq = [(E(Gm[i][0]) * Gm[0][j] + E(Gm[i][1]) * Gm[1][j]) + E(Gm[i][2]) * Gm[2][j] for i, j in HIJ]
        else:
            uu = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
            inside = has & (uu.v < h * h)                    # the f32 candidates reach 1.01 h^2; beyond h every term is 0
            v = d
            Kq = [E(np.full(uu.v.shape, 1.0 if i == j else 0.0)) for i, j in HIJ]
        w1r, w2 = _kernel_d2(_sqrt(uu), h, inside)
        ra = V * (w2 - w1r) / uu
        b = V * w1r
        for q, (i, j) in enumerate(HIJ):
            H[q] = _acc((ra * v[i]) * v[j] + b * Kq[q], inside)
        return H, inside.any(1)
    h2 = E(h) * h
    d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    qq = d2.v / (h * h)
    inside = has & (qq < 1.0)
    ne = (has & (np.abs(qq - 1.0) < 20 * U)).sum(1).astype(np.float64)       # candidates whose membership may flip
    eb = 20 * U
    u = 1.0 - d2 / h2
    uu = u * u
    wt = uu * u
    S = _acc(wt, inside, ne * eb ** 3)
    X = [_acc(wt * d[a], inside, ne * eb ** 3 * h) for a in range(3)]
    ex = [uu * d[a] for a in range(3)]
    T = [_acc(ex[a], inside, ne * eb ** 2 * h) for a in range(3)]
    M = {(i, j): _acc(ex[i] * d[j], inside, ne * eb ** 2 * h * h) for i, j in HIJ}
    S2 = _acc(u * u, inside, ne * eb ** 2)
    ed = [u * d[a] for a in range(3)]
    nn = {(i, j): ed[i] * d[j] for i, j in HIJ}
    N = {k: _acc(t, inside, ne * eb * h * h) for k, t in nn.items()}
    O = {}
    for (i, j) in HIJ:
        for c in range(j, 3):
            O[(i, j, c)] = _acc(nn[(i, j)] * d[c], inside, ne * eb * h ** 3)
    k6, kh = E(6.0) / h2, E(4.0) / h2
    ok = S.v > 0
    s = _sel(ok, S, 1.0)
    mv = [X[a] / s for a in range(3)]
    m2 = (mv[0] * mv[0] + mv[1] * mv[1]) + mv[2] * mv[2]
    nm = _sqrt(m2)
    okm = ok & (nm.v > 0)
    nms = _sel(okm, nm, 1.0)
    Mf = lambda i, j: M[(min(i, j), max(i, j))]  # noqa: E731
    grad = []
    for i in range(3):
        mm = (Mf(i, 0) * mv[0] + Mf(i, 1) * mv[1]) + Mf(i, 2) * mv[2]
        jm = (k6 * (mm - m2 * T[i])) / s
        grad.append((mv[i] - jm) / nms)
    mh = [mv[a] / nms for a in range(3)]
    J = [[(k6 * (Mf(i, j) - mv[i] * T[j])) / s for j in range(3)] for i in range(3)]
    B = [[(1.0 if i == j else 0.0) - J[i][j] for j in range(3)] for i in range(3)]
    cv = [(J[0][j] * mh[0] + J[1][j] * mh[1]) + J[2][j] * mh[2] for j in range(3)]
    sig = nm * S2 - ((mh[0] * T[0] + mh[1] * T[1]) + mh[2] * T[2])
    Of = lambda a, i, j: O[tuple(sorted((a, i, j)))]  # noqa: E731
    for q, (i, j) in enumerate(HIJ):
        om = (Of(0, i, j) * mh[0] + Of(1, i, j) * mh[1]) + Of(2, i, j) * mh[2]
        p = kh * (om - nm * N[(i, j)])
        if i == j:
            p = p + sig
        p = (p - T[i] * cv[j]) - cv[i] * T[j]
        first = (k6 * p) / s
        bb = (B[0][i] * B[0][j] + B[1][i] * B[1][j]) + B[2][i] * B[2][j]
        second = (bb - grad[i] * grad[j]) / nms
        H[q] = _sel(okm, -(first + second), 0.0)
    if mode == "rad":
        dl = E(dlt.astype(np.float64)[idx])
        ebd = float(np.abs(dlt).max()) if len(dlt) else 0.0
        Q = _acc(wt * dl, inside, ne * eb ** 3 * ebd)
        Uv = [_acc((uu * dl) * d[a], inside, ne * eb ** 2 * h * ebd) for a in range(3)]
        ud = u * dl
        S2d = _acc(u * ud, inside, ne * eb ** 2 * ebd)
        Nd = {(i, j): _acc((ud * d[i]) * d[j], inside, ne * eb * h * h * ebd) for i, j in HIJ}
        Rq = Q / s
        rg = [(k6 * (Uv[i] - Rq * T[i])) / s for i in range(3)]
        dg = Rq * S2 - S2d
        for q, (i, j) in enumerate(HIJ):
            p = kh * (Nd[(i, j)] - Rq * N[(i, j)])
            if i == j:
                p = p + dg
            p = (p - T[i] * rg[j]) - rg[i] * T[j]
            H[q] = _sel(ok, H[q] + (k6 * p) / s, 0.0)
    return H, ok


def _hess_matrix(H):
    """(m, 3, 3) from the six entries of a list of E or an (m, 6) array."""
    a = np.stack([x.v if isinstance(x, E) else x for x in H], 1) if isinstance(H, list) else H
    return a[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)


# ------------------------------------------------------------------ 1. the formula is the derivative ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_formula_is_the_derivative(cloud):
    """The float64 analytic Hessian of every supported mode against central differences (step 1e-5 h) of the float64 analytic
    gradient of levelset_field_harness.f64_field, at random off-grid points, relative to the largest Hessian norm; only the kink
    points of section 13.1 (|m| < 1e-3 h, averaged modes) are left out."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    h = float(h)
    lo, hi = p.min(0) - h, p.max(0) + h
    pts = np.random.default_rng(191).uniform(lo, hi, (400, 3))
    for mode in MODES:
        radii = mode_kwargs(splashsurf_b200, mode, p, KW).get("particle_radii")
        ctr, w, g6, dlt = f64_records(p, KW, mode, radii)
        v = f64_field(mode, ctr, w, g6, dlt, h, float(r), pts)[0]
        Hm = _hess_matrix(f64_hessian(mode, ctr, w, g6, dlt, h, pts)[0])
        step = 1e-5 * h
        fd = np.zeros_like(Hm)
        for a in range(3):
            e = np.zeros(3)
            e[a] = step
            fd[:, :, a] = (f64_field(mode, ctr, w, g6, dlt, h, float(r), pts + e)[1] - f64_field(mode, ctr, w, g6, dlt, h, float(r), pts - e)[1]) / (2 * step)
        keep = v != 0
        if mode in ("avg", "rad"):
            va = f64_field("avg", ctr, w, g6, dlt, h, float(r), pts)[0]
            keep &= (va != 0) & (h - va > 1e-3 * h)
        scale = np.linalg.norm(Hm[keep], axis=(1, 2)).max()
        err = np.abs(Hm[keep] - fd[keep]).max()
        print(cloud, mode, "largest |H - central differences| / largest |H|", float(err / scale), int(keep.sum()))
        assert keep.sum() > 50 and err <= 1e-5 * scale, (mode, err, scale)


# ------------------------------------------------------------------ 2. f32 oracle within float64 bounds ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_oracle_within_float64_bounds(cloud):
    """At 1500 random points (none excluded) every entry of the f32 oracle's Hessian lies within f64_hessian's per-point bound
    (times 1.25 for the second-order terms); prints the largest error / bound ratio of each mode.  The inputs are the f32 records
    the oracle folds (the anisotropic ones included), as exact real numbers."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    lo, hi = p.min(0) - float(h), p.max(0) + float(h)
    pts = np.random.default_rng(193).uniform(lo, hi, (1500, 3)).astype(np.float32)
    for mode in MODES:
        radii = mode_kwargs(splashsurf_b200, mode, p, KW).get("particle_radii")
        ctr, w, g6, dlt, _ = records(p, KW, mode, radii)
        oh = oracle_field(p, KW, mode, pts, radii)[2]
        H, reach = f64_hessian(mode, ctr, w, g6, dlt, float(h), pts)
        ref = np.stack([x.v for x in H], 1)
        bnd = 1.25 * np.stack([x.e for x in H], 1)
        err = np.abs(oh.astype(np.float64) - ref)
        assert np.all(oh[~reach] == 0.0)
        assert np.all(np.isfinite(bnd[reach])), (mode, int((~np.isfinite(bnd[reach])).sum()))
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(bnd > 0, err / bnd, np.where(err > 0, np.inf, 0.0))
        print(cloud, mode, "largest error / bound", float(ratio[reach].max()), "points", int(reach.sum()))
        assert np.all(err <= bnd), (mode, float(ratio.max()))


# ------------------------------------------------------------------ 4. one particle ----
ONE_PARTICLE_REL = 1e-3


@pytest.mark.parametrize("mode", MODES)
def test_emulated_one_particle_curvature(emu, mode):  # noqa: F811
    """One particle: the level sets are spheres about it, so at 0.2 h <= rho <= 0.9 h kappa_H = 1 / rho and kappa_G = 1 / rho^2
    within ONE_PARTICLE_REL; prints the largest relative errors."""
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    _, h, _ = _kw_abs(KW)
    rng = np.random.default_rng(171)
    dirs = rng.normal(size=(400, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rho = rng.uniform(0.2, 0.9, (400, 1)) * float(h)
    pts = (p[0].astype(np.float64) + rho * dirs).astype(np.float32)
    rho = np.linalg.norm(pts.astype(np.float64) - p[0], axis=1)
    f = emu.LevelSetField(p, **KW, **mode_kwargs(emu, mode, p, KW))
    try:
        kh, kg = f.curvature(pts)
    finally:
        f.close()
    eh = np.abs(kh * rho - 1.0)
    eg = np.abs(kg * rho * rho - 1.0)
    print(mode, "one particle: largest relative error of kappa_H", float(eh.max()), "kappa_G", float(eg.max()))
    assert eh.max() <= ONE_PARTICLE_REL and eg.max() <= ONE_PARTICLE_REL, (float(eh.max()), float(eg.max()))


# ------------------------------------------------------------------ 5. shape ----
BALL_REL = 0.10                  # kappa_H at the vertices against 1 / median vertex radius; measured -3.6 % .. +2.1 % (DESIGN.md 13.2)
SLAB_H = 0.25                    # median |kappa_H| at the interior top-face vertices, times h; measured 0.083 .. 0.185


def _slab(seed):
    """A flat jittered slab of 24 x 24 x 6 particles."""
    return _lattice(24, 24, 6, 0.1, seed)


@pytest.mark.parametrize("mode", MODES)
def test_emulated_ball_and_slab(emu, mode):  # noqa: F811
    """On a jittered ball of radius 12 r the median kappa_H at the mesh vertices (the anisotropic mode: the mean, DESIGN.md section
    13.2) is within BALL_REL of 1 / (median vertex radius); on a flat jittered slab the median |kappa_H| at the interior top-face
    vertices is below SLAB_H / h.  Prints both."""
    _, h, _ = _kw_abs(KW)
    p = _ball(0.1, 211)
    mk = mode_kwargs(emu, mode, p, KW)
    mesh, _ = emu.reconstruction_pipeline(p, levelset_curvature=True, **KW, **mk)
    v = mesh.mesh.vertices.astype(np.float64)
    rad = np.median(np.linalg.norm(v - p.astype(np.float64).mean(0), axis=1))
    kh = mesh.point_attributes["mean_curvature"]
    # the anisotropic surface is faceted at the scale of the spacing: its kappa_H spreads widely and its median is skewed
    mid = float(np.mean(kh) if mode == "aniso" else np.median(kh))
    print(mode, "ball: kappa_H * median radius - 1", mid * rad - 1.0, "median", float(np.median(kh)) * rad - 1.0,
          "5 / 95 percentile", (np.percentile(kh, [5, 95]) * rad).tolist(), "vertices", len(v))
    assert abs(mid * rad - 1.0) <= BALL_REL
    s = _slab(212)
    mk = mode_kwargs(emu, mode, s, KW)
    mesh, _ = emu.reconstruction_pipeline(s, levelset_curvature=True, **KW, **mk)
    v = mesh.mesh.vertices
    lo, hi = s.min(0), s.max(0)
    top = (v[:, 2] > 0.5 * (lo[2] + hi[2])) & np.all((v[:, :2] > lo[:2] + 2 * h) & (v[:, :2] < hi[:2] - 2 * h), axis=1)
    kh = mesh.point_attributes["mean_curvature"][top]
    med = float(np.median(np.abs(kh)) * h)
    print(mode, "slab: median |kappa_H| h", med, "vertices", int(top.sum()))
    assert top.sum() > 50 and med <= SLAB_H


# ------------------------------------------------------------------ 6. equal radii ----
def test_emulated_equal_radii_equal_plain_averaged(emu):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    rad = np.full(len(p), np.float32(_kw_abs(kw)[0]))
    a = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), **kw)
    b = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), particle_radii=rad, **kw)
    try:
        pts = random_points(a.grid, 2000, 198, pad=0.1)
        for x, y in zip(a.hessian(pts), b.hessian(pts)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
        for x, y in zip(a.curvature(pts), b.curvature(pts)):
            assert _same(x, y)
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ 7. refusals ----
def test_emulated_refusals(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    for corr_rad in (False, True):
        mk = dict(averaged_surface=ss.AveragedSurface(1.0, ss.JacobianCorrection()))
        if corr_rad:
            mk["particle_radii"] = mode_kwargs(ss, "rad", p, KW)["particle_radii"]
        f = ss.LevelSetField(p, **KW, **mk)
        try:
            pts = random_points(f.grid, 10, 3)
            for call in (f.hessian, f.curvature):
                with pytest.raises(ss.SplashsurfError, match="no Hessian") as e:
                    call(pts)
                assert e.value.code == 7                      # SS_ERR_UNSUPPORTED through the C entry
            L = f._ctx._L
            out, g, H, c = np.empty(10, np.float32), np.empty((10, 3), np.float32), np.empty((10, 6), np.float32), np.empty((10, 2), np.float32)
            assert L.ss_levelset_field_hessian_at_f32(f._s, pts.ctypes.data, 10, out.ctypes.data, g.ctypes.data, H.ctypes.data) == 7
            assert L.ss_levelset_field_curvature_at_f32(f._s, pts.ctypes.data, 10, out.ctypes.data, c.ctypes.data) == 7
            assert f.evaluate(pts).shape == (10,)              # the value query stays available
        finally:
            f.close()
    ctx = ss.Context()
    try:
        f = ss.LevelSetField(p, context=ctx, **KW)
        pts = random_points(f.grid, 50, 4)
        for call in (f.hessian, f.curvature):
            with pytest.raises(TypeError):
                call(pts.astype(np.float64))
            with pytest.raises(ValueError):
                call(pts[:, :2])
            nan = pts.copy()
            nan[7, 2] = np.nan
            with pytest.raises(ss.SplashsurfError, match="point 7"):
                call(nan)
        L = ctx._L
        out, g, H, c = np.empty(50, np.float32), np.empty((50, 3), np.float32), np.empty((50, 6), np.float32), np.empty((50, 2), np.float32)
        assert L.ss_levelset_field_hessian_at_f32(f._s, pts.ctypes.data, 50, out.ctypes.data, g.ctypes.data, None) == 6
        assert L.ss_levelset_field_hessian_at_f32(f._s, pts.ctypes.data, 50, out.ctypes.data, None, H.ctypes.data) == 6
        assert L.ss_levelset_field_hessian_at_f32(f._s, pts.ctypes.data, 50, None, g.ctypes.data, H.ctypes.data) == 6
        assert L.ss_levelset_field_curvature_at_f32(f._s, pts.ctypes.data, 50, out.ctypes.data, None) == 6
        assert L.ss_levelset_field_curvature_at_f32(f._s, None, 50, out.ctypes.data, c.ctypes.data) == 6
        assert L.ss_levelset_field_hessian_at_f32(f._s, pts.ctypes.data, 1 << 31, out.ctypes.data, g.ctypes.data, H.ctypes.data) != 0
        assert L.ss_levelset_field_curvature_at_f32(f._s, pts.ctypes.data, 1 << 31, out.ctypes.data, c.ctypes.data) != 0
        ss.reconstruct_surface(p, context=ctx, **KW)
        for call in (f.hessian, f.curvature):
            with pytest.raises(ss.SplashsurfError, match="gone"):
                call(pts)
        f.close()
    finally:
        ctx.close()


def test_emulated_pipeline_and_cli_refusals(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli
    p = _cube(6, 5)
    with pytest.raises(ValueError, match="Jacobian-corrected"):
        emu.reconstruction_pipeline(p, levelset_curvature=True, averaged_surface=emu.AveragedSurface(1.0, emu.JacobianCorrection()), **KW)
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "-o", str(tmp_path / "x.vtk")]
    for extra, msg in ((["--levelset-curvature=on", "--averaged-surface=on", "--averaged-correction=on"], "no Hessian"),
                       (["--levelset-curvature=on", "--partition=on"], "--partition=on")):
        with pytest.raises(ValueError, match=msg):
            cli.main(args + extra)
        assert not os.path.exists(tmp_path / "x.vtk")


# ------------------------------------------------------------------ 8. pipeline and CLI ----
@pytest.mark.parametrize("mode", ["sph", "aniso", "avg", "rad"])
def test_emulated_pipeline_levelset_curvature(emu, mode):  # noqa: F811
    """levelset_curvature=True: the attributes equal field.curvature() at the post-smoothing vertices bit for bit, with and without
    compute_normals; with levelset_normals also on the normals are those of levelset_normals alone."""
    p = _ball(0.1, 111)
    mk = mode_kwargs(emu, mode, p, KW)
    mesh, _ = emu.reconstruction_pipeline(p, levelset_curvature=True, mesh_smoothing_iters=2, **KW, **mk)
    assert set(mesh.point_attributes) == {"mean_curvature", "gaussian_curvature"}
    kh, kg = mesh.point_attributes["mean_curvature"], mesh.point_attributes["gaussian_curvature"]
    nv = len(mesh.mesh.vertices)
    assert kh.dtype == np.float32 and kh.shape == (nv,) and kg.shape == (nv,)
    f = emu.LevelSetField(p, **KW, **mk)
    try:
        rh, rg = f.curvature(np.ascontiguousarray(mesh.mesh.vertices, np.float32))
    finally:
        f.close()
    assert _same(kh, rh) and _same(kg, rg)
    both, _ = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, levelset_curvature=True, mesh_smoothing_iters=2,
                                          **KW, **mk)
    ln, _ = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, mesh_smoothing_iters=2, **KW, **mk)
    assert np.array_equal(both.point_attributes["normals"], ln.point_attributes["normals"])
    assert _same(both.point_attributes["mean_curvature"], kh) and _same(both.point_attributes["gaussian_curvature"], kg)
    area, _ = emu.reconstruction_pipeline(p, compute_normals=True, levelset_curvature=True, mesh_smoothing_iters=2, **KW, **mk)
    assert _same(area.point_attributes["mean_curvature"], kh)


def test_emulated_cli_levelset_curvature(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    out = tmp_path / "k.vtk"
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "--averaged-surface=on"]
    assert cli.main(args + ["--levelset-curvature=on", "-o", str(out)]) == 0
    p = io.read_particles(src)
    mesh, _ = emu.reconstruction_pipeline(p, particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False,
                                          levelset_curvature=True, averaged_surface=emu.AveragedSurface())
    _, _, _, point, _ = io.read_vtk_mesh(str(out))
    for name in ("mean_curvature", "gaussian_curvature"):
        assert _same(np.asarray(point[name], np.float32), mesh.point_attributes[name])
