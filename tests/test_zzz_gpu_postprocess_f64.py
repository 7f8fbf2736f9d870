"""The device post-processing (ss_post.cuh, and k_sph_normals of ss_kernels.cuh) against a float64 reference with a bound per value.

Every reference value is a pair (v, e): v is the reference's formula in real arithmetic on the same f32 inputs (evaluated in float64),
e bounds |f32 evaluation - v| for ANY f32 evaluation of that formula that rounds each operation once and sums in any order.  The bound
is carried operation by operation (class `E`): a rounding adds u (|v| + e), u = 2^-24; products, quotients and square roots propagate
the bounds of their operands; a sum of n terms gets gamma_(n-1) * sum(|t_j| + e_j) on top of the terms' own bounds.  The kernel is
evaluated on the f32 distance, so near the support edge, where (2 - q)^3 cancels, a term is held to what the error of q allows, and a
quotient whose divisor's bound reaches the divisor (a normal where the gradient cancels) is held to nothing.  Intermediates outside
the normal f32 range are flagged (`out`) and those values are not judged: that is where the reference itself stops being free of units.

The query points are placed where the queries can go wrong: a point at 0.9 h, 0.97 h or 0.995 h from exactly one particle, in all 26
directions, with point and particle on the two sides of a subdomain-tile face, edge or corner, or of a splat-bin face; points exactly on
those faces; a particle at exactly d^2 == h^2; points outside the grid.  The points become vertices without triangles of a real
reconstruction (ss_surface_replace_mesh_f32), so the smoothing weights, SPH normals and interpolation of the pipeline all see them, and
they go to the stand-alone SphInterpolator.  k_sph_normals, which picks its candidate bins from the brick of the vertex's edge, runs
on every vertex of reconstructions with R = h / c = 1, 6, 7, 8, 9 and 17 (17: bins of 16 cells).  The mesh kernels run on meshes built
here (degenerate and duplicate triangles, isolated vertices, a fan of 320, non-manifold edges).

The same tables run on the H100 (`ss`) and on the CPU executor of the CUDA sources (`emu`)."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)
from test_post_emulation import emul  # noqa: F401  (fixture: the post-processing kernels alone on the CPU executor)
from test_zzz_gpu_levelset_paths import _cube
from test_zzz_gpu_scale_and_offset import K_ALL, K_SOME, OFFSET_BANDS, REFUSED_BANDS, _scaled, band_offset, offset_band

U = 2.0 ** -24
F32_TINY, F32_BIG = float(np.finfo(np.float32).tiny), 2.0 ** 126


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1.0 - n * U)


class E:
    """A real value `v` (float64 array) with a bound `e` on |f32 evaluation - v|; `out`: an intermediate left the normal f32 range."""

    def __init__(self, v, e=0.0, out=False):
        self.v = np.asarray(v, np.float64)
        self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()
        self.out = np.broadcast_to(np.asarray(out, bool), self.v.shape).copy()

    @staticmethod
    def const(x, roundings):
        """A constant the device rounds to f32 in `roundings` operations."""
        return E(x, gamma(roundings) * abs(x))

    @staticmethod
    def rnd(v, e, out):
        a = np.abs(v)
        with np.errstate(invalid="ignore"):
            out = out | ((a != 0) & ((a < F32_TINY) | (a > F32_BIG)))
        return E(v, e + U * (a + e), out)

    def __getitem__(self, k):
        return E(self.v[k], self.e[k], self.out[k])

    def __add__(self, o):
        o = o if isinstance(o, E) else E(o)
        return E.rnd(self.v + o.v, self.e + o.e, self.out | o.out)

    def __sub__(self, o):
        o = o if isinstance(o, E) else E(o)
        return E.rnd(self.v - o.v, self.e + o.e, self.out | o.out)

    def __rsub__(self, o):
        return E(o) - self

    def __mul__(self, o):
        o = o if isinstance(o, E) else E(o)
        with np.errstate(invalid="ignore"):           # 0 * inf bound: NaN, i.e. not judged
            return E.rnd(self.v * o.v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e, self.out | o.out)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = o if isinstance(o, E) else E(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            m = np.abs(o.v) - o.e
            e = np.where(m > 0, (self.e + np.abs(v) * o.e) / np.where(m > 0, m, 1.0), np.inf)
        return E.rnd(v, e, self.out | o.out)

    def __rtruediv__(self, o):
        return E(o) / self

    def sqrt(self):
        a = np.maximum(self.v, 0.0)
        s = np.sqrt(a)
        e = np.maximum(np.sqrt(a + self.e) - s, s - np.sqrt(np.maximum(a - self.e, 0.0)))
        return E.rnd(s, e, self.out)

    @staticmethod
    def where(mask, a, b):
        return E(np.where(mask, a.v, b.v), np.where(mask, a.e, b.e), np.where(mask, a.out, b.out))


def segsum(t: E, seg, n) -> E:
    """sum_j t_j per segment, f32 in any order: the terms' bounds plus gamma_(n-1) sum(|t_j| + e_j)."""
    cnt = np.bincount(seg, minlength=n)
    v = np.bincount(seg, t.v, minlength=n)
    a = np.bincount(seg, np.abs(t.v) + t.e, minlength=n)
    e = np.bincount(seg, t.e, minlength=n) + gamma(np.maximum(cnt - 1, 0)) * a
    return E(v, e, np.bincount(seg, t.out, minlength=n) > 0)


# ------------------------------------------------------------------ the float64 reference ----
def _sub(a, b):
    """f32 difference of two f32 inputs."""
    return E.rnd(np.asarray(a, np.float64) - np.asarray(b, np.float64), 0.0, False)


def _d2(x, p):
    """Squared distance of f32 points, left to right like the device: (dx dx + dy dy) + dz dz."""
    d = [_sub(x[:, k], p[:, k]) for k in range(3)]
    return d, d[0] * d[0] + d[1] * d[1] + d[2] * d[2]


def pairs(points, particles, h):
    """(point, particle) pairs that can lie within h in f32: the real distance is within h (1 + 1e-5)."""
    from scipy.spatial import cKDTree
    tree = cKDTree(np.asarray(particles, np.float64))
    lists = tree.query_ball_point(np.asarray(points, np.float64), r=float(h) * (1 + 1e-5))
    cnt = np.fromiter((len(l) for l in lists), np.int64, len(lists))
    i = np.repeat(np.arange(len(lists)), cnt)
    j = np.fromiter((q for l in lists for q in l), np.int64, int(cnt.sum()))
    return i, j


def _q(d2, h):
    """q = 2 r / h (kernel.rs:73-107) with r = sqrt of the f32 squared distance."""
    r = d2.sqrt()
    return r, (r + r) / E(h)


def _x2(q):
    """2 - q, clamped at the support: exact in f32 for q in [1, 2], its bound is that of q (plus how far q lies past 2)."""
    return E(np.maximum(2.0 - q.v, 0.0), q.e + np.maximum(q.v - 2.0, 0.0), q.out)


def kernel(q, h):
    """CubicSplineKernel::evaluate (kernel.rs:73-107), constants rounded like fill_kernel_consts."""
    sig = E.const(8.0 / float(h) ** 3, 3)
    inner = E.const(3.0 / (2.0 * np.pi), 3) * ((E.const(2.0 / 3.0, 1) - q * q) + ((0.5 * q) * q) * q)
    x = _x2(q)
    outer = ((E.const(1.0 / (4.0 * np.pi), 3) * x) * x) * x
    f = E.where(q.v < 1.0, inner, outer)
    f.e = f.e + np.where(np.abs(q.v - 1.0) <= q.e, q.e * q.e, 0.0)      # the two pieces agree to first order at q = 1
    return sig * f


def kernel_dq(q):
    """d/dq of the kernel's shape (kernel.rs:83-94), constant 3 / (4 pi)."""
    k = E.const(3.0 / (4.0 * np.pi), 3)
    inner = k * ((-4.0) * q + (3.0 * q) * q)
    x = _x2(q)
    outer = (E(-k.v, k.e) * x) * x
    d = E.where(q.v < 1.0, inner, outer)
    d.e = d.e + np.where(np.abs(q.v - 1.0) <= q.e, 2.0 * k.v * q.e * q.e, 0.0)
    return d


class Ref:
    """Reference values with bounds at `points` for particles `x` (f32), densities `rho`, rest mass `m` and support radius `h`."""

    def __init__(self, x, rho, m, h, points):
        self.x, self.rho, self.h = np.asarray(x, np.float32), np.asarray(rho, np.float32), np.float32(h)
        self.m, self.p = np.float32(m), np.asarray(points, np.float32)
        self.i, self.j = pairs(self.p, self.x, self.h)
        self.d, self.d2 = _d2(self.x[self.j], self.p[self.i])
        self.r, self.q = _q(self.d2, self.h)
        self.vol = E(self.m) / E(self.rho[self.j])
        self.w = self.vol * kernel(self.q, self.h)
        self.den = segsum(self.w, self.i, len(self.p))
        self.n = np.bincount(self.i, minlength=len(self.p))

    def _drop(self, keep):
        """The same sums without the pairs where `keep` is False."""
        r = object.__new__(Ref)
        r.__dict__.update(self.__dict__)
        r.i, r.j, r.d2 = self.i[keep], self.j[keep], self.d2[keep]
        r.d, r.r, r.q, r.vol, r.w = [c[keep] for c in self.d], self.r[keep], self.q[keep], self.vol[keep], self.w[keep]
        r.den = segsum(r.w, r.i, len(self.p))
        return r

    def without_farthest(self):
        """The sums with the farthest in-support particle of every point left out."""
        inside = self.d2.v <= float(self.h) ** 2
        far = np.full(len(self.p), -1)
        order = np.lexsort((self.d2.v, self.i))
        last = np.r_[self.i[order][1:] != self.i[order][:-1], True]
        cand = order[last & inside[order]]
        far[self.i[cand]] = cand
        keep = np.ones(len(self.i), bool)
        keep[far[far >= 0]] = False
        return self._drop(keep)

    def interpolate(self, values, correction):
        """sph_interpolation.rs:210-258: sum_j A_j V_j W_ij, times 1 / sum_j V_j W_ij with the correction; NaN without particles."""
        a = values if isinstance(values, E) else E(np.asarray(values, np.float32))
        if a.v.ndim == 1:
            a = E(a.v[:, None], a.e[:, None], a.out[:, None])
        cols = []
        for k in range(a.v.shape[1]):
            num = segsum(a[self.j, k] * self.w, self.i, len(self.p))
            cols.append(num * (1.0 / self.den) if correction else num)
        out = E(np.stack([c.v for c in cols], 1), np.stack([c.e for c in cols], 1), np.stack([c.out for c in cols], 1))
        nan = (self.den.v == 0) & (self.den.e == 0)
        out.v[nan] = np.nan
        # the sum of weights decides between a number and NaN: a divisor that may be 0 leaves the value open
        open_ = ~nan & (self.den.v - self.den.e <= 0)
        out.e[open_] = np.inf
        return out, nan

    def normals(self):
        """sph_interpolation.rs:82-133: normalize(sum_j V_j (x_j - x_i) / r |grad W|(r)) over d^2 <= h^2."""
        gn = (E.const(8.0 / float(self.h) ** 3, 3) * kernel_dq(self.q)) * E.const(2.0 / float(self.h), 1)
        g = [segsum(((dk / self.r) * gn) * self.vol, self.i, len(self.p)) for dk in self.d]
        nrm = (g[0] * g[0] + g[1] * g[1] + g[2] * g[2]).sqrt()
        n = [gk / nrm for gk in g]
        out = E(np.stack([c.v for c in n], 1), np.stack([c.e for c in n], 1), np.stack([c.out for c in n], 1))
        nan = (self.n == 0) | np.array([(c.v == 0) & (c.e == 0) for c in g]).all(0)
        nan |= np.bincount(self.i, self.d2.v == 0, minlength=len(self.p)) > 0        # a point on a particle: 0 / 0
        out.v[nan] = np.nan
        return out, nan


def weighted_neighbor_counts(x, h) -> E:
    """reconstruct.rs:1190-1205: sum over j != i with d^2 < h^2 of 1 - clamp(d^2 / h^2, 0, 1)."""
    x = np.asarray(x, np.float32)
    i, j = pairs(x, x, h)
    keep = i != j
    i, j = i[keep], j[keep]
    _, d2 = _d2(x[j], x[i])
    ratio = d2 / E.const(float(h) ** 2, 1)
    ratio = E(np.minimum(ratio.v, 1.0), ratio.e, ratio.out)
    return segsum(1.0 - ratio, i, len(x))


def smoothstep(n, normalization) -> E:
    """reconstruct.rs:1220-1231: x = min(max(n, 0) / normalization, 1) with Rust's NaN-ignoring max; 6 x^5 - 15 x^4 + 10 x^3."""
    n = n if isinstance(n, E) else E(np.asarray(n, np.float32))
    v = np.where(np.isnan(n.v), 0.0, n.v)
    pos = E(np.maximum(v, 0.0), np.where(np.isnan(n.v), 0.0, n.e), n.out)
    with np.errstate(invalid="ignore"):
        x = pos / E(np.float32(normalization))
        one = x.v - x.e >= 1.0
    x = E(np.where(one, 1.0, np.minimum(x.v, 1.0)), np.where(one, 0.0, x.e), x.out & ~one)
    x3 = (x * x) * x
    x4 = x3 * x
    x5 = x4 * x
    return (x5 * 6.0 - x4 * 15.0) + x3 * 10.0


def csr(tris, nv):
    """Unique neighbours per vertex in ascending order (mesh.rs:290-306; a pair with equal indices is no edge)."""
    from oracle import postprocess as pp
    off, adj = pp.vertex_vertex_connectivity(np.asarray(tris, np.int64), nv)
    adj = np.concatenate([np.sort(adj[off[k]:off[k + 1]]) for k in range(nv)]) if len(adj) else adj
    return off, adj


def _vec(cols):
    return E(np.stack([c.v for c in cols], 1), np.stack([c.e for c in cols], 1), np.stack([c.out for c in cols], 1))


def laplacian(verts, off, adj, iterations, beta, weights) -> E:
    """postprocessing.rs:17-53 with the buffer swap at :31: the vertex blended with the neighbour mean is the one of two iterations ago."""
    nv = len(verts)
    seg = np.repeat(np.arange(nv), np.diff(off))
    deg = np.diff(off).astype(np.float64)
    w = weights if isinstance(weights, E) else E(np.asarray(weights, np.float32))
    cur = [E(np.asarray(verts, np.float32)[:, k]) for k in range(3)]
    buf = [E(c.v) for c in cur]
    be = E(np.float32(beta)) * w
    om = 1.0 - be
    for _ in range(iterations):
        cur, buf = buf, cur
        nxt = []
        for k in range(3):
            s = segsum(buf[k][adj], seg, nv)
            mean = E.where(deg > 0, s / E(np.maximum(deg, 1.0)), s)
            nxt.append(cur[k] * om + mean * be)
        cur = nxt
    return _vec(cur)


def smooth_normals(normals, off, adj, iterations) -> E:
    """postprocessing.rs:56-97: n_i = normalize(sum of the neighbours' normals)."""
    nv = len(normals)
    seg = np.repeat(np.arange(nv), np.diff(off))
    cur = [E(np.asarray(normals, np.float32)[:, k]) for k in range(3)]
    for _ in range(iterations):
        s = [segsum(c[adj], seg, nv) for c in cur]
        nrm = (s[0] * s[0] + s[1] * s[1] + s[2] * s[2]).sqrt()
        cur = [sk / nrm for sk in s]
    return _vec(cur)


def area_normals(verts, tris) -> E:
    """mesh.rs:812-821 + :899-905: sum over the incident triangles of cross(v1 - v0, v2 - v1), normalised."""
    v = np.asarray(verts, np.float32)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    a = [_sub(v[t[:, 1], k], v[t[:, 0], k]) for k in range(3)]
    b = [_sub(v[t[:, 2], k], v[t[:, 1], k]) for k in range(3)]
    cr = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    # incident (vertex, triangle) pairs, each once
    vt = np.unique(np.stack([t.ravel(), np.repeat(np.arange(len(t)), 3)], 1), axis=0) if len(t) else np.zeros((0, 2), np.int64)
    s = [segsum(c[vt[:, 1]], vt[:, 0], len(v)) for c in cr]
    nrm = (s[0] * s[0] + s[1] * s[1] + s[2] * s[2]).sqrt()
    return _vec([sk / nrm for sk in s])


# ------------------------------------------------------------------ judging ----
def check(got, ref: E, nan=None, what="", min_judged=0.0, f32=None):
    """Device values inside the bound wherever the bound is finite and the intermediates stay in range; NaN exactly where the
    reference has none.  The window is what the `out` flags leave: inside it at least `min_judged` of the values must have a finite
    bound (and so be judged); outside it the device must be non-finite exactly where `f32`, an f32 evaluation of the same formula,
    is.  Returns (fraction judged, fraction outside the window)."""
    g = np.asarray(got, np.float64).reshape(ref.v.shape)
    rows = ref.v.reshape(len(ref.v), -1)
    g2 = g.reshape(len(g), -1)
    nan = np.zeros(len(rows), bool) if nan is None else np.asarray(nan)
    gn = np.isnan(g2)
    assert gn[nan].all(), (what, "finite where the reference is NaN", np.nonzero(nan & ~gn.all(1))[0][:8])
    e = ref.e.reshape(len(rows), -1)
    out = ref.out.reshape(len(rows), -1).any(1) & ~nan
    judged = ~nan & np.isfinite(e).all(1) & ~out
    bad = judged & (gn.any(1) | (np.abs(g2 - rows) > e).any(1))
    if bad.any():
        k = np.nonzero(bad)[0]
        worst = k[np.argmax(np.nanmax(np.abs(g2[k] - rows[k]) / np.maximum(e[k], 1e-300), 1))]
        raise AssertionError(f"{what}: {len(k)} of {int(judged.sum())} values outside their bound; worst point {worst}: device "
                             f"{g2[worst].tolist()}, reference {rows[worst].tolist()} +- {e[worst].tolist()}")
    window = ~nan & ~out
    frac = float(judged.sum() / window.sum()) if window.any() else 1.0
    assert frac >= min_judged, (what, frac)
    if out.any():
        assert f32 is not None, (what, "values outside the f32 window and no f32 evaluation to hold them to")
        want = ~np.isfinite(np.asarray(f32, np.float64).reshape(len(g2), -1))
        have = ~np.isfinite(g2)
        diff = out & (want != have).any(1)
        assert not diff.any(), (what, "non-finite pattern outside the window differs from the f32 evaluation", np.nonzero(diff)[0][:8],
                                g2[diff][:4].tolist(), np.asarray(f32).reshape(len(g2), -1)[diff][:4].tolist())
    return float(judged.mean()) if len(judged) else 1.0, float(out.mean()) if len(out) else 0.0


def outside(got, ref: E, nan):
    """True where a value lies outside the bound (what a sensitive probe must do when a term is missing)."""
    g = np.asarray(got, np.float64).reshape(len(ref.v), -1)
    v, e = ref.v.reshape(len(g), -1), ref.e.reshape(len(g), -1)
    with np.errstate(invalid="ignore"):
        return (np.isnan(g).any(1) != nan) | (np.abs(g - v) > e).any(1)


# ------------------------------------------------------------------ probes ----
DIRS = [np.array(s, np.float64) for s in itertools.product((-1, 0, 1), repeat=3) if any(s)]
FRACTIONS = (0.9, 0.97, 0.995)


def probe_layout(gmin, c, S, be, h, origin_tile, kinds=("tile", "bin")):
    """Sole-neighbour probes.  For each kind of corner (a subdomain-tile corner, or a splat-bin corner inside a tile) and each octant s,
    one particle X sits just past the corner in that octant, 2 tiles away from any other; around it the points X - f h d for every
    direction d whose non-zero components have the signs of s (so point and particle lie on the two sides of 1, 2 or 3 faces), and
    the points on those faces.  Returns particles, points, and for each point the index of its particle (-1: none)."""
    gmin = np.asarray(gmin, np.float32)
    sub = np.float32(np.float32(c) * np.float32(S))
    delta = 0.003 * float(h)
    xs, pts, owner = [], [], []
    for n_site, (kind, s) in enumerate(itertools.product(kinds, itertools.product((-1, 1), repeat=3))):
        kt = np.asarray(origin_tile) + 2 * np.array([n_site % 4, (n_site // 4) % 2, n_site // 8])
        corner = (gmin + (kt.astype(np.float32) * sub).astype(np.float32)).astype(np.float32)
        if kind == "bin":
            corner = (corner + np.float32(be) * np.float32(c)).astype(np.float32)
        s = np.asarray(s, np.float64)
        x = (corner.astype(np.float64) + s * delta).astype(np.float32)
        xs.append(x)
        for d in DIRS:
            if np.any((d != 0) & (d != s)):
                continue
            u = d / np.linalg.norm(d)
            for f in FRACTIONS:
                pts.append((x.astype(np.float64) - f * float(h) * u).astype(np.float32)); owner.append(len(xs) - 1)
            on_face = x.copy()
            on_face[d != 0] = corner[d != 0]                                      # exactly on the face / edge / corner
            pts.append(on_face); owner.append(len(xs) - 1)
    return np.array(xs, np.float32), np.array(pts, np.float32), np.array(owner)


def check_probes_sensitive(ref: Ref, owner, n_particles_before):
    """Every probe point has exactly its own particle within h, and the reference without it lies outside the bound."""
    own = owner >= 0
    inside = ref.d2.v <= float(ref.h) ** 2
    cnt = np.bincount(ref.i[inside], minlength=len(ref.p))
    assert (cnt[own] == 1).all(), np.nonzero(own & (cnt != 1))[0][:8]
    assert np.array_equal(ref.j[inside & own[ref.i]], owner[ref.i[inside & own[ref.i]]] + n_particles_before)
    cut = ref.without_farthest()
    vals = np.linspace(1, 2, len(ref.x)).astype(np.float32)
    for corr in (True, False):
        a, nan = ref.interpolate(vals, corr)
        b, _ = cut.interpolate(vals, corr)
        fin = own & np.isfinite(a.e).all(1) & ~nan
        assert fin.sum() >= 0.9 * own.sum()
        assert outside(b.v, a, nan)[fin].all(), "a probe that does not see its only particle"
    nrm, nan = ref.normals()
    fin = own & np.isfinite(nrm.e).all(1) & ~nan
    assert outside(cut.normals()[0].v, nrm, nan)[fin].all()


# ------------------------------------------------------------------ device entries ----
def surface_queries(lib, x, kw, pts, aniso=False, normalization=13.0):
    """A reconstruction of x; its mesh replaced by `pts` (vertices without triangles), then every particle query of the surface there:
    smoothing weights (wnn, sw), SPH normals (k_pp_sph_normals) and interpolation of a scalar and a vector, with and without the
    correction.  Returns those, the reconstruction's filtered particles and densities, and its grid."""
    ctx = lib.Context()
    try:
        L = ctx._L
        p = lib.make_params(**kw)
        s = lib._reconstruct_raw(ctx, np.ascontiguousarray(x, np.float32), p, lib.Anisotropy() if aniso else None)
        try:
            n = L.ss_surface_num_particles(s)
            rho = np.empty(n, np.float32)
            lib._check(L, L.ss_surface_copy_particle_densities(s, rho.ctypes.data))
            g = lib._Grid()
            lib._check(L, L.ss_surface_grid(s, C.byref(g)))
            xf = x
            if p.has_particle_aabb:
                inside = np.empty(len(x), np.uint8)
                lib._check(L, L.ss_surface_copy_particle_inside_aabb(s, inside.ctypes.data))
                xf = x[inside.astype(bool)]
            assert len(xf) == n
            pts = np.ascontiguousarray(pts, np.float32)
            m = len(pts)
            lib._check(L, L.ss_surface_replace_mesh_f32(s, pts.ctypes.data, m, None, 0))
            out = {"x": xf, "rho": rho, "grid": (np.array(g.aabb_min[:], np.float32), np.array(g.aabb_max[:], np.float32)),
                   "wnn": np.empty(m, np.float32), "sw": np.empty(m, np.float32), "normals": np.empty((m, 3), np.float32)}
            lib._check(L, L.ss_surface_compute_smoothing_weights_f32(s, C.c_float(normalization), out["wnn"].ctypes.data, out["sw"].ctypes.data))
            lib._check(L, L.ss_surface_compute_normals_f32(s, 1))
            lib._check(L, L.ss_surface_copy_normals(s, out["normals"].ctypes.data))
            a1, a3 = _attributes(xf)
            for corr in (1, 0):
                for name, a in (("a1", a1), ("a3", a3)):
                    o = np.empty((m,) if a.ndim == 1 else (m, 3), np.float32)
                    lib._check(L, L.ss_surface_interpolate_quantity_f32(s, a.ctypes.data, a.ndim if a.ndim == 1 else 3, corr, o.ctypes.data))
                    out[f"{name}_{corr}"] = o
            return out
        finally:
            ctx.free_surface(s)
    finally:
        ctx.close()


def _attributes(x):
    a1 = np.ascontiguousarray((np.arange(len(x)) % 17 * 0.25 - 1).astype(np.float32))
    a3 = np.ascontiguousarray(np.random.default_rng(len(x)).normal(size=(len(x), 3)).astype(np.float32))
    return a1, a3


def f32_evaluations(x, rho, m, h, pts):
    """The same formulas evaluated in f32 (oracle/postprocess.py, oracle.sph_normals): what the device is held to outside the window."""
    import oracle
    from oracle import postprocess as pp
    with np.errstate(all="ignore"):
        wnn = pp.interpolate_quantity(x, rho, m, h, pp.weighted_neighbor_counts(x, h), pts, True)
        f = {"wnn": wnn, "sw": pp.smoothing_weights(wnn, 13.0),
             "normals": oracle.sph_normals(x, rho, pts, compact_support_radius=h, particle_rest_mass=m)}
        a1, a3 = _attributes(x)
        for corr in (1, 0):
            for name, a in (("a1", a1), ("a3", a3)):
                f[f"{name}_{corr}"] = pp.interpolate_quantity(x, rho, m, h, a, pts, bool(corr))
    return f


def check_surface_queries(out, m, h, pts, min_judged=0.9):
    """Every output of `surface_queries` against the float64 reference at the same points.  Returns the fractions outside the window."""
    x, rho = out["x"], out["rho"]
    # a point outside the grid has no particle within h: the grid reaches past every particle by more than h, so the clamped tile
    # lookup of ss_tile_of_position only ever serves points with an empty sum
    gmin, gmax = out["grid"]
    assert (gmin.astype(np.float64) <= x.min(0).astype(np.float64) - float(h)).all() and (gmax.astype(np.float64) >= x.max(0) + float(h)).all()
    ref = Ref(x, rho, m, h, pts)
    f32 = f32_evaluations(x, rho, m, h, pts)
    windows = {}
    wnc = weighted_neighbor_counts(x, h)
    wnn, nan = ref.interpolate(wnc, True)
    windows["wnn"] = check(out["wnn"], wnn, nan, "wnn", min_judged, f32["wnn"])[1]
    sw = smoothstep(E(wnn.v[:, 0], wnn.e[:, 0], wnn.out[:, 0]), 13.0)
    windows["sw"] = check(out["sw"], sw, None, "sw", min_judged, f32["sw"])[1]
    nrm, nan = ref.normals()
    windows["normals"] = check(out["normals"], nrm, nan, "k_pp_sph_normals", min_judged * 0.9, f32["normals"])[1]
    a1, a3 = _attributes(x)
    for corr in (1, 0):
        for name, a in (("a1", a1), ("a3", a3)):
            r, nan = ref.interpolate(a, bool(corr))
            key = f"{name}_{corr}"
            windows[key] = check(out[key], r, nan, f"interpolate {name} correction={corr}", min_judged, f32[key])[1]
    return windows


# ------------------------------------------------------------------ scales and offsets ----
def moved(x, pts, k=0, band=None, sign=1):
    """The scene scaled by 2^k (exact) or moved by (o, -o, o) into offset band `band` of test_zzz_gpu_scale_and_offset."""
    s = np.float32(2.0 ** k)
    x, pts = (x * s).astype(np.float32), (pts * s).astype(np.float32)
    if band is not None:
        o = sign * band_offset(band) * np.array([1.0, -1.0, 1.0])
        x, pts = (x.astype(np.float64) + o).astype(np.float32), (pts.astype(np.float64) + o).astype(np.float32)
        assert offset_band(float(np.abs(x).max())) == band
    return x, pts, float(s)


ACCEPTED_BANDS = [b for b in OFFSET_BANDS if b not in REFUSED_BANDS and b != -18]       # -18: a cloud at the origin, the k = 0 cases
OFFSETS = [(b, sign) for b in ACCEPTED_BANDS for sign in (1, -1)]


# ------------------------------------------------------------------ the probe cloud of a reconstruction ----
R_ = 0.025
PROBE_KW = dict(particle_radius=R_, smoothing_length=2.0, cube_size=0.5, subdomain_grid_auto_disable=False)


def probe_scene(oracle_mod, S):
    """A small jittered cube (a surface), two anchor particles that fix the grid, and the sole-neighbour probes of `probe_layout`
    on tiles of S cubes (c = 0.0125, h = 0.1, R = 8, bins of 8 cells).  The isolated probe particles make most subdomains sparse."""
    kw = dict(PROBE_KW, subdomain_num_cubes_per_dim=S)
    _, h, c = oracle_mod.absolute_params(R_, 2.0, 0.5)
    sub = float(c) * S
    hi = 0.35 + sub * 9
    anchors = np.array([[-0.1, -0.1, -0.1], [hi, 4.5 * sub + 0.3, 6.5 * sub + 0.3]], np.float32)
    g = oracle_mod.reconstruct(anchors, **kw)["grid"]
    tile0 = np.ceil((0.55 - g["aabb_min"]) / sub).astype(int)
    xs, pts, owner = probe_layout(g["aabb_min"], c, S, 8, h, tile0)
    body = _cube(5, 7)
    x = np.concatenate([anchors, body, xs]).astype(np.float32)
    assert oracle_mod.reconstruct(x, **kw)["grid"]["aabb_min"].tolist() == g["aabb_min"].tolist()
    # the body's vertices-to-be, and points outside the grid
    far = np.array([g["aabb_min"] - 0.05, g["aabb_max"] + 0.05, [g["aabb_min"][0] - 0.01, 0.1, 0.1]], np.float32)
    pts = np.concatenate([pts, far, (body[::7] + np.float32(0.3 * h)).astype(np.float32)])
    owner = np.concatenate([owner, -np.ones(len(pts) - len(owner), int)])
    return x, kw, pts, owner, 2 + len(body), h


PROBE_PATHS = {
    "S16": dict(subdomain_num_cubes_per_dim=16),
    "S32": dict(subdomain_num_cubes_per_dim=32),
    "S64": dict(subdomain_num_cubes_per_dim=64),
    "global": dict(subdomain_num_cubes_per_dim=16, subdomain_grid=False),
    "aniso": dict(subdomain_num_cubes_per_dim=16),
}


@pytest.mark.parametrize("S", [16, 32, 64])
def test_probe_reference_is_sensitive(oracle_mod, S):
    """CPU: each probe sees exactly its own particle, and leaving that particle out moves every output out of its bound."""
    x, kw, pts, owner, n0, h = probe_scene(oracle_mod, S)
    o = oracle_mod.reconstruct(x, **kw)
    assert o["used_decomposition"] and o["subdomain_sparse"].any() and not o["subdomain_sparse"].all()
    ref = Ref(x, o["particle_densities"], oracle_mod.sph_rest_mass(R_), h, pts)
    check_probes_sensitive(ref, owner, n0)


def run_probe_scene(lib, oracle_mod, path, k=0, band=None, sign=1):
    S = PROBE_PATHS[path]["subdomain_num_cubes_per_dim"]
    x, kw, pts, owner, n0, h = probe_scene(oracle_mod, S)
    x, pts, s = moved(x, pts, k, band, sign)
    kw = _scaled(dict(kw, **PROBE_PATHS[path]), s)
    out = surface_queries(lib, x, kw, pts, aniso=path == "aniso")
    return sum(check_surface_queries(out, oracle_mod.sph_rest_mass(kw["particle_radius"]), oracle_mod.absolute_params(kw["particle_radius"], 2.0, 0.5)[1],
                                     pts, min_judged(k)).values())


# ------------------------------------------------------------------ the stand-alone interpolator ----
HI = 0.125          # a power of two: points at exactly d^2 == h^2 exist in f32


def interpolator_scene(oracle_mod, k=0, band=None, sign=1):
    """Sole-neighbour probes on the SphInterpolator's own grid (cubes of h / 2, tiles of 64 cubes), plus a dense cluster
    (3x the rest density), a particle with a point at exactly h (the term counts with W = 0: NaN, like an empty sum), and points
    outside the grid; scaled by 2^k or moved into an offset band."""
    h = np.float32(HI)
    anchors = np.array([[-1, -1, -1], [36, 20, 20]], np.float32)
    g = oracle_mod.reconstruct(anchors, particle_radius=HI / 4, smoothing_length=2.0, cube_size=2.0, subdomain_grid_auto_disable=False)["grid"]
    xs, pts, owner = probe_layout(g["aabb_min"], h / 2, 64, 8, h, np.array([1, 1, 1]))
    rng = np.random.default_rng(11)
    cluster = (rng.uniform(-0.5, 0.5, (400, 3)) * 0.36 * float(h) + 2.0).astype(np.float32)     # ~3x rest density of r = h / 4
    edge_x = np.array([[1.0, 3.0, 1.0]], np.float32)
    edge_p = np.array([[1.0 - HI, 3.0, 1.0], [1.0, 3.0 + HI, 1.0]], np.float32)
    x = np.concatenate([anchors, cluster, edge_x, xs]).astype(np.float32)
    assert oracle_mod.reconstruct(x, particle_radius=HI / 4, smoothing_length=2.0, cube_size=2.0,
                                  subdomain_grid_auto_disable=False)["grid"]["aabb_min"].tolist() == g["aabb_min"].tolist()
    extra = np.concatenate([edge_p, (cluster[::5] + np.float32(0.1 * h)).astype(np.float32),
                            np.array([g["aabb_min"] - 1.0, [40, 1, 1], [-1.5, 3, 1]], np.float32)])
    pts = np.concatenate([pts, extra])
    owner = np.concatenate([owner, -np.ones(len(extra), int)])
    rho = np.full(len(x), 1000.0, np.float32) * rng.uniform(0.8, 1.2, len(x)).astype(np.float32)
    x, pts, s = moved(x, pts, k, band, sign)
    cl = np.arange(len(pts) - len(extra) + 2, len(pts) - 3)
    return x, rho, np.float32(1e-3 * s ** 3), np.float32(h * np.float32(s)), pts, owner, len(x) - len(xs), np.arange(2) + len(pts) - len(extra), cl


def test_interpolator_reference_is_sensitive(oracle_mod):
    """CPU: the sole-neighbour probes, and in the crowded cluster the loss of the farthest particle leaves the bound at most points."""
    x, rho, m, h, pts, owner, n0, edge, cl = interpolator_scene(oracle_mod)
    ref = Ref(x, rho, m, h, pts)
    check_probes_sensitive(ref, owner, n0)
    assert (ref.d2.v[np.isin(ref.i, edge)] == float(h) ** 2).any()
    assert ref.n[cl].min() > 100
    a1, _ = _attributes(x)
    r, nan = ref.interpolate(a1, False)
    cut, _ = ref.without_farthest().interpolate(a1, False)
    assert outside(cut.v[cl], r[cl], nan[cl]).mean() >= 0.5


def run_interpolator(lib, oracle_mod, k=0, band=None, sign=1, it_cls=None):
    x, rho, m, h, pts, owner, n0, edge, cl = interpolator_scene(oracle_mod, k, band, sign)
    from oracle import postprocess as pp
    import oracle
    it = (it_cls or lib.SphInterpolator)(x, rho, m, h)
    try:
        a1, a3 = _attributes(x)
        ref = Ref(x, rho, m, h, pts)
        windows = []
        with np.errstate(all="ignore"):
            for corr in (True, False):
                for a in (a1, a3):
                    got = np.asarray(it.interpolate_quantity(a, pts, first_order_correction=corr))
                    r, nan = ref.interpolate(a, corr)
                    windows.append(check(got, r, nan, f"SphInterpolator correction={corr}", min_judged(k), pp.interpolate_quantity(x, rho, m, h, a, pts, corr))[1])
                    assert np.isnan(got[edge]).all()
            got = np.asarray(it.interpolate_normals(pts))
            nrm, nan = ref.normals()
            windows.append(check(got, nrm, nan, "SphInterpolator normals", 0.8 * min_judged(k),
                                 oracle.sph_normals(x, rho, pts, compact_support_radius=h, particle_rest_mass=m))[1])
        assert np.isnan(got[edge]).all()
        return max(windows)
    finally:
        if hasattr(it, "close"):
            it.close()


# Windows found by the `out` flags of the float64 reference (DESIGN.md row f.1), per scene: (last k at which the share of values
# outside the normal f32 range is still the one at k = 0, that share summed over the outputs).  At k = 0 the only such values are
# smooth-step powers of tiny counts (probe scene) and kernel values of the particle at exactly h (interpolator).  Past the window,
# terms near the support edge underflow (gradients ~ V / h^4 first); at k = -36 the gradient term (dx / r) |grad W| overflows.
# Inside, every value with a finite bound is judged; outside, the device's non-finite pattern must be the f32 evaluation's.
WINDOWS = {"probe": (28, 0.0064), "interpolator": (30, 0.0038), "vertices": (25, 0.0)}


def assert_window(scene, k, share):
    last, at0 = WINDOWS[scene]
    if -22 <= k <= last:
        assert round(share, 4) == at0, (scene, k, share)
    if abs(k) == 36:
        assert share > at0, (scene, k, share)


def min_judged(k):
    return 0.9 if -22 <= k <= 25 else 0.0


# ------------------------------------------------------------------ k_sph_normals on every vertex ----
def _splash():
    from splashsurf_b200 import synthetic as syn
    return syn.splash((8, 8, 8), 2, 0.025, 105).astype(np.float32)


# name -> (cloud, cube_size, R, bin cells)
NORMAL_CASES = {
    "R1": (_splash, 4.0, 1, 8),
    "R6": (lambda: _cube(8, 1), 0.68, 6, 8),
    "R7": (_splash, 0.6, 7, 8),
    "R8": (_splash, 0.5, 8, 8),
    "R9": (_splash, 0.45, 9, 8),
    "R9_S32": (lambda: _cube(8, 1), 0.45, 9, 8),
    "R17": (lambda: _cube(5, 3), 0.2424, 17, 16),
}


def check_vertex_normals(lib, oracle_mod, name, k=0, band=None, sign=1):
    gen, cube, R, be = NORMAL_CASES[name]
    x, _, s = moved(gen(), np.zeros((0, 3), np.float32), k, band, sign)
    S = 32 if name.endswith("S32") else 16
    kw = _scaled(dict(particle_radius=R_, smoothing_length=2.0, cube_size=cube, subdomain_num_cubes_per_dim=S, subdomain_grid_auto_disable=False), s)
    ctx = lib.Context()
    try:
        res = lib.reconstruct_surface(x, sph_normals=True, with_debug=True, context=ctx, **kw)
    finally:
        ctx.close()
    assert res.levelset_paths["R"] == R and res.levelset_paths["bin_cells"] == be, res.levelset_paths
    v, keys = res.mesh.vertices, res.vertex_edge_keys
    ax = keys[:, 3]
    along = keys[np.arange(len(keys)), ax]
    assert (along % 8 == 7).any()                                                      # edges that leave their brick
    ortho = np.array([[keys[q, d] % S == 0 for d in range(3) if d != ax[q]] for q in range(len(keys))])
    if len(res.subdomains["flat"]) > 8:                                                # (R1: the grid is one tile)
        assert ortho.any(1).any() and ortho.all(1).any()                               # on tile faces and tile edges
    _, h, _ = oracle_mod.absolute_params(kw["particle_radius"], 2.0, cube)
    m = oracle_mod.sph_rest_mass(kw["particle_radius"])
    ref = Ref(x, res.particle_densities, m, h, v)
    nrm, nan = ref.normals()
    f32 = oracle_mod.sph_normals(x, res.particle_densities, v, compact_support_radius=h, particle_rest_mass=m)
    window = check(res.normals, nrm, nan, f"k_sph_normals {name}", min_judged(k), f32)[1]
    # k_pp_sph_normals and the other queries at the same vertices
    out = surface_queries(lib, x, kw, v)
    check(out["normals"], nrm, nan, f"k_pp_sph_normals {name}", min_judged(k), f32)
    return window


@pytest.mark.parametrize("name", ["R1", "R9"])
def test_vertex_reference_sees_a_lost_edge_particle(oracle_mod, name):
    """CPU: on the vertices of the cases where k_sph_normals used to lose particles, leaving out each vertex's farthest particle moves
    the normal out of its bound at a share of the vertices (there the bound alone decides whether a support-edge loss is seen)."""
    gen, cube, _, _ = NORMAL_CASES[name]
    x = gen()
    o = oracle_mod.reconstruct(x, particle_radius=R_, smoothing_length=2.0, cube_size=cube, subdomain_num_cubes_per_dim=16, subdomain_grid_auto_disable=False)
    _, h, _ = oracle_mod.absolute_params(R_, 2.0, cube)
    ref = Ref(x, o["particle_densities"], oracle_mod.sph_rest_mass(R_), h, o["vertices"])
    nrm, nan = ref.normals()
    frac = outside(ref.without_farthest().normals()[0].v, nrm, nan)[~nan].mean()
    assert frac >= LOST_PARTICLE_SEEN[name], frac


LOST_PARTICLE_SEEN = {"R1": 0.85, "R9": 0.85}          # 0.91 measured on both


# ------------------------------------------------------------------ the pipeline, and the wheel ----
def check_pipeline(x, rho, m, h, raw_v, tris, got, iterations, attrs, min_judged=0.9):
    """reconstruct.rs:1159-1391 on a given mesh: wnn / sw at the raw vertices, `iterations` of weighted smoothing (beta = 1), then SPH
    normals and corrected interpolation at the smoothed vertices `got["vertices"]`, each against the float64 reference."""
    raw_v = np.asarray(raw_v, np.float32)
    ref = Ref(x, rho, m, h, raw_v)
    wnn, nan = ref.interpolate(weighted_neighbor_counts(x, h), True)
    check(got["wnn"], wnn, nan, "pipeline wnn", min_judged)
    sw = smoothstep(E(wnn.v[:, 0], wnn.e[:, 0], wnn.out[:, 0]), 13.0)
    check(got["sw"], sw, None, "pipeline sw", min_judged)
    off, adj = csr(tris, len(raw_v))
    check(got["vertices"], laplacian(raw_v, off, adj, iterations, 1.0, sw), None, "pipeline smoothed vertices", min_judged)
    refs = Ref(x, rho, m, h, got["vertices"])
    nrm, nan = refs.normals()
    check(got["normals"], nrm, nan, "pipeline normals", min_judged * 0.9)
    for name, a in attrs.items():
        r, nan = refs.interpolate(a, True)
        check(got[name], r, nan, f"pipeline {name}", min_judged)


PIPELINE_CASES = {
    "cleanup_decimation": dict(mesh_cleanup=True, mesh_cleanup_snap_dist=0.5, decimate_barnacles=True),
    "particle_aabb": dict(aabb_min=[-0.05, -0.05, -0.05], aabb_max=[0.3, 0.25, 0.3]),
}


def check_device_pipeline(lib, case):
    """reconstruction_pipeline on the device; the mesh it post-processes is rebuilt with the free functions (clean-up + decimation)."""
    import oracle
    x = _splash()
    kw = dict(particle_radius=R_, smoothing_length=2.0, cube_size=0.6)
    a1, a3 = _attributes(x)
    extra = PIPELINE_CASES[case]
    mw, rec = lib.reconstruction_pipeline(x, attributes_to_interpolate={"a1": a1, "a3": a3}, **kw, **extra, mesh_smoothing_iters=3,
                                          output_mesh_smoothing_weights=True, compute_normals=True, sph_normals=True)
    mesh = rec.mesh.copy()
    if extra.get("mesh_cleanup"):
        lib.marching_cubes_cleanup(mesh, rec.grid, max_rel_snap_dist=0.5, max_iter=5)
        lib.barnacle_decimation(mesh)
        assert mesh.nvertices < rec.mesh.nvertices and np.array_equal(mw.mesh.triangles, mesh.triangles)
    inside = rec.particle_inside_aabb
    xf = x if inside is None else x[inside]
    if inside is not None:
        assert 0 < inside.sum() < len(x)
    _, h, _ = oracle.absolute_params(R_, 2.0, 0.6)
    got = dict(mw.point_attributes, vertices=mw.mesh.vertices)
    attrs = {k: (v if inside is None else v[inside]) for k, v in (("a1", a1), ("a3", a3))}
    check_pipeline(xf, rec.particle_densities, oracle.sph_rest_mass(R_), h, mesh.vertices, mesh.triangles, got, 3, attrs)


def test_wheel_inside_bounds(oracle_mod):
    """CPU, where the reference wheel is unpacked: its SphInterpolator and reconstruction_pipeline outputs lie inside the float64
    bounds -- this pins the reference's semantics (inclusion at d^2 <= h^2, NaN for an empty sum with and without the correction,
    the NaN-ignoring max, the buffer swap of the smoothing) to the float64 reference the device is judged by."""
    if not oracle_mod.reference_available():
        pytest.skip("oracle/_ref (reference wheel) not present")
    ps = oracle_mod.reference()
    run_interpolator(None, oracle_mod, it_cls=lambda x, rho, m, h: ps.SphInterpolator(x, rho, float(m), float(h)))
    x = _splash()
    kw = dict(particle_radius=R_, smoothing_length=2.0, cube_size=0.6)
    a1, a3 = _attributes(x)
    mw, rec = ps.reconstruction_pipeline(x, attributes_to_interpolate={"a1": a1, "a3": a3}, **kw, output_raw_mesh=True, mesh_smoothing_iters=3,
                                         output_mesh_smoothing_weights=True, compute_normals=True, sph_normals=True)
    got = {k: np.asarray(v) for k, v in mw.point_attributes.items()}
    got["vertices"] = np.asarray(mw.mesh.vertices)
    _, h, _ = oracle_mod.absolute_params(R_, 2.0, 0.6)
    check_pipeline(x, np.asarray(rec.particle_densities), oracle_mod.sph_rest_mass(R_), h, np.asarray(rec.mesh.vertices),
                   np.asarray(rec.mesh.triangles), got, 3, {"a1": a1, "a3": a3})


# ------------------------------------------------------------------ meshes built here ----
def built_mesh(nv_grid=23):
    """A height field of nv_grid^2 vertices plus: a fan of 320 triangles around one vertex, degenerate triangles (a repeated
    index), duplicated triangles, an edge shared by 4 triangles, and isolated vertices; nv is not a multiple of 128 or 256."""
    rng = np.random.default_rng(17)
    g = np.stack(np.meshgrid(np.arange(nv_grid), np.arange(nv_grid), indexing="ij"), -1).reshape(-1, 2).astype(np.float64) * 0.05
    z = 0.02 * np.sin(7 * g[:, 0]) * np.cos(5 * g[:, 1]) + rng.normal(0, 0.002, len(g))
    v = [np.column_stack([g, z])]
    tris = []
    for i in range(nv_grid - 1):
        for j in range(nv_grid - 1):
            a, b, c_, d = i * nv_grid + j, (i + 1) * nv_grid + j, i * nv_grid + j + 1, (i + 1) * nv_grid + j + 1
            tris += [(a, b, d), (a, d, c_)]
    n = len(v[0])
    centre, rim = n, n + 1 + np.arange(320)
    ang = np.linspace(0, 2 * np.pi, 320, endpoint=False)
    v.append(np.array([[2.0, 0.5, 0.1]]))
    v.append(np.column_stack([2.0 + 0.3 * np.cos(ang), 0.5 + 0.3 * np.sin(ang), 0.1 + 0.02 * rng.normal(size=320)]))
    tris += [(centre, rim[k], rim[(k + 1) % 320]) for k in range(320)]
    n = centre + 321
    v.append(np.array([[3.0, 0, 0], [3.1, 0, 0], [3.0, 0.1, 0.02], [3.0, -0.1, 0.01], [3.05, 0.05, 0.1], [3.05, -0.05, -0.1]]))
    tris += [(n, n + 1, n + 2), (n + 1, n, n + 3), (n, n + 1, n + 4), (n + 1, n, n + 5)]        # edge (n, n+1) in 4 triangles
    tris += [(5, 5, 6), (7, 8, 7), (9, 9, 9)]                                               # degenerate
    tris += [tris[10], tris[11], tris[10]]                                                  # duplicates
    v.append(rng.uniform(4, 5, (13, 3)))                                                    # isolated
    verts = np.concatenate(v).astype(np.float32)
    assert len(verts) % 128 and len(verts) % 256
    return verts, np.array(tris, np.uint64)


def test_mesh_reference_bounds_hold_the_f32_oracle():
    """CPU: the bound is not too tight: oracle/postprocess.py (f32, its own order of sums) lies inside it."""
    from oracle import postprocess as pp
    v, t = built_mesh()
    off, adj = csr(t, len(v))
    w = np.random.default_rng(2).uniform(0, 1, len(v)).astype(np.float32)
    for it in (1, 2, 5):
        check(pp.laplacian_smoothing(v, off, adj, it, 0.7, w), laplacian(v, off, adj, it, 0.7, w), what="laplacian", min_judged=1.0)
    n = pp.vertex_normals(v, t)
    an = area_normals(v, t)
    check(n, an, np.isnan(an.v).any(1), "area normals")
    n0 = np.nan_to_num(n).astype(np.float32)
    for it in (1, 3):
        ref = smooth_normals(n0, off, adj, it)
        check(pp.laplacian_smoothing_normals(n0, off, adj, it), ref, np.isnan(ref.v).any(1), "normal smoothing")
    # and the same on the surface of a reconstruction, with the particle sums
    x = _splash()
    import oracle as om
    o = om.reconstruct(x, particle_radius=R_, smoothing_length=2.0, cube_size=0.6)
    _, h, _ = om.absolute_params(R_, 2.0, 0.6)
    mass = om.sph_rest_mass(R_)
    ref = Ref(x, o["particle_densities"], mass, h, o["vertices"])
    check(pp.weighted_neighbor_counts(x, h), weighted_neighbor_counts(x, h), what="wnc", min_judged=1.0)
    vals = (x[:, 0] * 3 - 1).astype(np.float32)
    for corr in (True, False):
        r, nan = ref.interpolate(vals, corr)
        check(pp.interpolate_quantity(x, o["particle_densities"], mass, h, vals, o["vertices"], corr), r, nan, "interpolate", 0.99)
    nrm, nan = ref.normals()
    check(om.sph_normals(x, o["particle_densities"], o["vertices"], compact_support_radius=h, particle_rest_mass=mass), nrm, nan, "normals", 0.99)
    wnn, nan = ref.interpolate(weighted_neighbor_counts(x, h), True)
    check(pp.smoothing_weights(pp.interpolate_quantity(x, o["particle_densities"], mass, h, pp.weighted_neighbor_counts(x, h), o["vertices"], True),
                               13.0), smoothstep(E(wnn.v[:, 0], wnn.e[:, 0], wnn.out[:, 0]), 13.0), None, "sw", 0.99)


def test_mesh_reference_is_sensitive():
    """CPU: the bounds of the mesh reference are tight enough to see one lost neighbour, and the buffer swap of the smoothing."""
    v, t = built_mesh()
    off, adj = csr(t, len(v))
    w = np.random.default_rng(3).uniform(0, 1, len(v)).astype(np.float32)
    ref = laplacian(v, off, adj, 3, 0.7, w)
    # the last neighbour of every vertex left out
    seg_keep = np.ones(len(adj), bool)
    seg_keep[off[1:][np.diff(off) > 0] - 1] = False
    off2 = np.r_[0, np.cumsum(np.bincount(np.repeat(np.arange(len(v)), np.diff(off))[seg_keep], minlength=len(v)))]
    assert outside(laplacian(v, off2, adj[seg_keep], 3, 0.7, w).v, ref, np.zeros(len(v), bool)).sum() > len(v) // 2
    # without the swap the neighbours come from the initial vertices in every iteration, and the blended vertex is the previous one
    seg, deg = np.repeat(np.arange(len(v)), np.diff(off)), np.diff(off)
    mean0 = np.zeros((len(v), 3))
    np.add.at(mean0, seg, v[adj].astype(np.float64))
    mean0 = np.where(deg[:, None] > 0, mean0 / np.maximum(deg, 1)[:, None], mean0)
    be = 0.7 * w.astype(np.float64)[:, None]
    cur = v.astype(np.float64)
    for _ in range(3):
        cur = cur * (1 - be) + mean0 * be
    assert outside(cur, ref, np.zeros(len(v), bool)).sum() > len(v) // 2


def check_mesh_kernels(lib, iterations, beta, weights):
    v, t = built_mesh()
    nv = len(v)
    off, adj = csr(t, nv)
    mesh = lib.TriMesh3d(v.copy(), t.copy())
    conn = mesh.vertex_vertex_connectivity()
    assert np.array_equal(conn.offsets.astype(np.int64), off) and np.array_equal(conn.indices.astype(np.int64), adj)
    w = {"zero": np.zeros(nv, np.float32), "one": np.ones(nv, np.float32),
         "random": np.random.default_rng(iterations).uniform(0, 1, nv).astype(np.float32)}[weights]
    lib.laplacian_smoothing_parallel(mesh, conn, iterations=iterations, beta=beta, weights=w)
    check(mesh.vertices, laplacian(v, off, adj, iterations, beta, w), what="laplacian", min_judged=1.0)
    n = mesh.vertex_normals_parallel()
    ref = area_normals(mesh.vertices, t)
    check(n, ref, np.isnan(ref.v).any(1), "area normals", 0.9)
    n0 = np.nan_to_num(n).astype(np.float32)
    for it in (0, 1, iterations):
        s = n0.copy()
        lib.laplacian_smoothing_normals_parallel(s, conn, iterations=it)
        ref = smooth_normals(n0, off, adj, it)
        check(s, ref, np.isnan(ref.v).any(1), f"normal smoothing {it}", 0.9)


MESH_SETTINGS = [(it, b, w) for it in range(8) for b in (0.0, 0.7, 1.0) for w in ("zero", "one", "random") if it in (0, 1, 2, 7) or b == 0.7]


# ------------------------------------------------------------------ smoothstep ----
def smoothstep_inputs():
    f = np.float32
    dense0 = np.nextafter(f(0), f(1), dtype=f) * np.arange(-50, 50, dtype=f)
    around = np.linspace(-1e-3, 1e-3, 301, dtype=f)
    norm = np.float32(13.0)
    at_norm = (norm + np.arange(-200, 200, dtype=f) * np.spacing(norm)).astype(f)
    sweep = np.linspace(-5, 30, 2001, dtype=f)
    special = np.array([np.inf, -np.inf, np.nan, -np.nan, np.finfo(f).tiny, -np.finfo(f).tiny, np.finfo(f).max, -np.finfo(f).max, 1e-40, -1e-40], f)
    return np.concatenate([dense0, around, at_norm, sweep, special]).astype(f)


def test_smoothstep_reference(oracle_mod):
    """CPU: the f32 oracle inside the bound (NaN counts included: Rust's max ignores NaN), and special values by their definition."""
    from oracle import postprocess as pp
    n = smoothstep_inputs()
    ref = smoothstep(n, 13.0)
    check(pp.smoothing_weights(n, 13.0), ref, None, "oracle smoothstep", 0.95, pp.smoothing_weights(n, 13.0))
    got = pp.smoothing_weights(np.array([np.nan, np.inf, -np.inf, -1.0], np.float32), 13.0)
    assert got.tolist() == [0.0, 1.0, 0.0, 0.0]


def check_smoothstep(emul):
    """k_pp_smoothstep on chosen counts (the kernel stepped by the executor of tests/emul/post_emul.cpp).  On the device the same
    kernel sees the interpolated counts of the probe scenes, NaN (points without particles) included."""
    n = smoothstep_inputs()
    out = np.empty_like(n)
    emul.emul_smoothstep(C.c_uint32(len(n)), C.c_void_p(n.ctypes.data), C.c_float(13.0), C.c_void_p(out.ctypes.data))
    from oracle import postprocess as pp
    check(out, smoothstep(n, 13.0), None, "k_pp_smoothstep", 0.95, pp.smoothing_weights(n, 13.0))
    assert np.isfinite(out).all()


# ------------------------------------------------------------------ H100 ----
@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PROBE_PATHS))
def test_cuda_sole_neighbour_probes(ss, oracle_mod, path):
    run_probe_scene(ss, oracle_mod, path)


@pytest.mark.gpu
@pytest.mark.parametrize("k", K_ALL)
def test_cuda_sole_neighbour_probes_at_scale(ss, oracle_mod, k):
    assert_window("probe", k, run_probe_scene(ss, oracle_mod, "S16", k=k))


@pytest.mark.gpu
@pytest.mark.parametrize("band,sign", OFFSETS)
def test_cuda_sole_neighbour_probes_at_offset(ss, oracle_mod, band, sign):
    assert_window("probe", 0, run_probe_scene(ss, oracle_mod, "S16", band=band, sign=sign))


@pytest.mark.gpu
@pytest.mark.parametrize("k", K_ALL)
def test_cuda_interpolator_probes_at_scale(ss, oracle_mod, k):
    assert_window("interpolator", k, run_interpolator(ss, oracle_mod, k))


@pytest.mark.gpu
@pytest.mark.parametrize("band,sign", OFFSETS)
def test_cuda_interpolator_probes_at_offset(ss, oracle_mod, band, sign):
    assert_window("interpolator", 0, run_interpolator(ss, oracle_mod, band=band, sign=sign))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(NORMAL_CASES))
def test_cuda_sph_normals_every_vertex(ss, oracle_mod, name):
    check_vertex_normals(ss, oracle_mod, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["R1", "R9"])
@pytest.mark.parametrize("k", K_ALL)
def test_cuda_sph_normals_every_vertex_at_scale(ss, oracle_mod, name, k):
    assert_window("vertices", k, check_vertex_normals(ss, oracle_mod, name, k=k))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["R1", "R9"])
@pytest.mark.parametrize("band,sign", OFFSETS)
def test_cuda_sph_normals_every_vertex_at_offset(ss, oracle_mod, name, band, sign):
    assert_window("vertices", 0, check_vertex_normals(ss, oracle_mod, name, band=band, sign=sign))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PIPELINE_CASES))
def test_cuda_pipeline(ss, case):
    check_device_pipeline(ss, case)


@pytest.mark.gpu
@pytest.mark.parametrize("iterations,beta,weights", MESH_SETTINGS)
def test_cuda_mesh_kernels(ss, iterations, beta, weights):
    check_mesh_kernels(ss, iterations, beta, weights)


# ------------------------------------------------------------------ CPU executor ----
@pytest.mark.parametrize("path", list(PROBE_PATHS))
def test_emulated_sole_neighbour_probes(emu, oracle_mod, path):
    run_probe_scene(emu, oracle_mod, path)


@pytest.mark.parametrize("k", K_SOME + [-36, 36])
def test_emulated_sole_neighbour_probes_at_scale(emu, oracle_mod, k):
    assert_window("probe", k, run_probe_scene(emu, oracle_mod, "S16", k=k))


@pytest.mark.parametrize("band,sign", OFFSETS)
def test_emulated_sole_neighbour_probes_at_offset(emu, oracle_mod, band, sign):
    assert_window("probe", 0, run_probe_scene(emu, oracle_mod, "S16", band=band, sign=sign))


@pytest.mark.parametrize("k", K_ALL)
def test_emulated_interpolator_probes_at_scale(emu, oracle_mod, k):
    assert_window("interpolator", k, run_interpolator(emu, oracle_mod, k))


@pytest.mark.parametrize("band,sign", OFFSETS)
def test_emulated_interpolator_probes_at_offset(emu, oracle_mod, band, sign):
    assert_window("interpolator", 0, run_interpolator(emu, oracle_mod, band=band, sign=sign))


@pytest.mark.parametrize("name", list(NORMAL_CASES))
def test_emulated_sph_normals_every_vertex(emu, oracle_mod, name):
    check_vertex_normals(emu, oracle_mod, name)


@pytest.mark.parametrize("name", ["R1", "R9"])
@pytest.mark.parametrize("k", K_SOME + [-36, 36])
def test_emulated_sph_normals_every_vertex_at_scale(emu, oracle_mod, name, k):
    assert_window("vertices", k, check_vertex_normals(emu, oracle_mod, name, k=k))


@pytest.mark.parametrize("name", ["R1", "R9"])
@pytest.mark.parametrize("band,sign", OFFSETS)
def test_emulated_sph_normals_every_vertex_at_offset(emu, oracle_mod, name, band, sign):
    assert_window("vertices", 0, check_vertex_normals(emu, oracle_mod, name, band=band, sign=sign))


@pytest.mark.parametrize("case", list(PIPELINE_CASES))
def test_emulated_pipeline(emu, case):
    check_device_pipeline(emu, case)


@pytest.mark.parametrize("iterations,beta,weights", [(0, 1.0, "one"), (1, 0.7, "random"), (2, 1.0, "one"), (5, 0.7, "random"), (7, 1.0, "zero"),
                                                     (4, 0.0, "random")])
def test_emulated_mesh_kernels(emu, iterations, beta, weights):
    check_mesh_kernels(emu, iterations, beta, weights)


def test_emulated_smoothstep(emul):
    check_smoothstep(emul)
