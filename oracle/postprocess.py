"""CPU restatement of the reference's mesh post-processing steps (SURVEY §8f) -- TEST INFRASTRUCTURE ONLY.

numpy/scipy restatements of the steps `splashsurf reconstruct` runs on the reconstructed mesh
(splashsurf/src/reconstruct.rs:1094-1391), all in f32 like the reference's `R = f32` instantiation:

* `vertex_vertex_connectivity`       splashsurf_lib/src/mesh.rs:290-306
* `laplacian_smoothing`              splashsurf_lib/src/postprocessing.rs:17-53
* `laplacian_smoothing_normals`      splashsurf_lib/src/postprocessing.rs:56-97
* `vertex_normals`                   splashsurf_lib/src/mesh.rs:799-838, :888-906
* `interpolate_quantity`             splashsurf_lib/src/sph_interpolation.rs:210-258
* `weighted_neighbor_counts`         splashsurf/src/reconstruct.rs:1168-1205
* `smoothing_weights`                splashsurf/src/reconstruct.rs:1220-1231
* `pipeline`                         the order of the steps, reconstruct.rs:1094-1391

Parity status: PINNED against the reference wheel (tests/test_oracle_postprocess.py, tests/golden/postprocess_ref.npz).
Sums over neighbours run in a different order than the reference's (hash / R-tree order there), so parity is to f32
round-off (tests state 2e-5 relative), not bit-exact.
"""
from __future__ import annotations

import numpy as np

F = np.float32


# ------------------------------------------------------------------ connectivity ----
def vertex_vertex_connectivity(triangles: np.ndarray, nv: int):
    """CSR (offsets[nv+1], neighbours) of the unique neighbours of every vertex, in the reference's order of first
    appearance while walking the triangles (mesh.rs:295-303)."""
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    a, b, c = t[:, 0], t[:, 1], t[:, 2]
    src = np.stack([a, a, b, b, c, c], axis=1).ravel()
    dst = np.stack([b, c, a, c, a, b], axis=1).ravel()
    keep = src != dst
    src, dst = src[keep], dst[keep]
    key = src * np.int64(nv) + dst
    _, first = np.unique(key, return_index=True)
    first.sort()                                   # order of first appearance
    src, dst = src[first], dst[first]
    order = np.argsort(src, kind="stable")
    src, dst = src[order], dst[order]
    off = np.zeros(nv + 1, dtype=np.int64)
    np.add.at(off, src + 1, 1)
    return np.cumsum(off), dst


def _neighbor_sum(values: np.ndarray, off: np.ndarray, adj: np.ndarray) -> np.ndarray:
    """Sequential f32 sum of values[adj[...]] per row, neighbour by neighbour (left fold like the reference's loop)."""
    nv = len(off) - 1
    deg = np.diff(off)
    out = np.zeros((nv,) + values.shape[1:], dtype=F)
    for k in range(int(deg.max()) if nv else 0):
        rows = np.nonzero(deg > k)[0]
        out[rows] = (out[rows] + values[adj[off[rows] + k]]).astype(F)
    return out


# ------------------------------------------------------------------ smoothing ----
def laplacian_smoothing(vertices, off, adj, iterations: int, beta: float, weights) -> np.ndarray:
    """postprocessing.rs:17-53.  NOTE the buffer swap at :31: the vertex that is blended with the neighbour mean is the
    one from TWO iterations ago (the initial one in iterations 1 and 2), the neighbour mean is taken from the previous
    iteration.  This restatement follows that behaviour (pinned against the wheel)."""
    cur = np.ascontiguousarray(vertices, dtype=F).copy()          # mesh.vertices
    buf = cur.copy()                                               # vertex_buffer
    w = np.asarray(weights, dtype=F)
    deg = np.diff(off).astype(np.int64)
    has = deg > 0
    n = deg.astype(F)
    for _ in range(iterations):
        cur, buf = buf, cur                                        # :31 swap: `cur` is written, `buf` is read
        beta_eff = (F(beta) * w).astype(F)
        vsum = _neighbor_sum(buf, off, adj)
        vsum[has] = (vsum[has] / n[has, None]).astype(F)
        one_minus = (F(1.0) - beta_eff).astype(F)
        cur[:] = ((cur * one_minus[:, None]).astype(F) + (vsum * beta_eff[:, None]).astype(F)).astype(F)
    return cur


def laplacian_smoothing_normals(normals, off, adj, iterations: int) -> np.ndarray:
    """postprocessing.rs:56-97: n_i <- normalize(sum_j n_j) over the neighbours (the vertex itself is not included)."""
    cur = np.ascontiguousarray(normals, dtype=F).copy()
    for _ in range(iterations):
        s = _neighbor_sum(cur, off, adj)
        nrm = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]).astype(F) + (s[:, 2] * s[:, 2]).astype(F)).astype(F)
        with np.errstate(invalid="ignore", divide="ignore"):
            cur = (s / nrm[:, None]).astype(F)
    return cur


def vertex_normals(vertices, triangles) -> np.ndarray:
    """Area-weighted vertex normals, mesh.rs:812-821 + :899-905 (cross((v1-v0), (v2-v1)) added to the three corners)."""
    v = np.ascontiguousarray(vertices, dtype=F)
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    n = np.cross((v[t[:, 1]] - v[t[:, 0]]).astype(F), (v[t[:, 2]] - v[t[:, 1]]).astype(F)).astype(F)
    acc = np.zeros_like(v, dtype=np.float64)
    for k in range(3):
        np.add.at(acc, t[:, k], n.astype(np.float64))
    acc = acc.astype(F)
    nrm = np.sqrt((acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1] + acc[:, 2] * acc[:, 2]).astype(F)).astype(F)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (acc / nrm[:, None]).astype(F)


# ------------------------------------------------------------------ SPH interpolation ----
def _kernel(r: np.ndarray, h: float) -> np.ndarray:
    """CubicSplineKernel::evaluate, kernel.rs:73-107 (f32)."""
    r = r.astype(F)
    hh = F(h)
    q = ((r + r) / hh).astype(F)
    sigma = F(8.0) / (hh * hh * hh)
    inner = F(3.0 / (2.0 * np.pi)) * (F(2.0 / 3.0) - q * q + F(0.5) * q * q * q)
    x = (F(2.0) - q)
    outer = F(1.0 / (4.0 * np.pi)) * x * x * x
    f = np.where(q < 1.0, inner, np.where(q < 2.0, outer, F(0.0))).astype(F)
    return (sigma * f).astype(F)


def sphere_rest_mass(particle_radius: float, rest_density: float) -> np.float32:
    """reconstruct.rs:1126-1129: 4 * (pi/3) * r^3 * rho0 in f32."""
    r = F(particle_radius)
    return F(F(F(4.0) * F(np.pi / 3.0)) * F(r * r * r) * F(rest_density))


def _pairs_within(points, particles, radius):
    from scipy.spatial import cKDTree
    tree = cKDTree(np.asarray(particles, dtype=np.float64))
    lists = tree.query_ball_point(np.asarray(points, dtype=np.float64), r=float(radius) * (1.0 + 1e-6))
    cnt = np.fromiter((len(l) for l in lists), dtype=np.int64, count=len(lists))
    i = np.repeat(np.arange(len(lists), dtype=np.int64), cnt)
    j = np.fromiter((q for l in lists for q in l), dtype=np.int64, count=int(cnt.sum()))
    return i, j


def interpolate_quantity(particles, densities, rest_mass, h, values, points, first_order_correction=True) -> np.ndarray:
    """sph_interpolation.rs:210-258: sum_j A_j (V_j W_ij), V_j = m / rho_j, optionally divided by sum_j V_j W_ij;
    particles with |x_j - x_i|^2 <= h^2 (rstar locate_within_distance)."""
    x = np.ascontiguousarray(particles, dtype=F)
    p = np.ascontiguousarray(points, dtype=F)
    a = np.asarray(values, dtype=F)
    vec = a.ndim == 2
    a2 = a if vec else a[:, None]
    i, j = _pairs_within(p, x, h)
    d = (x[j] - p[i]).astype(F)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(F)
    ok = d2 <= F(h) * F(h)
    i, j, d2 = i[ok], j[ok], d2[ok]
    w = ((F(rest_mass) / np.asarray(densities, dtype=F)[j]).astype(F) * _kernel(np.sqrt(d2).astype(F), h)).astype(F)
    num = np.zeros((len(p), a2.shape[1]), dtype=np.float64)
    np.add.at(num, i, (a2[j] * w[:, None]).astype(np.float64))
    corr = np.zeros(len(p), dtype=np.float64)
    np.add.at(corr, i, w.astype(np.float64))
    num = num.astype(F)
    with np.errstate(invalid="ignore", divide="ignore"):
        if first_order_correction:
            num = (num * (F(1.0) / corr.astype(F))[:, None]).astype(F)
        else:                                      # :252-254: 0 * (1 / 0) + 1 is NaN for an empty sum as well
            num[corr.astype(F) == 0] = np.nan
    return num if vec else num[:, 0]


def weighted_neighbor_counts(particles, h) -> np.ndarray:
    """reconstruct.rs:1190-1205: sum over the neighbours j != i with d^2 < h^2 of 1 - clamp(d^2 / h^2, 0, 1)."""
    x = np.ascontiguousarray(particles, dtype=F)
    i, j = _pairs_within(x, x, h)
    keep = i != j
    i, j = i[keep], j[keep]
    d = (x[i] - x[j]).astype(F)
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(F)
    h2 = F(h) * F(h)
    ok = d2 < h2
    term = (F(1.0) - np.clip((d2[ok] / h2).astype(F), F(0.0), F(1.0))).astype(F)
    out = np.zeros(len(x), dtype=np.float64)
    np.add.at(out, i[ok], term.astype(np.float64))
    return out.astype(F)


def smoothing_weights(vertex_weighted_num_neighbors, normalization: float) -> np.ndarray:
    """reconstruct.rs:1220-1231: x = min(max(n - 0, 0) / normalization, 1); 6 x^5 - 15 x^4 + 10 x^3.  Rust's f32::max ignores
    NaN (NaN.max(0) = 0), so a NaN count (a vertex without particles in range) gets the weight 0: np.fmax, not np.maximum."""
    n = np.asarray(vertex_weighted_num_neighbors, dtype=F)
    x = np.minimum((np.fmax(n, F(0.0)) / F(normalization)).astype(F), F(1.0)).astype(F)
    x3 = (x * x * x).astype(F); x4 = (x3 * x).astype(F); x5 = (x4 * x).astype(F)
    return ((x5 * F(6.0)).astype(F) - (x4 * F(15.0)).astype(F) + (x3 * F(10.0)).astype(F)).astype(F)


# ------------------------------------------------------------------ the pipeline's order of steps ----
def pipeline(particles, densities, vertices, triangles, *, particle_radius, rest_density, compact_support_radius,
             mesh_smoothing_weights=True, mesh_smoothing_weights_normalization=13.0, mesh_smoothing_iters=None,
             compute_normals=False, sph_normals=False, normals_smoothing_iters=None, attributes=None,
             sph_normals_fn=None) -> dict:
    """reconstruct.rs:1094-1391 without cleanup / decimation / clamping / quads: weights at the raw vertices, smoothing,
    then normals and attribute interpolation at the smoothed vertices.  `particles`/`densities` are the filtered ones."""
    out = {}
    v = np.ascontiguousarray(vertices, dtype=F)
    nv = len(v)
    m = sphere_rest_mass(particle_radius, rest_density)
    h = float(compact_support_radius)
    off = adj = None
    if normals_smoothing_iters is not None or mesh_smoothing_iters is not None:
        off, adj = vertex_vertex_connectivity(triangles, nv)
    weights = None
    if mesh_smoothing_weights:
        wn = weighted_neighbor_counts(particles, h)
        wnn = interpolate_quantity(particles, densities, m, h, wn, v, True)
        weights = smoothing_weights(wnn, mesh_smoothing_weights_normalization)
        out["wnn"], out["sw"] = wnn, weights
    if mesh_smoothing_iters is not None:
        w = weights if weights is not None else np.ones(nv, dtype=F)
        v = laplacian_smoothing(v, off, adj, int(mesh_smoothing_iters), 1.0, w)
    out["vertices"] = v
    if compute_normals:
        if sph_normals:
            raw = sph_normals_fn(particles, densities, v, compact_support_radius=h, particle_rest_mass=float(m))
        else:
            raw = vertex_normals(v, triangles)
        if normals_smoothing_iters is not None:
            out["normals"] = laplacian_smoothing_normals(raw, off, adj, int(normals_smoothing_iters))
            out["raw_normals"] = raw
        else:
            out["normals"] = raw
    for name, a in (attributes or {}).items():
        out[name] = interpolate_quantity(particles, densities, m, h, a, v, True)
    return out
