"""Averaged-position surface (Zhu & Bridson 2005; splashsurf_b200.AveragedSurface, DESIGN.md section 12).

* the plain-C restatement (tests/averaged_oracle.c, built on the pinned oracle) against an independent float64 numpy restatement of
  the definition, within a per-point rounding bound derived below, plus properties of the definition;
* the device pipeline on the CPU executor of the CUDA sources (tests/emul) against the oracle, bit for bit: mesh, densities (also
  equal to the standard run's) and the kept level-set tile; every tier of the warp-per-brick cascade is reached;
* refusals, the command line, and the surface quality measured on the oracle.
The GPU-marked counterpart of the device cases is tests/test_zzz_gpu_averaged_surface.py."""
import ctypes as C
import os

import numpy as np
import pytest

import c_oracle
from test_anisotropic import KW, R, _aniso_params, _clustered, _cube, _lattice, _sphere, _splash
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

H = 4 * R                      # compact support radius of KW
EPS = 2.0 ** -24               # unit roundoff of f32

# ------------------------------------------------------------------ the averaged oracle (tests/averaged_oracle.c) ----
def _avg_lib():
    """tests/averaged_oracle.c (it includes the pinned oracle/splashsurf_oracle.c unchanged) with its entry point bound."""
    from oracle import _Params, _Result
    return c_oracle.build("averaged_oracle.c", {
        "so_reconstruct_averaged": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(_Params), C.c_float, C.POINTER(C.POINTER(_Result)),
                                              C.c_int64, C.c_void_p]),
        "so_free": (None, [C.POINTER(_Result)])})


def oracle_reconstruct_averaged(particles, *, particle_radius, smoothing_length, cube_size, rest_density=1000.0, iso_surface_threshold=0.6,
                                aabb_min=None, aabb_max=None, subdomain_grid=True, subdomain_num_cubes_per_dim=64, radius_factor=1.0,
                                tile_of_subdomain=None, **_ignored):
    """C-oracle reconstruction with the averaged-position surface (DESIGN.md section 12): the dict of `reconstruct` (plus "tile" when
    `tile_of_subdomain` is given), or {"rc": code} on a refusal.  Always decomposed."""
    from oracle import _Result, _grid_dict
    L = _avg_lib()
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    p = _aniso_params(particle_radius, smoothing_length, cube_size, rest_density, iso_surface_threshold, aabb_min, aabb_max,
                      subdomain_grid, subdomain_num_cubes_per_dim)
    S = int(subdomain_num_cubes_per_dim)
    tile = np.zeros((S + 1,) * 3, dtype=np.float32) if tile_of_subdomain is not None else None
    out = C.POINTER(_Result)()
    rc = L.so_reconstruct_averaged(xyz.ctypes.data, len(xyz), C.byref(p), float(np.float32(radius_factor)), C.byref(out),
                                   -1 if tile_of_subdomain is None else int(tile_of_subdomain), None if tile is None else tile.ctypes.data)
    try:
        if rc != 0:
            return {"rc": rc}
        res = out.contents
        n = res.n_filtered
        nv, nt, ns = res.nv, res.nt, res.n_subdomains
        d = {"rc": rc, "grid": _grid_dict(res.grid), "used_decomposition": bool(res.used_decomposition),
             "subdomain_grid": _grid_dict(res.subdomain_grid)}
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


def _busiest_tile(o):
    """Flat index of the subdomain with the most members (None without subdomains)."""
    f = o["subdomain_flat"]
    return int(f[int(np.argmax(o["subdomain_count"]))]) if len(f) else None


def _tile_points(o, flat, S):
    """f32 coordinates of the (S + 1)^3 grid points of subdomain `flat`, min + index * cell as the kernels compute them."""
    sg, gg = o["subdomain_grid"], o["grid"]
    nsd = sg["ncells"]
    ijk = np.array([flat // (nsd[1] * nsd[2]), (flat // nsd[2]) % nsd[1], flat % nsd[2]])
    idx = np.stack(np.meshgrid(*[np.arange(S + 1)] * 3, indexing="ij"), -1).reshape(-1, 3) + ijk * S
    gmin = np.asarray(gg["aabb_min"], np.float32)
    return gmin + idx.astype(np.float32) * np.float32(gg["cell_size"])


# ------------------------------------------------------------------ float64 restatement ----
def numpy_averaged(p, pts, h):
    """f(g) of DESIGN.md section 12 in float64 at the points `pts` (brute-force neighbours), the number n of particles within
    h (1 + 1e-6) of each point (the terms an f32 evaluation may count) and a bound on |f32 fold - f| per point.

    The bound (u = 2^-24, every term first order, the sum enlarged by a quarter for the second-order terms):
    * weights: with |d| <= h, d^2 carries 7 u h^2, q = d^2 / h^2 9 u q, the base b = 1 - q 9 u q + u b (1 - q is exact for q >= 1/2),
      w = b^3 three times the base's error times b^2 plus two roundings: dw_j <= u (27 b^2 q + 5 w).  A candidate whose f32
      membership can flip (|q - 1| < 20 u) has w <= (10 u)^3; that is added to such candidates.  Weight errors move the
      average x_bar = sum w d / S by sum dw_j (d_j - x_bar) / S', S' the perturbed sum >= S - sum dw_j -- relative errors of the
      weights cancel between numerator and denominator, so a lone candidate at the edge of the support costs nothing.  When
      S - sum dw_j <= 0 only |x_bar' - x_bar| <= 2 h (two convex combinations of points within h) is claimed.  With one candidate
      x_bar is its offset whatever its weight; if f32 drops it (ambiguous), f = 0 against h - |d| <= 20 u h.
    * offsets and products: u |d| + u w |d| per term, u h after dividing by S; the n additions of each sum: n u h on the
      numerator, n u |x_bar| <= n u h through the denominator;
    * value: three divisions, the squares and sums, the square root and h - ...: 6 u h.
    Where no particle is within h both are exactly 0."""
    from scipy.spatial import cKDTree
    u = EPS
    x = p.astype(np.float64)
    g = pts.astype(np.float64)
    f, n, bound = np.zeros(len(g)), np.zeros(len(g), int), np.zeros(len(g))
    if not len(x):
        return f, n, bound
    tree = cKDTree(x)
    for q, nb in enumerate(tree.query_ball_point(g, h * (1 + 1e-6))):
        n[q] = len(nb)
        if not nb:
            continue
        d = x[nb] - g[q]
        qq = (d * d).sum(1) / (h * h)
        base = np.where(qq < 1.0, 1.0 - qq, 0.0)
        w = base ** 3
        S = w.sum()
        xb = (w[:, None] * d).sum(0) / S if S > 0 else np.zeros(3)
        if S > 0:
            f[q] = h - np.linalg.norm(xb)
        dw = u * (27.0 * base * base * qq + 5.0 * w) + np.where(np.abs(qq - 1.0) < 20 * u, (10.0 * u) ** 3, 0.0)
        low = S - dw.sum()
        if n[q] == 1:
            move = 20 * u * h
        else:
            move = 2.0 * h if low <= 0 else min(2.0 * h, float((dw * np.linalg.norm(d - xb, axis=1)).sum()) / low)
        bound[q] = 1.25 * (move + u * h * (2 * n[q] + 8))
    return f, n, bound


ORACLE_CLOUDS = {
    "jittered_lattice": lambda: _cube(9, 701),
    "sphere": lambda: _sphere(5, 702),
    "slab": lambda: _lattice(14, 3, 14, 0.25, 703),
    "sparse_droplets": lambda: _splash((6, 3, 6), 5, 704),
}


@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_oracle_levelset_matches_float64_restatement(name):
    """The oracle's tile of one subdomain against f(g) in float64, point by point within the bound of numpy_averaged."""
    from oracle import absolute_params
    p = ORACLE_CLOUDS[name]()
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    flat = _busiest_tile(oracle_reconstruct_averaged(p, **kw))
    o = oracle_reconstruct_averaged(p, tile_of_subdomain=flat, **kw)
    h = float(absolute_params(R, 2.0, 0.5)[1])
    pts = _tile_points(o, flat, S)
    f, n, bound = numpy_averaged(p, pts, h)
    tile = o["tile"].reshape(-1).astype(np.float64)
    assert np.all(tile[n == 0] == 0.0)
    m = n > 0
    assert m.sum() > 100
    err = np.abs(tile[m] - f[m])
    assert np.all(err <= bound[m]), (err.max(), bound[m][np.argmax(err / bound[m])])
    assert np.median(bound[m]) < 1e-5 * h                            # the bound is tight where the weights are not all at the edge
    assert tile.min() >= -8 * np.spacing(np.float32(h))              # a convex combination of particles within h: f >= 0 up to rounding


def test_one_particle_is_a_sphere_of_radius_r_s():
    """One particle: f = h - |g - p| to a few ulp at every point within h, and every mesh vertex within c^2 / R_s (+ rounding) of the
    sphere of radius R_s, radially.  Bound: along a crossing edge (length c, axis-aligned) phi(t) = |x(t) - p| is convex with
    phi'' <= 1 / r, and r >= R_s - c on it (else both end points lie within R_s); marching cubes puts the vertex where the chord of
    phi meets R_s, where phi lies below the chord by at most c^2 / 8 / (R_s - c) <= 0.43 c^2 / R_s for c <= R_s / sqrt(2); |grad phi|
    = 1 turns that into the radial distance.  Rounding of f moves a vertex radially by about the error of f."""
    from oracle import absolute_params
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    r, h, c = (float(v) for v in absolute_params(R, 2.0, 0.5))
    rs = float(np.float32(1.0) * np.float32(r))
    assert c <= rs / np.sqrt(2.0)
    flat = _busiest_tile(oracle_reconstruct_averaged(p, **kw))
    o = oracle_reconstruct_averaged(p, tile_of_subdomain=flat, **kw)
    pts = _tile_points(o, flat, 16).astype(np.float64)
    dist = np.linalg.norm(pts - p[0].astype(np.float64), axis=1)
    tile = o["tile"].reshape(-1).astype(np.float64)
    within = dist < h * (1 - 1e-6)
    assert within.sum() > 100
    assert np.abs(tile[within] - (h - dist[within])).max() <= 8 * np.spacing(np.float32(h))
    assert np.all(tile[dist > h * (1 + 1e-6)] == 0.0)
    v = o["vertices"].astype(np.float64)
    assert len(v) > 50
    rad = np.linalg.norm(v - p[0].astype(np.float64), axis=1)
    slack = 32 * float(np.spacing(np.float32(h))) + 8 * float(np.spacing(np.float32(np.abs(v).max())))
    assert np.all(rad <= rs + slack) and np.all(rad >= rs - c * c / rs - slack), (rad.min(), rad.max(), rs)


# ------------------------------------------------------------------ a candidate at the edge of the support ----
SHELL_KW = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5, subdomain_num_cubes_per_dim=64)


def _shell_point(o, p):
    """Flat tile index and f32 coordinates of the grid points of the busiest tile of `o` at which particle p has
    fl(d2 / h2) = 1 - 2^-24 in the kernels' operation order (weight 2^-72, the smallest a candidate can have)."""
    from oracle import absolute_params
    h = np.float32(absolute_params(SHELL_KW["particle_radius"], 2.0, 0.5)[1])
    flat = _busiest_tile(o)
    g = _tile_points(o, flat, SHELL_KW["subdomain_num_cubes_per_dim"])
    d = p[None, :] - g
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    q = d2 / (h * h)
    return flat, np.nonzero(q == np.float32(1.0) - np.float32(2.0 ** -24))[0], g


def _edge_shell_particle():
    """One particle at r = 0.01 (h = 0.04) placed so that a grid point lies in the outermost f32 shell of its support: about h from
    that point along x, with its x coordinate stepped by ulps and its y coordinate by ulps off the grid line (a fine step of d2)."""
    from oracle import absolute_params
    h = np.float32(absolute_params(0.01, 2.0, 0.5)[1])
    target = np.float32(1.0) - np.float32(2.0 ** -24)
    p = np.array([0.1, 0.2, 0.3], np.float32)
    for _ in range(4):
        o = oracle_reconstruct_averaged(p[None], **SHELL_KW)
        if len(_shell_point(o, p)[1]):
            return p
        gmin, c = np.asarray(o["grid"]["aabb_min"], np.float32), np.float32(o["grid"]["cell_size"])
        gp = gmin + np.round((p - gmin) / c).astype(np.float32) * c          # a grid point near p (f32, as the kernels compute it)
        gp[0] = gmin[0] + np.float32(np.round((p[0] - h - gmin[0]) / c)) * c
        ys = (np.int32(gp[1].view(np.int32)) + np.arange(20000, dtype=np.int32)).view(np.float32)
        dy = ys - gp[1]
        x0 = np.float32(gp[0] + h).view(np.int32)
        for k in range(-40, 1):
            x = np.int32(x0 + k).view(np.float32)
            dx = np.float32(x - gp[0])
            q = ((dx * dx + dy * dy) + np.float32(0.0)) / (h * h)
            hit = np.nonzero(q == target)[0]
            if len(hit):
                p = np.array([x, ys[hit[0]], gp[2]], np.float32)
                break
    raise AssertionError("no grid point in the outermost shell")


def test_candidate_at_the_edge_of_the_support_stays_outside():
    """A grid point whose only candidate has weight 2^-72: the raw sums X = w dx are about 1e-23, their squares underflow, so a norm
    of the raw sums read f = h (inside) there and made a closed blob about h from the particle.  The norm of the averaged offset
    gives f = h - |d|, about 0: one closed sphere of radius R_s, equal to the float64 value within its bound."""
    from oracle import absolute_params
    p = _edge_shell_particle()
    o = oracle_reconstruct_averaged(p[None], tile_of_subdomain=None, **SHELL_KW)
    flat, hit, g = _shell_point(o, p)
    assert len(hit)
    o = oracle_reconstruct_averaged(p[None], tile_of_subdomain=flat, **SHELL_KW)
    r, h, c = (float(v) for v in absolute_params(0.01, 2.0, 0.5))
    tile = o["tile"].reshape(-1)
    f, n, bound = numpy_averaged(p[None], g[hit], h)
    assert np.all(n == 1) and np.all(np.abs(tile[hit].astype(np.float64) - f) <= bound) and np.all(tile[hit] < 1e-6 * h)
    ncomp, closed, chi = mesh_topology(o["triangles"])
    assert (ncomp, closed, chi) == (1, True, [2])
    rad = np.linalg.norm(o["vertices"].astype(np.float64) - p.astype(np.float64), axis=1)
    assert rad.max() <= r * (1 + 1e-4)


def test_isolated_particles_give_one_sphere_each():
    """4096 particles at r = 0.01 on a jittered lattice of spacing 0.12 > 2 (h + c): one closed sphere per particle and nothing else.
    The jitter places the grid points at many different offsets from the particles."""
    rng = np.random.default_rng(709)
    g = np.stack(np.meshgrid(*[np.arange(16)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.12
    p = (g + rng.uniform(-0.005, 0.005, g.shape)).astype(np.float32)
    o = oracle_reconstruct_averaged(p, **SHELL_KW)
    ncomp, closed, chi = mesh_topology(o["triangles"])
    assert ncomp == len(p) and closed and set(chi) == {2}


# ------------------------------------------------------------------ mesh topology ----
def mesh_topology(tris):
    """(components, closed, euler characteristic per component) of a triangle mesh: closed = every edge in exactly two triangles."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = np.asarray(tris, np.int64)
    if not len(t):
        return 0, True, []
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), axis=1)
    ue, cnt = np.unique(e, axis=0, return_counts=True)
    closed = bool(np.all(cnt == 2))
    used = np.unique(t)
    remap = -np.ones(t.max() + 1, np.int64)
    remap[used] = np.arange(len(used))
    a, b = remap[ue[:, 0]], remap[ue[:, 1]]
    ncomp, lab = connected_components(coo_matrix((np.ones(len(a)), (a, b)), shape=(len(used), len(used))), directed=False)
    chi = []
    tl = lab[remap[t[:, 0]]]
    el = lab[a]
    for k in range(ncomp):
        chi.append(int((lab == k).sum() - (el == k).sum() + (tl == k).sum()))
    return ncomp, closed, chi


def test_two_distant_particles_give_two_closed_components():
    from oracle import absolute_params
    r, h, c = (float(v) for v in absolute_params(R, 2.0, 0.5))
    p = np.array([[0.0, 0.0, 0.0], [2 * (h + c) * 1.05, 0.01, 0.0]], np.float32)
    o = oracle_reconstruct_averaged(p, **dict(KW, subdomain_num_cubes_per_dim=16))
    ncomp, closed, chi = mesh_topology(o["triangles"])
    assert ncomp == 2 and closed and chi == [2, 2]


def test_points_no_particle_reaches_are_zero():
    """Sparse droplets: every grid point of a tile without a particle within h is exactly 0 (outside, since t = h - R_s > 0)."""
    p = _splash((6, 3, 6), 5, 705)
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    o0 = oracle_reconstruct_averaged(p, **kw)
    from scipy.spatial import cKDTree
    tree = cKDTree(p.astype(np.float64))
    for flat in o0["subdomain_flat"][:: max(1, len(o0["subdomain_flat"]) // 4)]:
        o = oracle_reconstruct_averaged(p, tile_of_subdomain=int(flat), **kw)
        pts = _tile_points(o, int(flat), S).astype(np.float64)
        dmin, _ = tree.query(pts)
        far = dmin > H * (1 + 1e-6)
        assert far.any() and np.all(o["tile"].reshape(-1)[far] == 0.0)


# Measured on the oracle (ball of radius 9 d, lattice spacing d = 2 r, S = 32): at +-0.1 d jitter one closed component of euler
# characteristic 2; at +-0.25 d, where the anisotropic kernels open cavities inside the fluid, also one closed component, euler 2.
@pytest.mark.parametrize("jitter", [0.1, 0.25])
def test_jittered_ball_is_one_closed_sphere(jitter):
    p = _sphere(9, 706, jitter=jitter)
    o = oracle_reconstruct_averaged(p, **dict(KW, subdomain_num_cubes_per_dim=32))
    ncomp, closed, chi = mesh_topology(o["triangles"])
    assert (ncomp, closed, chi) == (1, True, [2]), (ncomp, closed, chi)


def test_oracle_refusals():
    p = _cube(5, 707)
    for rf in (0.0, -1.0, float("nan"), float("inf"), 4.0, 5.0):          # R_s = rf r must lie in (0, h = 4 r)
        assert oracle_reconstruct_averaged(p, radius_factor=rf, **KW)["rc"] == 6, rf
    assert oracle_reconstruct_averaged(p, subdomain_grid=False, **KW)["rc"] == 7
    assert oracle_reconstruct_averaged(p, radius_factor=3.9, **KW)["rc"] == 0


# ------------------------------------------------------------------ surface quality (oracle) ----
def test_quality_sphere_radii_spread():
    """Particle sphere (lattice jittered by +-0.1 d): the spread of the vertex radii drops against the standard mode.  Measured on the
    oracle: 0.00612 with AveragedSurface() against 0.00787 standard (ratio 0.777)."""
    import oracle
    p = _sphere(9, 609, jitter=0.1)
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    a = oracle_reconstruct_averaged(p, **kw)
    i = oracle.reconstruct(p, subdomain_grid_auto_disable=False, **kw)
    sa = np.linalg.norm(a["vertices"].astype(np.float64), axis=1).std()
    si = np.linalg.norm(i["vertices"].astype(np.float64), axis=1).std()
    assert sa < 0.85 * si, (sa, si)


def test_quality_slab_top_face_flatness():
    """Jittered slab (+-0.25 d): the spread of the heights of the top face's vertices (away from the edges) drops slightly against the
    standard mode.  Measured on the oracle: 0.00531 with AveragedSurface() against 0.00564 standard (ratio 0.941)."""
    import oracle
    p = _lattice(14, 3, 14, 0.25, 602)
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    a = oracle_reconstruct_averaged(p, **kw)
    i = oracle.reconstruct(p, subdomain_grid_auto_disable=False, **kw)

    def top_spread(v):
        v = v.astype(np.float64)
        mid = v[:, 1] > 0.05
        core = mid & (np.abs(v[:, 0] - 0.325) < 0.2) & (np.abs(v[:, 2] - 0.325) < 0.2)
        return v[core, 1].std()
    ta, ti = top_spread(a["vertices"]), top_spread(i["vertices"])
    assert ta < 0.98 * ti, (ta, ti)


# ------------------------------------------------------------------ device on the CPU executor ----
# name -> (cloud, reconstruction keywords, options); the anisotropic test's list with a non-default radius factor
CASES = {
    "cfg1_fixture": (lambda: np.load(os.path.join(os.path.dirname(__file__), "golden", "cfg1_particles.npy")),
                     dict(particle_radius=R, smoothing_length=2.0, cube_size=0.75), {}),
    "cube_S16": (lambda: _cube(10, 501), dict(KW, subdomain_num_cubes_per_dim=16), {}),
    "splash_S24": (lambda: _splash((9, 9, 9), 2, 502), dict(KW, cube_size=0.6, subdomain_num_cubes_per_dim=24), {}),
    "cube_S64": (lambda: _cube(9, 503), dict(KW, subdomain_num_cubes_per_dim=64), {}),
    "droplets_sparse": (lambda: _splash((12, 6, 12), 6, 504), dict(KW, cube_size=0.75, subdomain_num_cubes_per_dim=16), {}),
    "tile_batch_1": (lambda: _splash((9, 9, 9), 2, 505), dict(KW, cube_size=0.75, subdomain_num_cubes_per_dim=16), dict(tile_batch=1)),
    "particle_aabb": (lambda: _cube(10, 506), dict(KW, subdomain_num_cubes_per_dim=16, aabb_min=[0.05, 0.0, -1.0], aabb_max=[1.0, 0.3, 1.0]), {}),
    "clustered_overflow": (lambda: _clustered(507), dict(KW, subdomain_num_cubes_per_dim=16), dict(tier="avg_select")),
    "empty": (lambda: np.zeros((0, 3), np.float32), KW, {}),
    "one_particle": (lambda: np.array([[0.1, 0.2, 0.3]], np.float32), KW, {}),
    "radius_factor": (lambda: _cube(9, 508), dict(KW, subdomain_num_cubes_per_dim=24), dict(radius_factor=1.6)),
    "edge_of_support": (lambda: _edge_shell_particle()[None], SHELL_KW, {}),
}


def check_device_case(ss, oracle_mod, name):
    """Device (or CPU executor) vs oracle, bit for bit (mesh, densities, the kept tile); densities vs the standard run; two runs
    identical.  Returns the level-set path counters of the first run."""
    gen, kw, opts = CASES[name]
    p = gen()
    av = ss.AveragedSurface(opts.get("radius_factor", 1.0))
    o = oracle_reconstruct_averaged(p, radius_factor=av.radius_factor, **kw)
    assert o["rc"] == 0
    flat = _busiest_tile(o)
    if flat is not None:
        o = oracle_reconstruct_averaged(p, radius_factor=av.radius_factor, tile_of_subdomain=flat, **kw)
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


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_averaged_matches_oracle(emu, oracle_mod, name):  # noqa: F811
    check_device_case(emu, oracle_mod, name)


def test_emulated_averaged_refusals(emu):  # noqa: F811
    p = _cube(6, 708)
    ctx = emu.Context()
    try:
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, averaged_surface=emu.AveragedSurface(), subdomain_grid=False, **KW)
        assert e.value.code == 7
        for rf in (0.0, -1.0, float("nan"), float("inf"), 4.0):
            with pytest.raises(emu.SplashsurfError) as e:
                emu.reconstruct_surface(p, context=ctx, averaged_surface=emu.AveragedSurface(rf), **KW)
            assert e.value.code == 6, rf
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, averaged_surface=emu.AveragedSurface(), anisotropy=emu.Anisotropy(), **KW)
        assert e.value.code == 6
        # the context is back to the standard level set after a refused call
        base = emu.reconstruct_surface(p, context=ctx, subdomain_grid_auto_disable=False, with_debug=True, **KW)
        assert base.mesh.nvertices > 0 and base.levelset_paths["avg_512"] == 0
        # the partitioned (multi-GPU) entry
        L = ctx._L
        params = emu.make_params(**KW)
        grid = emu._Grid()
        emu._check(L, L.ss_grid_for_reconstruction_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid)))
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, C.byref(emu.AveragedSurface()._abi())))
        out = C.c_void_p()
        rc = L.ss_reconstruct_partition_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid), 0, 0, 100, 1, 0, 0, C.byref(out))
        assert rc == 7 and not out
        emu._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, None))
    finally:
        ctx.close()


def test_runner_refuses_averaged_surface_on_several_gpus():
    from splashsurf_b200 import AveragedSurface, distributed as ssd
    with pytest.raises(ValueError, match="averaged-position surface"):
        ssd.Runner(None, None, 2, 0, 0, device="cpu", averaged_surface=AveragedSurface())


def test_emulated_cli_averaged(emu, tmp_path):  # noqa: F811
    """`reconstruct --averaged-surface=on` writes the mesh of reconstruct_surface(averaged_surface=AveragedSurface()); it refuses
    --anisotropic=on and --partition=on, and --averaged-radius-factor without it."""
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q"]
    assert cli.main(args + ["--averaged-surface=on", "-o", str(tmp_path / "a.npz")]) == 0
    got = np.load(tmp_path / "a.npz")
    p = io.read_particles(src)
    want = emu.reconstruct_surface(p, particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False,
                                   averaged_surface=emu.AveragedSurface())
    assert np.array_equal(got["vertices"], want.mesh.vertices) and np.array_equal(got["triangles"], want.mesh.triangles)
    assert cli.main(args + ["--averaged-surface=on", "--averaged-radius-factor", "1.5", "-o", str(tmp_path / "b.npz")]) == 0
    assert not np.array_equal(np.load(tmp_path / "b.npz")["vertices"], got["vertices"])
    with pytest.raises(ValueError, match="--averaged-surface=on"):
        cli.main(args + ["--averaged-radius-factor", "1.5", "-o", str(tmp_path / "c.npz")])
    assert not os.path.exists(tmp_path / "c.npz")
    for other in ("--partition=on", "--anisotropic=on"):
        with pytest.raises(ValueError, match=other):
            cli.main(args + ["--averaged-surface=on", other, "-o", str(tmp_path / "c.npz")])
        assert not os.path.exists(tmp_path / "c.npz")
