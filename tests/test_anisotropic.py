"""Anisotropic kernels (Yu & Turk 2013; splashsurf_b200.Anisotropy, DESIGN.md section 11).

* the plain-C restatement (tests/anisotropic_oracle.c, built on the pinned oracle) against an independent float64 numpy
  restatement of the definition (guards against a formula error the restatement and the kernels would share), plus properties;
* the device pipeline on the CPU executor of the CUDA sources (tests/emul) against the oracle, bit for bit: smoothed centres,
  G matrices, particle densities (also equal to the isotropic run's), canonical mesh;
* refusals, the command line, and the surface quality gain measured on the oracle.
The GPU-marked counterpart of the device cases is tests/test_zzz_gpu_anisotropic.py."""
import ctypes as C
import os

import numpy as np
import pytest

import c_oracle
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

R = 0.025
KW = dict(particle_radius=R, smoothing_length=2.0, cube_size=0.5)


# ------------------------------------------------------------------ the anisotropic oracle (tests/anisotropic_oracle.c) ----
def _aniso_lib():
    """tests/anisotropic_oracle.c (it includes the pinned oracle/splashsurf_oracle.c unchanged) with its entry points bound."""
    from oracle import _Params, _Result
    vp = C.c_void_p
    return c_oracle.build("anisotropic_oracle.c", {
        "so_reconstruct_aniso": (C.c_int, [vp, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_float, C.c_uint32, C.POINTER(C.POINTER(_Result)),
                                           C.c_int64, vp, vp, vp]),
        "so_aniso_records": (C.c_int64, [vp, C.c_uint64, C.POINTER(_Params), C.c_float, C.c_float, C.c_uint32, vp, vp, vp, vp]),
        "so_free": (None, [C.POINTER(_Result)])})


def _aniso_params(particle_radius, smoothing_length, cube_size, rest_density, iso_surface_threshold, aabb_min, aabb_max,
                  subdomain_grid, subdomain_num_cubes_per_dim):
    from oracle import _Params, absolute_params
    r, h, c = absolute_params(particle_radius, smoothing_length, cube_size)
    p = _Params()
    p.particle_radius, p.rest_density, p.compact_support_radius = float(r), float(np.float32(rest_density)), float(h)
    p.cube_size, p.iso_surface_threshold = float(c), float(np.float32(iso_surface_threshold))
    p.has_particle_aabb = int(aabb_min is not None and aabb_max is not None)
    if p.has_particle_aabb:
        p.aabb_min = (C.c_float * 3)(*[float(np.float32(v)) for v in aabb_min])
        p.aabb_max = (C.c_float * 3)(*[float(np.float32(v)) for v in aabb_max])
    p.enable_simd, p.decomposition = 1, int(subdomain_grid)
    p.subdomain_num_cubes_per_dim, p.auto_disable = int(subdomain_num_cubes_per_dim), 0
    return p


def oracle_reconstruct_anisotropic(particles, *, particle_radius, smoothing_length, cube_size, rest_density=1000.0, iso_surface_threshold=0.6,
                            aabb_min=None, aabb_max=None, subdomain_grid=True, subdomain_num_cubes_per_dim=64, smoothing=0.9,
                            max_stretch=4.0, min_neighbors=10, tile_of_subdomain=None, **_ignored):
    """C-oracle reconstruction with anisotropic kernels (DESIGN.md section 11): the dict of `reconstruct` plus
    "smoothed_particles" (n, 3) and "anisotropy" (n, 6: g00 g01 g02 g11 g12 g22) of the filtered particles.  Always decomposed."""
    from oracle import _Result, _grid_dict
    L = _aniso_lib()
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    p = _aniso_params(particle_radius, smoothing_length, cube_size, rest_density, iso_surface_threshold, aabb_min, aabb_max,
                      subdomain_grid, subdomain_num_cubes_per_dim)
    S = int(subdomain_num_cubes_per_dim)
    tile = np.zeros((S + 1,) * 3, dtype=np.float32) if tile_of_subdomain is not None else None
    xbar = np.zeros((max(len(xyz), 1), 3), np.float32)
    g = np.zeros((max(len(xyz), 1), 6), np.float32)
    out = C.POINTER(_Result)()
    rc = L.so_reconstruct_aniso(xyz.ctypes.data, len(xyz), C.byref(p), float(np.float32(smoothing)), float(np.float32(max_stretch)),
                                int(min_neighbors), C.byref(out), -1 if tile_of_subdomain is None else int(tile_of_subdomain),
                                None if tile is None else tile.ctypes.data, xbar.ctypes.data, g.ctypes.data)
    try:
        if rc != 0:
            return {"rc": rc}
        res = out.contents
        n = res.n_filtered
        nv, nt, ns = res.nv, res.nt, res.n_subdomains
        d = {"rc": rc, "grid": _grid_dict(res.grid), "used_decomposition": bool(res.used_decomposition),
             "subdomain_grid": _grid_dict(res.subdomain_grid)}
        d["particle_densities"] = np.ctypeslib.as_array(res.densities, (n,)).copy() if n else np.zeros(0, np.float32)
        d["particle_inside_aabb"] = (np.ctypeslib.as_array(res.inside_aabb, (len(xyz),)).astype(bool).copy() if p.has_particle_aabb else None)
        d["vertices"] = np.ctypeslib.as_array(res.vertices, (nv, 3)).copy() if nv else np.zeros((0, 3), np.float32)
        d["triangles"] = np.ctypeslib.as_array(res.triangles, (nt, 3)).copy() if nt else np.zeros((0, 3), np.uint64)
        d["vertex_keys"] = np.ctypeslib.as_array(res.vertex_keys, (nv, 4)).copy() if nv else np.zeros((0, 4), np.int64)
        d["subdomain_flat"] = np.ctypeslib.as_array(res.subdomain_flat, (ns,)).copy() if ns else np.zeros(0, np.int64)
        d["subdomain_count"] = np.ctypeslib.as_array(res.subdomain_count, (ns,)).copy() if ns else np.zeros(0, np.uint64)
        d["smoothed_particles"], d["anisotropy"], d["tile"] = xbar[:n].copy(), g[:n].copy(), tile
        return d
    finally:
        L.so_free(out)



def oracle_anisotropy(particles, *, particle_radius, smoothing_length, cube_size, smoothing=0.9, max_stretch=4.0, min_neighbors=10,
                      subdomain_num_cubes_per_dim=64, rest_density=1000.0):
    """x_bar (n, 3) and G (n, 6: g00 g01 g02 g11 g12 g22) of every particle, from the anisotropic oracle."""
    o = oracle_reconstruct_anisotropic(particles, particle_radius=particle_radius, smoothing_length=smoothing_length, cube_size=cube_size,
                                       smoothing=smoothing, max_stretch=max_stretch, min_neighbors=min_neighbors,
                                       subdomain_num_cubes_per_dim=subdomain_num_cubes_per_dim, rest_density=rest_density)
    assert o["rc"] == 0, o
    return o["smoothed_particles"], o["anisotropy"]


# ------------------------------------------------------------------ clouds ----
def _cube(n, seed):
    from splashsurf_b200 import synthetic as syn
    return syn.jittered_cube(n, R, seed)


def _splash(n, drops, seed):
    from splashsurf_b200 import synthetic as syn
    return syn.splash(n, drops, R, seed)


def _lattice(nx, ny, nz, jitter=0.0, seed=0):
    d = 2 * R
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3).astype(np.float64) * d
    if jitter:
        g += np.random.default_rng(seed).uniform(-jitter * d, jitter * d, g.shape)
    return g.astype(np.float32)


def _sphere(radius_d, seed, jitter=0.25):
    p = _lattice(2 * radius_d + 1, 2 * radius_d + 1, 2 * radius_d + 1, jitter, seed) - np.float32(radius_d * 2 * R)
    return np.ascontiguousarray(p[np.linalg.norm(p.astype(np.float64), axis=1) <= radius_d * 2 * R])


def _clustered(seed):
    """A jittered cube plus 4400 particles inside a ball of radius 0.6 h: more candidates per brick than the 4096-slot slice."""
    rng = np.random.default_rng(seed)
    h = 4 * R
    v = rng.normal(size=(4400, 3))
    ball = (v / np.linalg.norm(v, axis=1, keepdims=True) * (0.6 * h * rng.uniform(0, 1, (4400, 1)) ** (1 / 3)) + 0.2).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([_cube(8, seed), ball]))


# name -> (cloud, reconstruction keywords, context options)
CASES = {
    "cfg1_fixture": (lambda: np.load(os.path.join(os.path.dirname(__file__), "golden", "cfg1_particles.npy")),
                     dict(particle_radius=R, smoothing_length=2.0, cube_size=0.75), {}),
    "cube_S16": (lambda: _cube(10, 501), dict(KW, subdomain_num_cubes_per_dim=16), {}),
    "splash_S24": (lambda: _splash((9, 9, 9), 2, 502), dict(KW, cube_size=0.6, subdomain_num_cubes_per_dim=24), {}),
    "cube_S64": (lambda: _cube(9, 503), dict(KW, subdomain_num_cubes_per_dim=64), {}),
    "droplets_sparse": (lambda: _splash((12, 6, 12), 6, 504), dict(KW, cube_size=0.75, subdomain_num_cubes_per_dim=16), {}),
    "tile_batch_1": (lambda: _splash((9, 9, 9), 2, 505), dict(KW, cube_size=0.75, subdomain_num_cubes_per_dim=16), dict(tile_batch=1)),
    "particle_aabb": (lambda: _cube(10, 506), dict(KW, subdomain_num_cubes_per_dim=16, aabb_min=[0.05, 0.0, -1.0], aabb_max=[1.0, 0.3, 1.0]), {}),
    "clustered_overflow": (lambda: _clustered(507), dict(KW, subdomain_num_cubes_per_dim=16), {}),
    "empty": (lambda: np.zeros((0, 3), np.float32), KW, {}),
    "one_particle": (lambda: np.array([[0.1, 0.2, 0.3]], np.float32), KW, {}),
    "custom_parameters": (lambda: _cube(9, 508), dict(KW, subdomain_num_cubes_per_dim=24), dict(aniso=dict(smoothing=0.5, max_stretch=2.5, min_neighbors=4))),
}


def check_device_case(ss, oracle_mod, name):
    """Device (or CPU executor) vs oracle, bit for bit; densities vs the isotropic run; two runs identical."""
    gen, kw, opts = CASES[name]
    p = gen()
    an = ss.Anisotropy(**opts.get("aniso", {}))
    ctx = ss.Context()
    try:
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        g = ss.reconstruct_surface(p, context=ctx, with_debug=True, anisotropy=an, **kw)
        g2 = ss.reconstruct_surface(p, context=ctx, with_debug=True, anisotropy=an, **kw)
        iso = ss.reconstruct_surface(p, context=ctx, subdomain_grid_auto_disable=False, **kw)
    finally:
        ctx.close()
    o = oracle_reconstruct_anisotropic(p, smoothing=an.smoothing, max_stretch=an.max_stretch, min_neighbors=an.min_neighbors, **kw)
    assert o["rc"] == 0
    assert np.array_equal(g.particle_densities, o["particle_densities"])
    assert np.array_equal(g.particle_densities, iso.particle_densities)
    assert np.array_equal(g.smoothed_particles, o["smoothed_particles"])
    assert np.array_equal(g.anisotropy_matrices.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]], o["anisotropy"])
    assert np.array_equal(g.subdomains["flat"], o["subdomain_flat"]) and np.array_equal(g.subdomains["count"], o["subdomain_count"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                               kw.get("subdomain_num_cubes_per_dim", 64))
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, m
    assert np.array_equal(g.mesh.vertices, g2.mesh.vertices) and np.array_equal(g.mesh.triangles, g2.mesh.triangles)
    assert np.array_equal(g.anisotropy_matrices, g2.anisotropy_matrices)
    if len(p) > 100:
        assert g.mesh.nvertices > 0


# ------------------------------------------------------------------ float64 restatement ----
def numpy_anisotropy(p, h, lam=0.9, kr=4.0, min_nb=10):
    """The definition of DESIGN.md section 11 in float64 (numpy eigh, brute-force neighbours).  Also returns per particle the
    neighbour count and whether a neighbour sits within 1e-5 h of the support radius (count ambiguous in f32)."""
    from scipy.spatial import cKDTree
    x = p.astype(np.float64)
    n = len(x)
    tree = cKDTree(x)
    xbar, G, det = x.copy(), np.tile(np.eye(3), (n, 1, 1)), np.ones(n)
    nn, amb = np.zeros(n, int), np.zeros(n, bool)
    for i, nb in enumerate(tree.query_ball_point(x, h * (1 + 1e-5))):
        nb = np.array([j for j in nb if j != i], int)
        d = x[nb] - x[i] if len(nb) else np.zeros((0, 3))
        r = np.linalg.norm(d, axis=1)
        amb[i] = bool(np.any(np.abs(r - h) < 1e-5 * h))
        keep = r < h
        d, r = d[keep], r[keep]
        nn[i] = len(d)
        w = np.concatenate([[1.0], 1.0 - (r / h) ** 3])
        off = np.concatenate([np.zeros((1, 3)), d])
        mu = (w[:, None] * off).sum(0) / w.sum()
        xbar[i] = x[i] + lam * mu
        e = off - mu
        C = (w[:, None, None] * e[:, :, None] * e[:, None, :]).sum(0) / w.sum()
        sig, V = np.linalg.eigh(C)
        sig, V = np.maximum(sig[::-1], 0.0), V[:, ::-1]
        if nn[i] < min_nb or sig[0] == 0.0:
            continue
        s = np.maximum(sig, sig[0] / kr) / sig[0]
        G[i] = V @ np.diag(1.0 / s) @ V.T
        det[i] = np.prod(1.0 / s)
    return xbar, G, det, nn, amb


def _w_cubic(r, h):
    """The cubic spline with support h (kernel.rs:51-107) in float64."""
    q = 2.0 * r / h
    f = np.where(q < 1.0, 1.5 / np.pi * (2.0 / 3.0 - q * q + 0.5 * q ** 3), np.where(q < 2.0, 0.25 / np.pi * (2.0 - q) ** 3, 0.0))
    return 8.0 / h ** 3 * f


ORACLE_CLOUDS = {
    "jittered_lattice": lambda: _cube(9, 601),
    "slab": lambda: _lattice(14, 3, 14, 0.25, 602),
    "sphere": lambda: _sphere(5, 603),
    "sparse_droplets": lambda: _splash((6, 3, 6), 5, 604),
    "two_particles": lambda: np.array([[0.0, 0.0, 0.0], [0.05, 0.01, 0.0]], np.float32),
}


@pytest.mark.parametrize("name", sorted(ORACLE_CLOUDS))
def test_oracle_anisotropy_matches_float64_restatement(oracle_mod, name):
    p = ORACLE_CLOUDS[name]()
    h = 4 * R
    xb, g = oracle_anisotropy(p, **KW)
    nxb, nG, _, _, amb = numpy_anisotropy(p, h)
    ok = ~amb
    assert np.abs(xb[ok].astype(np.float64) - nxb[ok]).max() <= 1e-5 * h
    G = g[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3).astype(np.float64)
    assert np.abs(G[ok] - nG[ok]).max() <= 1e-4


@pytest.mark.parametrize("name", ["jittered_lattice", "sphere", "slab"])
def test_oracle_levelset_matches_float64_restatement(oracle_mod, name):
    """The oracle's level-set tile of one subdomain against sum_j V_j det G_j W(|G_j (x - x_bar_j)|) in float64."""
    p = ORACLE_CLOUDS[name]()
    h = 4 * R
    S = 16
    kw = dict(KW, subdomain_num_cubes_per_dim=S)
    o0 = oracle_reconstruct_anisotropic(p, **kw)
    flat = int(o0["subdomain_flat"][len(o0["subdomain_flat"]) // 2])
    o = oracle_reconstruct_anisotropic(p, tile_of_subdomain=flat, **kw)
    nxb, nG, ndet, _, amb = numpy_anisotropy(p, h)
    if amb.any():
        pytest.skip("a neighbour at the support radius makes the neighbour count ambiguous in f32")
    sg, gg = o["subdomain_grid"], o["grid"]
    nsd = sg["ncells"]
    ijk = np.array([flat // (nsd[1] * nsd[2]), (flat // nsd[2]) % nsd[1], flat % nsd[2]])
    idx = np.stack(np.meshgrid(*[np.arange(S + 1)] * 3, indexing="ij"), -1).reshape(-1, 3) + ijk * S
    pts = gg["aabb_min"].astype(np.float64) + idx * float(gg["cell_size"])
    rest_mass = (2 * R) ** 3 * 1000.0
    V = rest_mass / o["particle_densities"].astype(np.float64) * ndet
    phi = np.zeros(len(pts))
    for j in range(len(p)):
        u = np.einsum("ab,nb->na", nG[j], nxb[j][None] - pts)
        r = np.linalg.norm(u, axis=1)
        phi += np.where(r < h, V[j] * _w_cubic(r, h), 0.0)
    tile = o["tile"].reshape(-1).astype(np.float64)
    assert np.abs(tile - phi).max() <= 1e-5 * max(np.abs(phi).max(), 1.0)


def test_interior_lattice_particle_is_isotropic(oracle_mod):
    p = _lattice(9, 9, 9)
    xb, g = oracle_anisotropy(p, **KW)
    centre = np.argmin(np.linalg.norm(p - p.mean(0), axis=1))
    assert np.abs(g[centre] - np.array([1, 0, 0, 1, 0, 1], np.float32)).max() < 1e-5
    assert np.abs(xb[centre] - p[centre]).max() < 1e-6


def test_sheet_surface_particle_is_flat_with_clamped_stretch(oracle_mod):
    """A one-layer sheet: zero variance along its normal -> the kernel's shortest axis lies along y, stretch clamped at k_r."""
    p = _lattice(13, 1, 13)
    xb, g = oracle_anisotropy(p, **KW)
    c = np.argmin(np.linalg.norm(p - p.mean(0), axis=1))
    G = g[c][[0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(3, 3).astype(np.float64)
    lam, vec = np.linalg.eigh(G)
    assert abs(lam[-1] - 4.0) < 1e-4 and abs(abs(vec[1, -1]) - 1.0) < 1e-4
    assert np.abs(lam[:2] - 1.0).max() < 1e-4
    # a jittered slab: at a top-face particle the shortest kernel axis (largest eigenvalue of G) is the slab normal
    s = _lattice(14, 3, 14, 0.25, 605)
    _, gs = oracle_anisotropy(s, **KW)
    top = np.where((s[:, 1] > 0.09) & (np.abs(s[:, 0] - 0.33) < 0.1) & (np.abs(s[:, 2] - 0.33) < 0.1))[0]
    assert len(top)
    for t in top:
        lam, vec = np.linalg.eigh(gs[t][[0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(3, 3).astype(np.float64))
        assert abs(vec[1, -1]) > 0.9 and lam[-1] > 1.5


def test_few_neighbours_give_identity_exactly(oracle_mod):
    p = _splash((5, 5, 5), 3, 606)
    _, g = oracle_anisotropy(p, min_neighbors=1000, **KW)
    assert np.array_equal(g, np.tile(np.array([1, 0, 0, 1, 0, 1], np.float32), (len(p), 1)))
    iso = np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]], np.float32)                 # no neighbours at all
    xb, g = oracle_anisotropy(iso, **KW)
    assert np.array_equal(xb, iso) and np.array_equal(g, np.tile(np.array([1, 0, 0, 1, 0, 1], np.float32), (2, 1)))


def test_no_stretch_no_smoothing_equals_isotropic_tiles(oracle_mod):
    """max_stretch = 1, smoothing = 0: x_bar = x, G = I up to rounding -> the isotropic exact tile to a few ulp."""
    p = _cube(9, 607)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    o0 = oracle_reconstruct_anisotropic(p, smoothing=0.0, max_stretch=1.0, **kw)
    flat = int(o0["subdomain_flat"][len(o0["subdomain_flat"]) // 2])
    a = oracle_reconstruct_anisotropic(p, smoothing=0.0, max_stretch=1.0, tile_of_subdomain=flat, **kw)
    assert np.array_equal(a["smoothed_particles"], p)
    b = oracle_mod.reconstruct(p, tile_of_subdomain=flat, subdomain_grid_auto_disable=False, simd=False, **kw)
    ta, tb = a["tile"].astype(np.float64), b["tile"].astype(np.float64)
    assert np.abs(ta - tb).max() <= 8 * np.spacing(np.float32(np.abs(tb).max()))


# ------------------------------------------------------------------ device on the CPU executor ----
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_anisotropic_matches_oracle(emu, oracle_mod, name):  # noqa: F811
    check_device_case(emu, oracle_mod, name)


def test_emulated_anisotropic_refusals(emu):  # noqa: F811
    p = _cube(6, 608)
    ctx = emu.Context()
    try:
        with pytest.raises(emu.SplashsurfError) as e:
            emu.reconstruct_surface(p, context=ctx, anisotropy=emu.Anisotropy(), subdomain_grid=False, **KW)
        assert e.value.code == 7
        for bad in (dict(smoothing=1.5), dict(smoothing=-0.1), dict(max_stretch=0.5), dict(max_stretch=float("nan")), dict(smoothing=float("nan"))):
            with pytest.raises(emu.SplashsurfError) as e:
                emu.reconstruct_surface(p, context=ctx, anisotropy=emu.Anisotropy(**bad), **KW)
            assert e.value.code == 6
        # the context is back to isotropic after a refused call
        assert emu.reconstruct_surface(p, context=ctx, **KW).mesh.nvertices > 0
        # the partitioned (multi-GPU) entry
        L = ctx._L
        params = emu.make_params(**KW)
        grid = emu._Grid()
        emu._check(L, L.ss_grid_for_reconstruction_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid)))
        emu._check(L, L.ss_context_set_anisotropy_f32(ctx._h, C.byref(emu.Anisotropy()._abi())))
        out = C.c_void_p()
        rc = L.ss_reconstruct_partition_f32(ctx._h, p.ctypes.data, len(p), C.byref(params), C.byref(grid), 0, 0, 100, 1, 0, 0, C.byref(out))
        assert rc == 7 and not out
        emu._check(L, L.ss_context_set_anisotropy_f32(ctx._h, None))
    finally:
        ctx.close()


def test_emulated_cli_anisotropic(emu, tmp_path):  # noqa: F811
    """`reconstruct --anisotropic=on` writes the mesh of reconstruct_surface(anisotropy=Anisotropy()); --partition=on refuses it."""
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q"]
    assert cli.main(args + ["--anisotropic=on", "-o", str(tmp_path / "a.npz")]) == 0
    got = np.load(tmp_path / "a.npz")
    p = io.read_particles(src)
    want = emu.reconstruct_surface(p, particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False,
                                   anisotropy=emu.Anisotropy())
    assert np.array_equal(got["vertices"], want.mesh.vertices) and np.array_equal(got["triangles"], want.mesh.triangles)
    assert cli.main(args + ["--anisotropic=on", "--aniso-max-stretch", "2", "-o", str(tmp_path / "b.npz")]) == 0
    assert not np.array_equal(np.load(tmp_path / "b.npz")["vertices"], got["vertices"])
    with pytest.raises(ValueError, match="--partition=on"):
        cli.main(args + ["--anisotropic=on", "--partition=on", "-o", str(tmp_path / "c.npz")])
    assert not os.path.exists(tmp_path / "c.npz")
    # as a process: exit code 1 and the message
    import subprocess
    import sys
    r = subprocess.run([sys.executable, "-m", "splashsurf_b200", *args, "--anisotropic=on", "--partition=on", "-o", str(tmp_path / "c.npz")],
                       capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), timeout=300)
    assert r.returncode == 1 and "--partition=on" in r.stderr


# ------------------------------------------------------------------ surface quality (oracle) ----
def test_quality_sphere_radii_spread():
    """Particle sphere (lattice jittered by +-0.1 d): the spread of the vertex radii drops with anisotropic kernels.  Measured on the
    oracle: 0.00688 with Anisotropy() against 0.00787 isotropic (ratio 0.874)."""
    import oracle
    p = _sphere(9, 609, jitter=0.1)
    kw = dict(KW, subdomain_num_cubes_per_dim=32)
    a = oracle_reconstruct_anisotropic(p, **kw)
    i = oracle.reconstruct(p, subdomain_grid_auto_disable=False, **kw)
    sa = np.linalg.norm(a["vertices"].astype(np.float64), axis=1).std()
    si = np.linalg.norm(i["vertices"].astype(np.float64), axis=1).std()
    assert sa < 0.95 * si, (sa, si)
