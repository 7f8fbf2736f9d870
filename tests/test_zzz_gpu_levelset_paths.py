"""Launch paths of the level-set stage, asserted: every kernel the stage can choose at run time against the oracle, bit for bit.

The stage picks its kernels from the data and the parameters (DESIGN.md section 3b / 4):
* certification: k_certify_warp with a 384-candidate slice (at most 16 candidate bin runs per brick, R = ceil(h / c) <= 8), with a
  576-candidate slice (17-32 runs: R = 9, and R = 17-25 where the bins are 16 cells wide), or the fused k_levelset (more runs);
* the exact pass and the fix-up pass: a cascade of k_exact_warp (512 candidates), k_exact_warp_mid (1024), k_exact_warp_big (4096,
  dynamic shared memory) and k_levelset's selection path;
* the anisotropic level set: k_aniso_levelset<512>, <4096>, then k_aniso_select;
* each of them in its GLOBAL (no subdomain grid) and COUNT (set_count_pairs) instantiation.
Every case of CASES states the paths it exists for, and the test reads them back from `levelset_paths` (ss_surface_levelset_paths):
a case that drifts off its path fails, and `test_path_matrix_is_covered` fails when the table stops covering a cell of REQUIRED.

Fix-up cascade beyond its first tier: not in REQUIRED.  A brick reaches the fix-up pass only with a point the certification marked,
and the certification marks nothing in a brick with more candidates than its slice (576 at most, extension plane included).  The
fix-up pass stages a subset of those (no extension plane), so its 4096 tier and the selection path cannot be reached.  Its 1024 tier
needs, in such a brick, 513-576 candidates or more than 224 within the support of one 4x4x4 sub-box, next to a certified point on a
surface-crossing edge; with a uniform density one sub-box support holds about 15 % of a brick's candidates, and no dense cluster
tried (R = 9 and R = 20, 530-570 particles, sigma 0.006-0.015; lattices of spacing 0.032-0.046) produced a fix-up brick at all.

The same table runs on the H100 (`ss` fixture) and on the CPU executor of the CUDA sources (`emu`).  The executor cannot check
what differs between these kernels on the device (shared-memory opt-in, slice sizes, mbarrier phases, register allocation): the
GPU run is the one that counts for them."""
import numpy as np
import pytest

from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

BASE = dict(particle_radius=0.025, smoothing_length=2.0)
TIERS = ("512", "1024", "4096", "select")
C05 = 0.5 * 0.025                                   # absolute cube size of cube_size = 0.5 (R = 8)


def _cube(n, seed, r=0.025):
    from splashsurf_b200 import synthetic as syn
    return syn.jittered_cube(n, r, seed)


def _cluster(n, sigma=0.004, seed=None):
    """n particles normally distributed around the origin: with sigma = 0.004 every one is a candidate of each of the 27 bricks
    around it (600: more than 512, 1500: more than 1024, 4500: more than 4096)."""
    return np.random.default_rng(n if seed is None else seed).normal(0, sigma, (n, 3)).astype(np.float32)


def _corner_cluster(n):
    """A cluster on the corner shared by 8 subdomains of 64 cubes, plus one particle at the origin that fixes the grid: the grid starts
    at -(R + 1) c (the kernel margin, rounded down to a cell), so the subdomain corner is at (64 - R - 1) c = 55 c on each axis.  The
    cluster's particles are ghost members of all 8 tiles, and the bricks of the lower tiles around it hold the index-64 planes."""
    return np.concatenate([np.zeros((1, 3), np.float32), _cluster(n) + np.float32(55 * C05)])


def _aniso_cluster(n_ball, seed):
    """test_anisotropic._clustered with n_ball particles in the ball of radius 0.6 h."""
    rng = np.random.default_rng(seed)
    h = 4 * 0.025
    v = rng.normal(size=(n_ball, 3))
    ball = (v / np.linalg.norm(v, axis=1, keepdims=True) * (0.6 * h * rng.uniform(0, 1, (n_ball, 1)) ** (1 / 3)) + 0.2).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([_cube(8, seed), ball]))


SUB = dict(subdomain_grid_auto_disable=False)
GLOBAL = dict(subdomain_grid=False)
# name -> (cloud, reconstruction keywords, context options, path cells the case must take)
CASES = {
    "cube_R8": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **SUB), {},
                ["cert/sub/384", "exact/sub/512", "fixup/sub/512"]),
    "cube_R8_global": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **GLOBAL), {},
                       ["cert/global/384", "exact/global/512", "fixup/global/512"]),
    "cube_R9": (lambda: _cube(8, 1), dict(BASE, cube_size=0.45, **SUB), {}, ["cert/sub/576_R9", "exact/sub/512", "fixup/sub/512"]),
    "cube_R9_global": (lambda: _cube(8, 1), dict(BASE, cube_size=0.45, **GLOBAL), {}, ["cert/global/576_R9", "exact/global/512"]),
    "cube_R14_fused": (lambda: _cube(8, 1), dict(BASE, cube_size=0.3, **SUB), {}, ["cert/sub/fused_R"]),
    "cube_R14_fused_global": (lambda: _cube(8, 1), dict(BASE, cube_size=0.3, **GLOBAL), {}, ["cert/global/fused_R"]),
    "cube_R20_bins16": (lambda: _cube(6, 1), dict(BASE, cube_size=0.2, **SUB), {}, ["cert/sub/576_R17_25", "exact/sub/512"]),
    "cube_R20_bins16_global": (lambda: _cube(6, 1), dict(BASE, cube_size=0.2, **GLOBAL), {}, ["cert/global/576_R17_25", "exact/global/512"]),
    "cluster_1024": (lambda: _cluster(600), dict(BASE, cube_size=0.5, **SUB), {}, ["exact/sub/1024"]),
    "cluster_1024_global": (lambda: _cluster(600), dict(BASE, cube_size=0.5, **GLOBAL), {}, ["exact/global/1024"]),
    "cluster_4096": (lambda: _cluster(1500), dict(BASE, cube_size=0.5, **SUB), {}, ["exact/sub/4096"]),
    "cluster_4096_global": (lambda: _cluster(1500), dict(BASE, cube_size=0.5, **GLOBAL), {}, ["exact/global/4096"]),
    "cluster_4096_scalar": (lambda: _cluster(1500), dict(BASE, cube_size=0.5, simd=False, **SUB), {}, ["exact/sub/4096", "scalar/sub/4096"]),
    "cluster_select": (lambda: _cluster(4500), dict(BASE, cube_size=0.5, **SUB), {}, ["exact/sub/select"]),
    "cluster_select_global": (lambda: _cluster(4500), dict(BASE, cube_size=0.5, **GLOBAL), {}, ["exact/global/select"]),
    "corner_cluster_batch_1": (lambda: _corner_cluster(1500), dict(BASE, cube_size=0.5, **SUB), dict(tile_batch=1),
                               ["corner/8_tiles", "exact/sub/512", "exact/sub/4096"]),
    "aniso_4096": (lambda: _aniso_cluster(1500, 511), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16), dict(aniso=True),
                   ["aniso/512", "aniso/4096"]),
    "aniso_clustered_overflow": (lambda: _aniso_cluster(4400, 507), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16),
                                 dict(aniso=True), ["aniso/select"]),
}

REQUIRED = sorted(
    [f"cert/{m}/{k}" for m in ("sub", "global") for k in ("384", "576_R9", "576_R17_25", "fused_R")]
    + [f"exact/{m}/{t}" for m in ("sub", "global") for t in TIERS]
    + ["fixup/sub/512", "fixup/global/512", "scalar/sub/4096", "corner/8_tiles", "aniso/4096", "aniso/select"])


def _finished(received):
    """Bricks each tier of a cascade finished: what it received minus what it passed on (the last tier passes nothing on)."""
    return [received[t] - (received[t + 1] if t + 1 < len(received) else 0) for t in range(len(received))]


def taken_cells(lp, kw, opts, subdomains):
    """The path cells of one reconstruction, from its levelset_paths."""
    m = "global" if lp["global"] else "sub"
    R = lp["R"]
    cells = set()
    if lp["cert_warp_384"]:
        cells.add(f"cert/{m}/384")
    if lp["cert_warp_576"]:
        assert R == 9 or 17 <= R <= 25, lp
        cells.add(f"cert/{m}/576_R9" if R == 9 else f"cert/{m}/576_R17_25")
    if lp["cert_fused"] and R >= 10 and not 17 <= R <= 25:
        cells.add(f"cert/{m}/fused_R")
    for cascade in ("exact", "fixup"):
        for t, n in zip(TIERS, _finished([lp[f"{cascade}_{t}"] for t in TIERS])):
            assert n >= 0, lp
            if n:
                cells.add(f"{cascade}/{m}/{t}")
                if cascade == "exact" and t != "512" and kw.get("simd") is False:
                    cells.add(f"scalar/{m}/{t}")
    for t, n in zip(("512", "4096", "select"), _finished([lp[f"aniso_{t}"] for t in ("512", "4096", "select")])):
        if n:
            cells.add(f"aniso/{t}")
    if opts.get("tile_batch") == 1 and kw.get("subdomain_num_cubes_per_dim", 64) == 64 and subdomains is not None \
            and len(subdomains["flat"]) == 8 and int(subdomains["count"].min()) >= 1500:
        cells.add("corner/8_tiles")
    return cells


def _run(lib, p, kw, opts, count):
    ctx = lib.Context()
    try:
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        ctx.set_count_pairs(count)
        an = lib.Anisotropy() if opts.get("aniso") else None
        return lib.reconstruct_surface(p, with_debug=True, context=ctx, anisotropy=an, **kw)
    finally:
        ctx.close()


def check_case(lib, oracle_mod, name):
    gen, kw, opts, expected = CASES[name]
    p = gen()
    g = _run(lib, p, kw, opts, False)
    if opts.get("aniso"):
        from test_anisotropic import oracle_reconstruct_anisotropic
        o = oracle_reconstruct_anisotropic(p, **kw)
        assert o["rc"] == 0
    else:
        o = oracle_mod.reconstruct(p, **kw)
    lp = g.levelset_paths
    cells = taken_cells(lp, kw, opts, g.subdomains)
    assert set(expected) <= cells, (name, sorted(set(expected) - cells), lp)
    assert lp["count_pairs"] == 0
    assert np.array_equal(g.particle_densities, o["particle_densities"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                               kw.get("subdomain_num_cubes_per_dim", 64))
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, (name, m)
    # the COUNT instantiations of the same kernels: same paths, same bits, and certification work counted exactly when certified
    gc = _run(lib, p, kw, opts, True)
    lpc = gc.levelset_paths
    assert lpc["count_pairs"] == 1 and {k: v for k, v in lpc.items() if k != "count_pairs"} == {k: v for k, v in lp.items() if k != "count_pairs"}
    assert np.array_equal(gc.particle_densities.view(np.uint32), g.particle_densities.view(np.uint32))
    assert np.array_equal(gc.mesh.vertices.view(np.uint32), g.mesh.vertices.view(np.uint32))
    assert np.array_equal(gc.mesh.triangles, g.mesh.triangles) and np.array_equal(gc.vertex_edge_keys, g.vertex_edge_keys)
    # certification evaluations: counted by k_certify_warp only, and by it whenever it swept a brick -- which it did when fewer bricks
    # than it received went on to the exact pass (a brick with more candidates than its slice goes there whole, unswept)
    cw = lpc["cert_warp_384"] + lpc["cert_warp_576"]
    if cw == 0:
        assert gc.timings["levelset_cert_evals"] == 0, (name, lpc)
    if lpc["exact_512"] < cw:
        assert gc.timings["levelset_cert_evals"] > 0, (name, lpc)
    if not opts.get("aniso"):                       # the anisotropic level set has no pair counter
        assert gc.timings["levelset_pairs"] > 0
    assert g.timings["levelset_pairs"] == 0 and g.timings["levelset_cert_evals"] == 0
    return cells


def numpy_pair_count(p, g, h, S):
    """(grid point, particle) pairs with |x - p| < h over every point of every tile, in float64: the in-support test d^2 < h^2 of the
    dense-subdomain kernels (every particle within h of a tile point is a member of that tile: the ghost margin is at least h).
    Returns the bounds for a band of 1e-6 relative around h, where the f32 test may go either way."""
    from scipy.spatial import cKDTree
    gmin = np.asarray(g.grid.aabb.min, np.float64)
    c = float(g.grid.cell_size)
    nsd = g.subdomain_grid.ncells_per_dim
    tree = cKDTree(p.astype(np.float64))
    lo = hi = 0
    ax = np.arange(S + 1)
    for f in g.subdomains["flat"]:
        ijk = np.array([f // (nsd[1] * nsd[2]), (f // nsd[2]) % nsd[1], f % nsd[2]])
        idx = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3) + ijk * S
        pts = gmin + c * idx
        lo += int(tree.query_ball_point(pts, h * (1 - 1e-6), return_length=True).sum())
        hi += int(tree.query_ball_point(pts, h * (1 + 1e-6), return_length=True).sum())
    return lo, hi


PAIR_CLOUDS = {
    "cube": lambda: _cube(6, 11),
    # 600 candidates per brick: variant 2 evaluates them in k_exact_warp_mid, variant 1 and exact everywhere in k_levelset's
    # selection path (more than its 512 staged candidates)
    "cluster_600": lambda: _cluster(600),
}


def check_pair_counter(lib, cloud):
    """levelset_pairs, the numerator of bench.py's roofline figures: with a threshold no point reaches, no box certifies, so every path
    evaluates the same (point, particle) pairs -- variant 2 (certification + exact cascade), variant 1, and exact everywhere -- and the
    count equals an independent float64 count."""
    p = PAIR_CLOUDS[cloud]()
    kw = dict(BASE, cube_size=0.5, iso_surface_threshold=1e6, **SUB)
    got = {}
    for variant, exact in ((2, False), (1, False), (2, True)):
        ctx = lib.Context()
        try:
            ctx.set_levelset_variant(variant)
            ctx.set_levelset_exact_everywhere(exact)
            ctx.set_count_pairs(True)
            g = lib.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
        finally:
            ctx.close()
        assert not g.subdomains["sparse"].any() and g.mesh.nvertices == 0
        got[(variant, exact)] = (g.timings["levelset_pairs"], g.levelset_paths)
    pairs = {k: v[0] for k, v in got.items()}
    assert len(set(pairs.values())) == 1, pairs
    assert got[(2, False)][1]["cert_warp_384"] and got[(1, False)][1]["cert_cta"] and got[(2, True)][1]["cert_fused"]
    lo, hi = numpy_pair_count(p, g, float(lib.make_params(**kw).compact_support_radius), 64)
    assert 0 < lo <= pairs[(2, False)] <= hi, (lo, pairs, hi)


# ------------------------------------------------------------------ H100 ----
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cuda_levelset_path(ss, oracle_mod, name):
    check_case(ss, oracle_mod, name)


@pytest.mark.gpu
@pytest.mark.parametrize("cloud", list(PAIR_CLOUDS))
def test_cuda_levelset_pair_counter(ss, cloud):
    check_pair_counter(ss, cloud)


# ------------------------------------------------------------------ CPU executor ----
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_levelset_path(emu, oracle_mod, name):
    check_case(emu, oracle_mod, name)


@pytest.mark.parametrize("cloud", list(PAIR_CLOUDS))
def test_emulated_levelset_pair_counter(emu, cloud):
    check_pair_counter(emu, cloud)


def test_path_matrix_is_covered():
    """The union of the cells the cases claim covers every required cell (each case's claim is checked by the tests above)."""
    covered = set()
    for _, _, _, expected in CASES.values():
        covered |= set(expected)
    assert not set(REQUIRED) - covered, sorted(set(REQUIRED) - covered)
    assert covered <= set(REQUIRED) | {"aniso/512"}, sorted(covered - set(REQUIRED))
