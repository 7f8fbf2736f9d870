"""GPU parity of level-set variant 1 (csrc/ss_certify.cuh: separate certification kernel + exact pass over the boxes it could
not certify; off by default) against the pinned oracle -- same assertions as the seeded parity tests of the default variant.
Kept in its own late-sorted file: written after the round's GPU budget was spent, so far it has only run on the CPU executor
(tests/test_emulated_pipeline.py::test_emulated_split_certification_variant, tools/fuzz_emulated.py --variant 1)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BASE = dict(particle_radius=0.025, smoothing_length=2.0)
CASES = [
    ("cube24", lambda syn: syn.jittered_cube(24, 0.025, 601), dict(BASE, cube_size=0.5)),
    ("splash_scalar", lambda syn: syn.splash((20, 20, 20), 5, 0.025, 602), dict(BASE, cube_size=0.6, simd=False)),
    ("splash_S20", lambda syn: syn.splash((18, 18, 18), 4, 0.025, 603), dict(BASE, cube_size=0.6, subdomain_num_cubes_per_dim=20,
                                                                             subdomain_grid_auto_disable=False)),
    ("splash_S32_c075", lambda syn: syn.splash((24, 24, 24), 6, 0.025, 604), dict(BASE, cube_size=0.75, subdomain_num_cubes_per_dim=32)),
    ("global_nodec", lambda syn: syn.splash((14, 14, 14), 4, 0.025, 605), dict(BASE, cube_size=0.75, subdomain_grid=False)),
    ("dam_small", lambda syn: syn.dam_break_scaled(120_000, 0.01, 606), dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)),
]


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("name,gen,kw", CASES, ids=[c[0] for c in CASES])
def test_cuda_split_certification_bit_exact_vs_oracle(ss, oracle_mod, name, gen, kw, variant):
    from splashsurf_b200 import synthetic as syn
    p = gen(syn)
    o = oracle_mod.reconstruct(p, **kw)
    ctx = ss.Context()
    try:
        ctx.set_levelset_variant(variant)
        g = ss.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
        assert g.timings["levelset_launches"] >= 2          # certification launch + exact pass (+ fix-up pass)
        g0 = None
        ctx.set_levelset_variant(0)
        g0 = ss.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
    finally:
        ctx.close()
    assert np.array_equal(g.particle_densities, o["particle_densities"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                               kw.get("subdomain_num_cubes_per_dim", 64))
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, m
    # and the two variants agree with each other element for element (same kernels decide and evaluate)
    assert np.array_equal(g.mesh.vertices, g0.mesh.vertices) and np.array_equal(g.mesh.triangles, g0.mesh.triangles)


@pytest.mark.parametrize("n,sigma", [(3000, 0.004), (400, 0.02), (260, 0.01), (6000, 0.004)], ids=["oversized_brick", "list_overflow", "dense_cluster", "extreme_cluster"])
def test_cuda_warp_per_brick_clustered_particles(ss, oracle_mod, n, sigma):
    """Variant 2 on pathological clustering (fallback of whole bricks to k_levelset, sub-box list overflow).  oversized_brick: the
    1024-candidate tier finishes no brick, the 4096 tier some, k_levelset's selection path the rest; extreme_cluster: every brick of
    the exact pass ends in the selection path (tests/test_zzz_gpu_levelset_paths.py holds the whole path matrix)."""
    kw = dict(BASE, cube_size=0.5, subdomain_grid_auto_disable=False)
    p = np.random.default_rng(n).normal(0, sigma, (n, 3)).astype(np.float32)
    o = oracle_mod.reconstruct(p, **kw)
    ctx = ss.Context()
    try:
        ctx.set_levelset_variant(2)
        g = ss.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
    finally:
        ctx.close()
    assert np.array_equal(g.particle_densities, o["particle_densities"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"], 64)
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, m
    lp = g.levelset_paths
    if n == 3000:
        assert lp["exact_1024"] == lp["exact_512"] > 0 and 0 < lp["exact_select"] < lp["exact_4096"] == lp["exact_1024"], lp
    if n == 6000:
        assert lp["exact_select"] == lp["exact_512"] > 0, lp


@pytest.mark.parametrize("case", ["cube24", "splash_scalar", "dam_small", "clump_rounds_and_pool_overflow", "clump_oversized_cell"])
def test_cuda_density_kernel_variants(ss, oracle_mod, case):
    """Cell-cooperative density kernel (default, csrc/ss_density.cuh) and the thread-per-particle kernel: densities bit-equal to
    the oracle and to each other, including the cooperative kernel's escape routes (rounds of 16 particles, pool overflow,
    oversized cell)."""
    from splashsurf_b200 import synthetic as syn
    kw = dict(BASE, cube_size=0.5, subdomain_grid_auto_disable=False)
    if case == "clump_rounds_and_pool_overflow":
        p = np.random.default_rng(7).normal(0, 0.01, (251, 3)).astype(np.float32)
    elif case == "clump_oversized_cell":
        p = np.random.default_rng(8).normal(0.05, 0.004, (420, 3)).astype(np.float32)
    else:
        _, gen, kw = [c for c in CASES if c[0] == case][0]
        p = gen(syn)
    o = oracle_mod.reconstruct(p, **kw)
    rho = []
    for dv in (2, 1, 0):
        ctx = ss.Context()
        try:
            ctx.set_density_variant(dv)
            g = ss.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
        finally:
            ctx.close()
        assert np.array_equal(g.particle_densities, o["particle_densities"]), dv
        rho.append(g.particle_densities)
    assert np.array_equal(rho[0], rho[1]) and np.array_equal(rho[0], rho[2])


@pytest.mark.parametrize("name,gen,kw", [c for c in CASES if c[0] != "global_nodec"], ids=[c[0] for c in CASES if c[0] != "global_nodec"])
def test_cuda_brick_pass_variants(ss, oracle_mod, name, gen, kw):
    """Warp-per-brick marching cubes + fix-up sweep (default, csrc/ss_mc.cuh) and the CTA-per-brick passes: both meshes equal the
    oracle's after canonical ordering (the order of vertices / triangles inside a brick differs between the two)."""
    from splashsurf_b200 import synthetic as syn
    p = gen(syn)
    o = oracle_mod.reconstruct(p, **kw)
    counts = []
    for mv in (1, 0):
        ctx = ss.Context()
        try:
            ctx.set_mc_variant(mv)
            g = ss.reconstruct_surface(p, with_debug=True, context=ctx, **kw)
        finally:
            ctx.close()
        m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                                   kw.get("subdomain_num_cubes_per_dim", 64))
        assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, (mv, m)
        counts.append((g.mesh.nvertices, g.mesh.ncells))
    assert counts[0] == counts[1]
