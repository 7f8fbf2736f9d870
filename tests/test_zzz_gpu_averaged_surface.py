"""Averaged-position surface (splashsurf_b200.AveragedSurface, DESIGN.md section 12) on the device: the mesh, the densities and the
kept level-set tile equal the C oracle bit for bit, the densities equal the standard run's, and the tier of the warp-per-brick
cascade each case took is read back; a 1 M-particle dam break gives a closed, manifold, reproducible mesh."""
import numpy as np
import pytest

from test_averaged_surface import CASES, check_device_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_averaged_matches_oracle(ss, oracle_mod, name):
    lp = check_device_case(ss, oracle_mod, name)
    tiers = {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")}
    print(name, tiers)
    if name == "clustered_overflow":
        assert tiers["avg_select"] > 0 and tiers["avg_4096"] >= tiers["avg_select"]


def test_cuda_averaged_dam_break_1m(ss):
    """1 M-particle dam break (cfg-4 proportions): closed and manifold, identical across two runs, densities of the standard run."""
    from splashsurf_b200 import synthetic as syn
    p = syn.dam_break_scaled(1_000_000)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        a = ss.reconstruct_surface(p, context=ctx, averaged_surface=ss.AveragedSurface(), with_debug=True, **kw)
        b = ss.reconstruct_surface(p, context=ctx, averaged_surface=ss.AveragedSurface(), **kw)
        std = ss.reconstruct_surface(p, context=ctx, **kw)
    finally:
        ctx.close()
    assert a.mesh.nvertices > 100_000
    assert np.array_equal(a.mesh.vertices, b.mesh.vertices) and np.array_equal(a.mesh.triangles, b.mesh.triangles)
    assert np.array_equal(a.particle_densities, std.particle_densities)
    rep = ss.check_mesh_consistency(a.mesh, a.grid, check_closed=True, check_manifold=True)
    assert rep is None, rep
    assert a.levelset_paths["avg_512"] > 0
    # no spurious blobs: a grid point read inside with nothing there becomes a closed component of a few vertices about h from the
    # fluid (one inside point: 6 vertices), while a lone particle's sphere of radius R_s = 2 cells has dozens; and every vertex lies
    # within c of an inside grid point, which has a particle within h: no vertex is farther than h + c from every particle
    from scipy.spatial import cKDTree
    from test_averaged_surface import mesh_topology
    ncomp, closed, _ = mesh_topology(a.mesh.triangles)
    sizes = np.bincount(_vertex_components(a.mesh.triangles, a.mesh.nvertices))
    dist, _ = cKDTree(p.astype(np.float64)).query(a.mesh.vertices.astype(np.float64))
    h, c, rs = 0.04, 0.005, 0.01
    print(f"dam break 1M averaged: {ncomp} components, smallest {sizes[sizes > 0].min()} vertices, vertex-particle distance "
          f"max {dist.max():.5f} (R_s = {rs}, h = {h}), beyond R_s + c: {(dist > rs + c).sum()}")
    assert closed and sizes[sizes > 0].min() >= 24, sorted(sizes[sizes > 0])[:10]
    assert dist.max() <= (h + c) * (1 + 1e-5)


def _vertex_components(tris, nv):
    """Component label of every vertex of a triangle mesh (isolated vertices get labels of their own)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = np.asarray(tris, np.int64)
    a, b = np.concatenate([t[:, 0], t[:, 1], t[:, 2]]), np.concatenate([t[:, 1], t[:, 2], t[:, 0]])
    return connected_components(coo_matrix((np.ones(len(a)), (a, b)), shape=(nv, nv)), directed=False)[1]
