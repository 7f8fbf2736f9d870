"""Jacobian correction of the averaged-position surface (splashsurf_b200.JacobianCorrection, DESIGN.md section 12.1) on the device:
the mesh, the densities and the kept level-set tile equal the C oracle bit for bit, the densities equal the standard run's, and the
tier of the warp-per-brick cascade each case took is read back; a 1 M-particle dam break gives a closed, manifold, reproducible mesh."""
import numpy as np
import pytest

from test_averaged_correction import check_device_case
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_corrected_matches_oracle(ss, oracle_mod, name):
    lp = check_device_case(ss, oracle_mod, name)
    tiers = {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")}
    print(name, tiers)
    if name == "clustered_overflow":
        assert tiers["avg_select"] > 0 and tiers["avg_4096"] >= tiers["avg_select"]


def test_cuda_corrected_dam_break_1m(ss):
    """1 M-particle dam break (cfg-4 proportions): closed and manifold, identical across two runs, densities of the standard run."""
    from splashsurf_b200 import synthetic as syn
    p = syn.dam_break_scaled(1_000_000)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    av = ss.AveragedSurface(correction=ss.JacobianCorrection())
    ctx = ss.Context()
    try:
        a = ss.reconstruct_surface(p, context=ctx, averaged_surface=av, with_debug=True, **kw)
        b = ss.reconstruct_surface(p, context=ctx, averaged_surface=av, **kw)
        std = ss.reconstruct_surface(p, context=ctx, **kw)
    finally:
        ctx.close()
    assert a.mesh.nvertices > 100_000
    assert np.array_equal(a.mesh.vertices, b.mesh.vertices) and np.array_equal(a.mesh.triangles, b.mesh.triangles)
    assert np.array_equal(a.particle_densities, std.particle_densities)
    rep = ss.check_mesh_consistency(a.mesh, a.grid, check_closed=True, check_manifold=True)
    assert rep is None, rep
    lp = a.levelset_paths
    print("dam break 1M corrected:", a.mesh.nvertices, "vertices,", {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")})
    assert lp["avg_512"] > 0
