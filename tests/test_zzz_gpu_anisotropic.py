"""Anisotropic kernels (splashsurf_b200.Anisotropy, DESIGN.md section 11) on the device: smoothed centres, G matrices and the mesh
equal the C oracle bit for bit; densities equal the isotropic run's bit for bit; a 1 M-particle dam break gives a closed, manifold,
reproducible mesh."""
import numpy as np
import pytest

from test_anisotropic import CASES, check_device_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_anisotropic_matches_oracle(ss, oracle_mod, name):
    check_device_case(ss, oracle_mod, name)


def test_cuda_anisotropic_dam_break_1m(ss):
    """1 M-particle dam break (cfg-4 proportions): closed and manifold, identical across two runs, densities of the isotropic run."""
    from splashsurf_b200 import synthetic as syn
    p = syn.dam_break_scaled(1_000_000)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        a = ss.reconstruct_surface(p, context=ctx, anisotropy=ss.Anisotropy(), **kw)
        b = ss.reconstruct_surface(p, context=ctx, anisotropy=ss.Anisotropy(), **kw)
        iso = ss.reconstruct_surface(p, context=ctx, **kw)
    finally:
        ctx.close()
    assert a.mesh.nvertices > 100_000
    assert np.array_equal(a.mesh.vertices, b.mesh.vertices) and np.array_equal(a.mesh.triangles, b.mesh.triangles)
    assert np.array_equal(a.smoothed_particles, b.smoothed_particles) and np.array_equal(a.anisotropy_matrices, b.anisotropy_matrices)
    assert np.array_equal(a.particle_densities, iso.particle_densities)
    rep = ss.check_mesh_consistency(a.mesh, a.grid, check_closed=True, check_manifold=True)
    assert rep is None, rep
    assert a.timings["anisotropy"] > 0.0
