"""Per-particle radii of the averaged-position surface (reconstruct_surface(particle_radii=...), DESIGN.md section 12.2) on the device:
the mesh, the densities and the kept level-set tile equal the C oracle bit for bit, plain and corrected, with the tier of the
warp-per-brick cascade each case took read back; host and device radii give identical results; a 1 M-particle dam break with radii
in [0.8, 1.2] r gives a closed, manifold, reproducible mesh with the standard run's densities."""
import ctypes as C

import numpy as np
import pytest

from test_averaged_radii import check_device_case, seeded_radii
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_radii_match_oracle(ss, oracle_mod, name, corrected):
    lp = check_device_case(ss, oracle_mod, name, corrected)
    tiers = {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")}
    print(name, "corrected" if corrected else "plain", tiers)
    if name == "clustered_overflow":
        assert tiers["avg_select"] > 0 and tiers["avg_4096"] >= tiers["avg_select"]


def _vertices(ss, ctx, p, params):
    L = ctx._L
    s = ctx.reconstruct_raw(p.ctypes.data, len(p), params)
    try:
        v = np.empty((L.ss_surface_num_vertices(s), 3), np.float32)
        ss._check(L, L.ss_surface_copy_vertices(s, v.ctypes.data))
        return v
    finally:
        L.ss_surface_free(s)


def test_cuda_host_and_device_radii_agree(ss):
    """The setter takes host or device memory: a torch CUDA tensor gives the mesh of the numpy array, and the context keeps its own
    copy (the tensor is overwritten before the reconstruction)."""
    import torch
    from test_anisotropic import KW, _cube
    p = _cube(12, 871)
    radii = seeded_radii(len(p), 872, KW["particle_radius"])
    av = ss.AveragedSurface()
    want = ss.reconstruct_surface(p, averaged_surface=av, particle_radii=radii, **KW)
    ctx = ss.Context()
    L = ctx._L
    try:
        dev = torch.from_numpy(radii).cuda()
        torch.cuda.synchronize()
        ss._check(L, L.ss_context_set_averaged_surface_f32(ctx._h, C.byref(av._abi())))
        ss._check(L, L.ss_context_set_averaged_radii_f32(ctx._h, dev.data_ptr(), dev.shape[0]))
        dev.fill_(float("nan"))
        torch.cuda.synchronize()
        v = _vertices(ss, ctx, p, ss.make_params(**KW))
    finally:
        ctx.close()
    assert np.array_equal(v, want.mesh.vertices)


@pytest.mark.parametrize("corrected", [False, True], ids=["plain", "corrected"])
def test_cuda_radii_dam_break_1m(ss, corrected):
    """1 M-particle dam break (cfg-4 proportions), radii uniform in [0.8, 1.2] r: closed and manifold, identical across two runs,
    densities of the standard run."""
    from splashsurf_b200 import synthetic as syn
    p = syn.dam_break_scaled(1_000_000)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    radii = seeded_radii(len(p), 873, 0.01, 0.8, 1.2)
    av = ss.AveragedSurface(correction=ss.JacobianCorrection() if corrected else None)
    ctx = ss.Context()
    try:
        a = ss.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=radii, with_debug=True, **kw)
        b = ss.reconstruct_surface(p, context=ctx, averaged_surface=av, particle_radii=radii, **kw)
        std = ss.reconstruct_surface(p, context=ctx, **kw)
    finally:
        ctx.close()
    assert a.mesh.nvertices > 100_000
    assert np.array_equal(a.mesh.vertices, b.mesh.vertices) and np.array_equal(a.mesh.triangles, b.mesh.triangles)
    assert np.array_equal(a.particle_densities, std.particle_densities)
    rep = ss.check_mesh_consistency(a.mesh, a.grid, check_closed=True, check_manifold=True)
    assert rep is None, rep
    lp = a.levelset_paths
    print(f"dam break 1M radii {'corrected' if corrected else 'plain'}:", a.mesh.nvertices, "vertices,",
          {k: lp[k] for k in ("avg_512", "avg_4096", "avg_select")})
    assert lp["avg_512"] > 0
