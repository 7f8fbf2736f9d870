"""The Hessian and curvature of the level set at arbitrary points (LevelSetField.hessian / .curvature, DESIGN.md section 13.2) on
the device (the device-versus-oracle cases of every query live in tests/test_zzz_gpu_levelset_field.py): host and device point
arrays give identical results, and on a 1 M-particle dam break in every mode with a Hessian the values and gradients equal
evaluate() and gradient() at the mesh vertices and at 10 M uniform points, value, gradient and Hessian are 0 outside the grid, and
the curvature is finite at every vertex with a nonzero gradient."""
import numpy as np
import pytest

from levelset_field_harness import GRAD_MODES as MODES, _ball, _same, mode_kwargs, random_points
from test_anisotropic import KW, R, _cube

pytestmark = pytest.mark.gpu


def test_cuda_host_and_device_points_agree(ss):
    import torch
    p = _cube(12, 881)
    for mode in MODES:
        f = ss.LevelSetField(p, **KW, **mode_kwargs(ss, mode, p, KW))
        try:
            pts = random_points(f.grid, 50000, 882, pad=0.1)
            dev = torch.from_numpy(pts).cuda()
            for h, d in zip(f.hessian(pts), f.hessian(dev)):
                assert d.is_cuda and np.array_equal(h.view(np.uint32), d.cpu().numpy().view(np.uint32))
            for h, d in zip(f.curvature(pts), f.curvature(dev)):
                assert d.is_cuda and d.shape == (len(pts),) and _same(h, d.cpu().numpy())
        finally:
            f.close()


def test_cuda_refusals(ss):
    p = _cube(6, 5)
    for corr_rad in (False, True):
        mk = dict(averaged_surface=ss.AveragedSurface(1.0, ss.JacobianCorrection()))
        if corr_rad:
            mk["particle_radii"] = np.full(len(p), np.float32(R))
        f = ss.LevelSetField(p, **KW, **mk)
        try:
            for call in (f.hessian, f.curvature):
                with pytest.raises(ss.SplashsurfError, match="no Hessian") as e:
                    call(random_points(f.grid, 10, 3))
                assert e.value.code == 7
        finally:
            f.close()


@pytest.mark.parametrize("mode", MODES)
def test_cuda_pipeline_levelset_curvature(ss, mode):
    p = _ball(0.1, 111)
    mk = mode_kwargs(ss, mode, p, KW)
    mesh, _ = ss.reconstruction_pipeline(p, levelset_curvature=True, mesh_smoothing_iters=2, **KW, **mk)
    f = ss.LevelSetField(p, **KW, **mk)
    try:
        kh, kg = f.curvature(np.ascontiguousarray(mesh.mesh.vertices, np.float32))
    finally:
        f.close()
    assert _same(mesh.point_attributes["mean_curvature"], kh) and _same(mesh.point_attributes["gaussian_curvature"], kg)
    rad = np.median(np.linalg.norm(mesh.mesh.vertices.astype(np.float64) - p.astype(np.float64).mean(0), axis=1))
    print(mode, "ball: median kappa_H * median radius", float(np.median(kh) * rad))


def test_cuda_dam_break(ss):
    """1 M-particle dam break, every mode with a Hessian: values and gradients equal evaluate() and gradient() bit for bit at the
    mesh vertices and at 10 M uniform points, value, gradient and Hessian are 0 outside the grid, and the curvature is finite at every
    vertex with a nonzero gradient.  Prints the tiers and the fraction of finite curvatures."""
    import torch
    from splashsurf_b200 import synthetic as syn
    x = syn.dam_break_scaled(1_000_000, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        for mode in MODES:
            mk = mode_kwargs(ss, mode, x, kw)
            g = ss.reconstruct_surface(x, context=ctx, subdomain_grid_auto_disable=False, **kw, **mk)
            f = ss.LevelSetField(x, context=ctx, **kw, **mk)
            v = g.mesh.vertices
            val, grad, H = f.hessian(v)
            assert np.array_equal(val.view(np.uint32), f.evaluate(v).view(np.uint32))
            assert np.array_equal(grad.view(np.uint32), f.gradient(v)[1].view(np.uint32))
            kh, kg = f.curvature(v)
            nz = np.any(grad != 0, axis=1)
            assert np.isfinite(kh[nz]).all() and np.isfinite(kg[nz]).all(), mode
            pts = torch.from_numpy(random_points(f.grid, 10_000_000, 883, pad=0.05)).cuda()
            pv, pg, pH = f.hessian(pts)
            paths = f.paths
            assert torch.equal(pv, f.evaluate(pts)) and torch.equal(pg, f.gradient(pts)[1])
            lo = torch.tensor(f.grid.aabb.min, device=pts.device, dtype=torch.float32)
            hi = torch.tensor(f.grid.aabb.max, device=pts.device, dtype=torch.float32)
            out = ((pts < lo) | (pts > hi)).any(1)
            assert bool((pv[out] == 0).all()) and bool((pg[out] == 0).all()) and bool((pH[out] == 0).all())
            print(mode, "vertices", len(v), "nonzero gradient", int(nz.sum()), "median kappa_H", float(np.median(kh[nz])), "tiers", paths)
            f.close()
            del pts, pv, pg, pH
    finally:
        ctx.close()
