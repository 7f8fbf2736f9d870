"""The gradient of the level set at arbitrary points (LevelSetField.gradient / .normals, DESIGN.md section 13.1) on the device (the
device-versus-oracle cases of every query live in tests/test_zzz_gpu_levelset_field.py): host and device point arrays give identical
results, and on a 1 M-particle dam break in every mode with a gradient the normals at the mesh vertices are finite and agree in
orientation with the area-weighted normals, while 10 M uniform points have value and gradient 0 outside the grid."""
import time

import numpy as np
import pytest

from levelset_field_harness import GRAD_MODES as MODES, _ball, mode_kwargs, random_points
from test_anisotropic import KW, R, _cube

pytestmark = pytest.mark.gpu

AREA_AGREEMENT = 0.95            # least fraction of dam-break vertices whose level-set normal faces like the area-weighted one


def test_cuda_host_and_device_points_agree(ss):
    import torch
    p = _cube(12, 881)
    for mode in MODES:
        f = ss.LevelSetField(p, **KW, **mode_kwargs(ss, mode, p, KW))
        try:
            pts = random_points(f.grid, 50000, 882, pad=0.1)
            hv, hg = f.gradient(pts)
            dv, dg = f.gradient(torch.from_numpy(pts).cuda())
            assert dv.is_cuda and dg.is_cuda and dg.shape == (len(pts), 3)
            assert np.array_equal(hv, dv.cpu().numpy()) and np.array_equal(hg, dg.cpu().numpy())
            hn, dn = f.normals(pts), f.normals(torch.from_numpy(pts).cuda()).cpu().numpy()
            assert np.array_equal(np.isnan(hn), np.isnan(dn)) and np.allclose(hn[~np.isnan(hn)], dn[~np.isnan(dn)], atol=1e-6)
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
            with pytest.raises(ss.SplashsurfError, match="no gradient"):
                f.gradient(random_points(f.grid, 10, 3))
        finally:
            f.close()


@pytest.mark.parametrize("mode", ["aniso", "avg"])
def test_cuda_pipeline_levelset_normals(ss, mode):
    p = _ball(0.1, 111)
    mk = mode_kwargs(ss, mode, p, KW)
    mesh, _ = ss.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, **KW, **mk)
    area, _ = ss.reconstruction_pipeline(p, compute_normals=True, **KW, **mk)
    n, a = mesh.point_attributes["normals"], area.point_attributes["normals"]
    assert np.abs(np.linalg.norm(n, axis=1) - 1.0).max() < 1e-5 and np.all((n * a).sum(1) > 0)


def _area_normals(v, t):
    v = v.astype(np.float64)
    t = t.astype(np.int64)
    fn = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, t[:, k], fn)
    return n


def test_cuda_dam_break(ss):
    """1 M-particle dam break, every mode with a gradient: values equal evaluate() bit for bit at the mesh vertices and at 10 M
    uniform points, the normals at the vertices are finite and face like the area-weighted normals at no fewer than AREA_AGREEMENT of
    them, and outside the grid value and gradient are 0.  Prints the tiers, the agreement and the pipeline's time with and without
    levelset_normals."""
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
            val, grad = f.gradient(v)
            assert np.array_equal(val.view(np.uint32), f.evaluate(v).view(np.uint32))
            n = f.normals(v)
            assert np.isfinite(n).all(), mode
            agree = float(((n.astype(np.float64) * _area_normals(v, g.mesh.triangles)).sum(1) > 0).mean())
            pts = torch.from_numpy(random_points(f.grid, 10_000_000, 883, pad=0.05)).cuda()
            pv, pg = f.gradient(pts)
            paths = f.paths
            assert torch.equal(pv, f.evaluate(pts))
            lo = torch.tensor(f.grid.aabb.min, device=pts.device, dtype=torch.float32)
            hi = torch.tensor(f.grid.aabb.max, device=pts.device, dtype=torch.float32)
            out = ((pts < lo) | (pts > hi)).any(1)
            assert bool((pv[out] == 0).all()) and bool((pg[out] == 0).all()) and bool(torch.isfinite(pg).all())
            print(mode, "vertices", len(v), "area agreement", agree, "tiers", paths)
            assert agree >= AREA_AGREEMENT, (mode, agree)
            f.close()
            del pts, pv, pg
            if mode in ("aniso", "avg"):
                t = []
                for ln in (False, True, False, True):
                    t0 = time.perf_counter()
                    ss.reconstruction_pipeline(x, compute_normals=True, levelset_normals=ln, context=ctx, **kw, **mk)
                    t.append(time.perf_counter() - t0)
                print(mode, "pipeline s: area normals", min(t[0], t[2]), "levelset normals", min(t[1], t[3]))
    finally:
        ctx.close()
