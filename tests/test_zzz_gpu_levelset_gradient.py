"""The gradient of the level set at arbitrary points (LevelSetField.gradient / .normals, DESIGN.md section 13.1) on the device: the
device cases of tests/test_levelset_gradient.py on the H100 (values and gradients equal the point-scan oracle bit for bit, values
equal evaluate() bit for bit, the tier of each case printed), host and device point arrays give identical results, and on a
1 M-particle dam break in every mode with a gradient the normals at the mesh vertices are finite and agree in orientation with the
area-weighted normals, while 10 M uniform points have value and gradient 0 outside the grid."""
import time

import numpy as np
import pytest

from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_surface import CASES
from test_levelset_field import _kw_abs, face_points, mode_kwargs, random_points, shell_points
from test_levelset_gradient import MODES, check_gradient_vs_oracle

pytestmark = pytest.mark.gpu

AREA_AGREEMENT = 0.95            # least fraction of dam-break vertices whose level-set normal faces like the area-weighted one


@pytest.mark.parametrize("mode", MODES)
def test_cuda_points_equal_oracle(ss, mode):
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = ss.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 20000, 41), random_points(f.grid, 2000, 42, pad=0.3)])
    f.close()
    print(mode, check_gradient_vs_oracle(ss, p, kw, mode, pts))
    one = np.array([[0.1, 0.2, 0.3]], np.float32)
    print(mode, "lone particle", check_gradient_vs_oracle(ss, one, KW, mode, np.concatenate([shell_points(one[0], _kw_abs(KW)[1]), one])))


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_cuda_faces_and_last_cells_equal_oracle(ss, Rc):
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = ss.LevelSetField(p, **kw)
    pts = face_points(f.grid, 16, 77 + Rc)
    f.close()
    for mode in MODES:
        print(Rc, mode, check_gradient_vs_oracle(ss, p, kw, mode, pts))


@pytest.mark.parametrize("mode", ["sph", "avg"])
def test_cuda_clustered_reaches_select(ss, mode):
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(61).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    print(mode, check_gradient_vs_oracle(ss, p, kw, mode, pts, expect_tier="select"))


def test_cuda_outside_and_empty_inputs(ss):
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    for mode in MODES:
        f = ss.LevelSetField(p, **kw, **mode_kwargs(ss, mode, p, kw))
        try:
            pts = random_points(f.grid, 5000, 51, pad=2.0)
            lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
            out = np.any((pts < lo) | (pts > hi), axis=1)
            v, g = f.gradient(pts)
            assert np.all(v[out] == 0.0) and np.all(g[out] == 0.0)
            v, g = f.gradient(np.zeros((0, 3), np.float32))
            assert v.shape == (0,) and g.shape == (0, 3)
        finally:
            f.close()
    f = ss.LevelSetField(np.zeros((0, 3), np.float32), **KW)
    v, g = f.gradient(np.array([[0, 0, 0], [1, 1, 1]], np.float32))
    assert np.all(v == 0.0) and np.all(g == 0.0)
    f.close()


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
    from test_levelset_gradient import _ball
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
