"""The Hessian and curvature of the level set at arbitrary points (LevelSetField.hessian / .curvature, DESIGN.md section 13.2) on
the device: the device cases of tests/test_levelset_curvature.py on the H100 (values, gradients, Hessians and curvatures equal the
point-scan oracle bit for bit, values and gradients equal evaluate() and gradient() bit for bit, the tier of each case printed),
host and device point arrays give identical results, and on a 1 M-particle dam break in every mode with a Hessian the values and
gradients equal evaluate() and gradient() at the mesh vertices and at 10 M uniform points, value, gradient and Hessian are 0 outside
the grid, and the curvature is finite at every vertex with a nonzero gradient."""
import numpy as np
import pytest

from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_surface import CASES
from test_levelset_curvature import _same, check_hessian_vs_oracle
from test_levelset_field import _kw_abs, face_points, mode_kwargs, random_points, shell_points
from test_levelset_gradient import MODES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", MODES)
def test_cuda_points_equal_oracle(ss, mode):
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = ss.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 20000, 141), random_points(f.grid, 2000, 142, pad=0.3)])
    f.close()
    print(mode, check_hessian_vs_oracle(ss, p, kw, mode, pts))
    one = np.array([[0.1, 0.2, 0.3]], np.float32)
    print(mode, "lone particle", check_hessian_vs_oracle(ss, one, KW, mode, np.concatenate([shell_points(one[0], _kw_abs(KW)[1]), one])))


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_cuda_faces_and_last_cells_equal_oracle(ss, Rc):
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = ss.LevelSetField(p, **kw)
    pts = face_points(f.grid, 16, 177 + Rc)
    f.close()
    for mode in MODES:
        print(Rc, mode, check_hessian_vs_oracle(ss, p, kw, mode, pts))


@pytest.mark.parametrize("mode", ["sph", "avg"])
def test_cuda_clustered_reaches_select(ss, mode):
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(161).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    print(mode, check_hessian_vs_oracle(ss, p, kw, mode, pts, expect_tier="select"))


def test_cuda_outside_and_empty_inputs(ss):
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    for mode in MODES:
        mk = mode_kwargs(ss, mode, p, kw)
        f = ss.LevelSetField(p, **kw, **mk)
        try:
            pts = random_points(f.grid, 5000, 151, pad=2.0)
            lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
            out = np.any((pts < lo) | (pts > hi), axis=1)
            v, g, H = f.hessian(pts)
            assert np.all(v[out] == 0.0) and np.all(g[out] == 0.0) and np.all(H[out] == 0.0)
            assert np.all(np.isnan(f.curvature(pts)[0][out]))
            inside = random_points(f.grid, 3000, 152)
            print(mode, "empty subdomains", check_hessian_vs_oracle(ss, p, kw, mode, inside))
            v, g, H = f.hessian(np.zeros((0, 3), np.float32))
            assert v.shape == (0,) and g.shape == (0, 3) and H.shape == (0, 6)
        finally:
            f.close()
    f = ss.LevelSetField(np.zeros((0, 3), np.float32), **KW)
    v, g, H = f.hessian(np.array([[0, 0, 0], [1, 1, 1]], np.float32))
    assert np.all(v == 0.0) and np.all(g == 0.0) and np.all(H == 0.0)
    kh, kg = f.curvature(np.array([[0, 0, 0]], np.float32))
    assert np.isnan(kh).all() and np.isnan(kg).all()
    f.close()


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
    from test_levelset_gradient import _ball
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
