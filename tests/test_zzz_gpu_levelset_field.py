"""The level set at arbitrary points and its derivatives (LevelSetField, DESIGN.md sections 13, 13.1 and 13.2) on the device: the
device cases of tests/test_levelset_field.py on the H100 (the field equals the reconstruction's tile in every mode, and every query
a mode supports -- values, gradients, Hessians, curvatures -- equals the point-scan oracle bit for bit, the tiers of each case
printed), host and device point arrays give identical values, and on a 1 M-particle dam break the two grid points of every mesh
vertex's edge straddle the threshold while 10 M random points are evaluated."""
import numpy as np
import pytest

from levelset_field_harness import (GRAD_MODES, MODES, _kw_abs, check_field_vs_oracle, check_field_vs_reconstruction, face_points,
                                    mode_kwargs, random_points, shell_points)
from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64", "tile_batch_1", "particle_aabb"])
def test_cuda_field_equals_reconstruction(ss, name, mode):
    check_field_vs_reconstruction(ss, name, mode)


@pytest.mark.parametrize("mode", MODES)
def test_cuda_points_equal_oracle(ss, mode):
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = ss.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 20000, 41), random_points(f.grid, 2000, 42, pad=0.3),
                          random_points(f.grid, 20000, 141), random_points(f.grid, 2000, 142, pad=0.3)])
    f.close()
    print(mode, check_field_vs_oracle(ss, p, kw, mode, pts))
    one = np.array([[0.1, 0.2, 0.3]], np.float32)
    print(mode, "lone particle", check_field_vs_oracle(ss, one, KW, mode, np.concatenate([shell_points(one[0], _kw_abs(KW)[1]), one])))


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_cuda_faces_and_last_cells_equal_oracle(ss, Rc):
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = ss.LevelSetField(p, **kw)
    pts = np.concatenate([face_points(f.grid, 16, 77 + Rc), face_points(f.grid, 16, 177 + Rc)])
    f.close()
    for mode in MODES:
        print(Rc, mode, check_field_vs_oracle(ss, p, kw, mode, pts))


@pytest.mark.parametrize("mode", ["sph", "avg", "corr"])
def test_cuda_clustered_reaches_select(ss, mode):
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(61).uniform(0.1, 0.3, (200, 3)).astype(np.float32),
                          np.random.default_rng(161).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    print(mode, check_field_vs_oracle(ss, p, kw, mode, pts, expect_tier="select"))


def test_cuda_outside_and_empty_inputs(ss):
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    none = np.zeros((0, 3), np.float32)
    for mode in MODES:
        grad = mode in GRAD_MODES
        f = ss.LevelSetField(p, **kw, **mode_kwargs(ss, mode, p, kw))
        try:
            pts = np.concatenate([random_points(f.grid, 5000, 51, pad=2.0), random_points(f.grid, 5000, 151, pad=2.0)])
            lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
            out = np.any((pts < lo) | (pts > hi), axis=1)
            inside = random_points(f.grid, 3000, 152)
            assert np.all(f.evaluate(pts)[out] == 0.0) and f.evaluate(none).shape == (0,)
            if grad:
                v, g, H = f.hessian(pts)
                assert np.all(v[out] == 0.0) and np.all(g[out] == 0.0) and np.all(H[out] == 0.0)
                assert np.all(np.isnan(f.curvature(pts)[0][out]))
                v, g, H = f.hessian(none)
                assert v.shape == (0,) and g.shape == (0, 3) and H.shape == (0, 6)
        finally:
            f.close()
        print(mode, "empty subdomains", check_field_vs_oracle(ss, p, kw, mode, inside))
    f = ss.LevelSetField(none, **KW)
    v, g, H = f.hessian(np.array([[0, 0, 0], [1, 1, 1]], np.float32))
    assert np.all(v == 0.0) and np.all(g == 0.0) and np.all(H == 0.0)
    kh, kg = f.curvature(np.array([[0, 0, 0]], np.float32))
    assert np.isnan(kh).all() and np.isnan(kg).all()
    f.close()


def test_cuda_host_and_device_points_agree(ss):
    import torch
    p = _cube(12, 881)
    f = ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(), **KW)
    try:
        pts = random_points(f.grid, 50000, 882, pad=0.1)
        host = f.evaluate(pts)
        dev = f.evaluate(torch.from_numpy(pts).cuda())
        assert dev.is_cuda and np.array_equal(host, dev.cpu().numpy())
    finally:
        f.close()


def test_cuda_dam_break_mesh_consistency(ss):
    """1 M-particle dam break, every mode: the end points of each vertex's grid edge lie on opposite sides of the threshold, and
    10 M uniform points evaluate with the outside ones at exactly 0."""
    from splashsurf_b200 import synthetic as syn
    x = syn.dam_break_scaled(1_000_000, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        for mode in MODES:
            mk = mode_kwargs(ss, mode, x, kw)
            g = ss.reconstruct_surface(x, context=ctx, with_debug=True, simd=False, subdomain_grid_auto_disable=False, **kw, **mk)
            f = ss.LevelSetField(x, context=ctx, **kw, **mk)
            assert np.array_equal(f.particle_densities, g.particle_densities)
            keys = np.asarray(g.vertex_edge_keys, np.int64).reshape(-1, 4)
            a = keys[:, :3].astype(np.float32)
            b = a.copy()
            b[np.arange(len(b)), keys[:, 3]] += 1
            lo, c = np.asarray(g.grid.aabb.min, np.float32), np.float32(g.grid.cell_size)
            va, vb = f.evaluate((lo + a * c).astype(np.float32)), f.evaluate((lo + b * c).astype(np.float32))
            assert len(keys) > 1000 and np.all((va > f.threshold) != (vb > f.threshold)), mode
            pts = random_points(f.grid, 10_000_000, 883, pad=0.05)
            v = f.evaluate(pts)
            outside = np.any((pts < np.asarray(f.grid.aabb.min)) | (pts > np.asarray(f.grid.aabb.max)), axis=1)
            assert np.all(v[outside] == 0.0) and np.isfinite(v).all() and (v > f.threshold).any()
            print(mode, f.paths, g.mesh.nvertices)
            f.close()
    finally:
        ctx.close()
