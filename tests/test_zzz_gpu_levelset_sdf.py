"""Narrow-band signed distance grids (LevelSetField.signed_distance, DESIGN.md section 14) on the H100: the device cases of
tests/test_levelset_sdf.py against the brute-force oracle with the tiers printed, host against device arrays, and a 1 M-particle
dam break in every mode at band 3 -- the properties of section 14 at every listed point and edge, and bit equality on 200 random
listed bricks (the oracle gets the triangles near each brick; the signs come from field.evaluate, which equals its own oracle)."""
import numpy as np
import pytest

from levelset_field_harness import (SDF_MODES, assert_sdf_equal, check_properties, check_sdf_vs_oracle, mode_kwargs, oracle_distance,
                                    oracle_sdf, raw_case)
from test_anisotropic import KW, R, _cube
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", SDF_MODES)
@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64"])
def test_cuda_sdf_equals_oracle(ss, name, mode):
    gen, kw, _ = CASES[name]
    f, rec, got = check_sdf_vs_oracle(ss, gen(), dict(kw), mode, 3)
    print(name, mode, "listed", len(got.brick_coords), "tiers", got.paths)
    f.close()


@pytest.mark.parametrize("band", [1, 8])
def test_cuda_sdf_bands_equal_oracle(ss, band):
    gen, kw, _ = CASES["splash_S24"]
    check_sdf_vs_oracle(ss, gen(), dict(kw), "avg", band)[0].close()


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_cuda_sdf_cube_sizes_equal_oracle(ss, Rc):
    p = _cube(6, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    check_sdf_vs_oracle(ss, p, kw, "sph", 3)[0].close()


def test_cuda_fan_takes_global_walk(ss):
    p = _cube(5, 11)
    f = ss.LevelSetField(p, **KW)
    try:
        lo, c = np.asarray(f.grid.aabb.min, np.float32), np.float32(f.grid.cell_size)
        ctr = (lo + np.float32(12) * c).astype(np.float32) * np.ones(3, np.float32)
        ang = np.linspace(0, 2 * np.pi, 401)[:-1]
        rim = np.stack([ctr + 0.6 * c * np.array([np.cos(a), np.sin(a), 0.3 * np.sin(3 * a)]) for a in ang]).astype(np.float32)
        v = np.concatenate([ctr[None], rim]).astype(np.float32)
        t = np.array([[0, 1 + k, 1 + (k + 1) % 400] for k in range(400)], np.uint64)
        got = f.signed_distance(ss.TriMesh3d(v, t), band=2)
        print("fan tiers", got.paths)
        assert got.paths["global"] > 0
        assert_sdf_equal(got, *oracle_sdf(p, KW, "sph", v, t, 2, f.grid, f.threshold), what="fan")
    finally:
        f.close()


def test_cuda_passes_equal_one_pass(ss):
    gen, kw, _ = CASES["splash_S24"]
    f, rec, _ = raw_case(ss, gen(), dict(kw), "sph")
    L = f._ctx._L
    try:
        one = f.signed_distance(rec.mesh)
        L.ss_sdf_set_pass_pairs(500)
        many = f.signed_distance(rec.mesh)
    finally:
        L.ss_sdf_set_pass_pairs(0)
        f.close()
    print("passes", one.passes, many.passes)
    assert many.passes["passes"] > 5 and many.passes["pairs"] == one.passes["pairs"]
    assert_sdf_equal(many, one.brick_coords, one.values, one.brick_inside, what="passes")


def test_cuda_host_and_device_arrays(ss):
    import torch
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec, _ = raw_case(ss, p, dict(kw), "avg")
    try:
        host = f.signed_distance(rec.mesh)
        v = torch.from_numpy(rec.mesh.vertices).cuda()
        for t in (torch.from_numpy(rec.mesh.triangles.astype(np.int64)).cuda(), torch.from_numpy(rec.mesh.triangles.astype(np.int32)).cuda()):
            dev = f.signed_distance((v, t))
            assert dev.values.is_cuda and dev.brick_coords.is_cuda and dev.brick_inside.is_cuda
            assert np.array_equal(dev.brick_coords.cpu().numpy(), host.brick_coords)
            assert np.array_equal(dev.values.cpu().numpy().view(np.uint32), host.values.view(np.uint32))
            assert np.array_equal(dev.brick_inside.cpu().numpy(), host.brick_inside)
            assert np.array_equal(dev.to_dense().view(np.uint32), host.to_dense().view(np.uint32))
        with pytest.raises(TypeError):
            f.signed_distance((v.double(), t))
    finally:
        f.close()


@pytest.mark.parametrize("mode", ["sph", "aniso", "avg", "corr", "rad"])
def test_cuda_dam_break(ss, mode):
    """1 M-particle dam break in every mode at band 3: the properties of section 14 everywhere, and bit equality on 200 random listed
    bricks against the oracle's distance to the triangles near each brick with the signs of field.evaluate."""
    from splashsurf_b200 import synthetic as syn
    x = syn.dam_break_scaled(1_000_000, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    mk = mode_kwargs(ss, mode, x, kw)
    rec = ss.reconstruct_surface(x, simd=False, subdomain_grid_auto_disable=False, with_debug=True, **kw, **mk)
    f = ss.LevelSetField(x, **kw, **mk)
    try:
        got = f.signed_distance(rec.mesh, band=3)
        print(mode, "triangles", rec.mesh.ncells, "listed", len(got.brick_coords), "tiers", got.paths, "passes", got.passes)
        check_properties(ss, f, rec, got)
        B, c = np.float32(got.background), np.float32(f.grid.cell_size)
        lo, npd = np.asarray(f.grid.aabb.min, np.float32), np.asarray(f.grid.npoints_per_dim)
        T = rec.mesh.vertices[rec.mesh.triangles.astype(np.int64)]
        tmin, tmax = T.min(1).astype(np.float64), T.max(1).astype(np.float64)
        reach = float(B) + float(c)
        for bi in np.random.default_rng(17).choice(len(got.brick_coords), min(200, len(got.brick_coords)), replace=False):
            b = got.brick_coords[bi].astype(np.int64)
            idx = 8 * b + np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)
            pts = (lo + idx.astype(np.float32) * c).astype(np.float32)
            near = np.all((tmax + reach >= pts.min(0)) & (tmin - reach <= pts.max(0)), axis=1)
            d = np.minimum(oracle_distance(rec.mesh.vertices, rec.mesh.triangles[near], pts), B)
            inside = f.evaluate(pts) > f.threshold
            want = np.where(np.all(idx < npd, axis=1), np.where(inside, -d, d), B).astype(np.float32)
            assert np.array_equal(got.values[bi].reshape(-1).view(np.uint32), want.view(np.uint32)), (mode, bi)
    finally:
        f.close()
