"""The level set at arbitrary points (LevelSetField / ss_levelset_field_*_f32, DESIGN.md section 13), on the CPU executor of the CUDA
sources (also run with SS_EMUL_GUARD=1):

* the point-scan oracle (tests/levelset_field_oracle.c) at points that are not grid points, against the float64 restatements of the
  averaged and corrected surfaces within their per-point bounds;
* the device equals the oracle bit for bit at random points, at points on tile, brick and bin faces and in the last cell of a brick
  for R = 1, 6, 7, 8, 9, 17, at 0.9 / 0.97 / 0.995 h from a lone particle in 26 directions, outside the grid and in empty
  subdomains (exactly 0), for m = 0 and n = 0, and in the clustered case that reaches the selection walk;
* the device equals the reconstruction's level-set tile bit for bit at the tile's own f32 grid coordinates (the standard level set
  with simd = False), and the densities are the reconstruction's;
* the two grid points of every mesh vertex's edge lie on opposite sides of the threshold;
* refusals, NaN points, a stale handle and one context reused across handles and reconstructions.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_field.py."""
import numpy as np
import pytest

from levelset_field_harness import (GRAD_MODES, MODES, _kw_abs, check_field_vs_oracle, check_field_vs_reconstruction, face_points,
                                    mode_kwargs, oracle_field, random_points, shell_points)
from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_correction import numpy_corrected
from test_averaged_surface import CASES, ORACLE_CLOUDS, numpy_averaged
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)


# ------------------------------------------------------------------ oracle vs float64 ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_oracle_within_float64_bounds_off_grid(cloud):
    """At random points that are not grid points the point-scan oracle lies within the float64 per-point bounds of DESIGN.md
    sections 12 (averaged) and 12.1 (corrected)."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, c = _kw_abs(KW)
    lo, hi = p.min(0) - float(h), p.max(0) + float(h)
    pts = np.random.default_rng(31).uniform(lo, hi, (3000, 3)).astype(np.float32)
    v = oracle_field(p, KW, "avg", pts)[0]
    f, n, bound = numpy_averaged(p, pts, float(h))
    m = n > 0
    assert np.all(v[~m] == 0.0) and m.sum() > 300
    assert np.all(np.abs(v[m] - f[m]) <= bound[m])
    v = oracle_field(p, KW, "corr", pts)[0]
    val, _ev, _fv, _plain, n, bound = numpy_corrected(p, pts, float(h), float(r))
    m = n > 0
    assert np.all(np.abs(v[m] - val[m]) <= bound[m])


# ------------------------------------------------------------------ device (CPU executor) ----
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64", "tile_batch_1", "particle_aabb"])
def test_emulated_field_equals_reconstruction(emu, name, mode):  # noqa: F811
    check_field_vs_reconstruction(emu, name, mode)


# Device == point-scan oracle for every query a mode supports (levelset_field_harness.check_field_vs_oracle).  Each case runs the
# point sets of two seed families at once.
@pytest.mark.parametrize("mode", MODES)
def test_emulated_random_points_equal_oracle(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = emu.LevelSetField(p, **kw)
    pts = np.concatenate([random_points(f.grid, 3000, 41), random_points(f.grid, 300, 42, pad=0.3),
                          random_points(f.grid, 2000, 141), random_points(f.grid, 200, 142, pad=0.3)])
    f.close()
    tiers = check_field_vs_oracle(emu, p, kw, mode, pts)
    assert all(t["512"] > 0 for t in tiers.values()), tiers


@pytest.mark.parametrize("mode", ["sph", "avg"])
@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_emulated_faces_and_last_cells_equal_oracle(emu, Rc, mode):  # noqa: F811
    """Points on tile, brick and bin faces and in the last cell of a brick at R = ceil(h / c) = Rc: the group's candidate bins
    must reach one cell past the brick's grid points."""
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f = emu.LevelSetField(p, **kw)
    assert int(np.ceil(np.float32(4 * R) / np.float32(f.grid.cell_size))) == Rc
    pts = np.concatenate([face_points(f.grid, 16, 77 + Rc), face_points(f.grid, 16, 177 + Rc)])
    f.close()
    check_field_vs_oracle(emu, p, kw, mode, pts)


@pytest.mark.parametrize("mode", MODES)
def test_emulated_lone_particle_shells(emu, mode):  # noqa: F811
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    _, h, _ = _kw_abs(KW)
    check_field_vs_oracle(emu, p, KW, mode, np.concatenate([shell_points(p[0], h), p]))


@pytest.mark.parametrize("mode", MODES)
def test_emulated_outside_and_empty_subdomains_are_zero(emu, mode):  # noqa: F811
    """Points outside the grid, far away, and in subdomains without members (the droplets' gaps) have value, gradient and Hessian
    exactly 0 and a NaN curvature; empty point arrays give empty outputs of the right shapes; a field without particles is 0
    everywhere with NaN normals; a field with particles but no points reaches no tier."""
    gen, kw, _ = CASES["droplets_sparse"]
    p = gen()
    grad = mode in GRAD_MODES
    f = emu.LevelSetField(p, **kw, **mode_kwargs(emu, mode, p, kw))
    try:
        far = np.array([[1e6, 0, 0], [-1e6, 5, 5], [0, 0, 3e38]], np.float32)
        lo, hi = np.asarray(f.grid.aabb.min), np.asarray(f.grid.aabb.max)
        outside = np.concatenate([random_points(f.grid, 500, 51, pad=2.0), random_points(f.grid, 500, 151, pad=2.0)])
        outside = np.concatenate([far, outside[np.any((outside < lo) | (outside > hi), axis=1)]])
        inside = np.concatenate([random_points(f.grid, 4000, 52), random_points(f.grid, 3000, 152)])
        for pts, least in ((outside, len(outside)), (inside, 101)):
            v = f.evaluate(pts)
            empty = v == 0
            if grad:
                _, g, H = f.hessian(pts)
                empty &= np.all(g == 0, axis=1) & np.all(H == 0, axis=1)
                assert np.all(np.isnan(f.curvature(pts[empty])[0]))
            assert empty.sum() >= least, (empty.sum(), least)
    finally:
        f.close()
    check_field_vs_oracle(emu, p, kw, mode, inside)
    none = np.zeros((0, 3), np.float32)

    def no_points(f):
        assert f.evaluate(none).shape == (0,)
        if grad:
            v, g, H = f.hessian(none)
            kh, kg = f.curvature(none)
            assert v.shape == (0,) and g.shape == (0, 3) and H.shape == (0, 6) and kh.shape == (0,) and kg.shape == (0,)
    f = emu.LevelSetField(none, **KW, **mode_kwargs(emu, mode, none, KW))
    try:
        no_points(f)
        pts = np.array([[0, 0, 0], [1, 1, 1]], np.float32)
        assert np.all(f.evaluate(pts) == 0.0) and len(f.particle_densities) == 0
        if grad:
            v, g, H = f.hessian(pts)
            assert np.all(v == 0.0) and np.all(g == 0.0) and np.all(H == 0.0)
            assert np.all(np.isnan(f.curvature(pts)[0])) and np.all(np.isnan(f.normals(pts[:1])))
    finally:
        f.close()
    p = _cube(5, 3)
    f = emu.LevelSetField(p, **KW, **mode_kwargs(emu, mode, p, KW))
    try:
        no_points(f)
        assert f.paths == {"512": 0, "4096": 0, "select": 0}
    finally:
        f.close()


@pytest.mark.parametrize("mode", ["sph", "avg", "corr"])
def test_emulated_clustered_reaches_select(emu, mode):  # noqa: F811
    """4400 particles in a ball of 0.6 h: the groups inside it exceed the 4096-slot slice and go to the selection walk."""
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    _, h, _ = _kw_abs(kw)
    pts = np.concatenate([shell_points(np.full(3, 0.2), h * np.float32(0.5)),
                          np.random.default_rng(61).uniform(0.1, 0.3, (200, 3)).astype(np.float32),
                          np.random.default_rng(161).uniform(0.1, 0.3, (200, 3)).astype(np.float32)])
    check_field_vs_oracle(emu, p, kw, mode, pts, expect_tier="select")


def test_emulated_refusals_and_reuse(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    with pytest.raises(TypeError):
        ss.LevelSetField(p.astype(np.float64), **KW)
    with pytest.raises(ss.SplashsurfError, match="error 1"):
        ss.LevelSetField(p, **dict(KW, cube_size=0.0))
    with pytest.raises(ss.SplashsurfError, match="radius_factor"):
        ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(100.0), **KW)
    with pytest.raises(ss.SplashsurfError, match="exclusive"):
        ss.LevelSetField(p, anisotropy=ss.Anisotropy(), averaged_surface=ss.AveragedSurface(), **KW)
    bad = np.full(len(p), np.float32(KW["particle_radius"]))
    bad[3] = np.nan
    with pytest.raises(ss.SplashsurfError, match="index 3"):
        ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(), particle_radii=bad, **KW)
    with pytest.raises(ValueError):
        ss.LevelSetField(p, particle_radii=bad, **KW)
    ctx = ss.Context()
    try:
        f1 = ss.LevelSetField(p, context=ctx, **KW)
        pts = random_points(f1.grid, 100, 71)
        v1 = f1.evaluate(pts)
        nan = pts.copy()
        nan[17, 1] = np.nan
        nan[40, 0] = np.inf
        with pytest.raises(ss.SplashsurfError, match="point 17"):
            f1.evaluate(nan)
        with pytest.raises(TypeError):
            f1.evaluate(pts.astype(np.float64))
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f1.evaluate(pts)
        f2 = ss.LevelSetField(p, context=ctx, averaged_surface=ss.AveragedSurface(), **KW)
        f3 = ss.LevelSetField(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f2.evaluate(pts)
        assert np.array_equal(f3.evaluate(pts), v1)
        for f in (f1, f2, f3):
            f.close()
        # the context's own settings are untouched: a reconstruction afterwards is the standard one
        g = ss.reconstruct_surface(p, context=ctx, **KW)
        assert np.array_equal(g.mesh.vertices, ss.reconstruct_surface(p, **KW).mesh.vertices)
    finally:
        ctx.close()
