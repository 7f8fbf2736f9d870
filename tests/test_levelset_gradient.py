"""The gradient of the level set at arbitrary points (LevelSetField.gradient / .normals, ss_levelset_field_gradient_at_f32,
DESIGN.md section 13.1), on the CPU executor of the CUDA sources (also run with SS_EMUL_GUARD=1):

* the float64 analytic gradient of every supported mode is the derivative of the float64 field (central differences);
* the f32 point-scan oracle (tests/levelset_field_oracle.c) lies within a per-point float64 bound at every point, including the
  1/u amplification at the edge of the support of the averaged modes, and in the narrow band around the surface its normal lies
  within a small angle of the float64 normal;
* the device equals the oracle bit for bit, and its values equal evaluate() bit for bit: the device-versus-oracle cases of every
  query live in tests/test_levelset_field.py;
* properties (radial normals of one particle, the standard mode against SphInterpolator.interpolate_normals, equal radii), refusals,
  and reconstruction_pipeline(levelset_normals=True) / reconstruct --levelset-normals=on.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_gradient.py."""
import os

import numpy as np
import pytest

import splashsurf_b200
from levelset_field_harness import (GRAD_MODES as MODES, U, _ball, _kw_abs, f64_field, f64_records, mode_kwargs, oracle_field, random_points,
                                    records)
from test_anisotropic import KW, _cube
from test_averaged_surface import CASES, ORACLE_CLOUDS
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)


# ------------------------------------------------------------------ 1. the formula is the derivative ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_formula_is_the_derivative(cloud):
    """The float64 analytic gradient of every supported mode against central differences of the float64 field (step 1e-5 h) at
    random off-grid points; only points with |m| < 1e-3 h (the kink of the norm, averaged modes) are left out."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    h = float(h)
    lo, hi = p.min(0) - h, p.max(0) + h
    pts = np.random.default_rng(91).uniform(lo, hi, (400, 3))
    for mode in MODES:
        radii = mode_kwargs(splashsurf_b200, mode, p, KW).get("particle_radii")
        ctr, w, g6, dlt = f64_records(p, KW, mode, radii)
        v, g, _, _ = f64_field(mode, ctr, w, g6, dlt, h, float(r), pts)
        step = 1e-5 * h
        fd = np.zeros_like(g)
        for a in range(3):
            e = np.zeros(3)
            e[a] = step
            fd[:, a] = (f64_field(mode, ctr, w, g6, dlt, h, float(r), pts + e)[0] - f64_field(mode, ctr, w, g6, dlt, h, float(r), pts - e)[0]) / (2 * step)
        keep = v != 0
        if mode in ("avg", "rad"):                             # |m| = h - the plain averaged value
            va = f64_field("avg", ctr, w, g6, dlt, h, float(r), pts)[0]
            keep &= (va != 0) & (h - va > 1e-3 * h)
        scale = np.linalg.norm(g[keep], axis=1).max()
        err = np.abs(g[keep] - fd[keep]).max()
        assert keep.sum() > 50 and err <= 1e-6 * scale, (mode, err, scale)


# ------------------------------------------------------------------ 2. f32 oracle within float64 bounds ----
@pytest.mark.parametrize("cloud", sorted(ORACLE_CLOUDS))
def test_oracle_within_float64_bounds(cloud):
    """At every random point (none excluded) the f32 oracle's gradient lies within f64_field's per-point bound; prints the largest
    error / bound ratio of each mode."""
    p = ORACLE_CLOUDS[cloud]()
    r, h, _ = _kw_abs(KW)
    lo, hi = p.min(0) - float(h), p.max(0) + float(h)
    pts = np.random.default_rng(93).uniform(lo, hi, (1500, 3)).astype(np.float32)
    for mode in ("sph", "avg", "rad"):                       # the f32 records of these modes are the float64 inputs
        radii = mode_kwargs(splashsurf_b200, mode, p, KW).get("particle_radii")
        ctr, w, g6, dlt, _ = records(p, KW, mode, radii)
        og = oracle_field(p, KW, mode, pts, radii)[1]
        _, g, bnd, nobound = f64_field(mode, ctr, w, g6, dlt, float(h), float(r), pts, bound=True)
        assert nobound == 0, (mode, nobound)
        err = np.linalg.norm(og.astype(np.float64) - g, axis=1)
        reach = bnd > 0
        assert np.all(og[~reach] == 0.0)
        ratio = err[reach] / bnd[reach]
        print(cloud, mode, "largest error / bound", float(ratio.max()), "points", int(reach.sum()))
        assert np.all(err <= bnd), (mode, float(ratio.max()))
    # the anisotropic records: the f32 oracle's own x_bar, G and V det G as exact inputs of the float64 restatement
    ctr, w, g6, dlt, _ = records(p, KW, "aniso")
    og = oracle_field(p, KW, "aniso", pts)[1]
    _, g, bnd, _ = f64_field("aniso", ctr, w, g6, dlt, float(h), float(r), pts, bound=True)
    err = np.linalg.norm(og.astype(np.float64) - g, axis=1)
    reach = bnd > 0
    print(cloud, "aniso", "largest error / bound", float((err[reach] / bnd[reach]).max()))
    assert np.all(err <= bnd)


# ------------------------------------------------------------------ 3. narrow band ----
NARROW_BAND_DEG = 0.1            # largest angle measured on the oracle 0.029 degrees (DESIGN.md section 13.1)


@pytest.mark.parametrize("mode", MODES)
def test_narrow_band_normal_angle(emu, mode):  # noqa: F811
    """At the mesh vertices and at vertices moved by up to half a cell, the f32 oracle's normal lies within NARROW_BAND_DEG of the
    float64 normal; prints the largest angle."""
    p = ORACLE_CLOUDS["sphere"]()
    r, h, c = _kw_abs(KW)
    mk = mode_kwargs(emu, mode, p, KW)
    g = emu.reconstruct_surface(p, subdomain_grid_auto_disable=False, **KW, **mk)
    v = g.mesh.vertices
    rng = np.random.default_rng(95)
    pts = np.concatenate([v, v + rng.uniform(-0.5, 0.5, v.shape) * float(c)]).astype(np.float32)
    radii = mk.get("particle_radii")
    ctr, w, g6, dlt, _ = records(p, KW, mode, radii)
    og = oracle_field(p, KW, mode, pts, radii)[1]
    _, fg, _, _ = f64_field(mode, ctr, w, g6, dlt, float(h), float(r), pts)
    cos = (og.astype(np.float64) * fg).sum(1) / (np.linalg.norm(og, axis=1) * np.linalg.norm(fg, axis=1))
    ang = np.degrees(np.arccos(np.clip(cos, -1.0, 1.0)))
    print(mode, "largest narrow-band angle (deg)", float(ang.max()), len(pts))
    assert np.all(ang <= NARROW_BAND_DEG), float(ang.max())


# ------------------------------------------------------------------ 5. properties ----
@pytest.mark.parametrize("mode", MODES)
def test_emulated_one_particle_normals_are_radial(emu, mode):  # noqa: F811
    """One particle: the outward normal at every vertex of its mesh points away from the particle (for the averaged modes within the
    1/u-free bound of a single candidate: offsets of about h / 2 carry a few u; the standard and anisotropic modes are radial by
    symmetry of each term)."""
    p = np.array([[0.1, 0.2, 0.3]], np.float32)
    mk = mode_kwargs(emu, mode, p, KW)
    g = emu.reconstruct_surface(p, subdomain_grid_auto_disable=False, **KW, **mk)
    f = emu.LevelSetField(p, **KW, **mk)
    try:
        v = g.mesh.vertices
        assert len(v) > 10
        n = f.normals(v)
        radial = (v - p[0]).astype(np.float64)
        radial /= np.linalg.norm(radial, axis=1, keepdims=True)
        # a single term: n = fl(d) / |fl(d)| up to the roundings of the fold; the averaged modes' M m - |m|^2 T cancels, and at the
        # surface (|d| = R_s = h / 4, b = 15 / 16) its rounding reaches the direction scaled by 6 |d|^2 / (h^2 b) < 1: tens of u
        assert np.abs(n - radial).max() <= 512 * U, np.abs(n - radial).max()
    finally:
        f.close()


def test_emulated_standard_normals_match_sph_interpolator(emu):  # noqa: F811
    """Standard mode: normals() equals SphInterpolator(...).interpolate_normals() up to summation order where the gradient is not
    negligible."""
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    r, h, _ = _kw_abs(kw)
    f = emu.LevelSetField(p, **kw)
    try:
        pts = random_points(f.grid, 3000, 97)
        _, g = f.gradient(pts)
        n = f.normals(pts)
        rest_mass = float(np.float32(np.float32(r + r) ** 3 * np.float32(kw.get("rest_density", 1000.0))))
        si = emu.SphInterpolator(p, f.particle_densities, rest_mass, float(h))
        ref = si.interpolate_normals(pts)
        si.close()
        gn = np.linalg.norm(g, axis=1)
        big = gn > 1e-3 * gn.max()
        assert big.sum() > 200
        assert np.abs(n[big] - ref[big]).max() <= 1e-4, np.abs(n[big] - ref[big]).max()
    finally:
        f.close()


def test_emulated_equal_radii_equal_plain_averaged(emu):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    rad = np.full(len(p), np.float32(_kw_abs(kw)[0]))
    a = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), **kw)
    b = emu.LevelSetField(p, averaged_surface=emu.AveragedSurface(), particle_radii=rad, **kw)
    try:
        pts = random_points(a.grid, 2000, 98, pad=0.1)
        va, ga = a.gradient(pts)
        vb, gb = b.gradient(pts)
        assert np.array_equal(va.view(np.uint32), vb.view(np.uint32)) and np.array_equal(ga.view(np.uint32), gb.view(np.uint32))
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ 6. refusals ----
def test_emulated_refusals(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    for corr_rad in (False, True):
        mk = dict(averaged_surface=ss.AveragedSurface(1.0, ss.JacobianCorrection()))
        if corr_rad:
            mk["particle_radii"] = mode_kwargs(ss, "rad", p, KW)["particle_radii"]
        f = ss.LevelSetField(p, **KW, **mk)
        try:
            pts = random_points(f.grid, 10, 3)
            with pytest.raises(ss.SplashsurfError, match="no gradient") as e:
                f.gradient(pts)
            assert e.value.code == 7                          # SS_ERR_UNSUPPORTED through the C entry
            with pytest.raises(ss.SplashsurfError, match="no gradient"):
                f.normals(pts)
            assert f.evaluate(pts).shape == (10,)              # the value query stays available
        finally:
            f.close()
    ctx = ss.Context()
    try:
        f = ss.LevelSetField(p, context=ctx, **KW)
        pts = random_points(f.grid, 50, 4)
        with pytest.raises(TypeError):
            f.gradient(pts.astype(np.float64))
        with pytest.raises(ValueError):
            f.gradient(pts[:, :2])
        nan = pts.copy()
        nan[7, 2] = np.nan
        with pytest.raises(ss.SplashsurfError, match="point 7"):
            f.gradient(nan)
        L = ctx._L
        out = np.empty(50, np.float32)
        assert L.ss_levelset_field_gradient_at_f32(f._s, pts.ctypes.data, 50, out.ctypes.data, None) == 6
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f.gradient(pts)
        f.close()
    finally:
        ctx.close()


def test_emulated_pipeline_and_cli_refusals(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli
    p = _cube(6, 5)
    with pytest.raises(ValueError, match="compute_normals"):
        emu.reconstruction_pipeline(p, levelset_normals=True, **KW)
    with pytest.raises(ValueError, match="exclusive"):
        emu.reconstruction_pipeline(p, compute_normals=True, sph_normals=True, levelset_normals=True, **KW)
    with pytest.raises(ValueError, match="Jacobian-corrected"):
        emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True,
                                    averaged_surface=emu.AveragedSurface(1.0, emu.JacobianCorrection()), **KW)
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "-o", str(tmp_path / "x.vtk")]
    for extra, msg in ((["--levelset-normals=on"], "--normals=on"),
                       (["--levelset-normals=on", "--normals=on", "--sph-normals=on"], "exclusive"),
                       (["--levelset-normals=on", "--normals=on", "--averaged-surface=on", "--averaged-correction=on"], "no gradient"),
                       (["--levelset-normals=on", "--normals=on", "--partition=on"], "--partition=on")):
        with pytest.raises(ValueError, match=msg):
            cli.main(args + extra)
        assert not os.path.exists(tmp_path / "x.vtk")


# ------------------------------------------------------------------ 7. pipeline and CLI ----
@pytest.mark.parametrize("mode", ["aniso", "avg"])
def test_emulated_pipeline_levelset_normals(emu, mode):  # noqa: F811
    """On a jittered ball: level-set normals are unit vectors whose dot product with the area-weighted normal is positive at every
    vertex, and normals_smoothing_iters is applied to them."""
    p = _ball(0.1, 111)
    mk = mode_kwargs(emu, mode, p, KW)
    mesh, rec = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, **KW, **mk)
    area, _ = emu.reconstruction_pipeline(p, compute_normals=True, **KW, **mk)
    n, a = mesh.point_attributes["normals"], area.point_attributes["normals"]
    assert len(n) > 100 and np.abs(np.linalg.norm(n, axis=1) - 1.0).max() < 1e-5
    assert np.all((n * a).sum(1) > 0)
    f = emu.LevelSetField(p, **KW, **mk)
    assert np.array_equal(n, f.normals(mesh.mesh.vertices))
    f.close()
    sm, _ = emu.reconstruction_pipeline(p, compute_normals=True, levelset_normals=True, normals_smoothing_iters=3, output_raw_normals=True,
                                        **KW, **mk)
    assert np.array_equal(sm.point_attributes["raw_normals"], n)
    assert not np.array_equal(sm.point_attributes["normals"], n)
    assert np.all((sm.point_attributes["normals"] * a).sum(1) > 0)


def test_emulated_cli_levelset_normals(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli, io
    src = os.path.join(os.path.dirname(__file__), "golden", "reference_data", "cube_2366_particles.vtk")
    out = tmp_path / "n.vtk"
    args = ["reconstruct", src, "-r", "0.025", "-l", "2.0", "-c", "0.75", "-q", "--averaged-surface=on"]
    assert cli.main(args + ["--normals=on", "--levelset-normals=on", "-o", str(out)]) == 0
    p = io.read_particles(src)
    mesh, _ = emu.reconstruction_pipeline(p, particle_radius=0.025, smoothing_length=2.0, cube_size=0.75, subdomain_grid_auto_disable=False,
                                          compute_normals=True, levelset_normals=True, averaged_surface=emu.AveragedSurface())
    _, _, _, point, _ = io.read_vtk_mesh(str(out))
    assert np.array_equal(np.asarray(point["normals"], np.float32), mesh.point_attributes["normals"])
