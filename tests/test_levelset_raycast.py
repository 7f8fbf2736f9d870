"""First crossings of the level-set field along rays and segments (LevelSetField.raycast / ss_levelset_field_raycast_f32, DESIGN.md
section 15), on the CPU executor of the CUDA sources (also run with SS_EMUL_GUARD=1):

* the device equals the sample-by-sample oracle (tests/levelset_raycast_oracle.c) bit for bit -- t, positions, values, status and
  gradients -- in all six modes on splash_S24 and droplets_sparse, for camera rays from outside the grid, random rays inside and
  outside the liquid, short segments, axis-aligned rays on brick / tile / bin faces, far and receding rays and t_max = 0, at
  refine 0 / 1 / 24 / 64 and steps of 0.13 / 0.5 / 3 cells; the standard and averaged modes also at R = 1 and 9;
* values, gradients, normals and inside flags equal evaluate(), gradient(), normals() and inside() at the positions;
* on a jittered ball the hits lie within sqrt(3) cells plus the bracket of the raw mesh's triangles along the same rays;
* the clustered cloud reaches the selection tier during a ray cast;
* refusals, float64, a stale handle, m = 0, n = 0, host numpy against ctypes arrays, the 2^24 sample cap, and one context reused
  across a field, ray casts, evaluate and a reconstruction.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_raycast.py."""
import ctypes as C

import numpy as np
import pytest

from levelset_field_harness import GRAD_MODES, MODES, _ball, _kw_abs, _same, mode_kwargs
from levelset_raycast_harness import (bricks_crossed, check_raycast_vs_oracle, oracle_raycast, random_rays, ray_sets, segment_rays)
from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_surface import CASES
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

STEPS_REFINES = [(0.5, 24), (0.13, 1), (3.0, 64), (0.5, 0)]


def _rays(S, seed, scale=1):
    def of(f, p):
        _, h, _ = _kw_abs(KW)
        return ray_sets(f.grid, h, S, seed, scale, targets=p)
    return of


# ------------------------------------------------------------------ device == oracle ----
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["splash_S24", "droplets_sparse"])
def test_emulated_raycast_equals_oracle(emu, name, mode):  # noqa: F811
    gen, kw, _ = CASES[name]
    p = gen()
    res = check_raycast_vs_oracle(emu, p, kw, mode, _rays(kw["subdomain_num_cubes_per_dim"], 300), STEPS_REFINES)
    print(name, mode, res)
    assert all(r["paths"]["512"] > 0 for r in res), res
    assert sum(r["status"][1] + r["status"][-1] for r in res) > 20, res


@pytest.mark.parametrize("mode", ["sph", "avg"])
@pytest.mark.parametrize("Rc", [1, 9])
def test_emulated_raycast_cube_sizes(emu, Rc, mode):  # noqa: F811
    """R = ceil(h / c) = 1 and 9: a brick's candidate bins must reach one cell past its grid points for every point a lane evaluates."""
    p = _cube(7, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    check_raycast_vs_oracle(emu, p, kw, mode, _rays(16, 310 + Rc), [(0.5, 24), (3.0, 8)])


def test_emulated_raycast_wide_steps_reenter_groups(emu):  # noqa: F811
    """At 3 cells a bracket can span two bricks, and its bisection re-enters the brick the march already left: a ray cast alone
    then takes more rounds than the bricks its samples crossed."""
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = emu.LevelSetField(p, **kw)
    try:
        o, d, _ = random_rays(f.grid, 60, 320, targets=p)
        step = float(np.float32(3.0) * np.float32(f.grid.cell_size))
        h0 = f.raycast(o, d, step=step, refine=0, normals=False)
        hit = np.flatnonzero(np.abs(h0.status) == 1)
        assert len(hit) > 10
        nb = bricks_crossed(f, o, d, h0.t, step)
        c, lo = np.float32(f.grid.cell_size), np.asarray(f.grid.aabb.min, np.float32)
        more = []
        for i in hit:
            dt = np.float32(step) / np.linalg.norm(d[i]).astype(np.float32)
            a = o[i] + np.float32(h0.t[i] - dt) * d[i]
            if np.array_equal(np.floor((a - lo) / c / 8), np.floor((h0.positions[i] - lo) / c / 8)):
                continue                                     # the bracket lies in one brick
            one = f.raycast(o[i:i + 1], d[i:i + 1], step=step, refine=64, normals=False)
            more.append((one.rounds, int(nb[i])))
        print("(rounds, bricks crossed) of rays whose bracket spans two bricks:", more)
        assert any(r > b for r, b in more), more
    finally:
        f.close()


# ------------------------------------------------------------------ consistency with the point queries ----
@pytest.mark.parametrize("mode", MODES)
def test_emulated_raycast_consistent_with_queries(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f = emu.LevelSetField(p, **kw, **mode_kwargs(emu, mode, p, kw))
    try:
        o, d, tm = ray_sets(f.grid, _kw_abs(kw)[1], 24, 330, targets=p)
        grad = mode in GRAD_MODES
        hits = f.raycast(o, d, t_max=tm, normals=grad)
        hit = np.abs(hits.status) == 1
        assert hit.sum() > 20
        assert np.all(np.isinf(hits.t[~hit])) and np.all(np.isnan(hits.values[~hit])) and np.all(np.isnan(hits.positions[~hit]))
        x = hits.positions[hit]
        assert _same(hits.values[hit], f.evaluate(x))
        assert np.array_equal(f.inside(x), ~f.inside(o[hit]))
        assert np.array_equal(hits.status[hit] == -1, f.inside(o[hit]))
        assert np.all(hits.t[hit] >= 0) and np.all(hits.t[hit] <= tm[hit])
        if grad:
            assert _same(hits.gradients[hit], f.gradient(x)[1])
            assert _same(hits.normals[hit], f.normals(x))
            assert np.all(np.isnan(hits.normals[~hit]))
        else:
            assert hits.normals is None
            with pytest.raises(emu.SplashsurfError, match="no gradient"):
                f.raycast(o, d, t_max=tm)
    finally:
        f.close()


# ------------------------------------------------------------------ geometry against the mesh ----
def _mesh_t(verts, tris, o, d):
    """Smallest t >= 0 of each ray o + t d against the triangles (float64 Moller-Trumbore); inf where none."""
    v = verts.astype(np.float64)
    a, b, c = v[tris[:, 0]], v[tris[:, 1]], v[tris[:, 2]]
    e1, e2 = b - a, c - a
    out = np.full(len(o), np.inf)
    for i in range(len(o)):
        dd = d[i].astype(np.float64)
        pv = np.cross(dd, e2)
        det = np.einsum("ij,ij->i", e1, pv)
        ok = np.abs(det) > 1e-18
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        tv = o[i].astype(np.float64) - a
        u = np.einsum("ij,ij->i", tv, pv) * inv
        qv = np.cross(tv, e1)
        w = (qv @ dd) * inv
        t = np.einsum("ij,ij->i", e2, qv) * inv
        sel = ok & (u >= 0) & (w >= 0) & (u + w <= 1) & (t >= 0)
        if sel.any():
            out[i] = t[sel].min()
    return out


@pytest.mark.parametrize("mode", ["sph", "avg", "rad"])
def test_emulated_raycast_matches_mesh_on_ball(emu, mode):  # noqa: F811
    p = _ball(0.1, 11)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    mk = mode_kwargs(emu, mode, p, kw)
    rec = emu.reconstruct_surface(p, simd=False, subdomain_grid_auto_disable=False, **kw, **mk)
    f = emu.LevelSetField(p, **kw, **mk)
    try:
        rng = np.random.default_rng(340)
        u = rng.normal(size=(150, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        ctr = p.mean(0).astype(np.float64)
        rad = float(np.linalg.norm(p - ctr, axis=1).max()) + 4 * float(_kw_abs(kw)[1])
        o = np.concatenate([np.repeat(ctr[None], 150, 0), ctr + rad * u]).astype(np.float32)
        d = np.concatenate([u, -u]).astype(np.float32)
        c = float(f.grid.cell_size)
        step, refine = 0.5 * c, 24
        hits = f.raycast(o, d, step=step, refine=refine, normals=False)
        tm = _mesh_t(rec.mesh.vertices, rec.mesh.triangles.astype(np.int64), o, d)
        both = (np.abs(hits.status) == 1) & np.isfinite(tm)
        assert both.sum() > 250
        nd = np.linalg.norm(d.astype(np.float64), axis=1)
        diff = np.abs(hits.t.astype(np.float64) * nd - tm * nd)[both]
        tol = np.sqrt(3.0) * c + step * 2.0 ** -refine
        print(mode, "largest |t_field - t_mesh| =", float(diff.max()), "cells:", float(diff.max()) / c)
        assert np.all(diff <= tol), (float(diff.max()), tol)
    finally:
        f.close()


# ------------------------------------------------------------------ tiers ----
def test_emulated_raycast_clustered_reaches_select(emu):  # noqa: F811
    p = _clustered(507)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)

    def rays(f, _p):
        rng = np.random.default_rng(350)
        o = rng.uniform(0.1, 0.3, (60, 3)).astype(np.float32)
        d = rng.normal(size=(60, 3)).astype(np.float32)
        return o, d, np.full(60, np.float32(0.2))
    res = check_raycast_vs_oracle(emu, p, kw, "sph", rays, [(0.5, 24)], expect_tier="select")
    print(res)


# ------------------------------------------------------------------ refusals and edges ----
def test_emulated_raycast_refusals(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    f = ss.LevelSetField(p, **KW)
    L = ss._LIB
    try:
        o, d, tm = segment_rays(f.grid, 10, 360)
        for bad, field, match in [(np.nan, "o", "ray 3 has a non-finite"), (np.inf, "d", "ray 3 has a non-finite"),
                                  (0.0, "d", "ray 3 has a zero direction"), (np.nan, "t", "ray 3 has a NaN or negative"),
                                  (-1.0, "t", "ray 3 has a NaN or negative")]:
            oo, dd, tt = o.copy(), d.copy(), tm.copy()
            if field == "o":
                oo[3, 1] = bad
                oo[7, 0] = bad
            elif field == "d":
                dd[3] = bad
                dd[7] = bad
            else:
                tt[3] = bad
                tt[7] = bad
            with pytest.raises(ss.SplashsurfError, match=match) as e:
                f.raycast(oo, dd, t_max=tt)
            assert e.value.code == ss.SS_ERR_INVALID_PARAMETER
        dd = d.copy()
        dd[5] = [1e-30, 0, 0]                           # dt = step / |d| overflows
        with pytest.raises(ss.SplashsurfError, match="ray 5 has a zero direction"):
            f.raycast(o, dd, t_max=tm)
        for kw_, match in [(dict(step=0.0), "step"), (dict(step=np.inf), "step"), (dict(step=-1.0), "step"), (dict(refine=65), "refine")]:
            with pytest.raises(ss.SplashsurfError, match=match):
                f.raycast(o, d, t_max=tm, **kw_)
        with pytest.raises(TypeError):
            f.raycast(o.astype(np.float64), d, t_max=tm)
        with pytest.raises(TypeError):
            f.raycast(o, d.astype(np.float64), t_max=tm)
        with pytest.raises(ValueError):
            f.raycast(o, d[:5], t_max=tm)
        # through the C entry: NULL arrays, m too large
        out = [np.empty(10, np.float32), np.empty((10, 3), np.float32), np.empty(10, np.float32), np.empty(10, np.int8)]
        ptrs = [a.ctypes.data for a in out]
        rc = L.ss_levelset_field_raycast_f32(f._s, None, d.ctypes.data, None, 10, C.c_float(0.01), 24, *ptrs, None, None)
        assert rc == ss.SS_ERR_INVALID_PARAMETER
        rc = L.ss_levelset_field_raycast_f32(f._s, o.ctypes.data, d.ctypes.data, None, 10, C.c_float(0.01), 24, ptrs[0], None, ptrs[2], ptrs[3],
                                             None, None)
        assert rc == ss.SS_ERR_INVALID_PARAMETER
        rc = L.ss_levelset_field_raycast_f32(f._s, o.ctypes.data, d.ctypes.data, None, 2 ** 31 - 1, C.c_float(0.01), 24, *ptrs, None, None)
        assert rc == ss.SS_ERR_INDEX_TOO_SMALL
        rc = L.ss_levelset_field_raycast_f32(f._s, o.ctypes.data, d.ctypes.data, None, 10, C.c_float(np.nan), 24, *ptrs, None, None)
        assert rc == ss.SS_ERR_INVALID_PARAMETER
        rc = L.ss_levelset_field_raycast_f32(f._s, o.ctypes.data, d.ctypes.data, None, 10, C.c_float(0.01), 65, *ptrs, None, None)
        assert rc == ss.SS_ERR_INVALID_PARAMETER
        # host numpy arrays and ctypes arrays give identical results
        rounds = C.c_uint64()
        rc = L.ss_levelset_field_raycast_f32(f._s, o.ctypes.data, d.ctypes.data, tm.ctypes.data, 10, C.c_float(0.01), 24, *ptrs, None, C.byref(rounds))
        assert rc == 0
        co, cd, ct = (C.c_float * 30)(*o.ravel()), (C.c_float * 30)(*d.ravel()), (C.c_float * 10)(*tm)
        cout = [(C.c_float * 10)(), (C.c_float * 30)(), (C.c_float * 10)(), (C.c_int8 * 10)()]
        rc = L.ss_levelset_field_raycast_f32(f._s, C.addressof(co), C.addressof(cd), C.addressof(ct), 10, C.c_float(0.01), 24,
                                             *[C.addressof(a) for a in cout], None, None)
        assert rc == 0
        for a, b in zip(out[:3], cout[:3]):
            assert _same(a.ravel(), np.ctypeslib.as_array(b).ravel())
        assert np.array_equal(out[3], np.ctypeslib.as_array(cout[3]))
        h = f.raycast(o, d, t_max=tm, step=0.01)
        assert _same(h.t, out[0]) and _same(h.positions, out[1]) and np.array_equal(h.status, out[3])
        # m = 0
        e = f.raycast(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32))
        assert e.t.shape == (0,) and e.positions.shape == (0, 3) and e.status.dtype == np.int8 and e.normals.shape == (0, 3) and e.rounds == 0
        # scalar t_max
        h1 = f.raycast(o, d, t_max=1.0)
        h2 = f.raycast(o, d, t_max=np.ones(10, np.float32))
        assert _same(h1.t, h2.t) and np.array_equal(h1.status, h2.status)
    finally:
        f.close()
    # a corrected field refuses normals, not the ray cast
    f = ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(1.0, ss.JacobianCorrection()), **KW)
    try:
        with pytest.raises(ss.SplashsurfError, match="no gradient") as e:
            f.raycast(o, d, t_max=tm)
        assert e.value.code == ss.SS_ERR_UNSUPPORTED
        assert f.raycast(o, d, t_max=tm, normals=False).normals is None
    finally:
        f.close()


def test_emulated_raycast_empty_field_sample_cap_and_reuse(emu):  # noqa: F811
    ss = emu
    # n = 0: every ray misses
    f = ss.LevelSetField(np.zeros((0, 3), np.float32), **KW)
    try:
        o, d, tm = random_rays(f.grid, 30, 370)
        h = f.raycast(o, d)
        assert np.all(h.status == 0) and np.all(np.isinf(h.t))
        # the sample cap: 2^24 samples inside the grid without a crossing give status 2 (and the oracle agrees)
        lo = np.asarray(f.grid.aabb.min, np.float32)
        o2 = np.repeat((lo + np.float32(0.5) * np.float32(f.grid.cell_size))[None], 3, 0).astype(np.float32)
        d2 = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
        step = float(np.float32(f.grid.cell_size) * np.float32(1e-8))
        h2 = f.raycast(o2, d2, step=step, normals=False)
        ot, _, _, ost, _, ev = oracle_raycast(np.zeros((0, 3), np.float32), KW, "sph", f.grid, f.threshold, o2, d2, None, step, 24, grad=False)
        assert np.all(h2.status == 2) and np.array_equal(ost, h2.status) and ev == 3 * 2 ** 24
    finally:
        f.close()
    # one context across a field, ray casts, evaluate and a reconstruction
    p = _cube(6, 5)
    ctx = ss.Context()
    try:
        f1 = ss.LevelSetField(p, context=ctx, **KW)
        o, d, tm = random_rays(f1.grid, 50, 380)
        a = f1.raycast(o, d)
        v = f1.evaluate(o)
        b = f1.raycast(o, d)
        assert _same(a.t, b.t) and _same(a.normals, b.normals) and np.array_equal(v, f1.evaluate(o))
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f1.raycast(o, d)
        f1.close()
        f2 = ss.LevelSetField(p, context=ctx, **KW)
        c = f2.raycast(o, d)
        assert _same(a.t, c.t) and _same(a.positions, c.positions) and np.array_equal(a.status, c.status)
        f2.close()
    finally:
        ctx.close()
