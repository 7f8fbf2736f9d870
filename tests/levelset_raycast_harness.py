"""What the ray-cast tests share (DESIGN.md section 15): the ray sets, the sample-by-sample oracle (tests/levelset_raycast_oracle.c)
and the device-versus-oracle check.  Not a test module: the cases live in tests/test_levelset_raycast.py (CPU executor) and
tests/test_zzz_gpu_levelset_raycast.py (H100)."""
import ctypes as C

import numpy as np

import c_oracle
from levelset_field_harness import GRAD_MODES, MODE_ID, T_HIGH, T_LOW, _kw_abs, _ptr, _same, face_points, mode_kwargs, records


def _lib():
    vp = C.c_void_p
    return c_oracle.build("levelset_raycast_oracle.c", {
        "so_raycast": (C.c_int64, [C.c_int, vp, vp, vp, vp, C.c_uint64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp,
                                   vp, vp, vp, C.c_uint64, C.c_float, C.c_uint32, vp, vp, vp, vp, vp])})


def oracle_raycast(p, kw, mode, grid, thr, o, d, t_max, step, refine, radii=None, grad=True):
    """(t, positions, values, status, gradients or None, samples evaluated) of section 15 by the oracle."""
    r, h, _ = _kw_abs(kw)
    ctr, w, g6, dlt, _ = records(p, kw, mode, radii)
    o, d = np.ascontiguousarray(o, np.float32), np.ascontiguousarray(d, np.float32)
    m = len(o)
    tm = None if t_max is None else np.ascontiguousarray(np.broadcast_to(np.asarray(t_max, np.float32), (m,)))
    t, pos, val, st = np.empty(m, np.float32), np.empty((m, 3), np.float32), np.empty(m, np.float32), np.empty(m, np.int8)
    g = np.empty((m, 3), np.float32) if grad else None
    gmin, gmax = np.asarray(grid.aabb.min, np.float32), np.asarray(grid.aabb.max, np.float32)
    arr = [np.ascontiguousarray(a) if a is not None else None for a in (ctr, w, g6, dlt)]
    ev = 0
    if m:
        ev = _lib().so_raycast(MODE_ID[mode], *[_ptr(a) for a in arr], len(ctr), h, r, T_LOW, T_HIGH, np.float32(thr), gmin.ctypes.data,
                               gmax.ctypes.data, o.ctypes.data, d.ctypes.data, _ptr(tm), m, np.float32(step), int(refine), t.ctypes.data,
                               pos.ctypes.data, val.ctypes.data, st.ctypes.data, _ptr(g))
    return t, pos, val, st, g, ev


# ------------------------------------------------------------------ ray sets ----
def _unit(rng, m):
    v = rng.normal(size=(m, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _box(grid):
    lo, hi = np.asarray(grid.aabb.min, np.float64), np.asarray(grid.aabb.max, np.float64)
    return lo, hi, 0.5 * (lo + hi), hi - lo


def camera_rays(grid, n, seed):
    """A pinhole camera outside the grid box looking at its centre, n x n pixels over the box."""
    lo, hi, ctr, ext = _box(grid)
    rng = np.random.default_rng(seed)
    eye = ctr + 1.5 * np.linalg.norm(ext) * _unit(rng, 1)[0]
    fwd = (ctr - eye) / np.linalg.norm(ctr - eye)
    up = np.cross(fwd, _unit(rng, 1)[0])
    up /= np.linalg.norm(up)
    right = np.cross(fwd, up)
    s = np.linspace(-0.45, 0.45, n)
    u, v = np.meshgrid(s, s, indexing="ij")
    d = fwd + u.reshape(-1, 1) * right + v.reshape(-1, 1) * up
    return np.repeat(eye[None], n * n, 0).astype(np.float32), d.astype(np.float32), None


def random_rays(grid, m, seed, targets=None):
    """Origins uniform in the grid box padded by 30 %, random directions (with `targets`, half of them aimed at a random target
    point), t_max = inf."""
    lo, hi, _, ext = _box(grid)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo - 0.3 * ext, hi + 0.3 * ext, (m, 3))
    u = _unit(rng, m)
    if targets is not None and len(targets):
        k = m // 2
        aim = targets[rng.integers(0, len(targets), k)].astype(np.float64) - o[:k]
        u[:k] = aim / np.linalg.norm(aim, axis=1, keepdims=True)
    return o.astype(np.float32), (u * rng.uniform(0.2, 3.0, (m, 1))).astype(np.float32), None


def segment_rays(grid, m, seed):
    """Segments x0 -> x0 + delta, |delta| up to 2 cells, as o = x0, d = delta, t_max = 1."""
    lo, hi, _, _ = _box(grid)
    rng = np.random.default_rng(seed)
    o = rng.uniform(lo, hi, (m, 3)).astype(np.float32)
    d = (_unit(rng, m) * rng.uniform(0.01, 2.0, (m, 1)) * grid.cell_size).astype(np.float32)
    return o, d, np.ones(m, np.float32)


def face_rays(grid, S, seed, m=40):
    """Axis-aligned rays in both directions along every axis from points on tile, brick and bin faces (face_points): the rays
    through a face point along the other two axes lie in its face."""
    pts = face_points(grid, S, seed)
    pts = pts[np.random.default_rng(seed).choice(len(pts), min(m, len(pts)), replace=False)]
    dirs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    return np.repeat(pts, 6, 0), np.tile(dirs, (len(pts), 1)), None


def far_rays(grid, h, m, seed):
    """Origins 1000 h outside the grid moving towards its centre, and origins outside moving away from it."""
    lo, hi, ctr, ext = _box(grid)
    rng = np.random.default_rng(seed)
    u = _unit(rng, m)
    o_far = ctr + u * (0.5 * np.linalg.norm(ext) + 1000.0 * float(h))
    o_out = ctr + u * (0.6 * np.linalg.norm(ext) + float(h))
    o = np.concatenate([o_far, o_out]).astype(np.float32)
    d = np.concatenate([-u + 0.05 * _unit(rng, m), u]).astype(np.float32)
    return o, d, None


def zero_rays(grid, m, seed):
    o, d, _ = random_rays(grid, m, seed)
    return o, d, np.zeros(m, np.float32)


def ray_sets(grid, h, S, seed, scale=1, targets=None):
    """Every ray set of section 15's tests, concatenated: (origins, directions, t_max per ray); `targets` (the particles) for the
    aimed half of the random rays and the segments' start points."""
    seg = segment_rays(grid, 40 * scale, seed + 2)
    if targets is not None and len(targets):
        seg[0][: len(seg[0]) // 2] = targets[np.random.default_rng(seed + 6).integers(0, len(targets), len(seg[0]) // 2)]
    sets = [camera_rays(grid, 6 * scale, seed), random_rays(grid, 40 * scale, seed + 1, targets), seg,
            face_rays(grid, S, seed + 3, 12 * scale), far_rays(grid, h, 8 * scale, seed + 4), zero_rays(grid, 8 * scale, seed + 5)]
    o = np.concatenate([s[0] for s in sets])
    d = np.concatenate([s[1] for s in sets])
    tm = np.concatenate([np.full(len(s[0]), np.inf, np.float32) if s[2] is None else s[2] for s in sets])
    return o, d, tm


# ------------------------------------------------------------------ device vs oracle ----
def check_raycast_vs_oracle(ss, p, kw, mode, rays_of, steps_refines, f=None, expect_tier=None):
    """For each (step in cells, refine): the device's t, positions, values, status and (modes with a gradient) gradients equal the
    oracle's bit for bit, NaN equal to NaN.  rays_of(field) gives (origins, directions, t_max).  Returns per call
    (rounds, paths, status counts, samples the oracle evaluated)."""
    mk = mode_kwargs(ss, mode, p, kw)
    own = f is None
    if own:
        f = ss.LevelSetField(p, **kw, **mk)
    out = []
    try:
        o, d, tm = rays_of(f, p)
        grad = mode in GRAD_MODES
        for step_c, refine in steps_refines:
            step = float(np.float32(step_c) * np.float32(f.grid.cell_size))
            got = f.raycast(o, d, t_max=tm, step=step, refine=refine, normals=grad)
            paths = f.paths
            ot, opos, oval, ost, og, ev = oracle_raycast(p, kw, mode, f.grid, f.threshold, o, d, tm, step, refine,
                                                         radii=mk.get("particle_radii"), grad=grad)
            what = (mode, step_c, refine)
            bad = np.flatnonzero(got.status != ost)
            assert len(bad) == 0, (what, len(bad), bad[:4], got.status[bad[:4]], ost[bad[:4]], got.t[bad[:4]], ot[bad[:4]])
            assert _same(got.t, ot), (what, np.flatnonzero(got.t.view(np.uint32) != ot.view(np.uint32))[:4])
            assert _same(got.positions, opos) and _same(got.values, oval), what
            if grad:
                assert _same(got.gradients, og), what
            if expect_tier:
                assert paths[expect_tier] > 0, (what, paths)
            out.append(dict(rounds=got.rounds, paths=paths, status={int(s): int((got.status == s).sum()) for s in (-1, 0, 1, 2)}, samples=ev))
        return out
    finally:
        if own:
            f.close()


def bricks_crossed(f, o, d, hits_t, step):
    """The bricks each ray's samples cross up to t (refine = 0: t is the crossing sample), counted by their distinct brick indices
    (empty bricks included, at most 4096 samples per ray); 0 without a crossing."""
    c = np.float64(f.grid.cell_size)
    lo = np.asarray(f.grid.aabb.min, np.float64)
    n = np.zeros(len(o), np.int64)
    for i in range(len(o)):
        dt = step / np.linalg.norm(d[i].astype(np.float64))
        tend = hits_t[i] if np.isfinite(hits_t[i]) else 0.0
        k = np.arange(0, min(int(np.rint(tend / dt)) + 1, 4096))     # t is a sample: T_j = j dt
        x = o[i].astype(np.float64) + (k * dt)[:, None] * d[i].astype(np.float64)
        b = np.floor((x - lo) / c / 8).astype(np.int64)
        n[i] = len(np.unique(b, axis=0)) if len(b) else 0
    return n
