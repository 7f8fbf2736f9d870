"""Narrow-band signed distance grids (LevelSetField.signed_distance / ss_levelset_field_sdf_f32, DESIGN.md section 14) on the CPU
executor of the CUDA sources (also run with SS_EMUL_GUARD=1):

* the device equals the brute-force oracle (tests/levelset_sdf_oracle.c, bound by tests/levelset_field_harness.py) bit for bit -- brick list, values and brick_inside -- in
  every mode (standard with simd off and on, anisotropic, averaged, corrected, radii), on section 12's clouds, at band 1 / 3 / 8,
  S = 16 / 24 / 64 and at cube sizes giving R = 1, 6, 7, 8, 9, 17;
* hand-made meshes through the C entry: single triangles on brick faces and corners, zero-area triangles, a triangle outside the
  grid, an empty mesh, and a fan that overflows the shared slice and takes the global walk;
* the f32 distances lie within a per-point float64 bound of the exact distance to the same f32 triangles, and the bound is tight
  enough to notice a missing nearest triangle;
* on raw meshes: the sign is the field's, adjacent listed values differ by at most a cell, every vertex's edge is listed with
  opposite signs within a cell, and to_dense() has the field's sign at every grid point;
* refusals, one context reused across fields, queries and grids, and the CLI's --output-sdf.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_sdf.py."""
import ctypes as C

import numpy as np
import pytest

from levelset_field_harness import (SDF_MODES, assert_sdf_equal, check_properties, check_sdf_vs_oracle, mode_kwargs, oracle_distance,
                                    oracle_sdf, raw_case)
from test_anisotropic import KW, R, _cube
from test_averaged_surface import CASES
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)


# ------------------------------------------------------------------ device vs oracle ----
@pytest.mark.parametrize("mode", SDF_MODES)
@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64"])
def test_emulated_sdf_equals_oracle(emu, name, mode):  # noqa: F811
    gen, kw, _ = CASES[name]
    f, rec, got = check_sdf_vs_oracle(emu, gen(), dict(kw), mode, 3)
    assert len(got.brick_coords) > 0 and got.paths["shared"] > 0
    f.close()


@pytest.mark.parametrize("band", [1, 8])
@pytest.mark.parametrize("mode", ["sph", "avg"])
def test_emulated_sdf_bands_equal_oracle(emu, mode, band):  # noqa: F811
    gen, kw, _ = CASES["cube_S16"]
    check_sdf_vs_oracle(emu, gen(), dict(kw), mode, band)[0].close()


@pytest.mark.parametrize("name", ["droplets_sparse", "particle_aabb", "tile_batch_1"])
def test_emulated_sdf_clouds_equal_oracle(emu, name):  # noqa: F811
    gen, kw, _ = CASES[name]
    check_sdf_vs_oracle(emu, gen(), dict(kw), "sph", 3)[0].close()


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
def test_emulated_sdf_cube_sizes_equal_oracle(emu, Rc):  # noqa: F811
    """R = ceil(h / c) = Rc: lattices on which the mesh's triangles sit on and across brick faces."""
    p = _cube(6, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f, rec, got = check_sdf_vs_oracle(emu, p, kw, "sph", 3)
    assert int(np.ceil(np.float32(4 * R) / np.float32(f.grid.cell_size))) == Rc
    f.close()


# ------------------------------------------------------------------ hand-made meshes ----
def test_emulated_hand_made_meshes(emu):  # noqa: F811
    ss = emu
    p = _cube(5, 11)
    f = ss.LevelSetField(p, **KW)
    try:
        g = f.grid
        lo, c = np.asarray(g.aabb.min, np.float32), np.float32(g.cell_size)
        q = lambda *i: (lo + np.asarray(i, np.float32) * c).astype(np.float32)  # noqa: E731
        n = np.asarray(g.npoints_per_dim)
        cases = {
            "brick_face": (np.stack([q(8, 1, 1), q(8, 6, 2), q(8, 3, 7)]), [[0, 1, 2]]),
            "brick_corner": (np.stack([q(8, 8, 8), q(9.5, 8, 8), q(8, 8.5, 9)]), [[0, 1, 2]]),
            "collinear": (np.stack([q(3, 3, 3), q(5, 5, 5), q(9, 9, 9)]), [[0, 1, 2]]),
            "one_point": (np.stack([q(4.25, 7.5, 8)] * 3), [[0, 1, 2]]),
            "two_equal": (np.stack([q(4, 4, 4), q(4, 4, 4), q(6, 5, 4)]), [[0, 1, 2]]),
            "outside": (np.stack([q(-40, -40, -40), q(-39, -40, -40), q(-40, -39, -40)]), [[0, 1, 2]]),
            "upper_corner": (np.stack([q(*(n - 1)), q(*(n - 1.5)), q(n[0] - 1, n[1] - 2, n[2] - 1)]), [[0, 1, 2]]),
            "empty": (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint64)),
        }
        for name, (v, t) in cases.items():
            t = np.asarray(t, np.uint64).reshape(-1, 3)
            got = f.signed_distance(ss.TriMesh3d(np.ascontiguousarray(v, np.float32), t), band=3)
            o = oracle_sdf(p, KW, "sph", v, t, 3, g, f.threshold)
            assert_sdf_equal(got, *o, what=name)
            if name in ("outside", "empty"):
                assert len(got.brick_coords) == 0 and got.brick_inside.shape == tuple((n + 7) // 8) and got.brick_inside.any()
            else:
                assert len(got.brick_coords) > 0, name
            if name == "one_point":
                assert np.min(np.abs(got.values)) < c
        # a fan of 400 triangles around one lattice point: one brick far over the shared slice takes the global walk
        ang = np.linspace(0, 2 * np.pi, 401)[:-1]
        ctr = q(12, 12, 12)
        rim = np.stack([ctr + 0.6 * c * np.array([np.cos(a), np.sin(a), 0.3 * np.sin(3 * a)]) for a in ang]).astype(np.float32)
        v = np.concatenate([ctr[None], rim]).astype(np.float32)
        t = np.array([[0, 1 + k, 1 + (k + 1) % 400] for k in range(400)], np.uint64)
        got = f.signed_distance(ss.TriMesh3d(v, t), band=2)
        assert got.paths["global"] > 0, got.paths
        assert_sdf_equal(got, *oracle_sdf(p, KW, "sph", v, t, 2, g, f.threshold), what="fan")
    finally:
        f.close()


@pytest.mark.parametrize("mode", ["sph", "avg"])
def test_emulated_passes_equal_one_pass(emu, mode):  # noqa: F811
    """A small pair bound splits the call into many slabs of brick columns: the grid is the oracle's bit for bit all the same."""
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec, mk = raw_case(emu, p, dict(kw), mode)
    L = f._ctx._L
    try:
        one = f.signed_distance(rec.mesh)
        L.ss_sdf_set_pass_pairs(500)
        many = f.signed_distance(rec.mesh)
    finally:
        L.ss_sdf_set_pass_pairs(0)
        f.close()
    assert one.passes["passes"] == 1 and many.passes["passes"] > 5 and many.passes["pairs"] == one.passes["pairs"], (one.passes, many.passes)
    assert many.paths == one.paths
    assert_sdf_equal(many, one.brick_coords, one.values, one.brick_inside, what="passes")
    assert_sdf_equal(one, *oracle_sdf(p, kw, mode, rec.mesh.vertices, rec.mesh.triangles, 3, f.grid, f.threshold,
                                      radii=mk.get("particle_radii")), what="oracle")


# ------------------------------------------------------------------ float64 bound ----
U = 2.0 ** -24 * (1 + 2.0 ** -20)          # f32 unit roundoff, with room for the float64 arithmetic of the bound itself


class _E:
    """A float64 value with a bound on the distance between the f32 computation and the exact value, carried operation by
    operation (section 3a's running error: every f32 operation adds u |result|)."""

    def __init__(self, v, e):
        self.v, self.e = v, e

    def __add__(self, o):
        v = self.v + o.v
        return _E(v, self.e + o.e + U * (np.abs(v) + self.e + o.e))

    def __sub__(self, o):
        v = self.v - o.v
        return _E(v, self.e + o.e + U * (np.abs(v) + self.e + o.e))

    def __mul__(self, o):
        v = self.v * o.v
        e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
        return _E(v, e + U * (np.abs(v) + e))


def _edot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _ecross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _ediv(a, b):
    """a / b; unbounded (inf) where |b| <= its error."""
    den = np.abs(b.v) - b.e
    v = np.divide(a.v, b.v, out=np.zeros_like(a.v), where=b.v != 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf)
    return _E(v, e + U * (np.abs(v) + e))


def exact_interval_d2(p, t):
    """[lo, hi] of the squared distance the f32 formula of section 14 can give for points p (P, 3) and triangles t (T, 9), both
    exact f32 values: per pair, the exact distance of each branch the f32 computation may take, widened by its running error."""
    P = [_E(p[:, None, d].astype(np.float64), np.zeros((len(p), 1))) for d in range(3)]
    V = [[_E(t[None, :, 3 * k + d].astype(np.float64), np.zeros((1, len(t)))) for d in range(3)] for k in range(3)]

    def edge(v0, v1):
        e = [v1[d] - v0[d] for d in range(3)]
        w = [P[d] - v0[d] for d in range(3)]
        ee = _edot(e, e)
        x = _ediv(_edot(w, e), ee)
        tv = np.clip(x.v, 0.0, 1.0)
        te = np.minimum(x.e, 1.0)
        tv = np.where(ee.v == 0, 0.0, tv)
        te = np.where(ee.v == 0, 0.0, te)
        T = _E(tv, te)
        r = [P[d] - (v0[d] + T * e[d]) for d in range(3)]
        return _edot(r, r)

    a, b, c = V
    edges = [edge(a, b), edge(b, c), edge(c, a)]
    elo = np.minimum.reduce([x.v - x.e for x in edges])
    ehi = np.minimum.reduce([x.v + x.e for x in edges])
    ab, ac = [b[d] - a[d] for d in range(3)], [c[d] - a[d] for d in range(3)]
    n = _ecross(ab, ac)
    nn = _edot(n, n)
    sides = []
    for v0, v1 in ((a, b), (b, c), (c, a)):
        sides.append(_edot(_ecross([v1[d] - v0[d] for d in range(3)], [P[d] - v0[d] for d in range(3)]), n))
    surely_in = (nn.v - nn.e > 0) & np.all([s.v - s.e >= 0 for s in sides], axis=0)
    maybe_in = (nn.v + nn.e > 0) & np.all([s.v + s.e >= 0 for s in sides], axis=0)
    dn = _edot([P[d] - a[d] for d in range(3)], n)
    f = _ediv(dn * dn, nn)
    flo, fhi = f.v - f.e, f.v + f.e
    lo = np.where(maybe_in, np.minimum(elo, flo), elo)
    hi = np.where(surely_in, np.minimum(ehi, fhi), ehi)
    return np.maximum(lo, 0.0), hi


def test_emulated_distance_within_float64_bound(emu):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec, mk = raw_case(emu, p, dict(kw), "sph")
    try:
        got = f.signed_distance(rec.mesh, band=3)
        B = np.float32(got.background)
        lo_g, c = np.asarray(f.grid.aabb.min, np.float32), np.float32(f.grid.cell_size)
        v, tri = rec.mesh.vertices, rec.mesh.triangles.astype(np.int64)
        T = v[tri].reshape(-1, 9)
        tmin, tmax = T.reshape(-1, 3, 3).min(1).astype(np.float64), T.reshape(-1, 3, 3).max(1).astype(np.float64)
        rng = np.random.default_rng(5)
        checked = sensitive = 0
        for bi in rng.choice(len(got.brick_coords), min(40, len(got.brick_coords)), replace=False):
            b = got.brick_coords[bi].astype(np.int64)
            idx = 8 * b + np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)
            pts = (lo_g + idx.astype(np.float32) * c).astype(np.float32)
            d = np.abs(got.values[bi].reshape(-1))
            keep = (d < B) & np.all(idx < np.asarray(f.grid.npoints_per_dim), axis=1)
            reach = float(B) + float(c)
            near = np.all((tmax + reach >= pts[keep].min(0)) & (tmin - reach <= pts[keep].max(0)), axis=1)
            if not keep.any():
                continue
            lo2, hi2 = exact_interval_d2(pts[keep], T[near])
            lo, hi = np.sqrt(lo2.min(1)) * (1 - U), np.sqrt(hi2.min(1)) * (1 + U)
            assert np.all((d[keep] >= lo) & (d[keep] <= hi)), bi
            checked += int(keep.sum())
            # sensitivity: without its nearest triangle a point's distance leaves the bound wherever the next-nearest is farther
            order = np.argsort(lo2, axis=1)
            nxt_lo = np.sqrt(np.take_along_axis(lo2, order[:, 1:2], 1)[:, 0]) * (1 - U) if lo2.shape[1] > 1 else np.full(len(lo), np.inf)
            far = nxt_lo > hi
            if far.any():
                nearest = np.flatnonzero(near)[order[far, 0]]
                pk = pts[keep][far]
                for j in range(min(len(pk), 5)):
                    rest = np.delete(np.flatnonzero(near), order[far][j, 0])
                    dd = oracle_distance(v, rec.mesh.triangles[rest], pk[j:j + 1])[0]
                    assert not (lo[far][j] <= dd <= hi[far][j]), (bi, j, nearest[j])
                sensitive += int(far.sum())
        assert checked > 1000 and sensitive > 0.2 * checked, (checked, sensitive)
    finally:
        f.close()


# ------------------------------------------------------------------ properties on raw meshes ----
@pytest.mark.parametrize("mode", ["sph", "aniso", "avg", "corr", "rad"])
def test_emulated_properties_on_raw_meshes(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    mk = mode_kwargs(emu, mode, p, kw)
    rec = emu.reconstruct_surface(p, simd=False, subdomain_grid_auto_disable=False, with_debug=True, **kw, **mk)
    f = emu.LevelSetField(p, **kw, **mk)
    try:
        check_properties(emu, f, rec, f.signed_distance(rec.mesh, band=3))
    finally:
        f.close()


# ------------------------------------------------------------------ refusals and handles ----
def test_emulated_refusals_and_reuse(emu):  # noqa: F811
    ss = emu
    p = _cube(6, 5)
    ctx = ss.Context()
    try:
        rec = ss.reconstruct_surface(p, context=ctx, simd=False, subdomain_grid_auto_disable=False, **KW)
        mesh = rec.mesh.copy()
        f1 = ss.LevelSetField(p, context=ctx, **KW)
        L = ctx._L
        v, t = mesh.vertices, mesh.triangles.astype(np.uint32)
        h = C.c_void_p()
        for band in (0, 9):
            with pytest.raises(ss.SplashsurfError, match="band"):
                f1.signed_distance(mesh, band=band)
        with pytest.raises(TypeError):
            f1.signed_distance((v.astype(np.float64), t))
        bad = v.copy()
        bad[7, 2] = np.nan
        with pytest.raises(ss.SplashsurfError, match="vertex 7"):
            f1.signed_distance((bad, t))
        tb = t.copy()
        tb[11, 1] = len(v)
        with pytest.raises(ss.SplashsurfError, match="triangle 11"):
            f1.signed_distance((v, tb))
        with pytest.raises(ValueError):
            f1.signed_distance((v, mesh.triangles.astype(np.int64) - 1))
        assert L.ss_levelset_field_sdf_f32(f1._s, None, len(v), t.ctypes.data, len(t), 3, C.byref(h)) != 0
        assert "NULL" in L.ss_last_error().decode()
        assert L.ss_levelset_field_sdf_f32(f1._s, v.ctypes.data, 1 << 32, t.ctypes.data, len(t), 3, C.byref(h)) == 4
        assert L.ss_levelset_field_sdf_f32(f1._s, v.ctypes.data, len(v), t.ctypes.data, len(t), 3, None) != 0
        # one context: queries, grids and a later field; the grid outlives the field's records
        pts = (np.asarray(f1.grid.aabb.min, np.float32) + 0.37).reshape(1, 3).astype(np.float32)
        e1 = f1.evaluate(pts)
        g1 = f1.signed_distance(mesh)
        assert np.array_equal(f1.evaluate(pts), e1)
        g2 = f1.signed_distance((v, t))
        assert_sdf_equal(g2, g1.brick_coords, g1.values, g1.brick_inside)
        ss.reconstruct_surface(p, context=ctx, **KW)
        with pytest.raises(ss.SplashsurfError, match="gone"):
            f1.signed_distance(mesh)
        f2 = ss.LevelSetField(p, context=ctx, **KW)
        assert_sdf_equal(f2.signed_distance(mesh), g1.brick_coords, g1.values, g1.brick_inside)
        assert g1.to_dense().shape == tuple(f2.grid.npoints_per_dim)
        f1.close()
        f2.close()
    finally:
        ctx.close()


# ------------------------------------------------------------------ CLI ----
def test_emulated_cli_output_sdf(emu, tmp_path):  # noqa: F811
    from splashsurf_b200 import __main__ as cli, io
    p = _cube(6, 21)
    src = tmp_path / "cube_{}.xyz"
    for k in (1, 2):
        io.write_particles(str(tmp_path / f"cube_{k}.xyz"), (p + np.float32(0.01 * k)).astype(np.float32))
    base = ["reconstruct", str(src), f"-r={KW['particle_radius']}", "-l=2.0", f"-c={KW['cube_size']}", "--subdomain-grid-auto-disable=on",
            "--simd=off", "-q", "--output-dir", str(tmp_path / "out")]
    assert cli.main(base + ["--output-sdf", str(tmp_path / "out" / "sdf_{}.npz"), "--sdf-band", "2", "--mesh-smoothing-iters=3"]) == 0
    for k in (1, 2):
        z = np.load(tmp_path / "out" / f"sdf_{k}.npz")
        q = (p + np.float32(0.01 * k)).astype(np.float32)
        rec = emu.reconstruct_surface(q, simd=False, subdomain_grid_auto_disable=False, **KW)
        f = emu.LevelSetField(q, **KW)
        want = f.signed_distance(rec.mesh, band=2)
        assert_sdf_equal(type("G", (), dict(brick_coords=z["brick_coords"], values=z["values"], brick_inside=z["brick_inside"])), want.brick_coords,
                         want.values, want.brick_inside)
        assert z["band"] == 2 and z["background"] == np.float32(want.background) and z["cell"] == np.float32(f.grid.cell_size)
        assert np.array_equal(z["min"], np.asarray(f.grid.aabb.min, np.float32)) and list(z["points_per_dim"]) == f.grid.npoints_per_dim
        f.close()
    with pytest.raises(ValueError, match="partition"):
        cli.main(base + ["--output-sdf", str(tmp_path / "x_{}.npz"), "--partition=on"])
