"""The level-set certification at thresholds inside the fluid, checked point by point (DESIGN.md section 4.3).

The certification sweep stores SS_MARKER at grid points whose cubic lower bound exceeds threshold * (1 + 1e-4), and never
computes their exact value.  Mesh parity cannot see an unsound bound: at the usual thresholds (0.1 .. 0.8) every interior value
is far above t, and near the surface the fix-up pass re-evaluates every marker that has an outside 6-neighbour, which repairs a
wrongly certified point there.  So this module takes its thresholds from the field itself -- the values v at the 50 %, 70 % and
90 % quantiles of the busiest tile's nonzero values, with t = v, the neighbouring floats of v, and v / (1 + 1e-4), which puts a
point right at the certification margin -- and reads the tile back as the certification and exact pass left it
(ss_context_keep_levelset_tile_raw, taken before the fix-up).  For every point of a touched brick:
* a marker must have an exact (oracle) value strictly above t;
* any other point must equal the oracle's value bit for bit.
Per case and threshold the mesh, densities and vertex keys also equal the oracle bit for bit for level-set variants 2, 1, 0 and
exact evaluation everywhere.  The equality thresholds put grid values exactly on t, where the subdomain path classifies by
v > t and the global path also counts v == t as above next to a point below; with the reference's wheel unpacked the oracle is
pinned to it there.

CASES is shared with tests/test_zzz_gpu_levelset_threshold.py (H100).  The CPU executor cannot reproduce the device's slice sizes,
mbarrier phases or register allocation: the H100 run is the one that counts for the sweep.  The sensitivity test below compiles
the executor from patched sources (bound scaled up; ring-1 sweep counting ring-0 candidates again) and requires the table to catch
both."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_emulated_pipeline import CSRC, EMUL_DIR, ROOT, build_emulated_library, emu  # noqa: F401  (emu: fixture)
from test_zzz_gpu_levelset_paths import _cluster, taken_cells

MARKER = np.float32(3.0e38)
CERT_MARGIN = 1e-4                     # relative margin of the certification test (ss_certify.cuh)
NEAR = 1e-3                            # "just above t": t < v <= t (1 + NEAR)

BASE = dict(particle_radius=0.025, smoothing_length=2.0)
SUB = dict(subdomain_grid_auto_disable=False)
GLOBAL = dict(subdomain_grid=False)
R_LAT = 2.0 ** -5                      # lattice radius: cube_size 0.5 gives the cell 2^-6, every grid coordinate is exact in f32


def _cube(n, seed):
    from splashsurf_b200 import synthetic as syn
    return syn.jittered_cube(n, 0.025, seed)


def _lattice(n):
    """n^3 particles with spacing 2 r on exact multiples of 2 r: with cube_size 0.5 each sits on a grid point (index 4 k + R + 1)."""
    ax = np.arange(n, dtype=np.float64) * 2 * R_LAT
    return np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)


def _droplets():
    from splashsurf_b200 import synthetic as syn
    return syn.splash((8, 8, 8), 4, 0.025, 41)


# name -> (cloud, reconstruction keywords, options, path cells the case must take)
# options: tile_batch, tile ("busiest" or "busiest_sparse"), certifies (at least one marker expected), mode ("aniso" / "averaged")
CASES = {
    "cube_S16_R8": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **SUB), {}, ["cert/sub/384"]),
    "cube_S16_R9": (lambda: _cube(8, 2), dict(BASE, cube_size=0.45, subdomain_num_cubes_per_dim=16, **SUB), {}, ["cert/sub/576_R9"]),
    "cube_S16_R14_fused": (lambda: _cube(6, 3), dict(BASE, cube_size=0.3, subdomain_num_cubes_per_dim=16, **SUB), {}, ["cert/sub/fused_R"]),
    "cube_S16_R20_bins16": (lambda: _cube(5, 4), dict(BASE, cube_size=0.2, subdomain_num_cubes_per_dim=16, **SUB), {},
                            ["cert/sub/576_R17_25"]),
    "cube_S64_R8": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **SUB), {}, ["cert/sub/384"]),
    "cube_S64_R9": (lambda: _cube(8, 1), dict(BASE, cube_size=0.45, **SUB), {}, ["cert/sub/576_R9"]),
    "cube_S64_R14_fused": (lambda: _cube(8, 1), dict(BASE, cube_size=0.3, **SUB), {}, ["cert/sub/fused_R"]),
    "cube_S64_R20_bins16": (lambda: _cube(6, 1), dict(BASE, cube_size=0.2, **SUB), {}, ["cert/sub/576_R17_25"]),
    "lattice_on_grid_points": (lambda: _lattice(8), dict(particle_radius=R_LAT, smoothing_length=2.0, cube_size=0.5, **SUB), {},
                               ["cert/sub/384"]),
    "droplets_sparse_scalar": (_droplets, dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, simd=False, **SUB),
                               dict(tile="busiest_sparse"), ["cert/sub/384"]),
    "cube_S16_tile_batch_1": (lambda: _cube(8, 5), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **SUB), dict(tile_batch=1),
                              ["cert/sub/384"]),
    "cube_global": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **GLOBAL), {}, ["cert/global/384"]),
    # the global path tiles its grid in 64-cube tiles whatever subdomain_num_cubes_per_dim says
    "cube_global_S16": (lambda: _cube(8, 8), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **GLOBAL), {}, ["cert/global/384"]),
    # more candidates than the 384 slice around every brick of the cluster: those bricks go to the exact cascade whole
    "cluster_whole_bricks": (lambda: _cluster(600), dict(BASE, cube_size=0.5, **SUB), dict(certifies=False), ["exact/sub/1024"]),
    # opt-in surfaces: exact values only
    "aniso_never_certifies": (lambda: _cube(8, 6), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **SUB),
                              dict(mode="aniso", certifies=False), []),
    "averaged_never_certifies": (lambda: _cube(8, 7), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **SUB),
                                 dict(mode="averaged", certifies=False), []),
}


def thresholds(vals):
    """(label, t, kind) from the nonzero grid values: the 50 / 70 / 90 % quantile values v (actual grid values) with t = v, the
    neighbouring floats of v and v / (1 + 1e-4) (a point right at the certification margin), and the control t = 0.6."""
    nz = np.sort(vals[vals > 0].astype(np.float32))
    out = []
    for q in (50, 70, 90):
        v = nz[int(q / 100 * (len(nz) - 1))]
        out += [(f"q{q}_eq", v, "eq"), (f"q{q}_up", np.nextafter(v, np.float32(np.inf)), "up"),
                (f"q{q}_down", np.nextafter(v, np.float32(-np.inf)), "down"),
                (f"q{q}_margin", np.float32(np.float64(v) / (1 + CERT_MARGIN)), "margin")]
    out.append(("control_0.6", np.float32(0.6), "control"))
    return out


def pick_tile(o, opts):
    """Flat index of the tile the case checks: the subdomain with most particles (sparse ones only for "busiest_sparse"); the
    global path's tile 0 (the clouds fit into one 64-cube tile)."""
    if not o["used_decomposition"]:
        return 0
    cnt = o["subdomain_count"].astype(np.int64)
    if opts.get("tile") == "busiest_sparse":
        assert o["subdomain_sparse"].any(), "no sparse subdomain"
        cnt = np.where(o["subdomain_sparse"], cnt, -1)
    return int(o["subdomain_flat"][int(np.argmax(cnt))])


def run(lib, p, kw, opts, flat, variant=2, exact=False, raw=True):
    """One reconstruction on a fresh context; returns (result with debug taps, raw tile, brick states, plain tile or None)."""
    ctx = lib.Context()
    L = ctx._L
    try:
        ctx.set_levelset_variant(variant)
        ctx.set_levelset_exact_everywhere(exact)
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        mode = opts.get("mode")
        plain = mode is not None                          # the opt-in modes: also the plain tap, which they equal
        lib._check(L, L.ss_context_keep_levelset_tile_raw(ctx._h, flat if raw else -1))
        lib._check(L, L.ss_context_keep_levelset_tile(ctx._h, flat if plain else -1))
        prm = lib.make_params(**kw)
        arr = np.ascontiguousarray(p)
        s = lib._reconstruct_raw(ctx, arr, prm, lib.Anisotropy() if mode == "aniso" else None,
                                 lib.AveragedSurface() if mode == "averaged" else None)
        try:
            g = lib._collect(ctx, s, len(arr), prm, True, plain)
            tile = bst = None
            if raw:
                npt = (64 if not kw.get("subdomain_grid", True) else kw.get("subdomain_num_cubes_per_dim", 64)) + 1
                nb = (npt + 7) // 8
                tile, bst = np.empty((npt,) * 3, np.float32), np.empty((nb,) * 3, np.uint8)
                lib._check(L, L.ss_surface_copy_levelset_tile_raw(s, tile.ctypes.data, bst.ctypes.data))
            return g, tile, bst, g.levelset_tile if plain else None
        finally:
            ctx.free_surface(s)
    finally:
        ctx.close()


def _parity(oracle_mod, a, b_v, b_t, b_k, kw):
    return oracle_mod.mesh_parity(a.mesh.vertices, a.mesh.triangles, a.vertex_edge_keys, b_v, b_t, b_k, kw.get("subdomain_num_cubes_per_dim", 64))


def raw_check(tile, bst, exact, t):
    """Markers against the exact values: (wrong markers, mismatching points, markers, realised margin min v / t - 1, touched).
    Mismatching points: evaluated points of touched bricks that differ from the exact value, and points of untouched bricks (the
    stage left them unwritten: no candidate) whose exact value is not 0."""
    n = tile.shape[0]
    idx = np.arange(n) // 8
    touched = bst[idx[:, None, None], idx[None, :, None], idx[None, None, :]] > 0
    mk = touched & (tile == MARKER)
    wrong = int((mk & ~(exact > t)).sum())
    ev = touched & ~mk
    mismatch = int((tile[ev].view(np.uint32) != exact[ev].view(np.uint32)).sum()) + int((exact[~touched] != 0).sum())
    margin = float((exact[mk].astype(np.float64) / np.float64(t) - 1).min()) if mk.any() else float("nan")
    return wrong, mismatch, int(mk.sum()), margin, touched


def _bricks_over_slice(p, g, flat, kw, cap):
    """Bricks of the tile with more than `cap` particles within h of their point box: they have more candidates than the slice."""
    h = float(np.float32(2 * kw["smoothing_length"] * kw["particle_radius"]))
    c = float(g.grid.cell_size)
    S = kw.get("subdomain_num_cubes_per_dim", 64)
    nsd = g.subdomain_grid.ncells_per_dim
    ijk = np.array([flat // (nsd[1] * nsd[2]), (flat // nsd[2]) % nsd[1], flat % nsd[2]])
    lo0 = np.asarray(g.grid.aabb.min, np.float64) + ijk * S * c
    nb = (S + 8) // 8
    over = np.zeros((nb,) * 3, bool)
    pp = p.astype(np.float64)
    for b in np.ndindex(*over.shape):
        lo = lo0 + np.array(b) * 8 * c
        hi = lo0 + np.minimum(np.array(b) * 8 + 7, S) * c
        d = np.maximum(np.maximum(lo - pp, pp - hi), 0)
        over[b] = int(((d ** 2).sum(1) < h * h).sum()) > cap
    return over


def check_case(lib, oracle_mod, name, variants=(2, 1, 0, "exact")):
    """All assertions of one case over its thresholds; returns the per-threshold report rows."""
    gen, kw, opts, expected = CASES[name]
    p = gen()
    o0 = oracle_mod.reconstruct(p, **kw)
    flat = pick_tile(o0, opts)
    exact = oracle_mod.reconstruct(p, tile_of_subdomain=flat, **kw)["tile"]
    mode = opts.get("mode")
    rows, n_markers, n_near_case = [], 0, 0
    for label, t, kind in thresholds(exact):
        kwt = dict(kw, iso_surface_threshold=float(t))
        g, tile, bst, plain = run(lib, p, kwt, opts, flat)
        n_eq = int((exact == t).sum())
        n_near = int(((exact > t) & (exact.astype(np.float64) <= np.float64(t) * (1 + NEAR))).sum())
        if kind == "eq" and mode is None:
            assert n_eq >= 1, (name, label)
        n_near_case += n_near
        wrong, mismatch, nm, margin, touched = raw_check(tile, bst, exact if plain is None else plain, t)
        assert touched.any(), (name, label)
        assert wrong == 0, (name, label, "markers at points whose exact value is not above t", wrong)
        assert mismatch == 0, (name, label, "evaluated points that differ from the oracle", mismatch)
        n_markers += nm
        rows.append((name, label, float(t), n_eq, n_near, nm, margin))
        print(f"{name:26s} {label:12s} t={float(t):.9g} v==t: {n_eq:4d}  t<v<=t(1+1e-3): {n_near:5d}  markers: {nm:6d}  "
              f"min v/t-1 over markers: {margin:.3e}")
        if mode is not None:
            assert nm == 0 and np.array_equal(tile[touched].view(np.uint32), plain[touched].view(np.uint32)), (name, label)
            continue
        cells = taken_cells(g.levelset_paths, kw, opts, g.subdomains)
        assert set(expected) <= cells, (name, label, sorted(set(expected) - cells), g.levelset_paths)
        if name == "cluster_whole_bricks":
            over = _bricks_over_slice(p, g, flat, kw, 384)
            assert over.any()
            idx = np.arange(tile.shape[0]) // 8
            in_over = over[idx[:, None, None], idx[None, :, None], idx[None, None, :]]
            assert not (in_over & (tile == MARKER)).any(), (name, label)
        if name == "lattice_on_grid_points":
            q = (p.astype(np.float64) - np.asarray(g.grid.aabb.min, np.float64)) / float(g.grid.cell_size)
            assert np.array_equal(q, np.rint(q)), "lattice particles are not on grid points"
        o = oracle_mod.reconstruct(p, **kwt)
        assert np.array_equal(g.particle_densities, o["particle_densities"]), (name, label)
        first = None
        for v in variants:
            if v == 2:
                gv = g
            else:
                # the CTA certification kernel (variant 1) and the fused kernel (variant 0) are checked marker by marker as well;
                # exact evaluation everywhere must leave no marker
                gv, tv, bv, _ = run(lib, p, kwt, opts, flat, variant=2 if v == "exact" else v, exact=v == "exact")
                wv, mv, nmv = raw_check(tv, bv, exact, t)[:3]
                assert wv == 0 and mv == 0, (name, label, v, "raw tile", wv, mv)
                assert nmv == 0 or v != "exact", (name, label, nmv)
            m = _parity(oracle_mod, gv, o["vertices"], o["triangles"], o["vertex_keys"], kw)
            assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, (name, label, v, m)
            if first is None:
                first = gv
            else:
                m = _parity(oracle_mod, gv, first.mesh.vertices, first.mesh.triangles, first.vertex_edge_keys, kw)
                assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, (name, label, v, m)
    if mode is None:
        assert n_near_case > 0, (name, "no grid value just above a threshold")
    if opts.get("certifies", True):
        assert n_markers > 0, name
    else:
        assert n_markers == 0, name
    return rows


def check_reference(oracle_mod, name):
    """The oracle equals the reference's wheel on the equality thresholds (the '>' rule of the subdomain path, the global path's
    '>= with a neighbour below' rule)."""
    gen, kw, opts, _ = CASES[name]
    p = gen()
    o0 = oracle_mod.reconstruct(p, **kw)
    exact = oracle_mod.reconstruct(p, tile_of_subdomain=pick_tile(o0, opts), **kw)["tile"]
    ps = oracle_mod.reference()
    compared = 0
    for label, t, kind in thresholds(exact):
        if kind != "eq":
            continue
        kwt = dict(kw, iso_surface_threshold=float(t))
        o = oracle_mod.reconstruct(p, **kwt)
        assert o["rc"] == 0, (name, label)
        try:
            r = ps.reconstruct_surface(p, multi_threading=False, **kwt)
        except RuntimeError as e:
            # the reference's global path marks a point with v == t "above" only in the cells next to its crossing edge, and in
            # another cell the same corner reads "below" (v > t fails): that cell then lacks a vertex the table needs and the
            # reference stops with this error, where the oracle and the device mark the point in every cell (DESIGN.md 4.3)
            assert not kw.get("subdomain_grid", True) and "Missing iso surface vertex" in str(e), (name, label, str(e)[:300])
            print(f"{name} {label}: the reference stops (missing iso-surface vertex); the oracle gives {len(o['vertices'])} vertices")
            continue
        compared += 1
        assert np.array_equal(np.asarray(r.particle_densities), o["particle_densities"]), (name, label)
        rv, rt = np.asarray(r.mesh.vertices), np.asarray(r.mesh.triangles)
        keys = oracle_mod.resolve_keys(rv, o["grid"]["aabb_min"], o["grid"]["cell_size"], o["vertex_keys"], rt, o["triangles"],
                                       known_vertices=o["vertices"])
        m = oracle_mod.mesh_parity(rv, rt, keys, o["vertices"], o["triangles"], o["vertex_keys"], kw.get("subdomain_num_cubes_per_dim", 64))
        assert m["keys_equal"] and m["triangles_equal"] and m["n_interior_not_bitexact"] == 0, (name, label, m)
    assert compared >= 2, name


STANDARD = [n for n, c in CASES.items() if c[2].get("mode") is None]


# ------------------------------------------------------------------ CPU executor ----
@pytest.mark.parametrize("name", list(CASES))
def test_emulated_levelset_threshold(emu, oracle_mod, name):
    check_case(emu, oracle_mod, name)


@pytest.mark.parametrize("name", ["cube_S16_R8", "cube_global", "lattice_on_grid_points"])
def test_oracle_equals_reference_at_equality_thresholds(oracle_mod, name):
    if not oracle_mod.reference_available():
        pytest.skip("oracle/_ref not unpacked")
    check_reference(oracle_mod, name)


def test_oracle_global_tile_whatever_the_subdomain_size(oracle_mod):
    """The oracle's tile tap on the global path returns the 65^3 points of a 64-cube tile of the global grid for every subdomain
    size, also when auto-disable falls back to the global path; the subdomain path returns (S + 1)^3 points."""
    p = _cube(4, 9)
    kw = dict(BASE, cube_size=0.5)
    want = oracle_mod.reconstruct(p, tile_of_subdomain=0, **kw, **GLOBAL)["tile"]
    assert want.shape == (65,) * 3 and (want > 0).sum() > 1000
    for S in (16, 32, 96):
        o = oracle_mod.reconstruct(p, subdomain_num_cubes_per_dim=S, tile_of_subdomain=0, **kw, **GLOBAL)
        assert not o["used_decomposition"] and np.array_equal(o["tile"].view(np.uint32), want.view(np.uint32)), S
    q = _cube(2, 9)                                    # a grid of at most 1.2 S cells: auto-disable takes the global path
    o = oracle_mod.reconstruct(q, subdomain_num_cubes_per_dim=32, tile_of_subdomain=0, **kw)
    assert not o["used_decomposition"] and o["tile"].shape == (65,) * 3
    assert np.array_equal(o["tile"], oracle_mod.reconstruct(q, tile_of_subdomain=0, **kw, **GLOBAL)["tile"])
    o = oracle_mod.reconstruct(p, subdomain_num_cubes_per_dim=16, tile_of_subdomain=int(pick_tile(oracle_mod.reconstruct(
        p, subdomain_num_cubes_per_dim=16, **kw, **SUB), {})), **kw, **SUB)
    assert o["used_decomposition"] and o["tile"].shape == (17,) * 3 and (o["tile"] > 0).any()


def test_case_table_covers_every_certification_path():
    """The path cells the standard cases claim cover every certification slice and the fused kernel on the subdomain path, and
    the global path (each case's claim, and the spread of its values around the thresholds, are checked by check_case)."""
    claimed = set()
    for name in STANDARD:
        claimed |= set(CASES[name][3])
    assert {"cert/sub/384", "cert/sub/576_R9", "cert/sub/576_R17_25", "cert/sub/fused_R", "cert/global/384"} <= claimed


# ------------------------------------------------------------------ sensitivity: patched sources must be caught ----
SCALES = (1.02, 1.05, 1.10)


def _patched_library(tmp, tag, patch):
    """Compiles the CPU executor from a patched copy of csrc/ (the flags of build_emulated_library); returns (Popen, .so path)."""
    src = os.path.join(tmp, tag, "splashsurf_b200", "csrc")
    shutil.copytree(CSRC, src)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, tag, "include"))
    patch(src)
    so = os.path.join(tmp, tag, "libsplashsurf_emul.so")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-w", "-x", "c++", "-DSS_HOST_EMUL", "-I" + cuda_inc,
           "-include", os.path.join(EMUL_DIR, "cuda_emul.h"), "-shared", "-fPIC", "-pthread",
           "-Wl,-Bsymbolic", "-o", so, os.path.join(src, "ss_pipeline.cu")]
    return subprocess.Popen(cmd), so


def _edit(path, old, new):
    s = open(path).read()
    assert s.count(old) == 1, (path, old)
    open(path, "w").write(s.replace(old, new))


def _scale_bound(k):
    def patch(src):
        path = os.path.join(src, "ss_kernels.cuh")
        s = open(path).read()
        for g in range(4):
            m = re.search(rf"#define SS_G{g} (-?[0-9.]+)f", s)
            s = s.replace(m.group(0), f"#define SS_G{g} ({m.group(1)}f * {k}f)")
        open(path, "w").write(s)
    return patch


def _ring0_twice(src):
    _edit(os.path.join(src, "ss_certify.cuh"), "keep = (db2 < A.r1sq) && !(db2 < A.r0sq);", "keep = (db2 < A.r1sq);")


def _detects(lib, oracle_mod, names):
    """Cases whose raw-tile check fails with the library `lib` is bound to (default launch path, every threshold of the case)."""
    caught = []
    for name in names:
        gen, kw, opts, _ = CASES[name]
        p = gen()
        o0 = oracle_mod.reconstruct(p, **kw)
        flat = pick_tile(o0, opts)
        exact = oracle_mod.reconstruct(p, tile_of_subdomain=flat, **kw)["tile"]
        for label, t, kind in thresholds(exact):
            _, tile, bst, _ = run(lib, p, dict(kw, iso_surface_threshold=float(t)), opts, flat)
            wrong, mismatch = raw_check(tile, bst, exact, t)[:2]
            if wrong or mismatch:
                caught.append([name, label, wrong, mismatch])
                break
    return caught


# one process per library: two copies of the CPU executor do not share a process
DETECT_WORKER = r"""
import ctypes as C, json, os, sys
sys.path[:0] = [os.environ["SS_ROOT"], os.path.join(os.environ["SS_ROOT"], "tests")]
import oracle, splashsurf_b200 as ss
import test_levelset_threshold as T
ss._LIB = ss._bind(C.CDLL(os.environ["SS_EMUL_SO"]))
print("CAUGHT " + json.dumps(T._detects(ss, oracle, json.loads(os.environ["SS_CASES"]))))
"""


SENSITIVITY_CASES = ["cube_S16_R8", "cube_S16_R9", "cube_S16_R14_fused", "lattice_on_grid_points", "cube_global"]


def test_emulated_raw_check_catches_unsound_certification(oracle_mod, tmp_path):
    """The raw-tile check fails for an executor whose cubic bound is scaled up (1.10: one model of the sweep puts the first wrong
    markers there on a jittered cube) and for one whose ring-1 sweep admits the ring-0 candidates again (counted twice); the
    unpatched executor passes.  Prints the smallest scale the table detects."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    base = build_emulated_library()                     # skips without the CUDA headers
    jobs = {f"scale_{k}": _patched_library(str(tmp_path), f"scale_{k}", _scale_bound(k)) for k in SCALES}
    jobs["ring0_twice"] = _patched_library(str(tmp_path), "ring0_twice", _ring0_twice)
    for tag, (proc, _) in jobs.items():
        assert proc.wait() == 0, tag
    import json
    import sys
    script = tmp_path / "detect.py"
    script.write_text(DETECT_WORKER)
    libs = dict({tag: so for tag, (_, so) in jobs.items()}, unpatched=base)
    procs = {tag: subprocess.Popen([sys.executable, str(script)], stdout=subprocess.PIPE, text=True,
                                   env=dict(os.environ, SS_ROOT=ROOT, SS_EMUL_SO=so, SS_CASES=json.dumps(SENSITIVITY_CASES), SS_EMUL_THREADS="2"))
             for tag, so in libs.items()}
    found = {}
    for tag, proc in procs.items():
        out, _ = proc.communicate(timeout=1800)
        assert proc.returncode == 0, (tag, out[-2000:])
        found[tag] = json.loads([ln for ln in out.splitlines() if ln.startswith("CAUGHT ")][-1][7:])
    assert found.pop("unpatched") == []
    for tag, caught in found.items():
        print(f"{tag:12s} caught by {len(caught)} of {len(SENSITIVITY_CASES)} cases: {caught}")
    detected = [k for k in SCALES if found[f"scale_{k}"]]
    print("smallest bound scale detected:", min(detected) if detected else None)
    assert found[f"scale_{SCALES[-1]}"], "a bound scaled by 1.10 went unnoticed"
    assert found["ring0_twice"], "a ring-1 sweep counting ring-0 candidates twice went unnoticed"
