"""The device path against the oracle across length scales and far from the origin.

The reference's f32 arithmetic is free of units: scale a cloud (particles, particle_radius, AABB) by 2^k and every operation is scaled
exactly, so its output is 2^k times the output at k = 0, for as long as nothing leaves the normal range.  The device must follow it
bit for bit at every such k, and do the same work: the level-set certification bound runs in coordinates scaled by a power of two
near 1 / h (DESIGN.md 4.3), so its decisions -- and with them `levelset_paths` and the work counters -- do not depend on k.

Far from the origin f32 grid coordinates round by a growing fraction of a cell c.  Offsets are classified by the band
log2(ulp(|coordinate|) / c); up to 1/64 the device must match the oracle bit for bit (level-set tile of one subdomain included),
and the oracle the reference's binary; past it the reconstruction is refused with SS_ERR_REAL_TOO_SMALL.

The same tables run on the H100 (`ss` fixture) and on the CPU executor of the CUDA sources (`emu`)."""
import math

import numpy as np
import pytest

from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)
from test_zzz_gpu_levelset_paths import _aniso_cluster, _cluster, _cube

BASE = dict(particle_radius=0.025, smoothing_length=2.0)
SUB = dict(subdomain_grid_auto_disable=False)


def _splash():
    from splashsurf_b200 import synthetic as syn
    return syn.splash((8, 8, 8), 2, 0.025, 105).astype(np.float32)


# name -> (cloud, reconstruction keywords, context options); the launch paths of test_zzz_gpu_levelset_paths that a scale can reach
CASES = {
    "cube_R8": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **SUB), {}),
    "splash_sparse": (_splash, dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16, **SUB), {}),
    "splash_aabb": (_splash, dict(BASE, cube_size=0.5, aabb_min=[-0.05, -0.05, -0.05], aabb_max=[0.3, 0.25, 0.3], **SUB), {}),
    "cube_scalar": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, simd=False, **SUB), {}),
    "cube_global": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, subdomain_grid=False), {}),
    "cube_R9": (lambda: _cube(8, 1), dict(BASE, cube_size=0.45, **SUB), {}),
    "cluster_1024": (lambda: _cluster(600), dict(BASE, cube_size=0.5, **SUB), {}),
    "cluster_4096": (lambda: _cluster(1500), dict(BASE, cube_size=0.5, **SUB), {}),
    "cube_exact_everywhere": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **SUB), dict(exact_everywhere=True)),
    "cube_variant1": (lambda: _cube(8, 1), dict(BASE, cube_size=0.5, **SUB), dict(variant=1)),
    "aniso": (lambda: _aniso_cluster(300, 511), dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16), dict(aniso=True)),
}

# Powers of two around h = 0.1 (k = 0).  Bands of the certification coefficients G_k / h^(2k) if they were taken in absolute
# units (what they were before the bound was scaled): g3 overflows for h < 5e-7 (k <= -18), is normal up to h = 2.8e6 (k <= 24),
# denormal up to h = 5e7 (k <= 28), zero beyond.  The bound must be sound and do the same work in every band.
K_ALL = [-36, -22, -18, -17, 0, 24, 25, 26, 27, 28, 29, 30, 36]
K_SOME = [-22, 0, 27, 30]
# k = -36 and 36: inside the reference's window (the oracle self-check below passes there); volumes reach 4e-38 at k = -36, a
# step further they leave the normal f32 range and the reference itself stops being free of units.
SCALES = [("cube_R8", k) for k in K_ALL] + [(n, k) for n in CASES if n != "cube_R8" for k in K_SOME]


def scale_band(k):
    """Where f32(G3 / h^6), the coefficient as it would be rounded in absolute units, lies at h = 0.1 * 2^k."""
    from test_certification_bound import _coeffs
    with np.errstate(over="ignore", under="ignore"):
        g3 = abs(np.float32(_coeffs()[3] / (0.1 * 2.0 ** k) ** 6))
    if not np.isfinite(g3):
        return "g3_overflow"
    if g3 == 0:
        return "g3_zero"
    return "g3_denormal" if g3 < np.finfo(np.float32).tiny else "normal"


def _scaled(kw, s):
    kw = dict(kw)
    kw["particle_radius"] = kw["particle_radius"] * s
    for a in ("aabb_min", "aabb_max"):
        if a in kw:
            kw[a] = [float(np.float32(v) * np.float32(s)) for v in kw[a]]
    return kw


def _run(lib, p, kw, opts, count=False, tile=None):
    ctx = lib.Context()
    try:
        ctx.set_count_pairs(count)
        if opts.get("exact_everywhere"):
            ctx.set_levelset_exact_everywhere(True)
        if opts.get("variant"):
            ctx.set_levelset_variant(opts["variant"])
        if opts.get("tile_batch"):
            ctx.set_tile_batch(opts["tile_batch"])
        an = lib.Anisotropy() if opts.get("aniso") else None
        return lib.reconstruct_surface(p, with_debug=True, context=ctx, anisotropy=an, keep_levelset_tile_of=tile, **kw)
    finally:
        ctx.close()


def _oracle(oracle_mod, p, kw, opts, tile=None):
    if opts.get("aniso"):
        from test_anisotropic import oracle_reconstruct_anisotropic
        o = oracle_reconstruct_anisotropic(p, tile_of_subdomain=tile, **kw)
        assert o["rc"] == 0
        return o
    return oracle_mod.reconstruct(p, tile_of_subdomain=tile, **kw)


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                  b.view(np.uint32) if b.dtype == np.float32 else b)


def check_device(lib, oracle_mod, p, kw, opts, tile=False):
    """Device vs oracle, bit for bit: densities, subdomain lists, mesh keys, triangles, vertices (and one level-set tile)."""
    g = _run(lib, p, kw, opts)
    o = _oracle(oracle_mod, p, kw, opts)
    assert _same_bits(g.particle_densities, o["particle_densities"])
    if o.get("used_decomposition") and not opts.get("aniso"):
        assert np.array_equal(g.subdomains["flat"], o["subdomain_flat"]) and np.array_equal(g.subdomains["count"], o["subdomain_count"])
        assert np.array_equal(g.subdomains["sparse"], o["subdomain_sparse"])
    m = oracle_mod.mesh_parity(g.mesh.vertices, g.mesh.triangles, g.vertex_edge_keys, o["vertices"], o["triangles"], o["vertex_keys"],
                               kw.get("subdomain_num_cubes_per_dim", 64))
    assert m["keys_equal"] and m["triangles_equal"] and m["n_not_bitexact"] == 0, m
    if tile and g.subdomains is not None and len(g.subdomains["flat"]):
        f = int(g.subdomains["flat"][len(g.subdomains["flat"]) // 2])
        gt = _run(lib, p, kw, opts, tile=f).levelset_tile
        ot = _oracle(oracle_mod, p, kw, opts, tile=f)["tile"]
        diff = np.argwhere(gt.view(np.uint32) != ot.view(np.uint32))
        assert len(diff) == 0, (f, len(diff), diff[:4].tolist(), [(float(gt[tuple(d)]), float(ot[tuple(d)])) for d in diff[:4]])
    return g, o


WORK = ("levelset_fixup_points", "bricks_fixscan", "levelset_cert_evals", "bricks_levelset", "bricks_mc")


def check_scale(lib, oracle_mod, name, k):
    gen, kw0, opts = CASES[name]
    p0 = gen()
    s = np.float32(2.0 ** k)
    p, kw = (p0 * s).astype(np.float32), _scaled(kw0, float(s))
    assert np.array_equal(p / s, p0)                                                # the scaling itself is exact
    # oracle self-check: the reference's arithmetic is free of units at this k
    o0, ok = _oracle(oracle_mod, p0, kw0, opts), _oracle(oracle_mod, p, kw, opts)
    assert _same_bits(ok["particle_densities"], o0["particle_densities"])
    assert _same_bits(ok["vertices"], (o0["vertices"] * s).astype(np.float32)) and np.array_equal(ok["triangles"], o0["triangles"])
    g, _ = check_device(lib, oracle_mod, p, kw, opts)
    # work invariance, with pair counting on: the same kernels on the same bricks, the same certification work
    if not opts.get("aniso"):
        c0, ck = _run(lib, p0, kw0, opts, count=True), _run(lib, p, kw, opts, count=True)
        assert ck.levelset_paths == c0.levelset_paths, (ck.levelset_paths, c0.levelset_paths)
        assert {w: ck.timings[w] for w in WORK} == {w: c0.timings[w] for w in WORK}
        assert ck.timings["levelset_pairs"] == c0.timings["levelset_pairs"]
    else:
        assert g.levelset_paths == _run(lib, p0, kw0, opts).levelset_paths


# ------------------------------------------------------------------ offsets ----
# band b: ulp(|coordinate|) / c in [2^b, 2^(b+1)), with c = 0.0125 (cube_size 0.5 of r = 0.025).  The cloud is centred on the
# origin, then offset by (o, -o, o) or (-o, o, -o), o = 1.5 * 2^e so that the whole grid stays in one binade.  Band -18 is the
# centred cloud, moved so that |coordinate| is in [0.5, 1): the closest to the origin a cloud of this extent gets.
C = 0.0125
OFFSET_BANDS = [-18, -10, -7, -5, -3, -1]
REFUSED_BANDS = [-5, -3, -1]                  # ulp / c > 1/64: SS_ERR_REAL_TOO_SMALL


def band_offset(b):
    e = math.floor(math.log2(C * 2.0 ** b)) + 24          # ulp in [2^e, 2^(e+1)) is 2^(e - 23) = c 2^b rounded down to a power of 2
    return 1.5 * 2.0 ** e


def offset_band(amax):
    return math.floor(math.log2(2.0 ** (math.floor(math.log2(amax)) - 23) / C))


OFFSET_PATHS = {
    "certify": (dict(BASE, cube_size=0.5, **SUB), {}),
    "exact_everywhere": (dict(BASE, cube_size=0.5, **SUB), dict(exact_everywhere=True)),
    "scalar": (dict(BASE, cube_size=0.5, simd=False, **SUB), {}),
    "global": (dict(BASE, cube_size=0.5, subdomain_grid=False), {}),
    "tile_batch_1": (dict(BASE, cube_size=0.5, **SUB), dict(tile_batch=1)),
    "aniso": (dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16), dict(aniso=True)),
}
OFFSETS = [(path, b, sign) for path in OFFSET_PATHS for b in OFFSET_BANDS for sign in (1, -1)
           if path in ("certify", "exact_everywhere") or sign == 1]


def _offset_cloud(path, b, sign):
    p = (_aniso_cluster(300, 511) if path == "aniso" else _splash()).astype(np.float64)
    half = 0.5 * float((p.max(0) - p.min(0)).max())
    o = sign * (max(0.75 - half, 0.0) if b == -18 else band_offset(b))      # band -18: |coordinate| in [0.5, 1)
    q = (p - 0.5 * (p.min(0) + p.max(0)) + np.array([o, -o, o])).astype(np.float32)
    assert offset_band(float(np.abs(q).max())) == b
    return q


def check_offset(lib, oracle_mod, path, b, sign):
    import splashsurf_b200 as ssmod
    kw, opts = OFFSET_PATHS[path]
    p = _offset_cloud(path, b, sign)
    if b in REFUSED_BANDS:
        with pytest.raises(ssmod.SplashsurfError) as ei:
            _run(lib, p, kw, opts)
        assert ei.value.code == ssmod.SS_ERR_REAL_TOO_SMALL and "ulp" in str(ei.value)
        return
    check_device(lib, oracle_mod, p, kw, opts, tile=path != "global")


# ------------------------------------------------------------------ H100 ----
@pytest.mark.gpu
@pytest.mark.parametrize("name,k", SCALES)
def test_cuda_scale_power_of_two(ss, oracle_mod, name, k):
    check_scale(ss, oracle_mod, name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("k", list(range(-8, 10)))
def test_cuda_scale_power_of_ten(ss, oracle_mod, name, k):
    gen, kw, opts = CASES[name]
    s = 10.0 ** k
    check_device(ss, oracle_mod, (gen().astype(np.float64) * s).astype(np.float32), _scaled(kw, s), opts)


@pytest.mark.gpu
@pytest.mark.parametrize("path,band,sign", OFFSETS)
def test_cuda_offset(ss, oracle_mod, path, band, sign):
    check_offset(ss, oracle_mod, path, band, sign)


# ------------------------------------------------------------------ CPU executor ----
@pytest.mark.parametrize("name,k", SCALES)
def test_emulated_scale_power_of_two(emu, oracle_mod, name, k):
    check_scale(emu, oracle_mod, name, k)


@pytest.mark.parametrize("k", list(range(-8, 10)))
def test_emulated_scale_power_of_ten(emu, oracle_mod, k):
    gen, kw, opts = CASES["cube_R8"]
    s = 10.0 ** k
    check_device(emu, oracle_mod, (gen().astype(np.float64) * s).astype(np.float32), _scaled(kw, s), opts)


@pytest.mark.parametrize("path,band,sign", OFFSETS)
def test_emulated_offset(emu, oracle_mod, path, band, sign):
    check_offset(emu, oracle_mod, path, band, sign)


# ------------------------------------------------------------------ oracle vs reference binary ----
# the offset bands the device accepts: there the oracle judges it, so there the oracle is pinned to the reference's binary
WHEEL_BANDS = [b for b in OFFSET_BANDS if b not in REFUSED_BANDS]


@pytest.mark.parametrize("case", [("offset", b) for b in WHEEL_BANDS] + [("scale", k) for k in (-36, -22, 30, 36)])
def test_oracle_vs_reference_binary_at_scale_and_offset(oracle_mod, case):
    """The oracle judges the device here, so it is pinned against the reference's own binary at the same offsets and scales."""
    if not oracle_mod.reference_available():
        pytest.skip("oracle/_ref not unpacked")
    ps = oracle_mod.reference()
    kind, v = case
    kw = dict(BASE, cube_size=0.5, subdomain_num_cubes_per_dim=16)
    if kind == "offset":
        p = _offset_cloud("certify", v, 1)
    else:
        p, kw = (_splash() * np.float32(2.0 ** v)).astype(np.float32), _scaled(kw, 2.0 ** v)
    ref = ps.reconstruct_surface(p, multi_threading=False, **kw)
    o = oracle_mod.reconstruct(p, **kw)
    assert _same_bits(np.asarray(ref.particle_densities), o["particle_densities"])
    rv, rt = np.asarray(ref.mesh.vertices), np.asarray(ref.mesh.triangles)
    assert len(rv) == len(o["vertices"]) > 0
    rk = oracle_mod.resolve_keys(rv, o["grid"]["aabb_min"], o["grid"]["cell_size"], o["vertex_keys"], rt, o["triangles"], known_vertices=o["vertices"])
    m = oracle_mod.mesh_parity(rv, rt, rk, o["vertices"], o["triangles"], o["vertex_keys"], 16)
    assert m["keys_equal"] and m["triangles_equal"] and m.get("n_interior_not_bitexact", 0) == 0, m


# ------------------------------------------------------------------ coverage ----
SCALE_BANDS = {"g3_overflow", "normal", "g3_denormal", "g3_zero"}


def test_scale_and_offset_tables_are_covered():
    """Every scale band on the certifying default path (with k on both sides of each band edge), and every offset band on it,
    in both signs; the refused bands are the ones past 1/64."""
    ks = [k for n, k in SCALES if n == "cube_R8"]
    assert {scale_band(k) for k in ks} == SCALE_BANDS, sorted({scale_band(k) for k in ks})
    edges = [(-18, -17), (24, 25), (26, 27), (28, 29)]                 # h = 5e-7, 2.8e6, 1e7, 5e7
    for lo, hi in edges:
        assert lo in ks and hi in ks and 0.1 * 2.0 ** lo < [5e-7, 2.8e6, 1e7, 5e7][edges.index((lo, hi))] < 0.1 * 2.0 ** hi
    for path in ("certify",):
        got = {(b, s) for pth, b, s in OFFSETS if pth == path}
        assert got == {(b, s) for b in OFFSET_BANDS for s in (1, -1)}
    assert set(OFFSET_BANDS) >= {-18, -10, -7, -5, -3, -1}
    assert all(2.0 ** b > 1 / 64 for b in REFUSED_BANDS) and all(2.0 ** (b + 1) <= 1 / 64 for b in OFFSET_BANDS if b not in REFUSED_BANDS)
    # both sides of the limit: the last accepted band is pinned to the reference's binary, the first refused one is refused
    assert max(b for b in OFFSET_BANDS if b not in REFUSED_BANDS) + 2 == min(REFUSED_BANDS) and -7 in WHEEL_BANDS
