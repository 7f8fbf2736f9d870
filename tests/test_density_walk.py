"""The density stage's neighbour walk (ss_kernels.cuh: k_cell_offsets, ss_walk_run, k_density) on the CPU executor of the CUDA
sources: densities equal the oracle's bit for bit and equal the cell-cooperative kernels' (density variants 1 and 2); neighbour
counts and CSR neighbour lists equal the oracle's, in order.  The clouds put particles where the walk's corner cases are:
hit lists of K - 1, K, K + 1 and 2K entries and more than 96 (K = SS_DENSITY_K, the slots of k_density's shared-memory list),
z-columns with empty cells at the start, in the middle and at the end, columns clipped at both faces of a subdomain's
neighbourhood-search grid, a particle alone in its subdomain, sparse subdomains, S = 16, 24 and 64, a particle AABB, the
global path and the anisotropic mode.  The GPU-marked counterpart is tests/test_zzz_gpu_density_walk.py."""
import os
import re

import numpy as np
import pytest

from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

R = 0.025
H = 4 * R                      # compact support radius at smoothing_length 2
KW = dict(particle_radius=R, smoothing_length=2.0, cube_size=0.5, subdomain_grid_auto_disable=False)


def list_slots() -> int:
    """K: the d^2 slots per thread of k_density's hit list."""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "splashsurf_b200", "csrc", "ss_kernels.cuh")).read()
    return int(re.search(r"#define SS_DENSITY_K (\d+)", src).group(1))


def _clumps(seed):
    """Clumps of K, K + 1, K + 2, 2K + 1 and 110 particles inside balls of diameter 0.4 h, 5 h apart: every particle of a clump of
    N has exactly the N - 1 others as neighbours."""
    k = list_slots()
    rng = np.random.default_rng(seed)
    parts = []
    for i, n in enumerate((k, k + 1, k + 2, 2 * k + 1, 110)):
        v = rng.normal(size=(n, 3))
        ball = v / np.linalg.norm(v, axis=1, keepdims=True) * (0.2 * H * rng.uniform(0, 1, (n, 1)) ** (1 / 3))
        parts.append(ball + np.array([0.13 + 5 * H * i, 0.27, 0.41]))
    return np.concatenate(parts).astype(np.float32)


def _holey_cube(n, seed):
    """A jittered cube with h-cells punched out: the neighbourhood-search cells are aligned to multiples of h, so removing the
    particles of [i h, (i + 1) h)^3 empties one cell.  A whole z-layer of cells goes too, and random cells elsewhere, so that
    columns have empty cells at their start, middle and end."""
    from splashsurf_b200 import synthetic as syn
    p = syn.jittered_cube(n, R, seed).astype(np.float64)
    rng = np.random.default_rng(seed)
    cell = np.floor(p / H).astype(np.int64)
    hi = cell.max(axis=0)
    drop = cell[:, 2] == 2
    for _ in range(max(4, int(np.prod(hi + 1)) // 5)):
        drop |= np.all(cell == rng.integers(0, hi + 1), axis=1)
    return np.ascontiguousarray(p[~drop].astype(np.float32))


def _cube_clumps_and_loner(seed):
    """Holey cube + clumps + one particle alone in its subdomain."""
    return np.concatenate([_holey_cube(9, seed), _clumps(seed) + np.float32(0.6), np.array([[3.0, -2.0, 1.0]], np.float32)])


def _droplets(seed):
    from splashsurf_b200 import synthetic as syn
    return np.concatenate([syn.splash((9, 6, 9), 6, R, seed), _clumps(seed) + np.float32(1.5)])


# name -> (cloud, reconstruction keywords)
CASES = {
    "clumps_S64": (lambda: _clumps(1), dict(KW, subdomain_num_cubes_per_dim=64)),
    "clumps_S16": (lambda: _clumps(2), dict(KW, subdomain_num_cubes_per_dim=16)),
    "holey_cube_S16": (lambda: _holey_cube(10, 3), dict(KW, subdomain_num_cubes_per_dim=16)),
    "holey_cube_S24": (lambda: _holey_cube(10, 4), dict(KW, subdomain_num_cubes_per_dim=24)),
    "mixed_S24": (lambda: _cube_clumps_and_loner(5), dict(KW, subdomain_num_cubes_per_dim=24)),
    "mixed_S64": (lambda: _cube_clumps_and_loner(6), dict(KW, subdomain_num_cubes_per_dim=64)),
    "sparse_droplets_S16": (lambda: _droplets(7), dict(KW, cube_size=0.75, subdomain_num_cubes_per_dim=16)),
    "particle_aabb_S16": (lambda: _cube_clumps_and_loner(8), dict(KW, subdomain_num_cubes_per_dim=16, aabb_min=[0.05, 0.0, -1.0], aabb_max=[1.0, 0.32, 1.0])),
    "global_path": (lambda: _cube_clumps_and_loner(9), dict(KW, subdomain_grid=False)),
}


def check_case(ss, oracle_mod, name):
    p, kw = CASES[name][0](), CASES[name][1]
    o = oracle_mod.reconstruct(p, want_neighbor_counts=True, **kw)
    assert o["rc"] == 0
    rho = {}
    ctx = ss.Context()
    try:
        for dv in (0, 1, 2):
            ctx.set_density_variant(dv)
            rho[dv] = ss.reconstruct_surface(p, context=ctx, **kw).particle_densities
        ctx.set_density_variant(0)
        nb = None if "aabb_min" in kw else ss.reconstruct_surface(p, context=ctx, global_neighborhood_list=True, **kw).particle_neighbors
    finally:
        ctx.close()
    assert np.array_equal(rho[0], o["particle_densities"])
    assert np.array_equal(rho[1], rho[0]) and np.array_equal(rho[2], rho[0])
    if nb is not None:
        on = oracle_mod.reconstruct(p, want_neighbors=True, **kw)["neighbors"]
        off = nb.offsets.astype(np.int64)
        assert np.array_equal(np.diff(off), o["neighbor_counts"])
        assert np.array_equal(off, on[0]) and np.array_equal(nb.indices.astype(np.int64), on[1])
    return o


def _assert_list_lengths(o):
    """The clumps give hit lists of K - 1, K, K + 1, 2K and more than 96 entries."""
    k = list_slots()
    counts = set(o["neighbor_counts"].tolist())
    assert {k - 1, k, k + 1, 2 * k} <= counts and max(counts) > 96, sorted(counts)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_density_walk_matches_oracle(emu, oracle_mod, name):  # noqa: F811
    o = check_case(emu, oracle_mod, name)
    if "clumps" in name or "mixed" in name:
        _assert_list_lengths(o)


def check_anisotropic(ss):
    """Anisotropic mode on the clumps and the holey cube: densities, x_bar and G equal the standard run's densities and the
    anisotropic oracle's restatement, bit for bit."""
    from test_anisotropic import oracle_reconstruct_anisotropic
    p = _cube_clumps_and_loner(10)
    kw = dict(KW, subdomain_num_cubes_per_dim=16)
    ctx = ss.Context()
    try:
        a = ss.reconstruct_surface(p, context=ctx, anisotropy=ss.Anisotropy(), **kw)
        std = ss.reconstruct_surface(p, context=ctx, **kw)
    finally:
        ctx.close()
    an = ss.Anisotropy()
    o = oracle_reconstruct_anisotropic(p, smoothing=an.smoothing, max_stretch=an.max_stretch, min_neighbors=an.min_neighbors, **kw)
    assert o["rc"] == 0
    assert np.array_equal(a.particle_densities, std.particle_densities)
    assert np.array_equal(a.particle_densities, o["particle_densities"])
    assert np.array_equal(a.smoothed_particles, o["smoothed_particles"])
    assert np.array_equal(a.anisotropy_matrices.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]], o["anisotropy"])


def test_emulated_density_walk_anisotropic(emu):  # noqa: F811
    check_anisotropic(emu)
