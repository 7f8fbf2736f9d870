"""CPU tests of the invariant behind the level-set certification pass (DESIGN.md 4.3): the cubic g(s) used by
`ss_certify_box` never exceeds the kernel shape, and partial sums built from it never exceed the reference's exact value."""
import math
import os
import re

import numpy as np

from conftest import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _coeffs():
    src = open(os.path.join(ROOT, "splashsurf_b200", "csrc", "ss_kernels.cuh")).read()
    return [float(re.search(rf"#define SS_G{k} (-?[0-9.]+)f", src).group(1)) for k in range(4)]


def _f(q):
    q = np.asarray(q, dtype=np.float64)
    return np.where(q <= 0.5, 1 - 6 * q ** 2 + 6 * q ** 3, np.where(q < 1, 2 * (1 - q) ** 3, 0.0))


def test_cubic_is_a_lower_bound_of_the_kernel_shape():
    g0, g1, g2, g3 = _coeffs()
    s = np.concatenate([np.linspace(0, 1.0, 2_000_001), np.linspace(1.0, 9.0, 200_001)])
    g = np.maximum(0.0, g0 + s * (g1 + s * (g2 + s * g3)))
    assert (g <= _f(np.sqrt(s)) + 1e-12).all()
    # float32 evaluation (as on the device, Horner with FMAs) stays below as well: the -1e-5 offset in G0 covers rounding
    s32 = s.astype(np.float32)
    g32 = np.maximum(np.float32(0), np.float32(g0) + s32 * (np.float32(g1) + s32 * (np.float32(g2) + s32 * np.float32(g3))))
    assert (g32.astype(np.float64) <= _f(np.sqrt(s32.astype(np.float64))) + 2e-6).all()
    q = np.linspace(0, 1.2, 240001)
    cap = 32 * np.sum(np.maximum(0.0, g0 + q * q * (g1 + q * q * (g2 + q * q * g3))) * q * q) * (q[1] - q[0])
    assert 0.93 < cap < 1.0          # captures ~94 % of the kernel's volume integral


def _device_coefficients(h):
    """k_certify_warp's operands as the host computes them (ss_pipeline.cu): coordinates scaled by cs = 2^-e with h cs in [1, 2),
    coefficients G_k / (h cs)^(2k) in double, rounded to f32."""
    g0, g1, g2, g3 = _coeffs()
    h = float(np.float32(h))
    e = math.frexp(h)[1] - 1                                     # ilogb
    hs = math.ldexp(h, -e)
    ih2 = 1.0 / (hs * hs)
    return np.float32(math.ldexp(1.0, -e)), np.float32(g0), np.float32(g1 * ih2), np.float32(g2 * ih2 ** 2), np.float32(g3 * ih2 ** 3)


def test_scaled_bound_is_below_the_kernel_shape_at_every_length_scale():
    """At every power-of-two h of the reference's f32 window, and at h with mantissas across [1, 2): the f32 Horner bound on
    scaled squared distances, with the host's coefficients, never exceeds the kernel shape.  Absolute-unit coefficients failed this
    from h ~ 1e7 (G3 / h^6 denormal, then zero) and certified nothing below h ~ 5e-7 (overflow)."""
    s = np.concatenate([np.linspace(0, 1.0, 200_001), np.linspace(1.0, 9.0, 20_001)])
    hs = [0.1 * 2.0 ** k for k in range(-40, 41)] + [2.0 ** k for k in range(-40, 41)] + list(np.linspace(1.0, 1.999, 37))
    for h in hs:
        cs, g0, g1, g2, g3 = _device_coefficients(h)
        assert all(np.isfinite(x) and (x == 0 or abs(x) >= np.finfo(np.float32).tiny) for x in (g1, g2, g3)), h
        h32 = np.float64(np.float32(h))
        d2 = (s * (h32 * float(cs)) ** 2).astype(np.float32)       # scaled squared distances, as the kernel forms them
        g = np.maximum(np.float32(0), g0 + d2 * (g1 + d2 * (g2 + d2 * g3)))
        q = np.sqrt(d2.astype(np.float64)) / (h32 * float(cs))
        assert (g.astype(np.float64) <= _f(q) + 2e-6).all(), h


def test_partial_sums_never_exceed_the_exact_level_set(oracle_mod):
    """On the reference's grid-loop fixture: for random grid points, the bound summed over ALL particles within 0.8 h (the
    largest set a warp can use) is <= the exact tile value (AVX and scalar arithmetic) times (1 + 1e-4)."""
    g = load_golden("grid_loop_subdomain_33")
    g0, g1, g2, g3 = _coeffs()
    h, c, m = float(g["h"]), float(g["cell_size"]), float(g["rest_mass"])
    common = dict(global_min=g["global_min"], cube_size=g["cell_size"], subdomain_ijk=g["subdomain_ijk"], subdomain_cubes=64,
                  subdomain_min=g["subdomain_min"], h=g["h"], rest_mass=g["rest_mass"])
    p, rho = g["particles"].astype(np.float64), g["densities"].astype(np.float64)
    vol = m / rho
    sigma = 8.0 / (np.pi * h ** 3)
    rng = np.random.default_rng(3)
    pts = rng.integers(0, 65, size=(400, 3))
    for mode in (0, 1):
        tile = oracle_mod.levelset_tile(g["particles"], g["densities"], mode=mode, **common).astype(np.float64)
        for i, j, k in pts:
            x = g["subdomain_min"].astype(np.float64) + np.array([i, j, k]) * c
            s = ((p - x[None]) ** 2).sum(1) / h ** 2
            sel = s < 0.64
            lb = sigma * np.sum(vol[sel] * np.maximum(0.0, g0 + s[sel] * (g1 + s[sel] * (g2 + s[sel] * g3))))
            assert lb <= tile[i, j, k] * (1 + 1e-4) + 1e-12, (mode, i, j, k, lb, tile[i, j, k])
