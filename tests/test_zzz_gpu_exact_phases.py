"""Phase timing of the exact level-set pass (Context.set_exact_phases): the instrumented k_exact_warp computes the same level set and
times every brick the 512-candidate tier takes, on the H100 (`ss`) and on the CPU executor of the CUDA sources (`emu`)."""
import numpy as np
import pytest

from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)

KW = dict(particle_radius=0.025, smoothing_length=2.0, cube_size=0.5)


def check_phases(lib):
    from splashsurf_b200 import synthetic as syn
    p = syn.splash((12, 12, 12), 2, 0.025, seed=3)
    ctx = lib.Context(0)
    try:
        plain = lib.reconstruct_surface(p, context=ctx, with_debug=True, **KW)
        ctx.set_exact_phases(True)
        timed = lib.reconstruct_surface(p, context=ctx, with_debug=True, **KW)
        ph = ctx.exact_phases()
        ctx.set_exact_phases(False)
    finally:
        ctx.close()
    assert np.array_equal(plain.mesh.vertices, timed.mesh.vertices) and np.array_equal(plain.mesh.triangles, timed.mesh.triangles)
    assert ph["bricks"] == int(timed.levelset_paths["exact_512"] + timed.levelset_paths["fixup_512"]) > 0
    assert set(ph) == set(lib.Context.EXACT_PHASES) | {"bricks"}
    assert ph["fold"] > 0


@pytest.mark.gpu
def test_cuda_exact_phases(ss):
    check_phases(ss)


def test_emulated_exact_phases(emu):
    check_phases(emu)
