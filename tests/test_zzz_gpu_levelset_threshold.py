"""The level-set certification at thresholds inside the fluid on the H100: the cases of tests/test_levelset_threshold.py, with every
marker of the raw tile (ss_context_keep_levelset_tile_raw) checked against its exact oracle value and every evaluated point against
the oracle bit for bit, and the meshes of level-set variants 2, 1, 0 and exact evaluation everywhere against the oracle.  This is
the run that counts for the certification sweep: the CPU executor cannot reproduce the device's slice sizes, mbarrier phases or
register allocation."""
import pytest

from test_levelset_threshold import CASES, check_case


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cuda_levelset_threshold(ss, oracle_mod, name):
    check_case(ss, oracle_mod, name)
