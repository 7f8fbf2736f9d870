"""The density stage's neighbour walk on the device (the cases of tests/test_density_walk.py): densities equal the oracle's bit for
bit and equal density variants 1 and 2; neighbour counts and CSR lists equal the oracle's; the anisotropic mode's densities, x_bar
and G equal the standard run's and the oracle's."""
import pytest

from test_density_walk import CASES, check_anisotropic, check_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_density_walk_matches_oracle(ss, oracle_mod, name):
    check_case(ss, oracle_mod, name)


def test_cuda_density_walk_anisotropic(ss):
    check_anisotropic(ss)
