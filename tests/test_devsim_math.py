"""The numerics batteries of tests/test_hostsim_math.py, run on the sm_90a build of t2d_math.cuh (tests/devsim) on the GPU.

The tests are the very same functions; only the ``sim`` fixture they take differs: here it is the device twin, whose entry
points copy their inputs to the GPU, run the header's arithmetic there and copy the results back."""

import pytest

from tests.test_hostsim_math import *  # noqa: F401,F403  (the tests to run, and the devsim fixture)
from tests.test_hostsim_math import test_devsim_builds_and_exports_the_hostsim_entry_points

pytestmark = pytest.mark.gpu

del test_devsim_builds_and_exports_the_hostsim_entry_points   # a build check without a GPU: it runs with the host tests


@pytest.fixture(scope="module")
def sim(devsim):
    return devsim
