"""Several envs per process, side streams, the host pipeline next to stream-ordered calls and back-to-back launches on
the real sm_90a library: the tests of tests/sharing_suite.py.  Run on an H100 with `pytest -m gpu`."""
import pytest

from tests import sharing_suite
from tests.backends import collect

collect(globals(), sharing_suite, "gpu")


@pytest.mark.parametrize("order", list(sharing_suite.ORDERS))
def test_sharing_layouts_cross_48k(order):
    """The restatement of plan_smem_layouts behind test A: each order's layouts shrink from handle to handle and stay
    over 48 KB, and it gives the sizes the layout arithmetic gives by hand."""
    sharing_suite.check_layouts(order)
    sizes = {o: [sharing_suite.smem_layouts(b) for b in bs] for o, bs in sharing_suite.ORDERS.items()}
    assert sizes["uniform"][0]["step"] == 119248 and sizes["uniform"][1]["step"] == 83856
    assert sizes["uniform"][0]["env"] == 91728 and sizes["uniform"][1]["env"] == 54080
    assert sizes["rem"][0]["step_rem"] == 54976 and sizes["rem"][1]["step_rem"] == 49392   # ta80: just over 48 KB
