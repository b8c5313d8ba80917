"""Dirty-sector stores of the state block on the real sm_90a library: the tests of tests/dirty_block_suite.py at GPU
sizes.  Run on an H100 with `pytest -m gpu`."""
from tests import dirty_block_suite
from tests.backends import collect

collect(globals(), dirty_block_suite, "gpu")
