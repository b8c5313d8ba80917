"""Dirty-sector stores of the step kernels on the real sm_90a library: the tests of tests/dirty_store_suite.py at GPU
sizes.  Run on an H100 with `pytest -m gpu`."""
from tests import dirty_store_suite
from tests.backends import collect

collect(globals(), dirty_store_suite, "gpu")
