"""The parity tests of tests/parity_suite.py on the real sm_90a library (jssenv_b200/libjss_b200.so, called through
the C-ABI).  Run on an H100 with `pytest -m gpu`."""
from tests import parity_suite
from tests.backends import collect

collect(globals(), parity_suite, "gpu")
