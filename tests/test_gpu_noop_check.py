"""The no-op check on designed states on the real sm_90a library: the tests of tests/noop_check_suite.py at GPU
sizes.  Run on an H100 with `pytest -m gpu`."""
from tests import noop_check_suite
from tests.backends import collect

collect(globals(), noop_check_suite, "gpu")
