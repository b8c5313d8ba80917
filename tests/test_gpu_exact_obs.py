"""real_obs and the scaled reward against their exact values on the real sm_90a library: the tests of
tests/exact_obs_suite.py at GPU sizes, with the full divide sweeps.  Run on an H100 with `pytest -m gpu`."""
from tests import exact_obs_suite
from tests.backends import collect

collect(globals(), exact_obs_suite, "gpu")
