"""jss_step_logits_record (a logits step recorded into the caller's rollout slot) and jss_refresh_obs on the real
sm_90a library: the tests of tests/record_suite.py at GPU sizes.  Run on an H100 with `pytest -m gpu`."""
from tests import record_suite
from tests.backends import collect

collect(globals(), record_suite, "gpu")
