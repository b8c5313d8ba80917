"""jss_step_logits_record (a logits step recorded into the caller's rollout slot) and jss_refresh_obs under HOST
EMULATION of the CUDA kernels (tests/emu): the tests of tests/record_suite.py at CPU-friendly sizes."""
from tests import record_suite
from tests.backends import collect

collect(globals(), record_suite, "emu")
