"""jss_rollout_priority_sample (whole episodes drawn from a caller's logit table in one launch, with each episode's
log-probability and its gradient) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/priority_sample_suite.py at CPU-friendly sizes."""
from tests import priority_sample_suite
from tests.backends import collect

collect(globals(), priority_sample_suite, "emu")
