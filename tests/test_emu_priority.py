"""jss_rollout_priority (a caller's static priority rule run to the end of every episode in one launch) under HOST
EMULATION of the CUDA kernels (tests/emu): the tests of tests/priority_suite.py at CPU-friendly sizes."""
from tests import priority_suite
from tests.backends import collect

collect(globals(), priority_suite, "emu")
