"""jss_lookahead_priority (every legal action valued by a greedy rollout of a caller's priority table to the end of the
episode, the envs left untouched) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/lookahead_priority_suite.py at CPU-friendly sizes."""
from tests import lookahead_priority_suite
from tests.backends import collect

collect(globals(), lookahead_priority_suite, "emu")
