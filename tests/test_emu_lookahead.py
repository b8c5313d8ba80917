"""jss_lookahead (every legal action valued by a dispatching-rule rollout to the end of the episode, the envs left
untouched) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of tests/lookahead_suite.py at CPU-friendly
sizes."""
from tests import lookahead_suite
from tests.backends import collect

collect(globals(), lookahead_suite, "emu")
