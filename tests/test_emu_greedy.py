"""jss_step_greedy and jss_step_greedy_record (greedy / epsilon-greedy decoding of action scores fused into the step)
under HOST EMULATION of the CUDA kernels (tests/emu): the tests of tests/greedy_suite.py at CPU-friendly sizes."""
from tests import greedy_suite
from tests.backends import collect

collect(globals(), greedy_suite, "emu")
