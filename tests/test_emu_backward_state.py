"""The replayed gradients of sample_episodes, order_log_prob and sample_without_replacement across the calls a training
loop makes between forward and backward, under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/backward_state_suite.py at CPU-friendly sizes."""
from tests import backward_state_suite
from tests.backends import collect

collect(globals(), backward_state_suite, "emu")
