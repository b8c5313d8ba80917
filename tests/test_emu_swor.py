"""jss_sample_without_replacement and jss_order_log_prob (distinct episodes drawn by stochastic beam search, and given
orders scored under a logit table, with a gradient) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/swor_suite.py at CPU-friendly sizes."""
from tests import swor_suite
from tests.backends import collect

collect(globals(), swor_suite, "emu")
