"""jss_beam_search (a caller's logit table decoded by beam search, the envs left untouched) under HOST EMULATION of the
CUDA kernels (tests/emu): the tests of tests/beam_search_suite.py at CPU-friendly sizes."""
from tests import beam_search_suite
from tests.backends import collect

collect(globals(), beam_search_suite, "emu")
