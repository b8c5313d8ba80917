"""real_obs and the scaled reward against their exact values under HOST EMULATION of the CUDA kernels (tests/emu): the
tests of tests/exact_obs_suite.py at CPU-friendly sizes."""
from tests import exact_obs_suite
from tests.backends import collect

collect(globals(), exact_obs_suite, "emu")
