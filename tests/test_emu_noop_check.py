"""The no-op check on designed states under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/noop_check_suite.py at CPU-friendly sizes."""
from tests import noop_check_suite
from tests.backends import collect

collect(globals(), noop_check_suite, "emu")
