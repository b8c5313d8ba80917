"""Dirty-sector stores of the step kernels under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/dirty_store_suite.py at CPU-friendly sizes."""
from tests import dirty_store_suite
from tests.backends import collect

collect(globals(), dirty_store_suite, "emu")
