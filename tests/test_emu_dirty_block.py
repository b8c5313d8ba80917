"""Dirty-sector stores of the state block under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/dirty_block_suite.py at CPU-friendly sizes, in the default schedule and again with the threads of a block run in
shuffled order and shared memory poisoned, so that a read of the staged block before every lane has written it fails."""
from tests import dirty_block_suite
from tests.backends import collect
from tests.emu.emu_backend import SHUFFLED

collect(globals(), dirty_block_suite, "emu")
collect(globals(), dirty_block_suite, "emu", schedule=(SHUFFLED, 1, 0xA5), suffix="_shuffle1_a5")
