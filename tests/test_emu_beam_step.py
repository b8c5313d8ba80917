"""jss_beam_step and ObsBeamSearch (beam search for a policy that reads the observation at every decision) under HOST
EMULATION of the CUDA kernels (tests/emu): the tests of tests/beam_step_suite.py at CPU-friendly sizes."""
from tests import beam_step_suite
from tests.backends import collect

collect(globals(), beam_step_suite, "emu")
