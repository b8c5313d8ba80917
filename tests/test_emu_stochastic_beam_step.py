"""jss_stochastic_beam_step and ObsBeamSearch(stochastic=True) (stochastic beam search for a policy that reads the
observation at every decision) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/stochastic_beam_step_suite.py at CPU-friendly sizes."""
from tests import stochastic_beam_step_suite
from tests.backends import collect

collect(globals(), stochastic_beam_step_suite, "emu")
