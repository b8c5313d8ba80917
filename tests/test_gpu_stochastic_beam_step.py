"""jss_stochastic_beam_step and ObsBeamSearch(stochastic=True) (stochastic beam search for a policy that reads the
observation at every decision) on the real sm_90a library: the tests of tests/stochastic_beam_step_suite.py at GPU
sizes and a full-size ta80 run.  Run on an H100 with `pytest -m gpu`."""
from tests import stochastic_beam_step_suite
from tests.backends import collect

collect(globals(), stochastic_beam_step_suite, "gpu")
