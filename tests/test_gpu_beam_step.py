"""jss_beam_step and ObsBeamSearch (beam search for a policy that reads the observation at every decision) on the real
sm_90a library: the tests of tests/beam_step_suite.py at GPU sizes and a full-size ta80 run.  Run on an H100 with
`pytest -m gpu`."""
from tests import beam_step_suite
from tests.backends import collect

collect(globals(), beam_step_suite, "gpu")
