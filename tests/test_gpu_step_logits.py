"""jss_step_logits (masked categorical draw from policy logits fused into the step) on the real sm_90a library: the
tests of tests/step_logits_suite.py at GPU sizes.  Run on an H100 with `pytest -m gpu`."""
from tests import step_logits_suite
from tests.backends import collect

collect(globals(), step_logits_suite, "gpu")
