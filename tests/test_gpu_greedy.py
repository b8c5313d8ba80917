"""jss_step_greedy and jss_step_greedy_record (greedy / epsilon-greedy decoding of action scores fused into the step)
on the real sm_90a library: the tests of tests/greedy_suite.py at GPU sizes, and the exploration distribution and a
full-size greedy evaluation.  Run on an H100 with `pytest -m gpu`."""
from tests import greedy_suite
from tests.backends import collect

collect(globals(), greedy_suite, "gpu")
