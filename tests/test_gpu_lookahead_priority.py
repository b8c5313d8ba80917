"""jss_lookahead_priority (every legal action valued by a greedy rollout of a caller's priority table to the end of the
episode, the envs left untouched) on the real sm_90a library: the tests of tests/lookahead_priority_suite.py at GPU
sizes, and a full-size ta80 run against the oracle.  Run on an H100 with `pytest -m gpu`."""
from tests import lookahead_priority_suite
from tests.backends import collect

collect(globals(), lookahead_priority_suite, "gpu")
