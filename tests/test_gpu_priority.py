"""jss_rollout_priority (a caller's static priority rule run to the end of every episode in one launch) on the real
sm_90a library: the tests of tests/priority_suite.py at GPU sizes, and a full-size ta80 run against the oracle.  Run on
an H100 with `pytest -m gpu`."""
from tests import priority_suite
from tests.backends import collect

collect(globals(), priority_suite, "gpu")
