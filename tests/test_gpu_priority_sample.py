"""jss_rollout_priority_sample (whole episodes drawn from a caller's logit table in one launch, with each episode's
log-probability and its gradient) on the real sm_90a library: the tests of tests/priority_sample_suite.py at GPU
sizes, the distribution of the draws and of the gradient, and a full-size ta80 run against one-env twins and the
oracle.  Run on an H100 with `pytest -m gpu`."""
from tests import priority_sample_suite
from tests.backends import collect

collect(globals(), priority_sample_suite, "gpu")
