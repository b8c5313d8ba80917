"""The policy-entropy forms of rollout_priority_sample, sample_episodes and order_log_prob on the real sm_90a library:
the tests of tests/entropy_suite.py at GPU sizes and a full-size ta80 run with both gradients.  Run on an H100 with
`pytest -m gpu`."""
from tests import entropy_suite
from tests.backends import collect

collect(globals(), entropy_suite, "gpu")
