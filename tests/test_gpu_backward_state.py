"""The replayed gradients of sample_episodes, order_log_prob and sample_without_replacement across the calls a training
loop makes between forward and backward, on the real sm_90a library: the tests of tests/backward_state_suite.py at GPU
sizes, and the producer x intervening-call matrix again on ta80 at N = 4 096.  Run on an H100 with `pytest -m gpu`."""
from tests import backward_state_suite
from tests.backends import collect

collect(globals(), backward_state_suite, "gpu")
