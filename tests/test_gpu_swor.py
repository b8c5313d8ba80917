"""jss_sample_without_replacement and jss_order_log_prob (distinct episodes drawn by stochastic beam search, and given
orders scored under a logit table, with a gradient) on the real sm_90a library: the tests of tests/swor_suite.py at GPU
sizes and a full-size ta80 run.  Run on an H100 with `pytest -m gpu`."""
from tests import swor_suite
from tests.backends import collect

collect(globals(), swor_suite, "gpu")
