"""Numeric edges of the draws from a caller's fp32 logits on the real sm_90a library: the tests of
tests/sampling_edges_suite.py at GPU sizes, and the uniformity of tied draws at N = 65 536.  Run on an H100 with
`pytest -m gpu`."""
from tests import sampling_edges_suite
from tests.backends import collect

collect(globals(), sampling_edges_suite, "gpu")
