"""jss_beam_search (a caller's logit table decoded by beam search, the envs left untouched) on the real sm_90a library:
the tests of tests/beam_search_suite.py at GPU sizes and a full-size ta80 run.  Run on an H100 with `pytest -m gpu`."""
from tests import beam_search_suite
from tests.backends import collect

collect(globals(), beam_search_suite, "gpu")
