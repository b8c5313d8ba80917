"""jss_lookahead_sample (every legal action valued by k episodes drawn from a caller's logit table after it, the envs
left untouched) on the sm_90a library: the tests of tests/lookahead_sample_suite.py at GPU sizes (`-m gpu`)."""
from tests import lookahead_sample_suite
from tests.backends import collect

collect(globals(), lookahead_sample_suite, "gpu")
