"""jss_sample_episodes (k episodes per env drawn from a caller's logit table, the envs left untouched, with a replayed
gradient and the best sample's schedule) on the real sm_90a library: the tests of tests/sample_episodes_suite.py at GPU
sizes, a full-size ta80 run, the score-function identity and a chi-square test of the draws.  Run on an H100 with
`pytest -m gpu`."""
from tests import sample_episodes_suite
from tests.backends import collect

collect(globals(), sample_episodes_suite, "gpu")
