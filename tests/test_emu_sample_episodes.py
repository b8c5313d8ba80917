"""jss_sample_episodes (k episodes per env drawn from a caller's logit table, the envs left untouched, with a replayed
gradient and the best sample's schedule) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of
tests/sample_episodes_suite.py at CPU-friendly sizes."""
from tests import sample_episodes_suite
from tests.backends import collect

collect(globals(), sample_episodes_suite, "emu")
