"""jss_step_logits (masked categorical draw from policy logits fused into the step) under HOST EMULATION of the CUDA
kernels (tests/emu): the tests of tests/step_logits_suite.py at CPU-friendly sizes."""
from tests import step_logits_suite
from tests.backends import collect

collect(globals(), step_logits_suite, "emu")
