"""The policy-entropy forms of rollout_priority_sample, sample_episodes and order_log_prob under HOST EMULATION of the
CUDA kernels (tests/emu): the tests of tests/entropy_suite.py at CPU-friendly sizes, and the twin test again under
the other thread schedules of tests/test_emu_schedules.py."""
from tests import entropy_suite
from tests.backends import collect
from tests.test_emu_schedules import SCHEDULES

collect(globals(), entropy_suite, "emu")
for _tag, _schedule in SCHEDULES.items():
    collect(globals(), entropy_suite, "emu", only={"entropy_twin": ["mixed"]}, schedule=_schedule, suffix="_" + _tag)
