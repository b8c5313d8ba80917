"""jss_lookahead_sample (every legal action valued by k episodes drawn from a caller's logit table after it, the envs
left untouched) under HOST EMULATION of the CUDA kernels (tests/emu): the tests of tests/lookahead_sample_suite.py at
CPU-friendly sizes, and the twin test again under the other thread schedules of tests/test_emu_schedules.py."""
from tests import lookahead_sample_suite
from tests.backends import collect
from tests.test_emu_schedules import SCHEDULES

collect(globals(), lookahead_sample_suite, "emu")
for _tag, _schedule in SCHEDULES.items():
    collect(globals(), lookahead_sample_suite, "emu", only={"lookahead_sample_twin": [("NJM", 1)]},
            schedule=_schedule, suffix="_" + _tag)
