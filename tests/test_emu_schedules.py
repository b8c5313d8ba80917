"""The kernels under HOST EMULATION (tests/emu) with other legal schedules: threads and blocks run in descending or
shuffled order, and every block's shared memory and every device allocation start as a poison byte.

The emulator's default runs the threads of a block, and the blocks of a launch, in ascending order, and zero-fills
shared memory.  A shared-memory hand-off that lacks its __syncwarp / __syncthreads, or a read of memory nothing wrote,
then still sees what it expects.  Here a chosen set of the native tests, at least one per kernel family that passes
data between threads through shared memory, runs again under three other schedules, each held to its own reference
(the C oracle, the float64 host restatements, float64 autograd) as in its home suite.  A self-test first shows that
each schedule does expose such hazards."""
import ctypes

import numpy as np
import pytest

from tests import (beam_search_suite, beam_step_suite, dirty_store_suite, exact_obs_suite, greedy_suite,
                   improve_orders_suite, lookahead_priority_suite, lookahead_suite, parity_suite, priority_sample_suite,
                   record_suite, sample_episodes_suite, step_logits_suite, stochastic_beam_step_suite, swor_suite)
from jssenv_b200 import _native
from tests.backends import collect, native_test
from tests.emu.emu_backend import ASCENDING, DESCENDING, SHUFFLED, use_emulation

SCHEDULES = {
    "descending_ff": (DESCENDING, 0, 0xFF),     # NaN floats, -1 integers
    "shuffle1_a5": (SHUFFLED, 1, 0xA5),
    "shuffle2_00": (SHUFFLED, 2, 0x00),
}

# declaration -> the parameter sets to run (None: its own emu cases)
CHOSEN = {
    improve_orders_suite: {"improve_orders_restatement": [("beam", 0)], "improve_orders_edge_cases": None,
                           "improve_orders_batch_invariance": None},
    beam_search_suite: {"beam_search_host_restatement": None, "beam_search_exhaustive": None},
    swor_suite: {"swor_host_restatement": None, "swor_exhaustive": None, "swor_gradient": None},
    beam_step_suite: {"beam_step_parity": [("NJM", True)], "beam_step_round_twins": None},
    stochastic_beam_step_suite: {"stochastic_beam_step_parity": [("NJM", True)],
                                 "stochastic_beam_step_round_twins": None},
    sample_episodes_suite: {"sample_episodes_twin": [("NJM", True)], "sample_episodes_gradient": None,
                            "sample_episodes_split_invariance": None},
    priority_sample_suite: {"priority_sample_autograd": None},
    lookahead_suite: {"lookahead_twin_mixed_batch": None, "lookahead_split_invariance": None},
    lookahead_priority_suite: {"lookahead_priority_twin": [("NJM", True)]},
    dirty_store_suite: {"dirty_random_actions": None, "dirty_step_sample": None, "dirty_row_steps": None,
                        "dirty_after_recording": None, "dirty_outputs_vs_oracle": None},
    step_logits_suite: {"step_logits_mixed_batch": None},
    greedy_suite: {"greedy_mixed_batch": [0.3]},
    record_suite: {"record_mixed_batch": None},
    exact_obs_suite: {"serial_episode": ["mixed_ta01"]},
    parity_suite: {"random_mixed_batch": None},
}

for _tag, _schedule in SCHEDULES.items():
    for _suite, _only in CHOSEN.items():
        collect(globals(), _suite, "emu", only=_only, schedule=_schedule, suffix="_" + _tag)


# ---- the schedules bite: a kernel with deliberate hazards (tests/emu/emu_selftest.cpp) ---------------------------
BLOCKS, WARPS, PAIRS = 6, 8, 16


def run_selftest(lib):
    """Per block: whether each of the 128 lane-pair reads and 4 warp-pair reads saw its write, and the word a block
    read before writing it; and the first word of a fresh device allocation."""
    lib.jss_emu_selftest.restype = ctypes.c_int
    lib.jss_emu_selftest.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    out = np.zeros((BLOCKS, lib.jss_emu_selftest_width()), np.int32)
    fresh = ctypes.c_int(0)
    assert lib.jss_emu_selftest(BLOCKS, out.ctypes.data, ctypes.byref(fresh)) == 0
    lanes, warps = out[:, :WARPS * PAIRS], out[:, WARPS * PAIRS:WARPS * PAIRS + WARPS // 2]
    assert np.isin(lanes, (0, 1)).all() and np.isin(warps, (0, 1)).all()
    return lanes, warps, out[:, -1].view(np.uint32), np.uint32(fresh.value & 0xFFFFFFFF)


def test_emu_selftest_default_schedule_hides_the_hazards():
    with use_emulation() as be:
        lanes, warps, unwritten, _ = run_selftest(be.library())
    assert lanes.all() and warps.all()          # every write runs before its read
    assert unwritten[0] == 0                    # shared memory starts zeroed, once per launch


@pytest.mark.parametrize("tag", list(SCHEDULES))
def test_emu_selftest_schedule_exposes_the_hazards(tag):
    order, _, poison = SCHEDULES[tag]
    with use_emulation(SCHEDULES[tag]) as be:
        lanes, warps, unwritten, fresh = run_selftest(be.library())
    if order == DESCENDING:                     # every read runs before its write
        assert not lanes.any() and not warps.any()
    else:                                       # a fresh draw per scheduling pass: some reads run first, some do not
        assert 0 < lanes.sum() < lanes.size and 0 < warps.sum() < warps.size
    pattern = np.uint32(poison * 0x01010101)
    assert (unwritten == pattern).all()         # in every block, not once per launch
    assert fresh == pattern


def test_emu_selftest_schedule_is_restored():
    with use_emulation(SCHEDULES["descending_ff"]):
        pass
    with use_emulation() as be:
        lanes, warps, unwritten, _ = run_selftest(be.library())
        assert lanes.all() and warps.all() and unwritten[0] == 0
        with pytest.raises(ValueError):
            use_emulation._set((ASCENDING, 0, 256))


@native_test(gpu=None)
def selftest_bound(make_env, backend):
    """The schedule reaches the tests `collect` binds: the hazard kernel misses writes and reads the poison there."""
    lanes, _, unwritten, _ = run_selftest(_native.backend.library())
    assert not lanes.all() and not (unwritten == 0x7E57).any()


for _tag, _schedule in SCHEDULES.items():
    collect(globals(), {"selftest_bound": selftest_bound}, "emu", schedule=_schedule, suffix="_" + _tag)
