"""The uniform-batch step kernels write back only the 32-byte sectors of an env's observation row that the step
changed.  That is right only while real_obs holds, at every step's entry, the observation of the env's state block, and
only if the step marks every job whose row it changes.  Declared once for both backends (tests/backends.py) and collected by
tests/test_emu_dirty_store.py and tests/test_gpu_dirty_store.py.

The reference for real_obs is its full re-emission from the same state: a twin handle of the same batch imports the
env's exported state (jss_import_state writes the whole block and the whole row), and the env's real_obs and mask must
equal the twin's bit for bit after every step.  Uniform batches are also checked against the CPU oracle after every
step."""
import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import batch_cfg, check_random_batch, np_, synthetic_instance

BIG = synthetic_instance(160, 5, seed=11)            # 129..256 jobs: the 8-jobs-per-lane class
MID = synthetic_instance(64, 10, seed=12)            # 33..64 jobs: 2 jobs per lane
MIXED = ["ta01", "ta31", "ta80", "ta01", "ta80", "ta31", "ta45", "ta01", "ta62"]
# The uniform-batch kernels store only changed sectors when the rows are whole 16-byte chunks (J a multiple of 4): one
# batch per lane class (ta21: 20 jobs, ta80: 100), and a mixed batch, whose kernel stores whole rows.
BATCHES = {"ta21": ["ta21"] * 6, "mid": [MID] * 5, "ta80": ["ta80"] * 6, "big": [BIG] * 4, "mixed": MIXED + [BIG]}


def _u32(t):
    x = np_(t)
    return x.view(np.uint32) if x.dtype == np.float32 else x


class Fresh:
    """A twin of `env` that re-emits the observation of env's current state on demand."""

    def __init__(self, make_env, names, **kw):
        cfg = batch_cfg(names, sort=False)
        self.env = make_env(len(names), cfg, **kw)
        self.twin = make_env(len(names), cfg, **kw)
        self.env.reset()
        self.twin.reset()
        self.times = 0
        self.advanced = 0

    def check(self, ctx):
        t0 = np_(self.twin.current_time_step).copy()
        self.twin.import_state(self.env.export_state())
        assert np.array_equal(_u32(self.env.real_obs), _u32(self.twin.real_obs)), ctx
        assert np.array_equal(np_(self.env.action_mask), np_(self.twin.action_mask)), ctx
        t1 = np_(self.env.current_time_step)
        self.advanced += int((t1 > t0).sum())
        self.times += int((t1 == t0).sum())


def _drive(f, n_steps, act, ctx):
    for step in range(n_steps):
        act(step)
        f.check(f"{ctx} step {step}")
    assert f.advanced > 0 and f.times > 0, ctx        # steps with and without a time advance


@native_test(emu=[(b, r) for b in BATCHES for r in (True, False)], gpu=[(b, r) for b in BATCHES for r in (True, False)])
def dirty_random_actions(make_env, backend, batch, auto_reset):
    """Random legal actions, the no-op when legal, a forced no-op and illegal actions (the error bit),
    JSS_ACTION_SKIP and JSS_ACTION_ADVANCE, done with and without auto-reset, in a batch of every lane class."""
    names = BATCHES[batch]
    f = Fresh(make_env, names, auto_reset=auto_reset, seed=5)
    rng = np.random.default_rng(5)
    n = len(names)

    def act(step):
        mask = np_(f.env.action_mask).copy()
        a = np.array([rng.choice(np.flatnonzero(m)) if m.any() else 0 for m in mask], np.int32)
        kind = rng.integers(0, 12, n)
        a[kind == 0] = N.ACTION_SKIP
        a[kind == 1] = N.ACTION_ADVANCE
        a[kind == 2] = f.env.env_jobs[kind == 2]         # forced no-op: the error bit when the queue is empty
        a[kind == 3] = 10_000                             # out of range: the error bit
        f.env.step(a)

    _drive(f, 400, act, "random actions")


@native_test(emu=[(b, r) for b in BATCHES for r in ("RANDOM", "MWR")],
             gpu=[(b, r) for b in BATCHES for r in ("RANDOM", "MWR")])
def dirty_step_sample(make_env, backend, batch, rule):
    """step_sample with the masked-uniform sampler (SAMPLE = 1) and a dispatching rule (SAMPLE = 2)."""
    f = Fresh(make_env, BATCHES[batch], auto_reset=True, seed=9)
    acts = f.env.policy(rule).clone()

    def act(step):
        nonlocal acts
        *_, acts = f.env.step_sample(acts, rule)

    _drive(f, 300, act, f"step_sample {rule}")


@native_test(emu=[("ta80", "logits", 0.0), ("ta80", "greedy", 0.0), ("mixed", "greedy", 0.3)],
             gpu=[("ta80", "logits", 0.0), ("ta80", "greedy", 0.0), ("mixed", "greedy", 0.3)])
def dirty_row_steps(make_env, backend, batch, kind, epsilon):
    """step_logits and step_greedy (epsilon = 0 and > 0), then plain steps."""
    f = Fresh(make_env, BATCHES[batch], auto_reset=True, seed=13)
    rng = np.random.default_rng(13)
    ld = f.env.jobs + 1

    def act(step):
        x = lc._to_dev(f.env, lc.random_logits(rng, f.env, np_(f.env.action_mask), ld))
        if step % 3 == 2:
            f.env.step(f.env.policy("RANDOM"))
        elif kind == "logits":
            f.env.step_logits(x)
        else:
            f.env.step_greedy(x, epsilon)

    _drive(f, 300, act, f"{kind} {epsilon}")


@native_test(emu=["ta80", "mixed"], gpu=["ta80", "mixed"])
def dirty_after_recording(make_env, backend, batch):
    """Recording steps (the row whole into the slot, real_obs left stale) followed by plain steps, which first
    re-emit the stale real_obs."""
    f = Fresh(make_env, BATCHES[batch], auto_reset=True, seed=17)
    rng = np.random.default_rng(17)
    ld = f.env.jobs + 1
    traj = f.env.logits_trajectory(4)
    for rnd in range(30):
        for k in range(4):
            x = lc._to_dev(f.env, lc.random_logits(rng, f.env, np_(traj["action_mask"][k]), ld))
            f.env.step_logits_record(x, traj, k)
        acts = f.env.policy("RANDOM").clone()
        for step in range(3):
            *_, acts = f.env.step_sample(acts, "RANDOM")
            f.check(f"round {rnd} step {step}")
        traj = f.env.logits_trajectory(4, out=traj)


@native_test(emu=[["ta80"] * 4, ["ta21"] * 4], gpu=[["ta80"] * 16, ["ta21"] * 16])
def dirty_outputs_vs_oracle(make_env, backend, names):
    """Uniform batches stepped by the dirty path: observation, mask, rewards and every exported field equal the
    oracle's after every step, forced no-ops included."""
    check_random_batch(make_env, names, 500, seed=23, state_every=1, noop_force_every=9)


@native_test(emu=None, gpu=())
def dirty_ta80_full_size(make_env, backend):
    """ta80 at N = 65 536 from the stationary pre-roll of bench.py's headline, a few hundred steps."""
    import torch
    from bench import TA80_EPISODE, preroll
    f = Fresh(make_env, ["ta80"] * 65536, auto_reset=True, seed=1234)
    acts = preroll(f.env, "RANDOM", TA80_EPISODE, torch)
    for step in range(300):
        *_, acts = f.env.step_sample(acts, "RANDOM")
        t0 = f.twin.current_time_step.clone()
        f.twin.import_state(f.env.export_state())
        assert torch.equal(f.env.real_obs.view(torch.int32), f.twin.real_obs.view(torch.int32)), step
        assert torch.equal(f.env.action_mask, f.twin.action_mask), step
        assert bool((f.env.current_time_step > t0).any()) or step == 0
