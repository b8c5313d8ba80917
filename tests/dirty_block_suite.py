"""The uniform-batch step kernels that take actions or a rule write back only the 32-byte sectors of an env's state block
that hold a job record word the step changed (plus the tail and the block's first sector).  That is right only if the
step marks every word it changes: a missed sector leaves a stale field in the block, which export_state() decodes.
Declared once for both backends (tests/backends.py) and collected by tests/test_emu_dirty_block.py and
tests/test_gpu_dirty_block.py.

The reference for the state is a twin stepped through a kernel that stores whole blocks: step_greedy at epsilon 0, on
scores one-hot at the same actions.  Both handles must agree on export_state(), real_obs, the mask and the scalar
records after every step.  The uniform batches' rows and their state against the oracle are checked by
tests/dirty_store_suite.py."""
import numpy as np

from tests.backends import native_test
from tests.dirty_store_suite import BATCHES, Fresh, _u32
from tests.parity_common import np_

UNIFORM = [b for b in BATCHES if b != "mixed"]   # one uniform batch per lane class


def _one_hot(env, acts):
    """Scores (N, J + 1) on env's device that make step_greedy at epsilon 0 take `acts` (int32 tensor; legal actions,
    or any action of a done env)."""
    import torch
    x = torch.zeros((env.num_envs, env.jobs + 1), dtype=torch.float32, device=env.device)
    return x.scatter_(1, acts.long().clamp(0, env.jobs).view(-1, 1), 1.0)


def _same_state(env, twin, ctx):
    """export_state(), real_obs, the mask and the scalar records of two handles, bit for bit."""
    a, b = env.export_state(), twin.export_state()
    assert set(a) == set(b), ctx
    for k in a:
        assert np.array_equal(np_(a[k]), np_(b[k])), (ctx, k)
    for x, y in ((env.real_obs, twin.real_obs), (env.action_mask, twin.action_mask), (env.reward, twin.reward),
                 (env.reward_raw, twin.reward_raw)):
        assert np.array_equal(_u32(x), _u32(y)), ctx


@native_test(emu=[(b, r) for b in UNIFORM for r in (True, False)], gpu=[(b, r) for b in UNIFORM for r in (True, False)])
def dirty_state_vs_whole_blocks(make_env, backend, batch, auto_reset):
    """step (SAMPLE = 0), step_sample with the masked-uniform sampler (1) and with a rule (2) on a uniform batch of
    every lane class against a twin stepped by step_greedy, which stores whole blocks, at the same random legal
    actions (the no-op when legal), until episodes end: the state agrees after every step."""
    import torch
    names = BATCHES[batch]
    f = Fresh(make_env, names, auto_reset=auto_reset, seed=29)
    env, twin = f.env, f.twin
    rng = np.random.default_rng(29)
    J = env.jobs
    ended = 0
    for step in range(J * int(env.machines) * 5 // 4):
        mask = np_(env.action_mask)[:, : J + 1]
        a = np.array([rng.choice(np.flatnonzero(m)) if m.any() else 0 for m in mask], np.int32)
        acts = torch.from_numpy(a).to(env.device)
        t0 = np_(env.current_time_step).copy()
        if step % 3 == 0:
            env.step(acts)
        else:
            env.step_sample(acts.clone(), "RANDOM" if step % 3 == 1 else "MWR")
        twin.step_greedy(_one_hot(twin, acts), 0.0)
        _same_state(env, twin, f"step {step}")
        t1 = np_(env.current_time_step)
        f.advanced += int((t1 > t0).sum())
        f.times += int((t1 == t0).sum())
        ended += int(np_(env.done).sum())
    assert f.advanced > 0 and f.times > 0 and ended > 0   # steps with and without a time advance; episodes ended


@native_test(emu=None, gpu=())
def dirty_state_ta80_full_size(make_env, backend):
    """ta80 at N = 65 536 from the stationary pre-roll of bench.py's headline: step_sample against a twin that imports
    the pre-rolled state and is stepped by step_greedy at the same actions, a few hundred steps."""
    import torch
    from bench import TA80_EPISODE, preroll
    f = Fresh(make_env, ["ta80"] * 65536, auto_reset=True, seed=1234)
    acts = preroll(f.env, "RANDOM", TA80_EPISODE, torch)
    f.twin.import_state(f.env.export_state())
    for step in range(300):
        a = acts.clone()
        *_, acts = f.env.step_sample(acts, "RANDOM")
        f.twin.step_greedy(_one_hot(f.twin, a), 0.0)
        x, y = f.env.export_state(), f.twin.export_state()
        assert all(torch.equal(x[k], y[k]) for k in x), step
        for u, v in ((f.env.real_obs, f.twin.real_obs), (f.env.reward, f.twin.reward)):
            assert torch.equal(u.view(torch.int32), v.view(torch.int32)), step
        assert torch.equal(f.env.action_mask, f.twin.action_mask), step
        assert torch.equal(f.env.reward_raw, f.twin.reward_raw), step
