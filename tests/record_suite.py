"""The tests of jss_step_logits_record (a logits step that records its transition into the caller's rollout slot) and
jss_refresh_obs, declared once for both backends (tests/backends.py) and collected by tests/test_emu_record.py and
tests/test_gpu_record.py.  The reference is a twin env stepped with jss_step_logits on the same logits: the slots, the
env's own outputs, its state and its statistics must equal the twin's bit for bit."""
import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import assert_twins_equal, batch_cfg, np_, synthetic_instance, twin_envs

MASK_SENTINEL = 0xAB


class _Recorded:
    """The recording env as assert_twins_equal sees it: its own outputs, state and statistics, with the observation
    taken from the trajectory slot (its real_obs is stale by design)."""

    def __init__(self, env, real_obs):
        self._env, self.real_obs = env, real_obs

    def __getattr__(self, name):
        return getattr(self._env, name)


def _state(env):
    return {k: np_(v).copy() for k, v in env.export_state().items()}


def _unchanged(before, after):
    """Envs whose exported state (the flags aside: the error bit is not a change) the step left as it was."""
    same = np.ones(len(before["t"]), bool)
    for k in before:
        if k != "flags":
            same &= (before[k] == after[k]).reshape(len(same), -1).all(1)
    return same


def check_slot(a_env, b_env, traj, k, info_b, unchanged, ctx):
    """Transition k of `traj` against the twin b_env that took the same step with step_logits: the draw, the next
    observation and mask, and the scalar record (reward 0 for the envs the step left unchanged)."""
    u32 = np.uint32
    assert np.array_equal(np_(traj["actions"][k]), np_(info_b["actions"])), ctx
    assert np.array_equal(np_(traj["log_prob"][k]).view(u32), np_(info_b["log_prob"]).view(u32)), ctx
    assert np.array_equal(np_(traj["real_obs"][k + 1]).view(u32), np_(b_env.real_obs).view(u32)), ctx
    assert np.array_equal(np_(traj["action_mask"][k + 1]), np_(b_env.action_mask)), ctx
    rew, raw = np_(b_env.reward).copy(), np_(b_env.reward_raw).copy()
    rew[unchanged], raw[unchanged] = 0.0, 0
    assert np.array_equal(np_(traj["reward"][k]).view(u32), rew.view(u32)), ctx
    assert np.array_equal(np_(traj["reward_raw"][k]), raw), ctx
    assert np.array_equal(np_(traj["time"][k]), np_(b_env.current_time_step)), ctx
    assert np.array_equal(np_(traj["done"][k]), np_(b_env.done)), ctx
    assert np.array_equal(np_(traj["_scalars"][k][:, 3]), np_(b_env._flags_done)), ctx
    assert_twins_equal(_Recorded(a_env, traj["real_obs"][k + 1]), b_env, ctx)


def check_record(make_env, names, n_steps, seed, traj_len=16, pad=3, auto_reset=True, state_every=25, oracle=True):
    """Env A records every transition into trajectories of `traj_len` steps (one dict, reused), twin B steps with
    step_logits on the same seeded logits; after every step the slot and A's outputs equal B's, and every
    `state_every` steps the exported state and the statistics too.  A's draws are also checked against the float64
    oracle of the draw (as for step_logits)."""
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=seed, auto_reset=auto_reset)
    rng = np.random.default_rng(seed)
    ld = a_env.jobs + 1 + pad
    traj, before, k = None, _state(b_env), 0
    unchanged_seen = 0
    for step in range(n_steps):
        if k == 0:
            traj = a_env.logits_trajectory(traj_len, out=traj)
            assert np.array_equal(np_(traj["real_obs"][0]), np_(b_env.real_obs)), step
            assert np.array_equal(np_(traj["action_mask"][0]), np_(b_env.action_mask)), step
        mask, done = np_(traj["action_mask"][k]).copy(), np_(a_env.done).copy()
        logits = lc.random_logits(rng, a_env, mask, ld, illegal=np.nan if step % 2 else 1e30)
        x = lc._to_dev(a_env, logits)
        _, _, _, _, info_a = a_env.step_logits_record(x, traj, k)
        _, _, _, _, info_b = b_env.step_logits(x)
        if oracle:
            lc.check_draws(a_env, logits, mask, done, np_(info_a["actions"]), np_(info_a["log_prob"]), step,
                           np_(a_env.flags), f"step {step}")
        after = _state(b_env)
        unchanged = _unchanged(before, after)
        unchanged_seen += int(unchanged.sum())
        check_slot(a_env, b_env, traj, k, info_b, unchanged, f"step {step}")
        if step % state_every == state_every - 1:
            assert_twins_equal(_Recorded(a_env, traj["real_obs"][k + 1]), b_env, step, state=True, stats=True)
        before, k = after, (k + 1) % traj_len
    a_env.refresh_obs()
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)
    return unchanged_seen


@native_test()
def record_mixed_batch(make_env, backend):
    # every lane class of the mixed step kernel, 129..256 jobs included; the ta01 envs finish (and auto-reset)
    if backend == "emu":
        big = synthetic_instance(200, 6, 7, max_dur=40)
        check_record(make_env, ["ta01", "ta01", "ta51", "ta80", "dmu16", big], n_steps=330, seed=3)
    else:
        big = synthetic_instance(200, 8, 9, max_dur=50)
        check_record(make_env, ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80", big] * 3,
                     n_steps=1200, seed=3, state_every=100)


@native_test()
def record_uniform_ta01(make_env, backend):
    check_record(make_env, seed=4, **{"emu": dict(names=["ta01"] * 9, n_steps=300),
                                      "gpu": dict(names=["ta01"] * 300, n_steps=700, state_every=100)}[backend])


@native_test()
def record_uniform_ta80(make_env, backend):
    check_record(make_env, seed=5, pad=0, **{"emu": dict(names=["ta80"] * 3, n_steps=150),
                                             "gpu": dict(names=["ta80"] * 40, n_steps=2600, state_every=200)}[backend])


@native_test()
def record_big_uniform(make_env, backend):
    # 129..256 jobs in a uniform batch: the 8-jobs-per-lane body of the uniform step kernel
    if backend == "emu":
        check_record(make_env, [synthetic_instance(200, 6, 7, max_dur=40)] * 2, n_steps=60, seed=6)
    else:
        check_record(make_env, [synthetic_instance(200, 8, 9, max_dur=50)] * 9, n_steps=400, seed=6, state_every=100)


@native_test()
def record_episode_ends_frozen(make_env, backend):
    """Without auto-reset: finished envs stay frozen and are recorded unchanged, with reward 0, step after step."""
    n = {"emu": 6, "gpu": 64}[backend]
    unchanged = check_record(make_env, ["ta01"] * n, n_steps=320, seed=8, auto_reset=False, traj_len=40)
    assert unchanged > 0


@native_test(emu=None)
def record_full_size_ta80(make_env):
    """The headline batch, ta80 at N = 65 536 with auto-reset, pre-rolled so that the envs are at staggered episode
    phases, then 8 recorded steps from seeded device logits: bit-identical to the twin stepped with step_logits."""
    import torch
    n, period = 65536, 2236
    a_env, b_env = twin_envs(make_env, ["ta80"] * n, seed=1234, auto_reset=True)
    quota = ((torch.arange(n, device=a_env.device) * 7919) % period).to(torch.int32)
    skip = torch.full((n,), N.ACTION_SKIP, dtype=torch.int32, device=a_env.device)
    for k in range(period):                               # env i takes (i * 7919) mod period transitions
        for env in (a_env, b_env):
            env.step(torch.where(quota > k, env.policy("RANDOM"), skip))
    gen = torch.Generator(device=a_env.device).manual_seed(0)
    traj, before = a_env.logits_trajectory(8), _state(b_env)
    for k in range(8):
        x = torch.randn((n, a_env.jobs + 1), device=a_env.device, generator=gen)
        a_env.step_logits_record(x, traj, k)
        _, _, _, _, info_b = b_env.step_logits(x)
        after = _state(b_env)
        check_slot(a_env, b_env, traj, k, info_b, _unchanged(before, after), f"step {k}")
        before = after
    assert_twins_equal(_Recorded(a_env, traj["real_obs"][8]), b_env, "end", state=True, stats=True)


@native_test()
def record_slot_isolation(make_env):
    """A recording step writes its own slot and nothing else: the other slots, and the bytes of its rows past J_i,
    keep a NaN / 0xAB sentinel."""
    big = synthetic_instance(200, 6, 7, max_dur=40)
    names = ["ta01", "ta51", "ta80", big, "ta01"]
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=12, auto_reset=True)
    K, n, J = 4, a_env.num_envs, a_env.jobs
    traj = a_env.logits_trajectory(K)
    traj["_obs"][1:] = float("nan")
    traj["_mask"][1:] = MASK_SENTINEL
    traj["_scalars"][:] = -7
    traj["actions"][:] = -7
    traj["log_prob"][:] = float("nan")
    # the bytes a row of env i may hold: 7 * J_i floats; the mask bytes up to the lane's last whole store
    kj = np.array([1 << (0 if Ji <= 32 else 1 if Ji <= 64 else 2 if Ji <= 128 else 3) for Ji in a_env.env_jobs])
    mask_used = -(-(a_env.env_jobs + 1) // kj) * kj
    rng = np.random.default_rng(12)
    for k in range(K):
        mask = np_(traj["action_mask"][k]).copy()
        x = lc._to_dev(a_env, lc.random_logits(rng, a_env, mask, J + 1))
        a_env.step_logits_record(x, traj, k)
        b_env.step_logits(x)
        obs = np_(traj["_obs"]).copy()
        rows = np_(traj["_mask"]).copy()
        for s in range(1, K + 1):
            slot_obs = obs[s][: n * J * 7].reshape(n, J * 7)
            slot_mask = rows[s][: n * a_env._b.mask_stride].reshape(n, -1)
            for i, Ji in enumerate(a_env.env_jobs):
                written = s <= k + 1                      # slots 1 .. k + 1 hold transitions 0 .. k
                assert np.isnan(slot_obs[i, 7 * Ji:]).all() and (slot_mask[i, mask_used[i]:] == MASK_SENTINEL).all(), (k, s, i)
                assert written == (not np.isnan(slot_obs[i, : 7 * Ji]).any()), (k, s, i)
                assert written == (not (slot_mask[i, : Ji + 1] == MASK_SENTINEL).any()), (k, s, i)
            assert np.isnan(obs[s][n * J * 7:]).all() and (rows[s][n * a_env._b.mask_stride:] == MASK_SENTINEL).all()
        assert (np_(traj["_scalars"][k + 1:]) == -7).all() and (np_(traj["actions"][k + 1:]) == -7).all(), k
        assert np.isnan(np_(traj["log_prob"][k + 1:])).all(), k
        for i, Ji in enumerate(a_env.env_jobs):
            assert np.array_equal(obs[k + 1][: n * J * 7].reshape(n, J, 7)[i, :Ji], np_(b_env.real_obs)[i, :Ji]), (k, i)


def _stale_twins(make_env, seed):
    """Twins without auto-reset, env 1 crafted done (frozen), after three recording steps on A and the same three
    step_logits on B: A's real_obs is stale."""
    a_env, b_env = twin_envs(make_env, ["ta01", "ta01", "ta31", "ta51"], sort=False, seed=seed)
    for env in (a_env, b_env):
        x = env.export_state()
        x["legal"][1] = 0
        x["flags"][1] = int(x["flags"][1]) | (N.FLAG_DONE << 8) | 1
        env.import_state(x)
    rng = np.random.default_rng(seed)
    traj = a_env.logits_trajectory(3)
    for k in range(3):
        x = lc._to_dev(a_env, lc.random_logits(rng, a_env, np_(traj["action_mask"][k]), a_env.jobs + 1))
        a_env.step_logits_record(x, traj, k)
        b_env.step_logits(x)
    assert np_(b_env.done)[1] and not np.array_equal(np_(a_env.real_obs), np_(b_env.real_obs))
    return a_env, b_env, rng


@native_test()
def record_stale_then_refresh(make_env):
    """After recording steps, refresh_obs() and every non-recording call leave real_obs equal to the twin's, frozen
    done envs included: refresh_obs, step, step_logits, reset(mask), rollout, step_host."""
    for seed, op in enumerate(("refresh_obs", "step", "step_logits", "reset_mask", "rollout", "step_host")):
        a_env, b_env, rng = _stale_twins(make_env, 40 + seed)
        if op == "refresh_obs":
            a_env.refresh_obs()
        else:
            acts = np_(b_env.policy("RANDOM", step_index=99)).copy()   # the same actions for both twins
            x = lc._to_dev(b_env, lc.random_logits(rng, b_env, np_(b_env.action_mask), b_env.jobs + 1))
            for env in (a_env, b_env):
                if op == "step":
                    env.step(acts)
                elif op == "step_logits":
                    env.step_logits(x)
                elif op == "reset_mask":
                    env.reset(np.array([1, 0, 0, 1], np.uint8))   # env 1, frozen done, is not reset
                elif op == "rollout":
                    env.rollout("FIFO", 5)
                else:
                    env.step_host(acts)
        assert_twins_equal(a_env, b_env, op, state=True, stats=True)


@native_test()
def record_edge_cases(make_env):
    """The edge-case batch of step_logits (one finite legal logit, NaN / +inf / all -inf on legal entries, only the
    no-op legal, a done env; with and without auto-reset): the error, no-op-only and done envs get correct slot rows,
    with reward 0 where the step changed nothing."""
    for auto_reset in (False, True):
        n = 8
        a_env, b_env = twin_envs(make_env, ["ta01"] * n, seed=5, auto_reset=auto_reset)
        J = a_env.jobs
        for env in (a_env, b_env):
            env.step(np.zeros(n, np.int32))               # every env allocates job 0: one machine busy
            x = env.export_state()
            x["legal"][6] = 0
            x["legal"][7] = 0
            x["flags"][6] = int(x["flags"][6]) | (N.FLAG_NOOP_LEGAL << 8)
            x["flags"][7] = int(x["flags"][7]) | (N.FLAG_DONE << 8) | 1
            env.import_state(x)
        traj = a_env.logits_trajectory(1)
        mask = np_(traj["action_mask"][0]).copy()
        assert not mask[6, :J].any() and mask[6, J] and not mask[7].any()
        logits = np.random.default_rng(1).standard_normal((n, J + 1)).astype(np.float32)
        logits[~mask] = 1e30
        logits[0, :J] = -np.inf; logits[0, 3] = 0.7
        logits[1, 2] = np.nan
        logits[2, 5] = np.inf
        logits[3, 1:J] = -np.inf
        logits[6, J] = np.nan
        before = _state(b_env)
        x = lc._to_dev(a_env, logits)
        _, _, _, _, info = a_env.step_logits_record(x, traj, 0)
        _, _, _, _, info_b = b_env.step_logits(x)
        unchanged = _unchanged(before, _state(b_env))
        expect = [False, True, True, True, False, False, False, not auto_reset]
        assert list(unchanged) == expect, (auto_reset, unchanged)
        acts = np_(info["actions"])
        assert acts[0] == 3 and all(acts[i] == N.ACTION_SKIP for i in (1, 2, 3)) and acts[6] == J and acts[7] == 0
        assert (np_(traj["_scalars"][0])[unchanged, :2] == 0).all()
        check_slot(a_env, b_env, traj, 0, info_b, unchanged, f"auto_reset={auto_reset}")
        a_env.refresh_obs()
        assert_twins_equal(a_env, b_env, auto_reset, state=True, stats=True)


@native_test()
def record_launch_counts(make_env):
    """One launch per recording step; the first non-recording call after them adds the refresh, one launch per lane
    class present (as a reset); exports, policies and statistics leave real_obs stale and add no refresh."""
    import torch
    names = ["ta01", "ta51", "ta80", "ta01"]              # lane classes 1, 2 and 4 jobs per lane
    env = make_env(len(names), batch_cfg(names, sort=False), seed=9)
    classes = 3
    traj = env.logits_trajectory(3)
    x = torch.zeros((env.num_envs, env.jobs + 1), device=env.device)
    c = env.launch_count
    for k in range(3):
        env.step_logits_record(x, traj, k)
        assert env.launch_count == c + k + 1
    c = env.launch_count
    env.export_state(); env.policy("RANDOM"); env.stats()
    assert env.launch_count == c + 2 * classes + 1
    c = env.launch_count
    env.step(env.policy("RANDOM"))
    assert env.launch_count == c + classes + classes + 1   # policy, refresh, step
    c = env.launch_count
    env.step(np.full(env.num_envs, N.ACTION_SKIP, np.int32))
    env.refresh_obs()
    assert env.launch_count == c + 1
    env.step_logits_record(x, traj, 0)
    c = env.launch_count
    env.refresh_obs(); env.refresh_obs()
    assert env.launch_count == c + classes


@native_test()
def record_abi_errors(make_env):
    """jss_step_logits_record returns JSS_ERR_INVALID for a NULL or misaligned slot pointer, and for the arguments
    jss_step_logits rejects; log_prob_out may be NULL.  step_logits_record rejects a step outside the trajectory."""
    import pytest
    import torch
    env = make_env(3, {"instance_paths": ["ta01", "ta31"], "env_to_instance": [0, 1, 0]})
    J = env.jobs
    traj = env.logits_trajectory(2)
    logits = torch.zeros((3, J + 1), dtype=torch.float32, device=env.device)
    acts = torch.zeros(3, dtype=torch.int32, device=env.device)
    L, h, st = env._L, env._h, env._stream()
    ptrs = [traj["_obs"][1].data_ptr(), traj["_mask"][1].data_ptr(), traj["_scalars"][0].data_ptr()]

    def call(obs, mask, scalars, logits_p=logits.data_ptr(), acts_p=acts.data_ptr(), ld=J + 1):
        return L.jss_step_logits_record(h, logits_p, ld, 0, 0, acts_p, None, obs, mask, scalars, st)

    for i in range(3):
        bad = list(ptrs)
        bad[i] = None
        assert call(*bad) == -1, i
        bad[i] = ptrs[i] + 4
        assert call(*bad) == -1, i
    assert b"jss_step_logits_record" in L.jss_last_error(h)
    assert call(*ptrs, logits_p=None) == -1 and call(*ptrs, acts_p=None) == -1 and call(*ptrs, ld=J) == -1
    assert call(*ptrs) == 0
    assert L.jss_refresh_obs(h, st) == 0 and L.jss_refresh_obs(None, st) == -1
    env.synchronize()
    assert (np_(acts) >= 0).all()
    with pytest.raises(ValueError):
        env.step_logits_record(logits, traj, 2)
    with pytest.raises(ValueError):
        env.step_logits_record(logits[:, :J], traj, 0)
    # a trajectory made for another batch (fewer envs) is refused instead of written past
    other = make_env(2, {"instance_paths": ["ta01", "ta31"], "env_to_instance": [0, 1]})
    small = other.logits_trajectory(2)
    with pytest.raises(ValueError):
        env.step_logits_record(logits, small, 0)
    with pytest.raises(ValueError):
        env.logits_trajectory(2, out=small)
