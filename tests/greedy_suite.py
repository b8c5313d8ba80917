"""The tests of jss_step_greedy and jss_step_greedy_record (greedy / epsilon-greedy decoding of action scores fused
into the step), declared once for both backends (tests/backends.py) and collected by tests/test_emu_greedy.py and
tests/test_gpu_greedy.py.  Every decision is checked against the float64 restatement in tests/greedy_oracle.py, the
step against a twin env stepped with jss_step(actions), and the recording form against a twin stepped with
jss_step_greedy."""
import numpy as np

from jssenv_b200 import _native as N
from tests import greedy_oracle as GO
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import assert_twins_equal, batch_cfg, np_, oracle_episode, synthetic_instance, twin_envs
from tests.record_suite import _Recorded, _state, _unchanged, check_slot

EPSILONS = [0.0, 0.05, 0.3, 1.0]


def random_scores(rng, env, mask, ld, step, illegal):
    """The seeded rows of lc.random_logits (-inf at random, `illegal` off the legal actions, NaN in the padding),
    rounded to whole numbers every third step: exact ties, and -0.0 next to +0.0."""
    x = lc.random_logits(rng, env, mask, ld, illegal=illegal)
    return np.round(x) if step % 3 == 2 else x


def check_decisions(env, scores, mask, done, epsilon, acts, logp, step_index, flags_after, ctx):
    """Every env's reported action equals the oracle's; its log_prob is within 1e-6 relative of the oracle's, and
    +0.0 bit for bit at epsilon = 0.  Returns the actions a twin stepped with jss_step takes (an out-of-range one
    where the env got the error bit) and the number of envs that explored."""
    twin = acts.copy()
    explored = 0
    for i, Ji in enumerate(env.env_jobs):
        legal = mask[i, : Ji + 1]
        a_ref, lp_ref, err = GO.greedy(scores[i], legal, bool(done[i]), epsilon, env.seed, env.env_id_base + i,
                                       step_index)
        a, lp = int(acts[i]), float(logp[i])
        where = (ctx, i, a, a_ref, lp, lp_ref)
        assert a == a_ref, where
        if err:
            assert np.isnan(lp) and flags_after[i] & N.FLAG_ERROR, where
            twin[i] = lc.BIG_ACTION
        elif np.isnan(lp_ref):
            assert np.isnan(lp), where
        else:
            assert abs(lp - lp_ref) <= 1e-6 * abs(lp_ref), where
            if epsilon == 0.0:
                assert logp[i:i + 1].view(np.uint32)[0] == 0, where
            explored += a != GO.greedy(scores[i], legal, bool(done[i]), 0.0, 0, 0, 0)[0]
    return twin, explored


def check_greedy(make_env, names, n_steps, seed, epsilon, pad=3, state_every=25, auto_reset=True):
    """step_greedy on a batch driven by seeded scores (with -inf entries, ties, +-0, huge values or NaN on illegal
    entries, ld > J+1): every decision against the oracle, and a twin env stepped with jss_step(actions)
    bit-identical after every step."""
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=seed, auto_reset=auto_reset)
    rng = np.random.default_rng(seed)
    ld = a_env.jobs + 1 + pad
    explored = 0
    for k in range(n_steps):
        mask, done = np_(a_env.action_mask).copy(), np_(a_env.done).copy()
        scores = random_scores(rng, a_env, mask, ld, k, illegal=np.nan if k % 2 else 1e30)
        step_index = a_env._step_index
        _, _, _, _, info = a_env.step_greedy(lc._to_dev(a_env, scores), epsilon)
        acts, logp = np_(info["actions"]).copy(), np_(info["log_prob"]).copy()
        twin, e = check_decisions(a_env, scores, mask, done, epsilon, acts, logp, step_index, np_(a_env.flags),
                                  f"epsilon {epsilon} step {k}")
        explored += e
        b_env.step(twin)
        full = k % state_every == state_every - 1
        assert_twins_equal(a_env, b_env, f"step {k}", state=full, stats=full)
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)
    assert (explored > 0) == (epsilon > 0.0), explored
    return a_env


@native_test(emu=EPSILONS, gpu=EPSILONS)
def greedy_mixed_batch(make_env, backend, epsilon):
    # every lane class of the mixed step kernel, 129..256 jobs included; the ta01 envs finish (and auto-reset)
    if backend == "emu":
        big = synthetic_instance(200, 6, 7, max_dur=40)
        env = check_greedy(make_env, ["ta01", "ta01", "ta51", "ta80", "dmu16", big], n_steps=300, seed=3,
                           epsilon=epsilon, state_every=50)
    else:
        big = synthetic_instance(200, 8, 9, max_dur=50)
        env = check_greedy(make_env, ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80",
                                      big] * 3, n_steps=1200, seed=3, epsilon=epsilon, state_every=100)
    assert np_(env.episode_count)[:2].min() > 0


@native_test(emu=EPSILONS, gpu=EPSILONS)
def greedy_uniform_ta01(make_env, backend, epsilon):
    check_greedy(make_env, seed=4, epsilon=epsilon, **{"emu": dict(names=["ta01"] * 9, n_steps=300),
                                                       "gpu": dict(names=["ta01"] * 300, n_steps=700,
                                                                   state_every=100)}[backend])


@native_test(emu=EPSILONS, gpu=EPSILONS)
def greedy_uniform_ta80(make_env, backend, epsilon):
    check_greedy(make_env, seed=5, pad=0, epsilon=epsilon, **{"emu": dict(names=["ta80"] * 3, n_steps=150),
                                                              "gpu": dict(names=["ta80"] * 40, n_steps=2600,
                                                                          state_every=200)}[backend])


@native_test(emu=EPSILONS, gpu=EPSILONS)
def greedy_big_instances(make_env, backend, epsilon):
    # 129..256 jobs: the 8-jobs-per-lane bodies of the uniform and the mixed step kernels
    if backend == "emu":
        big = synthetic_instance(200, 6, 7, max_dur=40)
        check_greedy(make_env, [big] * 2, n_steps=60, seed=6, epsilon=epsilon)
        check_greedy(make_env, [big, "ta01"], n_steps=60, seed=7, epsilon=epsilon)
    else:
        big = synthetic_instance(200, 8, 9, max_dur=50)
        check_greedy(make_env, [big] * 9, n_steps=400, seed=6, epsilon=epsilon, state_every=100)
        check_greedy(make_env, [big, "ta01", "ta51", "ta80"] * 2, n_steps=400, seed=7, epsilon=epsilon,
                     state_every=100)


def _edge_batch(make_env, auto_reset):
    """Twins of 10 ta01 envs after one step of job 0 (its machine busy), env 6 crafted with only the no-op legal and
    env 7 done, and their scores: one finite legal score among -inf (0), NaN / +inf / all -inf on legal entries (1, 2,
    3), an exact tie (4), -0.0 before +0.0 and +0.0 before -0.0 at the top (5, 9), NaN on the only legal action (6);
    huge values on illegal entries and in the padding, NaN there for env 8."""
    n = 10
    a_env, b_env = twin_envs(make_env, ["ta01"] * n, seed=5, auto_reset=auto_reset)
    J = a_env.jobs
    for env in (a_env, b_env):
        env.step(np.zeros(n, np.int32))
        x = env.export_state()
        x["legal"][6] = 0
        x["legal"][7] = 0                                 # a done env has no legal job
        x["flags"][6] = int(x["flags"][6]) | (N.FLAG_NOOP_LEGAL << 8)
        x["flags"][7] = int(x["flags"][7]) | (N.FLAG_DONE << 8) | 1
        env.import_state(x)
    mask = np_(a_env.action_mask).copy()
    assert not mask[6, :J].any() and mask[6, J] and not mask[7].any() and not mask[0, 0]
    ld = J + 1 + 5
    s = np.random.default_rng(1).standard_normal((n, ld)).astype(np.float32)
    off = ~np.pad(mask[:, : J + 1], ((0, 0), (0, ld - J - 1)))
    s[off] = 1e30
    s[8][off[8]] = np.nan
    s[0, :J] = -np.inf; s[0, 3] = 0.7
    s[1, 2] = np.nan
    s[2, 5] = np.inf
    s[3, 1:J] = -np.inf
    first = {i: np.flatnonzero(mask[i, :J]) for i in (4, 5, 9)}
    s[4, first[4]] = 2.5                                  # every legal job ties
    s[5, :J] = -1.0; s[5, first[5][0]] = -0.0; s[5, first[5][1]] = 0.0
    s[9, :J] = -1.0; s[9, first[9][0]] = 0.0; s[9, first[9][1]] = -0.0
    s[6, J] = np.nan
    return a_env, b_env, mask, s, {i: int(f[0]) for i, f in first.items()}


@native_test()
def greedy_edge_cases(make_env):
    """The edge-case rows, at epsilon 0 and 1, with and without auto-reset: ties and +-0 ties go to the lowest index,
    a single finite score wins, illegal and padding entries are never chosen, bad rows error at either epsilon, the
    no-op-only env takes J, the done env 0 (frozen or reset)."""
    for auto_reset in (False, True):
        for epsilon in (0.0, 1.0):
            ctx = (auto_reset, epsilon)
            a_env, b_env, mask, s, lowest = _edge_batch(make_env, auto_reset)
            J = a_env.jobs
            done = np_(a_env.done).copy()
            step_index = a_env._step_index
            _, _, _, _, info = a_env.step_greedy(lc._to_dev(a_env, s), epsilon)
            acts, logp = np_(info["actions"]).copy(), np_(info["log_prob"]).copy()
            twin, _ = check_decisions(a_env, s, mask, done, epsilon, acts, logp, step_index, np_(a_env.flags), ctx)
            flags = np_(a_env.flags)
            for i in (1, 2, 3):
                assert acts[i] == N.ACTION_SKIP and np.isnan(logp[i]) and flags[i] & N.FLAG_ERROR, (ctx, i)
            assert acts[6] == J and logp[6] == 0.0 and acts[7] == 0 and logp[7] == 0.0, (ctx, acts, logp)
            if epsilon == 0.0:
                assert acts[0] == 3 and acts[4] == lowest[4] and acts[5] == lowest[5] and acts[9] == lowest[9], ctx
            for i in (0, 4, 5, 8, 9):
                assert 0 <= acts[i] <= J and mask[i, acts[i]], (ctx, i)
            b_env.step(twin)
            assert_twins_equal(a_env, b_env, ctx, state=True, stats=True)
            if auto_reset:
                assert int(a_env.current_time_step[7]) == 0 and np_(a_env.action_mask)[7, :J].all(), ctx
            else:
                assert np_(a_env.done)[7], ctx


@native_test()
def greedy_seed_independence_and_null_log_prob(make_env):
    """At epsilon = 0 two envs with different seeds, stepped at different step indices, choose the same actions with
    log_prob +0.0; log_prob_out may be NULL, which changes nothing else."""
    import torch
    names = ["ta01", "ta51", "ta80", "ta01"]
    a_env = make_env(4, batch_cfg(names, sort=False), seed=1)
    b_env = make_env(4, batch_cfg(names, sort=False), seed=2)
    a_env.reset(); b_env.reset()
    b_env._step_index = 17
    rng = np.random.default_rng(2)
    for k in range(40):
        x = lc._to_dev(a_env, random_scores(rng, a_env, np_(a_env.action_mask), a_env.jobs + 1, k, 1e30))
        _, _, _, _, ia = a_env.step_greedy(x)
        acts = torch.full((4,), -7, dtype=torch.int32, device=b_env.device)
        rc = b_env._L.jss_step_greedy(b_env._h, x.data_ptr(), b_env.jobs + 1, 0.0, b_env.seed, b_env._step_index,
                                      acts.data_ptr(), None, b_env._stream())
        assert rc == 0
        b_env._step_index += 3
        assert np.array_equal(np_(ia["actions"]), np_(acts)), k
        assert (np_(ia["log_prob"]).view(np.uint32)[np_(ia["actions"]) >= 0] == 0).all(), k
        assert_twins_equal(a_env, b_env, k)
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)


@native_test(emu=dict(n_steps=60), gpu=dict(n_total=60, n_steps=600))
def greedy_shard_invariance(make_env, n_steps, n_total=12, seed=31, epsilon=0.3):
    """Shards created with env_id_base != 0 reproduce the unsharded batch's actions and log_probs bit for bit at
    epsilon > 0, and its outputs, transition for transition."""
    names = ["ta01", "ta31", "ta51", "ta80"]
    e2i = np.arange(n_total) % len(names)
    cuts = [0, 5, n_total]
    whole = make_env(n_total, {"instance_paths": names, "env_to_instance": e2i}, seed=seed, auto_reset=True)
    shards = [make_env(hi - lo, {"instance_paths": names, "env_to_instance": e2i[lo:hi]}, seed=seed, auto_reset=True,
                       env_id_base=lo) for lo, hi in zip(cuts[:-1], cuts[1:])]
    whole.reset()
    for s in shards:
        s.reset()
    rng = np.random.default_rng(seed)
    for k in range(n_steps):
        dev = lc._to_dev(whole, random_scores(rng, whole, np_(whole.action_mask), whole.jobs + 1, k, 1e30))
        _, _, _, _, iw = whole.step_greedy(dev, epsilon)
        aw, lw = np_(iw["actions"]).copy(), np_(iw["log_prob"]).copy()
        for s, lo, hi in zip(shards, cuts[:-1], cuts[1:]):
            _, _, _, _, i_s = s.step_greedy(dev[lo:hi, : s.jobs + 1], epsilon)   # the whole batch's row stride as ld
            assert np.array_equal(np_(i_s["actions"]), aw[lo:hi]), (k, lo)
            assert np.array_equal(np_(i_s["log_prob"]).view(np.uint32), lw[lo:hi].view(np.uint32)), (k, lo)
            assert_twins_equal(s, whole, k, rows=slice(lo, hi))


def check_greedy_record(make_env, names, n_steps, seed, epsilon, traj_len=16, pad=3, auto_reset=True, state_every=25):
    """Env A records every transition with step_greedy_record into trajectories of `traj_len` steps (one dict,
    reused), twin B steps with step_greedy on the same scores: after every step the slot and A's outputs equal B's,
    every `state_every` steps the exported state and the statistics too.  Returns how many env-steps were unchanged."""
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=seed, auto_reset=auto_reset)
    rng = np.random.default_rng(seed)
    ld = a_env.jobs + 1 + pad
    traj, before, k = None, _state(b_env), 0
    unchanged_seen = 0
    for step in range(n_steps):
        if k == 0:
            traj = a_env.logits_trajectory(traj_len, out=traj)
        mask = np_(traj["action_mask"][k]).copy()
        x = lc._to_dev(a_env, random_scores(rng, a_env, mask, ld, step, illegal=np.nan if step % 2 else 1e30))
        a_env.step_greedy_record(x, traj, k, epsilon)
        _, _, _, _, info_b = b_env.step_greedy(x, epsilon)
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
def greedy_record_mixed_batch(make_env, backend):
    if backend == "emu":
        big = synthetic_instance(200, 6, 7, max_dur=40)
        check_greedy_record(make_env, ["ta01", "ta01", "ta51", "ta80", "dmu16", big], n_steps=260, seed=3,
                            epsilon=0.3, state_every=50)
    else:
        big = synthetic_instance(200, 8, 9, max_dur=50)
        check_greedy_record(make_env, ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80",
                                       big] * 3, n_steps=1200, seed=3, epsilon=0.3, state_every=100)


@native_test()
def greedy_record_uniform(make_env, backend):
    if backend == "emu":
        check_greedy_record(make_env, ["ta01"] * 5, n_steps=100, seed=4, epsilon=0.05)
        check_greedy_record(make_env, ["ta80"] * 2, n_steps=50, seed=5, epsilon=0.0, pad=0)
    else:
        check_greedy_record(make_env, ["ta01"] * 300, n_steps=700, seed=4, epsilon=0.05, state_every=100)
        check_greedy_record(make_env, ["ta80"] * 40, n_steps=2600, seed=5, epsilon=0.0, pad=0, state_every=200)


@native_test()
def greedy_record_episode_ends(make_env, backend):
    """Episode ends with auto-reset (the envs are reset and recorded) and without (finished envs stay frozen and are
    recorded unchanged, with reward 0, step after step)."""
    n = {"emu": 4, "gpu": 64}[backend]
    check_greedy_record(make_env, ["ta01"] * n, n_steps=300, seed=9, epsilon=0.05, traj_len=40)
    unchanged = check_greedy_record(make_env, ["ta01"] * n, n_steps=300, seed=8, epsilon=0.0, auto_reset=False,
                                    traj_len=40)
    assert unchanged > 0


@native_test()
def greedy_record_edge_cases(make_env):
    """The edge-case rows recorded: the error, no-op-only and done envs get correct slot rows, reward 0 where the step
    changed nothing; the env's own outputs equal the twin's after refresh_obs()."""
    for auto_reset in (False, True):
        a_env, b_env, _, s, _ = _edge_batch(make_env, auto_reset)
        traj = a_env.logits_trajectory(1)
        before = _state(b_env)
        x = lc._to_dev(a_env, s)
        a_env.step_greedy_record(x, traj, 0, 0.3)
        _, _, _, _, info_b = b_env.step_greedy(x, 0.3)
        unchanged = _unchanged(before, _state(b_env))
        assert unchanged[[1, 2, 3]].all() and unchanged[7] == (not auto_reset), unchanged
        check_slot(a_env, b_env, traj, 0, info_b, unchanged, auto_reset)
        a_env.refresh_obs()
        assert_twins_equal(a_env, b_env, auto_reset, state=True, stats=True)


@native_test()
def greedy_record_stale_then_refresh(make_env):
    """After recording steps real_obs is stale; refresh_obs(), step_greedy and step leave it equal to the twin's."""
    for seed, op in enumerate(("refresh_obs", "step_greedy", "step")):
        a_env, b_env = twin_envs(make_env, ["ta01", "ta01", "ta31", "ta51"], sort=False, seed=60 + seed)
        rng = np.random.default_rng(seed)
        traj = a_env.logits_trajectory(3)
        for k in range(3):
            x = lc._to_dev(a_env, random_scores(rng, a_env, np_(traj["action_mask"][k]), a_env.jobs + 1, k, 1e30))
            a_env.step_greedy_record(x, traj, k, 0.3)
            b_env.step_greedy(x, 0.3)
        assert not np.array_equal(np_(a_env.real_obs), np_(b_env.real_obs))
        if op == "refresh_obs":
            a_env.refresh_obs()
        else:
            x = lc._to_dev(a_env, random_scores(rng, a_env, np_(b_env.action_mask), a_env.jobs + 1, 0, 1e30))
            acts = np_(b_env.policy("RANDOM", step_index=99)).copy()
            for env in (a_env, b_env):
                env.step_greedy(x, 0.3) if op == "step_greedy" else env.step(acts)
        assert_twins_equal(a_env, b_env, op, state=True, stats=True)


@native_test()
def greedy_record_launch_counts(make_env):
    """One launch per step_greedy / step_greedy_record call when nothing is stale; the first non-recording call after
    recording adds the refresh, one launch per lane class present."""
    import torch
    names = ["ta01", "ta51", "ta80", "ta01"]              # lane classes 1, 2 and 4 jobs per lane
    env = make_env(len(names), batch_cfg(names, sort=False), seed=9)
    env.reset()
    classes = 3
    x = torch.zeros((env.num_envs, env.jobs + 1), device=env.device)
    c = env.launch_count
    for k in range(3):
        env.step_greedy(x, 0.3 * k)
        assert env.launch_count == c + k + 1
    traj = env.logits_trajectory(3)
    c = env.launch_count
    for k in range(3):
        env.step_greedy_record(x, traj, k, 0.5)
        assert env.launch_count == c + k + 1
    c = env.launch_count
    env.step_greedy(x)
    assert env.launch_count == c + classes + 1


@native_test()
def greedy_abi_errors(make_env):
    """jss_step_greedy and jss_step_greedy_record return JSS_ERR_INVALID, with a message naming the function, for a
    NULL scores or actions_out pointer, ld < jobs_max + 1, epsilon NaN or outside [0, 1], and (recording) a NULL or
    misaligned slot pointer; step_greedy and step_greedy_record raise ValueError for a bad epsilon, bad scores or a
    step outside the trajectory."""
    import pytest
    import torch
    env = make_env(3, {"instance_paths": ["ta01", "ta31"], "env_to_instance": [0, 1, 0]})
    env.reset()
    J = env.jobs
    traj = env.logits_trajectory(2)
    scores = torch.zeros((3, J + 1), dtype=torch.float32, device=env.device)
    acts = torch.zeros(3, dtype=torch.int32, device=env.device)
    L, h, st = env._L, env._h, env._stream()
    ptrs = [traj["_obs"][1].data_ptr(), traj["_mask"][1].data_ptr(), traj["_scalars"][0].data_ptr()]

    def plain(eps=0.0, s=scores.data_ptr(), a=acts.data_ptr(), ld=J + 1):
        return L.jss_step_greedy(h, s, ld, eps, 0, 0, a, None, st)

    def record(eps=0.0, s=scores.data_ptr(), a=acts.data_ptr(), ld=J + 1, slot=ptrs):
        return L.jss_step_greedy_record(h, s, ld, eps, 0, 0, a, None, *slot, st)

    for call, name in ((plain, b"jss_step_greedy"), (record, b"jss_step_greedy_record")):
        for kw in (dict(s=None), dict(a=None), dict(ld=J), dict(eps=float("nan")), dict(eps=-0.01),
                   dict(eps=1.0 + 1e-9), dict(eps=float("inf"))):
            assert call(**kw) == -1, (name, kw)
            assert L.jss_last_error(h).startswith(name + b":"), (name, kw, L.jss_last_error(h))
        assert call(eps=0.0) == 0 and call(eps=1.0) == 0, name
    for i in range(3):
        bad = list(ptrs)
        bad[i] = None
        assert record(slot=bad) == -1, i
        bad[i] = ptrs[i] + 4
        assert record(slot=bad) == -1, i
        assert L.jss_last_error(h).startswith(b"jss_step_greedy_record:"), i
    env.synchronize()
    assert (np_(acts) >= 0).all()
    step_index = env._step_index
    for eps in (float("nan"), -0.5, 1.5):
        with pytest.raises(ValueError):
            env.step_greedy(scores, eps)
        with pytest.raises(ValueError):
            env.step_greedy_record(scores, traj, 0, eps)
    assert env._step_index == step_index                  # refused before the native call
    with pytest.raises(ValueError):
        env.step_greedy(scores[:, :J])
    with pytest.raises(ValueError):
        env.step_greedy_record(scores, traj, 2)
    env.step_greedy(scores, 0.5)
    env.step_greedy_record(scores, traj, 1, 0.5)
    assert env._step_index == step_index + 2


@native_test(emu=None)
def greedy_exploration_distribution(make_env):
    """ta01 at N = 65 536 right after reset (every job legal, the no-op not), one shared score row, epsilon = 0.25:
    the envs that left the greedy action are a binomial sample of epsilon (1 - 1/n), their actions are uniform over
    the other n - 1 actions, and log_prob takes only its two analytic values."""
    import torch
    from scipy.stats import binomtest, chisquare
    n_envs, epsilon = 65536, 0.25
    env = make_env(n_envs, {"instance_path": "ta01"}, seed=11)
    env.reset()
    J = env.jobs
    row = torch.randn(J + 1, generator=torch.Generator().manual_seed(0)).to(env.device)
    _, _, _, _, info = env.step_greedy(row.expand(n_envs, J + 1), epsilon)
    acts, logp = info["actions"].cpu().numpy(), info["log_prob"].cpu().numpy()
    g, n = int(torch.argmax(row[:J])), J
    assert acts.min() >= 0 and acts.max() < J
    away = acts != g
    test = binomtest(int(away.sum()), n_envs, epsilon * (1 - 1 / n))
    assert test.pvalue > 1e-6, (test, away.sum())
    hist = np.delete(np.bincount(acts[away], minlength=J), g)
    res = chisquare(hist)
    assert res.pvalue > 1e-6, (res, hist)
    e = GO.threshold(epsilon) * 2.0 ** -32
    want = np.where(away, np.log(e / n), np.log(1 - e + e / n))
    assert np.abs(logp - want).max() <= 1e-6 * np.abs(want).max()
    assert len(np.unique(logp)) == 2


@native_test(emu=None)
def greedy_static_priority_ta80(make_env):
    """ta80 at N = 65 536 without auto-reset, epsilon = 0, a fixed random score row per env (a static priority
    rule), stepped until every env is done: every env's raw return is 2 sum_op - M makespan, and for a sample of envs
    the makespan equals a CPU oracle replay of the same rule."""
    import torch
    n_envs, cap = 65536, 5000
    env = make_env(n_envs, {"instance_path": "ta80"}, seed=13, auto_reset=False)
    env.reset()
    J, M = env.jobs, env.machines
    sum_op = int(env.instance_scalars[0][2])
    scores = torch.randn((n_envs, J + 1), generator=torch.Generator(device=env.device).manual_seed(3), device=env.device)
    ret = torch.zeros(n_envs, dtype=torch.int64, device=env.device)
    steps = 0
    while steps < cap:
        live = ~env.done.clone()
        env.step_greedy(scores)
        ret += torch.where(live, env.reward_raw.to(torch.int64), 0)
        steps += 1
        if steps % 50 == 0 and bool(env.done.all()):
            break
    assert bool(env.done.all()), steps
    assert not (np_(env.flags) & N.FLAG_ERROR).any()
    makespan = np_(env.current_time_step).astype(np.int64)
    assert np.array_equal(np_(ret), 2 * sum_op - M * makespan)
    assert np.array_equal(np_(env.last_makespan), makespan)
    rows = scores.cpu().numpy()
    for i in (0, 1, 4097, 33333, 65535):
        def choose(o, step, x=rows[i]):
            legal = np.flatnonzero(np.asarray(o.get_legal_actions(), bool))
            return int(legal[np.argmax(x[legal])])
        assert oracle_episode("ta80", choose)[0] == makespan[i], i
