"""Backend-agnostic checks of jss_step_logits (the masked categorical draw from policy logits fused into the step):
the native env (tests/backends.py) against the float64 restatement of the draw in oracle/logits_oracle.py, and against
a twin env stepped with jss_step(actions)."""
import numpy as np

from jssenv_b200 import _native as N
from oracle import logits_oracle as LO
from tests.parity_common import assert_twins_equal, np_, twin_envs

BIG_ACTION = 1 << 20          # out of range: jss_step sets the error bit and leaves the env unchanged


def _to_dev(env, arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).to(env.device)


def random_logits(rng, env, mask, ld, p_ninf=0.1, illegal=1e30):
    """Seeded logits for the batch: N(0, 2^2) on the candidates, -inf at random (p_ninf), `illegal` (a huge value or
    NaN) on every action that is not legal under `mask`, NaN in the columns past J_i (never read)."""
    n = env.num_envs
    x = (2.0 * rng.standard_normal((n, ld))).astype(np.float32)
    x[rng.random((n, ld)) < p_ninf] = -np.inf
    for i, Ji in enumerate(env.env_jobs):
        row = x[i]
        row[: Ji + 1][~mask[i, : Ji + 1]] = illegal
        row[Ji + 1:] = np.nan
    return x


def check_draws(env, logits, mask, done, acts, logp, step_index, flags_after, ctx):
    """Every env's reported action / log_prob against the float64 oracle.  Returns (twin actions, decisions,
    decisions where the device picked the oracle's argmax)."""
    twin = acts.copy()
    decisions = agree = 0
    for i, Ji in enumerate(env.env_jobs):
        legal = mask[i, : Ji + 1]
        a_ref, lp_ref, err, scores = LO.draw(logits[i], legal, bool(done[i]), env.seed, env.env_id_base + i, step_index)
        a, lp = int(acts[i]), float(logp[i])
        where = (ctx, i, a, a_ref, lp, lp_ref)
        if err:
            assert a == N.ACTION_SKIP and np.isnan(lp) and flags_after[i] & N.FLAG_ERROR, where
            twin[i] = BIG_ACTION
            continue
        if scores is None:                                # done env / only the no-op legal / nothing legal
            assert a == a_ref and (lp == lp_ref or (np.isnan(lp) and np.isnan(lp_ref))), where
            continue
        assert 0 <= a <= Ji and legal[a], where           # a legal action, never an illegal one
        best = scores.max()
        assert scores[a] >= best - 1e-4 * (1.0 + abs(best)), where
        assert abs(lp - lp_ref) <= 1e-5 * (1.0 + abs(lp_ref)), where
        decisions += 1
        agree += a == a_ref
    return twin, decisions, agree


def check_step_logits(make_env, names, n_steps, seed, pad=3, state_every=25, auto_reset=True, make_logits=None):
    """jss_step_logits on a batch, driven by seeded random logits (with -inf entries, huge values on illegal entries,
    ld > J+1; or `make_logits(rng, env, mask, ld, k)` at step k): every draw against the oracle, and a twin env
    stepped with jss_step(actions) bit-identical after every step (the env of a bad-logits draw gets an out-of-range
    action there, which sets the same error bit)."""
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=seed, auto_reset=auto_reset)
    rng = np.random.default_rng(seed)
    ld = a_env.jobs + 1 + pad
    decisions = agree = 0
    for k in range(n_steps):
        mask, done = np_(a_env.action_mask).copy(), np_(a_env.done).copy()
        if make_logits is None:
            logits = random_logits(rng, a_env, mask, ld, illegal=np.nan if k % 2 else 1e30)
        else:
            logits = make_logits(rng, a_env, mask, ld, k)
        _, _, _, _, info = a_env.step_logits(_to_dev(a_env, logits))
        acts, logp = np_(info["actions"]).copy(), np_(info["log_prob"]).copy()
        twin, d, g = check_draws(a_env, logits, mask, done, acts, logp, k, np_(a_env.flags), f"step {k}")
        decisions += d; agree += g
        b_env.step(twin)
        full = k % state_every == state_every - 1
        assert_twins_equal(a_env, b_env, f"step {k}", state=full, stats=full)
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)
    assert decisions > 0 and agree >= 0.999 * decisions, (agree, decisions)
    return a_env


def check_step_logits_edge_cases(make_env):
    """One finite legal logit among -inf, NaN / +inf / all -inf on legal entries, +1e30 on illegal entries and in the
    padding columns, only the no-op legal, done envs (frozen and auto-reset)."""
    for auto_reset in (False, True):
        n = 8
        a_env = make_env(n, {"instance_path": "ta01"}, seed=5, auto_reset=auto_reset)
        b_env = make_env(n, {"instance_path": "ta01"}, seed=5, auto_reset=auto_reset)
        J = a_env.jobs
        a_env.reset(); b_env.reset()
        first = np.zeros(n, np.int32)                     # every env allocates job 0: one machine busy
        a_env.step(first); b_env.step(first)
        # env 6: only the no-op legal; env 7: done -- crafted through the snapshot interface on both twins
        for env in (a_env, b_env):
            x = env.export_state()
            x["legal"][6] = 0
            x["legal"][7] = 0                             # a done env has no legal job
            x["flags"][6] = int(x["flags"][6]) | (N.FLAG_NOOP_LEGAL << 8)
            x["flags"][7] = int(x["flags"][7]) | (N.FLAG_DONE << 8) | 1
            env.import_state(x)
        mask = np_(a_env.action_mask).copy()
        assert not mask[6, :J].any() and mask[6, J] and not mask[7].any() and not mask[0, 0]
        before = {k: np_(v).copy() for k, v in a_env.export_state().items()}
        obs0, mask0 = np_(a_env.real_obs).copy(), mask.copy()
        rng = np.random.default_rng(1)
        ld = J + 1 + 5
        logits = rng.standard_normal((n, ld)).astype(np.float32)
        logits[:, J + 1:] = 1e30                          # padding columns: never read
        logits[~np.pad(mask[:, : J + 1], ((0, 0), (0, ld - J - 1)))] = 1e30   # illegal entries: never chosen
        logits[0, :J] = -np.inf; logits[0, 3] = 0.7       # one finite legal logit among -inf
        logits[1, 2] = np.nan                             # NaN on a legal entry
        logits[2, 5] = np.inf                             # +inf on a legal entry
        logits[3, 1:J] = -np.inf                          # every legal logit -inf (job 0 is running)
        logits[6, J] = np.nan                             # the only legal action's logit is not read
        twin = np.array([3, BIG_ACTION, BIG_ACTION, BIG_ACTION, 0, 0, J, 0], np.int32)
        _, _, _, _, info = a_env.step_logits(_to_dev(a_env, logits))
        acts, logp = np_(info["actions"]).copy(), np_(info["log_prob"]).copy()
        twin[4], twin[5] = acts[4], acts[5]
        b_env.step(twin)
        ctx = f"auto_reset={auto_reset}"
        assert acts[0] == 3 and logp[0] == 0.0, (ctx, acts[0], logp[0])
        flags = np_(a_env.flags)
        for i in (1, 2, 3):
            assert acts[i] == N.ACTION_SKIP and np.isnan(logp[i]) and flags[i] & N.FLAG_ERROR, (ctx, i)
        for i in (4, 5):
            assert 1 <= acts[i] < J and mask[i, acts[i]], (ctx, i, acts[i])
        assert acts[6] == J and logp[6] == 0.0 and acts[7] == 0 and logp[7] == 0.0, (ctx, acts, logp)
        twin_check, _, _ = check_draws(a_env, logits, mask, np_(before["flags"]) & 1, acts, logp, 0, flags, ctx)
        assert np.array_equal(twin_check[[0, 4, 5, 6, 7]], twin[[0, 4, 5, 6, 7]])
        after = {k: np_(v).copy() for k, v in a_env.export_state().items()}
        for k in before:                                  # the erroring envs are unchanged
            if k != "flags":
                assert np.array_equal(before[k][1:4], after[k][1:4]), (ctx, k)
        assert np.array_equal(np_(a_env.real_obs)[1:4], obs0[1:4]) and np.array_equal(np_(a_env.action_mask)[1:4], mask0[1:4])
        if auto_reset:                                    # the done env was reset by the call
            assert int(a_env.current_time_step[7]) == 0 and np_(a_env.action_mask)[7, :J].all()
        else:                                             # ... or stays frozen
            assert np.array_equal(after["todo"][7], before["todo"][7]) and np_(a_env.done)[7]
        assert_twins_equal(a_env, b_env, ctx, state=True, stats=True)


def check_step_logits_shards(make_env, n_total=12, n_steps=120, seed=31):
    """Shards created with env_id_base != 0 reproduce the unsharded batch's actions and log_probs bit for bit, and its
    outputs, transition for transition."""
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
    ld = whole.jobs + 1
    for k in range(n_steps):
        logits = random_logits(rng, whole, np_(whole.action_mask), ld)
        dev = _to_dev(whole, logits)
        _, _, _, _, iw = whole.step_logits(dev)
        aw, lw = np_(iw["actions"]).copy(), np_(iw["log_prob"]).copy()
        for s, lo, hi in zip(shards, cuts[:-1], cuts[1:]):
            _, _, _, _, i_s = s.step_logits(dev[lo:hi, : s.jobs + 1])   # row stride of the whole batch passed through as ld
            assert np.array_equal(np_(i_s["actions"]), aw[lo:hi]), (k, lo)
            assert np.array_equal(np_(i_s["log_prob"]).view(np.uint32), lw[lo:hi].view(np.uint32)), (k, lo)
            assert_twins_equal(s, whole, k, rows=slice(lo, hi))
            m_s = np_(s.action_mask)
            assert np.array_equal(m_s, np_(whole.action_mask)[lo:hi, : s.jobs + 1]), k


def check_step_logits_abi_errors(make_env):
    """jss_step_logits returns JSS_ERR_INVALID for a NULL logits or actions_out pointer and for ld < jobs_max + 1;
    step_logits rejects logits of the wrong shape."""
    import ctypes

    import pytest
    import torch
    env = make_env(3, {"instance_paths": ["ta01", "ta31"], "env_to_instance": [0, 1, 0]})
    J = env.jobs
    logits = torch.zeros((3, J + 1), dtype=torch.float32, device=env.device)
    acts = torch.zeros(3, dtype=torch.int32, device=env.device)
    p_l, p_a, st = ctypes.c_void_p(logits.data_ptr()), ctypes.c_void_p(acts.data_ptr()), env._stream()
    L, h = env._L, env._h
    assert L.jss_step_logits(h, None, J + 1, 0, 0, p_a, None, st) == -1
    assert L.jss_step_logits(h, p_l, J + 1, 0, 0, None, None, st) == -1
    assert L.jss_step_logits(h, p_l, J, 0, 0, p_a, None, st) == -1
    assert b"jss_step_logits" in L.jss_last_error(h)
    assert L.jss_step_logits(h, p_l, J + 1, 0, 0, p_a, None, st) == 0   # log_prob_out may be NULL
    env.synchronize()
    assert (np_(acts) >= 0).all()
    with pytest.raises(ValueError):
        env.step_logits(logits[:, :J])
    with pytest.raises(ValueError):
        env.step_logits(logits[:2])
