"""The tests of jss_lookahead (every legal action valued by a dispatching-rule rollout to the end of the episode, the envs
left untouched), declared once for both backends (tests/backends.py) and collected by tests/test_emu_lookahead.py and
tests/test_gpu_lookahead.py.  A table is checked against its definition on a twin batch: the same state imported, the
candidate stepped, then the rule (policy + step, or jss_rollout under the device coin) until done; and against the CPU
oracle's replay."""
import ctypes

import numpy as np

from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv
from tests.backends import native_test
from tests.parity_common import _coin_uniform, assert_twins_equal, batch_cfg, np_, synthetic_instance

RULES = ("RANDOM", "SPT", "FIFO", "MWR", "LWR", "MOR", "LOR", "CR")
NONPERM = synthetic_instance(37, 5, 8, max_dur=30, permutation=False)
SMALL = synthetic_instance(9, 4, 21, max_dur=20)
TINY = synthetic_instance(6, 3, 22, max_dur=15)
BIG_GPU = synthetic_instance(200, 8, 9, max_dur=50)
# emulation: short episodes in the lane classes with 33..64, 65..128 and 129..256 jobs
EMU_CLASSES = [synthetic_instance(40, 3, 10, max_dur=30), synthetic_instance(70, 3, 11, max_dur=30),
               synthetic_instance(130, 2, 12, max_dur=30)]


def snapshot(env):
    return {k: v.clone() for k, v in env.export_state().items()}


def random_walk(env, k):
    """k steps of the device's masked-uniform sampler (a done env gets 0 and stays frozen without auto-reset).  Returns
    the actions taken, [k][N]."""
    taken = []
    for _ in range(k):
        acts = env.policy("RANDOM")
        taken.append(np_(acts).copy())
        env.step(acts)
    return taken


def twin_table(make_env, env, rule, coin, step_index, cr=None):
    """The table jss_lookahead must return for env's current state, computed on a twin batch by its definition."""
    import torch
    n, J, M = env.num_envs, env.jobs, env.machines
    cfg = {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    twin = make_env(n, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed)
    twin.reset()
    if cr is not None:
        twin.set_cr_due_date_factor(cr)
    snap = snapshot(env)
    legal = np_(env.action_mask)[:, :J + 1].astype(bool) & ~np_(env.done)[:, None]
    bound = 2 * J * M + 1
    out = np.full((n, J + 1), -1, np.int64)
    for a in range(J + 1):
        cand = legal[:, a]
        if not cand.any():
            continue
        twin.import_state(snap)
        twin.step(torch.full((n,), a, dtype=torch.int32, device=env.device))
        if coin == "device":
            twin._step_index = step_index
            twin.rollout(rule, bound, write_obs=False)
        else:
            for d in range(bound):
                if np_(twin.done)[cand].all():
                    break
                twin.step(twin.policy(rule, coin=coin, step_index=step_index + d))
        done, t = np_(twin.done), np_(twin.current_time_step)
        out[cand & done, a] = t[cand & done]
    return out


def check_table(env, q, want, ctx):
    q = np_(q)
    for i, Ji in enumerate(env.env_jobs):
        assert np.array_equal(q[i, :Ji + 1], want[i, :Ji + 1]), (ctx, i, q[i, :Ji + 1], want[i, :Ji + 1])


def check_twin(make_env, names, rule, coin, k, seed, cr=None):
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=5)
    env.reset()
    if cr is not None:
        env.set_cr_due_date_factor(cr)
    random_walk(env, k)
    si = env._step_index
    q = env.lookahead(rule, coin)
    assert env._step_index == si + 2 * env.jobs * env.machines + 1
    check_table(env, q, twin_table(make_env, env, rule, coin, si, cr), (rule, coin, k))
    return env, q


@native_test(emu=[(r, c) for r in RULES for c in ("never", "device")],
             gpu=[(r, c) for r in RULES for c in ("never", "device")])
def lookahead_twin_rules(make_env, backend, rule, coin):
    """Every rule under both coins, at reset and mid-episode (some envs done, some with only the no-op legal)."""
    names = {"emu": ["ta01", SMALL, SMALL, NONPERM], "gpu": ["ta01", "ta11", SMALL, NONPERM] * 3}[backend]
    k = {"emu": 120, "gpu": 150}[backend]
    check_twin(make_env, [SMALL, SMALL, SMALL], rule, coin, 0, seed=3)
    check_twin(make_env, names, rule, coin, k, seed=4)
    if rule == "CR":
        check_twin(make_env, names, rule, coin, k, seed=5, cr=0.8)


@native_test()
def lookahead_twin_mixed_batch(make_env, backend):
    """Every lane class in one batch, with MWR under the device coin."""
    if backend == "emu":
        names = ["ta01", SMALL, *EMU_CLASSES, NONPERM]
        check_twin(make_env, names, "MWR", "device", 170, seed=6)
    else:
        names = ["ta01", "ta11", "ta21", "ta31", "ta41", "ta51", "ta61", "ta71", "ta80", NONPERM, BIG_GPU] * 2
        check_twin(make_env, names, "MWR", "device", 400, seed=6)


def _outputs(env):
    x = {k: np_(getattr(env, k)).copy() for k in ("real_obs", "action_mask", "reward", "reward_raw", "done",
                                                  "current_time_step", "flags", "episode_count", "last_makespan",
                                                  "last_return")}
    x.update({"x_" + k: np_(v).copy() for k, v in env.export_state().items()})
    if env.solution is not None:
        x["solution"] = np_(env.solution).copy()
    return x


@native_test(emu=[False, True], gpu=[False, True])
def lookahead_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and the counters are bit-identical after the call; one launch
    per lane class present; after a recording step the call leaves real_obs stale for refresh_obs()."""
    import torch
    names = ["ta01", NONPERM, "ta01", SMALL] if backend == "emu" else ["ta01", "ta51", "ta80", NONPERM] * 8
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, record_solution=True, seed=8)
    env.reset()
    random_walk(env, 60)
    before, stats = _outputs(env), env.stats()
    c = env.launch_count
    for rule in ("MWR", "RANDOM"):
        env.lookahead(rule, "device")
    assert env.launch_count == c + 2 * (2 if backend == "emu" else 3)   # one launch per lane class present
    after = _outputs(env)
    for k, v in before.items():
        assert np.array_equal(v, after[k]), k
    assert env.stats() == stats
    # a recording step leaves real_obs stale: the call neither reads nor refreshes it
    cfg = batch_cfg(names, sort=False)
    a_env, b_env = (make_env(len(names), cfg, auto_reset=auto_reset, seed=9) for _ in range(2))
    a_env.reset(); b_env.reset()
    scores = torch.zeros((a_env.num_envs, a_env.jobs + 1), device=a_env.device)
    traj = a_env.logits_trajectory(1)
    stale = np_(a_env.real_obs).copy()
    a_env.step_greedy_record(scores, traj, 0)
    b_env.step_greedy(scores)
    qa, qb = a_env.lookahead("LWR"), b_env.lookahead("LWR")
    assert np.array_equal(np_(qa), np_(qb))
    assert np.array_equal(np_(a_env.real_obs), stale)
    a_env.refresh_obs()
    assert_twins_equal(a_env, b_env, "refreshed", state=True, stats=True)


@native_test()
def lookahead_padded_layout(make_env, backend):
    """With ld > J+1 and the padding poisoned, only columns 0..J_i are written."""
    import torch
    names = ["ta01", SMALL, NONPERM]
    env = make_env(len(names), batch_cfg(names, sort=False), seed=10)
    env.reset()
    random_walk(env, 30)
    J = env.jobs
    want = np_(env.lookahead("SPT", "never")).copy()
    out = torch.full((env.num_envs, J + 6), -777, dtype=torch.int32, device=env.device)
    env.lookahead("SPT", "never", out=out)
    o = np_(out)
    for i, Ji in enumerate(env.env_jobs):
        assert np.array_equal(o[i, :Ji + 1], want[i, :Ji + 1]), i
        assert (o[i, Ji + 1:] == -777).all(), i
        assert (want[i, Ji + 1:] == -1).all(), i             # the default table is filled with -1


def oracle_value(inst, prefix, a, rule, coin, seed, env_id, step_index):
    """The oracle's makespan after replaying `prefix`, taking `a` and then `rule` to the end (-1 if not done)."""
    o = OracleEnv(*(load_instance(inst) if isinstance(inst, str) else inst))
    o.reset()
    for x in prefix:
        o.step(int(x))
    _, _, done, _, _ = o.step(a)
    d = 0
    while not done:
        if rule == "RANDOM":
            act = o.masked_random_action(seed, env_id, step_index + d)
        else:
            act, _ = o.rule_action(rule, _coin_uniform(seed, env_id, step_index + d) if coin == "device" else 1.0)
        _, _, done, _, _ = o.step(act)
        d += 1
    return o.current_time_step


@native_test(emu=[("MWR", "never"), ("RANDOM", "device"), ("CR", "device")],
             gpu=[(r, c) for r in ("MWR", "RANDOM", "CR", "SPT") for c in ("never", "device")])
def lookahead_oracle(make_env, backend, rule, coin):
    """ta01 and a non-permutation instance mid-episode: every legal column equals the oracle's replay."""
    names = ["ta01", NONPERM, "ta01", NONPERM]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=11)
    env.reset()
    taken = random_walk(env, 60)
    si = env._step_index
    q, mask, done = np_(env.lookahead(rule, coin)), np_(env.action_mask), np_(env.done)
    for i, inst in enumerate(names):
        if done[i]:
            continue
        Ji = env.env_jobs[i]
        for a in np.flatnonzero(mask[i, :Ji + 1]):
            want = oracle_value(inst, [t[i] for t in taken], int(a), rule, coin, env.seed, i, si)
            assert q[i, a] == want, (rule, coin, i, a)


def _rule_makespan(make_env, env, rule):
    twin = make_env(env.num_envs, {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
                                   "env_to_instance": list(env.env_to_instance)}, auto_reset=False)
    twin.reset()
    for _ in range(2 * env.jobs * env.machines + 1):
        if np_(twin.done).all():
            break
        twin.step(twin.policy(rule, coin="never"))
    return np_(twin.current_time_step).copy()


@native_test(emu=["MWR", "SPT"], gpu=list(RULES[1:]))
def lookahead_rollout_improvement(make_env, backend, rule):
    """The rollout method (argmin of the table, ties to the lowest index, coin "never"): the per-env minimum never
    increases, the final makespan equals the last minimum and is at most the rule's own makespan."""
    import torch
    names = {"emu": [SMALL, SMALL, TINY], "gpu": ["ta01", "ta21", SMALL, NONPERM] * 4}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False)
    env.reset()
    base = _rule_makespan(make_env, env, rule)
    big = np.iinfo(np.int32).max
    last = np.full(env.num_envs, big, np.int64)
    for _ in range(2 * env.jobs * env.machines + 1):
        done = np_(env.done)
        if done.all():
            break
        q = env.lookahead(rule, "never")
        qn = np_(q).astype(np.int64)
        mins = np.where(qn >= 0, qn, big).min(1)
        alive = ~done
        assert (mins[alive] < big).all()
        assert (mins[alive] <= last[alive]).all(), rule
        last[alive] = mins[alive]
        env.step(q.where(q >= 0, torch.full_like(q, big)).argmin(1).to(torch.int32))
    assert np_(env.done).all()
    ms = np_(env.current_time_step)
    assert np.array_equal(ms, last), rule
    assert (ms <= base).all(), (rule, ms, base)


@native_test()
def lookahead_split_invariance(make_env, backend):
    """The same envs, ids and states give the same tables in a batch of 3 (one tile, so its candidates are split over
    several work items: S = 2 on the emulated two-SM device) and in a large batch (S = 1: the tiles fill the SMs)."""
    n_big = {"emu": 24, "gpu": 4096}[backend]
    big = make_env(n_big, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    big.reset()
    random_walk(big, 40)
    snap = snapshot(big)
    small = make_env(3, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    small.reset()
    small.import_state({k: v[:3] for k, v in snap.items()})
    small._step_index = big._step_index                  # the same RNG counters
    for rule, coin in (("RANDOM", "device"), ("MWR", "device"), ("LOR", "never")):
        qb, qs = np_(big.lookahead(rule, coin)), np_(small.lookahead(rule, coin))
        assert np.array_equal(qb[:3], qs), (rule, coin)


@native_test()
def lookahead_abi(make_env, backend):
    """JSS_ERR_INVALID for a bad rule or coin, a NULL or misaligned table and ld < jobs_max + 1; JSS_ERR_STATE before
    jss_assign; a bad rule name, coin or out raises ValueError before the native call."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    J = env.jobs
    out = torch.zeros((2, J + 1), dtype=torch.int32, device=env.device)
    L, h, st, p = env._L, env._h, env._stream(), out.data_ptr()
    for args in ((-1, 0, p, J + 1), (8, 0, p, J + 1), (3, 2, p, J + 1), (3, -1, p, J + 1), (3, 0, None, J + 1),
                 (3, 0, p + 2, J + 1), (3, 0, p, J)):
        rule, coin, ptr, ld = args
        assert L.jss_lookahead(h, rule, coin, 0, 0, ptr, ld, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_lookahead:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_lookahead(raw, 3, 0, 0, 0, p, J + 1, st) == -5
    L.jss_destroy(raw)
    si = env._step_index
    for kw in ({"rule": "BOGUS"}, {"coin": "sometimes"}, {"out": out[:, :J]}, {"out": out.to(torch.int64)},
               {"out": torch.zeros((3, J + 1), dtype=torch.int32, device=env.device)},
               {"out": torch.zeros((J + 1, 2), dtype=torch.int32, device=env.device).t()}):
        with pytest.raises(ValueError):
            env.lookahead(**kw)
    assert env._step_index == si


@native_test(emu=None)
def lookahead_full_size_ta80(make_env):
    """ta80 at N = 4 096 mid-episode: no -1 on a legal column, five sampled envs equal to the oracle."""
    n = 4096
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=14)
    env.reset()
    taken = random_walk(env, 500)
    si = env._step_index
    q, mask = np_(env.lookahead("MWR", "device")), np_(env.action_mask)[:, :env.jobs + 1].astype(bool)
    assert (q[mask] >= 0).all()
    assert (q[~mask] == -1).all()
    for i in np.random.default_rng(14).choice(n, 5, replace=False):
        for a in np.flatnonzero(mask[i])[:4]:
            want = oracle_value("ta80", [t[i] for t in taken], int(a), "MWR", "device", env.seed, int(i), si)
            assert q[i, a] == want, (i, a)
