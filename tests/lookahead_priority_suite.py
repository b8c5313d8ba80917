"""The tests of jss_lookahead_priority (every legal action valued by a greedy rollout of a caller's priority table to the
end of the episode, the envs left untouched), declared once for both backends (tests/backends.py) and collected by
tests/test_emu_lookahead_priority.py and tests/test_gpu_lookahead_priority.py.  A table of values is checked against its
definition on a twin batch: the same state imported, the candidate stepped, then rollout_priority(table) to the end;
against lookahead(rule, "never") for the built-in rules written as tables; and against the CPU oracle's replay."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv
from tests import logits_common as lc
from tests.backends import native_test
from tests.lookahead_suite import _outputs, check_table, random_walk, snapshot
from tests.parity_common import assert_twins_equal, batch_cfg, np_, synthetic_instance
from tests.priority_suite import _rule_tables, random_table

NONPERM = synthetic_instance(37, 5, 8, max_dur=30, permutation=False)
SMALL = synthetic_instance(9, 4, 21, max_dur=20)
TINY = synthetic_instance(6, 3, 22, max_dur=15)
BIG_GPU = synthetic_instance(200, 8, 9, max_dur=50)
# emulation: short episodes in the lane classes with 33..64, 65..128 and 129..256 jobs
EMU_CLASSES = [synthetic_instance(40, 3, 10, max_dur=30), synthetic_instance(70, 3, 11, max_dur=30),
               synthetic_instance(130, 2, 12, max_dur=30)]
SHAPES = ("NJM", "NJ1", "1JM")


def shaped_table(env, seed, ties, shape):
    """random_table(env, seed, ties) cut to (N, J, M), (N, J, 1) or (1, J, M)."""
    t = random_table(env, seed, ties)
    return {"NJM": t, "NJ1": t[:, :, :1], "1JM": t[:1]}[shape]


def twin_values(make_env, env, table):
    """The values lookahead_priority(table) must return in env's current state, by their definition on a twin batch:
    for each candidate column, import the state, step the candidate, run rollout_priority(table) to the end, and read
    the end time of the envs that are done (-1 for the others)."""
    import torch
    n, J = env.num_envs, env.jobs
    cfg = {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    twin = make_env(n, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed)
    twin.reset()
    snap = snapshot(env)
    table = lc._to_dev(twin, table)
    legal = np_(env.action_mask)[:, :J + 1].astype(bool) & ~np_(env.done)[:, None]
    out = np.full((n, J + 1), -1, np.int64)
    for a in range(J + 1):
        cand = legal[:, a]
        if not cand.any():
            continue
        twin.import_state(snap)
        twin.step(torch.full((n,), a, dtype=torch.int32, device=env.device))
        twin.rollout_priority(table)
        done, t = np_(twin.done), np_(twin.current_time_step)
        out[cand & done, a] = t[cand & done]
    return out


def values(env, table, **kw):
    """lookahead_priority of a host table; the RNG counter must not move."""
    si = env._step_index
    q = env.lookahead_priority(lc._to_dev(env, table), **kw)
    assert env._step_index == si
    return q


def noop_only(env):
    """The envs whose only legal action is the no-op."""
    mask = np_(env.action_mask)
    return np.array([not mask[i, :Ji].any() and bool(mask[i, Ji]) for i, Ji in enumerate(env.env_jobs)])


def check_twin(make_env, names, table_of, k, seed, craft_noop=False):
    """Values after k random decisions against the twin's, for the table table_of(env).  With craft_noop, the first env
    that is not done is first given only the no-op as legal action, through the snapshot interface (a random walk from
    reset does not reach such a state)."""
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=5)
    env.reset()
    random_walk(env, k)
    if craft_noop:
        i = int(np.flatnonzero(~np_(env.done))[0])
        x = env.export_state()
        x["legal"][i] = 0
        x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
        env.import_state(x)
    table = table_of(env)
    check_table(env, values(env, table), twin_values(make_env, env, table), (k, table.shape))
    return env


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def lookahead_priority_twin(make_env, backend, shape, ties):
    """Every lane class in one batch (129..256 jobs and a non-permutation instance included) at reset and mid-episode,
    with some envs done and some with only the no-op legal; and uniform tiny batches (J <= 4)."""
    if backend == "emu":
        names, k = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170
    else:
        names, k = ["ta01", "ta11", "ta21", "ta31", "ta41", "ta51", "ta61", "ta71", "ta80", NONPERM, BIG_GPU, SMALL,
                    TINY] * 2, 400
    seed = SHAPES.index(shape) + (10 if ties else 0)
    table_of = lambda env: shaped_table(env, seed, ties, shape)  # noqa: E731
    check_twin(make_env, names, table_of, 0, seed)
    env = check_twin(make_env, names, table_of, k, seed, craft_noop=True)
    done = np_(env.done)
    assert done.any() and not done.all() and noop_only(env).any(), done
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        check_twin(make_env, [synthetic_instance(J, M, J * 10 + M)] * 3, table_of, J, seed)


@native_test()
def lookahead_priority_builtin_rules(make_env, backend):
    """The SPT, MWR, LWR, MOR and LOR tables give values bit-identical to lookahead(rule, "never"), on mixed batches at
    reset and mid-episode, and on ta80."""
    batches = {"emu": [(["ta01", SMALL, "ta11", NONPERM, EMU_CLASSES[0]], 0), (["ta01", SMALL, "ta11", NONPERM], 60)],
               "gpu": [(["ta01", "ta21", "ta41", "ta80", NONPERM, BIG_GPU] * 4, 0),
                       (["ta01", "ta21", "ta41", "ta80", NONPERM, BIG_GPU, SMALL] * 4, 300),
                       (["ta80"] * 256, 700)]}[backend]
    for names, k in batches:
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=2)
        env.reset()
        random_walk(env, k)
        for rule, table in _rule_tables(env).items():
            want = np_(env.lookahead(rule, "never")).copy()
            got = np_(values(env, table)).copy()
            assert np.array_equal(got, want), (rule, k)
            assert (got >= 0).any()


@native_test()
def lookahead_priority_bad_tables(make_env, backend):
    """NaN, +inf and all-(-inf) entries on operations some rollouts reach: exactly the affected candidates read -1, the
    rest equal the twin and the clean table's values, no flag changes and the call returns normally.  Entries that are
    never read (finished operations, columns past J_i, operations past M_i) change nothing."""
    names = ["ta01", "ta01", "ta01", "ta01", SMALL, "ta01", "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
    env.reset()
    random_walk(env, 40 if backend == "emu" else 60)
    x = env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    mask = np_(env.action_mask)[:, :env.jobs + 1].astype(bool) & ~np_(env.done)[:, None]
    clean = random_table(env, 31)
    bad = clean.copy()
    jobs = {i: int(np.flatnonzero(legal[i])[0]) for i in (0, 1)}
    bad[0, jobs[0], todo[0, jobs[0]]] = np.nan            # a legal job's current operation
    bad[1, jobs[1], todo[1, jobs[1]]] = np.inf
    bad[2] = -np.inf                                      # every legal job at -inf at the first decision
    for j in range(env.jobs):                             # every job's current operation -inf, the rest finite
        bad[3, j, min(todo[3, j], env.machines - 1)] = -np.inf
    bad[4, 9:, :] = np.nan                                # columns past J_i = 9
    bad[4, :, 4:] = np.inf                                # operations past M_i = 4
    ops = np.arange(env.machines)
    bad[5][ops[None, :] < todo[5][:, None]] = np.nan      # finished operations
    flags = np_(env.flags).copy()
    q = np_(values(env, bad)).copy()
    assert np.array_equal(np_(env.flags), flags)
    assert not (flags & N.FLAG_ERROR).any()
    check_table(env, q, twin_values(make_env, env, bad), "bad")
    ok = np_(values(env, clean)).copy()
    assert (ok[mask] >= 0).all()
    for i in (0, 1):                                      # only the candidate that takes the bad job skips its entry
        cols = np.flatnonzero(mask[i])
        assert q[i, jobs[i]] == ok[i, jobs[i]], i
        assert (q[i, cols[cols != jobs[i]]] == -1).all(), i
    assert (q[2][mask[2]] == -1).all()
    assert (q[3][mask[3]] == -1).any()
    for i in (4, 5, 6):
        assert np.array_equal(q[i], ok[i]), i


@native_test(emu=[False, True], gpu=[False, True])
def lookahead_priority_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and the counters are bit-identical after the call; one launch
    per lane class present; after a recording step the call leaves real_obs stale for refresh_obs()."""
    import torch
    names = ["ta01", NONPERM, "ta01", SMALL] if backend == "emu" else ["ta01", "ta51", "ta80", NONPERM] * 8
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, record_solution=True, seed=8)
    env.reset()
    random_walk(env, 60)
    before, stats = _outputs(env), env.stats()
    c = env.launch_count
    for table in (random_table(env, 4), random_table(env, 5, ties=True)[:1]):
        values(env, table)
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
    table = random_table(a_env, 6)
    qa, qb = values(a_env, table), values(b_env, table)
    assert np.array_equal(np_(qa), np_(qb))
    assert np.array_equal(np_(a_env.real_obs), stale)
    a_env.refresh_obs()
    assert_twins_equal(a_env, b_env, "refreshed", state=True, stats=True)


@native_test()
def lookahead_priority_padded_layout(make_env, backend):
    """With ld > J+1 and the padding poisoned, only columns 0..J_i are written."""
    import torch
    names = ["ta01", SMALL, NONPERM]
    env = make_env(len(names), batch_cfg(names, sort=False), seed=10)
    env.reset()
    random_walk(env, 30)
    J = env.jobs
    table = random_table(env, 7)
    want = np_(values(env, table)).copy()
    out = torch.full((env.num_envs, J + 6), -777, dtype=torch.int32, device=env.device)
    assert values(env, table, out=out) is out
    o = np_(out)
    for i, Ji in enumerate(env.env_jobs):
        assert np.array_equal(o[i, :Ji + 1], want[i, :Ji + 1]), i
        assert (o[i, Ji + 1:] == -777).all(), i
        assert (want[i, Ji + 1:] == -1).all(), i             # the default table is filled with -1


@native_test()
def lookahead_priority_split_invariance(make_env, backend):
    """The same envs and states give the same values in a batch of 3 (one tile, so its candidates are split over
    several work items) and in a large batch (S = 1: the tiles fill the SMs), per-env and broadcast tables alike."""
    n_big = {"emu": 24, "gpu": 4096}[backend]
    big = make_env(n_big, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    big.reset()
    random_walk(big, 40)
    snap = snapshot(big)
    small = make_env(3, {"instance_path": "ta01"}, auto_reset=False, seed=99)   # the seed does not matter
    small.reset()
    small.import_state({k: v[:3] for k, v in snap.items()})
    full, ties = random_table(big, 13), random_table(big, 14, ties=True)
    for tb, ts in ((full, full[:3]), (ties[:1], ties[:1])):
        qb, qs = np_(values(big, tb)), np_(values(small, ts))
        assert np.array_equal(qb[:3], qs), tb.shape
        assert (qs >= 0).any()


def _priority_makespan(make_env, env, table):
    twin = make_env(env.num_envs, {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
                                   "env_to_instance": list(env.env_to_instance)}, auto_reset=False)
    twin.reset()
    twin.rollout_priority(lc._to_dev(twin, table))
    assert np_(twin.done).all()
    return np_(twin.current_time_step).copy()


@native_test(emu=[False, True], gpu=[False, True])
def lookahead_priority_rollout_improvement(make_env, backend, ties):
    """The rollout method over the table (argmin of the values, ties to the lowest index): the per-env minimum never
    increases, the final makespan equals the last minimum and is at most the table's own greedy makespan."""
    import torch
    names = {"emu": [SMALL, SMALL, TINY, NONPERM], "gpu": ["ta01", "ta21", SMALL, NONPERM] * 4}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False)
    env.reset()
    table = random_table(env, 15, ties)
    base = _priority_makespan(make_env, env, table)
    big = np.iinfo(np.int32).max
    last = np.full(env.num_envs, big, np.int64)
    for _ in range(2 * env.jobs * env.machines + 1):
        done = np_(env.done)
        if done.all():
            break
        q = values(env, table)
        qn = np_(q).astype(np.int64)
        mins = np.where(qn >= 0, qn, big).min(1)
        alive = ~done
        assert (mins[alive] < big).all()
        assert (mins[alive] <= last[alive]).all()
        last[alive] = mins[alive]
        env.step(q.where(q >= 0, torch.full_like(q, big)).argmin(1).to(torch.int32))
    assert np_(env.done).all()
    ms = np_(env.current_time_step)
    assert np.array_equal(ms, last)
    assert (ms <= base).all(), (ms, base)


def oracle_value(inst, prefix, a, table):
    """The oracle's makespan after replaying `prefix`, taking `a` and then the table's argmax over the legal jobs'
    current operations (the no-op when no job is legal) to the end."""
    o = OracleEnv(*(load_instance(inst) if isinstance(inst, str) else inst))
    o.reset()
    for x in prefix:
        o.step(int(x))
    _, _, done, _, _ = o.step(a)
    while not done:
        legal = np.asarray(o.get_legal_actions(), bool)
        jobs = np.flatnonzero(legal[:-1])
        act = int(jobs[np.argmax(table[jobs, np.asarray(o.todo_time_step_job)[jobs]])]) if len(jobs) else o.jobs
        _, _, done, _, _ = o.step(act)
    return o.current_time_step


def check_oracle(env, names, table, taken, envs, cols=None):
    q, mask, done = np_(values(env, table)), np_(env.action_mask), np_(env.done)
    full = np.broadcast_to(table, (env.num_envs, env.jobs, env.machines))
    for i in envs:
        if done[i]:
            continue
        Ji, Mi = (load_instance(names[i]) if isinstance(names[i], str) else names[i])[0].shape
        for a in np.flatnonzero(mask[i, :Ji + 1])[:cols]:
            want = oracle_value(names[i], [t[i] for t in taken], int(a), full[i, :Ji, :Mi])
            assert q[i, a] == want, (i, a)


@native_test(emu=[False, True], gpu=[False, True])
def lookahead_priority_oracle(make_env, backend, ties):
    """ta01 and a non-permutation instance mid-episode: every legal column equals the oracle's replay."""
    names = ["ta01", NONPERM, "ta01", NONPERM]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=11)
    env.reset()
    taken = random_walk(env, 60)
    check_oracle(env, names, random_table(env, 16, ties), taken, range(len(names)))


@native_test()
def lookahead_priority_abi(make_env, backend):
    """JSS_ERR_INVALID for a NULL or misaligned table or values, a negative stride and ld < jobs_max + 1; JSS_ERR_STATE
    before jss_assign; a bad table shape or out raises ValueError before the native call; a table that requires grad is
    read detached."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    out = torch.zeros((n, J + 1), dtype=torch.int32, device=env.device)
    L, h, st, p, o = env._L, env._h, env._stream(), t.data_ptr(), out.data_ptr()
    s = (J * M, M, 1)
    for args in ((None, *s, o, J + 1), (p + 2, *s, o, J + 1), (p, -1, M, 1, o, J + 1), (p, J * M, -M, 1, o, J + 1),
                 (p, J * M, M, -1, o, J + 1), (p, *s, None, J + 1), (p, *s, o + 2, J + 1), (p, *s, o, J)):
        assert L.jss_lookahead_priority(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_lookahead_priority:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_lookahead_priority(raw, p, *s, o, J + 1, st) == -5
    L.jss_destroy(raw)
    si = env._step_index
    for bad in (t[0], t[None], t[:, :J - 1], torch.zeros((3, J, M), device=env.device), t[:, :, :M - 1]):
        with pytest.raises(ValueError):
            env.lookahead_priority(bad)
    for bad_out in (out[:, :J], out.to(torch.int64), torch.zeros((3, J + 1), dtype=torch.int32, device=env.device),
                    torch.zeros((J + 1, 2), dtype=torch.int32, device=env.device).t()):
        with pytest.raises(ValueError):
            env.lookahead_priority(t, out=bad_out)
    assert env._step_index == si
    table = lc._to_dev(env, random_table(env, 17))
    want = np_(env.lookahead_priority(table)).copy()
    g = table.double().requires_grad_(True)
    assert np.array_equal(np_(env.lookahead_priority(g)), want)
    assert g.grad is None
    assert env._step_index == si


@native_test(emu=None)
def lookahead_priority_full_size_ta80(make_env):
    """ta80 at N = 4 096 after 500 random decisions with a finite random table: no -1 on a legal column, -1 on every
    illegal one, a few sampled envs equal to the oracle."""
    import torch
    n = 4096
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=14)
    env.reset()
    taken = random_walk(env, 500)
    table = torch.rand((n, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(22),
                       device=env.device)
    q, mask = np_(env.lookahead_priority(table)), np_(env.action_mask)[:, :env.jobs + 1].astype(bool)
    assert (q[mask] >= 0).all()
    assert (q[~mask] == -1).all()
    host = table.cpu().numpy()
    for i in np.random.default_rng(14).choice(n, 4, replace=False):
        for a in np.flatnonzero(mask[i])[:3]:
            want = oracle_value("ta80", [t[i] for t in taken], int(a), host[i])
            assert q[i, a] == want, (i, a)
