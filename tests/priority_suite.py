"""The tests of jss_rollout_priority (a caller's static priority rule run to the end of every episode in one launch),
declared once for both backends (tests/backends.py) and collected by tests/test_emu_priority.py and
tests/test_gpu_priority.py.  The rollout is checked against a twin env stepped with jss_step_greedy on the rows the
table gives at each decision (the priority of every job's current operation, the no-op at -inf), against twins
stepped with the built-in rules, and against the CPU oracle."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import assert_twins_equal, batch_cfg, np_, synthetic_instance, twin_envs


def random_table(env, seed, ties=False):
    """A seeded (N, J, M) float32 table; with ties, small integers, so that equal priorities and -0.0 / +0.0 meet."""
    rng = np.random.default_rng(seed)
    shape = (env.num_envs, env.jobs, env.machines)
    if ties:
        return (rng.integers(-2, 3, size=shape) * np.where(rng.random(shape) < 0.5, -1.0, 1.0)).astype(np.float32)
    return rng.standard_normal(shape).astype(np.float32)


def greedy_rows(env, table):
    """The step_greedy rows a static priority table gives in env's current state: the entry of every job's current
    operation (clamped for finished jobs and padding, which are never legal) and the no-op column at -inf."""
    n, J, M = env.num_envs, env.jobs, env.machines
    todo = np.clip(np_(env.export_state()["todo"]), 0, M - 1)
    rows = np.full((n, J + 1), -np.inf, np.float32)
    rows[:, :J] = np.take_along_axis(np.broadcast_to(table, (n, J, M)), todo[:, :, None], 2)[:, :, 0]
    rows[np.arange(n), env.env_jobs] = -np.inf           # env i's no-op is column J_i
    return rows


def greedy_steps(env, table, k):
    """Up to k twin steps of step_greedy(rows, 0) (fewer once every env is done: done envs are frozen)."""
    for _ in range(k):
        if np_(env.done).all():
            return
        env.step_greedy(lc._to_dev(env, greedy_rows(env, table)))


def assert_same(a_env, b_env, ctx):
    assert_twins_equal(a_env, b_env, ctx, state=True, stats=True)
    if a_env.solution is not None:
        assert np.array_equal(np_(a_env.solution), np_(b_env.solution)), (ctx, "solution")


def check_twin(make_env, names, seed, k, ties=False):
    """rollout_priority(P, k), then to the end, equals as many twin steps of step_greedy; a third env run to the end
    in one call ends where the twin ends."""
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    table = random_table(a_env, seed, ties)
    a_env.rollout_priority(lc._to_dev(a_env, table), k)
    greedy_steps(b_env, table, k)
    assert_same(a_env, b_env, ("partial", k))
    a_env.rollout_priority(lc._to_dev(a_env, table))
    bound = 2 * a_env.jobs * a_env.machines + 1
    greedy_steps(b_env, table, bound)
    assert np_(b_env.done).all()
    assert_same(a_env, b_env, "second call")
    c_env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    c_env.reset()
    c_env.rollout_priority(lc._to_dev(c_env, table))
    assert_same(c_env, b_env, "one call")
    assert not (np_(c_env.flags) & N.FLAG_ERROR).any()
    return c_env


BIG_GPU = synthetic_instance(200, 8, 9, max_dur=50)
NONPERM = synthetic_instance(37, 5, 8, max_dur=30, permutation=False)
# emulation: short episodes in every lane class (33..64, 65..128 and 129..256 jobs)
EMU_CLASSES = [synthetic_instance(40, 3, 10, max_dur=30), synthetic_instance(70, 3, 11, max_dur=30),
               synthetic_instance(130, 2, 12, max_dur=30)]


@native_test(emu=[False, True], gpu=[False, True])
def priority_twin_mixed_batch(make_env, backend, ties):
    # every lane class of the generic kernel, 129..256 jobs and a non-permutation instance included
    if backend == "emu":
        check_twin(make_env, ["ta01", "ta01", *EMU_CLASSES, NONPERM], seed=1, k=40, ties=ties)
    else:
        check_twin(make_env, ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80", NONPERM,
                              BIG_GPU] * 3, seed=1, k=300, ties=ties)


@native_test()
def priority_twin_uniform(make_env, backend):
    """Uniform tiny (J <= 4), ta01 and ta80 batches."""
    n = {"emu": 3, "gpu": 64}[backend]
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        check_twin(make_env, [synthetic_instance(J, M, J * 10 + M)] * n, seed=J + M, k=2, ties=True)
    check_twin(make_env, ["ta01"] * n, seed=2, k=60)
    if backend == "gpu":
        check_twin(make_env, ["ta80"] * n, seed=3, k=700)


def _rule_tables(env):
    """SPT, MWR, LWR, MOR and LOR as (N, J, M) priority tables built from each env's instance."""
    n, J, M = env.num_envs, env.jobs, env.machines
    t = {r: np.zeros((n, J, M), np.float32) for r in ("SPT", "MWR", "LWR", "MOR", "LOR")}
    for i, k in enumerate(env.env_to_instance):
        _, dur = env.instances[k]
        Ji, Mi = dur.shape
        rem = np.cumsum(dur[:, ::-1], axis=1)[:, ::-1]           # work remaining from operation k on
        ops = np.arange(Mi)
        t["SPT"][i, :Ji, :Mi] = -dur
        t["MWR"][i, :Ji, :Mi] = rem
        t["LWR"][i, :Ji, :Mi] = -rem
        t["MOR"][i, :Ji, :Mi] = Mi - ops
        t["LOR"][i, :Ji, :Mi] = ops - Mi
    return t


@native_test()
def priority_reproduces_builtin_rules(make_env, backend):
    """Each built-in static rule as a table, run to done, is bit-identical to a twin stepped with policy(rule,
    coin="never") + step()."""
    names = {"emu": ["ta01", "ta01", "ta11", NONPERM], "gpu": ["ta01", "ta21", "ta41", "ta80", NONPERM, BIG_GPU] * 4}
    for rule, table in _rule_tables(make_env(len(names[backend]), batch_cfg(names[backend], sort=False))).items():
        a_env, b_env = twin_envs(make_env, names[backend], sort=False, auto_reset=False, record_solution=True)
        a_env.rollout_priority(lc._to_dev(a_env, table))
        for _ in range(2 * a_env.jobs * a_env.machines + 1):
            if np_(b_env.done).all():
                break
            b_env.step(b_env.policy(rule, coin="never"))
        assert np_(a_env.done).all(), rule
        assert_same(a_env, b_env, rule)


def oracle_run(inst, table):
    """The oracle's episode under the table's argmax over the legal jobs' current operations (the no-op when nothing
    else is legal); returns the oracle at the end and its raw return."""
    o = OracleEnv(*(load_instance(inst) if isinstance(inst, str) else inst))
    o.reset()
    done, total = False, 0
    while not done:
        legal = np.asarray(o.get_legal_actions(), bool)
        jobs = np.flatnonzero(legal[:-1])
        if len(jobs):
            keys = table[jobs, np.asarray(o.todo_time_step_job)[jobs]]
            a = int(jobs[np.argmax(keys)])
        else:
            a = o.jobs
        _, _, done, _, _ = o.step(a)
        total += o.last_raw_reward
    return o, total


def check_oracle(env, names, rows):
    """Makespan, raw return and solution of env i against the oracle's replay of the table rows[i] (J, M), i in rows."""
    for i, table in rows.items():
        Ji, Mi = (load_instance(names[i]) if isinstance(names[i], str) else names[i])[0].shape
        o, ret = oracle_run(names[i], table[:Ji, :Mi])
        assert int(env.last_makespan[i]) == o.current_time_step, i
        assert int(env.last_return[i]) == ret, i
        assert np.array_equal(np_(env.solution)[i, :Ji, :Mi], np.asarray(o.solution)), i


@native_test()
def priority_matches_oracle(make_env, backend):
    names = {"emu": ["ta01", "ta41", NONPERM, "ta01"], "gpu": ["ta01", "ta41", "ta80", NONPERM, BIG_GPU] * 4}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    env.reset()
    table = random_table(env, 5, ties=True)
    env.rollout_priority(lc._to_dev(env, table))
    assert np_(env.done).all()
    check_oracle(env, names, {i: table[i] for i in range(0, len(names), 1 if backend == "emu" else 3)})


@native_test()
def priority_broadcasts(make_env, backend):
    """(N, J, 1), (1, J, M) and padded strides (ld_job > M, ld_env > J * ld_job, NaN in the padding) give what the
    materialised (N, J, M) table gives."""
    import torch
    names = {"emu": ["ta01", "ta21", "ta01"], "gpu": ["ta01", "ta21", "ta41", "ta80"] * 8}[backend]
    ref = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    n, J, M, dev = ref.num_envs, ref.jobs, ref.machines, ref.device
    rng = np.random.default_rng(7)
    per_job = torch.from_numpy(rng.standard_normal((n, J, 1)).astype(np.float32)).to(dev)
    shared = torch.from_numpy(rng.integers(-3, 4, size=(1, J, M)).astype(np.float32)).to(dev)
    full = torch.from_numpy(random_table(ref, 8)).to(dev)
    padded = torch.full((n, J + 2, M + 5), float("nan"), device=dev)
    padded[:, :J, :M] = full
    view = padded[:, :J, :M]
    assert view.stride() == ((J + 2) * (M + 5), M + 5, 1)
    for given, materialised in ((per_job, per_job.expand(n, J, M)), (shared, shared.expand(n, J, M)),
                                (view, full), (per_job.double(), per_job.expand(n, J, M))):
        a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
        a_env.rollout_priority(given)
        b_env.rollout_priority(materialised.contiguous())
        assert np_(a_env.done).all()
        assert_same(a_env, b_env, tuple(given.shape))


@native_test()
def priority_done_and_auto_reset(make_env):
    """Under auto-reset: an env that finishes stops there with episode_count + 1 once, a done env is untouched by the
    next call, and reset() plus a second call replays the same episode."""
    names = ["ta01", "ta01", "ta31", "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=True, record_solution=True)
    env.reset()
    table = lc._to_dev(env, random_table(env, 9))
    env.rollout_priority(table, 100)
    env.rollout_priority(table)                           # the ta01 envs finish long before the bound
    assert np_(env.done).all() and (np_(env.episode_count) == 1).all()
    first = {k: np_(getattr(env, k)).copy() for k in ("last_makespan", "last_return", "current_time_step", "solution")}
    before = {k: np_(v).copy() for k, v in env.export_state().items()}
    obs = np_(env.real_obs).copy()
    c = env.launch_count
    env.rollout_priority(table)                           # every env done at entry
    assert env.launch_count == c + 1                      # one lane class
    assert (np_(env.episode_count) == 1).all() and np.array_equal(np_(env.real_obs), obs)
    for k, v in env.export_state().items():
        assert np.array_equal(np_(v), before[k]), k
    env.reset(np.array([1, 0, 1, 0], np.uint8))
    env.rollout_priority(table)
    assert np.array_equal(np_(env.episode_count), [2, 1, 2, 1])
    for k, v in first.items():
        assert np.array_equal(np_(getattr(env, k)), v), k


@native_test()
def priority_bad_priorities(make_env, backend):
    """NaN / +inf on a legal current operation, or every legal job at -inf, set the error bit and stop the env where
    the step_greedy twin leaves it, at the first decision or mid-episode; NaN and inf on entries that are never read
    (illegal jobs, finished operations, columns past J_i, operations past M_i) change nothing."""
    names = ["ta01", "ta01", "ta01", "ta01", "ta01", "ta21", "ta01", "ta01"]
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    J = a_env.jobs
    clean = random_table(a_env, 11)
    t = clean.copy()
    t[0, 3, 0] = np.nan                                   # every job is legal at reset
    t[1, 2, 0] = np.inf
    t[2, :, 0] = -np.inf
    t[3, :, 4] = np.nan                                   # mid-episode, once a job reaches its operation 4
    t[4, :15, 6] = -np.inf                                # mid-episode, all legal -inf: whichever comes
    t[4, :15, 7:] = -np.inf
    t[6, 15:, :] = np.nan                                 # columns past J_i = 15
    t[6, :, 15:] = np.inf                                 # operations past M_i = 15
    a_env.rollout_priority(lc._to_dev(a_env, t))
    greedy_steps(b_env, t, 2 * J * a_env.machines + 1)
    assert_same(a_env, b_env, "bad")
    err = (np_(a_env.flags) & N.FLAG_ERROR) != 0
    assert err[:5].all() and not err[5:].any(), err
    assert (np_(a_env.current_time_step)[:3] == 0).all() and int(a_env.current_time_step[3]) > 0
    ref = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    ref.reset()
    ref.rollout_priority(lc._to_dev(ref, clean))
    for i in (5, 6, 7):
        for k in ("last_makespan", "last_return", "solution"):
            assert np.array_equal(np_(getattr(a_env, k))[i], np_(getattr(ref, k))[i]), (i, k)
    # illegal jobs and finished operations: poisoned after a partial call, between calls
    a_env, b_env = twin_envs(make_env, ["ta01"] * 4, sort=False, auto_reset=False, record_solution=True)
    table = random_table(a_env, 12)
    for env in (a_env, b_env):
        env.rollout_priority(lc._to_dev(env, table), 30)
    x = b_env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    poisoned = table.copy()
    ops = np.arange(a_env.machines)
    poisoned[ops[None, None, :] < todo[:, :, None]] = np.nan                 # finished operations
    for i, j in zip(*np.nonzero(~legal & (todo < a_env.machines))):
        poisoned[i, j, todo[i, j]] = np.inf if (i + j) % 2 else np.nan       # illegal jobs' current operations
    a_env.rollout_priority(lc._to_dev(a_env, poisoned), 1)
    b_env.rollout_priority(lc._to_dev(b_env, table), 1)
    assert_same(a_env, b_env, "illegal")
    poisoned = table.copy()
    todo = np_(b_env.export_state()["todo"])
    poisoned[ops[None, None, :] < todo[:, :, None]] = np.nan
    a_env.rollout_priority(lc._to_dev(a_env, poisoned))
    b_env.rollout_priority(lc._to_dev(b_env, table))
    assert_same(a_env, b_env, "finished")
    assert not (np_(a_env.flags) & N.FLAG_ERROR).any()


@native_test()
def priority_abi(make_env):
    """JSS_ERR_INVALID for a NULL or misaligned table, a negative stride or n_steps < 0, JSS_ERR_STATE before
    jss_assign; n_steps = 0 does nothing; one launch per lane class present; a call after a recording step first
    refreshes real_obs; a wrong rank or shape raises ValueError before the native call."""
    import pytest
    import torch
    names = ["ta01", "ta51", "ta80", "ta01"]             # lane classes 1, 2 and 4 jobs per lane
    env = make_env(len(names), batch_cfg(names, sort=False), seed=3)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    L, h, st = env._L, env._h, env._stream()
    p, s = t.data_ptr(), (J * M, M, 1)
    for args in ((None, *s, 5), (p + 2, *s, 5), (p, -1, M, 1, 5), (p, J * M, -M, 1, 5), (p, J * M, M, -1, 5),
                 (p, *s, -1)):
        assert L.jss_rollout_priority(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_rollout_priority:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_rollout_priority(raw, p, *s, 5, st) == -5
    L.jss_destroy(raw)
    before = {k: np_(getattr(env, k)).copy() for k in ("real_obs", "action_mask", "reward_raw", "current_time_step")}
    c = env.launch_count
    assert L.jss_rollout_priority(h, p, *s, 0, st) == 0
    assert env.launch_count == c
    for k, v in before.items():
        assert np.array_equal(np_(getattr(env, k)), v), k
    env.rollout_priority(t, 3)
    assert env.launch_count == c + 3
    step_index = env._step_index
    for bad in (t[0], t[None], t[:, :J - 1], torch.zeros((2, J, M), device=env.device), t[:, :, :M - 1]):
        with pytest.raises(ValueError):
            env.rollout_priority(bad)
    assert env._step_index == step_index                  # refused before the native call, and no RNG counter
    # after a recording step, real_obs is brought up to date before the rollout (env 0's bad row leaves it unchanged,
    # so only the refresh writes its observation)
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=4)
    table = random_table(a_env, 13)
    table[0] = np.nan
    table = lc._to_dev(a_env, table)
    scores = torch.zeros((n, J + 1), device=a_env.device)
    traj = a_env.logits_trajectory(1)
    a_env.step_greedy_record(scores, traj, 0)
    b_env.step_greedy(scores)
    for env_ in (a_env, b_env):
        env_.rollout_priority(table, 5)
    assert_twins_equal(a_env, b_env, "after record", state=True, stats=True)


@native_test(emu=None)
def priority_full_size_ta80(make_env):
    """ta80 at N = 65 536, a random per-operation table, one default call: every env done without the error bit, the
    raw return 2 sum_op - M makespan everywhere, five sampled envs equal to the oracle's replay."""
    import torch
    n_envs = 65536
    env = make_env(n_envs, {"instance_path": "ta80"}, auto_reset=False, record_solution=True)
    env.reset()
    J, M = env.jobs, env.machines
    sum_op = int(env.instance_scalars[0][2])
    gen = torch.Generator(device=env.device).manual_seed(21)
    table = torch.rand((n_envs, J, M), generator=gen, device=env.device)
    env.rollout_priority(table)
    assert np_(env.done).all()
    assert not (np_(env.flags) & N.FLAG_ERROR).any()
    makespan = np_(env.last_makespan).astype(np.int64)
    assert np.array_equal(np_(env.last_return).astype(np.int64), 2 * sum_op - M * makespan)
    assert np.array_equal(np_(env.current_time_step), makespan)
    picks = [0, 1, 4097, 33333, 65535]
    check_oracle(env, {i: "ta80" for i in picks}, {i: table[i].cpu().numpy() for i in picks})
