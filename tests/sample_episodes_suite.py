"""The tests of jss_sample_episodes (k episodes per env drawn from a caller's logit table, the envs left untouched, with
a replayed gradient and the schedule of a chosen sample), declared once for both backends (tests/backends.py) and
collected by tests/test_emu_sample_episodes.py and tests/test_gpu_sample_episodes.py.  Every sample is checked against
its definition on a twin batch: the same state imported, the RNG counter set to step_index + s*B, and one
rollout_priority_sample call, which is itself tested against step_logits and the CPU oracle."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv
from tests import logits_common as lc
from tests.backends import native_test
from tests.lookahead_priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, SHAPES, SMALL, TINY, noop_only, shaped_table
from tests.lookahead_suite import _outputs, random_walk, snapshot
from tests.parity_common import batch_cfg, np_, synthetic_instance
from tests.priority_sample_suite import Twin, assert_log_prob, sample_call
from tests.priority_suite import random_table


def bound(env):
    return 2 * env.jobs * env.machines + 1


def twin_samples(make_env, env, table, k, step_index, solution=False):
    """What sample_episodes(table, k) at RNG counter step_index must give in env's current state, by its definition:
    per sample s, a twin batch with env's state imported runs rollout_priority_sample(table) once at counter
    step_index + s*B.  Returns makespan (N, k), log_prob (N, k), the float64 gradients (k, N, J, M) (zero where the
    twin's are NaN: padding, or never written) and, with `solution`, the twins' solution tables (k, N, J, M)."""
    n, J, M = env.num_envs, env.jobs, env.machines
    cfg = {"instance_paths": [env.instances[i] for i in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    twin = make_env(n, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed, record_solution=solution)
    snap = snapshot(env)
    done0 = np_(env.done).copy()
    dev = lc._to_dev(twin, table)
    ms = np.full((n, k), -1, np.int64)
    lp = np.zeros((n, k), np.float32)
    grads = np.zeros((k, n, J, M))
    sols = np.zeros((k, n, J, M), np.int32) if solution else None
    for s in range(k):
        twin.reset()                                     # solution rows back to -1
        twin.import_state(snap)
        twin._step_index = step_index + s * bound(env)
        l, g = sample_call(twin, dev)
        done, t = np_(twin.done), np_(twin.current_time_step)
        ms[done & ~done0, s] = t[done & ~done0]
        lp[:, s] = l
        grads[s] = np.nan_to_num(g.astype(np.float64), nan=0.0)
        if solution:
            sols[s] = np_(twin.solution)
    twin.close()
    return ms, lp, grads, sols


def draw(env, table, k, **kw):
    """sample_episodes of a host table; the counter must advance by k*B.  Returns the dict and the counter used."""
    si = env._step_index
    out = env.sample_episodes(lc._to_dev(env, table), k, **kw)
    assert env._step_index == si + k * bound(env)
    return out, si


def check_against_twins(make_env, env, table, k, weights_seed=None, splits=(1,)):
    """makespan and log_prob bit for bit against the twins; `best` from them; with weights_seed, the gradient for
    random weights at each split within 1e-5 * sum |w| (1 + |G|) per entry, and a second backward bit-identical."""
    out, si = draw(env, table, k)
    ms, lp, grads, _ = twin_samples(make_env, env, table, k, si)
    got_ms = np_(out["makespan"]).astype(np.int64)
    assert np.array_equal(got_ms, ms), (got_ms, ms)
    assert_log_prob(np_(out["log_prob"]).ravel(), lp.ravel(), "log_prob")
    big = np.where(ms >= 0, ms, np.iinfo(np.int64).max)
    want_best = np.where((ms >= 0).any(1), big.argmin(1), -1)
    assert np.array_equal(np_(out["best"]), want_best)
    if weights_seed is not None:
        import torch
        w = np.random.default_rng(weights_seed).standard_normal((env.num_envs, k)).astype(np.float32)
        want = np.einsum("ns,snjm->njm", w.astype(np.float64), grads)
        scale = np.einsum("ns,snjm->njm", np.abs(w).astype(np.float64), 1 + np.abs(grads))
        x = lc._to_dev(env, table)
        wt = torch.from_numpy(w).to(env.device)
        for split in splits:
            g1 = np_(env._sample_episodes_grad(x, k, si, wt, split).sum(0)).astype(np.float64)
            g2 = np_(env._sample_episodes_grad(x, k, si, wt, split).sum(0)).astype(np.float64)
            assert np.array_equal(g1, g2), split
            assert (np.abs(g1 - want) <= 1e-5 * scale).all(), (split, np.abs(g1 - want).max())
    return out, ms


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def sample_episodes_twin(make_env, backend, shape, ties):
    """Every lane class in one batch (129..256 jobs and a non-permutation instance included) at reset and mid-episode,
    with some envs done and one with only the no-op legal; uniform tiny batches (J <= 4); (N, J, M), (N, J, 1) and
    (1, J, M) tables, with ties.  The gradient is checked with one chunk and with several."""
    if backend == "emu":
        names, walk, k = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170, 3
    else:
        names, walk, k = ["ta01", "ta11", "ta21", "ta31", "ta41", "ta51", "ta61", "ta71", "ta80", NONPERM, BIG_GPU,
                          SMALL, TINY] * 2, 400, 6
    seed = SHAPES.index(shape) + (10 if ties else 0)
    for steps in (0, walk):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=5)
        env.reset()
        random_walk(env, steps)
        if steps:
            i = int(np.flatnonzero(~np_(env.done))[0])
            x = env.export_state()
            x["legal"][i] = 0
            x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
            env.import_state(x)
            done = np_(env.done)
            assert done.any() and not done.all() and noop_only(env).any(), done
        table = shaped_table(env, seed, ties, shape)
        _, ms = check_against_twins(make_env, env, table, k, weights_seed=seed, splits=(1, k))
        assert (ms[~np_(env.done)] >= 0).any()
        assert (ms[np_(env.done)] == -1).all()
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        env = make_env(3, batch_cfg([synthetic_instance(J, M, J * 10 + M)] * 3), auto_reset=False, seed=seed)
        env.reset()
        check_against_twins(make_env, env, shaped_table(env, seed, ties, shape), 4, weights_seed=seed, splits=(1, 3))


@native_test()
def sample_episodes_split_invariance(make_env, backend):
    """A batch of 3 (one tile: the library spreads each env's samples over several work items) and a large batch (one
    work item per tile) give the same outputs for the same states, counters and tables."""
    n_big = {"emu": 24, "gpu": 4096}[backend]
    big = make_env(n_big, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    big.reset()
    random_walk(big, 40)
    snap = snapshot(big)
    small = make_env(3, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    small.reset()
    small.import_state({k: v[:3] for k, v in snap.items()})
    full, ties = random_table(big, 13), random_table(big, 14, ties=True)
    for tb, ts in ((full, full[:3]), (ties[:1], ties[:1])):
        ob, _ = draw(big, tb, 5)
        small._step_index = big._step_index - 5 * bound(big)
        os_, _ = draw(small, ts, 5)
        for key in ("makespan", "log_prob", "best"):
            a, b = np_(ob[key])[:3], np_(os_[key])
            assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                  b.view(np.uint32) if b.dtype == np.float32 else b), key
        assert (np_(os_["makespan"]) >= 0).all()


@native_test(emu=[False, True], gpu=[False, True])
def sample_episodes_untouched(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and flags are bit-identical after the draws, the gradient
    replay and the solution replay; the counter advances by k*B; the draws take one launch per lane class present; after
    a recording step the call leaves real_obs stale."""
    import torch
    names = ["ta01", NONPERM, "ta01", SMALL] if backend == "emu" else ["ta01", "ta51", "ta80", NONPERM] * 8
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, record_solution=True, seed=8)
    env.reset()
    random_walk(env, 60)
    before, stats = _outputs(env), env.stats()
    classes = 2 if backend == "emu" else 3
    table = random_table(env, 4)
    c = env.launch_count
    out, si = draw(env, table, 3)
    assert env.launch_count == c + classes
    draw(env, random_table(env, 5, ties=True)[:1], 2, solution=True)
    x = lc._to_dev(env, table)
    env._sample_episodes_grad(x, 3, si, torch.ones((env.num_envs, 3), device=env.device), 2)
    after = _outputs(env)
    for k, v in before.items():
        assert np.array_equal(v, after[k]), k
    assert env.stats() == stats
    assert not (np_(env.flags) & N.FLAG_ERROR).any()
    cfg = batch_cfg(names, sort=False)
    a_env, b_env = (make_env(len(names), cfg, auto_reset=auto_reset, seed=9) for _ in range(2))
    a_env.reset(); b_env.reset()
    scores = torch.zeros((a_env.num_envs, a_env.jobs + 1), device=a_env.device)
    traj = a_env.logits_trajectory(1)
    stale = np_(a_env.real_obs).copy()
    a_env.step_greedy_record(scores, traj, 0)
    b_env.step_greedy(scores)
    table = random_table(a_env, 6)
    oa, _ = draw(a_env, table, 2)
    ob, _ = draw(b_env, table, 2)
    assert np.array_equal(np_(oa["makespan"]), np_(ob["makespan"]))
    assert np.array_equal(np_(a_env.real_obs), stale)


@native_test()
def sample_episodes_gradient(make_env, backend):
    """log_prob.backward(w) against the float64 sum over the twins' gradients for (N, J, M), (N, J, 1), (1, J, M) and
    float64 tables; two backward passes bit-identical; NaN samples, done envs and zero weights add exactly nothing; a
    table changed in place between forward and backward raises; without requires_grad log_prob has no grad_fn."""
    import pytest
    import torch
    names = {"emu": ["ta01", SMALL, "ta01", TINY], "gpu": ["ta01", "ta21", "ta41", "ta80", SMALL] * 4}[backend]
    k = 4
    ref = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False)
    n, J, M, dev = ref.num_envs, ref.jobs, ref.machines, ref.device
    rng = np.random.default_rng(17)
    w = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).to(dev)
    for shape, dtype in (((n, J, M), torch.float32), ((n, J, 1), torch.float32), ((1, J, M), torch.float32),
                         ((n, J, M), torch.float64)):
        env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=3)
        env.reset()
        random_walk(env, 20)
        base = torch.from_numpy(rng.standard_normal(shape)).to(dev, dtype)
        x = base.clone().requires_grad_(True)
        si = env._step_index
        out = env.sample_episodes(x, k)
        assert out["log_prob"].grad_fn is not None and out["makespan"].grad_fn is None
        out["log_prob"].backward(w, retain_graph=True)
        g1 = x.grad.clone()
        x.grad = None
        out["log_prob"].backward(w)
        assert torch.equal(g1, x.grad), shape
        assert x.grad.dtype == dtype and x.grad.shape == shape
        table = base.to(torch.float32).expand(n, J, M).cpu().numpy()
        _, _, grads, _ = twin_samples(make_env, env, table, k, si)
        want = np.einsum("ns,snjm->njm", np_(w).astype(np.float64), grads)
        scale = np.einsum("ns,snjm->njm", np.abs(np_(w)).astype(np.float64), 1 + np.abs(grads))
        want = torch.from_numpy(want).sum_to_size(shape).numpy()
        scale = torch.from_numpy(scale).sum_to_size(shape).numpy()
        assert (np.abs(np_(x.grad).astype(np.float64) - want) <= 1e-5 * scale).all(), shape
    # NaN samples, done envs and zero weights
    env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=4)
    env.reset()
    random_walk(env, 30 if backend == "emu" else 200)
    table = random_table(env, 19)
    x_ = env.export_state()
    todo, legal = np_(x_["todo"]), np_(x_["legal"]).astype(bool)
    alive = np.flatnonzero(~np_(env.done))
    bad_env = int(alive[0])
    Ji, Mi = int(env.env_jobs[bad_env]), int(env.env_machines[bad_env])
    table[bad_env, :, min(int(todo[bad_env, :Ji].max()) + 1, Mi - 1):] = np.nan   # met later by most samples
    dev_t = lc._to_dev(env, table)
    out, si = draw(env, table, 6)
    lp = np_(out["log_prob"])
    nan = np.isnan(lp)
    assert nan[bad_env].any(), lp[bad_env]
    wn = rng.standard_normal((n, 6)).astype(np.float32)
    wz = wn.copy()
    wz[nan] = 0.0
    wz[np_(env.done)] = 0.0
    wz[:, 1] = 0.0
    wn[:, 1] = 0.0
    for split in (1, 3):
        ga = np_(env._sample_episodes_grad(dev_t, 6, si, torch.from_numpy(wn).to(dev), split))
        gb = np_(env._sample_episodes_grad(dev_t, 6, si, torch.from_numpy(wz).to(dev), split))
        assert np.array_equal(ga, gb), split
        for i in np.flatnonzero(np_(env.done)):
            assert (ga[:, i] == 0).all(), i
    _, _, grads, _ = twin_samples(make_env, env, table, 6, si)
    assert (grads[nan.T] == 0).all()
    # in-place change between forward and backward
    x = torch.from_numpy(random_table(env, 20)).to(dev).requires_grad_(True)
    y = x * 1.0
    out = env.sample_episodes(y, 2)
    with torch.no_grad():
        y.add_(1.0)
    with pytest.raises(RuntimeError):
        out["log_prob"].sum().backward()
    out = env.sample_episodes(torch.from_numpy(random_table(env, 21)).to(dev), 2)
    assert out["log_prob"].grad_fn is None


def check_schedule(inst, sol, makespan):
    """A full schedule of `inst` (machine, duration): job precedence, no overlap on a machine, and the makespan."""
    machine, duration = inst
    J, M = machine.shape
    assert (sol[:J, :M] >= 0).all()
    end = sol[:J, :M] + duration
    assert (sol[:J, 1:M] >= end[:, :M - 1]).all()
    for m in range(int(machine.max()) + 1):
        iv = sorted(zip(sol[:J, :M][machine == m], end[machine == m]))
        assert all(b[0] >= a[1] for a, b in zip(iv, iv[1:])), m
    assert int(end.max()) == makespan


@native_test()
def sample_episodes_solution(make_env, backend):
    """The best sample's schedule equals its twin's solution; from reset it is feasible and ends at makespan[best];
    mid-episode it is the env's own solution completed; without record_solution the rest reads -1; an env whose best
    is -1 keeps its row."""
    names = {"emu": ["ta01", SMALL, NONPERM, TINY], "gpu": ["ta01", "ta21", "ta80", NONPERM, SMALL] * 4}[backend]
    k = 4
    for record, steps in ((True, 0), (True, 25), (False, 25)):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=record, seed=5)
        env.reset()
        random_walk(env, steps)
        table = random_table(env, 22)
        before = np_(env.solution).copy() if record else None
        out, si = draw(env, table, k, solution=True)
        ms, _, _, sols = twin_samples(make_env, env, table, k, si, solution=True)
        best, sol = np_(out["best"]), np_(out["solution"])
        if record:
            assert np.array_equal(np_(env.solution), before)
        for i, b in enumerate(best):
            if b < 0:
                want = before[i] if record else np.full_like(sol[i], -1)
                assert np.array_equal(sol[i], want), i
                continue
            started = sols[b, i] >= 0
            assert np.array_equal(sol[i][started], sols[b, i][started]), i
            if record:
                assert np.array_equal(sol[i][~started], before[i][~started]), i
            else:
                assert (sol[i][~started] == -1).all(), i
            if steps == 0:
                inst = names[i] if not isinstance(names[i], str) else load_instance(names[i])
                check_schedule(inst, sol[i], int(ms[i, b]))


@native_test()
def sample_episodes_bad_tables(make_env, backend):
    """NaN / +inf on a legal current operation, or every legal job at -inf: only the samples that meet them read -1
    and NaN, as their twins do; no env gets the error bit; entries never read change nothing."""
    names = ["ta01", "ta01", "ta01", "ta01", SMALL, "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
    env.reset()
    random_walk(env, 40 if backend == "emu" else 60)
    x = env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    clean = random_table(env, 31)
    bad = clean.copy()
    j0 = int(np.flatnonzero(legal[0])[0])
    bad[0, j0, todo[0, j0]] = np.nan                      # a legal job's current operation: every sample
    bad[1, :, min(int(todo[1].max()) + 2, env.machines - 1)] = np.inf
    bad[2] = -np.inf                                      # every legal job at -inf at the first decision
    bad[4, 9:, :] = np.nan                                # columns past J_i = 9
    bad[4, :, 4:] = np.inf                                # operations past M_i = 4
    ops = np.arange(env.machines)
    bad[5][ops[None, :] < todo[5][:, None]] = np.nan      # finished operations
    flags = np_(env.flags).copy()
    k = 4
    out, si = draw(env, bad, k)
    assert np.array_equal(np_(env.flags), flags) and not (flags & N.FLAG_ERROR).any()
    ms, lp, _, _ = twin_samples(make_env, env, bad, k, si)
    got_ms, got_lp = np_(out["makespan"]), np_(out["log_prob"])
    assert np.array_equal(got_ms, ms)
    assert_log_prob(got_lp.ravel(), lp.ravel(), "bad")
    assert np.array_equal(np.isnan(got_lp), (got_ms < 0) & ~np_(env.done)[:, None])
    assert np.isnan(got_lp[2]).all() and np.isnan(got_lp[1]).any()
    env._step_index = si
    ok, _ = draw(env, clean, k)
    for i in (3, 4, 5):
        assert np.array_equal(np_(ok["makespan"])[i], got_ms[i]), i
        assert np.array_equal(np_(ok["log_prob"])[i].view(np.uint32), got_lp[i].view(np.uint32)), i


@native_test()
def sample_episodes_shards(make_env, backend):
    """Shards created with env_id_base != 0 give the rows of the unsharded batch, bit for bit."""
    n_total = {"emu": 8, "gpu": 96}[backend]
    names = {"emu": ["ta01", SMALL, "ta01", NONPERM], "gpu": ["ta01", "ta31", "ta51", "ta80"]}[backend]
    e2i = np.arange(n_total) % len(names)
    cuts = [0, 5, n_total]
    whole = make_env(n_total, {"instance_paths": names, "env_to_instance": e2i}, seed=31, auto_reset=False)
    whole.reset()
    table = random_table(whole, 14)
    ow, _ = draw(whole, table, 3)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        s = make_env(hi - lo, {"instance_paths": names, "env_to_instance": e2i[lo:hi]}, seed=31, auto_reset=False,
                     env_id_base=lo)
        s.reset()
        os_, _ = draw(s, table[lo:hi, :s.jobs, :s.machines], 3)
        assert np.array_equal(np_(os_["makespan"]), np_(ow["makespan"])[lo:hi]), lo
        assert np.array_equal(np_(os_["log_prob"]).view(np.uint32), np_(ow["log_prob"])[lo:hi].view(np.uint32)), lo


@native_test()
def sample_episodes_abi(make_env, backend):
    """JSS_ERR_INVALID for NULL or misaligned pointers, a negative stride, k < 1, ld < k, split < 1 or > k and k*B past
    2^64; JSS_ERR_STATE before jss_assign; a bad table shape or k raises ValueError before the native call."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    L, h, st = env._L, env._h, env._stream()
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    i32 = torch.zeros(n * 8, dtype=torch.int32, device=env.device)
    f32 = torch.zeros(n * 8, dtype=torch.float32, device=env.device)
    g = torch.zeros(8 * n * J * M, dtype=torch.float32, device=env.device)
    p, o, q, w, r = t.data_ptr(), i32.data_ptr(), f32.data_ptr(), f32.data_ptr(), g.data_ptr()
    s = (J * M, M, 1)
    huge = 1 << 62
    fwd = ((None, *s, 4, o, q, 4), (p + 2, *s, 4, o, q, 4), (p, -1, M, 1, 4, o, q, 4), (p, J * M, -M, 1, 4, o, q, 4),
           (p, J * M, M, -1, 4, o, q, 4), (p, *s, 0, o, q, 4), (p, *s, -3, o, q, 4), (p, *s, 4, o, q, 3),
           (p, *s, 4, None, q, 4), (p, *s, 4, o + 2, q, 4), (p, *s, 4, o, None, 4), (p, *s, 4, o, q + 2, 4),
           (p, *s, huge, o, q, huge))
    for args in fwd:
        assert L.jss_sample_episodes(h, *args[:4], 0, 0, *args[4:], st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_sample_episodes:"), args
    bwd = ((None, *s, 4, w, 4, 1, r), (p, -1, M, 1, 4, w, 4, 1, r), (p, *s, 0, w, 4, 1, r), (p, *s, 4, w, 3, 1, r),
           (p, *s, 4, None, 4, 1, r), (p, *s, 4, w + 2, 4, 1, r), (p, *s, 4, w, 4, 0, r), (p, *s, 4, w, 4, 5, r),
           (p, *s, 4, w, 4, 1, None), (p, *s, 4, w, 4, 1, r + 2), (p, *s, huge, w, huge, 1, r))
    for args in bwd:
        assert L.jss_sample_episodes_grad(h, *args[:4], 0, 0, *args[4:], st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_sample_episodes_grad:"), args
    for args in ((None, *s, o, o), (p, *s, o + 2, o), (p, *s, None, o), (p, *s, o, None), (p, *s, o, o + 2),
                 (p, J * M, -M, 1, o, o)):
        assert L.jss_sample_episodes_solution(h, *args[:4], 0, 0, *args[4:], st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_sample_episodes_solution:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_sample_episodes(raw, p, *s, 0, 0, 4, o, q, 4, st) == -5
    assert L.jss_sample_episodes_grad(raw, p, *s, 0, 0, 4, w, 4, 1, r, st) == -5
    assert L.jss_sample_episodes_solution(raw, p, *s, 0, 0, o, o, st) == -5
    L.jss_destroy(raw)
    si = env._step_index
    for bad in (t[0], t[None], t[:, :J - 1], torch.zeros((3, J, M), device=env.device)):
        with pytest.raises(ValueError):
            env.sample_episodes(bad, 2)
    for k in (0, -1):
        with pytest.raises(ValueError):
            env.sample_episodes(t, k)
    assert env._step_index == si


@native_test(emu=None)
def sample_episodes_full_size_ta80(make_env):
    """ta80 at N = 64, k = 1 024, per-env table, from reset: every sample ends done with a finite log_prob, a spread of
    columns equals the twins; the best sample's schedule is feasible, equals a step_logits twin's, and the twin's
    actions replayed through the CPU oracle give the same makespan and solution."""
    import torch
    n, k = 64, 1024
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=15)
    env.reset()
    J, M = env.jobs, env.machines
    table = torch.randn((n, J, M), generator=torch.Generator(device=env.device).manual_seed(23), device=env.device)
    si = env._step_index
    out = env.sample_episodes(table, k, solution=True)
    ms, lp = np_(out["makespan"]), np_(out["log_prob"])
    assert (ms > 0).all() and np.isfinite(lp).all()
    cols = [0, 1, 511, 1023]
    twin = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=15)
    twin.reset()
    snap = snapshot(twin)
    for c in cols:
        twin.import_state(snap)
        twin._step_index = si + c * bound(env)
        l, _ = sample_call(twin, table, grad=False)
        assert np.array_equal(np_(twin.current_time_step), ms[:, c]), c
        assert np.array_equal(l.view(np.uint32), lp[:, c].view(np.uint32)), c
    best, sol = np_(out["best"]), np_(out["solution"])
    inst = load_instance("ta80")
    host = table.cpu().numpy()
    for i in (0, 63):
        b = int(best[i])
        check_schedule(inst, sol[i], int(ms[i, b]))
        one = make_env(1, {"instance_path": "ta80"}, auto_reset=False, record_solution=True, seed=15, env_id_base=i)
        one.reset()
        tw = Twin(one)
        tw.steps(host[i:i + 1], bound(env), si + b * bound(env))
        assert np_(one.done).all() and np.array_equal(np_(one.solution)[0], sol[i]), i
        o = OracleEnv(*inst)
        o.reset()
        done = False
        for a in tw.actions[0]:
            assert not done
            _, _, done, _, _ = o.step(a)
        assert done and o.current_time_step == ms[i, b], i
        assert np.array_equal(np.asarray(o.solution), sol[i]), i
        one.close()


@native_test(emu=None)
def sample_episodes_score_function_identity(make_env):
    """E[grad log p] = 0: one ta01 env from reset, a (1, J, M) table, k = 4 096 samples.  The backward with weights
    1/64 on one group of 64 samples gives that group's mean gradient; over 64 groups the per-entry mean is zero within
    its standard error (chi-square of the z-scores over the entries with non-zero variance)."""
    import torch
    from scipy.stats import chi2
    env = make_env(1, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    env.reset()
    J, M = env.jobs, env.machines
    table = torch.randn((1, J, M), generator=torch.Generator().manual_seed(1)).to(env.device)
    k, groups = 4096, 64
    si = env._step_index
    out = env.sample_episodes(table, k)
    assert np.isfinite(np_(out["log_prob"])).all()
    means = []
    for gi in range(groups):                             # the mean gradient of samples gi*64 .. gi*64+63
        w = torch.zeros((1, k), device=env.device)
        w[0, gi * (k // groups):(gi + 1) * (k // groups)] = 1.0 / (k // groups)
        means.append(np_(env._sample_episodes_grad(table, k, si, w, 8).sum(0))[0].astype(np.float64))
    means = np.stack(means)
    mean, sd = means.mean(0), means.std(0, ddof=1)
    live = sd > 0
    z = mean[live] / (sd[live] / np.sqrt(groups))
    assert live.sum() > J * M // 2
    assert chi2.sf(float((z ** 2).sum()), int(live.sum())) > 1e-6


@native_test(emu=None)
def sample_episodes_first_decision_distribution(make_env):
    """k = 65 536 samples of one env from reset, on an instance where every job starts on machine 0 and a table whose
    second operations never compete with a first one: each sample's log_prob is that of the order in which the jobs take
    machine 0, a Plackett-Luce draw from the softmax of the first operations' entries.  The first job of each sample
    against the softmax, and the 24 orders against their probabilities, by chi-square."""
    import itertools
    import torch
    from scipy.stats import chisquare
    J = 4
    inst = (np.array([[0, 1]] * J, np.int32), np.array([[3, 1]] * J, np.int32))
    env = make_env(1, batch_cfg([inst]), auto_reset=False, seed=21)
    env.reset()
    x = np.array([0.0, 0.45, 1.05, -0.35])                # the 24 orders' log-probabilities lie >= 0.017 apart
    table = np.zeros((1, J, 2), np.float32)
    table[0, :, 0] = x
    table[0, :, 1] = -1e4 * np.arange(1, J + 1)           # deterministic among themselves, never against a first op
    k = 65536
    out = env.sample_episodes(torch.from_numpy(table).to(env.device), k)
    lp = np_(out["log_prob"])[0].astype(np.float64)
    perms = list(itertools.permutations(range(J)))
    plp = []
    for pi in perms:
        rest, v = list(range(J)), 0.0
        for j in pi:
            v += x[j] - np.log(np.exp(x[rest]).sum())
            rest.remove(j)
        plp.append(v)
    plp = np.array(plp)
    assert np.diff(np.sort(plp)).min() > 1e-3
    idx = np.abs(lp[:, None] - plp[None, :]).argmin(1)
    assert (np.abs(lp - plp[idx]) < 1e-4).all()
    hist = np.bincount(idx, minlength=len(perms))
    assert chisquare(hist, np.exp(plp) * k).pvalue > 1e-6, hist
    first = np.array([pi[0] for pi in perms])[idx]
    p0 = np.exp(x - np.log(np.exp(x).sum()))
    assert chisquare(np.bincount(first, minlength=J), p0 * k).pvalue > 1e-6
