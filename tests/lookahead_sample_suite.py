"""The tests of jss_lookahead_sample (every legal action valued by k episodes drawn from a caller's logit table after it,
the envs left untouched), declared once for both backends (tests/backends.py) and collected by
tests/test_emu_lookahead_sample.py and tests/test_gpu_lookahead_sample.py.  The values are checked against their
definition on a twin batch: the same state imported, the candidate stepped, then sample_episodes(table, k) at the same
RNG counter; and, for a table whose gaps exceed the Gumbel noise, against lookahead_priority of its ranks."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.lookahead_priority_suite import (BIG_GPU, EMU_CLASSES, NONPERM, SHAPES, SMALL, TINY, noop_only,
                                            shaped_table)
from tests.lookahead_suite import _outputs, check_table, random_walk, snapshot
from tests.parity_common import batch_cfg, np_, synthetic_instance
from tests.priority_suite import random_table

# a k above every split: the split is at most the resident CTAs of the device (2 under emulation, 8 per SM at most on
# an H100's 132 SMs)
K_BIG = {"emu": 5, "gpu": 1500}


def bound(env):
    return 2 * env.jobs * env.machines + 1


def twin_values(make_env, env, table, k, step_index):
    """The (N, J+1, k) values lookahead_sample(table, k) at RNG counter step_index must return in env's current state,
    by their definition on a twin batch: for each candidate column, import the state, step the candidate, and run
    sample_episodes(table, k) at step_index; a candidate that ends the episode holds its end time in every column, and
    a candidate step that sets the error bit reads -1."""
    import torch
    n, J = env.num_envs, env.jobs
    cfg = {"instance_paths": [env.instances[i] for i in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    twin = make_env(n, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed)
    twin.reset()
    snap = snapshot(env)
    dev = lc._to_dev(twin, table)
    legal = np_(env.action_mask)[:, :J + 1].astype(bool) & ~np_(env.done)[:, None]
    err0 = (np_(env.flags) & N.FLAG_ERROR) != 0
    out = np.full((n, J + 1, k), -1, np.int64)
    for a in range(J + 1):
        cand = legal[:, a]
        if not cand.any():
            continue
        twin.import_state(snap)
        twin.step(torch.full((n,), a, dtype=torch.int32, device=env.device))
        done, t = np_(twin.done).copy(), np_(twin.current_time_step).copy()
        err = ((np_(twin.flags) & N.FLAG_ERROR) != 0) & ~err0
        twin._step_index = step_index
        ms = np_(twin.sample_episodes(dev, k)["makespan"]).astype(np.int64)
        go = cand & ~done & ~err
        out[go, a] = ms[go]
        out[cand & done, a] = t[cand & done, None]
    twin.close()
    return out


def values(env, table, k, **kw):
    """lookahead_sample of a host table; the counter must advance by k*B.  Returns the dict and the counter used."""
    si = env._step_index
    r = env.lookahead_sample(lc._to_dev(env, table), k, **kw)
    assert env._step_index == si + k * bound(env)
    return r, si


def check_summaries(r):
    """"mean" and "min" from "makespan": over the samples that ended, NaN / -1 where none did."""
    ms = np_(r["makespan"]).astype(np.int64)
    ended = ms >= 0
    cnt = ended.sum(2)
    with np.errstate(invalid="ignore"):
        mean = (np.where(ended, ms, 0).sum(2) / cnt).astype(np.float32)
    best = np.where(cnt > 0, np.where(ended, ms, np.iinfo(np.int64).max).min(2), -1)
    got_mean = np_(r["mean"])
    assert r["mean"].dtype.is_floating_point and got_mean.dtype == np.float32
    assert np.array_equal(np.isnan(got_mean), cnt == 0)
    assert np.array_equal(got_mean[cnt > 0], mean[cnt > 0])
    assert np_(r["min"]).dtype == np.int32 and np.array_equal(np_(r["min"]), best)


def check_twin(make_env, names, table_of, k, walk, seed, craft_noop=False):
    """Values after `walk` random decisions against the twin's, for the table table_of(env).  With craft_noop, the first
    env that is not done is first given only the no-op as legal action, through the snapshot interface."""
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=5)
    env.reset()
    random_walk(env, walk)
    if craft_noop:
        i = int(np.flatnonzero(~np_(env.done))[0])
        x = env.export_state()
        x["legal"][i] = 0
        x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
        env.import_state(x)
    table = table_of(env)
    r, si = values(env, table, k)
    q = np_(r["makespan"]).astype(np.int64)
    want = twin_values(make_env, env, table, k, si)
    for s in range(k):
        check_table(env, q[:, :, s], want[:, :, s], (walk, k, s, table.shape))
    for i, Ji in enumerate(env.env_jobs):
        assert (q[i, Ji + 1:] == -1).all(), i          # the default table is filled with -1
    check_summaries(r)
    return env, q


@native_test(emu=[("NJM", 3), ("NJ1", 1), ("1JM", 1)], gpu=[(s, k) for s in SHAPES for k in (1, 3)])
def lookahead_sample_twin(make_env, backend, shape, k):
    """Every lane class in one batch (129..256 jobs and a non-permutation instance included) at reset and mid-episode,
    with some envs done and one with only the no-op legal; and uniform tiny batches (J <= 4).  env_id_base = 5."""
    if backend == "emu":
        names, walk = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170
    else:
        names, walk = ["ta01", "ta11", "ta21", "ta31", "ta41", "ta51", "ta61", "ta71", "ta80", NONPERM, BIG_GPU,
                       SMALL, TINY] * 2, 400
    seed = SHAPES.index(shape) + 20 * k
    table_of = lambda env: shaped_table(env, seed, False, shape)  # noqa: E731
    _, q = check_twin(make_env, names, table_of, k, 0, seed)
    assert (q >= 0).any()
    env, q = check_twin(make_env, names, table_of, k, walk, seed, craft_noop=True)
    done = np_(env.done)
    assert done.any() and not done.all() and noop_only(env).any(), done
    assert (q[done] == -1).all() and (q[~done] >= 0).any()
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        check_twin(make_env, [synthetic_instance(J, M, J * 10 + M)] * 3, table_of, k, J, seed)


@native_test()
def lookahead_sample_more_samples_than_split(make_env, backend):
    """A k above the split, so that a work item takes several samples of one candidate, on uniform tiny batches and
    with ties in the table."""
    k = K_BIG[backend]
    for J, M in ((2, 2), (3, 4)):
        for ties in (False, True):
            check_twin(make_env, [synthetic_instance(J, M, J * 10 + M)] * 3,
                       lambda env: random_table(env, 7, ties), k, 1, 7)  # noqa: B023


@native_test()
def lookahead_sample_split_invariance(make_env, backend):
    """The same envs, states and counters give the same values in a batch of 3 (one tile, so that its pairs are split
    over several work items) and in a large batch (S = 1: the tiles fill the SMs), per-env and broadcast tables alike."""
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
        small._step_index = big._step_index
        rb, _ = values(big, tb, 3)
        rs, _ = values(small, ts, 3)
        qb, qs = np_(rb["makespan"]), np_(rs["makespan"])
        assert np.array_equal(qb[:3], qs), tb.shape
        assert (qs >= 0).any()


def rank_table(env, seed):
    """Per env a random permutation of 0 .. J M - 1 as an (N, J, M) float32 table."""
    rng = np.random.default_rng(seed)
    n, J, M = env.num_envs, env.jobs, env.machines
    return np.stack([rng.permutation(J * M).reshape(J, M) for _ in range(n)]).astype(np.float32)


@native_test()
def lookahead_sample_deterministic_limit(make_env, backend):
    """Distinct ranks times 64: the gaps exceed the range of the Gumbel noise (below 21), so every draw is the table's
    argmax and every sample equals lookahead_priority of the ranks, at reset and mid-episode."""
    names = {"emu": ["ta01", SMALL, NONPERM, TINY, EMU_CLASSES[0]],
             "gpu": ["ta01", "ta41", "ta80", NONPERM, BIG_GPU, SMALL] * 4}[backend]
    for walk in (0, 50):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=6)
        env.reset()
        random_walk(env, walk)
        ranks = rank_table(env, walk)
        want = np_(env.lookahead_priority(lc._to_dev(env, ranks))).copy()
        r, _ = values(env, ranks * 64, 4)
        q = np_(r["makespan"])
        for s in range(4):
            assert np.array_equal(q[:, :, s], want), (walk, s)
        assert (want >= 0).any()


@native_test()
def lookahead_sample_bad_tables(make_env, backend):
    """NaN, +inf and all-(-inf) entries on operations some samples reach: exactly the pairs whose path meets one read
    -1 (the twin's rule), no flag changes and the call returns normally.  Entries that are never read (finished
    operations, columns past J_i, operations past M_i) change nothing."""
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
    k = 2
    flags = np_(env.flags).copy()
    r, si = values(env, bad, k)
    q = np_(r["makespan"]).copy()
    assert np.array_equal(np_(env.flags), flags)
    assert not (flags & N.FLAG_ERROR).any()
    want = twin_values(make_env, env, bad, k, si)
    for s in range(k):
        check_table(env, q[:, :, s], want[:, :, s], ("bad", s))
    env._step_index = si
    ok = np_(values(env, clean, k)[0]["makespan"]).copy()
    assert (ok[mask] >= 0).all()
    for i in (0, 1):                                      # only the candidate that takes the bad job skips its entry
        cols = np.flatnonzero(mask[i])
        assert np.array_equal(q[i, jobs[i]], ok[i, jobs[i]]), i
        assert (q[i, cols[cols != jobs[i]]] == -1).all(), i
    assert (q[2][mask[2]] == -1).all()
    assert (q[3][mask[3]] == -1).any()
    for i in (4, 5, 6):
        assert np.array_equal(q[i], ok[i]), i


@native_test(emu=[False, True], gpu=[False, True])
def lookahead_sample_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and the flags are bit-identical after the call, and the RNG
    counter advances by exactly k*B; one launch per lane class present; a caller's `out` is written and returned."""
    import torch
    names = ["ta01", NONPERM, "ta01", SMALL] if backend == "emu" else ["ta01", "ta51", "ta80", NONPERM] * 8
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, record_solution=True, seed=8)
    env.reset()
    random_walk(env, 60)
    before, stats = _outputs(env), env.stats()
    c = env.launch_count
    for table, k in ((random_table(env, 4), 2), (random_table(env, 5, ties=True)[:1], 3)):
        values(env, table, k)
    assert env.launch_count == c + 2 * (2 if backend == "emu" else 3)   # one launch per lane class present
    after = _outputs(env)
    for key, v in before.items():
        assert np.array_equal(v, after[key]), key
    assert env.stats() == stats
    si = env._step_index
    want = np_(values(env, random_table(env, 6), 2)[0]["makespan"]).copy()
    env._step_index = si
    out = torch.full((env.num_envs, env.jobs + 1, 2), -777, dtype=torch.int32, device=env.device)
    r, _ = values(env, random_table(env, 6), 2, out=out)
    assert r["makespan"] is out
    o = np_(out)
    for i, Ji in enumerate(env.env_jobs):
        assert np.array_equal(o[i, :Ji + 1], want[i, :Ji + 1]), i
        assert (o[i, Ji + 1:] == -777).all(), i


@native_test()
def lookahead_sample_abi(make_env, backend):
    """JSS_ERR_INVALID, launching nothing, for a NULL or misaligned table or output, a negative stride, k < 1, k*B past
    2^64 and ld < (jobs_max + 1) k; JSS_ERR_UNSUPPORTED for k >= 2^31 and tiles * (jobs_max + 1) * k >= 2^31;
    JSS_ERR_STATE before jss_assign; a bad table shape, k or out raises ValueError before the native call; a table that
    requires grad is read detached."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    L, h, st = env._L, env._h, env._stream()
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    out = torch.zeros((n, J + 1, 4), dtype=torch.int32, device=env.device)
    p, o = t.data_ptr(), out.data_ptr()
    s, ld = (J * M, M, 1), (J + 1) * 4
    huge = 1 << 62
    c = env.launch_count
    for args in ((None, *s, 4, o, ld), (p + 2, *s, 4, o, ld), (p, -1, M, 1, 4, o, ld), (p, J * M, -M, 1, 4, o, ld),
                 (p, J * M, M, -1, 4, o, ld), (p, *s, 0, o, ld), (p, *s, -3, o, ld), (p, *s, huge, o, huge),
                 (p, *s, 4, None, ld), (p, *s, 4, o + 2, ld), (p, *s, 4, o, ld - 1), (p, *s, 4, o, 4)):
        assert L.jss_lookahead_sample(h, *args[:4], 0, 0, *args[4:], st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_lookahead_sample:"), args
    for k in (1 << 31, (1 << 31) // (J + 1) + 1):          # k itself, and the work items of the one tile
        assert L.jss_lookahead_sample(h, p, *s, 0, 0, k, o, (J + 1) * k, st) == -4, k
        assert L.jss_last_error(h).startswith(b"jss_lookahead_sample:"), k
    assert env.launch_count == c
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_lookahead_sample(raw, p, *s, 0, 0, 4, o, ld, st) == -5
    L.jss_destroy(raw)
    si = env._step_index
    for bad in (t[0], t[None], t[:, :J - 1], torch.zeros((3, J, M), device=env.device), t[:, :, :M - 1]):
        with pytest.raises(ValueError):
            env.lookahead_sample(bad, 2)
    for k in (0, -1):
        with pytest.raises(ValueError):
            env.lookahead_sample(t, k)
    for bad_out in (out[:, :J], out.to(torch.int64), out[:, :, :3], torch.zeros((3, J + 1, 4), dtype=torch.int32,
                                                                                 device=env.device),
                    out.transpose(0, 2).contiguous().transpose(0, 2), out.view(n, -1), [[0]]):
        with pytest.raises(ValueError):
            env.lookahead_sample(t, 4, out=bad_out)
    assert env._step_index == si and env.launch_count == c
    table = lc._to_dev(env, random_table(env, 17))
    want = np_(env.lookahead_sample(table, 3)["makespan"]).copy()
    env._step_index = si
    g = table.double().requires_grad_(True)
    r = env.lookahead_sample(g, 3)
    assert np.array_equal(np_(r["makespan"]), want)
    assert g.grad is None and not r["mean"].requires_grad


@native_test(emu=None)
def lookahead_sample_full_size_ta80(make_env):
    """ta80 at N = 256 after 500 random decisions with a finite random table and k = 4: no -1 on a legal column, -1 on
    every illegal one, and a few sampled envs equal to their twins."""
    import torch
    n, k = 256, 4
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=14)
    env.reset()
    random_walk(env, 500)
    table = torch.rand((n, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(22),
                       device=env.device)
    r, si = values(env, table.cpu().numpy(), k)
    q, mask = np_(r["makespan"]), np_(env.action_mask)[:, :env.jobs + 1].astype(bool)
    assert (q[mask] >= 0).all()
    assert (q[~mask] == -1).all()
    want = twin_values(make_env, env, table.cpu().numpy(), k, si)
    assert np.array_equal(q.astype(np.int64), want)
