"""The tests of jss_stochastic_beam_step (one stochastic-beam-search round per group of W envs from per-beam logit rows)
and ObsBeamSearch(stochastic=True), declared once for both backends (tests/backends.py) and collected by
tests/test_emu_stochastic_beam_step.py and tests/test_gpu_stochastic_beam_step.py.  A search driven with rows gathered
from a table at each slot's todo must equal jss_sample_without_replacement of that table bit for bit, on a G-env batch
with env_id_base / W at the same seed and counter; every round's written slots must equal twins stepped one env at a
time; with rows that depend on the observation, slot 0 must follow the policy's distribution over complete episodes."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.beam import ObsBeamSearch
from tests.backends import native_test
from tests.beam_search_suite import enumerate_sequences, twin_of
from tests.beam_step_suite import beam_batch, crafted, gathered_rows, record
from tests.lookahead_priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, SHAPES, SMALL, TINY, shaped_table
from tests.lookahead_suite import snapshot
from tests.parity_common import batch_cfg, np_
from tests.priority_suite import random_table
from tests.swor_suite import replay_slots, seq_order, swor, tiny_instances


def rebased(make_env, base):
    """`make_env` with env_id_base = base (beam_batch builds W envs per env with the env's own base)."""
    return lambda *a, **k: make_env(*a, **{**k, "env_id_base": base})


def sbatch(make_env, env, W, walk=7):
    """beam_batch of `env` on a batch with env_id_base = W * env.env_id_base, so that group g has env g's global id."""
    return beam_batch(rebased(make_env, W * env.env_id_base), env, W, walk)


def sdrive(big, table, W, each=None, policy=None):
    """ObsBeamSearch(stochastic=True) on `big` with rows gathered from `table` (or `policy(big)`); `each(search)` after
    every round.  The counter must advance by J*M at start().  Returns the result (every slot's order) as numpy arrays
    and the counter c of round 0."""
    si = big._step_index
    s = ObsBeamSearch(big, W, stochastic=True).start()
    c = s._counter
    assert big._step_index == c + big.jobs * big.machines and c >= si
    while not s.done:
        s.step(policy(big) if policy else gathered_rows(big, table, W))
        if each:
            each(s)
    return {k: np_(v).copy() for k, v in s.result(order=True, all_orders=True).items()}, c


def check_parity(make_env, env, table, W, walk=7):
    """The stochastic search driven on W envs per env equals sample_without_replacement(table, W) on env (which has the
    groups' global ids and the seed) at the search's counter: makespan, score = log_prob and key (bits), best and every
    slot's order."""
    big = sbatch(make_env, env, W, walk)
    got, c = sdrive(big, table, W)
    env._step_index = c
    want, _ = swor(env, table, W)
    assert np.array_equal(got["makespan"], want["makespan"]), (got["makespan"], want["makespan"])
    for a, b in (("score", "log_prob"), ("key", "key")):
        assert np.array_equal(got[a].view(np.uint32), want[b].view(np.uint32)), (a, got[a], want[b])
    assert np.array_equal(got["best"], want["best"])
    for i in range(env.num_envs):
        Ji, Mi = env.env_jobs[i], env.env_machines[i]
        assert np.array_equal(got["orders"][i, :, :Ji, :Mi], want["order"][i, :, :Ji, :Mi]), i
    big.close()
    return got


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def stochastic_beam_step_parity(make_env, backend, shape, ties):
    """Every lane class at reset and mid-episode (a done env and one with only the no-op legal), (N, J, M), (N, J, 1)
    and (1, J, M) tables with ties: bit-identical to sample_without_replacement."""
    if backend == "emu":
        names, walk, W = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170, 2
    else:
        names, walk, W = ["ta01", "ta31", "ta51", "ta71", NONPERM, BIG_GPU, SMALL, TINY], 400, 4
    seed = SHAPES.index(shape) + (10 if ties else 0)
    for steps in (0, walk):
        env = crafted(make_env, names, steps, seed)
        if steps:
            assert np_(env.done).any()
        check_parity(make_env, env, shaped_table(env, seed, ties, shape), W)


@native_test(emu=[1, 4, 16, 32], gpu=[1, 4, 16, 32])
def stochastic_beam_step_widths(make_env, backend, width):
    """Widths 1, 4, 16 and 32 at reset and mid-episode, against sample_without_replacement."""
    names = {"emu": [SMALL, TINY, NONPERM], "gpu": ["ta01", "ta41", "ta80", NONPERM, BIG_GPU, TINY]}[backend]
    for steps in (0, 30):
        env = crafted(make_env, names, steps, width)
        check_parity(make_env, env, random_table(env, width, True), width)


@native_test()
def stochastic_beam_step_round_twins(make_env, backend):
    """After each call every written slot equals a twin that imported its parent's pre-call state, stepped the job and
    took the forced no-ops, bit for bit in exported state, real_obs, action_mask and scalar record; empty slots and
    untouched groups are byte-for-byte unchanged, keys included; the statistics, solution, error bit and the env's RNG
    counter do not move during the rounds."""
    import torch
    names = {"emu": [SMALL, TINY, "ta01", EMU_CLASSES[0]], "gpu": ["ta01", "ta41", "ta80", BIG_GPU, TINY] * 2}[backend]
    W = 4
    env = crafted(make_env, names, 0, 5)
    big = beam_batch(rebased(make_env, 0), env, W, record_solution=True)
    twin = twin_of(make_env, big, record_solution=True)
    table = random_table(env, 6, True)
    s = ObsBeamSearch(big, W, stochastic=True).start()
    stats, si, err, rounds = big.stats(), big._step_index, np_(big.flags).copy() & N.FLAG_ERROR, 0
    while not s.done and rounds < 40:
        before = record(big)
        pre = snapshot(big)
        score0, key0 = np_(s.score).copy(), np_(s.key).copy()
        s.step(gathered_rows(big, table, W))
        rounds += 1
        after = record(big)
        parent = np_(s._parent[s._round - 1]).copy()
        job = np_(s._action[s._round - 1]).copy()
        new = (parent >= 0) & (job >= 0)
        n = big.num_envs
        src = np.where(new, (np.arange(n) // W) * W + np.maximum(parent, 0), np.arange(n))
        twin.import_state({k: v[torch.from_numpy(src).to(big.device)].clone() for k, v in pre.items()})
        twin.step(torch.from_numpy(np.where(new, job, N.ACTION_SKIP).astype(np.int32)).to(big.device))
        while True:
            m = np_(twin.action_mask)
            need = new & np.array([not m[i, :Ji].any() and bool(m[i, Ji]) for i, Ji in enumerate(twin.env_jobs)])
            if not need.any():
                break
            twin.step(torch.from_numpy(np.where(need, twin.env_jobs, N.ACTION_SKIP).astype(np.int32)).to(big.device))
        want = record(twin)
        for k in ("real_obs", "action_mask", "reward", "reward_raw", "current_time_step", "flags", "done") + tuple(
                "x_" + k for k in pre):
            if k == "x_t" or k == "x_flags":
                continue
            assert np.array_equal(after[k][new].view(np.uint8), want[k][new].view(np.uint8)), (rounds, k)
            assert np.array_equal(after[k][~new].view(np.uint8), before[k][~new].view(np.uint8)), (rounds, k)
        for k in ("episode_count", "last_makespan", "last_return", "solution"):
            assert np.array_equal(after[k], before[k]), k
        moved = (np.isfinite(score0) & ~before["done"]).reshape(-1, W).any(1)
        untouched = np.repeat(~moved, W)
        assert (parent[untouched] == np.arange(n)[untouched] % W).all() and (job[untouched] == -1).all()
        for now, then in ((s.score, score0), (s.key, key0)):
            assert np.array_equal(np_(now)[untouched].view(np.uint32), then[untouched].view(np.uint32))
        empty = ~new & ~untouched
        assert (parent[empty] == -1).all() and np.isneginf(np_(s.score)[empty]).all()
        assert np.isneginf(np_(s.key)[empty]).all()
        assert np.isfinite(np_(s.key)[new]).all() and (np_(s.key)[new] <= 0).all()
    assert rounds > 0
    assert big.stats()["episodes"] == stats["episodes"] and big._step_index == si
    assert np.array_equal(np_(big.flags) & N.FLAG_ERROR, err)
    twin.close()
    big.close()


def linear_policy(w, temp=1.0):
    """A fixed linear score of real_obs per job, divided by `temp`, with a zero no-op column: (N, J + 1) rows."""
    import torch

    def rows(env):
        x = env.real_obs[:, :env.jobs, :]
        out = torch.zeros((env.num_envs, env.jobs + 1), device=env.device)
        out[:, :env.jobs] = (x @ torch.as_tensor(w, dtype=torch.float32, device=env.device)) / temp
        return out
    return rows


def sequence_probs(make_env, inst, seqs, policy):
    """The float64 probability of each complete job sequence of `inst` from reset under `policy` (rows from the
    observation), by replaying the sequences on a batch of len(seqs) twins one decision at a time (forced no-ops add
    nothing)."""
    import torch
    n = len(seqs)
    env = make_env(n, batch_cfg([inst] * n), auto_reset=False, seed=1)
    env.reset()
    J = env.jobs
    lp = np.zeros(n)
    at = np.zeros(n, np.int64)
    while True:
        m, done = np_(env.action_mask).astype(bool), np_(env.done)
        rows = np_(policy(env)).astype(np.float64)
        act = np.full(n, N.ACTION_SKIP, np.int32)
        for i in range(n):
            if not m[i, :J].any():
                if m[i, J] and not done[i]:
                    act[i] = J                           # forced no-op
                continue
            j = seqs[i][0][at[i]]
            assert m[i, j]
            v = rows[i, :J][m[i, :J]]
            mx = v.max()
            lp[i] += rows[i, j] - mx - np.log(np.exp(v - mx).sum())
            act[i] = j
            at[i] += 1
        if (act == N.ACTION_SKIP).all():
            break
        env.step(torch.from_numpy(act).to(env.device))
    assert np_(env.done).all() and (at == [len(s) for s, _ in seqs]).all()
    env.close()
    return np.exp(lp)


@native_test(emu={"groups": 256}, gpu={"groups": 4096})
def stochastic_beam_step_distribution(make_env, backend, groups):
    """Rows from a fixed linear score of real_obs on a tiny instance: every complete slot of a group is a distinct
    complete sequence of positive probability, and slot 0 over the groups (independent draws in one search) passes a
    chi-square test against the exact probabilities, enumerated by replaying every sequence (bins of expected count
    below 5 pooled)."""
    from scipy.stats import chisquare
    inst, seqs = next((i, s) for i, s in tiny_instances() if 4 <= len(s) <= 12)
    W = 3
    env = make_env(groups, batch_cfg([inst] * groups), auto_reset=False, seed=31)
    env.reset()
    J, M = env.jobs, env.machines
    policy = linear_policy(np.random.default_rng(3).standard_normal(env.real_obs.shape[-1]) * 2.0)
    p = sequence_probs(make_env, inst, seqs, policy)
    assert abs(p.sum() - 1) < 1e-6 and (p > 0).all()
    index = {seq_order(s, J, M).tobytes(): q for q, (s, _) in enumerate(seqs)}
    big = sbatch(make_env, env, W, walk=0)
    out, _ = sdrive(big, None, W, policy=policy)
    first = []
    for g in range(groups):
        full = out["makespan"][g] >= 0
        c = int(full.sum())
        assert c == min(W, len(seqs)) and full[:c].all(), g
        got = [index[out["orders"][g, s].astype(np.int64).tobytes()] for s in range(c)]
        assert len(set(got)) == c
        for s, q in enumerate(got):
            assert out["makespan"][g, s] == seqs[q][1]
        first.append(got[0])
    counts = np.bincount(first, minlength=len(seqs)).astype(np.float64)
    exp = p * groups
    ok = exp >= 5
    f, e = np.append(counts[ok], counts[~ok].sum()), np.append(exp[ok], exp[~ok].sum())
    if e[-1] == 0:
        f, e = f[:-1], e[:-1]
    assert chisquare(f, e * f.sum() / e.sum()).pvalue > 1e-3, (counts, exp)
    big.close()


@native_test()
def stochastic_beam_step_replay(make_env, backend):
    """Every complete slot's order replays with rollout_priority(-order) from the start state to its makespan (a
    feasible schedule), and order_log_prob of the table equals the slot's score bit for bit."""
    from jssenv_b200.instances import load_instance
    names = {"emu": ["ta01", SMALL, TINY, NONPERM], "gpu": ["ta01", "ta21", "ta61", "ta80", NONPERM, TINY] * 2}[backend]
    W = 4
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=2)
    env.reset()
    table = random_table(env, 12)
    out, _ = sdrive(sbatch(make_env, env, W), table, W)
    assert (out["best"] >= 0).all()
    insts = [n if not isinstance(n, str) else load_instance(n) for n in names]
    replay_slots(make_env, env, {"makespan": out["makespan"], "order": out["orders"], "log_prob": out["score"]}, table,
                 insts)


@native_test()
def stochastic_beam_step_determinism_and_shards(make_env, backend):
    """Two identical runs are bit-identical; another counter or seed changes the draws; two shards with env_id_base =
    0 and G1 * W equal the unsharded batch."""
    names = {"emu": [SMALL, TINY, NONPERM, SMALL], "gpu": ["ta01", "ta41", "ta80", NONPERM, TINY, "ta21"]}[backend]
    W = 4

    table = None

    def run(lo=0, hi=len(names), seed=6, counter=0):
        nonlocal table
        env = make_env(hi - lo, batch_cfg(names[lo:hi], sort=False), auto_reset=False, seed=seed, env_id_base=lo)
        env.reset()
        if table is None:
            table = random_table(env, 9)
        big = sbatch(make_env, env, W)
        big._step_index = counter
        out, c = sdrive(big, np.ascontiguousarray(table[lo:hi, :env.jobs, :env.machines]), W)
        assert c == counter
        big.close()
        return out, env

    ref, env = run()
    again, _ = run()
    for k in ref:
        assert np.array_equal(ref[k].view(np.uint8), again[k].view(np.uint8)), k
    for other, _ in (run(counter=5), run(seed=7)):
        assert not np.array_equal(other["key"].view(np.uint32), ref["key"].view(np.uint32))
    cut = len(names) // 2
    for lo, hi in ((0, cut), (cut, len(names))):
        so, sh = run(lo, hi)
        for k in ("makespan", "score", "key"):
            assert np.array_equal(so[k].view(np.uint8), ref[k][lo:hi].view(np.uint8)), k
        for i in range(hi - lo):
            Ji, Mi = sh.env_jobs[i], sh.env_machines[i]
            assert np.array_equal(so["orders"][i, :, :Ji, :Mi], ref["orders"][lo + i, :, :Ji, :Mi]), i


@native_test(emu=None)
def stochastic_beam_step_side_stream(make_env):
    """A search run on a side stream equals the same search on the default stream, bit for bit."""
    import torch
    names = ["ta01", "ta41", "ta80", NONPERM] * 2
    W = 4
    outs = []
    for side in (False, True):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
        env.reset()
        table = random_table(env, 3)
        big = sbatch(make_env, env, W)
        if side:
            stream = torch.cuda.Stream()
            stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(stream):
                out, _ = sdrive(big, table, W)
            torch.cuda.current_stream().wait_stream(stream)
        else:
            out, _ = sdrive(big, table, W)
        outs.append(out)
    for k in outs[0]:
        assert np.array_equal(outs[0][k].view(np.uint8), outs[1][k].view(np.uint8)), k


@native_test()
def stochastic_beam_step_bad_rows_and_dead_groups(make_env, backend):
    """A bad row in one beam drops it and sets the group's bad bit; bad rows in every beam empty the group and the
    result reads -1 / NaN / NaN; a group whose slots all start dead is untouched (scores and keys); a group done at
    start() reads -1 / 0 / 0."""
    import torch
    env = make_env(4, batch_cfg([SMALL, SMALL, TINY, TINY], sort=False), auto_reset=False, seed=4)
    env.reset()
    while not np_(env.done)[3]:                          # group 3: done at start
        a = env.policy("RANDOM")
        a[:3] = N.ACTION_SKIP
        env.step(a)
    W = 4
    big = sbatch(make_env, env, W)
    table = random_table(env, 4)
    s = ObsBeamSearch(big, W, stochastic=True).start()
    s.score[2 * W] = float("-inf")                       # group 2: every slot dead
    s.step(gathered_rows(big, table, W))
    s.step(gathered_rows(big, table, W))
    sc = np_(s.score).reshape(4, W)
    live = np.isfinite(sc)
    assert live[0].sum() >= 2 and live[1].sum() >= 2 and not live[2].any()
    rows = gathered_rows(big, table, W)
    b = int(np.flatnonzero(live[0])[0])
    j = int(np.flatnonzero(np_(big.action_mask)[b, :big.env_jobs[b]])[0])
    rows[b, j] = float("nan")                            # group 0: one beam's row bad
    rows[W:2 * W] = float("inf")                         # group 1: every beam's row bad
    before, key0 = np_(big.real_obs).copy(), np_(s.key).copy()
    parent, action, bad = (np_(t).copy() for t in big.stochastic_beam_step(rows, W, s.score, s.key,
                                                                            s._counter + s._round))
    assert list(bad) == [1, 1, 0, 0]
    assert (parent[W:2 * W] == -1).all() and np.isneginf(np_(s.score)[W:2 * W]).all()
    assert np.isneginf(np_(s.key)[W:2 * W]).all()
    assert b not in parent[:W] and (parent[:W] >= 0).any()
    assert (parent[2 * W:] == np.tile(np.arange(W), 2)).all() and (action[2 * W:] == -1).all()
    assert np.array_equal(np_(big.real_obs)[2 * W:], before[2 * W:])
    assert np.array_equal(np_(s.key)[2 * W:].view(np.uint32), key0[2 * W:].view(np.uint32))
    s._bad |= torch.as_tensor(bad, device=big.device)
    s._round += 1
    while not s.done:
        s.step(gathered_rows(big, table, W))
    out = {k: np_(v) for k, v in s.result().items()}
    assert (out["makespan"][1] == -1).all() and np.isnan(out["score"][1]).all() and np.isnan(out["key"][1]).all()
    assert out["best"][1] == -1 and (out["makespan"][0] >= 0).any()
    assert (out["makespan"][2] == -1).all() and np.isneginf(out["score"][2]).all() and np.isneginf(out["key"][2]).all()
    assert (out["makespan"][3] == -1).all() and (out["score"][3] == 0).all() and (out["key"][3] == 0).all()


@native_test()
def stochastic_beam_step_abi(make_env, backend):
    """JSS_ERR_INVALID for a NULL or misaligned key, env_id_base not a multiple of the width, a width that does not
    divide N, a group that mixes instances, and what jss_beam_step rejects; JSS_ERR_STATE before jss_assign;
    ValueError from the wrappers; an auto-reset env is refused by start(); one launch per lane class present; the
    default ObsBeamSearch has no key."""
    import pytest
    import torch
    env = make_env(8, batch_cfg(["ta01"] * 4 + [SMALL] * 4, sort=False), auto_reset=False, seed=1, env_id_base=8)
    env.reset()
    n, J = env.num_envs, env.jobs
    L, h, st = env._L, env._h, env._stream()
    rows = torch.zeros((n, J + 1), device=env.device)
    sc = torch.full((n,), float("-inf"), device=env.device)
    sc[::4] = 0.0
    ky = sc.clone()
    p_, a_, b_ = (torch.zeros(n, dtype=torch.int32, device=env.device) for _ in range(3))
    r, s, k, pp, ap, bp = rows.data_ptr(), sc.data_ptr(), ky.data_ptr(), p_.data_ptr(), a_.data_ptr(), b_.data_ptr()
    bad = ((r, J + 1, 4, s, None, pp, ap, bp), (r, J + 1, 4, s, k + 2, pp, ap, bp),
           (r, J + 1, 8, s, k, pp, ap, bp), (r, J + 1, 3, s, k, pp, ap, bp), (r, J + 1, 0, s, k, pp, ap, bp),
           (None, J + 1, 4, s, k, pp, ap, bp), (r, J, 4, s, k, pp, ap, bp), (r, J + 1, 4, None, k, pp, ap, bp),
           (r, J + 1, 4, s, k, pp, ap, None))
    for lg, ld, w, *bufs in bad:
        assert L.jss_stochastic_beam_step(h, lg, ld, w, 7, 0, *bufs, st) == -1, (lg, ld, w, bufs)
        assert L.jss_last_error(h).startswith(b"jss_stochastic_beam_step:"), (w, bufs)
    assert L.jss_stochastic_beam_step(h, r, J + 1, 4, 7, 0, s, k, pp, ap, bp, st) == 0
    assert L.jss_stochastic_beam_step(h, r, J + 1, 2, 7, 0, s, k, pp, ap, bp, st) == 0
    odd = make_env(8, batch_cfg(["ta01"] * 8), auto_reset=False, seed=1, env_id_base=2)
    odd.reset()
    assert L.jss_stochastic_beam_step(odd._h, r, J + 1, 4, 7, 0, s, k, pp, ap, bp, st) == -1
    assert b"env_id_base" in L.jss_last_error(odd._h)
    with pytest.raises(ValueError):
        odd.stochastic_beam_step(rows, 4, sc, ky, 0)
    with pytest.raises(ValueError):
        ObsBeamSearch(odd, 4, stochastic=True).start()
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_stochastic_beam_step(raw, r, J + 1, 2, 7, 0, s, k, pp, ap, bp, st) == -5
    L.jss_destroy(raw)
    for w in (0, 3, 33):
        with pytest.raises(ValueError):
            env.stochastic_beam_step(rows, w, sc, ky, 0)
    with pytest.raises(ValueError):
        env.stochastic_beam_step(rows, 4, sc, ky.double(), 0)
    with pytest.raises(ValueError):
        env.stochastic_beam_step(rows, 4, sc, ky[:4], 0)
    with pytest.raises(ValueError):
        ObsBeamSearch(env, 8, stochastic=True)           # mixes instances
    ar = make_env(4, {"instance_path": "ta01"}, auto_reset=True)
    with pytest.raises(ValueError):
        ObsBeamSearch(ar, 2, stochastic=True).start()
    mixed = make_env(8, batch_cfg(["ta01"] * 4 + [EMU_CLASSES[0]] * 4, sort=False), auto_reset=False, seed=1)
    mixed.reset()
    c, si = mixed.launch_count, mixed._step_index
    mixed.stochastic_beam_step(torch.zeros((8, mixed.jobs + 1), device=mixed.device), 4, sc.clone(), ky.clone(), 3)
    assert mixed.launch_count == c + 2 and mixed._step_index == si
    plain = ObsBeamSearch(mixed, 4).start()
    assert plain.key is None and mixed._step_index == si
    plain.step(torch.zeros((8, mixed.jobs + 1), device=mixed.device))
    assert "key" not in plain.result()


@native_test(emu=None)
def stochastic_beam_step_full_size_ta80(make_env):
    """ta80 at G = 256, W = 16 from reset: bit-identical to sample_without_replacement, every group's complete slots
    distinct, and every slot's order replays to its makespan."""
    import torch
    G, W = 256, 16
    env = make_env(G, {"instance_path": "ta80"}, auto_reset=False, seed=15, env_id_base=G)
    env.reset()
    table = torch.randn((G, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(23),
                        device=env.device).cpu().numpy()
    out = check_parity(make_env, env, table, W, walk=0)
    for g in range(G):
        c = int((out["makespan"][g] >= 0).sum())
        assert c == W and len({out["orders"][g, s].tobytes() for s in range(c)}) == c, g
    replay_slots(make_env, env, {"makespan": out["makespan"], "order": out["orders"], "log_prob": out["score"]})
