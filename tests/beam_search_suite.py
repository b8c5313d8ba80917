"""The tests of jss_beam_search (a caller's logit table decoded by beam search, the envs left untouched), declared once
for both backends (tests/backends.py) and collected by tests/test_emu_beam_search.py and tests/test_gpu_beam_search.py.
The best slot's order is replayed greedily on a twin (rollout_priority(-order)); width 1 is checked against the greedy
decode, tiny instances against an exhaustive enumeration on the CPU oracle, and whole searches against a float64 beam
search restated on the host over N*W twins (export, gather, select, import, step)."""
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
from tests.priority_suite import random_table
from tests.sample_episodes_suite import check_schedule


def search(env, table, width, order=True):
    """beam_search of a host (or device) table; the RNG counter must not move.  Returns the outputs as numpy arrays."""
    si = env._step_index
    out = env.beam_search(lc._to_dev(env, table) if isinstance(table, np.ndarray) else table, width, order=order)
    assert env._step_index == si
    return {k: np_(v).copy() for k, v in out.items()}


def twin_of(make_env, env, reps=1, **kw):
    """A batch with env's instances (each env repeated `reps` times), reset."""
    cfg = {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
           "env_to_instance": list(np.repeat(np.asarray(env.env_to_instance), reps))}
    twin = make_env(env.num_envs * reps, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed, **kw)
    twin.reset()
    return twin


def rounds(snap, env):
    """R_i: the operations not started in each env's state."""
    todo, tufco = np_(snap["todo"]).astype(np.int64), np_(snap["tufco"]).astype(np.int64)
    R = np.zeros(env.num_envs, np.int64)
    for i, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        R[i] = np.maximum(0, Mi - todo[i, :Ji] - (tufco[i, :Ji] > 0)).sum()
    return R


def replay(make_env, env, out):
    """Identity 1: rollout_priority(-order) from env's state on a twin with record_solution ends done at
    makespan[best] for every env with a complete beam.  Returns the twin's solution table."""
    import torch
    twin = twin_of(make_env, env, record_solution=True)
    twin.import_state(snapshot(env))
    twin.rollout_priority(torch.from_numpy(-out["order"].astype(np.float32)).to(env.device))
    best = out["best"]
    ok = best >= 0
    done, t = np_(twin.done), np_(twin.current_time_step)
    assert done[ok].all(), np.flatnonzero(ok & ~done)
    want = out["makespan"][np.arange(env.num_envs), np.maximum(best, 0)]
    assert np.array_equal(t[ok], want[ok]), (t[ok], want[ok])
    assert (out["order"][~ok] == -1).all()
    sol = np_(twin.solution).copy()
    twin.close()
    return sol


def order_log_prob(make_env, env, table, order):
    """The float64 log-likelihood under `table` of the sequence each env's `order` encodes (the greedy decode of
    -order), from env's state, stepped on a twin one decision at a time; forced no-ops add 0.  NaN where the order is
    all -1."""
    import torch
    n, J = env.num_envs, env.jobs
    twin = twin_of(make_env, env)
    twin.import_state(snapshot(env))
    tab = np.broadcast_to(np.asarray(table, np.float64), (n, J, env.machines))
    lp = np.zeros(n)
    live = (order.reshape(n, -1) >= 0).any(1) & ~np_(env.done)
    while True:
        x = twin.export_state()
        legal, todo = np_(x["legal"]).astype(bool)[:, :J], np_(x["todo"]).astype(np.int64)
        done = np_(twin.done)
        act = np.full(n, N.ACTION_SKIP, np.int32)
        for i in np.flatnonzero(live & ~done):
            Ji = int(env.env_jobs[i])
            lg = np.flatnonzero(legal[i, :Ji])
            if not lg.size:
                act[i] = Ji                              # forced no-op
                continue
            ks = todo[i, lg]
            j = int(lg[np.argmax(-order[i, lg, ks])])
            v = tab[i, lg, ks]
            mx = v.max()
            lp[i] += tab[i, j, todo[i, j]] - mx - np.log(np.exp(v - mx).sum())
            act[i] = j
        if (act == N.ACTION_SKIP).all():
            break
        twin.step(torch.from_numpy(act).to(env.device))
    twin.close()
    return np.where(live, lp, np.nan)


def check_scores(make_env, env, table, out):
    """Identity 4 for the best slot and the shape of the score rows: complete slots first, scores non-increasing, the
    best slot's score within 1e-5 (1 + R) of its order's float64 log-likelihood."""
    sc, ms = out["score"], out["makespan"]
    R = rounds(snapshot(env), env)
    done = np_(env.done)
    for i in range(env.num_envs):
        if done[i]:
            assert (ms[i] == -1).all() and (sc[i] == 0).all(), i
            continue
        full = ms[i] >= 0
        if not full.any():
            continue
        k = int(full.sum())
        assert full[:k].all() and np.isneginf(sc[i, k:]).all(), i
        assert (np.diff(sc[i, :k].astype(np.float64)) <= 0).all(), (i, sc[i])
    want = order_log_prob(make_env, env, table, out["order"])
    b = out["best"]
    for i in np.flatnonzero(b >= 0):
        assert abs(float(sc[i, b[i]]) - want[i]) <= 1e-5 * (1 + R[i]), (i, sc[i, b[i]], want[i])


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def beam_search_replay(make_env, backend, shape, ties):
    """Every lane class in one batch (129..256 jobs and a non-permutation instance included) at reset and mid-episode,
    with some envs done and one with only the no-op legal; uniform tiny batches; (N, J, M), (N, J, 1) and (1, J, M)
    tables, with ties: the best order replays to makespan[best] (from reset a feasible schedule), and the scores."""
    if backend == "emu":
        names, walk, W = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170, 3
    else:
        names, walk, W = ["ta01", "ta11", "ta21", "ta31", "ta41", "ta51", "ta61", "ta71", "ta80", NONPERM, BIG_GPU,
                          SMALL, TINY] * 2, 400, 8
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
        out = search(env, table, W)
        assert (out["best"][~np_(env.done)] >= 0).all()
        sol = replay(make_env, env, out)
        if not steps:
            for i, name in enumerate(names):
                inst = name if not isinstance(name, str) else load_instance(name)
                check_schedule(inst, sol[i], int(out["makespan"][i, out["best"][i]]))
        check_scores(make_env, env, table, out)
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        env = make_env(3, batch_cfg([synthetic_instance(J, M, J * 10 + M)] * 3), auto_reset=False, seed=seed)
        env.reset()
        table = shaped_table(env, seed, ties, shape)
        out = search(env, table, 4)
        replay(make_env, env, out)
        check_scores(make_env, env, table, out)


@native_test()
def beam_search_width_one_is_greedy(make_env, backend):
    """width = 1 on integer tables in [-64, 64] equals rollout_priority(table) on a twin, bit for bit in makespan and
    order (the twin's solution), at reset and mid-episode, in every lane class."""
    import torch
    names = {"emu": ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY],
             "gpu": ["ta01", "ta21", "ta41", "ta61", "ta80", NONPERM, BIG_GPU, SMALL, TINY] * 3}[backend]
    for steps, seed in ((0, 1), (60, 2)):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, record_solution=True)
        env.reset()
        random_walk(env, steps)
        rng = np.random.default_rng(seed)
        table = rng.integers(-64, 65, size=(env.num_envs, env.jobs, env.machines)).astype(np.float32)
        out = search(env, table, 1)
        twin = twin_of(make_env, env, record_solution=True)
        twin.import_state(snapshot(env))
        twin.rollout_priority(torch.from_numpy(table).to(env.device))
        t, done = np_(twin.current_time_step), np_(twin.done)
        live = ~np_(env.done)
        assert done.all() and np.array_equal(out["makespan"][live, 0], t[live])
        # the order's rounds are the greedy decode's allocation order: the twin's start times sorted the same way
        sol = np_(twin.solution)
        ours = replay(make_env, env, out)
        assert np.array_equal(ours[live], sol[live])
        twin.close()


def enumerate_sequences(inst):
    """Every complete job sequence of `inst` from reset (forced no-ops taken, never a voluntary one), by depth-first
    replays of the CPU oracle: a list of (sequence, makespan)."""
    J = inst[0].shape[0]
    found = []

    def play(seq):
        o = OracleEnv(*inst)
        o.reset()
        done = False
        for j in seq:
            done = forced(o)
            _, _, done, _, _ = o.step(j)
        return o, done

    def forced(o):
        while True:
            legal = np.asarray(o.get_legal_actions(), bool)
            if legal[:J].any() or not legal[J]:
                return False
            o.step(J)

    def walk(seq):
        o, done = play(seq)
        if done:
            found.append((tuple(seq), int(o.current_time_step)))
            return
        forced(o)
        legal = np.asarray(o.get_legal_actions(), bool)
        for j in np.flatnonzero(legal[:J]):
            walk(seq + [int(j)])

    walk([])
    return found


@native_test()
def beam_search_exhaustive(make_env, backend):
    """Synthetic instances with J, M <= 3 and at most 32 complete job sequences: width >= count returns every sequence
    once (the multiset of makespans), the rest of the slots read -1 / -inf, and makespan[best] is the optimum."""
    insts = []
    for J, M, seed in ((2, 2, 1), (2, 3, 2), (3, 2, 3), (3, 2, 4), (2, 2, 5), (3, 2, 6), (2, 3, 7), (3, 2, 8)):
        inst = synthetic_instance(J, M, seed, max_dur=9, permutation=seed % 2 == 0)
        seqs = enumerate_sequences(inst)
        if len(seqs) <= 32:
            insts.append((inst, seqs))
    assert len(insts) >= 4
    for inst, seqs in insts:
        env = make_env(2, batch_cfg([inst] * 2), auto_reset=False, seed=4)
        env.reset()
        table = random_table(env, 5)
        for W in sorted({len(seqs), 32}):
            out = search(env, table, W)
            for i in range(2):
                ms = out["makespan"][i]
                assert sorted(ms[ms >= 0]) == sorted(m for _, m in seqs), (W, ms, seqs)
                assert (ms[len(seqs):] == -1).all() and np.isneginf(out["score"][i, len(seqs):]).all()
                assert ms[out["best"][i]] == min(m for _, m in seqs)
            replay(make_env, env, out)


def host_beam(make_env, env, table, W):
    """A float64 beam search restated on the host over N*W twins: each round export, gather the table at todo, take
    the log-softmax and the W best candidates per env, import the parents into their slots, step.  Returns the
    makespans (N, W), the best slot's order (N, J, M) and whether the env's selections kept a margin of
    1e-6 (1 + |score|) at every cut and between the final slots (where float32 rounding cannot change them)."""
    import torch
    n, J, M = env.num_envs, env.jobs, env.machines
    twin = twin_of(make_env, env, reps=W)
    snap = snapshot(env)
    twin.import_state({k: v.repeat_interleave(W, 0) for k, v in snap.items()})
    tab = np.broadcast_to(np.asarray(table, np.float64), (n, J, M))
    R = rounds(snap, env)
    done0 = np_(env.done)
    score = np.full((n, W), -np.inf)
    score[:, 0] = 0.0
    live = np.zeros((n, W), bool)
    live[:, 0] = ~done0
    safe = np.ones(n, bool)
    trace = np.zeros((int(R.max()) if n else 0, n, W, 2), np.int64)
    dev = env.device
    for r in range(trace.shape[0]):
        act_on = R > r
        while True:                                       # forced no-ops
            x = twin.export_state()
            legal = np_(x["legal"]).astype(bool)[:, :J].reshape(n, W, J)
            noop = ((np_(x["flags"]) >> 8) & N.FLAG_NOOP_LEGAL).astype(bool).reshape(n, W)
            need = live & act_on[:, None] & ~legal.any(2) & noop
            if not need.any():
                break
            act = np.where(need.ravel(), np.repeat(env.env_jobs, W), N.ACTION_SKIP).astype(np.int32)
            twin.step(torch.from_numpy(act).to(dev))
        x = twin.export_state()
        legal = np_(x["legal"]).astype(bool)[:, :J].reshape(n, W, J)
        todo = np_(x["todo"]).astype(np.int64).reshape(n, W, J)
        parent = np.zeros((n, W), np.int64)
        job = np.full((n, W), N.ACTION_SKIP, np.int64)
        new_score = np.full((n, W), -np.inf)
        new_live = np.zeros((n, W), bool)
        for i in np.flatnonzero(act_on):
            cands = []
            for b in np.flatnonzero(live[i]):
                lg = np.flatnonzero(legal[i, b])
                if not lg.size:
                    continue
                v = tab[i, lg, np.minimum(todo[i, b, lg], M - 1)]
                if np.isnan(v).any() or np.isposinf(v).any() or np.isneginf(v).all():
                    continue
                mx = v.max()
                lp = v - mx - np.log(np.exp(v - mx).sum())
                cands += [(score[i, b] + l, b, j) for l, j in zip(lp, lg) if l > -np.inf]
            cands.sort(key=lambda c: (-c[0], c[1], c[2]))
            # the kept set depends on the gap at the cut; the slots' order (which labels parents, and orders the final
            # rows) on the gaps between the kept candidates only in the last round, as long as the cut never ties
            pairs = zip(cands[:W], cands[1:W + 1]) if r == R[i] - 1 else zip(cands[W - 1:W], cands[W:W + 1])
            for a, b in pairs:
                if a[0] - b[0] <= 1e-6 * (1 + abs(a[0])):
                    safe[i] = False
            for s, (sc, b, j) in enumerate(cands[:W]):
                parent[i, s], job[i, s], new_score[i, s], new_live[i, s] = b, j, sc, True
            trace[r, i] = np.stack([parent[i], job[i]], 1)
        carry = ~act_on                                   # envs past their rounds keep their slots
        parent[carry] = np.arange(W)
        new_score[carry], new_live[carry] = score[carry], live[carry]
        rows = (np.arange(n)[:, None] * W + parent).ravel()
        x = {k: v[torch.from_numpy(rows).to(v.device)].clone() for k, v in x.items()}
        twin.import_state(x)
        twin.step(torch.from_numpy(job.ravel().astype(np.int32)).to(dev))
        score, live = new_score, new_live
    done = np_(twin.done).reshape(n, W)
    t = np_(twin.current_time_step).reshape(n, W)
    ms = np.where(live & done, t, -1)
    order = np.full((n, J, M), -1, np.int64)
    for i in range(n):
        if not (ms[i] >= 0).any():
            continue
        big = np.where(ms[i] >= 0, ms[i], np.iinfo(np.int64).max)
        at, seen = int(big.argmin()), np.zeros(J, np.int64)
        for r in range(int(R[i]) - 1, -1, -1):
            b, j = trace[r, i, at]
            order[i, j, env.env_machines[i] - 1 - seen[j]] = r
            seen[j] += 1
            at = int(b)
    twin.close()
    return ms, order, safe


@native_test(emu=[(3, 40)], gpu=[(8, 0)])
def beam_search_host_restatement(make_env, backend, width, steps):
    """The search against its float64 restatement on N*W twins, with random normal tables: makespan and order equal for
    every env whose selection keeps its margins (most of them).  GPU: ta80 at N = 8, W = 8, from reset, with a sharper
    table (standard deviation 8): over ta80's 2 000 rounds a unit table's scores reach about -300, where near-ties
    within the margin 1e-6 (1 + |score|) turn up in nearly every env."""
    names = {"emu": ["ta01", SMALL, NONPERM, TINY, SMALL, TINY], "gpu": ["ta80"] * 8}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=9)
    env.reset()
    random_walk(env, steps)
    table = random_table(env, 19) * {"emu": 1, "gpu": 8}[backend]
    out = search(env, table, width)
    ms, order, safe = host_beam(make_env, env, table, width)
    assert safe.mean() >= 0.5, (safe, out["score"][:, 0])
    for i in np.flatnonzero(safe):
        assert np.array_equal(out["makespan"][i], ms[i]), (i, out["makespan"][i], ms[i])
        Ji, Mi = env.env_jobs[i], env.env_machines[i]
        assert np.array_equal(out["order"][i, :Ji, :Mi], order[i, :Ji, :Mi]), i


@native_test()
def beam_search_determinism(make_env, backend):
    """Repeated calls are bit-identical; a permuted batch and shards give the same per-env rows; widths 4, 8, 16 and 32
    each replay in every lane class."""
    names = {"emu": ["ta01", SMALL, NONPERM, *EMU_CLASSES[:1], TINY],
             "gpu": ["ta01", "ta31", "ta51", "ta80", NONPERM, BIG_GPU, SMALL, TINY] * 2}[backend]
    n = len(names)
    env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=31)
    env.reset()
    table = random_table(env, 14)
    W = 4
    a, b = search(env, table, W), search(env, table, W)
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    perm = np.random.default_rng(3).permutation(n)
    pe = make_env(n, batch_cfg([names[p] for p in perm], sort=False), auto_reset=False, seed=31)
    pe.reset()
    po = search(pe, np.ascontiguousarray(table[perm, :pe.jobs, :pe.machines]), W)
    for k in ("makespan", "score"):
        assert np.array_equal(po[k].view(np.uint8), a[k][perm].view(np.uint8)), k
    for i, p in enumerate(perm):
        Jp, Mp = env.env_jobs[p], env.env_machines[p]
        assert np.array_equal(po["order"][i, :Jp, :Mp], a["order"][p, :Jp, :Mp]), i
    cut = n // 2
    for lo, hi in ((0, cut), (cut, n)):
        s = make_env(hi - lo, batch_cfg(names[lo:hi], sort=False), auto_reset=False, seed=31, env_id_base=lo)
        s.reset()
        so = search(s, np.ascontiguousarray(table[lo:hi, :s.jobs, :s.machines]), W)
        assert np.array_equal(so["makespan"], a["makespan"][lo:hi]), lo
        assert np.array_equal(so["score"].view(np.uint32), a["score"][lo:hi].view(np.uint32)), lo
    for W in (4, 8, 16, 32):
        out = search(env, table, W)
        assert (out["best"] >= 0).all() and (out["makespan"][:, :min(W, 2)] >= 0).all(), W
        replay(make_env, env, out)
        if W == 4:
            assert np.array_equal(out["makespan"], a["makespan"])


@native_test(emu=[False, True], gpu=[False, True])
def beam_search_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and the counters are unchanged by the call, also with an
    order; one launch per lane class present; no error bit, and an env with the sticky bit is searched as any other;
    after a recording step the call leaves real_obs stale for refresh_obs()."""
    import torch
    names = {"emu": ["ta01", SMALL, *EMU_CLASSES[:1], TINY], "gpu": ["ta01", "ta41", "ta80", BIG_GPU, TINY] * 3}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, seed=7, record_solution=True)
    env.reset()
    random_walk(env, 30)
    x = env.export_state()
    x["flags"][0] = int(x["flags"][0]) | (N.FLAG_ERROR << 8)
    env.import_state(x)
    table = random_table(env, 3)
    before, stats = _outputs(env), env.stats()
    classes = len({0 if J <= 32 else 1 if J <= 64 else 2 if J <= 128 else 3 for J in env.env_jobs})
    c = env.launch_count
    out = search(env, table, 4)
    search(env, table, 3, order=False)
    assert env.launch_count == c + 2 * classes
    after = _outputs(env)
    for k, v in before.items():
        assert np.array_equal(v, after[k]), k
    assert env.stats() == stats
    assert out["best"][0] >= 0                           # the env with the error bit is searched
    cfg = batch_cfg(names, sort=False)
    a_env, b_env = (make_env(len(names), cfg, auto_reset=auto_reset, seed=9) for _ in range(2))
    a_env.reset(); b_env.reset()
    scores = torch.zeros((a_env.num_envs, a_env.jobs + 1), device=a_env.device)
    traj = a_env.logits_trajectory(1)
    stale = np_(a_env.real_obs).copy()
    a_env.step_greedy_record(scores, traj, 0)
    b_env.step_greedy(scores)
    qa, qb = search(a_env, table, 2), search(b_env, table, 2)
    for k in qa:
        assert np.array_equal(qa[k], qb[k]), k
    assert np.array_equal(np_(a_env.real_obs), stale)


@native_test()
def beam_search_bad_tables(make_env, backend):
    """A NaN on a reached operation drops the beams that reach it; a NaN never read changes nothing; -inf entries
    exclude their jobs; an all-bad table gives -1 / NaN; an imported state with nothing legal gives -1 / -inf."""
    names = ["ta01", "ta01", "ta01", SMALL, "ta01", "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
    env.reset()
    random_walk(env, 20)
    x = env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    clean = random_table(env, 31)
    ref = search(env, clean, 4)
    bad = clean.copy()
    j0 = int(np.flatnonzero(legal[0])[0])
    bad[0, j0, todo[0, j0]] = np.nan                      # a legal current operation: the root's decision
    bad[1] = -np.inf                                      # every legal job at -inf
    bad[3, 9:, :] = np.nan                                # columns past J_i = 9: never read
    bad[3, :, 4:] = np.inf                                # operations past M_i = 4
    ops = np.arange(env.machines)
    bad[4][ops[None, :] < todo[4][:, None]] = np.nan      # operations already allocated: never read
    jx = int(np.flatnonzero(legal[5])[0])
    bad[5, jx, todo[5, jx]] = -np.inf                     # one job excluded at the root
    flags = np_(env.flags).copy()
    out = search(env, bad, 4)
    assert np.array_equal(np_(env.flags), flags)
    for i in (0, 1):
        assert (out["makespan"][i] == -1).all() and np.isnan(out["score"][i]).all() and out["best"][i] == -1, i
        assert (out["order"][i] == -1).all()
    for i in (2, 3, 4):
        assert np.array_equal(out["makespan"][i], ref["makespan"][i]), i
        assert np.array_equal(out["score"][i].view(np.uint32), ref["score"][i].view(np.uint32)), i
    assert (out["order"][5][jx, todo[5, jx]] != 0), out["order"][5][jx]     # not the first allocation
    replay(make_env, env, out)
    # a NaN deeper on one path: the beams that reach it are dropped, the others complete
    deep = clean.copy()
    deep[2, :, env.machines - 1] = np.nan                 # every job's last operation: every beam reaches one
    deep[2, 0, env.machines - 1] = 0.0
    o2 = search(env, deep, 4)
    assert (o2["makespan"][2] == -1).all() and np.isnan(o2["score"][2]).all()
    x = env.export_state()
    x["legal"][2] = 0
    x["flags"][2] = int(x["flags"][2]) & ~(N.FLAG_NOOP_LEGAL << 8)
    env.import_state(x)
    o3 = search(env, clean, 4)
    assert (o3["makespan"][2] == -1).all() and np.isneginf(o3["score"][2]).all() and o3["best"][2] == -1


@native_test()
def beam_search_abi(make_env, backend):
    """JSS_ERR_INVALID for NULL or misaligned pointers (order_out may be NULL), a negative stride, width < 1 or > 32 and
    ld < width; JSS_ERR_STATE before jss_assign; a bad shape or width raises ValueError before the native call."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    L, h, st = env._L, env._h, env._stream()
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    i32 = torch.zeros(n * 64, dtype=torch.int32, device=env.device)
    f32 = torch.zeros(n * 64, dtype=torch.float32, device=env.device)
    od = torch.zeros(n * J * M, dtype=torch.int32, device=env.device)
    p, o, q, r = t.data_ptr(), i32.data_ptr(), f32.data_ptr(), od.data_ptr()
    s = (J * M, M, 1)
    bad = ((None, *s, 4, o, q, 4, r), (p + 2, *s, 4, o, q, 4, r), (p, -1, M, 1, 4, o, q, 4, r),
           (p, J * M, -M, 1, 4, o, q, 4, r), (p, J * M, M, -1, 4, o, q, 4, r), (p, *s, 0, o, q, 4, r),
           (p, *s, 33, o, q, 33, r), (p, *s, -1, o, q, 4, r), (p, *s, 4, o, q, 3, r), (p, *s, 4, None, q, 4, r),
           (p, *s, 4, o + 2, q, 4, r), (p, *s, 4, o, None, 4, r), (p, *s, 4, o, q + 2, 4, r), (p, *s, 4, o, q, 4, r + 2))
    for args in bad:
        assert L.jss_beam_search(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_beam_search:"), args
    assert L.jss_beam_search(h, p, *s, 32, o, q, 32, None, st) == 0
    assert L.jss_beam_search(h, p, *s, 1, o, q, 1, r, st) == 0
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_beam_search(raw, p, *s, 4, o, q, 4, r, st) == -5
    L.jss_destroy(raw)
    for badt in (t[0], t[None], t[:, :J - 1], torch.zeros((3, J, M), device=env.device)):
        with pytest.raises(ValueError):
            env.beam_search(badt, 2)
    for w in (0, 33):
        with pytest.raises(ValueError):
            env.beam_search(t, w)


@native_test(emu=None)
def beam_search_full_size_ta80(make_env):
    """ta80 at N = 256, W = 16, per-env random normal tables, from reset: every env's best order replays to its
    makespan with a feasible schedule, and a sample of envs' best scores match their orders' float64 log-likelihood."""
    import torch
    n, W = 256, 16
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=15)
    env.reset()
    table = torch.randn((n, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(23),
                        device=env.device)
    out = search(env, table, W)
    assert (out["makespan"] > 0).all() and np.isfinite(out["score"]).all()
    sol = replay(make_env, env, out)
    inst = load_instance("ta80")
    for i in range(n):
        check_schedule(inst, sol[i], int(out["makespan"][i, out["best"][i]]))
    host = table.cpu().numpy()
    pick = [0, 1, 100, 255]
    sub = make_env(len(pick), {"instance_path": "ta80"}, auto_reset=False, seed=15)
    sub.reset()
    lp = order_log_prob(make_env, sub, host[pick], out["order"][pick])
    R = env.jobs * env.machines
    for k, i in enumerate(pick):
        assert abs(float(out["score"][i, out["best"][i]]) - lp[k]) <= 1e-5 * (1 + R), (i, lp[k])
