"""The tests of jss_improve_orders (given operation orders improved by steepest descent on the critical path, the envs
left untouched), declared once for both backends (tests/backends.py) and collected by tests/test_emu_improve_orders.py
and tests/test_gpu_improve_orders.py.  The descent is restated on the host, independently of the kernel: each decision
is chosen in numpy from export_state, twin batches are stepped with jss_step in lockstep (one twin row per order, then
one per neighbour), the chain is walked in numpy and the move rule applied; every output must equal it bit for bit.
Returned orders are replayed with rollout_priority(-order) and on the CPU oracle."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv
from tests.backends import native_test
from tests.beam_search_suite import search
from tests.lookahead_priority_suite import EMU_CLASSES, NONPERM, SMALL, TINY, noop_only
from tests.lookahead_suite import _outputs, random_walk, snapshot
from tests.parity_common import assert_twins_equal, batch_cfg, np_
from tests.priority_suite import random_table
from tests.sample_episodes_suite import check_schedule
from tests.swor_suite import swor

UNLIMITED = None
OUT_KEYS = ("order", "makespan", "start_makespan", "moves")


def improve(env, order, max_moves=UNLIMITED):
    """improve_orders of host (or device) orders; the RNG counter must not move.  Returns numpy arrays."""
    import torch
    si = env._step_index
    o = torch.from_numpy(np.ascontiguousarray(order)).to(env.device) if isinstance(order, np.ndarray) else order
    out = env.improve_orders(o, max_moves)
    assert env._step_index == si
    return {k: np_(v).copy() for k, v in out.items()}


def inst_of(env, i):
    """(machine, duration) of env i's instance."""
    return load_instance(env.instances[int(env.env_to_instance[i])])


def replay_rows(make_env, env, snap, rows, orders):
    """Replays order r (host (R, J, M)) from the state of env rows[r] on a twin batch stepped in lockstep.  Each
    decision is taken in numpy from the twin's export_state: the legal job whose current operation has the smallest
    entry as fp32 of -entry (ties to the lowest job), the no-op only when no job is legal and it is; at most
    2 J_i M_i + 1 decisions.  Returns (makespan, rounds, starts): the end time (-1 unless done), and for each operation
    the round (job allocations counted from 0) and start time at which the replay allocates it (-1 otherwise)."""
    import torch
    R, J, M = len(rows), env.jobs, env.machines
    ext = np.concatenate([np.asarray(rows, np.int64), np.arange(env.num_envs)])   # env's rows too: the same maxima
    cfg = {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
           "env_to_instance": [int(env.env_to_instance[i]) for i in ext]}
    twin = make_env(len(ext), cfg, auto_reset=False)
    twin.reset()
    twin.import_state({k: v[torch.as_tensor(ext, device=env.device)] for k, v in snap.items()})
    Ji = np.asarray(env.env_jobs)[rows].astype(np.int64)
    Mi = np.asarray(env.env_machines)[rows].astype(np.int64)
    bound = 2 * Ji * Mi + 1
    key = -(np.asarray(orders).astype(np.int32).astype(np.float32))        # fp32 of -entry
    rounds = np.full((R, J, M), -1, np.int64)
    starts = np.full((R, J, M), -1, np.int64)
    rnd = np.zeros(R, np.int64)
    failed = np_(twin.done).astype(bool)[:R]             # done at entry, nothing legal, an erring step
    live = ~failed
    ar = np.arange(R)
    for d in range(int(bound.max())):
        x = twin.export_state()
        legal = np_(x["legal"]).astype(bool)[:R, :J]
        todo = np_(x["todo"]).astype(np.int64)[:R]
        flags = np_(twin.flags).astype(np.int64)[:R]
        t = np_(twin.current_time_step).astype(np.int64)[:R]
        live &= (flags & N.FLAG_DONE) == 0
        live &= d < bound
        if not live.any():
            break
        k = np.minimum(todo, M - 1)
        cand = np.where(legal, key[ar[:, None], np.arange(J)[None, :], k], -np.inf)
        any_legal = legal.any(1)
        act = np.where(any_legal, np.argmax(cand, 1), np.where(flags & N.FLAG_NOOP_LEGAL, Ji, N.ACTION_SKIP))
        failed |= live & (act == N.ACTION_SKIP)          # nothing legal: the replay stops before done
        act = np.where(live, act, N.ACTION_SKIP)
        live &= act != N.ACTION_SKIP
        job = live & any_legal & (todo[ar, np.where(any_legal, act, 0)] < M)   # a job without an operation errs
        r_, j_ = ar[job], act[job]
        rounds[r_, j_, todo[r_, j_]] = rnd[job]
        starts[r_, j_, todo[r_, j_]] = t[job]
        rnd += job
        err = flags & N.FLAG_ERROR
        full = np.concatenate([act, np.full(len(ext) - R, N.ACTION_SKIP)]).astype(np.int32)
        twin.step(torch.from_numpy(full).to(env.device))
        erred = live & ((np_(twin.flags).astype(np.int64)[:R] & N.FLAG_ERROR) != err)   # an erring step changes nothing
        failed |= erred
        live &= ~erred
    done = (np_(twin.flags).astype(np.int64)[:R] & N.FLAG_DONE) != 0
    ms = np.where(done & ~failed, np_(twin.current_time_step).astype(np.int64)[:R], -1)
    twin.close()
    return ms, rounds, starts


def chain(inst, rounds, starts, T):
    """The chain's pairs (u, v) of the canonical schedule (rounds, starts) that ends at T, as flat (j, k) pairs."""
    machine, duration = inst
    Ji, Mi = machine.shape
    rd, st = rounds[:Ji, :Mi], starts[:Ji, :Mi]
    end = st + duration
    incall = rd >= 0
    at = np.argwhere(incall & (end == T))
    if not len(at):
        return []
    o = tuple(max(map(tuple, at), key=lambda q: rd[q]))
    pairs = []
    while True:
        s0, m = st[o], machine[o]
        same = incall & (machine == m) & (rd < rd[o])
        pm = tuple(np.argwhere(same)[np.argmax(rd[same])]) if same.any() else None
        if pm is not None and end[pm] == s0:
            pairs.append((pm, o))
            o = pm
        elif o[1] > 0 and incall[o[0], o[1] - 1] and end[o[0], o[1] - 1] == s0:
            o = (o[0], o[1] - 1)
        else:
            return pairs


def restate(make_env, env, orders):
    """The descent restated on the host for (N, k, J, M) orders: for each order the list of (order, makespan) after
    0, 1, ... accepted moves (the canonical order of each; [] if the input's replay does not end done), and the
    input's makespan."""
    n, k, J, M = orders.shape
    snap = snapshot(env)
    rows = np.repeat(np.arange(n), k)
    ms, rounds, starts = replay_rows(make_env, env, snap, rows, orders.reshape(n * k, J, M))
    hist = [[(rounds[r], int(ms[r]))] if ms[r] >= 0 else [] for r in range(n * k)]
    cur = {r: (rounds[r], starts[r], int(ms[r])) for r in range(n * k) if ms[r] >= 0}
    insts = [inst_of(env, i) for i in range(n)]
    while cur:
        nb_rows, nb_orders, owner = [], [], []
        for r, (rd, st, T) in cur.items():
            for c, (u, v) in enumerate(chain(insts[rows[r]], rd, st, T)):
                o = rd.copy()
                o[u], o[v] = rd[v], rd[u]
                nb_rows.append(rows[r]); nb_orders.append(o); owner.append((r, c))
        if not nb_rows:
            break
        vals, nrd, nst = replay_rows(make_env, env, snap, np.asarray(nb_rows), np.stack(nb_orders))
        best = {}
        for x, (r, c) in enumerate(owner):
            if vals[x] >= 0 and (r not in best or vals[x] < vals[best[r]]):
                best[r] = x
        nxt = {}
        for r, (rd, st, T) in cur.items():
            x = best.get(r)
            if x is None or vals[x] >= T:
                continue                                  # a local optimum
            nxt[r] = (nrd[x], nst[x], int(vals[x]))
            hist[r].append((nrd[x], int(vals[x])))
        cur = nxt
    return hist, ms


def expected(hist, start, n, k, J, M, max_moves):
    """The outputs improve_orders(max_moves) must return, from restate()'s history."""
    want = {"order": np.full((n, k, J, M), -1, np.int64), "makespan": np.full((n, k), -1, np.int64),
            "start_makespan": start.reshape(n, k).astype(np.int64), "moves": np.zeros((n, k), np.int64)}
    for r, h in enumerate(hist):
        if not h:
            continue
        m = len(h) - 1 if max_moves is None else min(max_moves, len(h) - 1)
        i, s = divmod(r, k)
        want["order"][i, s], want["makespan"][i, s], want["moves"][i, s] = h[m][0], h[m][1], m
    return want


def check_outputs(env, got, want, ctx):
    n, k = want["makespan"].shape
    for key in ("makespan", "start_makespan", "moves"):
        g = got[key].reshape(n, k)
        assert np.array_equal(g, want[key]), (ctx, key, g, want[key])
    o = got["order"].reshape(want["order"].shape)
    for i, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        assert np.array_equal(o[i, :, :Ji, :Mi], want["order"][i, :, :Ji, :Mi]), (ctx, i)


def random_orders(env, k, seed):
    """Random non-canonical integer tables with ties, negatives and duplicates, within +-2^24."""
    rng = np.random.default_rng(seed)
    shape = (env.num_envs, k, env.jobs, env.machines)
    small = rng.integers(-4, 5, size=shape)
    big = rng.integers(-(1 << 24), (1 << 24) + 1, size=shape)
    return np.where(rng.random(shape) < 0.5, small, big).astype(np.int64)


def input_orders(env, kind, k, seed):
    """(N, k, J, M) orders of one kind: beam_search / sample_without_replacement orders or random tables."""
    table = random_table(env, seed)
    if kind == "beam":
        o = np.stack([search(env, table, w)["order"] for w in (1, 4, 2)[:k]], 1)
    elif kind == "swor":
        o = swor(env, table, k)[0]["order"]
    else:
        o = random_orders(env, k, seed)
    return o.astype(np.int64)


def check_restatement(make_env, env, orders, moves_list, ctx):
    """improve_orders equals the host restatement for each max_moves in moves_list; returns the unlimited outputs."""
    n, k, J, M = orders.shape
    hist, start = restate(make_env, env, orders)
    res = None
    for mm in moves_list:
        got = improve(env, orders if k > 1 else orders[:, 0], mm)
        check_outputs(env, got, expected(hist, start, n, k, J, M, mm), (ctx, mm))
        if mm is None:
            res = got
    return res


def replay_check(make_env, env, out, oracle_envs=()):
    """Every returned order replays on a twin with rollout_priority(-order) to its makespan; for the envs in
    oracle_envs (from reset), the oracle replays the same decisions to the same makespan with a feasible schedule."""
    import torch
    ms = out["makespan"].reshape(env.num_envs, -1)
    order = out["order"].reshape(env.num_envs, ms.shape[1], env.jobs, env.machines)
    snap = snapshot(env)
    cfg = {"instance_paths": [env.instances[k] for k in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    for s in range(ms.shape[1]):
        full = ms[:, s] >= 0
        twin = make_env(env.num_envs, cfg, auto_reset=False)
        twin.reset()
        twin.import_state(snap)
        twin.rollout_priority(torch.from_numpy(-order[:, s].astype(np.float32)).to(env.device))
        assert np_(twin.done)[full].all() and np.array_equal(np_(twin.current_time_step)[full], ms[full, s]), s
        twin.close()
        for i in oracle_envs:
            if not full[i]:
                continue
            inst = inst_of(env, i)
            Ji, Mi = inst[0].shape
            o = OracleEnv(*inst)
            o.reset()
            sol = np.full((Ji, Mi), -1, np.int64)
            done = False
            while not done:
                legal = np.flatnonzero(np.asarray(o.get_legal_actions(), bool)[:Ji])
                todo = np.asarray(o.todo_time_step_job)
                if len(legal):
                    a = int(legal[np.argmin(order[i, s, legal, todo[legal]])])
                    sol[a, todo[a]] = o.current_time_step
                else:
                    a = Ji
                _, _, done, _, _ = o.step(a)
            assert o.current_time_step == ms[i, s], (i, s)
            check_schedule(inst, sol, int(ms[i, s]))


# ---- tests -------------------------------------------------------------------------------------------------------

EMU_NAMES = [SMALL, TINY, *EMU_CLASSES]
GPU_NAMES = ["ta01", "ta41", SMALL, NONPERM, *EMU_CLASSES]


@native_test(emu=[("beam", 0), ("swor", 1), ("random", 0), ("random", 1)],
             gpu=[("beam", 0), ("swor", 1), ("random", 0), ("random", 1)])
def improve_orders_restatement(make_env, backend, kind, steps):
    """Bit for bit against the host restatement: every lane class (129..256 jobs included), from reset and after a
    random walk, k = 1 and 3, max_moves 0, 1, 2 and unlimited, on beam_search, sample_without_replacement and random
    non-canonical orders."""
    names = EMU_NAMES if backend == "emu" else GPU_NAMES
    walk = {"emu": 40, "gpu": 120}[backend] * steps
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3 + steps)
    env.reset()
    random_walk(env, walk)
    for k in (1, 3):
        orders = input_orders(env, kind, k, 10 * k + steps)
        out = check_restatement(make_env, env, orders, (0, 1, 2, UNLIMITED), (kind, steps, k))
        assert (out["makespan"] >= 0).any()
        if kind != "random" or steps == 0:
            replay_check(make_env, env, out, oracle_envs=range(2) if steps == 0 else ())


@native_test()
def improve_orders_descent(make_env, backend):
    """makespan <= start_makespan, strictly where moves > 0; max_moves 0 returns R(input), a beam order unchanged; a
    second call on an output that stopped before max_moves returns it with moves 0; k and position do not matter."""
    names = EMU_NAMES if backend == "emu" else GPU_NAMES * 2
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=5)
    env.reset()
    random_walk(env, 10)
    a, b = input_orders(env, "random", 1, 7), input_orders(env, "beam", 1, 8)
    ab = np.concatenate([a, b], 1)
    both = improve(env, ab)
    ms, st, mv = both["makespan"], both["start_makespan"], both["moves"]
    assert (ms <= st).all() and (ms[mv > 0] < st[mv > 0]).all() and (mv > 0).any()
    for s, x in enumerate((a, b)):                        # improving [A, B] equals improving A and B separately
        one = improve(env, x[:, 0])
        for key in OUT_KEYS:
            assert np.array_equal(one[key], both[key][:, s]), (s, key)
    ba = improve(env, ab[:, ::-1])
    for key in OUT_KEYS:
        assert np.array_equal(ba[key], both[key][:, ::-1]), key
    zero = improve(env, b[:, 0], 0)                       # a beam order is canonical
    assert np.array_equal(zero["order"], b[:, 0]) and (zero["moves"] == 0).all()
    assert np.array_equal(zero["makespan"], zero["start_makespan"])
    again = improve(env, both["order"].reshape(ab.shape), 3)
    assert np.array_equal(again["order"], both["order"]) and (again["moves"] == 0).all()
    assert np.array_equal(again["makespan"], both["makespan"])
    assert both["best"].shape == (env.num_envs,)


@native_test()
def improve_orders_edge_cases(make_env, backend):
    """Envs done at entry, no-op-only starts and an imported state that errs follow the -1 conventions; in place
    (order_out == order) equals a separate output; a repeat is bit-identical."""
    import torch
    names = [SMALL, TINY, SMALL, NONPERM, EMU_CLASSES[0], TINY] * (1 if backend == "emu" else 4)
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=9)
    env.reset()
    random_walk(env, 60)
    x = env.export_state()
    i = int(np.flatnonzero(~np_(env.done))[0])
    x["legal"][i] = 0                                     # only the no-op legal
    x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
    e = int(np.flatnonzero(~np_(env.done))[1])            # nothing legal at all: the replay stops before done
    x["legal"][e] = 0
    x["flags"][e] = int(x["flags"][e]) & ~(N.FLAG_NOOP_LEGAL << 8)
    env.import_state(x)
    done = np_(env.done).astype(bool)
    assert done.any() and noop_only(env).any()
    orders = input_orders(env, "random", 2, 3)
    out = check_restatement(make_env, env, orders, (UNLIMITED,), "edges")
    assert (out["makespan"][done] == -1).all() and (out["start_makespan"][done] == -1).all()
    assert (out["moves"][done] == 0).all() and (out["order"][done] == -1).all()
    assert (out["makespan"][e] == -1).all() and (out["order"][e] == -1).all()
    assert (out["makespan"][i] >= 0).all()
    assert np.array_equal(improve(env, orders)["order"], out["order"])
    # in place, through the C ABI
    o = torch.from_numpy(orders.astype(np.int32)).to(env.device).contiguous()
    n, k = env.num_envs, orders.shape[1]
    res = [torch.empty((n, k), dtype=torch.int32, device=env.device) for _ in range(3)]
    rc = env._L.jss_improve_orders(env._h, o.data_ptr(), k, 2 ** 31 - 1, o.data_ptr(), *(r.data_ptr() for r in res), k,
                                   env._stream())
    assert rc == 0
    oo = np_(o)
    for i_, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        assert np.array_equal(oo[i_, :, :Ji, :Mi], out["order"][i_, :, :Ji, :Mi]), i_
    for r, key in zip(res, ("makespan", "start_makespan", "moves")):
        assert np.array_equal(np_(r), out[key]), key


@native_test()
def improve_orders_erring_state(make_env, backend):
    """An imported state whose first decision errs (a legal job without an operation) reads -1 / -1 / 0 and -1."""
    env = make_env(2, batch_cfg([SMALL, SMALL]), auto_reset=False, seed=4)
    env.reset()
    random_walk(env, 5)
    x = env.export_state()
    j = int(np.flatnonzero(np_(x["legal"])[0][:9])[0])
    x["legal"][0] = 0
    x["legal"][0, j] = 1                                  # the only legal job, but its operations are all done
    x["todo"][0, j] = env.machines
    try:
        env.import_state(x)
    except Exception:                                      # the library refuses the state: nothing to check
        return
    orders = input_orders(env, "random", 1, 5)
    out = check_restatement(make_env, env, orders, (UNLIMITED,), "erring")
    assert out["makespan"][0] == -1 and (out["order"][0] == -1).all() and out["moves"][0] == 0


@native_test()
def improve_orders_batch_invariance(make_env, backend):
    """An env permutation and shards (env_id_base != 0) change nothing."""
    import torch
    names = [SMALL, NONPERM, TINY, EMU_CLASSES[0]] if backend == "emu" else GPU_NAMES
    n = len(names)
    env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=6)
    env.reset()
    random_walk(env, 20)
    snap = snapshot(env)
    orders = input_orders(env, "random", 2, 6)
    want = improve(env, orders)
    perm = np.random.default_rng(6).permutation(n)
    for base, idx in ((0, perm), (n, np.arange(n)), (7, perm)):
        cfg = batch_cfg([names[i] for i in idx], sort=False)
        other = make_env(n, cfg, auto_reset=False, seed=1, env_id_base=base)
        other.reset()
        t = torch.as_tensor(idx, device=env.device)
        other.import_state({k: v[t] for k, v in snap.items()})
        got = improve(other, orders[idx])
        for key in ("makespan", "start_makespan", "moves"):
            assert np.array_equal(got[key], want[key][idx]), (base, key)
        for a, i in enumerate(idx):
            Ji, Mi = env.env_jobs[i], env.env_machines[i]
            assert np.array_equal(got["order"][a, :, :Ji, :Mi], want["order"][i, :, :Ji, :Mi]), (base, a)


@native_test(emu=[False, True], gpu=[False, True])
def improve_orders_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution, flags and the RNG counter are bit-identical after the call;
    one launch per lane class present; after a recording step the call leaves real_obs stale for refresh_obs()."""
    import torch
    names = [SMALL, NONPERM, SMALL, EMU_CLASSES[0]] if backend == "emu" else ["ta01", "ta51", "ta80", NONPERM] * 8
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, record_solution=True, seed=8)
    env.reset()
    random_walk(env, 30)
    orders = input_orders(env, "random", 2, 2)
    before, stats = _outputs(env), env.stats()
    c = env.launch_count
    improve(env, orders)
    improve(env, orders[:, 0], 1)
    assert env.launch_count == c + 2 * (2 if backend == "emu" else 3)   # one launch per lane class present
    after = _outputs(env)
    for k, v in before.items():
        assert np.array_equal(v, after[k]), k
    assert env.stats() == stats
    cfg = batch_cfg(names, sort=False)
    a_env, b_env = (make_env(len(names), cfg, auto_reset=auto_reset, seed=9) for _ in range(2))
    a_env.reset(); b_env.reset()
    scores = torch.zeros((a_env.num_envs, a_env.jobs + 1), device=a_env.device)
    traj = a_env.logits_trajectory(1)
    stale = np_(a_env.real_obs).copy()
    a_env.step_greedy_record(scores, traj, 0)
    b_env.step_greedy(scores)
    qa, qb = improve(a_env, orders), improve(b_env, orders)
    for key in OUT_KEYS:
        assert np.array_equal(qa[key], qb[key]), key
    assert np.array_equal(np_(a_env.real_obs), stale)
    a_env.refresh_obs()
    assert_twins_equal(a_env, b_env, "refreshed", state=True, stats=True)


@native_test()
def improve_orders_abi(make_env, backend):
    """JSS_ERR_INVALID for a NULL or misaligned pointer, k < 1, ld < k, max_moves < 0 and every overlap but in place;
    JSS_ERR_STATE before jss_assign; bad shapes, dtypes and max_moves raise ValueError."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M, k = env.num_envs, env.jobs, env.machines, 2
    dev = env.device
    o = torch.zeros((n, k, J, M), dtype=torch.int32, device=dev)
    oo = torch.zeros_like(o)
    r = [torch.zeros((n, k), dtype=torch.int32, device=dev) for _ in range(3)]
    L, h, st = env._L, env._h, env._stream()
    po, pq, p1, p2, p3 = o.data_ptr(), oo.data_ptr(), *(x.data_ptr() for x in r)
    good = (po, k, 5, pq, p1, p2, p3, k)
    assert L.jss_improve_orders(h, *good, st) == 0
    bad = [(None, k, 5, pq, p1, p2, p3, k), (po + 2, k, 5, pq, p1, p2, p3, k), (po, k, 5, None, p1, p2, p3, k),
           (po, k, 5, pq + 2, p1, p2, p3, k), (po, k, 5, pq, None, p2, p3, k), (po, k, 5, pq, p1, p2 + 2, p3, k),
           (po, k, 5, pq, p1, p2, None, k), (po, 0, 5, pq, p1, p2, p3, k), (po, k, 5, pq, p1, p2, p3, k - 1),
           (po, k, -1, pq, p1, p2, p3, k), (po, k, 5, pq, p1, p1, p3, k), (po, k, 5, pq, p1, p2, p1 + 4, k),
           (po, k, 5, po + 16, p1, p2, p3, k), (po, k, 5, pq, po, p2, p3, k), (po, k, 5, pq, p1, p2, pq + 4, k)]
    for args in bad:
        assert L.jss_improve_orders(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_improve_orders:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_improve_orders(raw, *good, st) == -5
    L.jss_destroy(raw)
    for badin in (o[:1], o[:, :, :J - 1], torch.zeros((3, J, M), dtype=torch.int32, device=dev), o.float(),
                  o[:, :0], o.bool()):
        with pytest.raises(ValueError):
            env.improve_orders(badin)
    for mm in (-1, 1.5, True, 2 ** 31):
        with pytest.raises(ValueError):
            env.improve_orders(o, mm)
    x = improve(env, o.to(torch.int64))
    assert set(x) == set(OUT_KEYS) | {"best"} and x["order"].shape == (n, k, J, M)
    y = improve(env, o[:, 0])
    assert set(y) == set(OUT_KEYS) and y["order"].shape == (n, J, M) and y["makespan"].shape == (n,)


@native_test(emu=None)
def improve_orders_full_size_ta80(make_env):
    """ta80 at N = 256 from the best beam_search(16) orders: every output replays on twins to its makespan; 16 envs with
    max_moves = 5 equal the restatement bit for bit; ta01 at N = 4 096 runs unlimited against twin replays."""
    import torch
    n = 256
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=14)
    env.reset()
    table = torch.randn((n, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(3),
                        device=env.device)
    orders = env.beam_search(table, 16, order=True)["order"]
    out = improve(env, orders, 5)
    assert (out["makespan"] <= out["start_makespan"]).all() and (out["moves"] > 0).any()
    replay_check(make_env, env, out)
    small = make_env(16, {"instance_path": "ta80"}, auto_reset=False, seed=14)
    small.reset()
    check_restatement(make_env, small, np_(orders[:16]).astype(np.int64)[:, None], (5,), "ta80")
    big = make_env(4096, {"instance_path": "ta01"}, auto_reset=False, seed=15)
    big.reset()
    t01 = torch.randn((4096, big.jobs, big.machines), generator=torch.Generator(device=big.device).manual_seed(4),
                      device=big.device)
    o01 = big.beam_search(t01, 1, order=True)["order"]
    res = improve(big, o01)
    assert (res["makespan"] <= res["start_makespan"]).all() and (res["moves"] > 0).any()
    replay_check(make_env, big, res)
