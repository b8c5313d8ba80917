"""The tests of jss_beam_step (one beam-search round per group of W envs from per-beam logit rows) and its driver
ObsBeamSearch, declared once for both backends (tests/backends.py) and collected by tests/test_emu_beam_step.py and
tests/test_gpu_beam_step.py.  A search driven with rows gathered from a table at each slot's todo must equal
jss_beam_search of that table bit for bit; every round's written slots must equal twins stepped one env at a time."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.beam import ObsBeamSearch
from jssenv_b200.instances import load_instance
from tests.backends import native_test
from tests.beam_search_suite import search, twin_of
from tests.lookahead_priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, SHAPES, SMALL, TINY, shaped_table
from tests.lookahead_suite import random_walk, snapshot
from tests.parity_common import batch_cfg, np_
from tests.priority_suite import random_table
from tests.sample_episodes_suite import check_schedule


def beam_batch(make_env, env, W, walk=7, **kw):
    """A batch of W envs per env of `env` (group g runs env g's instance), the other slots walked at random, env g's
    state imported into slot 0 of group g only."""
    import torch
    big = twin_of(make_env, env, reps=W, **kw)
    random_walk(big, walk)
    x = snapshot(big)
    snap = snapshot(env)
    rows = torch.arange(env.num_envs, device=big.device) * W
    for k in x:
        x[k][rows] = snap[k]
    sel = torch.zeros(big.num_envs, dtype=torch.uint8, device=big.device)
    sel[rows] = 1
    big.import_state(x, mask=sel)
    return big


def gathered_rows(big, table, W):
    """Each slot's logit row: the table of its group gathered at its jobs' current operations, NaN at every job that is
    not legal and in the no-op column (so a read of those shows up as a bad row)."""
    import torch
    n, J, M = big.num_envs, big.jobs, big.machines
    G = n // W
    t = torch.as_tensor(np.broadcast_to(np.asarray(table, np.float32), (G, J, M)).copy(), device=big.device)
    t = t.repeat_interleave(W, 0)
    todo = big.export_state()["todo"].long().clamp(0, M - 1)
    vals = t.gather(2, todo[:, :, None]).squeeze(2)
    legal = big.action_mask[:, :J].clone()
    legal &= torch.arange(J, device=big.device)[None, :] < torch.as_tensor(np.asarray(big.env_jobs), device=big.device)[:, None]
    rows = torch.full((n, J + 1), float("nan"), device=big.device)
    rows[:, :J] = torch.where(legal, vals, torch.tensor(float("nan"), device=big.device))
    return rows


def drive(big, table, W, order=True, all_orders=False, each=None):
    """ObsBeamSearch on `big` with rows gathered from `table`; `each(search)` after every round.  Returns the result as
    numpy arrays."""
    s = ObsBeamSearch(big, W).start()
    while not s.done:
        s.step(gathered_rows(big, table, W))
        if each:
            each(s)
    return {k: np_(v).copy() for k, v in s.result(order=order, all_orders=all_orders).items()}


def check_parity(make_env, env, table, W, walk=7):
    """The search driven on W envs per env equals beam_search(table, W) on env: makespan, score (bits) and order."""
    want = search(env, table, W)
    big = beam_batch(make_env, env, W, walk)
    got = drive(big, table, W)
    assert np.array_equal(got["makespan"], want["makespan"]), (got["makespan"], want["makespan"])
    assert np.array_equal(got["score"].view(np.uint32), want["score"].view(np.uint32)), (got["score"], want["score"])
    assert np.array_equal(got["best"], want["best"])
    for i in range(env.num_envs):
        Ji, Mi = env.env_jobs[i], env.env_machines[i]
        assert np.array_equal(got["order"][i, :Ji, :Mi], want["order"][i, :Ji, :Mi]), i
    big.close()
    return got


def crafted(make_env, names, steps, seed):
    """A batch after `steps` random decisions; with steps > 0 the first env not done gets only the no-op legal."""
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=3)
    env.reset()
    random_walk(env, steps)
    if steps:
        i = int(np.flatnonzero(~np_(env.done))[0])
        x = env.export_state()
        x["legal"][i] = 0
        x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
        env.import_state(x)
    return env


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def beam_step_parity(make_env, backend, shape, ties):
    """Every lane class at reset and mid-episode (a done env and one with only the no-op legal), (N, J, M), (N, J, 1) and
    (1, J, M) tables with ties: bit-identical to beam_search."""
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
def beam_step_widths(make_env, backend, width):
    """Widths 1, 4, 16 and 32 at reset and mid-episode, against beam_search."""
    names = {"emu": [SMALL, TINY, NONPERM], "gpu": ["ta01", "ta41", "ta80", NONPERM, BIG_GPU, TINY]}[backend]
    for steps in (0, 30):
        env = crafted(make_env, names, steps, width)
        check_parity(make_env, env, random_table(env, width, True), width)


def record(env):
    """Every output row a beam round may write, and the exported state, as numpy copies (scalars before the export,
    which rewrites the time and flags fields)."""
    out = {k: np_(getattr(env, k)).copy() for k in ("real_obs", "action_mask", "reward", "reward_raw",
                                                     "current_time_step", "flags", "done", "episode_count",
                                                     "last_makespan", "last_return")}
    out.update({"x_" + k: np_(v).copy() for k, v in env.export_state().items()})
    if env.solution is not None:
        out["solution"] = np_(env.solution).copy()
    return out


@native_test()
def beam_step_round_twins(make_env, backend):
    """After each call every written slot equals a twin that imported its parent's pre-call state, stepped the job and
    took the forced no-ops, bit for bit in exported state, real_obs, action_mask and scalar record; empty slots and
    untouched groups are byte-for-byte unchanged; the episode statistics, solution and the RNG counter do not move."""
    import torch
    names = {"emu": [SMALL, TINY, "ta01", EMU_CLASSES[0]], "gpu": ["ta01", "ta41", "ta80", BIG_GPU, TINY] * 2}[backend]
    W = 4
    env = crafted(make_env, names, 0, 5)
    big = beam_batch(make_env, env, W, record_solution=True)
    twin = twin_of(make_env, big, record_solution=True)
    table = random_table(env, 6, True)
    s = ObsBeamSearch(big, W).start()
    stats, si, rounds = big.stats(), big._step_index, 0
    while not s.done and rounds < 40:
        before = record(big)
        pre = snapshot(big)
        score0 = np_(s.score).copy()
        s.step(gathered_rows(big, table, W))
        rounds += 1
        after = record(big)
        parent = np_(s._parent[s._round - 1]).copy()
        job = np_(s._action[s._round - 1]).copy()
        new = (parent >= 0) & (job >= 0)
        n = big.num_envs
        src = np.where(new, (np.arange(n) // W) * W + np.maximum(parent, 0), np.arange(n))
        idx = torch.from_numpy(src).to(big.device)
        twin.import_state({k: v[idx].clone() for k, v in pre.items()})
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
        assert np.array_equal(np_(s.score)[untouched].view(np.uint32), score0[untouched].view(np.uint32))
        empty = ~new & ~untouched
        assert (parent[empty] == -1).all() and np.isneginf(np_(s.score)[empty]).all()
    assert big.stats()["episodes"] == stats["episodes"] and big._step_index == si
    twin.close()
    big.close()


@native_test()
def beam_step_invariant_after(make_env, backend):
    """After some rounds, step_logits / step / step_sample on the handle are bit-identical to a twin imported from the
    same state (a partial row emission would break the dirty-sector stores of the step kernels)."""
    import torch
    names = {"emu": [SMALL, "ta01", NONPERM], "gpu": ["ta01", "ta41", "ta80", NONPERM] * 4}[backend]
    W = 4
    env = crafted(make_env, names, 10, 8)
    big = beam_batch(make_env, env, W)
    table = random_table(env, 8)
    s = ObsBeamSearch(big, W).start()
    for _ in range(12):
        s.step(gathered_rows(big, table, W))
    twin = twin_of(make_env, big)
    twin.import_state(snapshot(big))
    twin._step_index = big._step_index
    g = torch.Generator(device=big.device).manual_seed(1)
    for k in range(6):
        logits = torch.randn((big.num_envs, big.jobs + 1), generator=g, device=big.device)
        if k % 3 == 0:
            big.step_logits(logits); twin.step_logits(logits)
        elif k % 3 == 1:
            acts = big.policy("RANDOM", step_index=k)
            big.step(acts); twin.step(acts)
        else:
            a = big.policy("SPT", step_index=k)
            big.step_sample(a.clone(), "MWR"); twin.step_sample(a.clone(), "MWR")
        for name in ("real_obs", "action_mask", "reward", "reward_raw", "current_time_step", "flags"):
            x, y = (np.ascontiguousarray(np_(getattr(e, name))) for e in (big, twin))
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (k, name)


@native_test()
def beam_step_replay(make_env, backend):
    """rollout_priority(-order) from the start state ends done at the best makespan with a feasible schedule, and every
    slot's order under all_orders replays to its makespan."""
    import torch
    names = {"emu": ["ta01", SMALL, TINY, NONPERM], "gpu": ["ta01", "ta21", "ta61", "ta80", NONPERM, TINY] * 2}[backend]
    W = 4
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=2)
    env.reset()
    big = beam_batch(make_env, env, W)
    out = drive(big, random_table(env, 12), W, order=True, all_orders=True)
    assert (out["best"] >= 0).all()
    for s in range(W):
        ok = out["makespan"][:, s] >= 0
        twin = twin_of(make_env, env, record_solution=True)
        twin.import_state(snapshot(env))
        ords = out["order"] if s < 0 else out["orders"][:, s]
        twin.rollout_priority(torch.from_numpy(-ords.astype(np.float32)).to(env.device))
        assert np_(twin.done)[ok].all() and np.array_equal(np_(twin.current_time_step)[ok], out["makespan"][ok, s])
        assert (ords[~ok] == -1).all()
        twin.close()
    twin = twin_of(make_env, env, record_solution=True)
    twin.rollout_priority(torch.from_numpy(-out["order"].astype(np.float32)).to(env.device))
    sol = np_(twin.solution)
    for i, name in enumerate(names):
        inst = load_instance(name) if isinstance(name, str) else name
        check_schedule(inst, sol[i], int(out["makespan"][i, out["best"][i]]))


@native_test()
def beam_step_bad_rows_and_dead_groups(make_env, backend):
    """A bad row in one beam drops it and sets the group's bad bit; bad rows in every beam empty the group and the result
    reads -1 / NaN; a group whose slots all start dead is untouched; the no-op column and non-legal columns are never
    read (NaN there changes nothing, as the parity tests show)."""
    import torch
    env = make_env(3, batch_cfg([SMALL, SMALL, TINY], sort=False), auto_reset=False, seed=4)
    env.reset()
    W = 4
    big = beam_batch(make_env, env, W)
    table = random_table(env, 4)
    s = ObsBeamSearch(big, W).start()
    s.score[2 * W] = float("-inf")                       # group 2: every slot dead
    s.step(gathered_rows(big, table, W))
    s.step(gathered_rows(big, table, W))
    sc = np_(s.score).reshape(3, W)
    live = np.isfinite(sc)
    assert live[0].sum() >= 2 and live[1].sum() >= 2 and not live[2].any()
    rows = gathered_rows(big, table, W)
    b = int(np.flatnonzero(live[0])[0])
    j = int(np.flatnonzero(np_(big.action_mask)[b, :big.env_jobs[b]])[0])
    rows[b, j] = float("nan")                            # group 0: one beam's row bad
    rows[W:2 * W] = float("inf")                         # group 1: every beam's row bad
    before = np_(big.real_obs).copy()
    parent, action, bad = (np_(t).copy() for t in big.beam_step(rows, W, s.score))
    assert list(bad) == [1, 1, 0]
    assert (parent[W:2 * W] == -1).all() and np.isneginf(np_(s.score)[W:2 * W]).all()
    assert b not in parent[:W] and (parent[:W] >= 0).any()
    assert (parent[2 * W:] == np.arange(W)).all() and (action[2 * W:] == -1).all()
    assert np.array_equal(np_(big.real_obs)[2 * W:], before[2 * W:])
    s._bad |= torch.as_tensor(bad, device=big.device)
    s._round += 1
    while not s.done:
        s.step(gathered_rows(big, table, W))
    out = {k: np_(v) for k, v in s.result().items()}
    assert (out["makespan"][1] == -1).all() and np.isnan(out["score"][1]).all() and out["best"][1] == -1
    assert (out["makespan"][0] >= 0).any()
    assert (out["makespan"][2] == -1).all() and np.isneginf(out["score"][2]).all()


@native_test()
def beam_step_abi(make_env, backend):
    """JSS_ERR_INVALID for NULL or misaligned pointers, width outside 1..32, N % width != 0, ld < J + 1 and a group that
    mixes instances; JSS_ERR_STATE before jss_assign; ValueError from the wrappers; an auto-reset env is refused by
    start(); one launch per lane class present, plus the refresh's when real_obs is stale."""
    import pytest
    import torch
    env = make_env(8, batch_cfg(["ta01"] * 4 + [SMALL] * 4, sort=False), auto_reset=False, seed=1)
    env.reset()
    n, J = env.num_envs, env.jobs
    L, h, st = env._L, env._h, env._stream()
    rows = torch.zeros((n, J + 1), device=env.device)
    sc = torch.full((n,), float("-inf"), device=env.device)
    sc[::4] = 0.0
    p_, a_, b_ = (torch.zeros(n, dtype=torch.int32, device=env.device) for _ in range(3))
    r, s, pp, ap, bp = rows.data_ptr(), sc.data_ptr(), p_.data_ptr(), a_.data_ptr(), b_.data_ptr()
    bad = ((None, J + 1, 4, s, pp, ap, bp), (r + 2, J + 1, 4, s, pp, ap, bp), (r, J, 4, s, pp, ap, bp),
           (r, J + 1, 0, s, pp, ap, bp), (r, J + 1, 33, s, pp, ap, bp), (r, J + 1, 3, s, pp, ap, bp),
           (r, J + 1, 8, s, pp, ap, bp), (r, J + 1, 4, None, pp, ap, bp), (r, J + 1, 4, s + 2, pp, ap, bp),
           (r, J + 1, 4, s, None, ap, bp), (r, J + 1, 4, s, pp, ap + 1, bp), (r, J + 1, 4, s, pp, ap, None))
    for args in bad:
        assert L.jss_beam_step(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_beam_step:"), args
    assert L.jss_beam_step(h, r, J + 1, 4, s, pp, ap, bp, st) == 0
    assert L.jss_beam_step(h, r, J + 1, 2, s, pp, ap, bp, st) == 0
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_beam_step(raw, r, J + 1, 2, s, pp, ap, bp, st) == -5
    L.jss_destroy(raw)
    for w in (0, 3, 33):
        with pytest.raises(ValueError):
            env.beam_step(rows, w, sc)
    with pytest.raises(ValueError):
        ObsBeamSearch(env, 8)                            # mixes instances
    with pytest.raises(ValueError):
        env.beam_step(rows, 4, sc.double())
    ar = make_env(4, {"instance_path": "ta01"}, auto_reset=True)
    with pytest.raises(ValueError):
        ObsBeamSearch(ar, 2).start()
    mixed = make_env(8, batch_cfg(["ta01"] * 4 + [EMU_CLASSES[0]] * 4, sort=False), auto_reset=False, seed=1)
    mixed.reset()
    rows2 = torch.zeros((8, mixed.jobs + 1), device=mixed.device, requires_grad=True)
    c = mixed.launch_count
    mixed.beam_step(rows2, 4, sc.clone())
    assert mixed.launch_count == c + 2
    traj = mixed.logits_trajectory(1)
    mixed.step_greedy_record(torch.zeros((8, mixed.jobs + 1), device=mixed.device), traj, 0)
    c = mixed.launch_count
    mixed.beam_step(rows2, 4, sc.clone())
    assert mixed.launch_count == c + 2 + 2              # the refresh launches once per lane class too


@native_test()
def beam_step_group_permutation_and_shards(make_env, backend):
    """Results do not depend on the order of the groups in the batch, nor on sharding (env_id_base)."""
    names = {"emu": [SMALL, TINY, NONPERM, SMALL], "gpu": ["ta01", "ta41", "ta80", NONPERM, TINY, "ta21"]}[backend]
    W = 2
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=6)
    env.reset()
    table = random_table(env, 9)
    ref = drive(beam_batch(make_env, env, W), table, W)
    perm = np.random.default_rng(2).permutation(len(names))
    pe = make_env(len(names), batch_cfg([names[p] for p in perm], sort=False), auto_reset=False, seed=6)
    pe.reset()
    po = drive(beam_batch(make_env, pe, W), np.ascontiguousarray(table[perm, :pe.jobs, :pe.machines]), W)
    for k in ("makespan", "score"):
        assert np.array_equal(po[k].view(np.uint8), ref[k][perm].view(np.uint8)), k
    cut = len(names) // 2
    for lo, hi in ((0, cut), (cut, len(names))):
        sh = make_env(hi - lo, batch_cfg(names[lo:hi], sort=False), auto_reset=False, seed=6, env_id_base=lo * W)
        sh.reset()
        so = drive(beam_batch(make_env, sh, W), np.ascontiguousarray(table[lo:hi, :sh.jobs, :sh.machines]), W)
        assert np.array_equal(so["makespan"], ref["makespan"][lo:hi])
        assert np.array_equal(so["score"].view(np.uint32), ref["score"][lo:hi].view(np.uint32))


@native_test(emu=None)
def beam_step_side_stream(make_env):
    """A search run on a side stream equals the same search on the default stream, bit for bit."""
    import torch
    names = ["ta01", "ta41", "ta80", NONPERM] * 2
    W = 4
    outs = []
    for side in (False, True):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
        env.reset()
        table = random_table(env, 3)
        big = beam_batch(make_env, env, W)
        if side:
            stream = torch.cuda.Stream()
            stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(stream):
                out = drive(big, table, W)
            torch.cuda.current_stream().wait_stream(stream)
        else:
            out = drive(big, table, W)
        outs.append(out)
    for k in outs[0]:
        assert np.array_equal(outs[0][k].view(np.uint8), outs[1][k].view(np.uint8)), k


@native_test(emu=None)
def beam_step_full_size_ta80(make_env):
    """ta80 at G = 256, W = 16 from reset: bit-identical to beam_search, and the best order replays to its makespan with
    a feasible schedule."""
    import torch
    G, W = 256, 16
    env = make_env(G, {"instance_path": "ta80"}, auto_reset=False, seed=15)
    env.reset()
    table = torch.randn((G, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(23),
                        device=env.device).cpu().numpy()
    out = check_parity(make_env, env, table, W, walk=0)
    twin = twin_of(make_env, env, record_solution=True)
    twin.rollout_priority(torch.from_numpy(-out["order"].astype(np.float32)).to(env.device))
    sol, inst = np_(twin.solution), load_instance("ta80")
    for i in range(G):
        check_schedule(inst, sol[i], int(out["makespan"][i, out["best"][i]]))
