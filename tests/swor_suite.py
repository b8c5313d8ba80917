"""The tests of jss_sample_without_replacement (k distinct episodes per env drawn without replacement from a caller's
logit table by stochastic beam search, the envs left untouched) and jss_order_log_prob / _grad (the log-likelihood of
given operation orders under the table, with its gradient), declared once for both backends (tests/backends.py) and
collected by tests/test_emu_swor.py and tests/test_gpu_swor.py.  Tiny instances are checked against an exhaustive
enumeration and a chi-square test of the draws; every slot's order is replayed greedily on a twin
(rollout_priority(-order)) and scored by order_log_prob; whole searches are checked against a float64 stochastic beam
search restated on the host over N*W twins with the same uniforms (oracle/logits_oracle.py); the gradient against float64
autograd of the likelihood restated from the twins' decisions."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from jssenv_b200.instances import load_instance
from oracle.logits_oracle import uniforms
from tests import logits_common as lc
from tests.backends import native_test
from tests.beam_search_suite import enumerate_sequences, order_log_prob, rounds, search, twin_of
from tests.lookahead_priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, SHAPES, SMALL, TINY, shaped_table
from tests.lookahead_suite import _outputs, random_walk, snapshot
from tests.parity_common import batch_cfg, np_, synthetic_instance
from tests.priority_suite import random_table
from tests.sample_episodes_suite import check_schedule


def swor(env, table, k, order=True):
    """sample_without_replacement of a host (or device) table; the RNG counter must advance by J*M.  Returns the
    outputs as numpy arrays and the counter used."""
    si = env._step_index
    out = env.sample_without_replacement(lc._to_dev(env, table) if isinstance(table, np.ndarray) else table, k,
                                         order=order)
    assert env._step_index == si + env.jobs * env.machines
    return {k_: np_(v.detach()).copy() for k_, v in out.items()}, si


def olp(env, table, order):
    """order_log_prob of a host table and host orders (N, [k,] J, M): (log_prob, makespan) as numpy arrays."""
    import torch
    lp, ms = env.order_log_prob(lc._to_dev(env, table), torch.from_numpy(np.ascontiguousarray(order)).to(env.device))
    return np_(lp).copy(), np_(ms).copy()


def complete(out):
    return out["makespan"] >= 0


def seq_order(seq, J, M):
    """The order (J, M) of a job sequence from reset: the i-th allocation of job j is its operation i."""
    o = np.full((J, M), -1, np.int64)
    seen = np.zeros(J, np.int64)
    for r, j in enumerate(seq):
        o[j, seen[j]] = r
        seen[j] += 1
    return o


def tiny_instances(limit=32):
    """Synthetic instances with at most `limit` complete job sequences, with them: [(inst, [(seq, makespan)])]."""
    found = []
    for J, M, seed in ((2, 2, 1), (2, 3, 2), (3, 2, 3), (3, 2, 4), (2, 2, 5), (3, 2, 6), (2, 3, 7), (3, 2, 8)):
        inst = synthetic_instance(J, M, seed, max_dur=9, permutation=seed % 2 == 0)
        seqs = enumerate_sequences(inst)
        if len(seqs) <= limit:
            found.append((inst, seqs))
    return found


def seq_log_probs(make_env, inst, seqs, table):
    """The float64 log-likelihood of each sequence under the (1, J, M) table, from reset, on a batch of len(seqs)
    copies of `inst` stepped one decision at a time."""
    env = make_env(len(seqs), batch_cfg([inst] * len(seqs)), auto_reset=False, seed=1)
    env.reset()
    J, M = env.jobs, env.machines
    orders = np.stack([seq_order(s, J, M) for s, _ in seqs])
    lp = order_log_prob(make_env, env, table, orders)
    env.close()
    return lp


def check_slots(env, out):
    """The exact invariants on a clean table: complete slots first, key[:, 0] == 0 where a slot is complete, keys
    non-increasing over the complete slots, -1 / -inf / -inf after them, and the complete slots' orders pairwise
    distinct."""
    done = np_(env.done)
    for i in range(env.num_envs):
        ms, lp, key = out["makespan"][i], out["log_prob"][i], out["key"][i]
        if done[i]:
            assert (ms == -1).all() and (lp == 0).all() and (key == 0).all(), i
            continue
        full = ms >= 0
        c = int(full.sum())
        assert c >= 1 and full[:c].all(), (i, ms)
        assert key[0] == 0.0 and (np.diff(key[:c].astype(np.float64)) <= 0).all(), (i, key)
        assert np.isneginf(lp[c:]).all() and np.isneginf(key[c:]).all(), i
        if "order" in out:
            o = out["order"][i, :c].reshape(c, -1)
            assert len({row.tobytes() for row in o}) == c, i
            assert (out["order"][i, c:] == -1).all(), i


def replay_slots(make_env, env, out, table=None, schedules=None):
    """Every complete slot's order replays via rollout_priority(-order) on a twin to its makespan; with `table`, its
    log_prob equals order_log_prob(table, its order) bit for bit, and so does its makespan; with `schedules` (the
    instances), every replayed schedule is feasible (from reset)."""
    import torch
    n, k = out["makespan"].shape
    twin = twin_of(make_env, env, record_solution=schedules is not None)
    snap = snapshot(env)
    for s in range(k):
        full = out["makespan"][:, s] >= 0
        if not full.any():
            continue
        twin.reset()
        twin.import_state(snap)
        twin.rollout_priority(torch.from_numpy(-out["order"][:, s].astype(np.float32)).to(env.device))
        done, t = np_(twin.done), np_(twin.current_time_step)
        assert done[full].all() and np.array_equal(t[full], out["makespan"][full, s]), s
        if schedules is not None:
            sol = np_(twin.solution)
            for i in np.flatnonzero(full):
                check_schedule(schedules[i], sol[i], int(out["makespan"][i, s]))
    twin.close()
    if table is not None:
        lp, ms = olp(env, table, out["order"])
        full = complete(out)
        assert np.array_equal(lp[full].view(np.uint32), out["log_prob"][full].view(np.uint32))
        assert np.array_equal(ms[full], out["makespan"][full])


@native_test()
def swor_exhaustive(make_env, backend):
    """Tiny instances with at most 32 complete job sequences: width 32 returns every sequence exactly once, each slot's
    log_prob within 1e-5 (1 + R) of its sequence's float64 likelihood, and sum exp(log_prob) within 1e-5 of 1."""
    insts = tiny_instances()
    assert len(insts) >= 4
    for inst, seqs in insts:
        env = make_env(3, batch_cfg([inst] * 3), auto_reset=False, seed=4, env_id_base=2)
        env.reset()
        J, M = env.jobs, env.machines
        table = random_table(env, 5)[:1]
        want = seq_log_probs(make_env, inst, seqs, table)
        index = {seq_order(s, J, M).tobytes(): q for q, (s, _) in enumerate(seqs)}
        out, _ = swor(env, table, 32)
        for i in range(3):
            c = int(complete(out)[i].sum())
            assert c == len(seqs), (c, len(seqs))
            got = [index[out["order"][i, s].astype(np.int64).tobytes()] for s in range(c)]
            assert sorted(got) == list(range(c))
            for s, q in enumerate(got):
                assert out["makespan"][i, s] == seqs[q][1]
                assert abs(float(out["log_prob"][i, s]) - want[q]) <= 1e-5 * (1 + J * M), (s, q)
            assert abs(np.exp(out["log_prob"][i, :c].astype(np.float64)).sum() - 1.0) <= 1e-5
        check_slots(env, out)
        replay_slots(make_env, env, out, table)


@native_test(emu={"n": 384}, gpu={"n": 4096})
def swor_distribution(make_env, backend, n):
    """One call with a broadcast (1, J, M) table over n envs of one tiny instance, each env with its own noise: the
    frequency of slot 0's sequence against p(y), and of the ordered pair (slot 0, slot 1) against p(a) p(b) / (1 - p(a)),
    by chi-square tests at a fixed seed (bins of expected count below 5 pooled)."""
    from scipy.stats import chisquare
    inst, seqs = next((i, s) for i, s in tiny_instances() if 4 <= len(s) <= 12)
    env = make_env(n, batch_cfg([inst] * n), auto_reset=False, seed=21)
    env.reset()
    J, M = env.jobs, env.machines
    table = (np.random.default_rng(8).standard_normal((1, J, M)) * 0.7).astype(np.float32)
    p = np.exp(seq_log_probs(make_env, inst, seqs, table))
    assert abs(p.sum() - 1) < 1e-9
    index = {seq_order(s, J, M).tobytes(): q for q, (s, _) in enumerate(seqs)}
    out, _ = swor(env, table, 2)
    a = np.array([index[out["order"][i, 0].astype(np.int64).tobytes()] for i in range(n)])
    b = np.array([index[out["order"][i, 1].astype(np.int64).tobytes()] for i in range(n)])
    assert (a != b).all()

    def test(counts, probs):
        exp = probs * n
        big = exp >= 5
        f = np.append(counts[big], counts[~big].sum())
        e = np.append(exp[big], exp[~big].sum())
        if e[-1] == 0:
            f, e = f[:-1], e[:-1]
        return chisquare(f, e).pvalue

    c1 = np.bincount(a, minlength=len(seqs)).astype(np.float64)
    assert test(c1, p) > 1e-3, (c1, p * n)
    S = len(seqs)
    pair = (p[:, None] * p[None, :] / (1 - p[:, None])) * (1 - np.eye(S))
    c2 = np.bincount(a * S + b, minlength=S * S).astype(np.float64)
    assert test(c2, pair.ravel()) > 1e-3


@native_test(emu=[(s, t) for s in SHAPES for t in (False, True)], gpu=[(s, t) for s in SHAPES for t in (False, True)])
def swor_consistency(make_env, backend, shape, ties):
    """Every lane class in one batch (129..256 jobs and a non-permutation instance included) at reset and mid-episode,
    with some envs done; uniform tiny batches; (N, J, M), (N, J, 1) and (1, J, M) tables, with ties: the exact slot
    invariants; every slot's order replays to its makespan (from reset a feasible schedule) and its log_prob equals
    order_log_prob bit for bit; order_log_prob of beam_search's best order equals that slot's score bit for bit; and
    order_log_prob matches the float64 likelihood within 1e-5 (1 + R)."""
    if backend == "emu":
        names, walk, W = ["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY, SMALL], 170, 3
    else:
        names, walk, W = ["ta01", "ta21", "ta41", "ta61", "ta80", NONPERM, BIG_GPU, SMALL, TINY] * 2, 400, 8
    seed = SHAPES.index(shape) + (10 if ties else 0)
    for steps in (0, walk):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, env_id_base=5)
        env.reset()
        random_walk(env, steps)
        if steps:
            assert np_(env.done).any() and not np_(env.done).all()
        table = shaped_table(env, seed, ties, shape)
        out, _ = swor(env, table, W)
        check_slots(env, out)
        insts = [n if not isinstance(n, str) else load_instance(n) for n in names] if not steps else None
        replay_slots(make_env, env, out, table, insts)
        bs = search(env, table, W)
        lp, ms = olp(env, table, bs["order"])
        ok = bs["best"] >= 0
        best = bs["score"][np.arange(env.num_envs), np.maximum(bs["best"], 0)]
        assert np.array_equal(lp[ok].view(np.uint32), best[ok].view(np.uint32))
        R = rounds(snapshot(env), env)
        want = order_log_prob(make_env, env, table, out["order"][:, 0])
        live = complete(out)[:, 0]
        assert (np.abs(out["log_prob"][live, 0] - want[live]) <= 1e-5 * (1 + R[live])).all()
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        env = make_env(3, batch_cfg([synthetic_instance(J, M, J * 10 + M)] * 3), auto_reset=False, seed=seed)
        env.reset()
        table = shaped_table(env, seed, ties, shape)
        out, _ = swor(env, table, 4)
        check_slots(env, out)
        replay_slots(make_env, env, out, table)


def host_swor(make_env, env, table, W, step_index):
    """The stochastic beam search restated in float64 on the host over N*W twins, with the library's uniforms: each
    round export, gather the table at todo, take the log-softmax, perturb each candidate (G, Z, the key), keep the W best
    keys per env, import the parents into their slots, step.  Returns the makespans (N, W), the scores (N, W), the keys
    (N, W), the slots' orders (N, W, J, M) and whether the env's selections kept a margin of 2e-5 (1 + |key|) at every
    cut and between the final slots (where float32 rounding cannot change them)."""
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
    key = np.full((n, W), -np.inf)
    key[:, 0] = 0.0
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
        new_score, new_key = np.full((n, W), -np.inf), np.full((n, W), -np.inf)
        new_live = np.zeros((n, W), bool)
        for i in np.flatnonzero(act_on):
            u = uniforms(env.seed, env.env_id_base + i, step_index + r, W * 256).astype(np.float64)
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
                keep = lp > -np.inf
                lg, cs = lg[keep], score[i, b] + lp[keep]
                G = cs + -np.log(-np.log(u[b * 256 + lg]))
                z = int(np.argmax(G))
                T = key[i, b]
                with np.errstate(divide="ignore"):
                    d = G - G[z]
                    l1m = np.where(d > -np.log(2), np.log(-np.expm1(d)), np.log1p(-np.exp(d)))
                vv = T - G + l1m
                kv = np.minimum(T, T - np.maximum(vv, 0) - np.log1p(np.exp(-np.abs(vv))))
                kv[z] = T
                cands += [(kv[q], b, int(lg[q]), cs[q]) for q in range(lg.size)]
            cands.sort(key=lambda c: (-c[0], c[1], c[2]))
            pairs = zip(cands[:W], cands[1:W + 1]) if r == R[i] - 1 else zip(cands[W - 1:W], cands[W:W + 1])
            for a, b in pairs:
                if a[0] - b[0] <= 2e-5 * (1 + abs(a[0])):
                    safe[i] = False
            for s, (kv, b, j, cs) in enumerate(cands[:W]):
                parent[i, s], job[i, s], new_key[i, s], new_score[i, s], new_live[i, s] = b, j, kv, cs, True
            trace[r, i] = np.stack([parent[i], job[i]], 1)
        carry = ~act_on                                   # envs past their rounds keep their slots
        parent[carry] = np.arange(W)
        new_score[carry], new_key[carry], new_live[carry] = score[carry], key[carry], live[carry]
        rows = (np.arange(n)[:, None] * W + parent).ravel()
        x = {k: v[torch.from_numpy(rows).to(v.device)].clone() for k, v in x.items()}
        twin.import_state(x)
        twin.step(torch.from_numpy(job.ravel().astype(np.int32)).to(dev))
        score, key, live = new_score, new_key, new_live
    done = np_(twin.done).reshape(n, W)
    t = np_(twin.current_time_step).reshape(n, W)
    ms = np.where(live & done, t, -1)
    order = np.full((n, W, J, M), -1, np.int64)
    for i in range(n):
        for s in np.flatnonzero(ms[i] >= 0):
            at, seen = int(s), np.zeros(J, np.int64)
            for r in range(int(R[i]) - 1, -1, -1):
                b, j = trace[r, i, at]
                order[i, s, j, env.env_machines[i] - 1 - seen[j]] = r
                seen[j] += 1
                at = int(b)
    twin.close()
    return ms, score, key, order, safe


@native_test(emu=[(3, 40)], gpu=[(8, 0)])
def swor_host_restatement(make_env, backend, width, steps):
    """The search against its float64 restatement on N*W twins with the same uniforms: makespans and orders equal, and
    log_prob and key within 1e-5 (1 + R) and 1e-4 (1 + |key|), for every env whose selections keep their margins (most
    of them).  GPU: ta80 at N = 8, W = 8, from reset."""
    names = {"emu": ["ta01", SMALL, NONPERM, TINY, SMALL, TINY], "gpu": ["ta80"] * 8}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=9, env_id_base=3)
    env.reset()
    random_walk(env, steps)
    table = random_table(env, 19) * {"emu": 1, "gpu": 4}[backend]
    out, si = swor(env, table, width)
    ms, score, key, order, safe = host_swor(make_env, env, table, width, si)
    R = rounds(snapshot(env), env)
    assert safe.mean() >= 0.5, safe
    for i in np.flatnonzero(safe):
        assert np.array_equal(out["makespan"][i], ms[i]), (i, out["makespan"][i], ms[i])
        Ji, Mi = env.env_jobs[i], env.env_machines[i]
        assert np.array_equal(out["order"][i, :, :Ji, :Mi], order[i, :, :Ji, :Mi]), i
        full = ms[i] >= 0
        assert (np.abs(out["log_prob"][i, full] - score[i, full]) <= 1e-5 * (1 + R[i])).all(), i
        assert (np.abs(out["key"][i, full] - key[i, full]) <= 1e-4 * (1 + np.abs(key[i, full]))).all(), i


def decisions(make_env, env, order):
    """The decisions of each (env, order) episode from env's state on a twin: per env and order a list of (legal jobs,
    their current operations, the chosen job), forced no-ops left out; None where the order is all -1 or env is done."""
    import torch
    n, J = env.num_envs, env.jobs
    k = order.shape[1]
    twin = twin_of(make_env, env)
    snap = snapshot(env)
    res = [[None] * k for _ in range(n)]
    for s in range(k):
        twin.import_state(snap)
        o = order[:, s]
        live = (o.reshape(n, -1) >= 0).any(1) & ~np_(env.done)
        dec = [[] for _ in range(n)]
        while True:
            x = twin.export_state()
            legal, todo = np_(x["legal"]).astype(bool)[:, :J], np_(x["todo"]).astype(np.int64)
            done = np_(twin.done)
            act = np.full(n, N.ACTION_SKIP, np.int32)
            for i in np.flatnonzero(live & ~done):
                lg = np.flatnonzero(legal[i, :int(env.env_jobs[i])])
                if not lg.size:
                    act[i] = int(env.env_jobs[i])
                    continue
                ks = todo[i, lg]
                j = int(lg[np.argmax(-o[i, lg, ks])])
                dec[i].append((lg, ks, j))
                act[i] = j
            if (act == N.ACTION_SKIP).all():
                break
            twin.step(torch.from_numpy(act).to(env.device))
        for i in np.flatnonzero(live):
            res[i][s] = dec[i]
    twin.close()
    return res


def f64_grad(dec, table, w):
    """d/d table of sum w[i, s] log p_s[i] in float64 autograd, the likelihood restated from the decisions; the table
    any shape that broadcasts to (N, J, M)."""
    import torch
    x = torch.tensor(np.asarray(table, np.float64), requires_grad=True)
    n = len(dec)
    total = torch.zeros((), dtype=torch.float64)
    for i in range(n):
        xi = x[min(i, x.shape[0] - 1)]
        for s, d in enumerate(dec[i]):
            if d is None or w[i, s] == 0:
                continue
            lp = torch.zeros((), dtype=torch.float64)
            for lg, ks, j in d:
                v = xi[torch.from_numpy(lg), torch.from_numpy(np.minimum(ks, xi.shape[1] - 1))]
                lp = lp + v[int(np.flatnonzero(lg == j)[0])] - torch.logsumexp(v, 0)
            total = total + float(w[i, s]) * lp
    total.backward()
    return x.grad.numpy()


@native_test()
def swor_gradient(make_env, backend):
    """order_log_prob backward against float64 autograd of the restated likelihood for (N, J, M), (N, J, 1), (1, J, M)
    and float64 tables; splits agree within tolerance and a repeated split is bit-identical; SWOR's log_prob.backward(w)
    equals order_log_prob's on the returned orders bit for bit; NaN samples, done envs and zero weights add nothing; a
    table changed in place before backward raises."""
    import pytest
    import torch
    names = {"emu": ["ta01", SMALL, TINY, NONPERM], "gpu": ["ta01", "ta41", "ta80", SMALL, TINY] * 2}[backend]
    k = 3
    rng = np.random.default_rng(17)
    for shape_of, dtype in ((lambda n, J, M: (n, J, M), torch.float32), (lambda n, J, M: (n, J, 1), torch.float32),
                            (lambda n, J, M: (1, J, M), torch.float32), (lambda n, J, M: (n, J, M), torch.float64)):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
        env.reset()
        random_walk(env, 20)
        n, J, M, dev = env.num_envs, env.jobs, env.machines, env.device
        shape = shape_of(n, J, M)
        base = torch.from_numpy(rng.standard_normal(shape)).to(dev, dtype)
        w = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).to(dev)
        x = base.clone().requires_grad_(True)
        si = env._step_index
        out = env.sample_without_replacement(x, k, order=True)
        assert out["log_prob"].grad_fn is not None and out["key"].grad_fn is None
        out["log_prob"].backward(w, retain_graph=True)
        g_swor = x.grad.clone()
        x.grad = None
        out["log_prob"].backward(w)
        assert torch.equal(g_swor, x.grad)
        assert x.grad.dtype == dtype and tuple(x.grad.shape) == shape
        x.grad = None
        lp, _ = env.order_log_prob(x, out["order"])
        lp.backward(w)
        assert torch.equal(g_swor, x.grad), shape
        assert env._step_index == si + J * M
        order = np_(out["order"])
        dec = decisions(make_env, env, order)
        wn = np_(w).astype(np.float64)
        want = f64_grad(dec, base.to(torch.float32).cpu().numpy(), wn)
        assert np.abs(np_(x.grad).astype(np.float64) - want).max() <= 1e-4 * (1 + np.abs(want).max()), shape
        xo = lc._to_dev(env, base.to(torch.float32).cpu().numpy())
        o = out["order"].contiguous()
        g1 = np_(env._order_log_prob_grad(xo, o, w, 1).sum(0)).astype(np.float64)
        for split in (2, 3):
            ga = np_(env._order_log_prob_grad(xo, o, w, split)).copy()
            gb = np_(env._order_log_prob_grad(xo, o, w, split))
            assert np.array_equal(ga.view(np.uint32), gb.view(np.uint32)), split
            assert np.abs(ga.sum(0) - g1).max() <= 1e-5 * (1 + np.abs(g1).max()), split
    # NaN samples, done envs and zero weights
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=4)
    env.reset()
    random_walk(env, 30 if backend == "emu" else 200)
    n = env.num_envs
    table = random_table(env, 19)
    clean, _ = swor(env, table, 4)
    x_ = env.export_state()
    todo = np_(x_["todo"])
    bad_env = int(np.flatnonzero(~np_(env.done))[0])
    Ji, Mi = int(env.env_jobs[bad_env]), int(env.env_machines[bad_env])
    table[bad_env, :, min(int(todo[bad_env, :Ji].max()) + 1, Mi - 1):] = np.nan
    lp, _ = olp(env, table, clean["order"])
    nan = np.isnan(lp)
    assert nan[bad_env].any(), lp[bad_env]
    dev_t = lc._to_dev(env, table)
    o = torch.from_numpy(clean["order"]).to(env.device).contiguous()
    wn = rng.standard_normal((n, 4)).astype(np.float32)
    wz = wn.copy()
    wz[nan] = 0.0
    wz[np_(env.done)] = 0.0
    wz[:, 1] = 0.0
    wn[:, 1] = 0.0
    for split in (1, 3):
        ga = np_(env._order_log_prob_grad(dev_t, o, torch.from_numpy(wn).to(env.device), split))
        gb = np_(env._order_log_prob_grad(dev_t, o, torch.from_numpy(wz).to(env.device), split))
        assert np.array_equal(ga, gb), split
        for i in np.flatnonzero(np_(env.done)):
            assert (ga[:, i] == 0).all(), i
    # in-place change between forward and backward
    x = torch.from_numpy(random_table(env, 20)).to(env.device).requires_grad_(True)
    y = x * 1.0
    out = env.sample_without_replacement(y, 2)
    with torch.no_grad():
        y.add_(1.0)
    with pytest.raises(RuntimeError):
        out["log_prob"].sum().backward()
    y = x * 1.0
    lp, _ = env.order_log_prob(y, o[:, 0])
    with torch.no_grad():
        y.add_(1.0)
    with pytest.raises(RuntimeError):
        lp.sum().backward()
    out = env.sample_without_replacement(torch.from_numpy(random_table(env, 21)).to(env.device), 2)
    assert out["log_prob"].grad_fn is None


@native_test()
def swor_determinism(make_env, backend):
    """Repeated calls at the same counter are bit-identical; a permuted batch gives each env the rows of a one-env batch
    with its global env id; env_id_base shards give the same rows; widths 1, 4, 16 and 32 keep the invariants."""
    names = {"emu": ["ta01", SMALL, NONPERM, *EMU_CLASSES[:1], TINY],
             "gpu": ["ta01", "ta31", "ta51", "ta80", NONPERM, BIG_GPU, SMALL, TINY] * 2}[backend]
    n = len(names)
    env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=31)
    env.reset()
    table = random_table(env, 14)
    W = 4
    a, si = swor(env, table, W)
    env._step_index = si
    b, _ = swor(env, table, W)
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    cut = n // 2
    for lo, hi in ((0, cut), (cut, n)):
        s = make_env(hi - lo, batch_cfg(names[lo:hi], sort=False), auto_reset=False, seed=31, env_id_base=lo)
        s.reset()
        s._step_index = si
        so, _ = swor(s, np.ascontiguousarray(table[lo:hi, :s.jobs, :s.machines]), W)
        assert np.array_equal(so["makespan"], a["makespan"][lo:hi]), lo
        for k in ("log_prob", "key"):
            assert np.array_equal(so[k].view(np.uint32), a[k][lo:hi].view(np.uint32)), (lo, k)
        for i in range(hi - lo):
            Jp, Mp = s.env_jobs[i], s.env_machines[i]
            assert np.array_equal(so["order"][i, :, :Jp, :Mp], a["order"][lo + i, :, :Jp, :Mp]), i
    perm = np.random.default_rng(3).permutation(n)
    pe = make_env(n, batch_cfg([names[p] for p in perm], sort=False), auto_reset=False, seed=31)
    pe.reset()
    pe._step_index = si
    pt = np.ascontiguousarray(table[perm, :pe.jobs, :pe.machines])
    po, _ = swor(pe, pt, W)
    for i in range(0, n, max(1, n // 4)):
        one = make_env(1, batch_cfg([names[perm[i]]]), auto_reset=False, seed=31, env_id_base=i)
        one.reset()
        one._step_index = si
        oo, _ = swor(one, np.ascontiguousarray(pt[i:i + 1, :one.jobs, :one.machines]), W)
        for k in ("makespan", "log_prob", "key"):
            assert np.array_equal(oo[k][0].view(np.uint8), po[k][i].view(np.uint8)), (i, k)
    for W in (1, 4, 16, 32):
        out, _ = swor(env, table, W)
        check_slots(env, out)
        if W == 1:
            assert (out["makespan"][:, 0] >= 0).all()


@native_test(emu=[False, True], gpu=[False, True])
def swor_no_side_effects(make_env, backend, auto_reset):
    """Every output, the exported state, stats(), solution and flags are unchanged by the draws, order_log_prob and its
    gradient; one launch per lane class present per call; the counter advances by exactly J*M per draw and not at all
    for order_log_prob; after a recording step the calls leave real_obs stale."""
    import torch
    names = {"emu": ["ta01", SMALL, *EMU_CLASSES[:1], TINY], "gpu": ["ta01", "ta41", "ta80", BIG_GPU, TINY] * 3}[backend]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=auto_reset, seed=7, record_solution=True)
    env.reset()
    random_walk(env, 30)
    table = random_table(env, 3)
    before, stats = _outputs(env), env.stats()
    classes = len({0 if J <= 32 else 1 if J <= 64 else 2 if J <= 128 else 3 for J in env.env_jobs})
    c = env.launch_count
    out, _ = swor(env, table, 4)
    swor(env, table, 3, order=False)
    assert env.launch_count == c + 2 * classes
    si = env._step_index
    o = torch.from_numpy(out["order"]).to(env.device).contiguous()
    olp(env, table, out["order"])
    env._order_log_prob_grad(lc._to_dev(env, table), o, torch.ones((env.num_envs, 4), device=env.device), 2)
    assert env._step_index == si
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
    qa, _ = swor(a_env, table, 2)
    qb, _ = swor(b_env, table, 2)
    for k in qa:
        assert np.array_equal(qa[k].view(np.uint8), qb[k].view(np.uint8)), k
    olp(a_env, table, qa["order"])
    assert np.array_equal(np_(a_env.real_obs), stale)


@native_test()
def swor_bad_tables(make_env, backend):
    """A NaN on the root's decision or every legal job at -inf gives -1 / NaN / NaN (order_log_prob NaN); a NaN never
    read changes nothing; an env done at entry reads -1 / 0 / 0 (order_log_prob -1 / 0); an imported state with nothing
    legal gives -1 / -inf / -inf."""
    names = ["ta01", "ta01", "ta01", SMALL, "ta01", "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=3)
    env.reset()
    random_walk(env, 20)
    x = env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    clean = random_table(env, 31)
    ref, si = swor(env, clean, 4)
    bad = clean.copy()
    j0 = int(np.flatnonzero(legal[0])[0])
    bad[0, j0, todo[0, j0]] = np.nan
    bad[1] = -np.inf
    bad[3, 9:, :] = np.nan                                # columns past J_i = 9: never read
    bad[3, :, 4:] = np.inf                                # operations past M_i = 4
    ops = np.arange(env.machines)
    bad[4][ops[None, :] < todo[4][:, None]] = np.nan      # operations already allocated: never read
    env._step_index = si
    out, _ = swor(env, bad, 4)
    for i in (0, 1):
        assert (out["makespan"][i] == -1).all() and np.isnan(out["log_prob"][i]).all(), i
        assert np.isnan(out["key"][i]).all() and out["best"][i] == -1 and (out["order"][i] == -1).all(), i
    for i in (2, 3, 4, 5):
        for k in ("makespan", "log_prob", "key", "order"):
            assert np.array_equal(out[k][i].view(np.uint8), ref[k][i].view(np.uint8)), (i, k)
    lp, ms = olp(env, bad, ref["order"])
    assert np.isnan(lp[0]).all() and np.isnan(lp[1]).all() and (ms[:2] == -1).all()
    assert np.array_equal(lp[2:].view(np.uint32), ref["log_prob"][2:].view(np.uint32))
    # done at entry, and an imported state with nothing legal
    x = env.export_state()
    x["flags"][5] = int(x["flags"][5]) | (N.FLAG_DONE << 8)
    x["legal"][2] = 0
    x["flags"][2] = int(x["flags"][2]) & ~(N.FLAG_NOOP_LEGAL << 8)
    env.import_state(x)
    assert np_(env.done)[5]
    o3, _ = swor(env, clean, 4)
    assert (o3["makespan"][5] == -1).all() and (o3["log_prob"][5] == 0).all() and (o3["key"][5] == 0).all()
    assert (o3["makespan"][2] == -1).all() and np.isneginf(o3["log_prob"][2]).all() and o3["best"][2] == -1
    assert np.isneginf(o3["key"][2]).all()
    lp, ms = olp(env, clean, ref["order"])
    assert (lp[5] == 0).all() and (ms[5] == -1).all()


@native_test()
def swor_abi(make_env, backend):
    """JSS_ERR_INVALID for NULL or misaligned pointers (order_out may be NULL), a negative stride, width or k out of
    range, ld < width / k, and a split outside 1..k; JSS_ERR_STATE before jss_assign; a bad shape, k or order raises
    ValueError before the native call."""
    import pytest
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    L, h, st = env._L, env._h, env._stream()
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    i32 = torch.zeros(n * 64, dtype=torch.int32, device=env.device)
    f32 = torch.zeros(n * 64, dtype=torch.float32, device=env.device)
    g32 = torch.zeros(n * 64, dtype=torch.float32, device=env.device)
    od = torch.zeros(n * 32 * J * M, dtype=torch.int32, device=env.device)
    gr = torch.zeros(4 * n * J * M, dtype=torch.float32, device=env.device)
    p, o, q, kq, r, gp = t.data_ptr(), i32.data_ptr(), f32.data_ptr(), g32.data_ptr(), od.data_ptr(), gr.data_ptr()
    s = (J * M, M, 1)
    bad = ((None, *s, 4, o, q, kq, 4, r), (p + 2, *s, 4, o, q, kq, 4, r), (p, -1, M, 1, 4, o, q, kq, 4, r),
           (p, J * M, -M, 1, 4, o, q, kq, 4, r), (p, J * M, M, -1, 4, o, q, kq, 4, r), (p, *s, 0, o, q, kq, 4, r),
           (p, *s, 33, o, q, kq, 33, r), (p, *s, 4, o, q, kq, 3, r), (p, *s, 4, None, q, kq, 4, r),
           (p, *s, 4, o + 2, q, kq, 4, r), (p, *s, 4, o, None, kq, 4, r), (p, *s, 4, o, q + 2, kq, 4, r),
           (p, *s, 4, o, q, None, 4, r), (p, *s, 4, o, q, kq + 2, 4, r), (p, *s, 4, o, q, kq, 4, r + 2))
    for args in bad:
        a = args[:4] + (1, 0) + args[4:]
        assert L.jss_sample_without_replacement(h, *a, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_sample_without_replacement:"), args
    assert L.jss_sample_without_replacement(h, p, *s, 1, 0, 32, o, q, kq, 32, None, st) == 0
    assert L.jss_sample_without_replacement(h, p, *s, 1, 0, 1, o, q, kq, 1, r, st) == 0
    bad = ((None, *s, r, 2, o, q, 2), (p + 2, *s, r, 2, o, q, 2), (p, -1, M, 1, r, 2, o, q, 2),
           (p, *s, None, 2, o, q, 2), (p, *s, r + 2, 2, o, q, 2), (p, *s, r, 0, o, q, 2), (p, *s, r, 2, o, q, 1),
           (p, *s, r, 2, None, q, 2), (p, *s, r, 2, o + 2, q, 2), (p, *s, r, 2, o, None, 2), (p, *s, r, 2, o, q + 2, 2))
    for args in bad:
        assert L.jss_order_log_prob(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_order_log_prob:"), args
    assert L.jss_order_log_prob(h, p, *s, r, 2, o, q, 2, st) == 0
    bad = ((None, *s, r, 2, q, 2, 1, gp), (p, *s, None, 2, q, 2, 1, gp), (p, *s, r, 0, q, 2, 1, gp),
           (p, *s, r, 2, q, 1, 1, gp), (p, *s, r, 2, None, 2, 1, gp), (p, *s, r, 2, q + 2, 2, 1, gp),
           (p, *s, r, 2, q, 2, 0, gp), (p, *s, r, 2, q, 2, 3, gp), (p, *s, r, 2, q, 2, 1, None),
           (p, *s, r, 2, q, 2, 1, gp + 2), (p, J * M, -M, 1, r, 2, q, 2, 1, gp))
    for args in bad:
        assert L.jss_order_log_prob_grad(h, *args, st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_order_log_prob_grad:"), args
    assert L.jss_order_log_prob_grad(h, p, *s, r, 2, q, 2, 2, gp, st) == 0
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_sample_without_replacement(raw, p, *s, 1, 0, 4, o, q, kq, 4, r, st) == -5
    assert L.jss_order_log_prob(raw, p, *s, r, 2, o, q, 2, st) == -5
    assert L.jss_order_log_prob_grad(raw, p, *s, r, 2, q, 2, 1, gp, st) == -5
    L.jss_destroy(raw)
    for badt in (t[0], t[None], t[:, :J - 1], torch.zeros((3, J, M), device=env.device)):
        with pytest.raises(ValueError):
            env.sample_without_replacement(badt, 2)
        with pytest.raises(ValueError):
            env.order_log_prob(badt, torch.zeros((n, J, M), dtype=torch.int32, device=env.device))
    for k in (0, 33):
        with pytest.raises(ValueError):
            env.sample_without_replacement(t, k)
    for bo in (torch.zeros((n, J, M)), torch.zeros((n, J, M - 1), dtype=torch.int32),
               torch.zeros((n + 1, J, M), dtype=torch.int64), torch.zeros((n, 0, J, M), dtype=torch.int32),
               torch.zeros((J, M), dtype=torch.int32)):
        with pytest.raises(ValueError):
            env.order_log_prob(t, bo.to(env.device))


@native_test(emu=None)
def swor_full_size_ta80(make_env):
    """ta80 at N = 256, W = 16, per-env random normal tables, from reset: the exact invariants, every slot's order
    replays to its makespan with a feasible schedule, and its log_prob equals order_log_prob bit for bit."""
    import torch
    n, W = 256, 16
    env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=15)
    env.reset()
    table = torch.randn((n, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(23),
                        device=env.device)
    out, _ = swor(env, table, W)
    assert (out["makespan"] > 0).all() and np.isfinite(out["log_prob"]).all() and np.isfinite(out["key"]).all()
    check_slots(env, out)
    inst = load_instance("ta80")
    replay_slots(make_env, env, out, table.cpu().numpy(), [inst] * n)
