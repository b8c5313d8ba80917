"""The tests of the policy-entropy forms of the three differentiable log-probability producers
(rollout_priority_sample, sample_episodes and order_log_prob with entropy=True), declared once for both backends
(tests/backends.py) and collected by tests/test_emu_entropy.py and tests/test_gpu_entropy.py.  The entropy of each
decision is H_t = log S - T/S over the legal jobs (jss_b200.h); an episode's entropy is the fp32 sum of its H_t.  Each
call is checked against a twin env stepped with step_logits on the gathered rows, the entropy and both gradients
against a float64 torch restatement of the twin's decisions run through autograd, and the entropy forms against the
calls without entropy, bit for bit, for everything those report."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.lookahead_priority_suite import EMU_CLASSES, NONPERM, SMALL, TINY, noop_only
from tests.lookahead_suite import random_walk, snapshot
from tests.parity_common import assert_twins_equal, batch_cfg, np_, synthetic_instance, twin_envs
from tests.priority_suite import BIG_GPU, greedy_rows, random_table
from tests.sample_episodes_suite import bound

# The kernels form exp and log with the MUFU approximations (relative error about 2^-21 near 0, growing with |d|), so
# one decision's H_t, a sum of J terms e_j d_j / S next to log S, carries an absolute error of a few 1e-7 per term;
# 4e-6 per decision covers it with room.  1e-5 relative covers the fp32 summation of up to 2 J M + 1 decisions.
ENT_REL, ENT_PER_DECISION = 1e-5, 4e-6


class EntTwin:
    """Steps a twin env with step_logits on the gathered rows of a logit table (or, with `driver`, greedily on the
    rows of the table `driver`, as order_log_prob replays an order) and restates, in float64 torch, each env's episode
    entropy and log-probability over the decisions it takes, so that autograd gives both gradients with respect to the
    table."""

    def __init__(self, env, table, driver=None):
        import torch
        n, J, M = env.num_envs, env.jobs, env.machines
        self.env, self.driver = env, driver
        self.table = np.ascontiguousarray(np.broadcast_to(table, (n, J, M)), np.float32)
        self.x = torch.tensor(self.table.astype(np.float64), requires_grad=True)
        self.h = [[] for _ in range(n)]
        self.lp = [[] for _ in range(n)]
        self.count = np.zeros((n, J, M), np.int64)
        self.decisions = np.zeros(n, np.int64)
        self.bad = np.zeros(n, bool)
        self.actions = [[] for _ in range(n)]
        self.log_prob32 = np.zeros(n, np.float32)          # the twin's log_probs summed in fp32, as the kernel sums

    def steps(self, k, step_index):
        import torch
        env = self.env
        env._step_index = step_index
        for _ in range(k):
            if np_(env.done).all():
                return
            rows = greedy_rows(env, self.table)
            todo = np_(env.export_state()["todo"]).copy()
            mask = np_(env.action_mask).copy()
            done = np_(env.done).copy()
            if self.driver is None:
                _, _, _, _, info = env.step_logits(lc._to_dev(env, rows))
            else:
                _, _, _, _, info = env.step_greedy(lc._to_dev(env, greedy_rows(env, self.driver)))
            acts, lp = np_(info["actions"]), np_(info["log_prob"])
            if self.driver is None:
                self.log_prob32 = (self.log_prob32 + lp).astype(np.float32)
            for i in np.flatnonzero(~done):
                self.actions[i].append(int(acts[i]))
                js = np.flatnonzero(mask[i, :int(env.env_jobs[i])])
                if not len(js) or self.bad[i]:
                    continue                              # a forced no-op, or after the episode met a bad row
                x = rows[i, js]
                if np.isnan(x).any() or (x == np.inf).any() or x.max() == -np.inf:
                    self.bad[i] = True
                    continue
                ks = todo[i, js]
                ls = torch.log_softmax(self.x[i, js, ks], 0)
                live = torch.from_numpy(x > -np.inf)      # p = 0 at -inf: no 0 * -inf
                p = ls.exp()
                self.h[i].append(-(p[live] * ls[live]).sum())
                self.lp[i].append(ls[torch.from_numpy(js == acts[i])].sum())
                self.count[i, js, ks] += 1
                self.decisions[i] += 1

    def entropy(self):
        """Each env's float64 episode entropy, NaN for an env whose episode met a bad row."""
        h = np.array([float(sum(t).item()) if t else 0.0 for t in self.h])
        return np.where(self.bad, np.nan, h)

    def grads(self):
        """The float64 (dH/dx, dlogp/dx), zero rows for the envs whose episode met a bad row."""
        import torch
        if getattr(self, "_grads", None) is None:
            out = []
            for terms in (self.h, self.lp):
                total = sum((t for i, ts in enumerate(terms) if not self.bad[i] for t in ts),
                            torch.zeros((), dtype=torch.float64))
                g = (torch.autograd.grad(total, self.x, retain_graph=True, allow_unused=True)[0]
                     if total.requires_grad else None)
                out.append(np.zeros(self.table.shape) if g is None else g.numpy().copy())
            self._grads = out
        return self._grads


def ent_call(env, table, n_steps=None, grad=True):
    """rollout_priority_sample_entropy's native call: (log_prob, entropy, grad, entropy_grad), the gradient buffers
    pre-filled with NaN so that entries the call must not write stay NaN."""
    import torch
    n, J, M = env.num_envs, env.jobs, env.machines
    g = torch.full((n, J, M), float("nan"), device=env.device) if grad else None
    gh = torch.full((n, J, M), float("nan"), device=env.device) if grad else None
    lp, h = env._rollout_priority_sample(table, 2 * J * M + 1 if n_steps is None else n_steps, g, True, gh)
    return (np_(lp).copy(), np_(h).copy(), np_(g).copy() if grad else None, np_(gh).copy() if grad else None)


def plain_call(env, table, n_steps=None):
    """rollout_priority_sample's native call without entropy: (log_prob, grad)."""
    import torch
    n, J, M = env.num_envs, env.jobs, env.machines
    g = torch.full((n, J, M), float("nan"), device=env.device)
    lp = env._rollout_priority_sample(table, 2 * J * M + 1 if n_steps is None else n_steps, g)
    return np_(lp).copy(), np_(g).copy()


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def assert_entropy(got, twin, ctx):
    """The kernel's fp32 episode entropies against the twin's float64 ones: NaN exactly where the twin's episode met a
    bad row, else within ENT_REL relative plus ENT_PER_DECISION per decision."""
    want = twin.entropy()
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (ctx, got, want)
    tol = ENT_REL * np.abs(want[~nan]) + ENT_PER_DECISION * twin.decisions[~nan]
    assert (np.abs(got[~nan] - want[~nan]) <= tol).all(), (ctx, np.abs(got[~nan] - want[~nan]).max())


def assert_grads(env, g, gh, twin, ctx):
    """Both gradient tables against the float64 autograd of the twin's restatement, within 2e-5 per decision an entry
    took part in plus 1e-5 relative; zero rows for envs whose episode met a bad row; padding untouched (NaN)."""
    wh, wl = twin.grads()
    for i, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        for got, want, what in ((g, wl, "log_prob"), (gh, wh, "entropy")):
            a, b = got[i, :Ji, :Mi].astype(np.float64), want[i, :Ji, :Mi]
            if twin.bad[i]:
                assert (a == 0).all(), (ctx, what, i)
            else:
                tol = 2e-5 * (1 + twin.count[i, :Ji, :Mi]) + 1e-5 * np.abs(b)
                assert (np.abs(a - b) <= tol).all(), (ctx, what, i, np.abs(a - b).max())
            assert np.isnan(got[i, Ji:]).all() and np.isnan(got[i, :, Mi:]).all(), (ctx, what, i, "padding written")


def check_rollout(make_env, names, table, k, walk=0, noop_env=False, seed=1):
    """rollout_priority_sample(entropy=True) for k decisions, then to the end, from reset or after `walk` random
    steps: state, counter, log_prob and d log_prob / dx bit for bit those of the call without entropy on a twin batch;
    entropy and both gradients against the float64 restatement of a step_logits twin.  Returns the twins of the two
    calls."""
    envs = [make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True, seed=seed)
            for _ in range(3)]
    for e in envs:
        e.reset()
        random_walk(e, walk)
    if noop_env:
        x = envs[0].export_state()
        i = int(np.flatnonzero(~np_(envs[0].done))[0])
        x["legal"][i] = 0
        x["flags"][i] = int(x["flags"][i]) | (N.FLAG_NOOP_LEGAL << 8)
        for e in envs:
            e.import_state(x)
        assert noop_only(envs[0])[i]
    a_env, c_env, b_env = envs
    dev = lc._to_dev(a_env, table)
    si = a_env._step_index
    twins = []
    for n_steps in (k, None):
        counter = a_env._step_index
        lp, h, g, gh = ent_call(a_env, dev, n_steps)
        lp_c, g_c = plain_call(c_env, dev, n_steps)
        assert a_env._step_index == c_env._step_index
        assert_twins_equal(a_env, c_env, ("entropy off", n_steps), state=True, stats=True)
        assert np.array_equal(np_(a_env.solution), np_(c_env.solution))
        assert np.array_equal(bits(lp), bits(lp_c)), n_steps
        assert np.array_equal(g, g_c, equal_nan=True), n_steps
        twin = EntTwin(b_env, table)
        twin.steps(2 * a_env.jobs * a_env.machines + 1 if n_steps is None else n_steps, counter)
        assert_twins_equal(a_env, b_env, ("twin", n_steps), state=True)
        assert_entropy(h, twin, n_steps)
        assert_grads(a_env, g, gh, twin, n_steps)
        twins.append(twin)
    assert a_env._step_index > si
    return twins


@native_test(emu=["mixed", "uniform"], gpu=["mixed", "uniform"])
def entropy_twin(make_env, backend, batch):
    """Every lane class (129..256 jobs and a non-permutation instance included) and uniform batches (J <= 4 and ta01),
    from reset and mid-episode with an env whose only legal action is the no-op: the entropy form against the plain call
    and the float64 restatement, entropy and both gradients."""
    if batch == "mixed":
        names = (["ta01", "ta01", *EMU_CLASSES, NONPERM] if backend == "emu" else
                 ["ta01", "ta21", "ta41", "ta61", "ta80", NONPERM, BIG_GPU, SMALL] * 2)
        for walk, k in ((0, 17), (30, 40)):
            env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False)
            check_rollout(make_env, names, random_table(env, 3 + walk), k, walk=walk, noop_env=walk > 0)
    else:
        for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
            names = [synthetic_instance(J, M, J * 10 + M)] * 3
            env = make_env(3, batch_cfg(names), auto_reset=False)
            check_rollout(make_env, names, random_table(env, J + M, ties=True), 2)
        names = ["ta01"] * {"emu": 3, "gpu": 16}[backend]
        env = make_env(len(names), batch_cfg(names), auto_reset=False)
        check_rollout(make_env, names, random_table(env, 5), 60, walk=20)


@native_test()
def entropy_edges(make_env, backend):
    """One job of nonzero probability (one legal job, or every other legal job at -inf): entropy and its gradient
    exactly 0; -inf entries among legal jobs; a constant table (H_t = log |L_t|, dH/dx = 0); large and shifted logits;
    bad rows (NaN exactly where log_prob is NaN, zero rows); envs done at entry (0)."""
    import torch
    # a single job: every decision has one legal job
    one = [synthetic_instance(1, 4, 7)] * 3
    env = make_env(3, batch_cfg(one), auto_reset=False, seed=2)
    env.reset()
    lp, h, g, gh = ent_call(env, lc._to_dev(env, random_table(env, 1)))
    assert np_(env.done).all()
    assert (bits(h) == 0).all() and (bits(lp) == 0).all(), (h, lp)
    assert (gh[:, :1, :4] == 0).all() and not np.signbit(gh[:, :1, :4]).any()
    # every legal job but one at -inf: the first decision from reset on ta01
    names = ["ta01"] * 4
    env = make_env(4, batch_cfg(names), auto_reset=False, seed=2)
    env.reset()
    t = random_table(env, 2)
    t[:, 1:, 0] = -np.inf
    lp, h, g, gh = ent_call(env, lc._to_dev(env, t), 1)
    assert (bits(h) == 0).all() and (bits(lp) == 0).all(), (h, lp)
    assert (gh == 0).all() and (g == 0).all()
    # -inf among legal jobs, constant, large and shifted tables
    base = random_table(env, 4)
    ninf = base.copy()
    ninf[np.random.default_rng(5).random(base.shape) < 0.3] = -np.inf
    for what, table in (("ninf", ninf), ("constant", np.full_like(base, 0.25)), ("large", base * 1e3),
                        ("shifted", base + 1e4)):
        first, _ = check_rollout(make_env, names, table, 4 if what == "ninf" else 25, walk=3, seed=6)
        if what == "ninf":                                # a job at -inf ends its episode with a bad row once it is
            assert not first.bad.all(), what              # the last legal one, so the first call checks the rest
    # the constant table's entropy is the sum of log |L_t|
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, seed=6)
    const = np.zeros((4, a_env.jobs, a_env.machines), np.float32)
    sizes = np.zeros(4)
    b_env._step_index = 0
    while not np_(b_env.done).all():
        m = np_(b_env.action_mask)[:, :b_env.jobs]
        live = ~np_(b_env.done)
        sizes[live] += np.log(np.maximum(m[live].sum(1), 1))
        b_env.step_logits(lc._to_dev(b_env, greedy_rows(b_env, const)))
    _, h, _, gh = ent_call(a_env, lc._to_dev(a_env, const))
    assert (np.abs(h - sizes) <= ENT_REL * sizes + ENT_PER_DECISION * 2 * a_env.jobs * a_env.machines).all(), (h, sizes)
    assert np.abs(gh).max() <= 1e-4
    # bad rows: NaN where log_prob is NaN, zero rows; entries never read change nothing
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, seed=7)
    bad = random_table(a_env, 11)
    bad[0, 3, 0] = np.nan
    bad[1, :, 4] = np.inf
    bad[2, :, 0] = -np.inf
    lp, h, g, gh = ent_call(a_env, lc._to_dev(a_env, bad))
    lp_b, g_b = plain_call(b_env, lc._to_dev(b_env, bad))
    assert np.array_equal(bits(lp), bits(lp_b)) and np.array_equal(g, g_b, equal_nan=True)
    assert np.array_equal(np.isnan(h), np.isnan(lp)) and np.isnan(h[:3]).all() and np.isfinite(h[3])
    for i in range(3):
        assert (gh[i, :15, :15] == 0).all() and (g[i, :15, :15] == 0).all(), i
    # envs done at entry: 0 everywhere, for every producer
    env = make_env(4, batch_cfg(names), auto_reset=False, seed=8)
    env.reset()
    table = lc._to_dev(env, random_table(env, 12))
    ent_call(env, table)
    assert np_(env.done).all()
    lp, h, g, gh = ent_call(env, table)
    assert (bits(h) == 0).all() and (bits(lp) == 0).all() and (gh[:, :15, :15] == 0).all()
    out = env.sample_episodes(table, 3, entropy=True)
    assert (bits(np_(out["entropy"])) == 0).all() and (np_(out["makespan"]) == -1).all()
    order = torch.zeros((4, 2, env.jobs, env.machines), dtype=torch.int32, device=env.device)
    lp_o, ms_o, h_o = env.order_log_prob(table, order, entropy=True)
    assert (bits(np_(h_o)) == 0).all() and (bits(np_(lp_o)) == 0).all()


def sample_twins(make_env, env, table, k, step_index):
    """What sample_episodes(table, k, entropy=True) at counter step_index must give, sample by sample: a twin batch
    with env's state imported runs rollout_priority_sample_entropy once at counter step_index + s*B.  Returns
    makespan, log_prob, entropy (N, k) and the float64 gradients G, G_H (k, N, J, M), zero where the twins' are NaN."""
    n, J, M = env.num_envs, env.jobs, env.machines
    cfg = {"instance_paths": [env.instances[i] for i in range(len(env.instances))],
           "env_to_instance": list(env.env_to_instance)}
    twin = make_env(n, cfg, auto_reset=False, env_id_base=env.env_id_base, seed=env.seed)
    snap = snapshot(env)
    done0 = np_(env.done).copy()
    dev = lc._to_dev(twin, table)
    ms = np.full((n, k), -1, np.int64)
    lp, h = np.zeros((n, k), np.float32), np.zeros((n, k), np.float32)
    g, gh = np.zeros((k, n, J, M)), np.zeros((k, n, J, M))
    for s in range(k):
        twin.reset()
        twin.import_state(snap)
        twin._step_index = step_index + s * bound(env)
        lp[:, s], h[:, s], gs, ghs = ent_call(twin, dev)
        done, t = np_(twin.done), np_(twin.current_time_step)
        ms[done & ~done0, s] = t[done & ~done0]
        g[s], gh[s] = np.nan_to_num(gs.astype(np.float64)), np.nan_to_num(ghs.astype(np.float64))
    twin.close()
    return ms, lp, h, g, gh


@native_test()
def entropy_sample_episodes(make_env, backend):
    """Column s of sample_episodes(entropy=True) equals a twin's rollout_priority_sample(entropy=True) at counter
    step_index + s*B, bit for bit; makespan and log_prob equal the call without entropy; the outputs do not depend on
    the split, on env_id_base or on sharding; the envs are untouched."""
    from tests.lookahead_suite import _outputs
    names = (["ta01", SMALL, *EMU_CLASSES[:1], NONPERM, TINY] if backend == "emu" else
             ["ta01", "ta21", "ta41", "ta80", NONPERM, BIG_GPU, SMALL, TINY] * 2)
    k = 3 if backend == "emu" else 6
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=4, env_id_base=3)
    env.reset()
    random_walk(env, 25)
    table = random_table(env, 9)
    dev = lc._to_dev(env, table)
    before, stats = _outputs(env), env.stats()
    si = env._step_index
    out = env.sample_episodes(dev, k, entropy=True)
    assert env._step_index == si + k * bound(env)
    env._step_index = si
    plain = env.sample_episodes(dev, k)
    for key in ("makespan", "log_prob", "best"):
        a, b = np_(out[key]), np_(plain[key])
        assert np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                              b.view(np.uint32) if b.dtype == np.float32 else b), key
    after = _outputs(env)
    for key, v in before.items():
        assert np.array_equal(v, after[key]), key
    assert env.stats() == stats
    ms, lp, h, _, _ = sample_twins(make_env, env, table, k, si)
    assert np.array_equal(np_(out["makespan"]).astype(np.int64), ms)
    assert np.array_equal(bits(np_(out["log_prob"])), bits(lp))
    assert np.array_equal(bits(np_(out["entropy"])), bits(h))
    # split: one small batch (several work items per tile) against the rows of a large one (one per tile)
    n_big = {"emu": 24, "gpu": 4096}[backend]
    big = make_env(n_big, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    big.reset()
    random_walk(big, 30)
    small = make_env(3, {"instance_path": "ta01"}, auto_reset=False, seed=12)
    small.reset()
    small.import_state({key: v[:3] for key, v in snapshot(big).items()})
    t_big = random_table(big, 13)
    ob = big.sample_episodes(lc._to_dev(big, t_big), 5, entropy=True)
    small._step_index = big._step_index - 5 * bound(big)
    os_ = small.sample_episodes(lc._to_dev(small, t_big[:3]), 5, entropy=True)
    assert np.array_equal(bits(np_(ob["entropy"])[:3]), bits(np_(os_["entropy"])))
    # shards with env_id_base != 0
    n_total = {"emu": 8, "gpu": 96}[backend]
    e2i = np.arange(n_total) % 2
    inst = ["ta01", SMALL] if backend == "emu" else ["ta01", "ta80"]
    whole = make_env(n_total, {"instance_paths": inst, "env_to_instance": e2i}, seed=31, auto_reset=False)
    whole.reset()
    tw = random_table(whole, 14)
    ow = whole.sample_episodes(lc._to_dev(whole, tw), 3, entropy=True)
    for lo, hi in ((0, 5), (5, n_total)):
        s = make_env(hi - lo, {"instance_paths": inst, "env_to_instance": e2i[lo:hi]}, seed=31, auto_reset=False,
                     env_id_base=lo)
        s.reset()
        o = s.sample_episodes(lc._to_dev(s, tw[lo:hi, :s.jobs, :s.machines]), 3, entropy=True)
        assert np.array_equal(bits(np_(o["entropy"])), bits(np_(ow["entropy"])[lo:hi])), lo


@native_test()
def entropy_backward(make_env, backend):
    """(w log_prob + v entropy).sum().backward() against the float64 sum of the twins' gradients for (N, J, M),
    (N, J, 1), (1, J, M) and float64 tables, at split 1 and above; a loss on the entropy alone and on log_prob alone;
    with v = 0 the replay adds what the replay without entropy adds, bit for bit; the same for order_log_prob."""
    import torch
    names = {"emu": ["ta01", SMALL, "ta01", TINY], "gpu": ["ta01", "ta21", "ta41", "ta80", SMALL] * 4}[backend]
    k = 4
    ref = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False)
    n, J, M, dev = ref.num_envs, ref.jobs, ref.machines, ref.device
    rng = np.random.default_rng(17)
    w = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).to(dev)
    v = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).to(dev)
    for shape, dtype in (((n, J, M), torch.float32), ((n, J, 1), torch.float32), ((1, J, M), torch.float32),
                         ((n, J, M), torch.float64)):
        env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=3)
        env.reset()
        random_walk(env, 20)
        base = torch.from_numpy(rng.standard_normal(shape)).to(dev, dtype)
        table = base.to(torch.float32).expand(n, J, M).cpu().numpy()
        si = env._step_index
        _, _, _, g, gh = sample_twins(make_env, env, table, k, si)
        for wl, vl in ((w, v), (None, v), (w, None)):
            x = base.clone().requires_grad_(True)
            env._step_index = si
            out = env.sample_episodes(x, k, entropy=True)
            assert out["entropy"].grad_fn is not None and out["makespan"].grad_fn is None
            loss = 0
            if wl is not None:
                loss = loss + (wl * out["log_prob"]).sum()
            if vl is not None:
                loss = loss + (vl * out["entropy"]).sum()
            loss.backward()
            ww = np_(wl).astype(np.float64) if wl is not None else np.zeros((n, k))
            vv = np_(vl).astype(np.float64) if vl is not None else np.zeros((n, k))
            want = np.einsum("ns,snjm->njm", ww, g) + np.einsum("ns,snjm->njm", vv, gh)
            scale = (np.einsum("ns,snjm->njm", np.abs(ww), 1 + np.abs(g)) +
                     np.einsum("ns,snjm->njm", np.abs(vv), 1 + np.abs(gh)))
            want = torch.from_numpy(want).sum_to_size(shape).numpy()
            scale = torch.from_numpy(scale).sum_to_size(shape).numpy()
            assert x.grad.dtype == dtype and x.grad.shape == shape
            assert (np.abs(np_(x.grad).astype(np.float64) - want) <= 1e-5 * scale).all(), (shape, wl is None)
    # splits, and v = 0 against the plain replay, bit for bit
    env = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=5)
    env.reset()
    random_walk(env, 15)
    dev_t = lc._to_dev(env, random_table(env, 21))
    si = env._step_index
    env.sample_episodes(dev_t, k, entropy=True)
    zero = torch.zeros_like(v)
    for split in (1, 3):
        a = np_(env._sample_episodes_grad(dev_t, k, si, w, split, zero))
        b = np_(env._sample_episodes_grad(dev_t, k, si, w, split))
        assert np.array_equal(a, b), split
        c = np_(env._sample_episodes_grad(dev_t, k, si, w, split, v)).sum(0)
        d = np_(env._sample_episodes_grad(dev_t, k, si, w, 1, v)).sum(0)
        assert np.allclose(c, d, rtol=1e-5, atol=1e-5), split
    order = env.sample_without_replacement(dev_t, 3, order=True)["order"]
    for split in (1, 2):
        a = np_(env._order_log_prob_grad(dev_t, order, w[:, :3], split, zero[:, :3]))
        b = np_(env._order_log_prob_grad(dev_t, order, w[:, :3], split))
        assert np.array_equal(a, b), split
    # order_log_prob: the entropy's gradient against the float64 restatement of the replayed orders
    x = dev_t.clone().requires_grad_(True)
    lp_o, ms_o, h_o = env.order_log_prob(x, order, entropy=True)
    (v[:, :3] * h_o).sum().backward()
    got = np_(x.grad).astype(np.float64)
    want = np.zeros_like(got)
    for s in range(3):
        tw = make_env(n, batch_cfg(names, sort=False), auto_reset=False, seed=5)
        tw.reset()
        tw.import_state(snapshot(env))
        twin = EntTwin(tw, np_(dev_t), driver=-np_(order[:, s]).astype(np.float32))
        twin.steps(bound(env), 0)
        wh, _ = twin.grads()
        want += np_(v)[:, s, None, None].astype(np.float64) * wh
        assert_entropy(np_(h_o.detach())[:, s], twin, ("order", s))
    assert np.allclose(got, want, rtol=1e-4, atol=1e-4), np.abs(got - want).max()


def episode_orders(twin, env):
    """The round order (beam_search's format) of each env's episode the twin took: the decision index at which each
    operation was drawn, -1 for operations not drawn."""
    n, J, M = env.num_envs, env.jobs, env.machines
    order = np.full((n, J, M), -1, np.int32)
    for i, acts in enumerate(twin.actions):
        nxt = np.zeros(J, np.int64)
        for t, a in enumerate(acts):
            if a < J and a < int(env.env_jobs[i]):
                order[i, a, nxt[a]] = t
                nxt[a] += 1
    return order


@native_test()
def entropy_cross_source(make_env, backend):
    """The round order of an episode drawn by rollout_priority_sample(entropy=True), replayed by order_log_prob(
    entropy=True), reports that episode's entropy and log_prob bit for bit; beam_search's best order's entropy
    against the float64 restatement of its replay."""
    names = (["ta01", SMALL, NONPERM, TINY, *EMU_CLASSES[:1]] if backend == "emu" else
             ["ta01", "ta21", "ta41", "ta80", NONPERM, SMALL] * 4)
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, seed=9)
    table = random_table(a_env, 33)
    dev = lc._to_dev(a_env, table)
    lp, h, _, _ = ent_call(a_env, dev)
    twin = EntTwin(b_env, table)
    twin.steps(bound(a_env), 0)
    order = episode_orders(twin, a_env)
    c_env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=9)
    c_env.reset()
    lp_o, ms_o, h_o = c_env.order_log_prob(dev, lc._to_dev(c_env, order), entropy=True)
    assert np.array_equal(bits(np_(lp_o)), bits(lp)) and np.array_equal(bits(np_(h_o)), bits(h))
    assert np.array_equal(np_(ms_o), np_(a_env.current_time_step))
    best = c_env.beam_search(dev, 4, order=True)
    bo = best["order"]
    lp_b, ms_b, h_b = c_env.order_log_prob(dev, bo, entropy=True)
    lp_p, ms_p = c_env.order_log_prob(dev, bo)
    assert np.array_equal(bits(np_(lp_b)), bits(np_(lp_p))) and np.array_equal(np_(ms_b), np_(ms_p))
    d_env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=9)
    d_env.reset()
    rep = EntTwin(d_env, table, driver=-np_(bo).astype(np.float32))
    rep.steps(bound(a_env), 0)
    assert_entropy(np_(h_b), rep, "beam")


@native_test()
def entropy_abi(make_env, backend):
    """The five entry points: JSS_ERR_INVALID for NULL or misaligned pointers, a negative stride, k < 1, ld < k and a
    split outside 1..k, with their own names in the error text; JSS_ERR_STATE before jss_assign."""
    import torch
    env = make_env(2, {"instance_path": "ta01"}, seed=13)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    L, h, st = env._L, env._h, env._stream()
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    i32 = torch.zeros(n * 8, dtype=torch.int32, device=env.device)
    f32 = torch.zeros(n * 8, dtype=torch.float32, device=env.device)
    g = torch.zeros(8 * n * J * M, dtype=torch.float32, device=env.device)
    order = torch.zeros((n, 4, J, M), dtype=torch.int32, device=env.device)
    p, o, q, r, od = t.data_ptr(), i32.data_ptr(), f32.data_ptr(), g.data_ptr(), order.data_ptr()
    s = (J * M, M, 1)

    def refused(fn, name, *args):
        assert getattr(L, fn)(h, *args) == -1, (fn, args)
        assert L.jss_last_error(h).startswith(name.encode() + b":"), (fn, L.jss_last_error(h))

    fn = "jss_rollout_priority_sample_entropy"
    for args in ((None, *s, 0, 0, 5, q, q, r, r), (p + 2, *s, 0, 0, 5, q, q, r, r), (p, -1, M, 1, 0, 0, 5, q, q, r, r),
                 (p, *s, 0, 0, -1, q, q, r, r), (p, *s, 0, 0, 5, None, q, r, r), (p, *s, 0, 0, 5, q, None, r, r),
                 (p, *s, 0, 0, 5, q, q + 2, r, r), (p, *s, 0, 0, 5, q, q, r + 2, r), (p, *s, 0, 0, 5, q, q, r, r + 2)):
        refused(fn, fn, *args, st)
    assert L.jss_rollout_priority_sample_entropy(h, p, *s, 0, 0, 0, q, q, None, None, st) == 0
    fn = "jss_sample_episodes_entropy"
    for args in ((None, *s, 0, 0, 4, o, q, q, 4), (p, *s, 0, 0, 0, o, q, q, 4), (p, *s, 0, 0, 4, o, q, q, 3),
                 (p, *s, 0, 0, 4, None, q, q, 4), (p, *s, 0, 0, 4, o, q + 2, q, 4), (p, *s, 0, 0, 4, o, q, None, 4),
                 (p, *s, 0, 0, 4, o, q, q + 2, 4), (p, J * M, -M, 1, 0, 0, 4, o, q, q, 4)):
        refused(fn, fn, *args, st)
    fn = "jss_sample_episodes_entropy_grad"
    for args in ((None, *s, 0, 0, 4, q, q, 4, 1, r), (p, *s, 0, 0, 0, q, q, 4, 1, r), (p, *s, 0, 0, 4, q, q, 3, 1, r),
                 (p, *s, 0, 0, 4, None, q, 4, 1, r), (p, *s, 0, 0, 4, q, None, 4, 1, r),
                 (p, *s, 0, 0, 4, q, q + 2, 4, 1, r), (p, *s, 0, 0, 4, q, q, 4, 0, r), (p, *s, 0, 0, 4, q, q, 4, 5, r),
                 (p, *s, 0, 0, 4, q, q, 4, 1, None), (p, *s, 0, 0, 4, q, q, 4, 1, r + 2)):
        refused(fn, fn, *args, st)
    fn = "jss_order_log_prob_entropy"
    for args in ((None, *s, od, 4, o, q, q, 4), (p, *s, None, 4, o, q, q, 4), (p, *s, od + 2, 4, o, q, q, 4),
                 (p, *s, od, 0, o, q, q, 4), (p, *s, od, 4, o, q, q, 3), (p, *s, od, 4, None, q, q, 4),
                 (p, *s, od, 4, o, None, q, 4), (p, *s, od, 4, o, q, None, 4), (p, *s, od, 4, o, q, q + 2, 4)):
        refused(fn, fn, *args, st)
    fn = "jss_order_log_prob_entropy_grad"
    for args in ((None, *s, od, 4, q, q, 4, 1, r), (p, *s, None, 4, q, q, 4, 1, r), (p, *s, od, 0, q, q, 4, 1, r),
                 (p, *s, od, 4, q, q, 3, 1, r), (p, *s, od, 4, None, q, 4, 1, r), (p, *s, od, 4, q, None, 4, 1, r),
                 (p, *s, od, 4, q, q + 2, 4, 1, r), (p, *s, od, 4, q, q, 4, 0, r), (p, *s, od, 4, q, q, 4, 5, r),
                 (p, *s, od, 4, q, q, 4, 1, None), (p, *s, od, 4, q, q, 4, 1, r + 2)):
        refused(fn, fn, *args, st)
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_rollout_priority_sample_entropy(raw, p, *s, 0, 0, 5, q, q, r, r, st) == -5
    assert L.jss_sample_episodes_entropy(raw, p, *s, 0, 0, 4, o, q, q, 4, st) == -5
    assert L.jss_sample_episodes_entropy_grad(raw, p, *s, 0, 0, 4, q, q, 4, 1, r, st) == -5
    assert L.jss_order_log_prob_entropy(raw, p, *s, od, 4, o, q, q, 4, st) == -5
    assert L.jss_order_log_prob_entropy_grad(raw, p, *s, od, 4, q, q, 4, 1, r, st) == -5
    L.jss_destroy(raw)


@native_test(emu=None)
def entropy_full_size_ta80(make_env):
    """ta80 at N = 65 536, a seeded torch.randn table, one call with both gradients: no error bits, every entropy
    finite and positive, log_prob and state bit for bit the call without entropy; five envs' entropy and gradient rows
    against the float64 restatement of one-env step_logits twins."""
    import torch
    n = 65536
    a_env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=5)
    c_env = make_env(n, {"instance_path": "ta80"}, auto_reset=False, seed=5)
    a_env.reset(); c_env.reset()
    J, M = a_env.jobs, a_env.machines
    table = torch.randn((n, J, M), generator=torch.Generator(device=a_env.device).manual_seed(21), device=a_env.device)
    lp, h, g, gh = ent_call(a_env, table)
    lp_c, g_c = plain_call(c_env, table)
    assert np_(a_env.done).all() and not (np_(a_env.flags) & N.FLAG_ERROR).any()
    assert np.isfinite(h).all() and (h > 0).all()
    assert np.array_equal(bits(lp), bits(lp_c)) and np.array_equal(g, g_c)
    assert_twins_equal(a_env, c_env, "ta80", state=True, stats=True)
    for i in (0, 1, 4097, 33333, 65535):
        one = make_env(1, {"instance_path": "ta80"}, auto_reset=False, seed=5, env_id_base=i)
        one.reset()
        twin = EntTwin(one, table[i:i + 1].cpu().numpy())
        twin.steps(2 * J * M + 1, 0)
        assert np_(one.done).all()
        assert_entropy(h[i:i + 1], twin, i)
        wh, wl = twin.grads()
        tol = 2e-5 * (1 + twin.count[0]) + 1e-5 * np.abs(wh[0])
        assert (np.abs(gh[i] - wh[0]) <= tol).all(), (i, np.abs(gh[i] - wh[0]).max())
        assert (np.abs(g[i] - wl[0]) <= 2e-5 * (1 + twin.count[0])).all(), i
        one.close()
