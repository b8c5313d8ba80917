"""The tests of jss_rollout_priority_sample (whole episodes drawn from a caller's logit table in one launch, with each
episode's log-probability and its gradient with respect to the table), declared once for both backends
(tests/backends.py) and collected by tests/test_emu_priority_sample.py and tests/test_gpu_priority_sample.py.  The
call is checked against a twin env stepped with jss_step_logits on the rows the table gives at each decision (the
entry of every job's current operation, the no-op at -inf), the gradient against its float64 restatement from the
twin's decisions, and, at full size, against the CPU oracle's replay of the twin's actions."""
import ctypes

import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import assert_twins_equal, batch_cfg, np_, twin_envs
from tests.priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, assert_same, greedy_rows, random_table, synthetic_instance


class Twin:
    """Steps a twin env with step_logits on the gathered rows of a table and keeps what a sampled call over the same
    decisions must report: each env's log_prob (the twin's per-step log_probs summed in fp32 in step order), the float64
    gradient of it with respect to the table, the number of decisions each entry took part in, and the actions.  `call`
    holds these over the steps since the last start(), `all` over every step."""

    def __init__(self, env):
        self.env = env
        self.all = self._zero()
        self.call = self._zero()
        self.actions = [[] for _ in range(env.num_envs)]

    def _zero(self):
        n, J, M = self.env.num_envs, self.env.jobs, self.env.machines
        return {"log_prob": np.zeros(n, np.float32), "grad": np.zeros((n, J, M)), "count": np.zeros((n, J, M), np.int64)}

    def start(self):
        self.call = self._zero()

    def steps(self, table, k, step_index, check=None):
        """Up to k twin steps from RNG counter step_index (fewer once every env is done); `check(rows, mask, done,
        actions, log_prob, counter)`, if given, sees each step's draw."""
        env = self.env
        J = env.jobs
        env._step_index = step_index
        for t in range(k):
            if np_(env.done).all():
                return
            rows = greedy_rows(env, table)
            todo = np_(env.export_state()["todo"]).copy()
            mask = np_(env.action_mask).copy()
            legal = mask[:, :J]
            done = np_(env.done).copy()
            _, _, _, _, info = env.step_logits(lc._to_dev(env, rows))
            acts, lp = np_(info["actions"]), np_(info["log_prob"])
            if check is not None:
                check(rows, mask, done, acts, lp, step_index + t)
            for d in (self.all, self.call):
                d["log_prob"] = (d["log_prob"] + lp).astype(np.float32)
            for i in np.flatnonzero(~done):
                self.actions[i].append(int(acts[i]))
                js = np.flatnonzero(legal[i])
                x = rows[i, js].astype(np.float64)
                if not len(js) or np.isnan(x).any() or not np.isfinite(x.max()):
                    continue                              # the no-op, or a bad row (the env errs, its gradient is 0)
                p = np.exp(x - x.max())
                p /= p.sum()
                for d in (self.all, self.call):
                    d["grad"][i, js, todo[i, js]] += (js == acts[i]) - p
                    d["count"][i, js, todo[i, js]] += 1


def sample_call(env, table, n_steps=None, grad=True):
    """rollout_priority_sample's native call on a (materialised or strided) device table: returns log_prob and the
    gradient buffer, pre-filled with NaN so that entries the call must not write stay NaN (None without grad)."""
    import torch
    n, J, M = env.num_envs, env.jobs, env.machines
    g = torch.full((n, J, M), float("nan"), device=env.device) if grad else None
    lp = env._rollout_priority_sample(table, 2 * J * M + 1 if n_steps is None else n_steps, g)
    return np_(lp).copy(), (np_(g).copy() if grad else None)


def assert_log_prob(got, want, ctx):
    """Bit for bit, NaN where the twin has NaN."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (ctx, got, want)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32)), (ctx, got, want)


def assert_grad(env, got, want, ctx, err=None):
    """The kernel's gradient rows against the twin's float64 restatement `want` (Twin.call or Twin.all) within
    1e-5 (1 + decisions the entry took part in), zero rows for the envs that erred in the call, and the entries past
    J_i / M_i untouched (NaN)."""
    for i, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        g, w = got[i, :Ji, :Mi], want["grad"][i, :Ji, :Mi]
        if err is not None and err[i]:
            assert (g == 0).all(), (ctx, i)
        else:
            assert (np.abs(g - w) <= 1e-5 * (1 + want["count"][i, :Ji, :Mi])).all(), (ctx, i, np.abs(g - w).max())
        assert np.isnan(got[i, Ji:]).all() and np.isnan(got[i, :, Mi:]).all(), (ctx, i, "padding written")


def check_twin(make_env, names, seed, k, ties=False):
    """rollout_priority_sample(P, k), then to the end, equals as many twin steps of step_logits from the same counter,
    log_prob bit for bit and the gradient within tolerance (zero for operations drawn before the second call and for
    envs done at its start); a third env run to the end in one call ends where the twin ends."""
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    table = random_table(a_env, seed, ties)
    dev = lc._to_dev(a_env, table)
    twin = Twin(b_env)
    lp, g = sample_call(a_env, dev, k)
    twin.steps(table, k, 0)
    assert a_env._step_index == k
    assert_same(a_env, b_env, ("partial", k))
    assert_log_prob(lp, twin.call["log_prob"], ("partial", k))
    assert_grad(a_env, g, twin.call, ("partial", k))
    twin.start()
    lp, g = sample_call(a_env, dev)
    twin.steps(table, 2 * a_env.jobs * a_env.machines + 1, k)
    assert np_(b_env.done).all()
    assert_same(a_env, b_env, "second call")
    assert_log_prob(lp, twin.call["log_prob"], "second call")
    assert_grad(a_env, g, twin.call, "second call")
    c_env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    c_env.reset()
    lp, g = sample_call(c_env, dev)
    assert_same(c_env, b_env, "one call")
    assert not (np_(c_env.flags) & N.FLAG_ERROR).any()
    assert_log_prob(lp, twin.all["log_prob"], "one call")
    assert_grad(c_env, g, twin.all, "one call")


@native_test(emu=[False, True], gpu=[False, True])
def priority_sample_twin_mixed_batch(make_env, backend, ties):
    # every lane class of the generic kernel, 129..256 jobs and a non-permutation instance included
    if backend == "emu":
        check_twin(make_env, ["ta01", "ta01", *EMU_CLASSES, NONPERM], seed=1, k=40, ties=ties)
    else:
        check_twin(make_env, ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80", NONPERM,
                              BIG_GPU] * 3, seed=1, k=300, ties=ties)


@native_test()
def priority_sample_twin_uniform(make_env, backend):
    """Uniform tiny (J <= 4), ta01 and ta80 batches."""
    n = {"emu": 3, "gpu": 64}[backend]
    for J, M in ((2, 2), (3, 4), (4, 3), (1, 2)):
        check_twin(make_env, [synthetic_instance(J, M, J * 10 + M)] * n, seed=J + M, k=2, ties=True)
    check_twin(make_env, ["ta01"] * n, seed=2, k=60)
    if backend == "gpu":
        check_twin(make_env, ["ta80"] * n, seed=3, k=700)


@native_test()
def priority_sample_autograd(make_env, backend):
    """log_prob.backward(w) gives the kernel's gradient weighted by w, summed over the broadcast dimensions, for
    (N, J, M), (N, J, 1), (1, J, M) and a float64 table (gradient in float64); without requires_grad log_prob has no
    grad_fn; a call without a gradient buffer leaves what a call with one leaves."""
    import torch
    names = {"emu": ["ta01", "ta21", "ta01"], "gpu": ["ta01", "ta21", "ta41", "ta80"] * 8}[backend]
    ref = make_env(len(names), batch_cfg(names, sort=False))
    n, J, M, dev = ref.num_envs, ref.jobs, ref.machines, ref.device
    rng = np.random.default_rng(17)
    w = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(dev)
    for shape, dtype in (((n, J, M), torch.float32), ((n, J, 1), torch.float32), ((1, J, M), torch.float32),
                         ((n, J, M), torch.float64)):
        base = torch.from_numpy(rng.standard_normal(shape)).to(dev, dtype)
        a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False)
        x = base.clone().requires_grad_(True)
        _, _, _, _, info = a_env.rollout_priority_sample(x)
        assert info["log_prob"].grad_fn is not None and info["log_prob"].dtype == torch.float32
        info["log_prob"].backward(w)
        lp, g = sample_call(b_env, base.to(torch.float32).expand(n, J, M).contiguous())
        assert_twins_equal(a_env, b_env, shape, state=True, stats=True)
        assert np.array_equal(np_(info["log_prob"].detach()).view(np.uint32), lp.view(np.uint32)), shape
        g = torch.from_numpy(np.nan_to_num(g, nan=0.0)).to(dev)
        want = (w[:, None, None] * g).sum_to_size(shape).to(dtype)
        assert x.grad.dtype == dtype and x.grad.shape == shape
        assert torch.allclose(x.grad, want, rtol=1e-6, atol=1e-6), shape
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False)
    table = lc._to_dev(a_env, random_table(a_env, 18))
    _, _, _, _, info = a_env.rollout_priority_sample(table)
    assert info["log_prob"].grad_fn is None
    with torch.no_grad():
        _, _, _, _, info2 = b_env.rollout_priority_sample(table.clone().requires_grad_(True))
    assert info2["log_prob"].grad_fn is None
    assert_twins_equal(a_env, b_env, "no grad", state=True, stats=True)
    assert np.array_equal(np_(info["log_prob"]).view(np.uint32), np_(info2["log_prob"]).view(np.uint32))
    # through the C ABI: grad_out NULL against a buffer
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False)
    lp_a, _ = sample_call(a_env, table, 37, grad=False)
    lp_b, _ = sample_call(b_env, table, 37, grad=True)
    assert_twins_equal(a_env, b_env, "NULL grad_out", state=True, stats=True)
    assert np.array_equal(lp_a.view(np.uint32), lp_b.view(np.uint32))


@native_test()
def priority_sample_broadcasts(make_env, backend):
    """(N, J, 1), (1, J, M) and padded strides (ld_job > M, ld_env > J * ld_job, NaN in the padding) give what the
    materialised (N, J, M) table gives: state, log_prob and gradient."""
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
        lp_a, g_a = sample_call(a_env, given)
        lp_b, g_b = sample_call(b_env, materialised.contiguous())
        assert np_(a_env.done).all()
        assert_same(a_env, b_env, tuple(given.shape))
        assert np.array_equal(lp_a.view(np.uint32), lp_b.view(np.uint32)), tuple(given.shape)
        assert np.array_equal(g_a, g_b, equal_nan=True), tuple(given.shape)


@native_test()
def priority_sample_bad_tables(make_env):
    """NaN / +inf on a legal current operation, or every legal job at -inf, set the error bit and stop the env where
    the step_logits twin leaves it, at the first decision or mid-episode, with log_prob NaN and zero gradient rows; NaN
    and inf on entries that are never read change nothing."""
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
    lp, g = sample_call(a_env, lc._to_dev(a_env, t))
    twin = Twin(b_env)
    twin.steps(t, 2 * J * a_env.machines + 1, 0)
    assert_same(a_env, b_env, "bad")
    err = (np_(a_env.flags) & N.FLAG_ERROR) != 0
    assert err[:5].all() and not err[5:].any(), err
    assert np.isnan(lp[:5]).all() and not np.isnan(lp[5:]).any(), lp
    assert_log_prob(lp, twin.call["log_prob"], "bad")
    assert_grad(a_env, g, twin.call, "bad", err)
    assert (np_(a_env.current_time_step)[:3] == 0).all() and int(a_env.current_time_step[3]) > 0
    ref = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, record_solution=True)
    ref.reset()
    lp_ref, g_ref = sample_call(ref, lc._to_dev(ref, clean))
    for i in (5, 6, 7):
        for k in ("last_makespan", "last_return", "solution"):
            assert np.array_equal(np_(getattr(a_env, k))[i], np_(getattr(ref, k))[i]), (i, k)
        assert lp[i] == lp_ref[i] and np.array_equal(g[i], g_ref[i], equal_nan=True), i
    # illegal jobs and finished operations: poisoned after a partial call, between calls
    a_env, b_env = twin_envs(make_env, ["ta01"] * 4, sort=False, auto_reset=False, record_solution=True)
    table = random_table(a_env, 12)
    for env in (a_env, b_env):
        sample_call(env, lc._to_dev(env, table), 30)
    x = b_env.export_state()
    todo, legal = np_(x["todo"]), np_(x["legal"]).astype(bool)
    poisoned = table.copy()
    ops = np.arange(a_env.machines)
    poisoned[ops[None, None, :] < todo[:, :, None]] = np.nan                 # finished operations
    for i, j in zip(*np.nonzero(~legal & (todo < a_env.machines))):
        poisoned[i, j, todo[i, j]] = np.inf if (i + j) % 2 else np.nan       # illegal jobs' current operations
    lp_a, g_a = sample_call(a_env, lc._to_dev(a_env, poisoned), 1)
    lp_b, g_b = sample_call(b_env, lc._to_dev(b_env, table), 1)
    assert_same(a_env, b_env, "illegal")
    assert np.array_equal(lp_a, lp_b) and np.array_equal(g_a, g_b, equal_nan=True)
    poisoned = table.copy()
    todo = np_(b_env.export_state()["todo"])
    poisoned[ops[None, None, :] < todo[:, :, None]] = np.nan
    lp_a, g_a = sample_call(a_env, lc._to_dev(a_env, poisoned))
    lp_b, g_b = sample_call(b_env, lc._to_dev(b_env, table))
    assert_same(a_env, b_env, "finished")
    assert np.array_equal(lp_a, lp_b) and np.array_equal(g_a, g_b, equal_nan=True)
    assert not (np_(a_env.flags) & N.FLAG_ERROR).any()


@native_test()
def priority_sample_done_and_auto_reset(make_env):
    """Under auto-reset: an env that finishes stops there with episode_count + 1 once; a done env is untouched by the
    next call, with log_prob 0 and zero gradient rows; the RNG counter advances by n_steps per call."""
    names = ["ta01", "ta01", "ta31", "ta01"]
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=True, record_solution=True)
    env.reset()
    table = lc._to_dev(env, random_table(env, 9))
    sample_call(env, table, 100)
    assert env._step_index == 100
    sample_call(env, table)
    assert env._step_index == 100 + 2 * env.jobs * env.machines + 1
    assert np_(env.done).all() and (np_(env.episode_count) == 1).all()
    before = {k: np_(v).copy() for k, v in env.export_state().items()}
    obs = np_(env.real_obs).copy()
    c = env.launch_count
    lp, g = sample_call(env, table)                       # every env done at entry
    assert env.launch_count == c + 1                      # one lane class
    assert (lp == 0).all() and not np.signbit(lp).any()
    for i, (Ji, Mi) in enumerate(zip(env.env_jobs, env.env_machines)):
        assert (g[i, :Ji, :Mi] == 0).all(), i
    assert (np_(env.episode_count) == 1).all() and np.array_equal(np_(env.real_obs), obs)
    for k, v in env.export_state().items():
        assert np.array_equal(np_(v), before[k]), k


@native_test()
def priority_sample_abi(make_env):
    """JSS_ERR_INVALID for a NULL or misaligned table or log_prob_out, a misaligned grad_out, a negative stride or
    n_steps < 0, JSS_ERR_STATE before jss_assign; n_steps = 0 does nothing; one launch per lane class present; a wrong
    rank or shape raises ValueError before the native call and leaves the counter; a call after a recording step first
    refreshes real_obs."""
    import pytest
    import torch
    names = ["ta01", "ta51", "ta80", "ta01"]             # lane classes 1, 2 and 4 jobs per lane
    env = make_env(len(names), batch_cfg(names, sort=False), seed=3)
    env.reset()
    n, J, M = env.num_envs, env.jobs, env.machines
    t = torch.zeros((n, J, M), dtype=torch.float32, device=env.device)
    lp = torch.zeros(n + 1, dtype=torch.float32, device=env.device)
    g = torch.zeros(n * J * M + 1, dtype=torch.float32, device=env.device)
    L, h, st = env._L, env._h, env._stream()
    p, s, q, r = t.data_ptr(), (J * M, M, 1), lp.data_ptr(), g.data_ptr()
    for args in ((None, *s, 5, q, r), (p + 2, *s, 5, q, r), (p, -1, M, 1, 5, q, r), (p, J * M, -M, 1, 5, q, r),
                 (p, J * M, M, -1, 5, q, r), (p, *s, -1, q, r), (p, *s, 5, None, r), (p, *s, 5, q + 2, r),
                 (p, *s, 5, q, r + 2)):
        assert L.jss_rollout_priority_sample(h, *args[:4], 0, 0, *args[4:], st) == -1, args
        assert L.jss_last_error(h).startswith(b"jss_rollout_priority_sample:"), args
    raw = ctypes.c_void_p()
    assert L.jss_create(ctypes.byref(raw), 0, 2, 0, 0) == 0
    assert L.jss_rollout_priority_sample(raw, p, *s, 0, 0, 5, q, r, st) == -5
    L.jss_destroy(raw)
    before = {k: np_(getattr(env, k)).copy() for k in ("real_obs", "action_mask", "reward_raw", "current_time_step")}
    c = env.launch_count
    assert L.jss_rollout_priority_sample(h, p, *s, 0, 0, 0, q, r, st) == 0
    assert L.jss_rollout_priority_sample(h, p, *s, 0, 0, 0, q, None, st) == 0
    assert env.launch_count == c
    for k, v in before.items():
        assert np.array_equal(np_(getattr(env, k)), v), k
    step_index = env._step_index
    env.rollout_priority_sample(t, 3)
    assert env.launch_count == c + 3
    assert env._step_index == step_index + 3
    for bad in (t[0], t[None], t[:, :J - 1], torch.zeros((2, J, M), device=env.device), t[:, :, :M - 1]):
        with pytest.raises(ValueError):
            env.rollout_priority_sample(bad)
    assert env._step_index == step_index + 3              # refused before the native call
    # after a recording step, real_obs is brought up to date before the call (env 0's bad table leaves it unchanged,
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
        env_.rollout_priority_sample(table, 5)
    assert_twins_equal(a_env, b_env, "after record", state=True, stats=True)


@native_test()
def priority_sample_shards(make_env, backend):
    """Shards created with env_id_base != 0 reproduce the unsharded batch: state, log_prob bit for bit, gradient."""
    n_total = {"emu": 8, "gpu": 96}[backend]
    names = {"emu": ["ta01", "ta31", "ta01", "ta41"], "gpu": ["ta01", "ta31", "ta51", "ta80"]}[backend]
    e2i = np.arange(n_total) % len(names)
    cuts = [0, 5, n_total]                               # every shard has the batch maxima J and M
    whole = make_env(n_total, {"instance_paths": names, "env_to_instance": e2i}, seed=31, auto_reset=False)
    shards = [make_env(hi - lo, {"instance_paths": names, "env_to_instance": e2i[lo:hi]}, seed=31, auto_reset=False,
                       env_id_base=lo) for lo, hi in zip(cuts[:-1], cuts[1:])]
    whole.reset()
    table = random_table(whole, 14)
    for k in (60, None):
        lp_w, g_w = sample_call(whole, lc._to_dev(whole, table), k)
        for s, lo, hi in zip(shards, cuts[:-1], cuts[1:]):
            if k == 60:
                s.reset()
            lp_s, g_s = sample_call(s, lc._to_dev(s, table[lo:hi, : s.jobs, : s.machines]), k)
            assert np.array_equal(lp_s.view(np.uint32), lp_w[lo:hi].view(np.uint32)), (k, lo)
            assert np.array_equal(g_s, g_w[lo:hi, : s.jobs, : s.machines], equal_nan=True), (k, lo)
            assert_twins_equal(s, whole, k, rows=slice(lo, hi))


@native_test(emu=None)
def priority_sample_first_decision_distribution(make_env):
    """ta01 at N = 65 536 from reset (every job legal, the no-op not), one broadcast (1, J, M) table, one decision: the
    histogram of the drawn jobs against the softmax of the entries of the jobs' first operations, and every log_prob
    against log_softmax."""
    import torch
    from scipy.stats import chisquare
    n = 65536
    env = make_env(n, {"instance_path": "ta01"}, seed=11, auto_reset=False)
    env.reset()
    J, M = env.jobs, env.machines
    table = torch.randn((1, J, M), generator=torch.Generator().manual_seed(0)).to(env.device)
    _, _, _, _, info = env.rollout_priority_sample(table, 1)
    running = np_(env.export_state()["tufco"]) > 0
    assert (running.sum(1) == 1).all()
    acts = running.argmax(1)
    logp = torch.log_softmax(table[0, :, 0].double(), 0).cpu().numpy()
    hist = np.bincount(acts, minlength=J)
    res = chisquare(hist, np.exp(logp) * n)
    assert res.pvalue > 1e-6, (res, hist)
    assert np.abs(np_(info["log_prob"]) - logp[acts]).max() <= 1e-5 * (1 + np.abs(logp).max())


@native_test(emu=None)
def priority_sample_score_function_identity(make_env):
    """E[grad log pi] = 0: with one broadcast (1, J, M) table on ta01 from reset to done, the per-entry mean of the
    gradient over 65 536 episodes is zero within its standard error (chi-square of the z-scores over the entries with
    non-zero variance).  A biased draw or a wrong gradient shows up here."""
    import torch
    from scipy.stats import chi2
    n = 65536
    env = make_env(n, {"instance_path": "ta01"}, seed=12, auto_reset=False)
    env.reset()
    J, M = env.jobs, env.machines
    table = torch.randn((1, J, M), generator=torch.Generator().manual_seed(1)).to(env.device)
    _, g = sample_call(env, table)
    assert np_(env.done).all() and not (np_(env.flags) & N.FLAG_ERROR).any()
    g = g.astype(np.float64)
    mean, sd = g.mean(0), g.std(0, ddof=1)
    live = sd > 0
    z = mean[live] / (sd[live] / np.sqrt(n))
    stat = float((z ** 2).sum())
    assert live.sum() > J * M // 2
    assert chi2.sf(stat, int(live.sum())) > 1e-6, (stat, int(live.sum()))


@native_test(emu=None)
def priority_sample_full_size_ta80(make_env):
    """ta80 at N = 65 536, a seeded torch.randn table, one default call: every env done without the error bit, the raw
    return 2 sum_op - M makespan everywhere, every gradient table summing to 0; five sampled envs equal to one-env
    twins stepped with step_logits from the same counter, and the twins' actions replayed through the oracle give the
    same makespan, return and solution, and the float64 gradient the env's rows."""
    import torch
    from oracle.jss_oracle import OracleEnv
    from jssenv_b200.instances import load_instance
    n_envs = 65536
    env = make_env(n_envs, {"instance_path": "ta80"}, auto_reset=False, record_solution=True, seed=5)
    env.reset()
    J, M = env.jobs, env.machines
    sum_op = int(env.instance_scalars[0][2])
    gen = torch.Generator(device=env.device).manual_seed(21)
    table = torch.randn((n_envs, J, M), generator=gen, device=env.device)
    lp, g = sample_call(env, table)
    assert np_(env.done).all()
    assert not (np_(env.flags) & N.FLAG_ERROR).any() and np.isfinite(lp).all()
    makespan = np_(env.last_makespan).astype(np.int64)
    assert np.array_equal(np_(env.last_return).astype(np.int64), 2 * sum_op - M * makespan)
    # each of the J * M decisions that draw a job adds 1 - sum p = 0
    assert (np.abs(g.astype(np.float64).sum((1, 2))) <= 1e-6 * J * M).all()
    solution = np_(env.solution)
    x = env.export_state()
    for i in (0, 1, 4097, 33333, 65535):
        rows = table[i:i + 1].cpu().numpy()
        twin_env = make_env(1, {"instance_path": "ta80"}, auto_reset=False, record_solution=True, seed=5,
                            env_id_base=i)
        twin_env.reset()
        twin = Twin(twin_env)
        twin.steps(rows, 2 * J * M + 1, 0)
        assert np_(twin_env.done).all()
        assert_twins_equal(twin_env, env, i, rows=slice(i, i + 1))
        for k, v in twin_env.export_state().items():
            assert np.array_equal(np_(v)[0], np_(x[k])[i]), (i, k)
        assert np.array_equal(np_(twin_env.solution)[0], solution[i]), i
        assert_log_prob(lp[i:i + 1], twin.all["log_prob"], i)
        assert (np.abs(g[i] - twin.all["grad"][0]) <= 1e-5 * (1 + twin.all["count"][0])).all(), i
        o = OracleEnv(*load_instance("ta80"))
        o.reset()
        done, ret = False, 0
        for a in twin.actions[0]:
            assert not done
            _, _, done, _, _ = o.step(a)
            ret += o.last_raw_reward
        assert done and o.current_time_step == makespan[i] and ret == int(env.last_return[i])
        assert np.array_equal(np.asarray(o.solution), solution[i]), i
        twin_env.close()
