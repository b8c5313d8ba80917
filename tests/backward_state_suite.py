"""The tests of the replayed gradients across the calls a training loop makes between forward and backward, declared
once for both backends (tests/backends.py) and collected by tests/test_emu_backward_state.py and
tests/test_gpu_backward_state.py.  sample_episodes, order_log_prob and sample_without_replacement replay their episodes
from the envs' state at backward time: after a call that may change that state, or after close(), their backward must
raise before any launch; after a call that leaves the envs untouched it must give, bit for bit, the gradient it gives
with nothing in between, which is held to the float64 references of the producers' own suites.
rollout_priority_sample writes its gradient during forward and must give the same gradient after any call.  Every
public method of JssVecEnv is classified here as changing the envs or not, and the classification is checked."""
import inspect

import numpy as np

from jssenv_b200 import JssVecEnv
from jssenv_b200 import _native as N
from jssenv_b200.beam import ObsBeamSearch
from tests import logits_common as lc
from tests.backends import native_test
from tests.entropy_suite import EntTwin, sample_twins
from tests.lookahead_priority_suite import EMU_CLASSES, NONPERM, SMALL, TINY, noop_only
from tests.lookahead_suite import _outputs, random_walk, snapshot
from tests.parity_common import batch_cfg, np_
from tests.priority_suite import greedy_rows, random_table
from tests.sample_episodes_suite import twin_samples
from tests.swor_suite import decisions, f64_grad

BATCHES = {"emu": {"mixed": (["ta01", SMALL, *EMU_CLASSES, NONPERM, TINY], 90, 2)},
           "gpu": {"mixed": (["ta01", "ta41", *EMU_CLASSES, NONPERM, SMALL, TINY], 30, 4),
                   "ta80": (["ta80"] * 4096, 200, 3)}}


def _skip(env):
    import torch
    return torch.full((env.num_envs,), N.ACTION_SKIP, dtype=torch.int32, device=env.device)


def _host_step(packed=False, dma_fraction=0.0):
    def call(env, c):
        env.host_step_begin(np_(env.policy("RANDOM")), packed=packed, dma_fraction=dma_fraction)
        env.host_wait_obs()
    return call


def _record(what, *extra):
    def call(env, c):
        getattr(env, what)(c.rows, env.logits_trajectory(1), 0, *extra)
    return call


def _mirror_step(env, c):
    env.host["actions"][:] = np_(env.policy("RANDOM"))
    env.step_export_host()


def _beam_step(env, c, stochastic=False):
    import torch
    score = torch.zeros(env.num_envs, dtype=torch.float32, device=env.device)
    if stochastic:
        env.stochastic_beam_step(c.rows, 1, score, score.clone(), 0)
    else:
        env.beam_step(c.rows, 1, score)


# Every call that may change an env's state, as (method, call(env, case)).  The reset that selects no env, the step of
# JSS_ACTION_SKIP everywhere and the import of the state the envs already hold change nothing, and count all the same.
MUTATING = [
    ("reset", lambda env, c: env.reset()),
    ("reset", lambda env, c: env.reset(np.zeros(env.num_envs, bool))),
    ("step", lambda env, c: env.step(env.policy("RANDOM"))),
    ("step", lambda env, c: env.step(_skip(env))),
    ("step_sample", lambda env, c: env.step_sample(env.policy("RANDOM"), "MWR")),
    ("step_logits", lambda env, c: env.step_logits(c.rows)),
    ("step_greedy", lambda env, c: env.step_greedy(c.rows, 0.25)),
    ("step_logits_record", _record("step_logits_record")),
    ("step_greedy_record", _record("step_greedy_record", 0.25)),
    ("rollout", lambda env, c: env.rollout("MWR", 3)),
    ("rollout_record", lambda env, c: env.rollout_record("SPT", 2)),
    ("rollout_priority", lambda env, c: env.rollout_priority(c.table, n_steps=3)),
    ("rollout_priority_sample", lambda env, c: env.rollout_priority_sample(c.table, n_steps=3)),
    ("beam_step", _beam_step),
    ("stochastic_beam_step", lambda env, c: _beam_step(env, c, True)),
    ("import_state", lambda env, c: env.import_state(snapshot(env))),
    ("step_host", lambda env, c: env.step_host(np_(env.policy("RANDOM")))),
    ("host_step_begin", _host_step()),
    ("host_step_begin", _host_step(packed=True)),
    ("host_step_begin", _host_step(packed=True, dma_fraction=0.5)),
    ("step_export_host", _mirror_step),
]

# Every public method that leaves the envs' state alone, as (method, call(env, case)).
UNTOUCHED = [
    ("lookahead", lambda env, c: env.lookahead("MWR")),
    ("lookahead_priority", lambda env, c: env.lookahead_priority(c.table)),
    ("lookahead_sample", lambda env, c: env.lookahead_sample(c.table, 1)),
    ("beam_search", lambda env, c: env.beam_search(c.table, 2, order=True)),
    ("sample_without_replacement", lambda env, c: env.sample_without_replacement(c.table, 2, order=True)),
    ("sample_episodes", lambda env, c: env.sample_episodes(c.table, 2, solution=True, entropy=True)),
    ("order_log_prob", lambda env, c: env.order_log_prob(c.table, c.order, entropy=True)),
    ("improve_orders", lambda env, c: env.improve_orders(c.order[:, 0], max_moves=1)),
    ("policy", lambda env, c: env.policy("RANDOM")),
    ("export_state", lambda env, c: env.export_state()),
    ("refresh_obs", lambda env, c: env.refresh_obs()),
    ("stats", lambda env, c: env.stats()),
    ("logits_trajectory", lambda env, c: env.logits_trajectory(1)),
    ("get_legal_actions", lambda env, c: env.get_legal_actions()),
    ("set_cr_due_date_factor", lambda env, c: env.set_cr_due_date_factor(1.5)),
    ("host_masked_random", lambda env, c: env.host_masked_random(np_(env.action_mask), 5)),
    ("host_wait_mask", lambda env, c: env.host_wait_mask()),
    ("host_wait_obs", lambda env, c: env.host_wait_obs()),
    ("synchronize", lambda env, c: env.synchronize()),
]

# Methods without an env (static), and the one that ends the handle.
STATIC = {"host_configure", "host_set_simd"}
ENDS = {"close"}


class Case:
    """A batch with a host mirror in a fixed state and RNG counter, after a random walk, with one env run to done and
    the host-step pipeline primed; the table, logit rows and orders the calls take; restore() puts the batch back."""

    def __init__(self, make_env, backend, batch, seed=3):
        import torch
        names, walk, self.k = BATCHES[backend][batch]
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=seed, host_mirror=True)
        env.reset()
        random_walk(env, walk)
        while not bool(np_(env.done)[-1]):                # the last env to done, the others held by JSS_ACTION_SKIP
            a = _skip(env)
            a[-1] = env.policy("RANDOM")[-1]
            env.step(a)
        done = np_(env.done)
        assert done.any() and not done.all(), done
        env.host_step_begin(np_(_skip(env)))
        env.host_wait_obs()
        self.env, self.snap, self.counter = env, snapshot(env), env._step_index
        self.host_table = random_table(env, seed + 1)
        self.table = lc._to_dev(env, self.host_table)
        self.rows = lc._to_dev(env, greedy_rows(env, self.host_table))
        self.order = env.sample_without_replacement(self.table, self.k, order=True)["order"]
        rng = np.random.default_rng(seed)
        self.w = torch.from_numpy(rng.standard_normal((env.num_envs, self.k)).astype(np.float32)).to(env.device)
        self.v = torch.from_numpy(rng.standard_normal((env.num_envs, self.k)).astype(np.float32)).to(env.device)

    def restore(self):
        self.env.import_state(self.snap)
        self.env._step_index = self.counter

    def leaf(self):
        return self.table.clone().requires_grad_(True)


def _losses(c, lp, h=None):
    """The losses on a producer's outputs: on log_prob alone, and with the entropy on it alone and on both."""
    if h is None:
        return {"log_prob": (c.w * lp).sum()}
    return {"log_prob": (c.w * lp).sum(), "entropy": (c.v * h).sum(), "both": (c.w * lp).sum() + (c.v * h).sum()}


# The replayed producers, as call(env, case, x) -> {loss name: loss}.
REPLAYED = {
    "sample_episodes": lambda env, c, x: _losses(c, env.sample_episodes(x, c.k)["log_prob"]),
    "sample_episodes_entropy": lambda env, c, x: _losses(
        c, *(lambda o: (o["log_prob"], o["entropy"]))(env.sample_episodes(x, c.k, entropy=True))),
    "order_log_prob": lambda env, c, x: _losses(c, env.order_log_prob(x, c.order)[0]),
    "order_log_prob_entropy": lambda env, c, x: _losses(
        c, *(lambda o: (o[0], o[2]))(env.order_log_prob(x, c.order, entropy=True))),
    "sample_without_replacement": lambda env, c, x: _losses(c, env.sample_without_replacement(x, c.k)["log_prob"]),
}


def _stored(env, c, x, entropy):
    _, _, _, _, info = env.rollout_priority_sample(x, n_steps=8, entropy=entropy)
    w, v = c.w[:, 0], c.v[:, 0]
    return (w * info["log_prob"]).sum() + ((v * info["entropy"]).sum() if entropy else 0)


def _bits(t):
    return np_(t).view(np.uint32).copy()


class References:
    """The float64 gradients of the producers' losses in the case's state and counter, by the references of the
    producers' own suites, each computed once: sample_episodes_suite.twin_samples (sample_episodes_gradient),
    entropy_suite.sample_twins (entropy_backward), swor_suite.decisions + f64_grad (swor_gradient) and, for the
    entropy of given orders, entropy_suite.EntTwin driven by the orders (entropy_backward)."""

    def __init__(self, make_env, c):
        self.make_env, self.c, self.memo = make_env, c, {}

    def _once(self, key, fn):
        if key not in self.memo:
            self.memo[key] = fn()
        return self.memo[key]

    def _order_entropy_grads(self):
        c, env = self.c, self.c.env
        out = []
        for s in range(c.k):
            tw = self.make_env(env.num_envs, {"instance_paths": list(env.instances),
                                              "env_to_instance": list(env.env_to_instance)}, auto_reset=False,
                               seed=env.seed)
            tw.reset()
            tw.import_state(c.snap)
            twin = EntTwin(tw, c.host_table, driver=-np_(c.order)[:, s].astype(np.float32))
            twin.steps(2 * env.jobs * env.machines + 1, 0)
            out.append(twin.grads()[0])
            tw.close()
        return np.stack(out)

    def __call__(self, producer, loss):
        """(want, tolerance per entry) of `loss` of `producer`."""
        c, env = self.c, self.c.env
        w, v = np_(c.w).astype(np.float64), np_(c.v).astype(np.float64)
        if loss == "entropy":
            w = np.zeros_like(w)
        if loss == "log_prob":
            v = np.zeros_like(v)
        if producer == "sample_episodes":
            g = self._once("twin_samples", lambda: twin_samples(self.make_env, env, c.host_table, c.k, c.counter)[2])
            return np.einsum("ns,snjm->njm", w, g), 1e-5 * np.einsum("ns,snjm->njm", np.abs(w), 1 + np.abs(g))
        if producer == "sample_episodes_entropy":
            g, gh = self._once("sample_twins",
                               lambda: sample_twins(self.make_env, env, c.host_table, c.k, c.counter)[3:])
            want = np.einsum("ns,snjm->njm", w, g) + np.einsum("ns,snjm->njm", v, gh)
            return want, 1e-5 * (np.einsum("ns,snjm->njm", np.abs(w), 1 + np.abs(g)) +
                                 np.einsum("ns,snjm->njm", np.abs(v), 1 + np.abs(gh)))
        # order_log_prob and sample_without_replacement: the search at the case's counter gives the case's orders
        dec = self._once("decisions", lambda: decisions(self.make_env, env, np_(c.order)))
        want = f64_grad(dec, c.host_table, w) if w.any() else np.zeros((env.num_envs, env.jobs, env.machines))
        tol = 1e-4 * (1 + np.abs(want).max())
        if v.any():
            gh = self._once("order_entropy", self._order_entropy_grads)
            want = want + np.einsum("ns,snjm->njm", v, gh)
            tol = tol + 1e-4 * (1 + np.abs(want))
        return want, np.broadcast_to(tol, want.shape)


def _forward_all(c):
    """Every producer's forward from the case's state: the stored ones first (each from the restored state; they step
    the envs), then the replayed ones at the case's counter.  Returns [(producer, loss name, x, loss)]."""
    env = c.env
    made = []
    for entropy in (False, True):
        c.restore()
        x = c.leaf()
        made.append(("rollout_priority_sample" + ("_entropy" if entropy else ""), "both", x, _stored(env, c, x, entropy)))
    c.restore()
    for producer, run in REPLAYED.items():
        env._step_index = c.counter
        x = c.leaf()
        made += [(producer, name, x, loss) for name, loss in run(env, c, x).items()]
    return made


def _grad(x, loss):
    x.grad = None
    loss.backward(retain_graph=True)
    g = _bits(x.grad)
    x.grad = None
    return g


@native_test(emu=["mixed"], gpu=["mixed", "ta80"])
def backward_state_matrix(make_env, backend, batch):
    """Every producer (sample_episodes and order_log_prob with and without entropy, losses on log_prob, entropy and
    both; sample_without_replacement; rollout_priority_sample with and without entropy) against every intervening
    call: with nothing in between each gradient is held to its float64 reference (at the mixed batch); after each call
    that leaves the envs untouched it is that gradient bit for bit; after each call that may change them the replayed
    producers raise and leave x.grad None, and rollout_priority_sample gives its gradient bit for bit."""
    import pytest
    c = Case(make_env, backend, batch)
    env = c.env
    made = _forward_all(c)
    nothing = {(p, name): _grad(x, loss) for p, name, x, loss in made}
    if batch == "mixed":
        ref = References(make_env, c)
        for p, name, x, loss in made:
            if p.startswith("rollout_priority_sample"):
                continue
            want, tol = ref(p, name)
            got = nothing[(p, name)].view(np.float32).astype(np.float64)
            assert (np.abs(got - want) <= tol).all(), (p, name, np.abs(got - want).max())
    # one loss per forward (both terms with entropy): the replays are what take the time
    made = [m for m in _forward_all(c) if m[1] == "both" or (m[1] == "log_prob" and not m[0].endswith("_entropy"))]
    for method, call in UNTOUCHED:
        call(env, c)
        for p, name, x, loss in made:
            assert np.array_equal(_grad(x, loss), nothing[(p, name)]), (method, p, name)
    for i, (method, call) in enumerate(MUTATING):
        made = _forward_all(c)
        call(env, c)
        for p, name, x, loss in made:
            if p.startswith("rollout_priority_sample"):
                assert np.array_equal(_grad(x, loss), nothing[(p, name)]), (method, i, p)
                continue
            with pytest.raises(RuntimeError, match=f"^{p.replace('_entropy', '')}: backward after a call"):
                loss.backward(retain_graph=True)
            assert x.grad is None, (method, i, p, name)
    env.close()


@native_test()
def backward_state_classification(make_env, backend):
    """Every public method of JssVecEnv is listed as changing the envs, leaving them untouched, static, or ending the
    handle (found by introspection, so a new method fails here until it is listed).  Each untouched one leaves
    export_state(), real_obs, action_mask, the scalar records and stats() bit for bit; after each changing one, and after
    close(), a gradient drawn before it refuses."""
    import pytest
    public = {name for name, v in inspect.getmembers(JssVecEnv) if not name.startswith("_") and callable(v)}
    listed = {m for m, _ in MUTATING} | {m for m, _ in UNTOUCHED} | STATIC | ENDS
    assert public == listed, ("not listed", public - listed, "not methods", listed - public)
    assert not {m for m, _ in MUTATING} & {m for m, _ in UNTOUCHED}
    for name in STATIC:
        assert isinstance(inspect.getattr_static(JssVecEnv, name), staticmethod), name
    c = Case(make_env, backend, "mixed")
    env = c.env
    for method, call in UNTOUCHED:
        before, stats = _outputs(env), env.stats()
        call(env, c)
        after = _outputs(env)
        for key, val in before.items():
            assert np.array_equal(val.view(np.uint32) if val.dtype == np.float32 else val,
                                  after[key].view(np.uint32) if val.dtype == np.float32 else after[key]), (method, key)
        assert env.stats() == stats, method
    for method, call in MUTATING + [("close", lambda env, c: env.close())]:
        c.restore()
        x = c.leaf()
        lp, _ = env.order_log_prob(x, c.order[:, :1])
        call(env, c)
        with pytest.raises(RuntimeError, match="^order_log_prob: backward after"):
            lp.sum().backward()
        assert x.grad is None, method


@native_test()
def backward_state_reported_flow(make_env, backend):
    """The flow of a training loop that steps its envs before loss.backward(): the backward raises and leaves x.grad
    None, where it used to return the gradient of other episodes; the same draw backed before the step gives the
    gradient of the twins' episodes."""
    import pytest
    import torch
    env = make_env(4, {"instance_path": "ta01"}, seed=3, auto_reset=False)
    env.reset()
    table = torch.from_numpy(np.random.default_rng(5).standard_normal((4, 15, 15)).astype(np.float32))
    x = table.to(env.device).clone().requires_grad_(True)
    si = env._step_index
    env.sample_episodes(x, 4)["log_prob"].sum().backward()
    _, _, grads, _ = twin_samples(make_env, env, table.numpy(), 4, si)
    want = grads.sum(0)
    assert (np.abs(np_(x.grad) - want) <= 1e-5 * (1 + np.abs(grads)).sum(0)).all()
    x.grad = None
    env._step_index = si
    lp = env.sample_episodes(x, 4)["log_prob"]
    env.step(env.policy("RANDOM"))
    with pytest.raises(RuntimeError, match="run sample_episodes again"):
        lp.sum().backward()
    assert x.grad is None


@native_test()
def backward_state_graphs(make_env, backend):
    """The graph shapes autograd allows, each against the float64 references: two forwards on one handle summed into
    one loss; backward(retain_graph=True) twice, bit for bit; the backward of an older forward after a newer one; a
    forward on handle A while handle B is stepped; and a backward after close() raises for every replayed producer."""
    import pytest
    import torch
    names = {"emu": ["ta01", SMALL, NONPERM, TINY], "gpu": ["ta01", "ta51", NONPERM, EMU_CLASSES[2], SMALL]}[backend]
    k = 3
    env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=7)
    env.reset()
    random_walk(env, 12)
    n = env.num_envs
    table = random_table(env, 8)
    dev = lc._to_dev(env, table)
    rng = np.random.default_rng(9)
    w1, w2 = (torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)).to(env.device) for _ in range(2))
    si = env._step_index
    _, _, grads, _ = twin_samples(make_env, env, table, k, si)
    want_se = np.einsum("ns,snjm->njm", np_(w1).astype(np.float64), grads)
    tol_se = 1e-5 * np.einsum("ns,snjm->njm", np.abs(np_(w1)).astype(np.float64), 1 + np.abs(grads))
    order = env.sample_without_replacement(dev, k, order=True)["order"]
    want_o = f64_grad(decisions(make_env, env, np_(order)), table, np_(w2).astype(np.float64))
    tol_o = 1e-4 * (1 + np.abs(want_o).max())

    def close_to(got, want, tol, ctx):
        assert (np.abs(np_(got).astype(np.float64) - want) <= tol).all(), (ctx, np.abs(np_(got) - want).max())

    # two forwards on one handle, one loss
    x = dev.clone().requires_grad_(True)
    env._step_index = si
    lp1 = env.sample_episodes(x, k)["log_prob"]
    lp2, _ = env.order_log_prob(x, order)
    ((w1 * lp1).sum() + (w2 * lp2).sum()).backward()
    close_to(x.grad, want_se + want_o, tol_se + tol_o, "summed")
    # retain_graph twice
    x = dev.clone().requires_grad_(True)
    env._step_index = si
    loss = (w1 * env.sample_episodes(x, k)["log_prob"]).sum()
    loss.backward(retain_graph=True)
    g1 = x.grad.clone()
    x.grad = None
    loss.backward()
    assert np.array_equal(_bits(g1), _bits(x.grad))
    close_to(g1, want_se, tol_se, "retained")
    # an older forward after a newer one
    x = dev.clone().requires_grad_(True)
    env._step_index = si
    old = (w1 * env.sample_episodes(x, k)["log_prob"]).sum()
    y = dev.clone().requires_grad_(True)
    new = (w1 * env.sample_episodes(y, k)["log_prob"]).sum()
    new_o = (w2 * env.sample_without_replacement(y, k)["log_prob"]).sum()
    old.backward()
    close_to(x.grad, want_se, tol_se, "older")
    (new + new_o).backward()
    assert torch.isfinite(y.grad).all()
    # handle A draws while handle B steps
    other = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=7)
    other.reset()
    x = dev.clone().requires_grad_(True)
    env._step_index = si
    lp1 = env.sample_episodes(x, k)["log_prob"]
    lp2, _ = env.order_log_prob(x, order)
    random_walk(other, 3)
    ((w1 * lp1).sum() + (w2 * lp2).sum()).backward()
    close_to(x.grad, want_se + want_o, tol_se + tol_o, "other handle stepped")
    # an order_log_prob loss on B while A steps refuses only B's
    xb = lc._to_dev(other, table).requires_grad_(True)
    lb, _ = other.order_log_prob(xb, torch.zeros((n, env.jobs, env.machines), dtype=torch.int32, device=env.device))
    env.step(env.policy("RANDOM"))
    lb.sum().backward()
    assert xb.grad is not None
    other.close()
    # close()
    x = dev.clone().requires_grad_(True)
    losses = {"sample_episodes": env.sample_episodes(x, k, entropy=True)["entropy"].sum(),
              "order_log_prob": env.order_log_prob(x, order)[0].sum(),
              "sample_without_replacement": env.sample_without_replacement(x, k)["log_prob"].sum()}
    env.close()
    for who, loss in losses.items():
        with pytest.raises(RuntimeError, match=f"^{who}: backward after close"):
            loss.backward()
        assert x.grad is None, who


@native_test()
def backward_state_obs_beam_search(make_env, backend):
    """ObsBeamSearch: a gradient drawn before a round's step() refuses; start() steps only to take forced no-ops, so a
    gradient drawn before it refuses when slot 0 of a group had only the no-op legal and is the one drawn without
    start() in between otherwise, bit for bit; result() leaves a gradient drawn before it alone."""
    import pytest
    W = 2
    names = {"emu": ["ta01"] * 2 + [SMALL] * 2, "gpu": ["ta01"] * 4 + ["ta41"] * 4}[backend]
    for forced in (False, True):
        env = make_env(len(names), batch_cfg(names, sort=False), auto_reset=False, seed=11)
        env.reset()
        if forced:                                       # at reset every job is legal: start() takes no step
            random_walk(env, 6)
            x_ = env.export_state()
            x_["legal"][0] = 0
            x_["flags"][0] = int(x_["flags"][0]) | (N.FLAG_NOOP_LEGAL << 8)
            env.import_state(x_)
            assert noop_only(env)[0]
        table = random_table(env, 12)
        dev = lc._to_dev(env, table)
        x = dev.clone().requires_grad_(True)
        lp = env.sample_episodes(x, 2)["log_prob"].sum()
        lp.backward(retain_graph=True)
        alone = _bits(x.grad)
        x.grad = None
        s = ObsBeamSearch(env, W)
        s.start()
        if forced:
            with pytest.raises(RuntimeError, match="^sample_episodes: backward after"):
                lp.backward()
            assert x.grad is None
        else:
            lp.backward()
            assert np.array_equal(_bits(x.grad), alone)
        y = dev.clone().requires_grad_(True)
        lo, _ = env.order_log_prob(y, np.zeros((env.num_envs, env.jobs, env.machines), np.int32))
        s.result(order=True)
        lo.sum().backward(retain_graph=True)
        y.grad = None
        s.step(lc._to_dev(env, greedy_rows(env, table)))
        with pytest.raises(RuntimeError, match="^order_log_prob: backward after"):
            lo.sum().backward()
        assert y.grad is None
        env.close()
