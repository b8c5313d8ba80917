"""Backend-agnostic parity checks: the native env (real CUDA library with `-m gpu`, host emulation of the same kernels
in the CPU suite; tests/backends.py) against the CPU oracle and the golden fixtures recorded from the unmodified Python
reference.

Bars: bit-exact action_mask / done / current_time_step / raw integer reward / integer state; real_obs and the scaled
reward bit for bit the reference's float64 quotients rounded once to fp32 (assert_obs_exact, assert_reward_exact).  Each
reference entry is one float64 division of two integers below 2^24, so it is correctly rounded, and rounding it to fp32
gives the correctly rounded fp32 quotient (53 >= 2 * 24 + 2: no double-rounding error) -- the value the kernels' jss_div
claims to emit.  The facade's float64 observation is the device's fp32 one widened, its float64 reward the reference's
own quotient.
"""
import numpy as np

from jssenv_b200 import JssEnv
from jssenv_b200 import _native as N
from jssenv_b200.dispatching import DISPATCHING_RULES, get_rule
from jssenv_b200.instances import load_instance
from oracle.jss_oracle import OracleEnv, OracleError
from oracle.logits_oracle import hash3
from tests.helpers import load_json, load_trace, replay_optimal

OUTPUTS = ("action_mask", "real_obs", "reward", "reward_raw", "done", "current_time_step", "flags", "episode_count",
           "last_makespan", "last_return")


def np_(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def batch_cfg(names, sort=True):
    """Config of a batch whose env i runs names[i]: an instance name, or a parsed (machine, duration) pair, which is
    told apart from the others by identity.  The instances are numbered in name order, or with sort=False in order of
    first appearance; the numbering decides the tile layout the kernels run."""
    def same(a, b):
        return a is b or (isinstance(a, str) and a == b)
    uniq = []
    for n in names:
        if not any(same(n, u) for u in uniq):
            uniq.append(n)
    if sort:
        uniq.sort()
    return {"instance_paths": uniq, "env_to_instance": [next(k for k, u in enumerate(uniq) if same(n, u)) for n in names]}


def twin_envs(make_env, names, sort=True, **kw):
    """Two envs of the same batch (batch_cfg(names, sort)) and arguments, both reset."""
    cfg = batch_cfg(names, sort)
    a_env, b_env = make_env(len(names), cfg, **kw), make_env(len(names), cfg, **kw)
    a_env.reset(); b_env.reset()
    return a_env, b_env


def assert_twins_equal(a_env, b_env, ctx, rows=slice(None), state=False, stats=False):
    """Every per-env output of a_env equals that of b_env's envs `rows`, bit for bit; with state / stats, the exported
    state and the statistics too."""
    for name in OUTPUTS:
        x, y = np_(getattr(a_env, name)), np_(getattr(b_env, name))[rows]
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        assert np.array_equal(x, y), (ctx, name)
    if state:
        xa, xb = a_env.export_state(), b_env.export_state()
        for k in xa:
            assert np.array_equal(np_(xa[k]), np_(xb[k])[rows]), (ctx, k)
    if stats:
        assert a_env.stats() == b_env.stats(), ctx


def oracle_episode(inst, choose):
    """One oracle episode of `inst` (a name or a parsed pair) from reset to done, `choose(o, step)` picking each action.
    Returns the makespan, the raw return and the number of steps."""
    o = OracleEnv(*(load_instance(inst) if isinstance(inst, str) else inst))
    o.reset()
    done, step, total = False, 0, 0
    while not done:
        _, _, done, _, _ = o.step(choose(o, step))
        total += o.last_raw_reward
        step += 1
    return o.current_time_step, total, step


def _assert_f32_exact(got, ref, what, ctx):
    got = np.asarray(got)
    assert got.dtype == np.float32, (ctx, what, got.dtype)
    want = np.asarray(ref, np.float64).astype(np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    if bad.any():
        k = tuple(int(i) for i in np.argwhere(bad)[0]) if bad.ndim else ()
        raise AssertionError(f"{ctx}: {what} differs from the correctly rounded reference at {int(bad.sum())} entries; "
                             f"first at {k}: got {got[k]!r}, want {want[k]!r} (float64 {np.asarray(ref)[k]!r})")


def assert_obs_exact(got_f32, ref_f64, ctx=""):
    """The device's fp32 observation entries equal the reference's float64 ones rounded once to fp32, bit for bit."""
    _assert_f32_exact(got_f32, ref_f64, "real_obs", ctx)


def assert_reward_exact(got_f32, ref_f64, ctx=""):
    """The device's fp32 scaled reward(s) equal the reference's float64 ones rounded once to fp32, bit for bit."""
    _assert_f32_exact(got_f32, ref_f64, "reward", ctx)


def assert_facade_obs_exact(got_f64, ref_f64, ctx=""):
    """The facade's float64 observation is the device's fp32 one widened: float64(float32(reference)), bit for bit."""
    got = np.asarray(got_f64)
    assert got.dtype == np.float64, (ctx, got.dtype)
    want = np.asarray(ref_f64, np.float64).astype(np.float32).astype(np.float64)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), f"{ctx}: facade real_obs"


def compare_env_to_oracle(env, i, o, obs, reward=None, done=None, raw=None, ctx=""):
    J = o.jobs
    mask = np_(obs["action_mask"][i])
    assert np.array_equal(mask[: J + 1], o.legal_actions), f"{ctx}: mask env {i}"
    assert not mask[J + 1:].any(), f"{ctx}: padding mask bytes must stay 0"
    ro = np_(obs["real_obs"][i])
    assert_obs_exact(ro[:J], o.state, f"{ctx}: env {i}")
    assert ro.min() >= 0.0 and ro.max() <= 1.0
    assert int(env.current_time_step[i]) == o.current_time_step, f"{ctx}: time env {i}"
    if reward is not None:
        assert_reward_exact(np.float32(reward[0]), reward[1], f"{ctx}: env {i}")
    if raw is not None:
        assert int(raw[0]) == int(raw[1]), f"{ctx}: raw reward {raw}"
    if done is not None:
        assert bool(done[0]) == bool(done[1]), f"{ctx}: done"


def compare_exported_state(env, oracles, alive=None, ctx=""):
    """Every integer array of the reference, including the derived ones."""
    x = {k: np_(v) for k, v in env.export_state().items()}
    env.synchronize()
    for i, o in enumerate(oracles):
        if alive is not None and not alive[i]:
            continue
        J, M = o.jobs, o.machines
        assert np.array_equal(x["todo"][i, :J], o.todo_time_step_job), f"{ctx} todo {i}"
        assert np.array_equal(x["tufco"][i, :J], o.time_until_finish_current_op_jobs), f"{ctx} tufco {i}"
        assert np.array_equal(x["idle_last"][i, :J], o.idle_time_jobs_last_op), f"{ctx} idle_last {i}"
        assert np.array_equal(x["total_idle"][i, :J], o.total_idle_time_jobs), f"{ctx} total_idle {i}"
        assert np.array_equal(x["tuam"][i, :M], o.time_until_available_machine), f"{ctx} tuam {i}"
        assert np.array_equal(x["legal"][i, :J].astype(bool), o.legal_actions[:J]), f"{ctx} legal {i}"
        assert np.array_equal(x["blocked"][i, :J].astype(bool), o.action_illegal_no_op), f"{ctx} blocked {i}"
        assert int(x["t"][i]) == o.current_time_step
        # stale column 4 numerator (appendix A.3)
        col4 = x["col4"][i, :J].astype(np.float64) / o.max_time_op
        assert np.abs(col4 - o.state[:, 4]).max() <= 1e-12, f"{ctx} col4 {i}"


def check_random_batch(make_env, names, n_steps, seed, state_every=25, noop_force_every=0):
    """Mixed batch; the ORACLE side picks masked-random actions (optionally a forced no-op
    whenever an event is pending, like tests/test_solutions.py:762), both sides step."""
    env = make_env(len(names), batch_cfg(names))
    oracles = [OracleEnv(*load_instance(n)) for n in names]
    rng = np.random.default_rng(seed)
    obs = env.reset()
    for o in oracles:
        o.reset()
    for i, o in enumerate(oracles):
        compare_env_to_oracle(env, i, o, obs, ctx="reset")
    alive = np.ones(len(names), bool)
    for step in range(n_steps):
        acts = np.full(len(names), N.ACTION_SKIP, np.int32)
        for i, o in enumerate(oracles):
            if not alive[i]:
                continue
            legal = np.flatnonzero(o.legal_actions)
            if noop_force_every and step % noop_force_every == noop_force_every - 1 and len(o.next_time_step) > 0:
                acts[i] = o.jobs
            else:
                acts[i] = int(legal[rng.integers(len(legal))])
        obs, reward, done, trunc, info = env.step(acts)
        reward, done, raw = np_(reward), np_(done), np_(env.reward_raw)
        assert not np_(trunc).any() and info == {}
        for i, o in enumerate(oracles):
            if not alive[i]:
                continue
            try:
                oo, r, d, _, _ = o.step(int(acts[i]))
            except OracleError:
                # forced no-op that empties the event queue: the reference raises, the device flags it
                assert int(env.flags[i]) & N.FLAG_ERROR, f"step {step} env {i}: expected error bit"
                alive[i] = False
                continue
            assert not (int(env.flags[i]) & N.FLAG_ERROR), f"step {step} env {i}: unexpected error bit"
            compare_env_to_oracle(env, i, o, obs, (reward[i], r), (done[i], d), (raw[i], o.last_raw_reward),
                                  ctx=f"step {step} action {acts[i]}")
            if d:
                alive[i] = False
                assert int(env.last_makespan[i]) == o.current_time_step
        if step % state_every == 0:
            compare_exported_state(env, oracles, alive, ctx=f"step {step}")
        if not alive.any():
            break
    return env, oracles


def check_golden_trace(make_env, path):
    """Replay a trace recorded from the unmodified Python reference (tests/golden)."""
    tr = load_trace(path)
    env = make_env(1, {"instance_path": tr["inst"]})
    obs = env.reset()
    J = tr["mask"].shape[1] - 1

    def check(k):
        assert np.array_equal(np_(obs["action_mask"][0])[: J + 1], tr["mask"][k]), f"mask {k}"
        assert_obs_exact(np_(obs["real_obs"][0])[:J], tr["obs"][k], f"obs {k}")
        assert int(env.current_time_step[0]) == tr["t"][k]

    check(0)
    for k, a in enumerate(tr["actions"]):
        obs, reward, done, _, _ = env.step(np.array([a], np.int32))
        assert_reward_exact(np_(reward)[0], tr["reward"][k], f"reward {k}")
        assert bool(done[0]) == bool(tr["done"][k])
        check(k + 1)
        if k % 50 == 0:
            x = {n: np_(v) for n, v in env.export_state().items()}
            assert np.array_equal(x["todo"][0, :J], tr["todo"][k + 1])
            assert np.array_equal(x["blocked"][0, :J].astype(bool), tr["blocked"][k + 1])
            assert np.array_equal(x["tuam"][0, : tr["tuam"].shape[1]], tr["tuam"][k + 1])


def check_facade_optimal(inst):
    """The reference's known-answer replays (tests/test_solutions.py) through the JssEnv facade,
    including its attribute surface (machine_legal, needed_machine_jobs, next_time_step ...)."""
    spec = load_json("optimal_sequences.json")[inst]
    env = JssEnv({"instance_path": inst})
    assert replay_optimal(env, spec) == spec["makespan"]
    assert env.last_time_step == spec["makespan"]
    assert env.solution.min() != -1 and (env.todo_time_step_job == env.machines).all()
    assert len(env.next_time_step) == 0
    env.reset()
    assert env.current_time_step == 0
    env.close()


def check_facade_attributes(inst, n_steps, seed):
    """Every attribute the reference exposes, against the oracle, along a random trace."""
    env = JssEnv({"instance_path": inst})
    o = OracleEnv(*load_instance(inst))
    rng = np.random.default_rng(seed)
    obs, _ = env.reset(), o.reset()
    assert env.jobs == o.jobs and env.machines == o.machines
    assert (env.max_time_op, env.max_time_jobs, env.sum_op) == (o.max_time_op, o.max_time_jobs, o.sum_op)
    assert np.array_equal(env.instance_matrix, o.instance_matrix)
    done = False
    for _ in range(n_steps):
        for name in ("legal_actions", "machine_legal", "needed_machine_jobs", "todo_time_step_job",
                     "time_until_available_machine", "time_until_finish_current_op_jobs",
                     "total_perform_op_time_jobs", "total_idle_time_jobs", "idle_time_jobs_last_op",
                     "action_illegal_no_op", "illegal_actions", "solution"):
            assert np.array_equal(getattr(env, name), getattr(o, name)), name
        assert env.nb_legal_actions == o.nb_legal_actions and env.nb_machine_legal == o.nb_machine_legal
        assert env.next_time_step == o.next_time_step
        assert env.current_time_step == o.current_time_step
        assert obs["real_obs"].dtype == np.float64 and obs["real_obs"].shape == (o.jobs, 7)
        assert_facade_obs_exact(env.state, o.state)
        if done:
            break
        legal = np.flatnonzero(o.legal_actions)
        a = int(legal[rng.integers(len(legal))])
        obs, r, done, trunc, info = env.step(a)
        _, r2, d2, _, _ = o.step(a)
        assert r == r2 and done == d2 and trunc is False and info == {}     # float64 quotient, bit-equal
    env.close()


def check_rules_seeded(inst):
    """Rule episodes with np.random.seed(0) reproduce the reference's makespans (dispatching.py)."""
    gold = load_json("rule_makespans.json")[inst]
    env = JssEnv({"instance_path": inst})
    for name, rule in DISPATCHING_RULES.items():
        np.random.seed(0)
        total, makespan = rule.run_episode(env)
        assert makespan == gold[name]["makespan"], (inst, name)
        assert abs(total - gold[name]["total_reward"]) <= 1e-3, (inst, name)
    if inst in load_json("cr_factor_makespans.json"):      # CriticalRatio(due_date_factor) as a launch parameter
        from jssenv_b200.dispatching import CriticalRatio
        for f, exp in load_json("cr_factor_makespans.json")[inst].items():
            np.random.seed(0)
            total, makespan = CriticalRatio(due_date_factor=float(f)).run_episode(env)
            assert makespan == exp["makespan"] and abs(total - exp["total_reward"]) <= 1e-3, (inst, f)
        np.random.seed(0)
        assert DISPATCHING_RULES["CR"].run_episode(env)[1] == gold["CR"]["makespan"]   # default factor restored
    try:
        get_rule("NOPE")
        raise AssertionError("get_rule must raise ValueError")   # tests/test_dispatching.py:39-47
    except ValueError:
        pass
    env.close()


def check_policy_kernels(make_env, names, n_steps, seed):
    """jss_policy for every rule vs the oracle's rule functions on identical states, with the
    coin uniform taken from the shared counter RNG; RANDOM vs the oracle's sampler and the
    host helper jss_host_masked_random."""
    env = make_env(len(names), batch_cfg(names), seed=seed)
    oracles = [OracleEnv(*load_instance(n)) for n in names]
    obs = env.reset()
    for o in oracles:
        o.reset()
    rules = ["SPT", "FIFO", "MWR", "LWR", "MOR", "LOR", "CR"]
    alive = np.ones(len(names), bool)
    for step in range(n_steps):
        # every rule on the CURRENT state (explicit step_index so all rules see the same coin)
        for rule in rules:
            a_dev = np_(env.policy(rule, coin="device", step_index=step)).copy()
            a_never = np_(env.policy(rule, coin="never", step_index=step)).copy()
            for i, o in enumerate(oracles):
                if not alive[i]:
                    continue
                u = _coin_uniform(env.seed, env.env_id_base + i, step)
                exp, consumed = o.rule_action(rule, u)
                assert a_dev[i] == exp, (step, rule, i, a_dev[i], exp)
                exp_never, _ = o.rule_action(rule, 1.0)
                assert a_never[i] == exp_never, (step, rule, i)
        a = np_(env.policy("RANDOM", step_index=step)).copy()
        host = env.host_masked_random(np.ascontiguousarray(np_(env.action_mask)), step)
        for i, o in enumerate(oracles):
            if alive[i]:
                assert a[i] == o.masked_random_action(env.seed, env.env_id_base + i, step), (step, i)
                assert a[i] == host[i]
            else:
                a[i] = N.ACTION_SKIP
        obs, _, done, _, _ = env.step(a)
        for i, o in enumerate(oracles):
            if alive[i]:
                _, _, d, _, _ = o.step(int(a[i]))
                compare_env_to_oracle(env, i, o, obs, ctx=f"policy step {step}")
                alive[i] = not d
        if not alive.any():
            break


def _coin_uniform(seed, env, ctr):
    """u = hash3(seed, env, ctr) / 2^32"""
    return hash3(seed, env, ctr) / 4294967296.0


def check_rollout_matches_steps(make_env, names, rule, n_steps, seed):
    """The fused rollout kernel == policy kernel + step kernel, transition for transition;
    and both == the oracle driven by the same counter RNG."""
    a_env, b_env = twin_envs(make_env, names, seed=seed, auto_reset=True)
    a_env.rollout(rule, n_steps, write_obs=True)
    for _ in range(n_steps):
        b_env.step(b_env.policy(rule))
    assert_twins_equal(a_env, b_env, rule, state=True, stats=True)
    # oracle with the same RNG (auto-reset: a done env is reset by the next transition)
    for i, n in enumerate(names):
        o = OracleEnv(*load_instance(n))
        o.reset()
        done, episodes, makespan = False, 0, -1
        for step in range(n_steps):
            if done:
                o.reset(); done = False
                continue
            if rule == "RANDOM":
                a = o.masked_random_action(seed, i, step)
            else:
                a, _ = o.rule_action(rule, _coin_uniform(seed, i, step))
            _, _, done, _, _ = o.step(a)
            if done:
                episodes += 1; makespan = o.current_time_step
        assert int(a_env.episode_count[i]) == episodes, (i, n)
        if episodes:
            assert int(a_env.last_makespan[i]) == makespan
        assert int(a_env.current_time_step[i]) == o.current_time_step
        J = o.jobs
        if not done:
            assert np.array_equal(np_(a_env.action_mask[i])[: J + 1], o.legal_actions)
            assert_obs_exact(np_(a_env.real_obs[i])[:J], o.state, (n, i))
    return a_env


def check_errors_and_freeze(make_env):
    """Reference exceptions -> sticky error bit, env unchanged; done envs freeze; masked reset."""
    env = make_env(4, {"instance_path": "ta01"})
    o = OracleEnv(*load_instance("ta01"))
    obs = env.reset(); o.reset()
    before = {k: np_(v).copy() for k, v in env.export_state().items()}
    mask0, obs0 = np_(env.action_mask).copy(), np_(env.real_obs).copy()
    # env0: no-op with empty queue (IndexError jss_env.py:517); env1: out of range; env2: skip; env3: legal
    env.step(np.array([env.jobs, 99, N.ACTION_SKIP, 3], np.int32))
    flags = np_(env.flags)
    assert flags[0] & N.FLAG_ERROR and flags[1] & N.FLAG_ERROR and not flags[2] & N.FLAG_ERROR and not flags[3] & N.FLAG_ERROR
    after = {k: np_(v).copy() for k, v in env.export_state().items()}
    for k in before:
        if k == "flags":
            continue
        assert np.array_equal(before[k][:3], after[k][:3]), k
    assert np.array_equal(np_(env.action_mask)[:3], mask0[:3]) and np.array_equal(np_(env.real_obs)[:3], obs0[:3])
    o.step(3)
    compare_env_to_oracle(env, 3, o, env._obs(), ctx="legal env next to erroring envs")
    # illegal job action: job 3 is now running -> not legal
    env.step(np.array([N.ACTION_SKIP] * 3 + [3], np.int32))
    assert np_(env.flags)[3] & N.FLAG_ERROR
    compare_env_to_oracle(env, 3, o, env._obs(), ctx="illegal action leaves the env unchanged")
    # masked reset clears only env 0 and 3
    env.reset(np.array([1, 0, 0, 1], np.uint8))
    flags = np_(env.flags)
    assert flags[0] == 0 and flags[3] == 0 and flags[1] & N.FLAG_ERROR
    assert int(env.current_time_step[3]) == 0 and np_(env.action_mask)[3, : env.jobs].all()
    return env


def check_auto_reset_and_stats(make_env, name, seed):
    env = make_env(6, {"instance_path": name}, seed=seed, auto_reset=True)
    o = OracleEnv(*load_instance(name))
    env.reset()
    n_steps = 2 * (2 * env.jobs * env.machines) + 10
    mk_o, ret_o = [], []
    o.reset(); done = False; ret = 0
    for step in range(n_steps):
        if done:
            o.reset(); done = False; ret = 0
            continue
        a = o.masked_random_action(seed, 0, step)
        _, _, done, _, _ = o.step(a)
        ret += o.last_raw_reward
        if done:
            mk_o.append(o.current_time_step); ret_o.append(ret)
    for _ in range(n_steps):
        env.step(env.policy("RANDOM"))
    st = env.stats()
    assert int(env.episode_count[0]) == len(mk_o) and int(env.last_makespan[0]) == mk_o[-1]
    assert int(env.last_return[0]) == ret_o[-1]
    # identity (SURVEY a9): raw episode return = 2*sum_op - M*makespan
    assert ret_o[-1] == 2 * o.sum_op - o.machines * mk_o[-1]
    assert st["episodes"] == int(np_(env.episode_count).sum()) and st["episodes"] >= 6
    assert st["min_makespan"] <= st["max_makespan"] and st["envs_error"] == 0
    lm = np_(env.last_makespan)
    assert st["min_makespan"] <= lm.min() and st["max_makespan"] >= lm.max()
    return env


def check_snapshot_restore(make_env, name, seed):
    env = make_env(3, {"instance_path": name}, seed=seed)
    env.reset()
    for _ in range(40):
        env.step(env.policy("RANDOM"))
    snap = {k: v.clone() for k, v in env.export_state().items()}
    mask, obs = np_(env.action_mask).copy(), np_(env.real_obs).copy()
    hist = []
    for k in range(30):
        a = env.policy("RANDOM", step_index=1000 + k).clone()
        env.step(a)
        hist.append((np_(a).copy(), np_(env.action_mask).copy(), np_(env.reward_raw).copy()))
    env.import_state(snap)
    assert np.array_equal(np_(env.action_mask), mask) and np.array_equal(np_(env.real_obs), obs)
    for k in range(30):
        a = env.policy("RANDOM", step_index=1000 + k)
        assert np.array_equal(np_(a), hist[k][0])
        env.step(a)
        assert np.array_equal(np_(env.action_mask), hist[k][1]) and np.array_equal(np_(env.reward_raw), hist[k][2])
    return env


def check_step_host(make_env, name, seed):
    env = make_env(5, {"instance_path": name}, seed=seed)
    ref = make_env(5, {"instance_path": name}, seed=seed)
    env.reset(); ref.reset()
    mask = np.ascontiguousarray(np_(env.action_mask))
    for k in range(60):
        a = env.host_masked_random(mask, k)
        obs, rew, done, trunc, _ = env.step_host(a)
        ref.step(a)
        assert np.array_equal(obs["action_mask"], np_(ref.action_mask))
        assert np.array_equal(obs["real_obs"], np_(ref.real_obs))
        assert np.array_equal(rew, np_(ref.reward)) and np.array_equal(done, np_(ref.done))
        mask = obs["action_mask"]
    return env


def check_step_sample(make_env, names, rule, n_steps, seed):
    """jss_step_sample (step fused with the next decision) == policy kernel + step kernel."""
    a_env, b_env = twin_envs(make_env, names, seed=seed, auto_reset=True)
    act_a = a_env.policy(rule).clone()             # step_index 0
    b_env._step_index = 0
    for k in range(n_steps):
        act_b = b_env.policy(rule)                 # step_index k
        assert np.array_equal(np_(act_a), np_(act_b)), f"actions differ at step {k}"
        b_env.step(act_b)
        *_, act_a = a_env.step_sample(act_a, rule)  # applies step k, samples with step_index k+1
        assert_twins_equal(a_env, b_env, k, stats=k == n_steps - 1)
    return a_env


def check_host_pipeline(make_env, name, seed):
    """The pipelined host-buffer path (begin / wait_mask / wait_obs) == the device-resident path."""
    env = make_env(7, {"instance_path": name}, seed=seed)
    ref = make_env(7, {"instance_path": name}, seed=seed)
    env.reset(); ref.reset()
    mask = np.ascontiguousarray(np_(env.action_mask))
    a = env.host_masked_random(mask, 0)
    env.host_step_begin(a)
    for k in range(1, 80):
        mask, rew, done = env.host_wait_mask()
        ref.step(a)
        assert np.array_equal(mask, np_(ref.action_mask)), k
        assert np.array_equal(rew, np_(ref.reward)) and np.array_equal(done, np_(ref.done))
        nxt = env.host_masked_random(mask, k)
        obs_prev_expected = np_(ref.real_obs).copy()
        env.host_step_begin(nxt)                       # next step enqueued while the previous obs may still stream
        assert np.array_equal(env.host_wait_obs(previous=True), obs_prev_expected), k
        a = nxt
    return env


def check_host_pipeline_packed(make_env, names, seed, n_steps=80):
    """Packed host-buffer path: 10-byte integer rows over the wire + host expansion == device real_obs BIT FOR BIT
    (and mask / reward / done as in the plain path), on a mixed batch, through done/auto-reset transitions."""
    env, ref = twin_envs(make_env, names, seed=seed, auto_reset=True)
    # get past the trivial all-zero start: a few hundred device steps on both
    for k in range(120):
        a0 = ref.policy("RANDOM", step_index=k)
        ref.step(a0); env.step(np_(a0))
    mask = np.ascontiguousarray(np_(env.action_mask))
    a = env.host_masked_random(mask, 1000)
    env.host_step_begin(a, packed=True)
    for k in range(1, n_steps):
        mask, rew, done = env.host_wait_mask()
        ref.step(a)
        assert np.array_equal(mask, np_(ref.action_mask)), k
        assert np.array_equal(rew, np_(ref.reward)) and np.array_equal(done, np_(ref.done))
        nxt = env.host_masked_random(mask, 1000 + k)
        expected = np_(ref.real_obs).copy()
        # next step enqueued while the previous rows may still stream; every third step ships a share of the envs as
        # final fp32 rows by DMA (hybrid)
        env.host_step_begin(nxt, packed=True, dma_fraction=(0.0, 0.0, 0.4)[k % 3] if len(names) >= 4 else 0.0)
        env.host_set_simd(k % 3)                       # scalar / AVX2 / AVX-512 expansion paths in turn
        got = env.host_wait_obs(previous=True)
        for i, J in enumerate(env.env_jobs):
            assert np.array_equal(got[i, :J].view(np.uint32), expected[i, :J].view(np.uint32)), (k, i)
        a = nxt
    env.host_set_simd(2)
    env.host_wait_obs()
    return env


def synthetic_instance(J, M, seed, max_dur=99, permutation=True):
    """Random instance; with permutation=False a job may visit a machine several times / skip others
    (the reference accepts that: it only requires M (machine, duration) pairs per job)."""
    rng = np.random.default_rng(seed)
    if permutation:
        machine = np.stack([rng.permutation(M) for _ in range(J)]).astype(np.int32)
    else:
        machine = rng.integers(0, M, size=(J, M)).astype(np.int32)
    duration = rng.integers(1, max_dur + 1, size=(J, M)).astype(np.int32)
    return machine, duration


def check_synthetic_shapes(make_env, shapes, n_steps, seed):
    """Edge shapes: kernel limits (J = 128, M = 32, duration 2047), partially filled lanes (J = 33, 65, 127),
    tiny instances (J = 1, M = 2), non-permutation machine sequences -- each against the oracle."""
    insts = [synthetic_instance(J, M, seed + k, md, perm) for k, (J, M, md, perm) in enumerate(shapes)]
    env = make_env(len(insts), {"instance_paths": insts, "env_to_instance": list(range(len(insts)))})
    oracles = [OracleEnv(m, d) for m, d in insts]
    rng = np.random.default_rng(seed)
    obs = env.reset()
    for o in oracles:
        o.reset()
    alive = np.ones(len(insts), bool)
    for i, o in enumerate(oracles):
        compare_env_to_oracle(env, i, o, obs, ctx="reset")
    for step in range(n_steps):
        acts = np.full(len(insts), N.ACTION_SKIP, np.int32)
        for i, o in enumerate(oracles):
            if alive[i]:
                legal = np.flatnonzero(o.legal_actions)
                acts[i] = int(legal[rng.integers(len(legal))])
        obs, reward, done, _, _ = env.step(acts)
        reward, done, raw = np_(reward), np_(done), np_(env.reward_raw)
        for i, o in enumerate(oracles):
            if not alive[i]:
                continue
            _, r, d, _, _ = o.step(int(acts[i]))
            compare_env_to_oracle(env, i, o, obs, (reward[i], r), (done[i], d), (raw[i], o.last_raw_reward),
                                  ctx=f"shape {shapes[i]} step {step}")
            alive[i] = not d
        if step % 40 == 0:
            compare_exported_state(env, oracles, alive, ctx=f"step {step}")
        if not alive.any():
            break
    return env


def check_abi_error_codes(make_env):
    """jss_load_instances / jss_assign / jss_step argument validation (rc < 0 -> NativeError with a message)."""
    import pytest
    from jssenv_b200._native import NativeError
    bad = [
        (synthetic_instance(257, 4, 1), "exceeds"),                      # J > JSS_MAX_JOBS
        (synthetic_instance(4, 33, 1), "exceeds"),                       # M > JSS_MAX_MACHINES
        ((np.zeros((3, 1), np.int32), np.ones((3, 1), np.int32)), "machines"),   # "We need at least 2 machines"
    ]
    for inst, msg in bad:
        with pytest.raises((NativeError, ValueError), match=msg):
            make_env(2, {"instance_path": inst})
    m, d = synthetic_instance(5, 3, 2)
    d0 = d.copy(); d0[1, 1] = 0
    with pytest.raises(NativeError, match="duration"):                   # zero-length op (see DESIGN.md section 1)
        make_env(2, {"instance_path": (m, d0)})
    d1 = d.copy(); d1[0, 0] = 2048
    with pytest.raises(NativeError, match="duration"):
        make_env(2, {"instance_path": (m, d1)})
    with pytest.raises(NativeError, match="out of range"):
        make_env(2, {"instance_paths": [(m, d)], "env_to_instance": [0, 1]})


def check_facade_errors():
    """Reference exceptions through the facade: IndexError once, env unchanged and usable afterwards."""
    import pytest
    env = JssEnv({"instance_path": "ta01"})
    o = OracleEnv(*load_instance("ta01"))
    env.reset(); o.reset()
    with pytest.raises(IndexError):            # no-op with an empty event queue (jss_env.py:517)
        env.step(env.jobs)
    with pytest.raises(IndexError):            # raw advance with an empty event queue
        env.increase_time_step()
    obs, r, done, _, _ = env.step(2)
    o.step(2)
    assert np.array_equal(env.legal_actions, o.legal_actions) and env.current_time_step == o.current_time_step
    with pytest.raises(IndexError):            # job 2 is running now: not legal
        env.step(2)
    with pytest.raises(IndexError):
        env.step(env.jobs + 5)
    obs, r, done, _, _ = env.step(4)           # still usable, still in lock-step with the oracle
    oo, r2, d2, _, _ = o.step(4)
    assert np.array_equal(obs["action_mask"], oo["action_mask"]) and r == r2 and done == d2
    assert env.render() is not None and len(env.render()) == 2
    env.close()


def check_dispatching_api(make_env):
    """tests/test_dispatching.py restated for the mirror module: every rule returns a legal action after reset
    (:49-58), get_rule raises on unknown names (:39-47), compare_rules result keys (:96-107), makespan > 0 (:109-121)."""
    from jssenv_b200.dispatching import compare_rules, compare_rules_batched
    env = JssEnv({"instance_path": "ta01"})
    env.reset()
    for name, rule in DISPATCHING_RULES.items():
        a = rule(env)
        assert 0 <= a <= env.jobs and env.get_legal_actions()[a], name
        assert rule.get_name() == name and isinstance(rule.get_description(), str)
    res = compare_rules(env, rules=["SPT", "MWR"], num_episodes=1)
    assert set(res) == {"SPT", "MWR"} and all(set(v) == {"avg_reward", "avg_makespan"} for v in res.values())
    assert all(v["avg_makespan"] > 0 for v in res.values())
    env.close()
    venv = make_env(4, {"instance_paths": ["ta01", "ta31"], "env_to_instance": [0, 0, 1, 1]}, seed=3)
    resb = compare_rules_batched(venv, rules=["FIFO", "LOR"])
    assert set(resb) == {"FIFO", "LOR"} and all(v["avg_makespan"] > 0 for v in resb.values())


def check_tiny_uniform_batches(make_env, seed=50, shapes=((2, 2), (3, 4), (4, 3), (4, 32), (1, 2), (5, 5)), max_steps=None):
    """Uniform batches of tiny instances (J <= 4, so Jcap = 4 and 7 * Jcap < 32): the per-warp scratch must
    still hold _check_no_op's 32-entry horizon table (ADVICE r1: shared-memory overflow in the rollout kernel).
    16 envs of one instance: fused rollout == policy + step kernels == oracle, transition for transition."""
    for k, (J, M) in enumerate(shapes):
        inst = synthetic_instance(J, M, seed + k, max_dur=30)
        n = 16
        for rule in ("RANDOM", "SPT"):
            a_env, b_env = twin_envs(make_env, [inst] * n, seed=seed + k, auto_reset=True)
            n_steps = 6 * J * M + 7 if max_steps is None else min(max_steps, 6 * J * M + 7)
            a_env.rollout(rule, n_steps, write_obs=True)
            oracles = [OracleEnv(*inst) for _ in range(n)]
            done = [False] * n
            for o in oracles:
                o.reset()
            for step in range(n_steps):
                acts = b_env.policy(rule)
                b_env.step(acts)
                a_host = np_(acts)
                for i, o in enumerate(oracles):
                    if done[i]:
                        o.reset(); done[i] = False
                    else:
                        exp = (o.masked_random_action(seed + k, i, step) if rule == "RANDOM"
                               else o.rule_action(rule, _coin_uniform(seed + k, i, step))[0])
                        assert a_host[i] == exp, (J, M, rule, step, i)
                        _, _, done[i], _, _ = o.step(int(a_host[i]))
                    compare_env_to_oracle(b_env, i, o, b_env._obs(), ctx=f"tiny {J}x{M} {rule} step {step}")
            assert_twins_equal(a_env, b_env, (J, M, rule), stats=True)
            assert a_env.stats()["envs_error"] == 0


def check_shard_invariance(make_env, n_total=24, n_steps=350, seed=77):
    """SURVEY.md section 4 (end) / 8(e): results must not depend on how the global batch is sharded.
    One env of N_total envs == the shards [0, N/2) and [N/2, N) created with env_id_base = 0 and N/2 (and an
    uneven 3-way split), transition for transition, with the on-device policies (RNG keyed by GLOBAL env id)."""
    names = ["ta01", "ta31", "ta51", "ta80"]
    e2i = np.arange(n_total) % len(names)
    for rule in ("RANDOM", "FIFO"):
        cuts = [0, n_total // 2, n_total]
        cuts3 = [0, 5, 5 + 9, n_total]
        for cut in (cuts, cuts3):
            # fresh envs per split: episode_count / last_makespan are cumulative statistics that reset() keeps
            whole = make_env(n_total, {"instance_paths": names, "env_to_instance": e2i}, seed=seed, auto_reset=True)
            shards = [make_env(hi - lo, {"instance_paths": names, "env_to_instance": e2i[lo:hi]}, seed=seed,
                               auto_reset=True, env_id_base=lo) for lo, hi in zip(cut[:-1], cut[1:])]
            whole.reset(); whole._step_index = 0
            for s in shards:
                s.reset()
            for k in range(n_steps):
                aw = whole.policy(rule)
                for s, lo, hi in zip(shards, cut[:-1], cut[1:]):
                    a_s = s.policy(rule)
                    assert np.array_equal(np_(a_s), np_(aw)[lo:hi]), (rule, k, lo)
                    s.step(a_s)
                whole.step(aw)
                for s, lo, hi in zip(shards, cut[:-1], cut[1:]):
                    assert_twins_equal(s, whole, (rule, k), rows=slice(lo, hi))
            # the gathered per-shard statistics equal the statistics of the unsharded batch
            from jssenv_b200.distributed import combine_stats, STATS_KEYS
            comb = combine_stats([[s.stats()[key] for key in STATS_KEYS] for s in shards])
            assert comb == {**whole.stats(), "min_makespan": comb["min_makespan"]} or comb == whole.stats()
            for s in shards:
                s.close()
            whole.close()


def check_rollout_record(make_env, names, rule, n_steps, seed):
    """jss_rollout_traj: slot k of the recorded trajectory == the outputs after transition k of policy + step."""
    a_env, b_env = twin_envs(make_env, names, seed=seed, auto_reset=True)
    tr = a_env.rollout_record(rule, n_steps)
    for k in range(n_steps):
        acts = b_env.policy(rule)
        assert np.array_equal(np_(tr["actions"][k]), np_(acts)), k
        b_env.step(acts)
        assert np.array_equal(np_(tr["action_mask"][k]), np_(b_env.action_mask)), k
        assert np.array_equal(np_(tr["real_obs"][k]), np_(b_env.real_obs)), k
        assert np.array_equal(np_(tr["reward"][k]), np_(b_env.reward)) and np.array_equal(np_(tr["done"][k]), np_(b_env.done)), k
        assert np.array_equal(np_(tr["time"][k]), np_(b_env.current_time_step)), k
    assert_twins_equal(a_env, b_env, "end", stats=True)


def check_big_uniform_batches(make_env, seed=60, max_steps=150):
    """Uniform batches of instances with 129..256 jobs (8 jobs per lane, 16 bits per lane in the state block): fused
    rollout == policy + step kernels == oracle; fused step + sampler; packed host path; single-env facade."""
    check_tiny_uniform_batches(make_env, seed=seed, shapes=((130, 4), (256, 6)), max_steps=max_steps)
    inst = synthetic_instance(200, 8, seed + 9, max_dur=50)
    a_env, b_env = twin_envs(make_env, [inst] * 9, seed=seed, auto_reset=True)
    act_a = a_env.policy("MWR").clone()
    b_env._step_index = 0
    for k in range(max_steps):
        act_b = b_env.policy("MWR")
        assert np.array_equal(np_(act_a), np_(act_b)), k
        b_env.step(act_b)
        *_, act_a = a_env.step_sample(act_a, "MWR")
        assert_twins_equal(a_env, b_env, k)
    # packed rows + host expansion == device real_obs, bit for bit
    mask = np.ascontiguousarray(np_(a_env.action_mask))
    a_env.host_step_begin(a_env.host_masked_random(mask, 7), packed=True)
    a_env.host_wait_mask()
    got = a_env.host_wait_obs()
    assert np.array_equal(got.view(np.uint32), np_(a_env.real_obs).view(np.uint32))
    # facade on a 200-job instance
    env = JssEnv({"instance_path": inst})
    o = OracleEnv(*inst)
    obs, _ = env.reset(), o.reset()
    rng = np.random.default_rng(seed)
    for _ in range(max_steps):
        legal = np.flatnonzero(o.legal_actions)
        a = int(legal[rng.integers(len(legal))])
        obs, r, done, _, _ = env.step(a)
        oo, r2, d2, _, _ = o.step(a)
        assert np.array_equal(obs["action_mask"], oo["action_mask"])
        assert_facade_obs_exact(obs["real_obs"], oo["real_obs"])
        assert r == r2 and done == d2
        assert np.array_equal(env.todo_time_step_job, o.todo_time_step_job) and np.array_equal(env.machine_legal, o.machine_legal)
        if done:
            break
    env.close()
