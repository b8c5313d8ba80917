"""Parity tests proper: the real sm_90a library (jssenv_b200/libjss_b200.so, called
through the C-ABI) against the CPU oracle and the golden fixtures recorded from the
unmodified Python reference.  Run on an H100 with `pytest -m gpu`."""
import glob
import os

import numpy as np
import pytest

from tests import parity_common as pc
from tests.helpers import GOLDEN, load_json

pytestmark = pytest.mark.gpu


def make_env(n, cfg, **kw):
    from jssenv_b200 import JssVecEnv
    return JssVecEnv(n, cfg, **kw)


def test_gpu_library_is_the_cuda_one():
    import torch
    from jssenv_b200 import _native
    assert torch.cuda.is_available()
    assert _native.backend.name == "cuda"
    assert os.path.basename(_native.LIB_PATH) == "libjss_b200.so" and os.path.exists(_native.LIB_PATH)
    env = make_env(2, {"instance_path": "ta01"})
    assert env.real_obs.is_cuda and env.action_mask.is_cuda and env.launch_count >= 1


def test_gpu_random_mixed_batch_all_shapes():
    names = ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "dmu20", "ta51", "ta61", "ta71", "ta80"] * 3
    pc.check_random_batch(make_env, names, n_steps=3000, seed=11, state_every=50)


def test_gpu_full_episodes_ta80_many_envs():
    pc.check_random_batch(make_env, ["ta80"] * 24, n_steps=3000, seed=5, state_every=200)


def test_gpu_forced_noops():
    pc.check_random_batch(make_env, ["ta01", "ta15", "ta45", "ta62", "ta80", "dmu17"] * 2, n_steps=1500, seed=3,
                          noop_force_every=5)
    pc.check_random_batch(make_env, ["ta01", "ta41", "ta80"], n_steps=1500, seed=4, noop_force_every=2)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "trace_*.npz"))),
                         ids=lambda p: os.path.basename(p)[6:-4])
def test_gpu_golden_reference_trace(path):
    pc.check_golden_trace(make_env, path)


@pytest.mark.parametrize("inst", sorted(load_json("optimal_sequences.json")))
def test_gpu_facade_optimal_makespan(inst):
    """The reference's 12 known-answer tests (tests/test_solutions.py) through the drop-in facade."""
    pc.check_facade_optimal(inst)


@pytest.mark.parametrize("inst,steps", [("ta01", 400), ("ta51", 300), ("ta80", 300)])
def test_gpu_facade_attributes(inst, steps):
    pc.check_facade_attributes(inst, steps, seed=2)


@pytest.mark.parametrize("inst", ["ta01", "ta41", "dmu16", "ta80"])
def test_gpu_rules_seeded(inst):
    pc.check_rules_seeded(inst)


def test_gpu_policy_kernels():
    pc.check_policy_kernels(make_env, ["ta01", "ta21", "ta31", "ta51", "ta62", "ta80", "dmu18"], n_steps=400, seed=9)


@pytest.mark.parametrize("rule", ["RANDOM", "SPT", "FIFO", "MWR", "LWR", "MOR", "LOR", "CR"])
def test_gpu_rollout_matches_steps(rule):
    pc.check_rollout_matches_steps(make_env, ["ta01", "ta01", "ta31", "ta51", "ta80", "ta80"], rule, n_steps=2600, seed=4)


@pytest.mark.parametrize("rule", ["RANDOM", "SPT", "FIFO", "MWR", "MOR", "LOR", "CR"])
def test_gpu_step_sample_fused(rule):
    pc.check_step_sample(make_env, ["ta01", "ta31", "ta51", "ta80", "ta80"], rule, n_steps=2600, seed=12)


def test_gpu_step_sample_alternating_rules_big_instances():
    """MWR stages the suffix-sum table and FIFO does not, so the fused step kernel runs with two shared-memory layouts.
    With 256-job instances both need more than 48 KB: switching rules back and forth must keep launching, and must
    equal the policy kernel + step kernel (uniform and mixed batches)."""
    big = pc.synthetic_instance(256, 32, seed=31)
    for insts, e2i in (([big], [0] * 16), ([big, "ta01"], [0, 1] * 8)):
        cfg = {"instance_paths": insts, "env_to_instance": e2i}
        a_env = make_env(16, cfg, seed=4, auto_reset=True)
        b_env = make_env(16, cfg, seed=4, auto_reset=True)
        a_env.reset(); b_env.reset()
        act_a = a_env.policy("MWR").clone()
        b_env._step_index = 0
        prev = "MWR"
        for k, rule in enumerate(["MWR", "FIFO"] * 12):
            act_b = b_env.policy(prev)
            assert np.array_equal(pc._np(act_a), pc._np(act_b)), (len(insts), k)
            b_env.step(act_b)
            *_, act_a = a_env.step_sample(act_a, rule)
            for name in ("action_mask", "real_obs", "reward", "done"):
                assert np.array_equal(pc._np(getattr(a_env, name)), pc._np(getattr(b_env, name))), (len(insts), k, name)
            prev = rule


def test_gpu_errors_freeze_reset():
    pc.check_errors_and_freeze(make_env)


def test_gpu_auto_reset_and_stats():
    pc.check_auto_reset_and_stats(make_env, "ta01", seed=6)
    pc.check_auto_reset_and_stats(make_env, "ta51", seed=7)


def test_gpu_snapshot_restore():
    pc.check_snapshot_restore(make_env, "ta31", seed=8)
    pc.check_snapshot_restore(make_env, "ta80", seed=8)


def test_gpu_step_host():
    pc.check_step_host(make_env, "ta01", seed=1)
    pc.check_step_host(make_env, "ta80", seed=1)


def test_gpu_batched_rules_match_oracle_episodes():
    """run_batch (fused rollouts) for every rule: per-env makespan == oracle episode driven by the same RNG."""
    from jssenv_b200.dispatching import DISPATCHING_RULES
    from jssenv_b200.instances import load_instance
    from oracle.jss_oracle import OracleEnv
    names = ["ta01", "ta41", "ta80"]
    env = make_env(3, {"instance_paths": names, "env_to_instance": [0, 1, 2]}, seed=21)
    for rule in DISPATCHING_RULES.values():
        base = env._step_index
        ret, mk = rule.run_batch(env)
        for i, n in enumerate(names):
            o = OracleEnv(*load_instance(n))
            o.reset()
            done, step, total = False, 0, 0
            while not done:
                a, _ = o.rule_action(rule.name, pc._coin_uniform(21, i, base + step))
                _, _, done, _, _ = o.step(a)
                total += o.last_raw_reward
                step += 1
            assert int(mk[i]) == o.current_time_step and int(ret[i]) == total, (rule.name, n)


def test_gpu_large_batch_invariants():
    """BASELINE.json full size (N = 65 536 ta80): size-independent properties.
    Envs driven by the same RNG stream agree; obs in [0,1]; finished episodes satisfy
    sum(raw reward) = 2*sum_op - M*makespan; all ops scheduled at done (tests/test_state.py)."""
    import torch
    n = 65536
    env = make_env(n, {"instance_path": "ta80"}, seed=99, auto_reset=False)
    env.reset()
    sum_op, M = int(env.instance_scalars[0, 2]), env.machines
    for k in range(2700):
        env.step(env.policy("RANDOM"))
        if k % 300 == 0:
            ro = env.real_obs
            assert float(ro.min()) >= 0.0 and float(ro.max()) <= 1.0 and bool(torch.isfinite(ro).all())
            legal = env.action_mask[:, : env.jobs]
            x = env.export_state()
            assert bool((legal == x["legal"].bool()).all())
            assert bool(((legal.sum(1) == 0) == env.done).all())
    st = env.stats()
    assert st["envs_error"] == 0 and st["envs_done"] == n and st["episodes"] == n
    mk, ret = env.last_makespan.long(), env.last_return.long()
    assert bool((ret == 2 * sum_op - M * mk).all())
    x = env.export_state()
    assert bool((x["todo"] == M).all()) and bool((x["tuam"] == 0).all())
    assert st["min_makespan"] == int(mk.min()) and st["max_makespan"] == int(mk.max())
    assert st["sum_makespan"] == int(mk.sum())
    # spot-check 4 envs of the big batch against the oracle replaying the same RNG stream
    from jssenv_b200.instances import load_instance
    from oracle.jss_oracle import OracleEnv
    for i in (0, 1, 4097, n - 1):
        o = OracleEnv(*load_instance("ta80"))
        o.reset()
        done, step = False, 0
        while not done:
            _, _, done, _, _ = o.step(o.masked_random_action(99, i, step))
            step += 1
        assert int(mk[i]) == o.current_time_step


def test_gpu_config2_ta01_n4096_random():
    """BASELINE.json configs[1]: ta01 N = 4096, masked-random policy; every 256th env replayed by the oracle."""
    from jssenv_b200.instances import load_instance
    from oracle.jss_oracle import OracleEnv
    n = 4096
    env = make_env(n, {"instance_path": "ta01"}, seed=31)
    env.reset()
    acts = env.policy("RANDOM").clone()
    for _ in range(400):
        *_, acts = env.step_sample(acts, "RANDOM")
    st = env.stats()
    assert st["envs_done"] == n and st["envs_error"] == 0 and st["episodes"] == n
    mk = env.last_makespan.cpu().numpy()
    ret = env.last_return.cpu().numpy()
    sum_op = int(env.instance_scalars[0, 2])
    assert (ret == 2 * sum_op - 15 * mk).all()
    for i in range(0, n, 256):
        o = OracleEnv(*load_instance("ta01"))
        o.reset()
        done, step = False, 0
        while not done:
            _, _, done, _, _ = o.step(o.masked_random_action(31, i, step))
            step += 1
        assert mk[i] == o.current_time_step, i


def test_gpu_config5_mixed_ta01_ta80_rules():
    """BASELINE.json configs[4]: env i runs ta{(i mod 80)+1}, N = 65 536, on-device FIFO and MWR
    (fused rollouts, device coin).  Episode identity for all envs, oracle replay for a sample."""
    import torch
    from jssenv_b200.dispatching import get_rule
    from jssenv_b200.instances import load_instance
    from oracle.jss_oracle import OracleEnv
    names = ["ta%02d" % (k + 1) for k in range(80)]
    n = 65536
    env = make_env(n, {"instance_paths": names, "env_to_instance": np.arange(n) % 80}, seed=77)
    sc = env.instance_scalars[env.env_to_instance]
    sum_op = torch.as_tensor(sc[:, 2], device=env.device)
    M = torch.as_tensor(env.env_machines.astype(np.int64), device=env.device)
    for rule in ("FIFO", "MWR"):
        base = env._step_index
        ret, mk = get_rule(rule).run_batch(env)
        st = env.stats()
        assert st["envs_done"] == n and st["envs_error"] == 0
        assert bool((ret.long() == 2 * sum_op - M * mk.long()).all()), rule
        for i in (0, 1, 14, 40, 79, 80 * 400 + 50, n - 1):
            o = OracleEnv(*load_instance(names[i % 80]))
            o.reset()
            done, step = False, 0
            while not done:
                a, _ = o.rule_action(rule, pc._coin_uniform(77, i, base + step))
                _, _, done, _, _ = o.step(a)
                step += 1
            assert int(mk[i]) == o.current_time_step, (rule, i)


def test_gpu_host_pipeline():
    pc.check_host_pipeline(make_env, "ta01", seed=3)
    pc.check_host_pipeline(make_env, "ta80", seed=4)


def test_gpu_edge_shapes_and_limits():
    """Kernel limits and ragged shapes, full episodes: J = 1 .. 256, M = 2 .. 32, durations to 2047,
    partially filled lanes, non-permutation machine sequences."""
    shapes = [(1, 2, 9, True), (2, 2, 5, True), (33, 3, 30, True), (65, 5, 99, True), (127, 7, 50, True),
              (128, 32, 2047, True), (32, 32, 200, True), (64, 20, 99, True), (17, 6, 40, False), (100, 20, 99, False),
              (128, 32, 99, False), (96, 31, 700, True),
              (129, 3, 60, True), (200, 10, 99, True), (256, 32, 2047, True), (255, 5, 30, False)]      # 8 jobs per lane
    pc.check_synthetic_shapes(make_env, shapes, n_steps=12000, seed=100)


def test_gpu_abi_error_codes():
    pc.check_abi_error_codes(make_env)


@pytest.mark.parametrize("rule", ["RANDOM", "CR", "FIFO"])
def test_gpu_step_sample_fused_uniform_batch(rule):
    """Uniform batches take the kernel variant that reads the instance scalars from kernel parameters."""
    pc.check_step_sample(make_env, ["ta80"] * 3, rule, n_steps=2600, seed=13)
    pc.check_step_sample(make_env, ["ta01"] * 9, rule, n_steps=600, seed=14)


def test_gpu_facade_errors():
    pc.check_facade_errors()


def test_gpu_dispatching_api():
    pc.check_dispatching_api(make_env)


def test_gpu_soak_auto_reset_full_size():
    """N = 65 536 ta80, 7 000 fused step+sample launches with auto-reset (about three episodes per env):
    no error bits, every finished episode satisfies sum(raw reward) = 2*sum_op - M*makespan, statistics agree."""
    n = 65536
    env = make_env(n, {"instance_path": "ta80"}, seed=2024, auto_reset=True)
    env.reset()
    acts = env.policy("RANDOM").clone()
    sum_op, M = int(env.instance_scalars[0, 2]), env.machines
    for k in range(7000):
        *_, acts = env.step_sample(acts, "RANDOM")
        if k % 1000 == 999:
            mk, ret, cnt = env.last_makespan.long(), env.last_return.long(), env.episode_count
            fin = cnt > 0
            assert bool((ret[fin] == 2 * sum_op - M * mk[fin]).all())
    st = env.stats()
    assert st["envs_error"] == 0 and int(env.episode_count.min()) >= 2
    assert st["episodes"] == int(env.episode_count.sum()) and st["steps"] <= 7000 * n
    assert 5800 <= st["min_makespan"] <= st["max_makespan"] <= 7500      # masked-random ta80 makespans
    ro = env.real_obs
    assert float(ro.min()) >= 0.0 and float(ro.max()) <= 1.0


def test_gpu_tiny_uniform_batches():
    pc.check_tiny_uniform_batches(make_env)


def test_gpu_shard_invariance():
    pc.check_shard_invariance(make_env, n_total=48, n_steps=2400)


def test_gpu_host_pipeline_packed():
    pc.check_host_pipeline_packed(make_env, ["ta01", "ta11", "ta31", "ta51", "ta62", "ta80", "dmu16"] * 9, seed=5, n_steps=600)
    pc.check_host_pipeline_packed(make_env, ["ta80"] * 3, seed=6)


@pytest.mark.parametrize("rule", ["RANDOM", "FIFO"])
def test_gpu_rollout_record(rule):
    pc.check_rollout_record(make_env, ["ta01"] * 5 + ["ta31", "ta51", "ta80", "ta80"], rule, n_steps=2500, seed=3)


def test_gpu_big_uniform_batches():
    pc.check_big_uniform_batches(make_env, max_steps=1500)
