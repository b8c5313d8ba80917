"""The parity tests, declared once for both backends (tests/backends.py) and collected by tests/test_emu_parity.py
and tests/test_gpu_parity.py: the native library, called through the C-ABI, against the CPU oracle and the golden
fixtures recorded from the unmodified Python reference.  The GPU run is the authoritative one, and some full-size
checks run only there; the emulation runs at sizes that keep the CPU suite fast."""
import os

import numpy as np
import pytest

from tests import parity_common as pc
from tests.backends import native_test
from tests.helpers import GOLDEN, golden_traces, load_json

UNIFORM_BATCH_RULES = ["RANDOM", "CR", "FIFO"]
RECORD_RULES = ["RANDOM", "FIFO"]


@native_test(emu=None)
def library_is_the_cuda_one(make_env):
    import torch
    from jssenv_b200 import _native
    assert torch.cuda.is_available()
    assert _native.backend.name == "cuda"
    assert os.path.basename(_native.LIB_PATH) == "libjss_b200.so" and os.path.exists(_native.LIB_PATH)
    env = make_env(2, {"instance_path": "ta01"})
    assert env.real_obs.is_cuda and env.action_mask.is_cuda and env.launch_count >= 1


@native_test(names={"emu": "test_emu_random_mixed_batch_all_lane_classes",
                    "gpu": "test_gpu_random_mixed_batch_all_shapes"})
def random_mixed_batch(make_env, backend):
    # KJ=1 (15, 20, 30 jobs), KJ=2 (50 jobs), KJ=4 (100 jobs), Demirkol (durations to 200)
    pc.check_random_batch(make_env, seed=11, **{
        "emu": dict(names=["ta01", "ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80"],
                    n_steps=400),
        "gpu": dict(names=["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "dmu20", "ta51", "ta61", "ta71", "ta80"] * 3,
                    n_steps=3000, state_every=50)}[backend])


@native_test(names={"emu": "test_emu_full_episode_ta80", "gpu": "test_gpu_full_episodes_ta80_many_envs"})
def full_episodes_ta80(make_env, backend):
    pc.check_random_batch(make_env, n_steps=3000, seed=5, **{"emu": dict(names=["ta80"], state_every=100),
                                                             "gpu": dict(names=["ta80"] * 24, state_every=200)}[backend])


@native_test()
def forced_noops(make_env, backend):
    for args in {"emu": [dict(names=["ta01", "ta45", "ta62", "ta80"], n_steps=500, seed=3, noop_force_every=5)],
                 "gpu": [dict(names=["ta01", "ta15", "ta45", "ta62", "ta80", "dmu17"] * 2, n_steps=1500, seed=3,
                              noop_force_every=5),
                         dict(names=["ta01", "ta41", "ta80"], n_steps=1500, seed=4, noop_force_every=2)]}[backend]:
        pc.check_random_batch(make_env, **args)


@native_test(emu=[pytest.param(t, id="trace_" + t)
                  for t in ("ta01_random0", "ta01_forcednoop3", "ta41_lowest0", "dmu16_random7", "ta80_highest0")],
             gpu=[os.path.basename(p)[6:-4] for p in golden_traces()])
def golden_reference_trace(make_env, trace):
    pc.check_golden_trace(make_env, os.path.join(GOLDEN, f"trace_{trace}.npz"))


@native_test(emu=["ta01", "ta41", "ta51"], gpu=sorted(load_json("optimal_sequences.json")))
def facade_optimal_makespan(inst):
    """The reference's known-answer tests (tests/test_solutions.py) through the drop-in facade."""
    pc.check_facade_optimal(inst)


@native_test(emu=dict(inst="ta01", steps=400), gpu=[("ta01", 400), ("ta51", 300), ("ta80", 300)])
def facade_attributes(inst, steps):
    pc.check_facade_attributes(inst, steps, seed=2)


@native_test(emu=dict(inst="ta01"), gpu=["ta01", "ta41", "dmu16", "ta80"], names={"emu": "test_emu_rules_seeded_ta01"})
def rules_seeded(inst):
    pc.check_rules_seeded(inst)


@native_test()
def policy_kernels(make_env, backend):
    pc.check_policy_kernels(make_env, seed=9, **{
        "emu": dict(names=["ta01", "ta31", "ta51", "ta80"], n_steps=150),
        "gpu": dict(names=["ta01", "ta21", "ta31", "ta51", "ta62", "ta80", "dmu18"], n_steps=400)}[backend])


@native_test(emu=["RANDOM", "FIFO", "MWR", "CR"], gpu=["RANDOM", "SPT", "FIFO", "MWR", "LWR", "MOR", "LOR", "CR"])
def rollout_matches_steps(make_env, backend, rule):
    pc.check_rollout_matches_steps(make_env, rule=rule, seed=4, **{
        "emu": dict(names=["ta01", "ta01", "ta51", "ta80"], n_steps=330),
        "gpu": dict(names=["ta01", "ta01", "ta31", "ta51", "ta80", "ta80"], n_steps=2600)}[backend])


@native_test(emu=["RANDOM", "MWR", "LOR"], gpu=["RANDOM", "SPT", "FIFO", "MWR", "MOR", "LOR", "CR"])
def step_sample_fused(make_env, backend, rule):
    pc.check_step_sample(make_env, rule=rule, seed=12, **{
        "emu": dict(names=["ta01", "ta51", "ta80"], n_steps=300),
        "gpu": dict(names=["ta01", "ta31", "ta51", "ta80", "ta80"], n_steps=2600)}[backend])


@native_test(emu=UNIFORM_BATCH_RULES, gpu=UNIFORM_BATCH_RULES)
def step_sample_fused_uniform_batch(make_env, backend, rule):
    """Uniform batches take the kernel variant that reads the instance scalars from kernel parameters."""
    steps_ta80, steps_ta01 = {"emu": (200, 200), "gpu": (2600, 600)}[backend]
    pc.check_step_sample(make_env, ["ta80"] * 3, rule, n_steps=steps_ta80, seed=13)
    pc.check_step_sample(make_env, ["ta01"] * 9, rule, n_steps=steps_ta01, seed=14)


@native_test(emu=None)
def step_sample_alternating_rules_big_instances(make_env):
    """MWR stages the suffix-sum table and FIFO does not, so the fused step kernel runs with two shared-memory layouts.
    With 256-job instances both need more than 48 KB: switching rules back and forth must keep launching, and must
    equal the policy kernel + step kernel (uniform and mixed batches)."""
    big = pc.synthetic_instance(256, 32, seed=31)
    for batch, names in (("uniform", [big] * 16), ("mixed", [big, "ta01"] * 8)):
        a_env, b_env = pc.twin_envs(make_env, names, sort=False, seed=4, auto_reset=True)
        act_a = a_env.policy("MWR").clone()
        b_env._step_index = 0
        prev = "MWR"
        for k, rule in enumerate(["MWR", "FIFO"] * 12):
            act_b = b_env.policy(prev)
            assert np.array_equal(pc.np_(act_a), pc.np_(act_b)), (batch, k)
            b_env.step(act_b)
            *_, act_a = a_env.step_sample(act_a, rule)
            pc.assert_twins_equal(a_env, b_env, (batch, k))
            prev = rule


@native_test(gpu=None)
def uniform_many_tiles(make_env):
    """Uniform batch with more tiles than (emulated) persistent CTAs, last tile partial."""
    pc.check_step_sample(make_env, ["ta01"] * 70, "RANDOM", n_steps=40, seed=21)
    pc.check_step_sample(make_env, ["ta01"] * 70, "LOR", n_steps=25, seed=22)


@native_test()
def errors_freeze_reset(make_env):
    pc.check_errors_and_freeze(make_env)


@native_test()
def auto_reset_and_stats(make_env, backend):
    for name, seed in {"emu": [("ta01", 6)], "gpu": [("ta01", 6), ("ta51", 7)]}[backend]:
        pc.check_auto_reset_and_stats(make_env, name, seed=seed)


@native_test()
def snapshot_restore(make_env, backend):
    for name in {"emu": ["ta31"], "gpu": ["ta31", "ta80"]}[backend]:
        pc.check_snapshot_restore(make_env, name, seed=8)


@native_test()
def step_host(make_env, backend):
    for name in {"emu": ["ta01"], "gpu": ["ta01", "ta80"]}[backend]:
        pc.check_step_host(make_env, name, seed=1)


@native_test()
def host_pipeline(make_env, backend):
    for name, seed in {"emu": [("ta01", 3)], "gpu": [("ta01", 3), ("ta80", 4)]}[backend]:
        pc.check_host_pipeline(make_env, name, seed=seed)


@native_test()
def host_pipeline_packed(make_env, backend):
    mixed = {"emu": dict(names=["ta01", "ta31", "ta51", "ta80", "dmu16"]),
             "gpu": dict(names=["ta01", "ta11", "ta31", "ta51", "ta62", "ta80", "dmu16"] * 9, n_steps=600)}[backend]
    pc.check_host_pipeline_packed(make_env, seed=5, **mixed)
    pc.check_host_pipeline_packed(make_env, ["ta80"] * 3, seed=6)


@native_test(emu=None)
def batched_rules_match_oracle_episodes(make_env):
    """run_batch (fused rollouts) for every rule: per-env makespan == oracle episode driven by the same RNG."""
    from jssenv_b200.dispatching import DISPATCHING_RULES
    names = ["ta01", "ta41", "ta80"]
    env = make_env(3, {"instance_paths": names, "env_to_instance": [0, 1, 2]}, seed=21)
    for rule in DISPATCHING_RULES.values():
        base = env._step_index
        ret, mk = rule.run_batch(env)
        for i, n in enumerate(names):
            mk_o, ret_o, _ = pc.oracle_episode(
                n, lambda o, step: o.rule_action(rule.name, pc._coin_uniform(21, i, base + step))[0])
            assert int(mk[i]) == mk_o and int(ret[i]) == ret_o, (rule.name, n)


@native_test(emu=None)
def large_batch_invariants(make_env):
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
    for i in (0, 1, 4097, n - 1):
        assert int(mk[i]) == pc.oracle_episode("ta80", lambda o, step: o.masked_random_action(99, i, step))[0]


@native_test(emu=None)
def config2_ta01_n4096_random(make_env):
    """BASELINE.json configs[1]: ta01 N = 4096, masked-random policy; every 256th env replayed by the oracle."""
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
        assert mk[i] == pc.oracle_episode("ta01", lambda o, step: o.masked_random_action(31, i, step))[0], i


@native_test(emu=None)
def config5_mixed_ta01_ta80_rules(make_env):
    """BASELINE.json configs[4]: env i runs ta{(i mod 80)+1}, N = 65 536, on-device FIFO and MWR
    (fused rollouts, device coin).  Episode identity for all envs, oracle replay for a sample."""
    import torch
    from jssenv_b200.dispatching import get_rule
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
            mk_o, _, _ = pc.oracle_episode(
                names[i % 80], lambda o, step: o.rule_action(rule, pc._coin_uniform(77, i, base + step))[0])
            assert int(mk[i]) == mk_o, (rule, i)


@native_test(emu=None)
def soak_auto_reset_full_size(make_env):
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


@native_test(gpu=None)
def gym_vector_adapter_autoreset():
    """next-step autoreset through the VectorEnv-style adapter: the step after `done` returns the reset obs."""
    from jssenv_b200 import JssGymVectorEnv
    env = JssGymVectorEnv(3, {"instance_path": "ta01"}, to_numpy=True, seed=5)
    obs, info = env.reset()
    assert obs["real_obs"].shape == (3, 15, 7) and obs["action_mask"][:, :15].all() and info == {}
    seen_done = np.zeros(3, bool)
    for k in range(600):
        acts = np.array([np.flatnonzero(m)[0] if m.any() else 0 for m in obs["action_mask"]], np.int32)
        prev_done = seen_done.copy()
        obs, rew, done, trunc, info = env.step(acts)
        for i in np.flatnonzero(prev_done & ~done):     # the transition right after a terminal one = reset
            assert obs["action_mask"][i, :15].all() and rew[i] == 0.0 and obs["real_obs"][i, :, 1:].max() == 0.0
        seen_done = done.copy()
        if env.vec.episode_count.min() >= 2:
            break
    assert int(env.vec.episode_count.min()) >= 2
    env.close()


@native_test()
def edge_shapes_and_limits(make_env, backend):
    """Kernel limits and ragged shapes: J = 1 .. 256, M = 2 .. 32, durations to 2047, partially filled lanes,
    non-permutation machine sequences; full episodes on the GPU."""
    shapes = [(1, 2, 9, True), (2, 2, 5, True), (33, 3, 30, True), (65, 5, 99, True), (127, 7, 50, True),
              (128, 32, 2047, True), (32, 32, 200, True), (64, 20, 99, True), (17, 6, 40, False), (100, 20, 99, False)]
    big = [(129, 3, 60, True), (200, 10, 99, True), (256, 32, 2047, True), (255, 5, 30, False)]   # 8 jobs per lane
    pc.check_synthetic_shapes(make_env, seed=100, **{
        "emu": dict(shapes=shapes + big, n_steps=260),
        "gpu": dict(shapes=shapes + [(128, 32, 99, False), (96, 31, 700, True)] + big, n_steps=12000)}[backend])


@native_test()
def abi_error_codes(make_env):
    pc.check_abi_error_codes(make_env)


@native_test()
def facade_errors():
    pc.check_facade_errors()


@native_test()
def dispatching_api(make_env):
    pc.check_dispatching_api(make_env)


@native_test()
def tiny_uniform_batches(make_env):
    pc.check_tiny_uniform_batches(make_env)


@native_test()
def shard_invariance(make_env, backend):
    pc.check_shard_invariance(make_env, **{"emu": dict(n_steps=150), "gpu": dict(n_total=48, n_steps=2400)}[backend])


@native_test(emu=RECORD_RULES, gpu=RECORD_RULES)
def rollout_record(make_env, backend, rule):
    pc.check_rollout_record(make_env, rule=rule, seed=3, **{
        "emu": dict(names=["ta01", "ta01", "ta51", "ta80"], n_steps=300),
        "gpu": dict(names=["ta01"] * 5 + ["ta31", "ta51", "ta80", "ta80"], n_steps=2500)}[backend])


@native_test()
def big_uniform_batches(make_env, backend):
    pc.check_big_uniform_batches(make_env, max_steps={"emu": 60, "gpu": 1500}[backend])
