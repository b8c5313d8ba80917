"""The tests of jss_step_logits (masked categorical draw from policy logits fused into the step), declared once for
both backends (tests/backends.py) and collected by tests/test_emu_step_logits.py and tests/test_gpu_step_logits.py:
the checks of tests/logits_common.py at GPU sizes and at CPU-friendly sizes under the host emulation of the kernels,
and on the GPU also the distribution of the draw and its repeatability."""
import numpy as np

from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import synthetic_instance


@native_test()
def step_logits_mixed_batch(make_env, backend):
    # every lane class of the mixed step kernel; the ta01 envs finish (and auto-reset) within the window
    lc.check_step_logits(make_env, seed=3, **{
        "emu": dict(names=["ta01", "ta01", "ta51", "ta80", "dmu16"], n_steps=330),
        "gpu": dict(names=["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80"] * 3,
                    n_steps=1200, state_every=100)}[backend])


@native_test()
def step_logits_uniform_ta01(make_env, backend):
    lc.check_step_logits(make_env, seed=4, **{"emu": dict(names=["ta01"] * 9, n_steps=300),
                                              "gpu": dict(names=["ta01"] * 300, n_steps=700, state_every=100)}[backend])


@native_test()
def step_logits_uniform_ta80(make_env, backend):
    # on the GPU through the end of the first episodes (about 2 236 transitions)
    lc.check_step_logits(make_env, seed=5, pad=0, **{
        "emu": dict(names=["ta80"] * 3, n_steps=150),
        "gpu": dict(names=["ta80"] * 40, n_steps=2600, state_every=200)}[backend])


@native_test()
def step_logits_big_instances(make_env, backend):
    # 129..256 jobs: the 8-jobs-per-lane bodies of the uniform and the mixed step kernels
    if backend == "emu":
        big = synthetic_instance(200, 6, 7, max_dur=40)
        lc.check_step_logits(make_env, [big] * 2, n_steps=60, seed=6)
        lc.check_step_logits(make_env, [big, "ta01"], n_steps=60, seed=7)
    else:
        big = synthetic_instance(200, 8, 9, max_dur=50)
        lc.check_step_logits(make_env, [big] * 9, n_steps=400, seed=6, state_every=100)
        lc.check_step_logits(make_env, [big, "ta01", "ta51", "ta80"] * 2, n_steps=400, seed=7, state_every=100)


@native_test()
def step_logits_edge_cases(make_env):
    lc.check_step_logits_edge_cases(make_env)


@native_test()
def step_logits_shard_invariance(make_env, backend):
    lc.check_step_logits_shards(make_env, **{"emu": dict(n_steps=80), "gpu": dict(n_total=60, n_steps=600)}[backend])


@native_test()
def step_logits_abi_errors(make_env):
    lc.check_step_logits_abi_errors(make_env)


@native_test(emu=None)
def step_logits_distribution(make_env):
    """ta01 at N = 65 536 right after reset (every job legal, the no-op not), one shared logits row, one call: the
    histogram of the drawn actions against the masked softmax, and every log_prob against log_softmax."""
    import torch
    from scipy.stats import chisquare
    n = 65536
    env = make_env(n, {"instance_path": "ta01"}, seed=11)
    env.reset()
    J = env.jobs
    row = torch.randn(J + 1, generator=torch.Generator().manual_seed(0)).to(env.device)
    _, _, _, _, info = env.step_logits(row.expand(n, J + 1))   # stride-0 rows: made contiguous by step_logits
    acts = info["actions"].cpu().numpy()
    assert acts.min() >= 0 and acts.max() < J
    logp = torch.log_softmax(row[:J].double(), 0).cpu().numpy()
    hist = np.bincount(acts, minlength=J)
    res = chisquare(hist, np.exp(logp) * n)
    assert res.pvalue > 1e-6, (res, hist)
    assert np.abs(info["log_prob"].cpu().numpy() - logp[acts]).max() <= 1e-5 * (1 + np.abs(logp).max())


@native_test(emu=None)
def step_logits_repeatable(make_env):
    """Same seed, same step index, same logits: identical actions and log_probs, whether from a second env or from
    the same env after a reset."""
    import torch
    names = ["ta01", "ta41", "ta80"]
    n = 3 * 1365
    cfg = {"instance_paths": names, "env_to_instance": np.arange(n) % 3}
    a_env, b_env = make_env(n, cfg, seed=21), make_env(n, cfg, seed=21)
    a_env.reset(); b_env.reset()
    logits = torch.randn((n, a_env.jobs + 1), generator=torch.Generator().manual_seed(1)).to(a_env.device)
    runs = []
    for env in (a_env, b_env, a_env):
        env.reset()
        env._step_index = 7
        _, _, _, _, info = env.step_logits(logits)
        runs.append((info["actions"].cpu().numpy(), info["log_prob"].cpu().numpy().view(np.uint32)))
    for acts, lp in runs[1:]:
        assert np.array_equal(acts, runs[0][0]) and np.array_equal(lp, runs[0][1])
