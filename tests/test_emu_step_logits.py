"""jss_step_logits (masked categorical draw from policy logits fused into the step) under HOST EMULATION of the CUDA
kernels (tests/emu): the same checks as tests/test_gpu_step_logits.py at CPU-friendly sizes."""
import pytest

from tests import logits_common as lc
from tests.emu.emu_backend import use_emulation
from tests.parity_common import synthetic_instance


@pytest.fixture(autouse=True)
def _emu():
    with use_emulation():
        yield


def make_env(n, cfg, **kw):
    from jssenv_b200 import JssVecEnv
    return JssVecEnv(n, cfg, **kw)


def test_emu_step_logits_mixed_batch():
    # every lane class of the mixed step kernel; the ta01 envs finish (and auto-reset) within the window
    lc.check_step_logits(make_env, ["ta01", "ta01", "ta51", "ta80", "dmu16"], n_steps=330, seed=3)


def test_emu_step_logits_uniform_ta01():
    lc.check_step_logits(make_env, ["ta01"] * 9, n_steps=300, seed=4)


def test_emu_step_logits_uniform_ta80():
    lc.check_step_logits(make_env, ["ta80"] * 3, n_steps=150, seed=5, pad=0)


def test_emu_step_logits_big_instances():
    # 129..256 jobs: the 8-jobs-per-lane bodies of the uniform and the mixed step kernels
    big = synthetic_instance(200, 6, 7, max_dur=40)
    lc.check_step_logits(make_env, [big] * 2, n_steps=60, seed=6)
    lc.check_step_logits(make_env, [big, "ta01"], n_steps=60, seed=7)


def test_emu_step_logits_edge_cases():
    lc.check_step_logits_edge_cases(make_env)


def test_emu_step_logits_shard_invariance():
    lc.check_step_logits_shards(make_env, n_steps=80)


def test_emu_step_logits_abi_errors():
    lc.check_step_logits_abi_errors(make_env)
