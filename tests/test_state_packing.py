"""The per-env state block keeps the five per-job integers in 10 bytes (jss_types.h): todo in 6 bits, tufco and col4
in 11 bits each, idle_last and total_idle in 24 bits each.  These tests push every field to the edges of its range
through jss_import_state / jss_export_state, and check that values outside the range are flagged instead of wrapped.
Each check runs on both backends of tests/backends.py."""
import numpy as np

from tests import parity_common as pc
from tests.backends import collect, native_test

JSS_FLAG_ERROR = 2
IDLE_MAX = (1 << 24) - 1
DUR_MAX = 2047
JOB_FIELDS = ("todo", "tufco", "col4", "idle_last", "total_idle")
SHAPES = [(256, 32), (100, 20)]      # the largest supported shape (8 jobs per lane) and ta80's shape (4 per lane)


def _field_max(name, M):
    return {"todo": M, "tufco": DUR_MAX, "col4": DUR_MAX, "idle_last": IDLE_MAX, "total_idle": IDLE_MAX}[name]


def _snapshot(env):
    return {k: v.clone() for k, v in env.export_state().items()}


def _set_row(x, name, i, J, values):
    import torch
    x[name][i, :J] = torch.as_tensor(np.asarray(values, np.int32)).to(x[name].device)


@native_test()
def state_roundtrip_at_field_limits(make_env):
    """export -> import -> export returns every field unchanged, with every field at its maximum on some jobs, at 0
    on others, and random in-range values elsewhere (a field bleeding into its neighbour changes the result)."""
    insts = [pc.synthetic_instance(J, M, seed=70 + k, max_dur=DUR_MAX) for k, (J, M) in enumerate(SHAPES)]
    n = 2 * len(insts)
    env = make_env(n, {"instance_paths": insts, "env_to_instance": [i % len(insts) for i in range(n)]})
    env.reset()
    x = _snapshot(env)
    rng = np.random.default_rng(5)
    want = {}
    for i in range(n):
        J, M = SHAPES[i % len(SHAPES)]
        for name in JOB_FIELDS:
            hi = _field_max(name, M)
            v = rng.integers(0, hi + 1, size=J)
            if i < len(SHAPES):
                v[:] = hi                          # env 0 / 1: every job at the maximum of every field
            else:
                v[::7] = hi                        # env 2 / 3: maxima, zeros and random values interleaved
                v[3::7] = 0
            _set_row(x, name, i, J, v)
            want[(i, name)] = v
    env.import_state(x)
    y = {k: pc.np_(v).copy() for k, v in env.export_state().items()}
    env.synchronize()
    for (i, name), v in want.items():
        J = SHAPES[i % len(SHAPES)][0]
        assert np.array_equal(y[name][i, :J], v), (i, name)
    assert not ((y["flags"] >> 8) & JSS_FLAG_ERROR).any()
    xt = {k: pc.np_(v) for k, v in x.items()}
    for name in ("tuam", "legal", "blocked", "t"):
        assert np.array_equal(y[name], xt[name]), name


@native_test()
def out_of_range_import_flagged(make_env):
    """A value outside its field's range gives the env the sticky error bit and is clamped into the range; the
    other envs of the batch are imported as they are."""
    J, M = SHAPES[1]
    inst = pc.synthetic_instance(J, M, seed=71, max_dur=DUR_MAX)
    cases = []
    for name in JOB_FIELDS:
        hi = _field_max(name, M)
        cases += [(name, -1, 0), (name, hi + 1, hi), (name, -(1 << 31), 0), (name, (1 << 31) - 1, hi)]
    n = len(cases) + 1                             # env 0 stays in range
    env = make_env(n, {"instance_paths": [inst], "env_to_instance": [0] * n})
    env.reset()
    x = _snapshot(env)
    rng = np.random.default_rng(6)
    base = {name: rng.integers(0, _field_max(name, M) + 1, size=J) for name in JOB_FIELDS}
    for i in range(n):
        for name in JOB_FIELDS:
            _set_row(x, name, i, J, base[name])
    for k, (name, bad, _) in enumerate(cases):
        v = base[name].copy()
        v[J - 1 - k % 4] = bad                     # a job slot of the last lanes, different ones across cases
        _set_row(x, name, k + 1, J, v)
    env.import_state(x)
    y = {k: pc.np_(v).copy() for k, v in env.export_state().items()}
    env.synchronize()
    err = (y["flags"] >> 8) & JSS_FLAG_ERROR
    assert err[0] == 0
    for name in JOB_FIELDS:
        assert np.array_equal(y[name][0, :J], base[name]), name
    for k, (name, bad, clamped) in enumerate(cases):
        i = k + 1
        assert err[i] != 0, (name, bad)
        v = base[name].copy()
        v[J - 1 - k % 4] = clamped
        assert np.array_equal(y[name][i, :J], v), (name, bad)


collect(globals(), globals(), "emu", "gpu")
