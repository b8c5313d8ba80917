"""Numeric edges of the draws from a caller's fp32 logits (jss_step_logits, jss_step_logits_record and
jss_rollout_priority_sample), declared once for both backends (tests/backends.py) and collected by
tests/test_emu_sampling_edges.py and tests/test_gpu_sampling_edges.py:

- shifting every logit by one constant changes nothing, bit for bit: the draw, log_prob, the gradient and the env;
- tied logits at +-1e30 and +-FLT_MAX, one legal logit at FLT_MAX among -FLT_MAX, and spreads past exp's range draw
  what the float64 oracle draws (on the GPU: uniformly over the tied actions, at N = 65 536), without a NaN;
- with two finite logits x0 and x0 + d, the second is drawn with probability sigmoid(d), at offsets 0 and 2^20.

A draw keyed on logit + g in fp32 fails all three once the logits are large: the ulp of the logit swallows the noise g,
the keys tie and the lowest index wins, while log_prob still describes the softmax."""
import numpy as np

from jssenv_b200 import _native as N
from tests import logits_common as lc
from tests.backends import native_test
from tests.parity_common import assert_twins_equal, np_, synthetic_instance, twin_envs
from tests.priority_sample_suite import Twin, assert_grad, assert_log_prob, sample_call
from tests.priority_suite import BIG_GPU, EMU_CLASSES, NONPERM, assert_same

FLT_MAX = float(np.finfo(np.float32).max)
# |c| <= 2^20 keeps x + c exact for x on the 1/8 grid of [-8, 8] (24 significant bits), and then
# (x + c) - (mx + c) = x - mx exactly (Sterbenz): the shifted draw must be the unshifted one
SHIFTS = np.float32([2.0 ** 10, -2.0 ** 10, 2.0 ** 16, -2.0 ** 16, 2.0 ** 20, -2.0 ** 20])
U32 = np.uint32

# every lane class of the step kernels (1, 2, 4 and 8 jobs per lane); the ta01 envs finish (and auto-reset)
STEP_BATCH = {"emu": (["ta01", "ta01", "ta51", "ta80", "dmu16", synthetic_instance(200, 6, 7, max_dur=40)], 330),
              "gpu": (["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80",
                       synthetic_instance(200, 8, 9, max_dur=50)] * 3, 1200)}
# every lane class of the rollout kernel, a non-permutation instance included
ROLLOUT_BATCH = {"emu": ["ta01", "ta01", *EMU_CLASSES, NONPERM],
                 "gpu": ["ta01", "ta11", "ta21", "ta31", "ta41", "dmu16", "ta51", "ta61", "ta71", "ta80", NONPERM,
                         BIG_GPU] * 3}


def grid_logits(rng, shape, p_ninf=0.1):
    """Seeded logits on the 1/8 grid of [-8, 8], -inf at random (p_ninf)."""
    x = (rng.integers(-64, 65, size=shape) / 8).astype(np.float32)
    x[rng.random(shape) < p_ninf] = -np.inf
    return x


def row_shifts(n, k):
    """Env i's shift at step k: every env goes through every shift, and a batch mixes them."""
    return SHIFTS[(np.arange(n) + k) % len(SHIFTS)]


def assert_same_draw(info_a, info_b, ctx):
    assert np.array_equal(np_(info_a["actions"]), np_(info_b["actions"])), ctx
    assert np.array_equal(np_(info_a["log_prob"]).view(U32), np_(info_b["log_prob"]).view(U32)), ctx


# ---- a. exact shift invariance --------------------------------------------------------------------------------------
@native_test()
def shift_invariance_step_logits(make_env, backend):
    """step_logits on grid logits and on the same logits shifted per env by +-2^10, +-2^16 or +-2^20: the same
    actions and log_probs bit for bit, and twin envs bit-identical after every step."""
    names, n_steps = STEP_BATCH[backend]
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=3, auto_reset=True)
    n, ld = a_env.num_envs, a_env.jobs + 4
    rng = np.random.default_rng(3)
    for k in range(n_steps):
        x = grid_logits(rng, (n, ld))
        _, _, _, _, info_a = a_env.step_logits(lc._to_dev(a_env, x))
        _, _, _, _, info_b = b_env.step_logits(lc._to_dev(b_env, x + row_shifts(n, k)[:, None]))
        assert_same_draw(info_a, info_b, k)
        full = k % 50 == 49
        assert_twins_equal(a_env, b_env, k, state=full, stats=full)
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)


@native_test()
def shift_invariance_step_logits_record(make_env, backend):
    """step_logits_record on grid logits and on shifted ones: identical slots, draws and envs."""
    names, n_steps = STEP_BATCH[backend]
    a_env, b_env = twin_envs(make_env, names, sort=False, seed=4, auto_reset=True)
    n, ld, traj_len = a_env.num_envs, a_env.jobs + 1, 16
    rng = np.random.default_rng(4)
    ta = tb = None
    for k in range(n_steps):
        slot = k % traj_len
        if slot == 0:
            ta, tb = a_env.logits_trajectory(traj_len, out=ta), b_env.logits_trajectory(traj_len, out=tb)
        x = grid_logits(rng, (n, ld))
        _, _, _, _, info_a = a_env.step_logits_record(lc._to_dev(a_env, x), ta, slot)
        _, _, _, _, info_b = b_env.step_logits_record(lc._to_dev(b_env, x + row_shifts(n, k)[:, None]), tb, slot)
        assert_same_draw(info_a, info_b, k)
        if slot == traj_len - 1 or k == n_steps - 1:
            for name, v in ta.items():
                bits = [np.ascontiguousarray(np_(t)).view(np.uint8) for t in (v, tb[name])]
                assert np.array_equal(*bits), (k, name)
    a_env.refresh_obs(); b_env.refresh_obs()
    assert_twins_equal(a_env, b_env, "end", state=True, stats=True)


@native_test()
def shift_invariance_priority_sample(make_env, backend):
    """rollout_priority_sample on a grid (N, J, M) table shifted per env, and on a broadcast (1, J, M) table shifted
    by each constant, to the end of the episodes: the same state, log_prob and gradient, bit for bit."""
    import torch
    names = ROLLOUT_BATCH[backend]
    rng = np.random.default_rng(5)
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    n, J, M = a_env.num_envs, a_env.jobs, a_env.machines
    table = grid_logits(rng, (n, J, M), p_ninf=0.001)
    shifted = table + row_shifts(n, 0)[:, None, None]
    for k in (40, None):                                  # a partial call, then to the end
        lp_a, g_a = sample_call(a_env, lc._to_dev(a_env, table), k)
        lp_b, g_b = sample_call(b_env, lc._to_dev(b_env, shifted), k)
        assert_same(a_env, b_env, ("table", k))
        assert np.array_equal(lp_a.view(U32), lp_b.view(U32)), ("table", k)
        assert np.array_equal(g_a.view(U32), g_b.view(U32)), ("table", k)
    done, err = np_(a_env.done), (np_(a_env.flags) & N.FLAG_ERROR) != 0   # an env whose legal entries are all -inf errs
    assert (done | err).all() and done.sum() > len(names) // 2, (done, err)
    shared = grid_logits(rng, (1, J, M), p_ninf=0.001)
    a_env, _ = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    lp_a, g_a = sample_call(a_env, torch.from_numpy(shared).to(a_env.device))
    for c in SHIFTS:
        _, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
        lp_b, g_b = sample_call(b_env, torch.from_numpy(shared + c).to(b_env.device))
        assert_same(a_env, b_env, ("broadcast", c))
        assert np.array_equal(lp_a.view(U32), lp_b.view(U32)), ("broadcast", c)
        assert np.array_equal(g_a.view(U32), g_b.view(U32)), ("broadcast", c)


# ---- b. tied and extreme magnitudes ---------------------------------------------------------------------------------
TIES = (1e30, -1e30, FLT_MAX, -FLT_MAX)
SPREAD = np.array([0.0, 0.5, 1.0, 2.0, 3.0, 89.0, 104.0, 200.0, 1000.0])   # below the largest: exp(-89) is 0 in fp32


def extreme_logits(rng, env, mask, ld, k):
    """Env i's legal logits at step k by case (i + k) % 6: all equal at 1e30, -1e30, FLT_MAX or -FLT_MAX; one at
    FLT_MAX and the rest at -FLT_MAX (x - mx overflows to -inf); a spread past exp's range below 0 or 1e4.  NaN on the
    illegal entries and in the padding (never read)."""
    x = np.full((env.num_envs, ld), np.nan, np.float32)
    for i, Ji in enumerate(env.env_jobs):
        legal = np.flatnonzero(mask[i, : Ji + 1])
        case = (i + k) % 6
        if case < 4:
            x[i, legal] = TIES[case]
        elif case == 4:
            x[i, legal] = -FLT_MAX
            if len(legal):
                x[i, rng.choice(legal)] = FLT_MAX
        else:
            x[i, legal] = rng.choice([0.0, 1e4]) - rng.choice(SPREAD, size=len(legal))
    return x


def extreme_table(rng, n, J, M):
    """Env i's (J, M) table by case i % 6: every entry 1e30, -1e30, FLT_MAX or -FLT_MAX; FLT_MAX on a tenth of the
    entries and -FLT_MAX elsewhere; a spread past exp's range below 0 or 1e4."""
    t = np.empty((n, J, M), np.float32)
    for i in range(n):
        case = i % 6
        if case < 4:
            t[i] = TIES[case]
        elif case == 4:
            t[i] = np.where(rng.random((J, M)) < 0.1, FLT_MAX, -FLT_MAX)
        else:
            t[i] = rng.choice([0.0, 1e4]) - rng.choice(SPREAD, size=(J, M))
    return t


@native_test()
def extreme_step_logits(make_env, backend):
    """step_logits on tied, overflowing and wide-spread logits (extreme_logits): every draw against the float64
    oracle, log_prob within its tolerance (so never NaN), twin envs stepped with the drawn actions bit-identical."""
    names, n_steps = STEP_BATCH[backend]
    lc.check_step_logits(make_env, names, n_steps, seed=6, state_every=100, make_logits=extreme_logits)


@native_test()
def extreme_priority_sample(make_env, backend):
    """rollout_priority_sample to the end of the episodes on tied, overflowing and wide-spread tables
    (extreme_table): the step_logits twin's every draw against the float64 oracle, and the call equal to the twin,
    log_prob bit for bit and the gradient within tolerance, neither of them NaN."""
    names = ROLLOUT_BATCH[backend]
    a_env, b_env = twin_envs(make_env, names, sort=False, auto_reset=False, record_solution=True)
    n, J, M = a_env.num_envs, a_env.jobs, a_env.machines
    table = extreme_table(np.random.default_rng(7), n, J, M)
    lp, g = sample_call(a_env, lc._to_dev(a_env, table))
    seen = {"decisions": 0}

    def check(rows, mask, done, acts, log_prob, counter):
        _, d, agree = lc.check_draws(b_env, rows, mask, done, acts, log_prob, counter, np_(b_env.flags), counter)
        assert agree == d, (counter, agree, d)
        seen["decisions"] += d

    twin = Twin(b_env)
    twin.steps(table, 2 * J * M + 1, 0, check)
    assert np_(a_env.done).all() and not (np_(a_env.flags) & N.FLAG_ERROR).any()
    assert seen["decisions"] >= sum(int(j) * int(m) for j, m in zip(a_env.env_jobs, a_env.env_machines))
    assert_same(a_env, b_env, "extreme")
    assert not np.isnan(lp).any(), lp
    assert_log_prob(lp, twin.call["log_prob"], "extreme")
    assert_grad(a_env, g, twin.call, "extreme")


@native_test(emu=None)
def tied_draws_uniform(make_env):
    """ta01 at N = 65 536 from reset (15 jobs legal, the no-op not), every logit equal at +-1e30 or +-FLT_MAX: the
    jobs drawn by step_logits and by rollout_priority_sample(table, 1) are uniform (chi-square), and every log_prob is
    -log 15."""
    import torch
    from scipy.stats import chisquare
    n = 65536
    env = make_env(n, {"instance_path": "ta01"}, seed=13, auto_reset=False)
    J, M = env.jobs, env.machines
    for v in TIES:
        for entry in ("step_logits", "rollout_priority_sample"):
            env.reset()
            if entry == "step_logits":
                _, _, _, _, info = env.step_logits(torch.full((J + 1,), v, device=env.device).expand(n, J + 1))
                acts = np_(info["actions"])
            else:
                _, _, _, _, info = env.rollout_priority_sample(torch.full((1, J, M), v, device=env.device), 1)
                running = np_(env.export_state()["tufco"]) > 0
                assert (running.sum(1) == 1).all(), (v, entry)
                acts = running.argmax(1)
            assert acts.min() >= 0 and acts.max() < J, (v, entry)
            hist = np.bincount(acts, minlength=J)
            res = chisquare(hist)
            assert res.pvalue > 1e-6, (v, entry, res, hist)
            assert np.abs(np_(info["log_prob"]) + np.log(J)).max() <= 1e-5 * (1 + np.log(J)), (v, entry)


# ---- c. calibration of the noise ------------------------------------------------------------------------------------
D_GRID = np.arange(-64, 65) / 8


def calibration_chi2(d, second):
    """(statistic, degrees of freedom, p-value) of the draws of the second action against sigmoid(d): one binomial
    z-score per value of d with n p (1 - p) >= 4, one per sign of d for the other values pooled, their squares
    summed."""
    from scipy.stats import chi2
    vals, inv = np.unique(d, return_inverse=True)
    cnt, hit = np.bincount(inv), np.bincount(inv, weights=second)
    p = 1.0 / (1.0 + np.exp(-vals))
    mean, var = cnt * p, cnt * p * (1.0 - p)
    big = var >= 4.0
    terms = list((hit[big] - mean[big]) ** 2 / var[big])
    for side in (vals < 0, vals > 0):
        m = side & ~big
        if m.any():
            terms.append((hit[m].sum() - mean[m].sum()) ** 2 / var[m].sum())
    stat = float(sum(terms))
    return stat, len(terms), float(chi2.sf(stat, len(terms)))


@native_test(emu={"n": len(D_GRID) * 16}, gpu={"n": 65536})
def two_way_calibration(make_env, n):
    """ta01 from reset, env i with exactly two finite logits, x0 on job j1 and x0 + d_i on job j2 (a seeded pair, d_i
    on the 1/8 grid of [-8, 8]), every other job at -inf: the share of envs that draw j2 follows sigmoid(d) (per-d
    binomial z-scores in one chi-square, p > 1e-6) and log_prob is log sigmoid(+-d), at x0 = 0 and 2^20, for
    step_logits and for one decision of rollout_priority_sample.  Each draw weighs two Gumbel variates, so both
    branches of jss_gumbel (log for u < 1/2, log1p above) meet in the difference."""
    env = make_env(n, {"instance_path": "ta01"}, seed=17, auto_reset=False)
    J, M = env.jobs, env.machines
    rng = np.random.default_rng(17)
    d = D_GRID[np.arange(n) % len(D_GRID)]
    j1, j2 = np.argsort(rng.random((n, J)), axis=1)[:, :2].T
    envs = np.arange(n)
    for x0 in (0.0, 2.0 ** 20):
        x = np.full((n, J + 1), -np.inf, np.float32)
        x[envs, j1] = x0
        x[envs, j2] = x0 + d                              # exact: d is on the 1/8 grid
        for entry in ("step_logits", "rollout_priority_sample"):
            env.reset()
            if entry == "step_logits":
                _, _, _, _, info = env.step_logits(lc._to_dev(env, x))
                acts = np_(info["actions"])
            else:
                table = np.full((n, J, M), -np.inf, np.float32)
                table[:, :, 0] = x[:, :J]                  # every job's current operation is its first
                _, _, _, _, info = env.rollout_priority_sample(lc._to_dev(env, table), 1)
                running = np_(env.export_state()["tufco"]) > 0
                assert (running.sum(1) == 1).all(), (x0, entry)
                acts = running.argmax(1)
            second = acts == j2
            assert (second | (acts == j1)).all(), (x0, entry)
            want = -np.logaddexp(0.0, np.where(second, -d, d))   # log sigmoid(d) for j2, log sigmoid(-d) for j1
            lp = np_(info["log_prob"]).astype(np.float64)
            assert np.abs(lp - want).max() <= 1e-5 * (1 + np.abs(want).max()), (x0, entry)
            stat, df, p = calibration_chi2(d, second)
            assert p > 1e-6, (x0, entry, stat, df)
