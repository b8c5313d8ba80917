"""real_obs and the scaled reward against their exact values, declared once for both backends (tests/backends.py) and
collected by tests/test_emu_exact_obs.py and tests/test_gpu_exact_obs.py.

Every observation entry is a quotient of two integers: column 1 tufco / max_time_op, 2 todo / M, 3 (t - total_idle, or
jobs_length once todo = M) / max_time_jobs, 4 col4 / max_time_op, 5 idle_last / sum_op, 6 total_idle / sum_op; the
scaled reward is raw / max_time_op.  The kernels claim the correctly rounded fp32 quotient (jss_div).  The reference
for it is np.float32(np.float64(x) / y): a float64 quotient of integers below 2^24 is correctly rounded, and rounding
it once more to fp32 cannot err (53 >= 2 * 24 + 2).  reference_is_correctly_rounded checks that argument against exact
rational rounding instead of relying on it.

The divide sweeps write their numerators straight into the state through import_state, over every divisor the limits
allow for max_time_op and M and at the edges of the ranges of max_time_jobs and sum_op, and read the entries back from
every path that emits a row: the import itself (the generic kernel), refresh_obs after a recording step, and the
packed host rows expanded by the scalar, AVX2 and AVX-512 code.  The serialised episodes put every operation on
machine 0, so that time, idle_last and total_idle run up to sum_op = 256 * 32 * 2047 = 2^24 - 8192, the largest the
24-bit fields of the state block have to hold."""
import fractions

import numpy as np

from jssenv_b200 import _native as N
from oracle.jss_oracle import OracleEnv
from tests.backends import native_test
from tests.parity_common import assert_obs_exact, batch_cfg, compare_env_to_oracle, compare_exported_state, np_

MAX_DUR = 2047
MAX_SUM_OP = 256 * 32 * MAX_DUR                  # 16 769 024 = 2^24 - 8192
FROZEN = (N.FLAG_DONE << 8) | 1                  # an imported env marked done: no step changes it


def _is_prime(n):
    return n > 1 and all(n % p for p in range(2, int(n ** 0.5) + 1))


def _prime_below(n):
    while not _is_prime(n):
        n -= 1
    return n


def _prime_above(n):
    while not _is_prime(n):
        n += 1
    return n


MAX_TIME_JOBS = [32 * MAX_DUR, 32 * MAX_DUR - 1, 2 ** 15 - 1, 49151, 2 ** 15, 2 ** 15 + 1,
                 _prime_below(32 * MAX_DUR), _prime_above(2 ** 15 + 2), _prime_below(40000)]
SUM_OP = [MAX_SUM_OP, 2 ** 23 - 1, 2 ** 23, 2 ** 23 + 1, 3 * 2 ** 22,
          _prime_below(MAX_SUM_OP), _prime_below(2 ** 23 - 2), _prime_above(2 ** 23 + 2)]


def exact_f32(x, y):
    """The reference's entry: one float64 division of two integers, rounded once to fp32."""
    return (np.asarray(x, np.float64) / np.asarray(y, np.float64)).astype(np.float32)


def rounded_f32(x, y):
    """x / y rounded to the nearest fp32, ties to even, by exact rational arithmetic (|x| < 2^25, 0 < y < 2^25)."""
    q = fractions.Fraction(abs(int(x)), int(y))
    if q == 0:
        return np.float32(0.0)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if q < fractions.Fraction(2) ** e:
        e -= 1                                    # now 2^e <= q < 2^(e+1)
    m = q * fractions.Fraction(2) ** (23 - e)     # in [2^23, 2^24)
    r = int(m)
    if m - r > fractions.Fraction(1, 2) or (m - r == fractions.Fraction(1, 2) and r % 2):
        r += 1
    v = np.float32(r * 2.0 ** (e - 23))           # exact: r <= 2^24
    return -v if x < 0 else v


def _spread(total, n):
    """n positive integers no larger than MAX_DUR that add up to `total`, as equal as possible."""
    base, rem = divmod(int(total), n)
    d = np.full(n, base, np.int32)
    d[:rem] += 1
    assert 1 <= d.min() and d.max() <= MAX_DUR, (total, n)
    return d


def _instance(rng, J, M, durations):
    machine = np.stack([rng.permutation(M) for _ in range(J)]).astype(np.int32)
    return machine, np.asarray(durations, np.int32).reshape(J, M)


def _near_midpoints(y, k):
    """The k numerators in [1, y] whose quotients by y lie closest to a midpoint between two fp32 values: where a
    divide that is off by the least amount, such as one with a reciprocal one ulp low, rounds the wrong way."""
    best = []
    for a in range(1, y + 1, 1 << 22):
        x = np.arange(a, min(y + 1, a + (1 << 22)), dtype=np.float64)
        m = np.ldexp(x / y, (23 - np.floor(np.log2(x / y))).astype(np.int64))     # the 24-bit significand, unrounded
        d = np.abs(m - np.floor(m) - 0.5)
        keep = np.argsort(d)[:k]
        best.append(np.stack([d[keep], x[keep]]))
    best = np.concatenate(best, 1)
    return best[1, np.argsort(best[0])[:k]].astype(np.int64)


def _numerators(rng, y, edge, n_random, n_hard, slots):
    """The n_hard numerators nearest a rounding midpoint, every numerator in [0, edge] and in [y - edge, y], and
    n_random uniform ones in [0, y], repeated to fill `slots`."""
    x = np.concatenate([_near_midpoints(y, n_hard), np.arange(0, min(edge, y) + 1),
                        np.arange(max(0, y - edge), y + 1), rng.integers(0, y + 1, n_random)])
    assert len(x) <= slots, (len(x), slots)
    return np.resize(x, slots)


class Planted:
    """A batch whose envs all have J jobs, into whose state import_state writes chosen integers."""

    def __init__(self, make_env, insts, env_to_instance):
        self.env = make_env(len(env_to_instance), {"instance_paths": insts, "env_to_instance": env_to_instance})
        e = self.env
        self.J = int(e.jobs)
        assert (e.env_jobs == self.J).all()
        sc = e.instance_scalars[e.env_to_instance]
        self.mto, self.mtj, self.sop = (sc[:, k:k + 1].astype(np.int64) for k in range(3))
        self.M = e.env_machines[:, None].astype(np.int64)
        self.len = np.stack([insts[k][1].sum(1) for k in e.env_to_instance]).astype(np.int64)

    def random_state(self, rng):
        """In-range integers for every field: each entry of the row in [0, 1]."""
        n, J = self.env.num_envs, self.J
        u = lambda hi: (rng.random((n, J)) * (hi + 1)).astype(np.int64)      # uniform in [0, hi] per row
        t = u(self.mtj)[:, :1]
        total = np.minimum(u(self.sop), t)
        return {"todo": u(self.M), "tufco": u(self.mto), "col4": u(self.mto), "idle_last": u(self.sop),
                "total_idle": total, "legal": rng.integers(0, 2, (n, J)), "t": t[:, 0]}

    def quotients(self, st):
        """Numerator and divisor of every entry of the rows (column 0 is the legal bit over 1)."""
        perf = np.where(st["todo"] < self.M, st["t"][:, None] - st["total_idle"], self.len)
        num = np.stack([st["legal"], st["tufco"], st["todo"], perf, st["col4"], st["idle_last"], st["total_idle"]], -1)
        den = np.stack(np.broadcast_arrays(np.ones_like(self.mto), self.mto, self.M, self.mtj, self.mto, self.sop,
                                           self.sop), -1)
        return num, np.broadcast_to(den, num.shape)

    def check(self, st, ctx):
        """Imports `st` and checks the rows each emitting path writes: the import, refresh_obs after a recording step,
        and the packed host rows under each SIMD level (a JSS_ACTION_SKIP step ships every env's row)."""
        import torch
        env, J = self.env, self.J
        x = env.export_state()
        for k in ("todo", "tufco", "col4", "idle_last", "total_idle", "legal"):
            x[k][:, :J].copy_(torch.as_tensor(np.ascontiguousarray(st[k]), dtype=x[k].dtype))
        x["blocked"].zero_()
        x["tuam"].zero_()
        x["t"].copy_(torch.as_tensor(np.asarray(st["t"], np.int32)))
        x["flags"].fill_(FROZEN)
        env.import_state(x)
        assert not (np_(env.flags) & N.FLAG_ERROR).any(), f"{ctx}: an imported value was out of range"
        num, den = self.quotients(st)
        want = exact_f32(num, den)
        assert (num >= 0).all() and (num <= den).all()

        def same(got, path):
            got = np.asarray(got)[:, :J]
            assert_obs_exact(got, want, f"{ctx} {path}")
            assert got.min() >= 0.0 and got.max() <= 1.0, (ctx, path)
            assert (got[num == den] == 1.0).all(), (ctx, path)

        same(np_(env.real_obs), "import_state")
        env.real_obs.fill_(float("nan"))
        traj = env.logits_trajectory(1)
        env.step_logits_record(torch.zeros((env.num_envs, J + 1), dtype=torch.float32, device=env.device), traj, 0)
        env.refresh_obs()
        same(np_(env.real_obs), "refresh_obs")
        skip = np.full(env.num_envs, N.ACTION_SKIP, np.int32)
        try:
            for level in (0, 1, 2):
                env.host_set_simd(level)
                env.host_step_begin(skip, packed=True)
                env.host_wait_mask()
                same(env.host_wait_obs().copy(), f"packed rows, SIMD level {level}")
        finally:
            env.host_set_simd(2)


@native_test(emu=())
def reference_is_correctly_rounded():
    """np.float32(np.float64(x) / y) is the correctly rounded fp32 quotient, checked by exact rational rounding on a
    few thousand pairs from every divisor family of the sweeps, and on the scaled rewards raw / max_time_op."""
    rng = np.random.default_rng(1)
    pairs = []
    for y in list(rng.integers(1, MAX_DUR + 1, 300)) + [1, 3, 7, MAX_DUR] + list(range(2, 33)) + MAX_TIME_JOBS + SUM_OP:
        y = int(y)
        xs = np.concatenate([[0, 1, y - 1, y], rng.integers(0, y + 1, 12)])
        pairs += [(int(x), y) for x in xs if x >= 0]
    for y in rng.integers(1, MAX_DUR + 1, 200):
        pairs += [(int(x), int(y)) for x in rng.integers(-32 * MAX_DUR, MAX_DUR + 1, 4)]   # |raw| <= M * max_time_op
    pairs += [(-61410, MAX_DUR), (2 ** 24 - 1, 3), (2 ** 24 - 1, MAX_SUM_OP)]
    assert len(pairs) > 3000
    for x, y in pairs:
        assert exact_f32(x, y).view(np.uint32) == rounded_f32(x, y).view(np.uint32), (x, y)


@native_test(emu=dict(imports=1), gpu=dict(imports=8))
def divide_max_time_op(make_env, backend, imports):
    """Every max_time_op 1..2047, one env each (256 jobs), with the numerators 0..max_time_op in both tufco (column 1)
    and col4 (column 4): chunk k of 256 goes to tufco ascending from 0 and to col4 descending from max_time_op, so
    8 imports cover every numerator (the emulation's one import the lowest and the highest 256)."""
    rng = np.random.default_rng(2)
    J, M = 256, 2
    insts = []
    for y in range(1, MAX_DUR + 1):
        d = rng.integers(1, y + 1, J * M)
        d[rng.integers(J * M)] = y
        insts.append(_instance(rng, J, M, d))
    p = Planted(make_env, insts, np.arange(len(insts)))
    for k in range(imports):
        st = p.random_state(rng)
        lo = (k * J + np.arange(J)[None, :]) % (p.mto + 1)
        st["tufco"], st["col4"] = lo, p.mto - lo
        p.check(st, f"max_time_op import {k}")


@native_test(emu=(), gpu=())
def divide_machines(make_env, backend):
    """Every M 2..32, one env each (64 jobs), with every todo 0..M (column 2); todo = M also makes column 3
    jobs_length / max_time_jobs."""
    rng = np.random.default_rng(3)
    J = 64
    insts = [_instance(rng, J, M, rng.integers(1, 100, J * M)) for M in range(2, 33)]
    p = Planted(make_env, insts, np.arange(len(insts)))
    for k in range(2):
        st = p.random_state(rng)
        st["todo"] = (np.arange(J)[None, :] + k * 7) % (p.M + 1)
        p.check(st, f"machines import {k}")


@native_test(emu=dict(envs=2, imports=2, edge=200, n_random=300, n_hard=64),
             gpu=dict(envs=64, imports=7, edge=4096, n_random=100_000, n_hard=4096))
def divide_max_time_jobs(make_env, backend, envs, imports, edge, n_random, n_hard):
    """max_time_jobs (column 3) at 65 504 (the largest: 32 operations of 2047), 65 503, 32 767, 49 151, 2^15, 2^15 + 1
    and primes, with the n_hard numerators nearest a rounding midpoint, every numerator in [0, edge] and [y - edge, y]
    and n_random random ones, as t - total_idle (t = y); `envs` envs of 256 jobs per divisor, `imports` imports each."""
    rng = np.random.default_rng(4)
    J, M = 256, 32
    insts = []
    for y in MAX_TIME_JOBS:
        d = rng.integers(1, y // M + 1, (J, M))
        d[0] = _spread(y, M)                                  # job 0 is the longest: y
        insts.append(_instance(rng, J, M, d))
    p = Planted(make_env, insts, np.repeat(np.arange(len(insts)), envs))
    assert [int(v) for v in p.mtj[::envs, 0]] == MAX_TIME_JOBS
    per_env = []
    for y in MAX_TIME_JOBS:
        per_env.append(_numerators(rng, y, edge, n_random, n_hard, envs * imports * J).reshape(envs, imports, J))
    xs = np.concatenate(per_env)                              # (n, imports, J)
    for k in range(imports):
        st = p.random_state(rng)
        st["todo"] = np.minimum(st["todo"], p.M - 1)          # unfinished: column 3 is t - total_idle
        st["t"] = p.mtj[:, 0]
        st["total_idle"] = p.mtj - xs[:, k]
        st["idle_last"] = np.minimum(st["idle_last"], st["total_idle"])
        p.check(st, f"max_time_jobs import {k}")


@native_test(emu=dict(envs=1, imports=2, edge=100, n_random=100, n_hard=64),
             gpu=dict(envs=64, imports=7, edge=4096, n_random=100_000, n_hard=4096))
def divide_sum_op(make_env, backend, envs, imports, edge, n_random, n_hard):
    """sum_op (columns 5 and 6) at 16 769 024 (the largest: 256 x 32 operations of 2047), 2^23 - 1, 2^23, 2^23 + 1,
    3 * 2^22 and primes near 2^24 and 2^23, with the n_hard numerators nearest a rounding midpoint, every numerator in
    [0, edge] and [y - edge, y] (x = y and y - 1 among them) and n_random random ones, in both idle_last and
    total_idle; finished jobs (todo = M), so that column 3 stays jobs_length / max_time_jobs."""
    rng = np.random.default_rng(5)
    J, M = 256, 32
    insts = [_instance(rng, J, M, _spread(y, J * M)[rng.permutation(J * M)]) for y in SUM_OP]
    p = Planted(make_env, insts, np.repeat(np.arange(len(insts)), envs))
    assert [int(v) for v in p.sop[::envs, 0]] == SUM_OP
    per_env = []
    for y in SUM_OP:
        per_env.append(_numerators(rng, y, edge, n_random, n_hard, envs * imports * J).reshape(envs, imports, J))
    xs = np.concatenate(per_env)
    for k in range(imports):
        st = p.random_state(rng)
        st["todo"] = np.broadcast_to(p.M, st["todo"].shape).copy()
        st["idle_last"] = xs[:, k]
        st["total_idle"] = np.roll(xs[:, k], 1, axis=1)
        st["t"] = p.sop[:, 0]
        p.check(st, f"sum_op import {k}")


# ---- serialised episodes at the 24-bit time limit ------------------------------------------------------------------

def serial_instance(J, M=32, seed=None):
    """Every operation on machine 0: all 2047 long, or (with a seed) random durations with job 0 all 2047.  Machine 0
    never idles, so every complete schedule ends at sum_op; no job is ever blocked by a no-op, because every
    unfinished job waits for machine 0."""
    d = np.full((J, M), MAX_DUR, np.int32)
    if seed is not None:
        d = np.random.default_rng(seed).integers(1, MAX_DUR + 1, (J, M)).astype(np.int32)
        d[0] = MAX_DUR
    return np.zeros((J, M), np.int32), d


def _serial_insts(backend):
    J = {"emu": 64, "gpu": 256}[backend]
    return serial_instance(J), serial_instance(J, seed=6)


SERIAL_PATHS = ["step", "step_sample_RANDOM", "step_sample_MWR", "step_logits", "mixed_ta01", "rollout", "packed"]


@native_test(emu=["step", "step_sample_MWR", "mixed_ta01", "packed"], gpu=SERIAL_PATHS)
def serial_episode(make_env, backend, path):
    """One serialised episode per env to done, compared with the oracle after every step (mask, exact real_obs and
    scaled reward, raw reward, done, time, and every exported integer), through one entry point: step with random
    legal actions, step_sample (RANDOM, MWR), step_logits, step on a mixed batch with ta01 (the mixed kernel),
    rollout(write_obs=True) one transition per call, or the packed host path.  The no-op is never legal.  At the end
    t = sum_op and the last job to finish has waited sum_op - 32 * 2047."""
    import torch
    big, rnd = _serial_insts(backend)
    names = {"step": [big], "step_sample_RANDOM": [big], "step_sample_MWR": [rnd], "step_logits": [rnd],
             "mixed_ta01": [big, rnd, "ta01"], "rollout": [big], "packed": [big, rnd]}[path]
    from jssenv_b200.instances import load_instance
    env = make_env(len(names), batch_cfg(names, sort=False), seed=8)
    oracles = [OracleEnv(*(load_instance(n) if isinstance(n, str) else n)) for n in names]
    obs = env.reset()
    for o in oracles:
        o.reset()
    rng = np.random.default_rng(9)
    n = len(names)
    alive = np.ones(n, bool)
    acts = env.policy(path[12:]).clone() if path.startswith("step_sample") else None
    step = 0
    peak_t, peak_idle = np.zeros(n, np.int64), np.zeros(n, np.int64)
    while alive.any():
        mask = np_(env.action_mask).copy()
        if path.startswith("step_sample"):
            a = np_(acts).copy()
            obs, reward, done, _, _, acts = env.step_sample(acts, path[12:])
        elif path == "rollout":
            base = env._step_index
            a = np.array([o.masked_random_action(env.seed, i, base) for i, o in enumerate(oracles)], np.int32)
            obs, reward, done, _, _ = env.rollout("RANDOM", 1, write_obs=True)
        elif path == "step_logits":
            x = torch.as_tensor(rng.standard_normal((n, env.jobs + 1)).astype(np.float32), device=env.device)
            obs, reward, done, _, info = env.step_logits(x)
            a = np_(info["actions"]).copy()
        else:
            a = np.array([rng.choice(np.flatnonzero(m)) if m.any() else N.ACTION_SKIP for m in mask], np.int32)
            if path == "packed":
                env.host_step_begin(a, packed=True)
                hmask, reward, done = env.host_wait_mask()
                obs = {"action_mask": hmask, "real_obs": env.host_wait_obs()}
            else:
                obs, reward, done, _, _ = env.step(a)
        reward, done, raw = np_(reward), np_(done), np_(env.reward_raw)
        for i, o in enumerate(oracles):
            if not alive[i]:
                continue
            assert isinstance(names[i], str) or not mask[i, o.jobs], f"{path} step {step} env {i}: the no-op is legal"
            _, r, d, _, _ = o.step(int(a[i]))
            compare_env_to_oracle(env, i, o, obs, (reward[i], r), (done[i], d), (raw[i], o.last_raw_reward),
                                  ctx=f"{path} step {step} action {a[i]}")
            alive[i] = not d
        compare_exported_state(env, oracles, alive | np_(env.done), ctx=f"{path} step {step}")
        x = env.export_state()
        peak_t = np.maximum(peak_t, np_(x["t"]))
        peak_idle = np.maximum(peak_idle, np_(x["total_idle"]).max(1))
        step += 1
    for i, o in enumerate(oracles):
        assert int(env.last_makespan[i]) == o.current_time_step
        if not isinstance(names[i], str):                     # the serialised instances
            S = o.sum_op
            assert peak_t[i] == S and peak_idle[i] >= S - o.machines * MAX_DUR, (i, peak_t[i], peak_idle[i], S)
    print(f"{path}: {step} steps, largest t {peak_t.max()}, largest total_idle {peak_idle.max()}")


@native_test(emu=dict(look_from_end=40), gpu=dict(look_from_end=None))
def serial_known_answers(make_env, backend, look_from_end):
    """On the serialised all-2047 instance every complete schedule has makespan sum_op and raw return
    2 * sum_op - 32 * sum_op (-503 070 720 at 256 x 32, an int32 without wrap-around), whatever decides: every built-in
    rule (run_batch), rollout_priority, rollout_priority_sample, sample_episodes and beam_search (W = 4) from reset, and
    lookahead, every legal entry of which is sum_op (from reset; in the emulation from `look_from_end` transitions
    before the end).  stats() sums and bounds the episodes."""
    import torch
    from jssenv_b200.dispatching import DISPATCHING_RULES
    big, _ = _serial_insts(backend)
    J, M = big[0].shape
    S = J * M * MAX_DUR
    ret_want = 2 * S - M * S
    assert ret_want >= -2 ** 31
    n = 2
    env = make_env(n, {"instance_path": big}, seed=10)
    episodes = 0

    def ended(what):
        nonlocal episodes
        assert np_(env.done).all() and (np_(env.last_makespan) == S).all(), what
        assert (np_(env.last_return) == ret_want).all(), what
        episodes += n

    for name, rule in DISPATCHING_RULES.items():
        ret, mk = rule.run_batch(env)
        assert (np_(mk) == S).all() and (np_(ret) == ret_want).all(), name
        ended(name)
    rng = np.random.default_rng(11)
    table = torch.as_tensor(rng.standard_normal((n, J, M)).astype(np.float32), device=env.device)
    env.reset()
    env.rollout_priority(table)
    ended("rollout_priority")
    env.reset()
    _, _, _, _, info = env.rollout_priority_sample(table)
    assert np.isfinite(np_(info["log_prob"])).all()
    ended("rollout_priority_sample")
    env.reset()
    assert (np_(env.sample_episodes(table, 4)["makespan"]) == S).all()
    assert (np_(env.beam_search(table, 4)["makespan"]) == S).all()
    if look_from_end:
        env.rollout("RANDOM", J * M - look_from_end, write_obs=False)     # an episode is J * M allocations
    assert not np_(env.done).any()
    mask = np_(env.action_mask).copy()
    assert mask[:, :J].any(1).all() and not mask[:, J].any()
    values = np_(env.lookahead("MWR"))[:, : J + 1]
    assert (values[mask] == S).all() and (values[~mask] == -1).all(), values
    st = env.stats()
    assert st["episodes"] == episodes and st["envs_error"] == 0
    assert st["min_makespan"] == st["max_makespan"] == S and st["sum_makespan"] == episodes * S
    assert st["sum_return"] == episodes * ret_want
