"""Several envs per process, the caller's side streams, the host pipeline next to stream-ordered calls, and long chains
of back-to-back launches, each against a twin: the same batch, seed and inputs, run alone on the default stream with a
device synchronise after every call.  Results are compared bit for bit (floats as uint32 bits).

The library keeps CUDA state that outlives one handle, one stream and one launch: a kernel's dynamic shared-memory
opt-in is per process and device, the host pipeline runs on the handle's own non-blocking streams, and the step kernels
launch with programmatic dependent launch (PDL).  The host emulation runs every launch in order, so these tests are
GPU-only; collected by tests/test_gpu_sharing.py.

Tests that need work to land late put a sleep of SLEEP_CYCLES on the producing stream, and assert their own premise:
that stream is still busy once the call under test is enqueued, and it is non-blocking (the default stream does not
wait for it)."""
import contextlib

import numpy as np

from tests.backends import native_test
from tests.parity_common import OUTPUTS, batch_cfg, np_, synthetic_instance, twin_envs

SLEEP_CYCLES = 100_000_000        # torch.cuda._sleep: about 50 ms at the H100's 1.98 GHz SM clock

U256 = synthetic_instance(256, 32, seed=41, max_dur=60)
U230 = synthetic_instance(230, 20, seed=42, max_dur=60)
U200 = synthetic_instance(200, 10, seed=43, max_dur=60)
U127 = synthetic_instance(127, 7, seed=44, max_dur=60)
# the orders of handles of test A (each run twice through): each later batch has a smaller layout of the kernels they
# share, all over 48 KB, so that a handle that lowered a kernel's opt-in would break the ones before it
ORDERS = {"uniform": [[U256] * 8, [U200] * 8],                                  # 8-jobs-per-lane step + generic kernels
          "mixed": [["ta01"] * 3 + [U256] * 5, ["ta01"] * 3 + [U200] * 5],      # jss_step_mixed_kernel<_, true>
          "rem": [[U127] * 8, ["ta80"] * 8],                                    # MWR step_sample: 53.7 vs 48.2 KB
          "three": [[U230] * 8, [U256] * 8, [U200] * 8]}


# ---------------------------------------------------------------- the shared-memory layouts (plan_smem_layouts)
def smem_layouts(names):
    """Dynamic shared memory in bytes of the generic kernel ("env") and the step kernels without / with the suffix-sum
    table and with a logits row, for a batch of `names`: a restatement of plan_smem_layouts in jss_api.cu."""
    from jssenv_b200.instances import load_instance
    shapes = [(n if not isinstance(n, str) else load_instance(n))[0].shape for n in names]
    J, M = max(s[0] for s in shapes), max(s[1] for s in shapes)
    ops, rem = max(j * m for j, m in shapes), max(j * (m + 1) for j, m in shapes)
    up = lambda x, m: -(-x // m) * m
    slots = max(4, 1 << (0 if J <= 32 else 1 if J <= 64 else 2 if J <= 128 else 3))
    jcap, mcap = up(J, slots), up(M, 4)
    words = 2 * jcap + up(jcap, 8) // 2 + mcap + 2 * slots + 4
    scratch = max(7 * jcap, 32) * 4
    off_rem = 80 + up(ops, 8) * 2 + up(J, 4) * 4           # sizeof(JssInst) = 80
    off_warp0 = off_rem + up(rem, 8) * 2
    step_warp = 16 + words * 4 + scratch + words * 4
    return {"env": off_warp0 + 8 * scratch, "step": off_rem + 8 * step_warp, "step_rem": off_warp0 + 8 * step_warp,
            "step_logits": off_rem + 8 * (step_warp + up(4 * (J + 1), 16))}


def check_layouts(order):
    """The premise of test A for `order`: the last handle's layout of each kernel the order exercises is over 48 KB
    and smaller than every earlier handle's."""
    kernels = ["step_rem"] if order == "rem" else ["env", "step", "step_logits"]
    sizes = [smem_layouts(b) for b in ORDERS[order]]
    for earlier in sizes[:-1]:
        for k in kernels:
            assert earlier[k] > sizes[-1][k] > 48 * 1024, (order, k, earlier[k], sizes[-1][k])


# ---------------------------------------------------------------- helpers
def _bits(t):
    x = np.ascontiguousarray(np_(t))
    return x.view(np.uint32) if x.dtype == np.float32 else x.view(np.uint8) if x.dtype == np.bool_ else x


def _assert_same(got, want, ctx):
    """Two lists of (call, {name: tensor}) equal, bit for bit."""
    assert [g[0] for g in got] == [w[0] for w in want], ctx
    for (call, a), (_, b) in zip(got, want):
        assert a.keys() == b.keys(), (ctx, call)
        for k in a:
            assert np.array_equal(_bits(a[k]), _bits(b[k])), (ctx, call, k)


def _outputs(env):
    return {name: getattr(env, name).clone() for name in OUTPUTS}


def _sleep(stream):
    import torch
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)


def _side_stream():
    """A new torch side stream, once checked to be non-blocking: a default-stream op completes while it sleeps.  (The op
    runs once before the sleep: a kernel's first launch in the process loads it, which waits for the device.)"""
    import torch
    side = torch.cuda.Stream()
    x = torch.ones(4, device="cuda")
    (x * 2).sum().item()
    _sleep(side)
    y = x * 2
    torch.cuda.default_stream().synchronize()
    assert not side.query() and float(y.sum()) == 8.0, "the side stream must be non-blocking"
    side.synchronize()
    return side


def _prep(env, seed, n_rows=4, k=2):
    """Seeded device inputs of the script: rows for the row-driven steps, a logit / priority table, weights."""
    import torch
    rng = np.random.default_rng(seed)
    n, J, M = env.num_envs, env.jobs, env.machines
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(env.device)
    return {"rows": dev(rng.standard_normal((n_rows, n, J + 1)).astype(np.float32)),
            "table": dev(rng.standard_normal((n, J, M)).astype(np.float32)),
            "w": dev(rng.standard_normal(n).astype(np.float32)),
            "wk": dev(rng.standard_normal((n, k)).astype(np.float32)),
            "reset_mask": dev((rng.random(n) < 0.5).astype(np.uint8))}


def _script(env, inp, late, rnd):
    """Every entry-point family once, as (call, fn, flags): fn() runs the call and returns what it produced besides the
    env's outputs.  `late(t)` is the call's copy of a prepared input.  Flags: "syncs" (the call synchronises its
    stream), "outside" (run outside the side stream's context)."""
    import torch
    s = {}

    def policy():
        s["a"] = env.policy("RANDOM").clone()
        return {"a": s["a"]}

    def step():
        env.step(late(s["a"]))
        return {}

    def step_sample(rule):
        *_, s["a"] = env.step_sample(late(s["a"]), rule)
        return {"a": s["a"]}

    def row(what, k, *extra):
        _, _, _, _, info = getattr(env, what)(late(inp["rows"][k]), *extra)
        return dict(info)

    def record(what, k, *extra):
        getattr(env, what)(late(inp["rows"][k]), s["traj"], k, *extra)
        return {}

    def trajectory():
        s["traj"] = env.logits_trajectory(2)
        return {}

    def traj_out(t):
        return {k: t[k].clone() for k in ("_obs", "_mask", "_scalars", "actions") + (("log_prob",) if "log_prob" in t else ())}

    def prio_sample():
        x = late(inp["table"]).requires_grad_()
        _, _, _, _, info = env.rollout_priority_sample(x, n_steps=30)
        s["x1"], s["loss1"] = x, (info["log_prob"] * late(inp["w"])).sum()
        return {"log_prob": info["log_prob"].detach().clone()}

    def episodes():
        x = late(inp["table"]).requires_grad_()
        out = env.sample_episodes(x, 2, solution=True)
        s["x2"], s["loss2"] = x, (out["log_prob"] * late(inp["wk"])).sum()
        return {k: v.detach().clone() for k, v in out.items()}

    def backward(i):
        s[f"loss{i}"].backward()
        return {"grad": s[f"x{i}"].grad.clone()}

    def export():
        s["snap"] = {k: v.clone() for k, v in env.export_state().items()}
        return dict(s["snap"])

    def stats():
        return {"stats": torch.tensor(list(env.stats().values()))}

    out = "outside" if rnd % 2 else ""
    return [
        ("reset", lambda: env.reset(late(inp["reset_mask"])) and {}, ""),
        ("rollout", lambda: env.rollout("SPT", 40) and {}, ""),
        ("policy", policy, ""), ("step", step, ""),
        ("export_state", export, ""),
        ("step_sample RANDOM", lambda: step_sample("RANDOM"), ""),
        ("step_sample MWR", lambda: step_sample("MWR"), ""), ("step", step, ""),
        ("step_logits", lambda: row("step_logits", 0), ""),
        ("step_greedy", lambda: row("step_greedy", 1, 0.3), ""),
        ("logits_trajectory", trajectory, ""),
        ("step_logits_record", lambda: record("step_logits_record", 0), ""),
        ("step_greedy_record", lambda: record("step_greedy_record", 1, 0.3), ""),
        ("trajectory", lambda: traj_out(s["traj"]), ""),
        ("refresh_obs", lambda: env.refresh_obs() or {}, ""),
        ("rollout_record", lambda: traj_out(env.rollout_record("MWR", 8)), ""),
        ("rollout_priority", lambda: env.rollout_priority(late(inp["table"]), n_steps=30) and {}, ""),
        ("rollout_priority_sample", prio_sample, ""), ("backward", lambda: backward(1), out),
        ("lookahead", lambda: {"v": env.lookahead("MWR")}, ""),
        ("lookahead_priority", lambda: {"v": env.lookahead_priority(late(inp["table"]))}, ""),
        ("sample_episodes", episodes, ""), ("backward", lambda: backward(2), out),
        ("import_state", lambda: env.import_state({k: late(v) for k, v in s["snap"].items()}) or {}, ""),
        ("stats", stats, "syncs"),
        ("export_state", export, ""),
    ]


def run_script(env, inp, rnd, side=None):
    """The script on `env`: with side=None on the default stream with a device synchronise after every call (the twin);
    else every call inside torch.cuda.stream(side) behind a sleep on side, its inputs copied and its outputs cloned on
    side, and one synchronise at the end.  Returns [(call, {name: tensor})]."""
    import torch
    late = lambda t: t.clone()          # a fresh leaf per call: gradients never accumulate across calls
    res = []
    for call, fn, flags in _script(env, inp, late, rnd):
        if side is None:
            res.append((call, {**fn(), **_outputs(env)}))
            torch.cuda.synchronize()
            continue
        _sleep(side)
        with contextlib.nullcontext() if "outside" in flags else torch.cuda.stream(side):
            res.append((call, {**fn(), **_outputs(env)}))
        if "syncs" not in flags:
            assert not side.query(), f"the sleep did not cover {call}: raise SLEEP_CYCLES"
    torch.cuda.synchronize()
    return res


def _make(make_env, names, **kw):
    return make_env(len(names), batch_cfg(names, sort=False), seed=11, auto_reset=True, record_solution=True, **kw)


# ---------------------------------------------------------------- A: handles that share kernels
@native_test(emu=None, gpu=list(ORDERS))
def sharing_handles(make_env, backend, order):
    """Handles of different batches created and run one after another in one process (the order twice through, every
    entry point family each time) equal each batch run alone: a later handle with a smaller layout of a kernel must
    not lower the kernel's shared-memory opt-in under an earlier one."""
    check_layouts(order)
    batches = ORDERS[order]
    envs = [_make(make_env, b) for b in batches]
    got = [[] for _ in batches]
    for rnd in range(2):
        for i, e in enumerate(envs):                    # each handle creates its layouts on first use, in this order
            got[i].append(run_script(e, _prep(e, 100 + i), rnd))
    for i, b in enumerate(batches):
        alone = _make(make_env, b)
        for rnd in range(2):
            _assert_same(got[i][rnd], run_script(alone, _prep(alone, 100 + i), rnd), (order, i, rnd))


# ---------------------------------------------------------------- B: the caller's stream
B_BATCH = ["ta01", "ta31", "ta80", "ta51", "ta80", "ta01", U200, "ta31", "ta80", "ta51"]


@native_test(emu=None, gpu=())
def sharing_side_stream(make_env, backend):
    """Every stream-ordered entry point inside torch.cuda.stream(side), its inputs written on side behind a sleep and its
    outputs copied on side, equals the twin; both autograd backwards run inside the context in the first round and
    outside it in the second.  The twin runs first, so that no kernel is loaded (which waits for the device) under
    the sleep."""
    side = _side_stream()
    env, twin = _make(make_env, B_BATCH), _make(make_env, B_BATCH)
    for rnd in range(2):
        want = run_script(twin, _prep(twin, 200 + rnd), rnd)
        _assert_same(run_script(env, _prep(env, 200 + rnd), rnd, side=side), want, rnd)


@native_test(emu=None, gpu=())
def sharing_construct_on_side_stream(make_env, backend):
    """An N = 65 536 ta80 batch constructed inside torch.cuda.stream(side) and stepped on side at once equals its twin:
    the construction's own reset on the legacy default stream has completed when the constructor returns."""
    import torch
    side = _side_stream()
    names = ["ta80"] * 65536
    with torch.cuda.stream(side):
        env = _make(make_env, names)
        acts = env.policy("RANDOM")
        for _ in range(8):
            *_, acts = env.step_sample(acts, "RANDOM")
        got = {**_outputs(env), "a": acts.clone()}
    torch.cuda.synchronize()
    twin = _make(make_env, names)
    acts = twin.policy("RANDOM")
    for _ in range(8):
        *_, acts = twin.step_sample(acts, "RANDOM")
        torch.cuda.synchronize()
    _assert_same([("steps", got)], [("steps", {**_outputs(twin), "a": acts.clone()})], "construct")
    _assert_same([("state", env.export_state())], [("state", twin.export_state())], "construct")
    assert env.stats() == twin.stats()


# ---------------------------------------------------------------- C: host pipeline meets stream-ordered calls
C_BATCH = ["ta01", "ta80", "ta31", "ta80", "ta01", "ta51", "ta80", "ta31"]
C_CALLS = ["step", "step_sample", "policy", "export_state", "stats", "step_host", "reset", "import_state",
           "sample_episodes"]
C_SYNCS = ("stats", "step_host", "import_state")     # these return once their stream (or the pipeline) is done


def _call(env, call, b, snap, inp):
    """One stream-ordered call on the default stream after the host step, and what it produced."""
    import torch
    bd = torch.from_numpy(b).to(env.device)
    if call == "step":
        env.step(bd)
        return {}
    if call == "step_sample":
        return {"a": env.step_sample(bd, "RANDOM")[-1].clone()}
    if call == "policy":
        return {"a": env.policy("RANDOM", step_index=500).clone()}
    if call == "export_state":
        return {k: v.clone() for k, v in env.export_state().items()}
    if call == "stats":
        return {"stats": torch.tensor(list(env.stats().values()))}
    if call == "step_host":
        obs, rew, done, _, _ = env.step_host(b)
        return {"mask": torch.from_numpy(obs["action_mask"].copy()), "obs": torch.from_numpy(obs["real_obs"].copy()),
                "reward": torch.from_numpy(rew.copy())}
    if call == "reset":
        env.reset(inp["reset_mask"])
        return {}
    if call == "import_state":
        env.import_state(snap)
        return {}
    out = env.sample_episodes(inp["table"], 2, solution=True)
    return {k: v.clone() for k, v in out.items()}


def _pair_after_steps(make_env, names, n_steps=6):
    """An env and its twin, stepped alike to a state past the start, and the host actions a (for the pipelined step)
    and b (legal after a), and a snapshot taken before a."""
    import torch
    env, twin = _make(make_env, names), _make(make_env, names)
    for e in (env, twin):
        for _ in range(n_steps):
            e.step(e.policy("RANDOM"))
    torch.cuda.synchronize()
    a = np_(twin.policy("RANDOM", step_index=300)).copy()
    snap = {k: v.clone() for k, v in twin.export_state().items()}
    return env, twin, a, snap


@native_test(emu=None, gpu=C_CALLS)
def sharing_pipeline_then(make_env, backend, call):
    """host_step_begin(a) enqueued behind a sleep on a side stream, then a stream-ordered call on the default stream:
    the call acts on the state after a, as the twin's step(a) followed by the same call does, and the pipeline's own
    host results are those of step(a)."""
    import torch
    env, twin, a, snap = _pair_after_steps(make_env, C_BATCH)
    inp = _prep(twin, 7)
    twin.step(a)
    after_a = {"mask": np_(twin.action_mask).copy(), "obs": np_(twin.real_obs).copy(), "reward": np_(twin.reward).copy()}
    b = np_(twin.policy("RANDOM", step_index=301)).copy()
    want = {**_call(twin, call, b, snap, inp), **_outputs(twin)}
    warm = _make(make_env, C_BATCH)                   # the sequence once untimed: first-use costs land outside the sleep
    warm.host_step_begin(a)
    _call(warm, call, b, snap, inp)
    warm.host_wait_obs()
    torch.cuda.synchronize()
    side = _side_stream()
    _sleep(side)
    with torch.cuda.stream(side):
        env.host_step_begin(a)
    assert not side.query(), "the sleep did not cover host_step_begin"
    got = {**_call(env, call, b, snap, inp), **_outputs(env)}
    if call not in C_SYNCS:
        assert not side.query(), f"the sleep did not cover {call}: raise SLEEP_CYCLES"
    torch.cuda.synchronize()
    mask, reward, _ = env.host_wait_mask()
    obs = env.host_wait_obs()
    assert np.array_equal(mask, after_a["mask"]) and np.array_equal(_bits(reward), _bits(after_a["reward"])), call
    assert np.array_equal(_bits(obs), _bits(after_a["obs"])), call
    _assert_same([(call, got)], [(call, want)], "pipeline then call")
    _assert_same([("state", env.export_state())], [("state", twin.export_state())], call)
    assert env.stats() == twin.stats(), call


@native_test(emu=None, gpu=[("plain", False, 0.0), ("packed", True, 0.0), ("hybrid", True, 0.4)])
def sharing_pipeline_mask_then_step(make_env, backend, mode, packed, dma_fraction):
    """After host_wait_mask() alone, a device step does not change what host_wait_obs() then returns: the step waits
    for the begin's observation transfer."""
    import torch
    names = ["ta80"] * 4096
    env, twin, a, _ = _pair_after_steps(make_env, names)
    twin.step(a)
    obs_a = np_(twin.real_obs).copy()
    b = np_(twin.policy("RANDOM", step_index=301)).copy()
    twin.step(b)
    env.host_step_begin(a, packed=packed, dma_fraction=dma_fraction)
    env.host_wait_mask()
    env.step(torch.from_numpy(b).to(env.device))
    obs = env.host_wait_obs()
    assert np.array_equal(_bits(obs), _bits(obs_a)), mode
    torch.cuda.synchronize()
    _assert_same([("step", _outputs(env))], [("step", _outputs(twin))], mode)
    _assert_same([("state", env.export_state())], [("state", twin.export_state())], mode)


# ---------------------------------------------------------------- D: back-to-back launches
MIXED_ALL = ["ta01", "ta51", "ta80", U200]           # lane classes 0 .. 3, 129..256 jobs included
D_BATCHES = {"ta80": (["ta80"] * 16384, 64),          # more tiles than resident CTAs
             "mixed": ([MIXED_ALL[i % 4] for i in range(4096)], 64),   # 512 tiles: grid > one resident CTA per SM
             "ta01": (["ta01"] * 8, 256)}             # one CTA
D_KINDS = ["step", "step_sample RANDOM", "step_sample MWR", "step_logits", "step_greedy", "record"]


def _chain(env, kind, K, acts, rows, sync):
    """K launches of `kind` on `env`, every input prepared in `acts` / `rows`; sync: a device synchronise after each.
    Returns the buffers the chain wrote."""
    import torch
    n, dev = env.num_envs, env.device
    if kind == "record":
        traj = env.logits_trajectory(K)
    elif kind.startswith("step_sample"):
        buf = torch.empty((K + 1, n), dtype=torch.int32, device=dev)
        buf[0] = env.policy(kind.split()[1])
    else:
        out_a = torch.zeros((K, n), dtype=torch.int32, device=dev)
        out_lp = torch.zeros((K, n), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    for k in range(K):
        if kind == "step":
            env.step(acts[k])
        elif kind.startswith("step_sample"):
            env.step_sample(buf[k], kind.split()[1], out=buf[k + 1])
        elif kind == "step_logits":
            env.step_logits(rows[k], actions_out=out_a[k], log_prob_out=out_lp[k])
        elif kind == "step_greedy":
            env.step_greedy(rows[k], 0.3, actions_out=out_a[k], log_prob_out=out_lp[k])
        elif k % 2:
            env.step_greedy_record(rows[k], traj, k, epsilon=0.3)
        else:
            env.step_logits_record(rows[k], traj, k)
        if sync:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    if kind == "record":
        return {k: traj[k] for k in ("_obs", "_mask", "_scalars", "actions", "log_prob")}
    return {"a": buf} if kind.startswith("step_sample") else {"a": out_a, "log_prob": out_lp}


def _chain_rows(env, K, seed):
    """K seeded logit / score rows for `env`'s batch, as slices of one device tensor."""
    import torch
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.standard_normal((K, env.num_envs, env.jobs + 1)).astype(np.float32)).to(env.device)


@native_test(emu=None, gpu=[(b, k) for b in D_BATCHES for k in D_KINDS])
def sharing_back_to_back(make_env, backend, batch, kind):
    """A chain of launches with no torch op and no host synchronise between them (each step may start under PDL before
    the previous one drains) equals the same chain with a device synchronise after every launch: every recorded slot
    and action, the final outputs, the exported state and the statistics."""
    import torch
    names, K = D_BATCHES[batch]
    env, twin = twin_envs(make_env, names, sort=False, seed=19, auto_reset=True)
    rows = _chain_rows(twin, K, 19)
    acts = None
    if kind == "step":                                  # actions of a synchronised masked-random run of a third copy
        pilot = make_env(len(names), batch_cfg(names, sort=False), seed=19, auto_reset=True)
        acts = torch.empty((K, len(names)), dtype=torch.int32, device=env.device)
        for k in range(K):
            acts[k] = pilot.policy("RANDOM")
            pilot.step(acts[k])
            torch.cuda.synchronize()
        pilot.close()
    got = _chain(env, kind, K, acts, rows, sync=False)
    want = _chain(twin, kind, K, acts, rows, sync=True)
    _assert_same([(kind, {**got, **_outputs(env)})], [(kind, {**want, **_outputs(twin)})], batch)
    _assert_same([("state", env.export_state())], [("state", twin.export_state())], (batch, kind))
    assert env.stats() == twin.stats(), (batch, kind)


@native_test(emu=None, gpu=())
def sharing_two_streams_interleaved(make_env, backend):
    """Two envs of different batches, each on its own side stream, their launches interleaved with no synchronise
    between them, each equal to its twin."""
    import torch
    K = 96
    b1, b2 = ["ta80"] * 4096, [MIXED_ALL[i % 4] for i in range(1024)]
    e1, t1 = twin_envs(make_env, b1, sort=False, seed=23, auto_reset=True)
    e2, t2 = twin_envs(make_env, b2, sort=False, seed=29, auto_reset=True)
    rows = _chain_rows(e2, K, 29)
    bufs, outs = [], []
    for e in (e1, t1):
        bufs.append(torch.empty((K + 1, e.num_envs), dtype=torch.int32, device=e.device))
        bufs[-1][0] = e.policy("RANDOM")
    for e in (e2, t2):
        outs.append((torch.zeros((K, e.num_envs), dtype=torch.int32, device=e.device),
                     torch.zeros((K, e.num_envs), dtype=torch.float32, device=e.device)))
    torch.cuda.synchronize()
    s1, s2 = _side_stream(), _side_stream()
    for k in range(K):
        with torch.cuda.stream(s1):
            e1.step_sample(bufs[0][k], "RANDOM", out=bufs[0][k + 1])
        with torch.cuda.stream(s2):
            e2.step_greedy(rows[k], 0.2, actions_out=outs[0][0][k], log_prob_out=outs[0][1][k])
    for k in range(K):
        t1.step_sample(bufs[1][k], "RANDOM", out=bufs[1][k + 1])
        t2.step_greedy(rows[k], 0.2, actions_out=outs[1][0][k], log_prob_out=outs[1][1][k])
        torch.cuda.synchronize()
    torch.cuda.synchronize()
    _assert_same([("e1", {"a": bufs[0], **_outputs(e1)})], [("e1", {"a": bufs[1], **_outputs(t1)})], "stream 1")
    _assert_same([("e2", {"a": outs[0][0], "lp": outs[0][1], **_outputs(e2)})],
                 [("e2", {"a": outs[1][0], "lp": outs[1][1], **_outputs(t2)})], "stream 2")
    for e, t in ((e1, t1), (e2, t2)):
        _assert_same([("state", e.export_state())], [("state", t.export_state())], "two streams")
        assert e.stats() == t.stats()
