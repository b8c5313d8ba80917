#!/usr/bin/env python
"""k episodes per env drawn from a caller's logit table, the envs left untouched (JssVecEnv.sample_episodes,
jss_sample_episodes), timed against what a caller does without it:

  ta80, N = 1, k = 4 096, a (1, J, M) table, from reset: sample_episodes against reset + rollout_priority_sample on a
    4 096-env batch (the same number of episodes drawn from reset, N*k envs instead of N);
  ta80, N = 256, k = 64, a per-env (N, J, M) table, after a fixed 500-decision random pre-roll: sample_episodes against
    the definitional loop, per sample s import_state(snapshot), RNG counter step_index + s*B and
    rollout_priority_sample on the whole batch, its makespans and log-probabilities gathered into column s;
  ta01, N = 4 096, k = 16, a per-env table, from reset, forward and backward: sample_episodes on a table that requires
    grad and log_prob.backward(w), against the same loop with a gradient buffer per sample and sum_s w_s G_s.

Before timing, the fused outputs are checked against the loop bit for bit (makespan and log_prob; for the first
workload, four columns against one-env twins), and the gradient within float32 rounding.  Each round runs both paths
with CUDA events around work that ends in a device synchronise, alternating.  Decisions per call are the operations not
yet started at the call, summed over the samples (every sample ends done; the sampler never draws the no-op from a
state a step produced).  The JSON line gives, per workload, each path's median and range in ms per call, episodes/s
and decisions/s, with the card and its power limit.  Writes nothing.

  python tools/bench_sample_episodes.py [--rounds R] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402


def timed(fn):
    import torch
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)


def undrawn_ops(env):
    """Operations not yet started, per env (int64 tensor)."""
    x = env.export_state()
    started = x["todo"].long() + (x["tufco"] > 0).long()
    return (env.machines - started).clamp(min=0)[:, :env.jobs].sum(1)


def result(workload, ms, episodes, decisions, parity):
    med = {k: statistics.median(v) for k, v in ms.items()}
    fused, other = list(ms)
    return {"workload": workload, "episodes_per_call": episodes, "decisions_per_call": decisions,
            "ms_per_call": {k: {"median": med[k], "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()},
            "episodes_per_s": {k: episodes / (med[k] * 1e-3) for k in ms},
            "decisions_per_s": {k: decisions / (med[k] * 1e-3) for k in ms},
            f"speedup_{fused}_vs_{other}": med[other] / med[fused], "parity": parity}


def loop_samples(env, table, k, snap, step_index, makespan, log_prob, weights=None, grad=None, gbuf=None):
    """The definitional loop: per sample s, import the snapshot, set the counter, one rollout_priority_sample."""
    import torch
    B = 2 * env.jobs * env.machines + 1
    for s in range(k):
        env.import_state(snap)
        env._step_index = step_index + s * B
        lp = env._rollout_priority_sample(table, B, gbuf)
        makespan[:, s] = torch.where(env.done, env.current_time_step, -1)
        log_prob[:, s] = lp
        if grad is not None:
            grad.add_(weights[:, s, None, None] * gbuf.nan_to_num())
    env.import_state(snap)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    dev = torch.device("cuda", args.device)
    results = []

    # 1. ta80, one env, k = 4 096 from reset, broadcast table, against a 4 096-env batch
    k = 4096
    env = JssVecEnv(1, {"instance_path": "ta80"}, device=args.device, auto_reset=False, seed=1)
    batch = JssVecEnv(k, {"instance_path": "ta80"}, device=args.device, auto_reset=False, seed=1)
    twin = JssVecEnv(1, {"instance_path": "ta80"}, device=args.device, auto_reset=False, seed=1)
    J, M = env.jobs, env.machines
    B = 2 * J * M + 1
    table = torch.randn((1, J, M), generator=torch.Generator(device=dev).manual_seed(7), device=dev)
    env.reset()
    out = env.sample_episodes(table, k)
    for s in (0, 1, 2047, k - 1):
        twin.reset()
        twin._step_index = s * B
        _, _, _, _, info = twin.rollout_priority_sample(table)
        if not (int(twin.current_time_step[0]) == int(out["makespan"][0, s])
                and torch.equal(info["log_prob"].view(torch.int32), out["log_prob"][:, s].view(torch.int32))):
            raise SystemExit(f"ta80 N=1 k={k}: sample {s} differs from its twin")
    if (out["makespan"] < 0).any():
        raise SystemExit("ta80 N=1: a sample did not end")
    ms = {"sample_episodes": [], "batch_rollout": []}
    for _ in range(args.rounds):
        ms["sample_episodes"].append(timed(lambda: env.sample_episodes(table, k)))
        ms["batch_rollout"].append(timed(lambda: (batch.reset(), batch.rollout_priority_sample(table))))
    results.append(result(f"ta80 ({J}x{M}) N=1 k={k} from reset, broadcast (1, J, M) table, against reset + "
                          f"rollout_priority_sample on a {k}-env batch", ms, k, k * J * M,
                          "four sample columns == one-env twins (import, counter, rollout_priority_sample)"))
    for e in (env, batch, twin):
        e.close()

    # 2. ta80, N = 256, k = 64, per-env table after 500 random decisions, against the definitional loop
    # 3. ta01, N = 4 096, k = 16, per-env table from reset, forward + backward against the loop with gradients
    for inst, n, k, preroll, backward in (("ta80", 256, 64, 500, False), ("ta01", 4096, 16, 0, True)):
        env, loop = (JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
                     for _ in range(2))
        J, M = env.jobs, env.machines
        for e in (env, loop):
            e.reset()
            for _ in range(preroll):
                e.step(e.policy("RANDOM"))
        snap = {key: v.clone() for key, v in loop.export_state().items()}
        decisions = int(undrawn_ops(loop).sum()) * k
        gen = torch.Generator(device=dev).manual_seed(8)
        table = torch.randn((n, J, M), generator=gen, device=dev)
        weights = torch.randn((n, k), generator=gen, device=dev)
        mk, lp = torch.empty((n, k), dtype=torch.int32, device=dev), torch.empty((n, k), device=dev)
        grad = torch.zeros((n, J, M), device=dev) if backward else None
        gbuf = torch.empty((n, J, M), device=dev) if backward else None
        x = table.clone().requires_grad_(backward)

        def fused():
            out = env.sample_episodes(x, k)
            if backward:
                x.grad = None
                out["log_prob"].backward(weights)
            return out

        def run_loop():
            if backward:
                grad.zero_()
            loop_samples(loop, table, k, snap, env._step_index - k * (2 * J * M + 1), mk, lp, weights, grad, gbuf)

        out = fused()
        run_loop()
        if not (torch.equal(out["makespan"], mk) and torch.equal(out["log_prob"].view(torch.int32), lp.view(torch.int32))):
            raise SystemExit(f"{inst} N={n} k={k}: fused and loop samples differ")
        if (mk < 0).any():
            raise SystemExit(f"{inst} N={n} k={k}: a sample did not end")
        parity = "makespan and log_prob bit-identical to the loop"
        if backward:
            err = float((x.grad - grad).abs().max())
            tol = 1e-5 * float(weights.abs().sum(1).max()) * (1 + float(grad.abs().max()))
            if err > tol:
                raise SystemExit(f"{inst} N={n} k={k}: gradient differs from the loop's by {err}")
            parity += f"; gradient max |diff| {err:.3g}"
        ms = {"sample_episodes": [], "loop": []}
        for _ in range(args.rounds):
            ms["sample_episodes"].append(timed(fused))
            ms["loop"].append(timed(run_loop))
        results.append(result(f"{inst} ({J}x{M}) N={n} k={k}, {preroll} random decisions before the call, per-env "
                              f"(N, J, M) table{', forward + backward' if backward else ''}, against import_state + "
                              f"counter + rollout_priority_sample per sample", ms, n * k, decisions, parity))
        for e in (env, loop):
            e.close()
    print(json.dumps({"rounds": args.rounds, "results": results, "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
