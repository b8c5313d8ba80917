#!/usr/bin/env python
"""The policy entropy of table-drawn episodes (entropy=True on JssVecEnv.rollout_priority_sample and sample_episodes),
timed against the same calls without it and against what a caller writes without it:

  ta80, N = 65 536, a per-env (N, J, M) table, reset to done: rollout_priority_sample with entropy off, on, and on with
    both gradients stored plus the torch backward of (w log_prob + v entropy).sum();
  ta01, N = 4 096, k = 64, a per-env table, from reset: sample_episodes forward, and forward + backward (the replay),
    entropy off and on;
  ta01, N = 256, reset to done: the per-decision loop a caller writes today (export_state, a torch gather at todo, the
    masked softmax's entropy, step_logits on the gathered row) against rollout_priority_sample(entropy=True).

Before timing, the entropy forms' log_prob (and makespan) are checked bit for bit against the calls without entropy,
and the loop's episode entropies against the fused call's within 1e-4 relative.  Each round runs every variant of a
workload once with CUDA events around work that ends in a device synchronise, alternating.  The JSON line gives, per
workload, each variant's median and range in ms per call, with the card and its power limit.  Writes nothing.

  python tools/bench_entropy.py [--rounds R] [--device D]
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


def rounds(variants, n, setup=None):
    """Each variant timed once per round, alternating; `setup(name)` runs untimed before each."""
    ms = {k: [] for k in variants}
    for _ in range(n):
        for name, fn in variants.items():
            if setup is not None:
                setup(name)
            ms[name].append(timed(fn))
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()}


def loop_entropy(env, table):
    """The per-decision loop: export_state, gather each job's current entry, the masked softmax's entropy and
    step_logits on the row, until every env is done.  Returns each env's fp32 sum of the decisions' entropies."""
    import torch
    n, J = env.num_envs, env.jobs
    h = torch.zeros(n, device=table.device)
    rows = torch.full((n, J + 1), float("-inf"), device=table.device)
    while not bool(env.done.all()):
        x = env.export_state()
        todo = x["todo"].long().clamp(max=env.machines - 1)
        legal = x["legal"].bool()
        rows[:, :J] = table.gather(2, todo[:, :, None])[:, :, 0]
        lg = torch.where(legal, rows[:, :J], float("-inf"))
        ls = torch.log_softmax(lg, 1)
        p = ls.exp()
        ht = -torch.where(p > 0, p * ls, 0.0).sum(1)
        decide = legal.any(1) & ~env.done
        h += torch.where(decide, ht, 0.0)
        env.step_logits(rows)
    return h


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

    # 1. ta80, N = 65 536, reset to done
    n = 65536
    env = JssVecEnv(n, {"instance_path": "ta80"}, device=args.device, auto_reset=False, seed=1)
    J, M = env.jobs, env.machines
    gen = torch.Generator(device=dev).manual_seed(3)
    table = torch.randn((n, J, M), generator=gen, device=dev)
    w, v = torch.randn(n, generator=gen, device=dev), torch.randn(n, generator=gen, device=dev)
    x = table.clone().requires_grad_(True)

    def backward():
        x.grad = None
        _, _, _, _, info = env.rollout_priority_sample(x, entropy=True)
        (w * info["log_prob"] + v * info["entropy"]).sum().backward()

    variants = {"entropy_off": lambda: env.rollout_priority_sample(table),
                "entropy_on": lambda: env.rollout_priority_sample(table, entropy=True),
                "entropy_on_grad_backward": backward}
    outs = []
    for name in ("entropy_off", "entropy_on"):
        env.reset()
        env._step_index = 0
        outs.append(variants[name]()[4])
    if not torch.equal(outs[0]["log_prob"].view(torch.int32), outs[1]["log_prob"].view(torch.int32)):
        raise SystemExit("ta80: log_prob differs with entropy on")
    if not bool(torch.isfinite(outs[1]["entropy"]).all()):
        raise SystemExit("ta80: an entropy is not finite")

    def setup(_):
        env.reset()
        env._step_index = 0
    results.append({"workload": f"ta80 ({J}x{M}) N={n} rollout_priority_sample reset to done, per-env table",
                    "ms_per_call": rounds(variants, args.rounds, setup), "parity": "log_prob bit-identical"})
    env.close()

    # 2. ta01, N = 4 096, k = 64, from reset, sample_episodes forward and forward + backward
    n, k = 4096, 64
    env = JssVecEnv(n, {"instance_path": "ta01"}, device=args.device, auto_reset=False, seed=1)
    env.reset()
    J, M = env.jobs, env.machines
    table = torch.randn((n, J, M), generator=gen, device=dev)
    w, v = torch.randn((n, k), generator=gen, device=dev), torch.randn((n, k), generator=gen, device=dev)
    x = table.clone().requires_grad_(True)
    a = env.sample_episodes(table, k)
    env._step_index = 0
    b = env.sample_episodes(table, k, entropy=True)
    if not (torch.equal(a["makespan"], b["makespan"]) and
            torch.equal(a["log_prob"].view(torch.int32), b["log_prob"].view(torch.int32))):
        raise SystemExit("ta01: sample_episodes differs with entropy on")

    def fwd_bwd(entropy):
        def run():
            x.grad = None
            out = env.sample_episodes(x, k, entropy=entropy)
            loss = (w * out["log_prob"]).sum()
            if entropy:
                loss = loss + (v * out["entropy"]).sum()
            loss.backward()
        return run

    variants = {"forward_entropy_off": lambda: env.sample_episodes(table, k),
                "forward_entropy_on": lambda: env.sample_episodes(table, k, entropy=True),
                "forward_backward_entropy_off": fwd_bwd(False), "forward_backward_entropy_on": fwd_bwd(True)}
    results.append({"workload": f"ta01 ({J}x{M}) N={n} k={k} sample_episodes from reset, per-env table",
                    "ms_per_call": rounds(variants, args.rounds),
                    "parity": "makespan and log_prob bit-identical"})
    env.close()

    # 3. ta01, N = 256, reset to done: the per-decision torch loop against the fused call
    n = 256
    fused, loop = (JssVecEnv(n, {"instance_path": "ta01"}, device=args.device, auto_reset=False, seed=1)
                   for _ in range(2))
    J, M = fused.jobs, fused.machines
    table = torch.randn((n, J, M), generator=gen, device=dev)
    for e in (fused, loop):
        e.reset()
        e._step_index = 0
    _, _, _, _, info = fused.rollout_priority_sample(table, entropy=True)
    h_loop = loop_entropy(loop, table)
    if not torch.equal(fused.current_time_step, loop.current_time_step):
        raise SystemExit("ta01 loop: the loop's episodes differ from the fused call's")
    err = float(((h_loop - info["entropy"]).abs() / info["entropy"].abs().clamp(min=1)).max())
    if err > 1e-4:
        raise SystemExit(f"ta01 loop: entropies differ by {err:.3g} relative")

    def setup(_):
        for e in (fused, loop):
            e.reset()
            e._step_index = 0
    variants = {"rollout_priority_sample_entropy": lambda: fused.rollout_priority_sample(table, entropy=True),
                "torch_loop": lambda: loop_entropy(loop, table)}
    results.append({"workload": f"ta01 ({J}x{M}) N={n} reset to done, per-env table: the fused entropy against "
                                "export_state + gather + masked softmax entropy + step_logits per decision",
                    "ms_per_call": rounds(variants, args.rounds, setup),
                    "parity": f"same episodes; entropy max relative diff {err:.3g}"})
    print(json.dumps({"rounds": args.rounds, "results": results, "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
