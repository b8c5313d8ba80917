#!/usr/bin/env python
"""Whole episodes drawn from a caller's logit table, timed on ta80 at N = 65 536 from reset to done, with a seeded
torch.randn per-operation table (N, J, M):

  sample:       JssVecEnv.rollout_priority_sample(P) without the gradient (jss_rollout_priority_sample, grad_out
                NULL), one call to the end of every episode;
  sample_grad:  the same with P.requires_grad, then backward() of log_prob.sum() (the kernel writes the gradient
                table, the backward weights and returns it);
  greedy:       rollout_priority(P), the argmax of the same table (jss_rollout_priority);
  loop:         the same draws the only way possible without the fused call: per decision, export_state(), a torch
                gather of P at todo, the no-op column at -inf, then step_logits(rows), its log_prob summed in fp32.

The loop checks every --poll decisions whether every env is done.  Every round resets the envs and sets the RNG counter
to 0, and runs each path with CUDA events around work that ends in a device synchronise.  Before the timed rounds, an
untimed round checks that sample and loop leave bit-identical makespans, raw returns, solutions and log-prob sums; the
timed rounds check it again.  The JSON line gives each path's median and range over --rounds alternating rounds, in ms
per batch, episodes/s and decisions/s, and the card with its power limit.  Writes nothing.

  python tools/bench_priority_sample.py [--envs N] [--instance ta80] [--rounds R] [--poll P] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--instance", default="ta80")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--poll", type=int, default=50, help="decisions between the loop's all-done checks")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    N = args.envs
    names = ("sample", "sample_grad", "greedy", "loop")
    envs = {name: JssVecEnv(N, {"instance_path": args.instance}, device=args.device, auto_reset=False,
                            record_solution=True, seed=1)
            for name in names}
    env0 = envs["sample"]
    J, M, dev = env0.jobs, env0.machines, env0.device
    gen = torch.Generator(device=dev).manual_seed(0)
    table = torch.randn((N, J, M), device=dev, generator=gen)
    ninf = torch.full((N, 1), float("-inf"), device=dev)
    log_prob = {}

    def sample(env):
        log_prob["sample"] = env.rollout_priority_sample(table)[4]["log_prob"]

    def sample_grad(env):
        x = table.clone().requires_grad_(True)
        lp = env.rollout_priority_sample(x)[4]["log_prob"]
        lp.sum().backward()
        log_prob["sample_grad"] = lp.detach()

    def loop(env):
        total = torch.zeros(N, dtype=torch.float32, device=dev)
        while True:
            for _ in range(args.poll):
                todo = env.export_state()["todo"].clamp(max=M - 1).long()
                rows = torch.cat([table.gather(2, todo.unsqueeze(2)).squeeze(2), ninf], 1)
                total += env.step_logits(rows)[4]["log_prob"]
            if bool(env.done.all()):
                log_prob["loop"] = total
                return

    paths = {"sample": sample, "sample_grad": sample_grad, "greedy": lambda env: env.rollout_priority(table),
             "loop": loop}

    def run(name):
        env = envs[name]
        env.reset()
        env._step_index = 0
        steps0 = env.stats()["steps"]
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        paths[name](env)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1)
        if not bool(env.done.all()):
            raise SystemExit(f"{name}: not every env is done")
        return ms, env.stats()["steps"] - steps0

    def check():
        a, b = envs["sample"], envs["loop"]
        for f in ("last_makespan", "last_return", "solution"):
            if not torch.equal(getattr(a, f), getattr(b, f)):
                raise SystemExit(f"sample and loop differ in {f}")
        if not torch.equal(log_prob["sample"].view(torch.int32), log_prob["loop"].view(torch.int32)):
            raise SystemExit("sample and loop differ in the log-prob sums")
        if not torch.equal(log_prob["sample"].view(torch.int32), log_prob["sample_grad"].view(torch.int32)):
            raise SystemExit("sample and sample_grad differ in the log-prob sums")

    for name in paths:                                   # untimed: warm-up and the bit-identity check
        run(name)
    check()
    ms = {name: [] for name in paths}
    decisions = {}
    for _ in range(args.rounds):
        for name in paths:
            t, d = run(name)
            ms[name].append(t)
            decisions[name] = d
        check()
    err = {name: int(env.stats()["envs_error"]) for name, env in envs.items()}
    mean_makespan = {name: float(env.last_makespan.double().mean()) for name, env in envs.items()}
    mean_log_prob = float(log_prob["sample"].double().mean())
    for env in envs.values():
        env.close()
    med = {name: statistics.median(v) for name, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.instance} ({J}x{M}) N={N} from reset to the end of every episode, seeded torch.randn "
                    f"per-operation logit table (N, J, M)",
        "rounds": args.rounds, "parity": "sample == loop in makespan, raw return, solution and log-prob sum (bits), "
                                         "before timing and every round",
        "ms_per_batch": {name: {"median": med[name], "min": min(v), "max": max(v), "runs": v} for name, v in ms.items()},
        "episodes_per_s": {name: N / (med[name] * 1e-3) for name in ms},
        "decisions_per_batch": decisions,
        "decisions_per_s": {name: decisions[name] / (med[name] * 1e-3) for name in ms},
        "ratio_vs_sample": {name: med[name] / med["sample"] for name in ms},
        "mean_makespan": mean_makespan, "mean_log_prob": mean_log_prob, "envs_error": err,
        "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
