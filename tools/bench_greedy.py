#!/usr/bin/env python
"""Greedy and epsilon-greedy stepping from action scores, timed on the headline batch (ta80, N = 65 536, auto-reset,
pre-rolled like bench.py's headline), from one seeded torch.randn (N, J+1) fp32 score tensor:

  greedy:      JssVecEnv.step_greedy(scores, 0) (jss_step_greedy): masked argmax + step, one launch;
  greedy_0.05: step_greedy(scores, 0.05): the epsilon-greedy behaviour policy of a value-based agent, one launch;
  torch:       what a user writes without it: scores.masked_fill(~action_mask, -inf).argmax(1).int(), then step();
  logits:      step_logits(scores), the masked categorical draw, on the same env and scores.

Two twin envs first run --check steps the greedy and the torch way from the same state and scores; the actions and
every env output must be bit-identical after every step.  Then the four paths are timed with CUDA events over --steps
steps each, in --rounds alternating rounds; the JSON line gives each path's median and range over the rounds in
microseconds per step, the achieved bandwidth of the fused paths for the bytes a ta80 env-step moves (those of
jss_step_logits: the scores row is read as the logits row is), and the card.  Writes nothing.

  python tools/bench_greedy.py [--envs N] [--instance ta80] [--steps S] [--rounds R] [--check C] [--warmup W]
                               [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import TA80_EPISODE, gpu_info, preroll   # noqa: E402
from bench_logits import logits_step_bytes           # noqa: E402

OUTPUTS = ("real_obs", "action_mask", "reward", "reward_raw", "done", "current_time_step", "flags", "episode_count",
           "last_makespan", "last_return")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--instance", default="ta80")
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--check", type=int, default=64, help="steps of the greedy / torch equality check")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import numpy as np
    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    N = args.envs
    envs = [JssVecEnv(N, {"instance_path": args.instance}, device=args.device, auto_reset=True, seed=1234)
            for _ in range(2)]
    J, M = envs[0].jobs, envs[0].machines
    for env in envs:
        env.reset()
        preroll(env, "RANDOM", TA80_EPISODE if J * M >= 2000 else int(1.13 * J * M), torch)
    fused_env, torch_env = envs
    scores = torch.randn((N, J + 1), device=fused_env.device,
                         generator=torch.Generator(device=fused_env.device).manual_seed(0))
    acts = torch.empty(N, dtype=torch.int32, device=fused_env.device)
    logp = torch.empty(N, dtype=torch.float32, device=fused_env.device)
    ninf = torch.tensor(float("-inf"), device=fused_env.device)

    def greedy(eps):
        def fn(k):
            fused_env.step_greedy(scores, eps, actions_out=acts, log_prob_out=logp)
        return fn

    def torch_path(k):
        torch_env.step(scores.masked_fill(~torch_env.action_mask, ninf).argmax(1).int())

    def logits(k):
        fused_env.step_logits(scores, actions_out=acts, log_prob_out=logp)

    # the same transitions both ways from the same state: bit-identical actions and env outputs
    def bits(t):
        return t.view(torch.int32) if t.dtype == torch.float32 else t
    for k in range(args.check):
        want = scores.masked_fill(~torch_env.action_mask, ninf).argmax(1).int()
        torch_env.step(want)
        greedy(0.0)(k)
        if not torch.equal(acts, want):
            raise SystemExit(f"step {k}: greedy and torch actions differ")
        bad = [f for f in OUTPUTS if not torch.equal(bits(getattr(fused_env, f)), bits(getattr(torch_env, f)))]
        if bad:
            raise SystemExit(f"step {k}: greedy and torch envs differ in {bad}")
    torch.cuda.synchronize()

    def timed(fn):
        for k in range(max(3, args.warmup)):
            fn(k)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for k in range(args.steps):
            fn(k)
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) * 1e3 / args.steps

    paths = {"greedy": greedy(0.0), "greedy_0.05": greedy(0.05), "torch": torch_path, "logits": logits}
    us = {name: [] for name in paths}
    for _ in range(args.rounds):
        for name, fn in paths.items():
            us[name].append(timed(fn))
    b = float(np.mean([logits_step_bytes(j, m) for j, m in zip(fused_env.env_jobs.tolist(),
                                                                 fused_env.env_machines.tolist())]))
    for env in envs:
        env.close()
    med = {name: statistics.median(v) for name, v in us.items()}
    print(json.dumps({
        "workload": f"{args.instance} ({J}x{M}) N={N}, auto-reset, pre-rolled like bench.py; actions decoded from one "
                    f"fixed torch.randn (N, J+1) fp32 score tensor",
        "steps_per_round": args.steps, "rounds": args.rounds, "greedy_equals_torch_steps": args.check,
        "us_per_step": {name: {"median": med[name], "min": min(v), "max": max(v), "runs": v} for name, v in us.items()},
        "speedup_greedy_vs_torch": med["torch"] / med["greedy"],
        "greedy_over_logits": med["greedy"] / med["logits"],
        "bytes_per_env_step": b,
        "achieved_GBps": {name: b * N / (med[name] * 1e-6) / 1e9 for name in ("greedy", "greedy_0.05", "logits")},
        "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
