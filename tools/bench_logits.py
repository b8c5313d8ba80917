#!/usr/bin/env python
"""Stepping from policy logits, timed two ways on the headline batch (ta80, N = 65 536, auto-reset, pre-rolled like
bench.py's headline), from the same seeded torch.randn (N, J+1) fp32 logits tensor, CUDA events over --steps steps:

  fused: JssVecEnv.step_logits (jss_step_logits): masked Gumbel-max draw + log_prob + step, one launch;
  torch: what a caller writes without it: masked_fill(~mask, -inf), Categorical(logits=...).sample() and .log_prob(),
         .int(), step().

Prints one JSON line with the microseconds per step of each, the bytes the fused launch moves per env-step and its
achieved rate.  Writes nothing.

  python tools/bench_logits.py [--envs N] [--instance ta80] [--steps K] [--warmup W] [--device D]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import TA80_EPISODE, gpu_info, preroll   # noqa: E402


def logits_step_bytes(J, M):
    """HBM bytes a jss_step_logits launch moves per env-step (J <= 128): the state block read and written, real_obs,
    the mask row, the scalar record, the logits row (J + 1 floats) and the action and log_prob written."""
    jc, mc = (J + 3) & ~3, (M + 3) & ~3
    block = 4 * (2 * jc + ((jc + 7) & ~7) // 2 + mc + 8 + 4)      # jss_block_geom in csrc/jss_types.h
    return 2 * block + 28 * J + ((J + 1 + 3) & ~3) + 16 + 4 * (J + 1) + 4 + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--instance", default="ta80")
    ap.add_argument("--steps", type=int, default=2400)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    N = args.envs
    env = JssVecEnv(N, {"instance_path": args.instance}, device=args.device, auto_reset=True, seed=1234)
    J, M = env.jobs, env.machines
    env.reset()
    preroll(env, "RANDOM", TA80_EPISODE if J * M >= 2000 else int(1.13 * J * M), torch)
    logits = torch.randn((N, J + 1), device=env.device, generator=torch.Generator(device=env.device).manual_seed(0))
    acts = torch.empty(N, dtype=torch.int32, device=env.device)
    logp = torch.empty(N, dtype=torch.float32, device=env.device)
    mask = env.action_mask
    col0 = torch.zeros((1, J + 1), dtype=torch.bool, device=env.device)
    col0[0, 0] = True

    def fused():
        env.step_logits(logits, actions_out=acts, log_prob_out=logp)

    def torch_path():
        # a done env (auto-reset pending) has no legal action: it gets action 0, as from the fused call; without
        # argument validation (which would synchronise with the host every step)
        legal = mask | (col0 & ~mask.any(1, keepdim=True))
        d = torch.distributions.Categorical(logits=logits.masked_fill(~legal, float("-inf")), validate_args=False)
        a = d.sample()
        d.log_prob(a)
        env.step(a.int())

    def timed(fn):
        for _ in range(max(3, args.warmup)):
            fn()
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.steps):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) * 1e3 / args.steps

    us_fused = timed(fused)
    us_torch = timed(torch_path)
    env.close()
    nbytes = logits_step_bytes(J, M)
    print(json.dumps({
        "workload": f"{args.instance} ({J}x{M}) N={N}, auto-reset, pre-rolled like bench.py's headline; actions drawn "
                    "from one fixed torch.randn (N, J+1) fp32 logits tensor, masked by action_mask",
        "steps": args.steps, "fused_us_per_step": us_fused, "torch_us_per_step": us_torch,
        "speedup": us_torch / us_fused, "fused_bytes_per_env_step": nbytes,
        "fused_achieved_GBps": nbytes * N / (us_fused * 1e-6) / 1e9, "gpu": gpu_info(args.device),
        "fused": "jss_step_logits: Gumbel-max draw over the legal actions + log_prob + step, one launch",
        "torch": "masked_fill(~mask, -inf) -> Categorical(logits, validate_args=False).sample() / .log_prob() -> "
                 ".int() -> step()"}))


if __name__ == "__main__":
    main()
