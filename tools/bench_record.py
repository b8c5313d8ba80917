#!/usr/bin/env python
"""Collecting a rollout from policy logits, timed on the headline batch (ta80, N = 65 536, auto-reset, pre-rolled like
bench.py's headline) or, with --mixed, on bench.py's cfg5 batch (env i runs ta((i mod 80) + 1)), from one seeded
torch.randn (N, J+1) fp32 logits tensor, writing into K-slot trajectory buffers (step k goes to slot k mod K):

  record: JssVecEnv.step_logits_record (jss_step_logits_record): draw + step, the observation, mask and scalar record
          written straight into the slot, one launch;
  copy:   what a collector writes without it: step_logits() into the slot's actions / log_prob, then torch copies of
          real_obs, action_mask, reward, reward_raw, done and time into the slot;
  logits: step_logits() alone, on the same env and logits (what record adds to the plain logits step, in one session).

Two twin envs first run K steps the record and the copy way from the same state and logits, and the two trajectories
must be bit-identical.  Then the three paths are timed with CUDA events over --steps steps each, in --rounds
alternating rounds; the JSON line gives each path's median and range over the rounds in microseconds per step, the
bytes each moves per env-step (mean over the batch) and the card.  --profile adds, from a separate torch.profiler run
of 100 steps per path, the mean device time per step of each kernel.  Writes nothing.

  python tools/bench_record.py [--envs N] [--instance ta80 | --mixed] [--steps S] [--rounds R] [--slots K] [--warmup W]
                               [--profile] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import TA80_EPISODE, gpu_info, preroll   # noqa: E402
from bench_logits import logits_step_bytes           # noqa: E402

FIELDS = ("real_obs", "action_mask", "actions", "log_prob", "reward", "reward_raw", "done", "time")


def record_step_bytes(J, M):
    """HBM bytes a jss_step_logits_record launch moves per env-step (J <= 128): those of jss_step_logits, plus the mask
    row and the 16-byte scalar record written a second time (to the slot as well as to the env's buffers)."""
    return logits_step_bytes(J, M) + ((J + 1 + 3) & ~3) + 16


def copy_step_bytes(J, M):
    """jss_step_logits plus the collector's copies, each read once and written once: the observation (28 J), the mask
    (J + 1 bools) and the reward, raw reward, done and time fields (4 + 4 + 1 + 4)."""
    return logits_step_bytes(J, M) + 2 * (28 * J + (J + 1) + 13)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--instance", default="ta80")
    ap.add_argument("--mixed", action="store_true", help="bench.py's cfg5 batch: env i runs ta((i mod 80) + 1)")
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import numpy as np
    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    N, K = args.envs, args.slots
    if args.mixed:
        cfg = {"instance_paths": ["ta%02d" % (k + 1) for k in range(80)], "env_to_instance": np.arange(N) % 80}
    else:
        cfg = {"instance_path": args.instance}
    envs = [JssVecEnv(N, cfg, device=args.device, auto_reset=True, seed=1234) for _ in range(2)]
    J, M = envs[0].jobs, envs[0].machines
    for env in envs:
        env.reset()
        preroll(env, "RANDOM", TA80_EPISODE if args.mixed or J * M >= 2000 else int(1.13 * J * M), torch)
    rec_env, copy_env = envs
    logits = torch.randn((N, J + 1), device=rec_env.device, generator=torch.Generator(device=rec_env.device).manual_seed(0))
    rec_traj, copy_traj = rec_env.logits_trajectory(K), copy_env.logits_trajectory(K)
    acts = torch.empty(N, dtype=torch.int32, device=rec_env.device)
    logp = torch.empty(N, dtype=torch.float32, device=rec_env.device)

    def record(k):
        rec_env.step_logits_record(logits, rec_traj, k % K)

    def copy(k):
        k %= K
        copy_env.step_logits(logits, actions_out=copy_traj["actions"][k], log_prob_out=copy_traj["log_prob"][k])
        copy_traj["real_obs"][k + 1].copy_(copy_env.real_obs)
        copy_traj["action_mask"][k + 1].copy_(copy_env.action_mask)
        for f, src in (("reward", copy_env.reward), ("reward_raw", copy_env.reward_raw), ("done", copy_env.done),
                       ("time", copy_env.current_time_step)):
            copy_traj[f][k].copy_(src)

    def plain(k):
        copy_env.step_logits(logits, actions_out=acts, log_prob_out=logp)

    # the same K transitions both ways from the same state: bit-identical trajectories (every env changes in every step
    # -- auto-reset, finite logits -- so the copied rewards equal the recorded ones too)
    for k in range(K):
        record(k)
        copy(k)
    torch.cuda.synchronize()

    def bits(t):
        return t.view(torch.int32) if t.dtype == torch.float32 else t
    mismatched = [f for f in FIELDS if not torch.equal(bits(rec_traj[f]), bits(copy_traj[f]))]
    if mismatched:
        raise SystemExit(f"record and copy trajectories differ in {mismatched}")

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

    paths = {"record": record, "copy": copy, "logits": plain}
    us = {name: [] for name in paths}
    for _ in range(args.rounds):
        for name, fn in paths.items():
            us[name].append(timed(fn))
    kernels = {}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name, fn in paths.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for k in range(100):
                    fn(k)
                torch.cuda.synchronize()
            kernels[name] = {
                e.key[:80]: round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 100, 2)
                for e in prof.key_averages() if getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) > 0}
    jm = list(zip(rec_env.env_jobs.tolist(), rec_env.env_machines.tolist()))
    b_rec = float(np.mean([record_step_bytes(j, m) for j, m in jm]))
    b_copy = float(np.mean([copy_step_bytes(j, m) for j, m in jm]))
    b_plain = float(np.mean([logits_step_bytes(j, m) for j, m in jm]))
    for env in envs:
        env.close()
    med = {name: statistics.median(v) for name, v in us.items()}
    out = {
        "workload": ("cfg5 mixed ta01..ta80" if args.mixed else f"{args.instance} ({J}x{M})") +
                    f" N={N}, auto-reset, pre-rolled like bench.py; actions drawn from one fixed torch.randn (N, J+1) "
                    f"fp32 logits tensor; {K}-slot trajectory",
        "steps_per_round": args.steps, "rounds": args.rounds,
        "us_per_step": {name: {"median": med[name], "min": min(v), "max": max(v), "runs": v} for name, v in us.items()},
        "speedup_record_vs_copy": med["copy"] / med["record"],
        "record_over_logits": med["record"] / med["logits"], "trajectories_identical": True,
        "bytes_per_env_step": {"record": b_rec, "copy": b_copy, "logits": b_plain},
        "achieved_GBps": {"record": b_rec * N / (med["record"] * 1e-6) / 1e9,
                          "copy": b_copy * N / (med["copy"] * 1e-6) / 1e9,
                          "logits": b_plain * N / (med["logits"] * 1e-6) / 1e9},
        "gpu": gpu_info(args.device)}
    if kernels:
        out["kernel_us_per_step"] = kernels
    print(json.dumps(out))


if __name__ == "__main__":
    main()
