#!/usr/bin/env python
"""Sampling without replacement by stochastic beam search (JssVecEnv.sample_without_replacement,
jss_sample_without_replacement), timed against beam_search at the same width and sample_episodes at the same k:

  ta80, N = 256, k = 16, per-env random normal tables, from reset and after a fixed 500-decision random pre-roll;
  ta01, N = 4 096, k = 8, from reset;
  the backward (jss_order_log_prob_grad on the returned orders) against sample_episodes' backward (the replayed draws),
  ta01, N = 4 096, k = 8, unit weights.

Before timing, every slot's order is checked by replay: rollout_priority(-order) on a twin in the same state ends done
at that slot's makespan.  Each round runs every path with CUDA events around work that ends in a device synchronise,
alternating; the line gives each path's median and range in ms per call.

Decode quality: ta41..ta80, one env each, from reset, the table x[j][k] = (work remaining in job j from operation k
on) / (T * mean duration) at T = 0.5, 0.05 and 0.01: the mean best makespan of greedy decoding (rollout_priority),
best-of-k sampling (sample_episodes), beam search and SWOR at k = 4 and 16, and sample_episodes' duplicate rate, the
share of its k samples per env whose (makespan, log_prob) pair equals an earlier sample's.  Writes nothing.

  python tools/bench_sample_without_replacement.py [--rounds R] [--device D]

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (CUDA 12.9 build, median of three rounds, ms per call):

  workload                                   SWOR     beam_search   sample_episodes
  ta80, N = 256, k = 16, from reset          38.7     30.5          9.15
  ta80, N = 256, k = 16, after 500 random    29.8     23.7          7.26
  ta01, N = 4 096, k = 8, from reset         11.1     9.11          4.45
  ta01, N = 4 096, k = 8, backward           5.59 (order_log_prob_grad)    5.87 (sample_episodes' replay)

  mean best makespan, ta41..ta80    greedy    best-of-k   beam     SWOR     sample_episodes duplicates
  T = 0.5,  k = 4                   3706.7    3670.1      3698.5   3668.6   0
  T = 0.5,  k = 16                  3706.7    3637.2      3697.9   3627.6   0
  T = 0.05, k = 4                   3706.7    3673.5      3702.8   3672.1   0
  T = 0.05, k = 16                  3706.7    3654.6      3695.8   3654.8   0
  T = 0.01, k = 4                   3706.7    3683.6      3694.0   3683.8   1.9 %
  T = 0.01, k = 16                  3706.7    3668.0      3689.8   3670.8   8.9 %
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402
from tools.bench_beam_search import remaining_work_table, timed   # noqa: E402


def replay_check(env, out, what):
    """Every complete slot's order replays via rollout_priority(-order) on a twin in env's state to its makespan."""
    import torch
    from jssenv_b200 import JssVecEnv
    twin = JssVecEnv(env.num_envs, {"instance_paths": list(env.instances), "env_to_instance": list(env.env_to_instance)},
                     device=env.device_index, auto_reset=False, seed=env.seed)
    twin.reset()
    snap = {k: v.clone() for k, v in env.export_state().items()}
    for s in range(out["makespan"].shape[1]):
        full = out["makespan"][:, s] >= 0
        twin.import_state(snap)
        twin.rollout_priority(-out["order"][:, s].float())
        if not (bool(full.all()) and bool(twin.done.all()) and torch.equal(twin.current_time_step,
                                                                            out["makespan"][:, s])):
            raise SystemExit(f"{what}: slot {s} does not replay to its makespan")
    twin.close()


def duplicate_rate(out):
    """The share of samples whose (makespan, log_prob) pair equals an earlier sample's of the same env."""
    ms, lp = out["makespan"].cpu().numpy(), out["log_prob"].detach().cpu().numpy()
    dup = 0
    for i in range(ms.shape[0]):
        dup += ms.shape[1] - len(set(zip(ms[i].tolist(), lp[i].view("uint32").tolist())))
    return dup / ms.size


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
    for inst, n, k, preroll in (("ta80", 256, 16, 0), ("ta80", 256, 16, 500), ("ta01", 4096, 8, 0)):
        env = JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
        J, M = env.jobs, env.machines
        env.reset()
        for _ in range(preroll):
            env.step(env.policy("RANDOM"))
        table = torch.randn((n, J, M), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
        out = env.sample_without_replacement(table, k, order=True)
        replay_check(env, out, f"{inst} N={n} k={k}")
        lp, _ = env.order_log_prob(table, out["order"])
        if not torch.equal(lp, out["log_prob"]):
            raise SystemExit("order_log_prob does not equal the slots' log_prob")
        ms = {"sample_without_replacement": [], "beam_search": [], "sample_episodes": []}
        env.beam_search(table, k)                       # one untimed call of each path first
        env.sample_episodes(table, k)
        for _ in range(args.rounds):
            ms["sample_without_replacement"].append(timed(lambda: env.sample_without_replacement(table, k)))
            ms["beam_search"].append(timed(lambda: env.beam_search(table, k)))
            ms["sample_episodes"].append(timed(lambda: env.sample_episodes(table, k)))
        med = {key: statistics.median(v) for key, v in ms.items()}
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n} k={k}, {preroll} random decisions before the call, per-env (N, J, M) "
                        f"random normal table",
            "ms_per_call": {key: {"median": med[key], "min": min(v), "max": max(v), "runs": v} for key, v in ms.items()},
            "parity": "every slot's order replays to its makespan; order_log_prob equals log_prob bit for bit"})
        if inst == "ta01":
            w = torch.ones((n, k), device=dev)
            bw = {"sample_without_replacement_backward": [], "sample_episodes_backward": []}
            for warm in [True] + [False] * args.rounds:   # the first pass untimed: it carries the process's one-time
                x = table.clone().requires_grad_(True)    # setup of the first backward
                o = env.sample_without_replacement(x, k)
                t = timed(lambda: o["log_prob"].backward(w))
                if not warm:
                    bw["sample_without_replacement_backward"].append(t)
                x = table.clone().requires_grad_(True)
                o = env.sample_episodes(x, k)
                t = timed(lambda: o["log_prob"].backward(w))
                if not warm:
                    bw["sample_episodes_backward"].append(t)
            results[-1]["backward_ms"] = {key: {"median": statistics.median(v), "min": min(v), "max": max(v),
                                               "runs": v} for key, v in bw.items()}
        env.close()

    names = [f"ta{i}" for i in range(41, 81)]
    quality = {}
    for temp in (0.5, 0.05, 0.01):
        for k in (4, 16):
            env = JssVecEnv(len(names), {"instance_paths": names, "env_to_instance": list(range(len(names)))},
                            device=args.device, auto_reset=False, seed=3)
            table = torch.from_numpy(remaining_work_table(names, env.jobs, env.machines, temp)).to(dev)
            env.reset()

            def best(o):
                return o["makespan"].gather(1, o["best"][:, None])[:, 0]
            beam = best(env.beam_search(table, k))
            samp_out = env.sample_episodes(table, k)
            samp = best(samp_out)
            sw = best(env.sample_without_replacement(table, k))
            env.rollout_priority(table)
            g = env.current_time_step.clone()
            if not (bool((beam > 0).all()) and bool((samp > 0).all()) and bool((sw > 0).all())
                    and bool(env.done.all())):
                raise SystemExit("decode quality: a decode did not finish")
            quality[f"T={temp} k={k}"] = {
                "greedy": float(g.double().mean()), "best_of_k_samples": float(samp.double().mean()),
                "beam_search": float(beam.double().mean()), "swor": float(sw.double().mean()),
                "sample_episodes_duplicate_rate": duplicate_rate(samp_out)}
            env.close()
    print(json.dumps({"rounds": args.rounds, "results": results,
                      "decode_quality_ta41_ta80_mean_best_makespan": {
                          "table": "remaining work / (T * mean duration)", **quality},
                      "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
