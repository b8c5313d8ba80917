#!/usr/bin/env python
"""Beam search over a caller's logit table, the envs left untouched (JssVecEnv.beam_search, jss_beam_search), timed
against what a caller does without it, a torch loop over a batch of N*W envs that at every round exports the state,
gathers the table at todo, takes a log-softmax and the W best candidates per env (score, then parent slot, then job),
imports the chosen parents into their slots and steps:

  ta80, N = 256, W = 16, per-env random normal tables, from reset and after a fixed 500-decision random pre-roll;
  ta01, N = 4 096, W = 8, from reset.

Before timing, the fused outputs are checked by replay: rollout_priority(-order) on a twin in the same state ends done
at makespan[best] for every env.  The loop's log-softmax is torch's, not the kernel's fast exp / log, so the JSON line
reports how many envs' makespan rows it matches rather than requiring all.  Decisions per call are the operations not
yet started, summed over the envs, times W.  Each round runs both paths with CUDA events around work that ends in a
device synchronise, alternating; the line gives each path's median and range in ms per call and decisions/s.

Decode quality: ta41..ta80, one env each, from reset, the table x[j][k] = (work remaining in job j from operation k
on) / (T * mean duration) with T = 0.5: the mean best makespan of greedy decoding (rollout_priority), best-of-W sampling
(sample_episodes, k = W) and beam search at W, for W = 4 and 16.  Writes nothing.

  python tools/bench_beam_search.py [--rounds R] [--device D]
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


def replay_check(env, out, what):
    """rollout_priority(-order) on a twin in env's state ends done at makespan[best] in every env."""
    import torch
    from jssenv_b200 import JssVecEnv
    twin = JssVecEnv(env.num_envs, {"instance_paths": list(env.instances), "env_to_instance": list(env.env_to_instance)},
                     device=env.device_index, auto_reset=False, seed=env.seed)
    twin.reset()
    twin.import_state({k: v.clone() for k, v in env.export_state().items()})
    twin.rollout_priority(-out["order"].float())
    best = out["best"]
    want = out["makespan"].gather(1, best.clamp(min=0)[:, None])[:, 0]
    if not (bool((best >= 0).all()) and bool(twin.done.all()) and torch.equal(twin.current_time_step, want)):
        raise SystemExit(f"{what}: the best order does not replay to makespan[best]")
    twin.close()


def torch_loop(loop, table, W, snap, R):
    """The beam search a caller writes without the kernel, on `loop`, a batch of N*W envs.  Returns the makespans
    (N, W), -1 for an empty slot."""
    import torch
    n, J, M = table.shape
    dev = table.device
    ar = torch.arange(n, device=dev)
    loop.import_state({k: v.repeat_interleave(W, 0) for k, v in snap.items()})
    score = torch.full((n, W), float("-inf"), device=dev)
    score[:, 0] = 0.0
    jobs_i = torch.as_tensor(loop.env_jobs, device=dev, dtype=torch.int32)
    tab = table[:, None].expand(n, W, J, M)
    for r in range(int(R.max())):
        act_on = (R > r)[:, None].expand(n, W)
        live = score > float("-inf")
        while True:                                       # forced no-ops
            x = loop.export_state()
            legal = x["legal"][:, :J].bool().view(n, W, J)
            noop = ((x["flags"] >> 8) & 4).bool().view(n, W)
            need = live & act_on & ~legal.any(2) & noop
            if not bool(need.any()):
                break
            loop.step(torch.where(need.reshape(-1), jobs_i, -1).to(torch.int32))
        todo = x["todo"][:, :J].long().view(n, W, J).clamp(max=M - 1)
        v = tab.gather(3, todo[..., None])[..., 0].masked_fill(~legal, float("-inf"))
        cand = (score[..., None] + torch.log_softmax(v, 2)).masked_fill(~live[..., None], float("-inf"))
        vals, idx = torch.sort(cand.reshape(n, W * J), dim=1, descending=True, stable=True)
        new_score, top = vals[:, :W], idx[:, :W]
        parent, job = top // J, (top % J).to(torch.int32)
        keep = act_on & (new_score > float("-inf"))
        parent = torch.where(act_on, parent, torch.arange(W, device=dev)[None])
        score = torch.where(act_on, new_score, score)
        rows = (ar[:, None] * W + parent).reshape(-1)
        loop.import_state({k: v[rows] for k, v in x.items()})
        loop.step(torch.where(keep, job, -1).reshape(-1))
    ended = loop.done.view(n, W) & (score > float("-inf"))
    return torch.where(ended, loop.current_time_step.view(n, W), -1)


def remaining_work_table(names, J, M, temperature):
    import numpy as np
    from jssenv_b200.instances import load_instance
    t = np.full((len(names), J, M), -1e4, np.float32)
    for i, name in enumerate(names):
        _, dur = load_instance(name)
        rem = np.cumsum(dur[:, ::-1], 1)[:, ::-1]
        t[i, :dur.shape[0], :dur.shape[1]] = rem / (temperature * dur.mean())
    return t


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
    for inst, n, W, preroll in (("ta80", 256, 16, 0), ("ta80", 256, 16, 500), ("ta01", 4096, 8, 0)):
        env = JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
        loop = JssVecEnv(n * W, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
        J, M = env.jobs, env.machines
        env.reset()
        loop.reset()
        for _ in range(preroll):
            env.step(env.policy("RANDOM"))
        snap = {k: v.clone() for k, v in env.export_state().items()}
        R = undrawn_ops(env)
        decisions = int(R.sum()) * W
        table = torch.randn((n, J, M), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
        out = env.beam_search(table, W, order=True)
        replay_check(env, out, f"{inst} N={n} W={W}")
        ref = torch_loop(loop, table, W, snap, R)
        agree = int((ref == out["makespan"]).all(1).sum())
        ms = {"beam_search": [], "torch_loop": []}
        for _ in range(args.rounds):
            ms["beam_search"].append(timed(lambda: env.beam_search(table, W)))
            ms["torch_loop"].append(timed(lambda: torch_loop(loop, table, W, snap, R)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n} W={W}, {preroll} random decisions before the call, per-env (N, J, M) "
                        f"random normal table, against the torch loop on {n * W} envs",
            "decisions_per_call": decisions,
            "ms_per_call": {k: {"median": med[k], "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()},
            "decisions_per_s": {k: decisions / (med[k] * 1e-3) for k in ms},
            "speedup_beam_search_vs_torch_loop": med["torch_loop"] / med["beam_search"],
            "parity": "best order replays to makespan[best] in every env",
            "torch_loop_rows_equal": f"{agree}/{n}"})
        env.close()
        loop.close()

    names = [f"ta{k}" for k in range(41, 81)]
    quality = {}
    for W in (4, 16):
        env = JssVecEnv(len(names), {"instance_paths": names, "env_to_instance": list(range(len(names)))},
                        device=args.device, auto_reset=False, seed=3)
        table = torch.from_numpy(remaining_work_table(names, env.jobs, env.machines, 0.5)).to(dev)
        env.reset()
        beam = env.beam_search(table, W)
        b = beam["makespan"].gather(1, beam["best"][:, None])[:, 0]
        samp = env.sample_episodes(table, W)
        s = samp["makespan"].gather(1, samp["best"][:, None])[:, 0]
        env.rollout_priority(table)
        g = env.current_time_step.clone()
        if not (bool((b > 0).all()) and bool((s > 0).all()) and bool(env.done.all())):
            raise SystemExit("decode quality: a decode did not finish")
        quality[f"W={W}"] = {"greedy": float(g.double().mean()), f"best_of_{W}_samples": float(s.double().mean()),
                             f"beam_{W}": float(b.double().mean())}
        env.close()
    print(json.dumps({"rounds": args.rounds, "results": results,
                      "decode_quality_ta41_ta80_mean_best_makespan": {
                          "table": "remaining work / (0.5 * mean duration)", **quality},
                      "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
