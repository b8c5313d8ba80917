#!/usr/bin/env python
"""Every legal action valued by k episodes drawn from a caller's logit table after it (JssVecEnv.lookahead_sample,
jss_lookahead_sample), timed against the loop a caller writes without it:

  fused: env.lookahead_sample(table, k), one launch per lane class;
  loop:  per candidate column a: import_state(snapshot), step(a) on every env, sample_episodes(table, k) at the same
         RNG counter, and a torch.where of its makespans into column a (a legal; the end time in every sample where
         the step alone ends the episode; else -1).

Workloads: ta80 at N = 256, k = 16 from reset and after a fixed 500-decision random pre-roll, and ta01 at N = 4 096,
k = 8 from reset, each with a seeded per-env (N, J, M) table.  One untimed call of each path first, checked bit for
bit; then each round runs both paths, alternating, with CUDA events around work that ends in a device synchronise, and
checks them bit for bit again.  The JSON line gives, per workload, each path's median and range in ms per call, the
(legal candidate, sample) pairs per call and per second and the speedup, with the card and its power limit.  Writes
nothing.

  python tools/bench_lookahead_sample.py [--rounds R] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402

WORKLOADS = (("ta80", 256, 16, 0), ("ta80", 256, 16, 500), ("ta01", 4096, 8, 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    results = []
    for inst, n, k, preroll in WORKLOADS:
        fused, loop = (JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
                       for _ in range(2))
        J, M = fused.jobs, fused.machines
        for env in (fused, loop):
            env.reset()
            for _ in range(preroll):
                env.step(env.policy("RANDOM"))
        legal = (loop.action_mask[:, :J + 1] != 0) & ~loop.done[:, None]
        pairs = int(legal.sum()) * k
        si = fused._step_index
        table = torch.randn((n, J, M), generator=torch.Generator(device=fused.device).manual_seed(7),
                            device=fused.device)
        out = torch.empty((n, J + 1, k), dtype=torch.int32, device=fused.device)
        values = torch.empty_like(out)

        def run_fused():
            fused._step_index = si
            fused.lookahead_sample(table, k, out=out)

        def run_loop():
            root = {key: v.clone() for key, v in loop.export_state().items()}   # the caller's snapshot
            for a in range(J + 1):
                loop.import_state(root)
                loop.step(torch.full((n,), a, dtype=torch.int32, device=loop.device))
                done, t = loop.done.clone(), loop.current_time_step.clone()
                loop._step_index = si
                ms = loop.sample_episodes(table, k)["makespan"]
                col = torch.where(done[:, None], t[:, None].to(torch.int32), ms)
                values[:, a] = torch.where(legal[:, a, None], col, -1)
            loop.import_state(root)

        def timed(fn):
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            fn()
            ev1.record()
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1)

        def check(when):
            if not torch.equal(out, values):
                raise SystemExit(f"{inst} N={n} k={k} pre-roll {preroll} ({when}): the fused and loop values differ")

        run_fused()
        run_loop()
        torch.cuda.synchronize()
        check("untimed call")
        ms = {"fused": [], "loop": []}
        for _ in range(args.rounds):
            ms["fused"].append(timed(run_fused))
            ms["loop"].append(timed(run_loop))
            check("timed round")
        med = {key: statistics.median(v) for key, v in ms.items()}
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n}, k={k}, {preroll} random decisions before the call, per-env (N, J, M) "
                        f"table",
            "candidate_sample_pairs": pairs,
            "ms_per_call": {key: {"median": med[key], "min": min(v), "max": max(v), "runs": v} for key, v in ms.items()},
            "pairs_per_s": {key: pairs / (med[key] * 1e-3) for key in ms},
            "speedup_fused_vs_loop": med["loop"] / med["fused"],
            "parity": "fused values == loop values, untimed call and every round"})
        for env in (fused, loop):
            env.close()
    print(json.dumps({"rounds": args.rounds, "results": results, "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
