#!/usr/bin/env python
"""Every legal action valued by a dispatching-rule rollout to the end of the episode (JssVecEnv.lookahead,
jss_lookahead), timed against the loop a caller writes without it:

  fused: env.lookahead(rule, coin="device"), one launch per lane class;
  loop:  per candidate column a: import_state(snapshot), step(a) on every env, rollout(rule, 2JM+1, write_obs=False)
         and a torch.where of current_time_step into column a (a legal and the env done, else -1).

Workloads: ta80 at N = 4 096 from reset and after a fixed 500-decision random pre-roll (the batch fills the GPU:
one work item per tile), ta80 at N = 32 (each env's candidates split over several work items), and ta01 at
N = 65 536.  Each round runs both paths with CUDA events around work that ends in a device synchronise, alternating,
and checks that the two tables are bit-identical.  Decisions per call are counted on the device, in an untimed pass:
the loop env's episode step statistics over rollouts of the candidate envs alone (import_state with a mask).  The
JSON line gives, per workload, each path's median and range in ms per call, candidate rollouts/s, decisions/s and the
speedup, with the card and its power limit.  Writes nothing.

  python tools/bench_lookahead.py [--rule MWR] [--rounds R] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402

WORKLOADS = (("ta80", 4096, 0), ("ta80", 4096, 500), ("ta80", 32, 0), ("ta01", 65536, 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rule", default="MWR")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    results = []
    for inst, n, preroll in WORKLOADS:
        fused, loop = (JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
                       for _ in range(2))
        J, M = fused.jobs, fused.machines
        bound = 2 * J * M + 1
        for env in (fused, loop):
            env.reset()
            for _ in range(preroll):
                env.step(env.policy("RANDOM"))
        si = fused._step_index
        snap = {k: v.clone() for k, v in loop.export_state().items()}
        legal = (loop.action_mask[:, :J + 1] != 0) & ~loop.done[:, None]
        n_cand = int(legal.sum())
        out = torch.empty((n, J + 1), dtype=torch.int32, device=fused.device)
        table = torch.empty_like(out)

        def run_fused():
            fused._step_index = si
            fused.lookahead(args.rule, "device", out=out)

        def run_loop(root=None, mask=False):
            if root is None:                             # the caller's snapshot of the root state
                root = {k: v.clone() for k, v in loop.export_state().items()}
            for a in range(J + 1):
                loop.import_state(root, mask=legal[:, a] if mask else None)
                loop.step(torch.full((n,), a, dtype=torch.int32, device=loop.device))
                loop._step_index = si
                loop.rollout(args.rule, bound, write_obs=False)
                table[:, a] = torch.where(legal[:, a] & loop.done, loop.current_time_step, -1)
            loop.import_state(root)

        # decisions per call, counted on the device: only the candidate envs take decisions (every other env is
        # left done by a first rollout, and a masked import restores the candidates alone)
        loop._step_index = si
        loop.rollout(args.rule, bound, write_obs=False)
        steps0 = loop.stats()["steps"]
        run_loop(snap, mask=True)
        decisions = loop.stats()["steps"] - steps0

        def timed(fn):
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            fn()
            ev1.record()
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1)

        ms = {"fused": [], "loop": []}
        for _ in range(args.rounds):
            ms["fused"].append(timed(run_fused))
            ms["loop"].append(timed(run_loop))
            if not torch.equal(out, table):
                raise SystemExit(f"{inst} N={n} pre-roll {preroll}: the fused and loop tables differ")
        med = {k: statistics.median(v) for k, v in ms.items()}
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n}, {preroll} random decisions before the call, rule {args.rule}, "
                        f"coin device",
            "candidates": n_cand, "decisions_per_call": decisions,
            "ms_per_call": {k: {"median": med[k], "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()},
            "candidate_rollouts_per_s": {k: n_cand / (med[k] * 1e-3) for k in ms},
            "decisions_per_s": {k: decisions / (med[k] * 1e-3) for k in ms},
            "speedup_fused_vs_loop": med["loop"] / med["fused"],
            "parity": "fused table == loop table, every round"})
        for env in (fused, loop):
            env.close()
    print(json.dumps({"rounds": args.rounds, "results": results, "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
