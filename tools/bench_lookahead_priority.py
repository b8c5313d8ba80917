#!/usr/bin/env python
"""Every legal action valued by a greedy rollout of a caller's priority table to the end of the episode
(JssVecEnv.lookahead_priority, jss_lookahead_priority), timed against the loop a caller writes without it:

  fused: env.lookahead_priority(table), one launch per lane class;
  loop:  per candidate column a: import_state(snapshot), step(a) on every env, rollout_priority(table) and a
         torch.where of current_time_step into column a (a legal and the env done, else -1);
  and, for context, env.lookahead("MWR", "never") beside env.lookahead_priority(MWR table): the same values (checked
  bit for bit), so their difference in time is the cost of reading the table from L2 / HBM instead of the suffix sums
  from shared memory.

Workloads: ta80 at N = 4 096 from reset and after a fixed 500-decision random pre-roll, ta80 at N = 32 (each env's
candidates split over several work items), and ta01 at N = 65 536; each with a seeded per-env (N, J, M) table and a
seeded broadcast (1, J, M) table.  Each round runs every path with CUDA events around work that ends in a device
synchronise, alternating, and checks that the fused and loop values are bit-identical (and the MWR pair).  Decisions
per call are counted on the device, in an untimed pass: the loop env's episode step statistics over rollouts of the
candidate envs alone (import_state with a mask).  The JSON line gives, per workload and table, each path's median and
range in ms per call, candidate rollouts/s, decisions/s and the speedup, with the card and its power limit.  Writes
nothing.

  python tools/bench_lookahead_priority.py [--rounds R] [--device D]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402

WORKLOADS = (("ta80", 4096, 0), ("ta80", 4096, 500), ("ta80", 32, 0), ("ta01", 65536, 0))


def mwr_table(env):
    """MWR as a (1, J, M) priority table: the work remaining from each operation on (a uniform batch)."""
    import torch
    _, dur = env.instances[0]
    rem = dur[:, ::-1].cumsum(axis=1)[:, ::-1].copy()
    return torch.from_numpy(rem).to(torch.float32).to(env.device)[None]


def main():
    ap = argparse.ArgumentParser()
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
        for env in (fused, loop):
            env.reset()
            for _ in range(preroll):
                env.step(env.policy("RANDOM"))
        snap = {k: v.clone() for k, v in loop.export_state().items()}
        legal = (loop.action_mask[:, :J + 1] != 0) & ~loop.done[:, None]
        n_cand = int(legal.sum())
        gen = torch.Generator(device=fused.device).manual_seed(7)
        tables = {"per-env (N, J, M)": torch.rand((n, J, M), generator=gen, device=fused.device),
                  "broadcast (1, J, M)": torch.rand((1, J, M), generator=gen, device=fused.device)}
        out = torch.empty((n, J + 1), dtype=torch.int32, device=fused.device)
        values = torch.empty_like(out)

        def run_loop(table, root=None, mask=False):
            if root is None:                             # the caller's snapshot of the root state
                root = {k: v.clone() for k, v in loop.export_state().items()}
            for a in range(J + 1):
                loop.import_state(root, mask=legal[:, a] if mask else None)
                loop.step(torch.full((n,), a, dtype=torch.int32, device=loop.device))
                loop.rollout_priority(table)
                values[:, a] = torch.where(legal[:, a] & loop.done, loop.current_time_step, -1)
            loop.import_state(root)

        def timed(fn):
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            fn()
            ev1.record()
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1)

        for name, table in tables.items():
            # decisions per call, counted on the device: only the candidate envs take decisions (every other env is
            # left done by a first rollout, and a masked import restores the candidates alone)
            loop.rollout_priority(table)
            steps0 = loop.stats()["steps"]
            run_loop(table, snap, mask=True)
            decisions = loop.stats()["steps"] - steps0
            ms = {"fused": [], "loop": []}
            for _ in range(args.rounds):
                ms["fused"].append(timed(lambda: fused.lookahead_priority(table, out=out)))
                ms["loop"].append(timed(lambda: run_loop(table)))
                if not torch.equal(out, values):
                    raise SystemExit(f"{inst} N={n} pre-roll {preroll} {name}: the fused and loop values differ")
            med = {k: statistics.median(v) for k, v in ms.items()}
            results.append({
                "workload": f"{inst} ({J}x{M}) N={n}, {preroll} random decisions before the call, {name} table",
                "candidates": n_cand, "decisions_per_call": decisions,
                "ms_per_call": {k: {"median": med[k], "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()},
                "candidate_rollouts_per_s": {k: n_cand / (med[k] * 1e-3) for k in ms},
                "decisions_per_s": {k: decisions / (med[k] * 1e-3) for k in ms},
                "speedup_fused_vs_loop": med["loop"] / med["fused"],
                "parity": "fused values == loop values, every round"})

        # the rule MWR against the same rule as a table: same values, suffix sums in shared memory vs table reads
        mwr = mwr_table(fused)
        rule_out = torch.empty_like(out)
        ms = {"lookahead_rule": [], "lookahead_priority_table": []}
        for _ in range(args.rounds):
            ms["lookahead_rule"].append(timed(lambda: fused.lookahead("MWR", "never", out=rule_out)))
            ms["lookahead_priority_table"].append(timed(lambda: fused.lookahead_priority(mwr, out=out)))
            if not torch.equal(out, rule_out):
                raise SystemExit(f"{inst} N={n} pre-roll {preroll}: lookahead(MWR) and the MWR table differ")
        med = {k: statistics.median(v) for k, v in ms.items()}
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n}, {preroll} random decisions before the call, MWR rule vs (1, J, M) "
                        f"MWR table",
            "candidates": n_cand,
            "ms_per_call": {k: {"median": med[k], "min": min(v), "max": max(v), "runs": v} for k, v in ms.items()},
            "table_over_rule": med["lookahead_priority_table"] / med["lookahead_rule"],
            "parity": "lookahead(MWR, never) == lookahead_priority(MWR table), every round"})
        for env in (fused, loop):
            env.close()
    print(json.dumps({"rounds": args.rounds, "results": results, "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
