#!/usr/bin/env python
"""A static priority rule run to the end of every episode, timed on ta80 at N = 65 536 from reset, with a seeded
random priority table:

  fused_op:    JssVecEnv.rollout_priority(P) with per-operation priorities P (N, J, M) (jss_rollout_priority), one
               call to the end of every episode;
  loop_op:     the same table the only way possible without it: per decision, export_state(), a torch gather of P at
               todo, the no-op column at -inf, then step_greedy(rows);
  fused_job:   rollout_priority with per-job priorities (N, J, 1);
  loop_job:    the step_greedy loop on the static row of the same per-job priorities.

The loops check every --poll decisions whether every env is done.  Every round resets the envs, runs each path with
CUDA events around work that ends in a device synchronise, and checks that fused_op and loop_op, and fused_job and
loop_job, left bit-identical makespans, raw returns and solutions.  The JSON line gives each path's median and range
over --rounds alternating rounds, in ms per batch, episodes/s and decisions/s (from the summed per-env episode step
counts), and the card with its power limit.  Writes nothing.

  python tools/bench_priority.py [--envs N] [--instance ta80] [--rounds R] [--poll P] [--device D]
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
    ap.add_argument("--poll", type=int, default=50, help="decisions between the loops' all-done checks")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    N = args.envs
    envs = {name: JssVecEnv(N, {"instance_path": args.instance}, device=args.device, auto_reset=False,
                            record_solution=True)
            for name in ("fused_op", "loop_op", "fused_job", "loop_job")}
    env0 = envs["fused_op"]
    J, M, dev = env0.jobs, env0.machines, env0.device
    gen = torch.Generator(device=dev).manual_seed(0)
    per_op = torch.rand((N, J, M), device=dev, generator=gen)
    per_job = torch.rand((N, J, 1), device=dev, generator=gen)
    ninf = torch.full((N, 1), float("-inf"), device=dev)
    job_rows = torch.cat([per_job[:, :, 0], ninf], 1)

    def loop(env, rows_of):
        while True:
            for _ in range(args.poll):
                env.step_greedy(rows_of(env))
            if bool(env.done.all()):
                return

    def op_rows(env):
        todo = env.export_state()["todo"].clamp(max=M - 1).long()
        return torch.cat([per_op.gather(2, todo.unsqueeze(2)).squeeze(2), ninf], 1)

    paths = {"fused_op": lambda env: env.rollout_priority(per_op),
             "loop_op": lambda env: loop(env, op_rows),
             "fused_job": lambda env: env.rollout_priority(per_job),
             "loop_job": lambda env: loop(env, lambda e: job_rows)}

    def run(name):
        env = envs[name]
        env.reset()
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

    def same(a, b):
        ea, eb = envs[a], envs[b]
        return all(torch.equal(getattr(ea, f), getattr(eb, f)) for f in ("last_makespan", "last_return", "solution"))

    ms = {name: [] for name in paths}
    decisions = {}
    for _ in range(args.rounds):
        for name in paths:
            t, d = run(name)
            ms[name].append(t)
            decisions[name] = d
        for a, b in (("fused_op", "loop_op"), ("fused_job", "loop_job")):
            if not same(a, b):
                raise SystemExit(f"{a} and {b} differ in makespan, raw return or solution")
    err = {name: int(env.stats()["envs_error"]) for name, env in envs.items()}
    mean_makespan = {name: float(env.last_makespan.double().mean()) for name, env in envs.items()}
    for env in envs.values():
        env.close()
    med = {name: statistics.median(v) for name, v in ms.items()}
    print(json.dumps({
        "workload": f"{args.instance} ({J}x{M}) N={N} from reset to the end of every episode, seeded torch.rand "
                    f"priority tables (N, J, M) and (N, J, 1)",
        "rounds": args.rounds, "parity": "fused_op == loop_op and fused_job == loop_job in makespan, raw return and "
                                          "solution, every round",
        "ms_per_batch": {name: {"median": med[name], "min": min(v), "max": max(v), "runs": v} for name, v in ms.items()},
        "episodes_per_s": {name: N / (med[name] * 1e-3) for name in ms},
        "decisions_per_batch": decisions,
        "decisions_per_s": {name: decisions[name] / (med[name] * 1e-3) for name in ms},
        "speedup_fused_vs_loop": {"op": med["loop_op"] / med["fused_op"], "job": med["loop_job"] / med["fused_job"]},
        "mean_makespan": mean_makespan, "envs_error": err,
        "gpu": gpu_info(args.device)}))


if __name__ == "__main__":
    main()
