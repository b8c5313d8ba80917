#!/usr/bin/env python
"""Critical-path descent on operation orders (JssVecEnv.improve_orders, jss_improve_orders), timed against the host
loop it replaces.  Per move that loop runs, for every order of the batch in lockstep: beam_search(-O, 1, order=True)
for the canonical rounds (width 1 is the greedy replay), a twin rollout_priority(-R) with solution recording for the
start times, the chain walk in numpy, order_log_prob with a zero (1, J, M) table on the neighbours padded to the
longest chain, and the argmin.  Workloads (per-env random normal tables, at most --max-moves moves per order):

  ta80, N = 256, the best order of beam_search(W = 16), from reset and after a fixed 500-decision random pre-roll;
  ta80, N = 256, all k = 16 orders of sample_without_replacement, from reset;
  ta01, N = 4 096, the best order of beam_search(W = 16), from reset.

Before timing, the two paths are checked bit for bit (final order, makespan, start makespan and moves).  One untimed
call of each path, then --rounds alternating rounds with CUDA events around work that ends in a device synchronise;
the line gives each path's median and range in ms per call, with the chain length and moves measured.

Quality: ta41..ta80, one env each, from reset, DESIGN.md's remaining-work table at T = 0.5: the mean best makespan of
greedy decoding, beam search at W = 16 and sampling without replacement at k = 16 (all 16 orders improved), before and
after improve_orders without a move limit, with the mean moves.  Writes nothing.

  python tools/bench_improve_orders.py [--rounds R] [--max-moves K] [--device D]

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit (CUDA 12.9 build, median of three rounds, ms per call,
max_moves = 3):

  workload                                          improve_orders   host loop   mean moves
  ta80, N = 256, beam W = 16 best, from reset       167.9            1 330       2.61
  ta80, N = 256, beam W = 16 best, after 500        108.7            1 006       2.63
  ta80, N = 256, SWOR k = 16, from reset            1 919            19 962      2.64
  ta01, N = 4 096, beam W = 16 best, from reset     16.3             1 276       1.68

  mean best makespan, ta41..ta80, T = 0.5    before    after     mean moves
  greedy                                     3706.7    3653.4    3.18
  beam W = 16                                3697.9    3648.4    3.53
  SWOR k = 16                                3636.0    3581.5    3.65
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench import gpu_info   # noqa: E402
from tools.bench_beam_search import remaining_work_table, timed   # noqa: E402


def chain(machine, duration, rd, st, T):
    """The chain's pairs (flat u, flat v) of the canonical schedule (rounds rd, starts st: (J_i, M_i)) ending at T."""
    M = machine.shape[1]
    mf, r, s = machine.ravel(), rd.ravel(), st.ravel()
    e = s + duration.ravel()
    q = np.flatnonzero(r >= 0)
    srt = q[np.lexsort((r[q], mf[q]))]                   # in-call operations by machine, then round
    pm = np.full(r.size, -1, np.int64)
    same = mf[srt[1:]] == mf[srt[:-1]]
    pm[srt[1:][same]] = srt[:-1][same]
    at = q[e[q] == T]
    if not len(at):
        return []
    o = int(at[np.argmax(r[at])])
    pm, r, s, e = pm.tolist(), r.tolist(), s.tolist(), e.tolist()
    pairs = []
    while True:
        p, s0 = pm[o], s[o]
        if p >= 0 and e[p] == s0:
            pairs.append((p, o))
            o = p
        elif o % M > 0 and r[o - 1] >= 0 and e[o - 1] == s0:
            o -= 1
        else:
            return pairs


class HostLoop:
    """The host loop over an (R, J, M) batch of orders, each row replayed from its env's state (rows: one env per
    order, states imported once)."""

    def __init__(self, env, k, snap):
        import torch
        from jssenv_b200 import JssVecEnv
        from jssenv_b200.instances import load_instance
        n = env.num_envs
        cfg = {"instance_paths": list(env.instances),
               "env_to_instance": list(np.repeat(np.asarray(env.env_to_instance), k))}
        idx = torch.arange(n, device=env.device).repeat_interleave(k)
        self.rows = JssVecEnv(n * k, cfg, device=env.device_index, auto_reset=False, seed=1)
        self.twin = JssVecEnv(n * k, cfg, device=env.device_index, auto_reset=False, record_solution=True, seed=1)
        self.snap = {key: v[idx].clone() for key, v in snap.items()}
        for e in (self.rows, self.twin):
            e.reset()
            e.import_state(self.snap)
        self.insts = [load_instance(env.instances[int(i)]) for i in self.rows.env_to_instance]
        self.zero = torch.zeros((1, env.jobs, env.machines), device=env.device)

    def run(self, order, max_moves):
        import torch
        rows, twin = self.rows, self.twin
        R, J, M = rows.num_envs, rows.jobs, rows.machines
        o = order.reshape(R, J, M)
        moves = np.zeros(R, np.int64)
        active = np.ones(R, bool)
        start, cur, pairs_seen = None, None, []
        for mv in range(max_moves + 1):
            canon = rows.beam_search(-o.float(), 1, order=True)
            rd = canon["order"]
            ms = canon["makespan"][:, 0].cpu().numpy().astype(np.int64)
            if start is None:
                start, cur = ms.copy(), ms.copy()
                active &= ms >= 0
            if mv == max_moves or not active.any():
                break
            twin.import_state(self.snap)
            twin.rollout_priority(-rd.float())
            sol, rdh = twin.solution.cpu().numpy(), rd.cpu().numpy()
            ch = []
            for i in range(R):
                mach, dur = self.insts[i]
                Ji, Mi = mach.shape
                ch.append(chain(mach, dur, rdh[i, :Ji, :Mi], sol[i, :Ji, :Mi], cur[i]) if active[i] else [])
            C = max(len(c) for c in ch)
            pairs_seen.append(float(np.mean([len(c) for c, a in zip(ch, active) if a])) if active.any() else 0.0)
            if C == 0:
                break
            nb = np.repeat(rdh[:, None], C, 1)
            for i, c in enumerate(ch):
                Mi = self.insts[i][0].shape[1]
                for x, (u, v) in enumerate(c):
                    (ju, ku), (jv, kv) = divmod(u, Mi), divmod(v, Mi)
                    nb[i, x, ju, ku], nb[i, x, jv, kv] = rdh[i, jv, kv], rdh[i, ju, ku]
            _, vals = rows.order_log_prob(self.zero, torch.from_numpy(nb).to(rows.device))
            v = vals.cpu().numpy().astype(np.int64)
            v = np.where(v >= 0, v, np.iinfo(np.int64).max)
            c = v.argmin(1)
            best = v[np.arange(R), c]
            take = active & (best < cur)
            if not take.any():
                break
            nxt = rdh.copy()
            nxt[take] = nb[np.flatnonzero(take), c[take]]
            cur[take], moves[take] = best[take], moves[take] + 1
            active &= take
            o = torch.from_numpy(nxt).to(rows.device)
        return {"order": rd, "makespan": cur, "start_makespan": start, "moves": moves, "pairs": pairs_seen}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-moves", type=int, default=3)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    torch.cuda.set_device(args.device)
    dev = torch.device("cuda", args.device)
    info = gpu_info(args.device)
    results = []
    for inst, n, src, preroll in (("ta80", 256, "beam16", 0), ("ta80", 256, "beam16", 500), ("ta80", 256, "swor16", 0),
                                  ("ta01", 4096, "beam16", 0)):
        env = JssVecEnv(n, {"instance_path": inst}, device=args.device, auto_reset=False, seed=1)
        J, M = env.jobs, env.machines
        env.reset()
        for _ in range(preroll):
            env.step(env.policy("RANDOM"))
        table = torch.randn((n, J, M), generator=torch.Generator(device=dev).manual_seed(8), device=dev)
        if src == "swor16":
            order = env.sample_without_replacement(table, 16, order=True)["order"]
        else:
            b = env.beam_search(table, 16, order=True)
            order = b["order"][:, None]
        k = order.shape[1]
        host = HostLoop(env, k, {key: v.clone() for key, v in env.export_state().items()})
        ref = host.run(order, args.max_moves)            # the untimed call of each path, checked bit for bit
        got = env.improve_orders(order, args.max_moves)
        for key in ("makespan", "start_makespan", "moves"):
            if not np.array_equal(got[key].reshape(-1).cpu().numpy(), ref[key]):
                raise SystemExit(f"{inst} {src}: {key} differs between improve_orders and the host loop")
        if not torch.equal(got["order"].reshape(ref["order"].shape), ref["order"]):
            raise SystemExit(f"{inst} {src}: the final orders differ")
        ms = {"improve_orders": [], "host_loop": []}
        for _ in range(args.rounds):
            ms["improve_orders"].append(timed(lambda: env.improve_orders(order, args.max_moves)))
            ms["host_loop"].append(timed(lambda: host.run(order, args.max_moves)))
        mv = got["moves"].double()
        results.append({
            "workload": f"{inst} ({J}x{M}) N={n}, {src} orders (k={k}), {preroll} random decisions before the call, "
                        f"max_moves={args.max_moves}",
            "ms_per_call": {key: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                            for key, v in ms.items()},
            "mean_moves": float(mv.mean()), "mean_chain_pairs_per_move": ref["pairs"],
            "mean_makespan": {"start": float(got["start_makespan"].double().mean()),
                              "final": float(got["makespan"].double().mean())},
            "parity": "order, makespan, start_makespan and moves equal the host loop's bit for bit"})
        env.close()

    names = [f"ta{i}" for i in range(41, 81)]
    env = JssVecEnv(len(names), {"instance_paths": names, "env_to_instance": list(range(len(names)))},
                    device=args.device, auto_reset=False, seed=3)
    table = torch.from_numpy(remaining_work_table(names, env.jobs, env.machines, 0.5)).to(dev)
    env.reset()
    quality = {}
    decodes = {"greedy": env.beam_search(table, 1, order=True)["order"][:, None],
               "beam_W16": env.beam_search(table, 16, order=True)["order"][:, None],
               "swor_k16": env.sample_without_replacement(table, 16, order=True)["order"]}
    for name, order in decodes.items():
        out = env.improve_orders(order)
        if not bool((out["makespan"] > 0).all()):
            raise SystemExit(f"quality: {name} did not finish")
        quality[name] = {"before": float(out["start_makespan"].min(1).values.double().mean()),
                         "after": float(out["makespan"].min(1).values.double().mean()),
                         "mean_moves": float(out["moves"].double().mean())}
    print(json.dumps({"rounds": args.rounds, "results": results,
                      "quality_ta41_ta80_mean_best_makespan": {"table": "remaining work / (0.5 * mean duration)",
                                                               **quality},
                      "gpu": info}))


if __name__ == "__main__":
    main()
