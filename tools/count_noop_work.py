#!/usr/bin/env python
"""Counts the work of the no-op check (env_check_no_op, the reference's _check_no_op) per env-step, on the host
emulation of the kernels (tests/emu): no GPU needed, and no time is measured.

Workloads: bench.py's headline at a reduced N -- auto-reset, masked-random (step_sample "RANDOM"), env i pre-rolled
(i * 7919) mod period transitions -- on ta80 (4 jobs per lane) and ta01 (1 job per lane), and the mixed cfg5 batch
(env i runs ta((i mod 80) + 1), pre-rolled as bench.py does).  After every timed step the state the step's check ran on
is read back with export_state() and the check is replayed here, counting:
  - gate: the share of env-steps that pass the gate (an event pending, <= 3 legal machines, <= 4 legal jobs);
  - pass 1: the legal jobs the reference visits, in ascending order, and the share that returns "not legal" there
    (some legal job ends before the next event);
  - pass 2, for the env-steps that reach it: per job slot, the share of steps that run the slot, the walks it starts
    (jobs whose case sets up a walk), the lane iterations, and the warp's trip count (the longest walk of the slot
    over the lanes, which the warp pays for); the slot after which the slot-by-slot check exits early;
  - the trip count of one interleaved loop over every slot (the longest walk of any lane, no early exit) against
    the sum of the slot-by-slot trips;
  - the walk steps and trips when the walks are bounded by the largest final per-machine horizon instead of the
    reference's max_horizon, and whether every result stays the same.
Reset steps of auto-reset envs (where no check runs) are left out.

  python tools/count_noop_work.py [--envs N] [--steps S] [--workloads ta80,ta01,cfg5]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from bench import TA80_EPISODE, preroll   # noqa: E402


def lane_kj(J):
    return 1 if J <= 32 else 2 if J <= 64 else 4 if J <= 128 else 8


class Tally:
    def __init__(self):
        self.steps = 0
        self.gated = 0
        self.p1_visits = 0
        self.p1_return = 0
        self.p2 = 0
        self.noop_legal = 0
        self.slot_run = {}
        self.slot_walks = {}
        self.slot_iters = {}
        self.slot_trip = {}
        self.exit_after = {}
        self.trip_slotwise = 0
        self.trip_interleaved = 0
        self.iters_h = 0
        self.trip_slotwise_h = 0

    def add(self, d, k, v=1):
        d[k] = d.get(k, 0) + v


def replay(T, machine, duration, KJ, t, todo, tufco, tuam, legal, blocked, max_time_op):
    """One env's check on its state; adds its counts to T and returns the check's result."""
    J, M = machine.shape
    T.steps += 1
    ops_m = np.where(todo < M, machine[np.arange(J), np.minimum(todo, M - 1)], -1)
    ops_d = np.where(todo < M, duration[np.arange(J), np.minimum(todo, M - 1)], 0)
    lj = np.flatnonzero(legal)
    ML = set(int(m) for m in ops_m[lj])
    pending = tuam[tuam > 0]
    if pending.size == 0 or len(ML) > 3 or lj.size > 4:
        return False
    T.gated += 1
    next_event = t + int(pending.min())
    maxh = t
    hz = {}
    for j in lj:                                              # pass 1, ascending job index
        T.p1_visits += 1
        m, end = int(ops_m[j]), t + int(ops_d[j])
        if end < next_event:
            T.p1_return += 1
            return False
        hz[m] = min(hz.get(m, t + max_time_op), end)
        maxh = max(maxh, hz[m])
    T.p2 += 1
    bounded = walk(T, machine, duration, KJ, t, todo, tufco, tuam, legal, blocked, hz, ML, max(hz.values()),
                   count_h=True)
    result = walk(T, machine, duration, KJ, t, todo, tufco, tuam, legal, blocked, hz, ML, maxh)
    assert bounded == result                                  # the bound changes the work, never the result
    return result


def walk(T, machine, duration, KJ, t, todo, tufco, tuam, legal, blocked, hz, ML, maxh, count_h=False):
    """Pass 2 with the walks bounded by maxh; counts into T (with count_h, only the bounded-by-H totals)."""
    J, M = machine.shape
    ops_m = np.where(todo < M, machine[np.arange(J), np.minimum(todo, M - 1)], -1)
    want = set()
    exited = None
    lengths = np.zeros((32, KJ), np.int64)                    # each lane's walk per slot
    for i in range(KJ):
        if not count_h:
            T.add(T.slot_run, i)
        for lane in range(32):
            j = KJ * lane + i
            if j >= J or legal[j] or todo[j] >= M:
                continue
            if tufco[j] > 0:
                ts, tm = int(todo[j]) + 1, t + int(tufco[j])
            elif not blocked[j]:
                ts, tm = int(todo[j]), t + int(tuam[ops_m[j]])
            else:
                continue
            if not count_h:
                T.add(T.slot_walks, i)
            n = 0
            while ts < M - 1 and maxh > tm:
                m = int(machine[j, ts])
                if m in hz and hz[m] > tm:
                    want.add(m)
                tm += int(duration[j, ts])
                ts += 1
                n += 1
            lengths[lane, i] = n
        if count_h:
            T.iters_h += int(lengths[:, i].sum())
            T.trip_slotwise_h += int(lengths[:, i].max())
        else:
            T.add(T.slot_iters, i, int(lengths[:, i].sum()))
            T.add(T.slot_trip, i, int(lengths[:, i].max()))
            T.trip_slotwise += int(lengths[:, i].max())
        if i + 1 < KJ and ML and want == ML:
            exited = i
            break
    if count_h:
        return bool(ML) and want == ML
    T.trip_interleaved += int(lengths.max())
    T.add(T.exit_after, "none" if exited is None else exited)
    if ML and want == ML:
        T.noop_legal += 1
    return bool(ML) and want == ML


def report(T, KJ):
    g, p2 = max(T.gated, 1), max(T.p2, 1)
    return {
        "env_steps": T.steps,
        "gate_share": round(T.gated / max(T.steps, 1), 4),
        "pass1_visits_per_gated_step": round(T.p1_visits / g, 3),
        "pass1_return_share_of_gated": round(T.p1_return / g, 4),
        "pass2_share_of_steps": round(T.p2 / max(T.steps, 1), 4),
        "noop_legal_share_of_pass2": round(T.noop_legal / p2, 4),
        "per_slot_per_pass2_step": {i: {"run": round(T.slot_run.get(i, 0) / p2, 4),
                                        "walks": round(T.slot_walks.get(i, 0) / p2, 3),
                                        "lane_iterations": round(T.slot_iters.get(i, 0) / p2, 3),
                                        "warp_trips": round(T.slot_trip.get(i, 0) / p2, 3)} for i in range(KJ)},
        "lane_iterations_per_pass2_step": round(sum(T.slot_iters.values()) / p2, 3),
        "early_exit_after_slot_share": {str(k): round(v / p2, 4) for k, v in sorted(T.exit_after.items(), key=str)},
        "warp_trips_per_pass2_step": {"slot_by_slot_with_exits": round(T.trip_slotwise / p2, 3),
                                      "one_interleaved_loop": round(T.trip_interleaved / p2, 3)},
        "walks_bounded_by_largest_minimum": {"lane_iterations": round(T.iters_h / p2, 3),
                                             "warp_trips_slot_by_slot": round(T.trip_slotwise_h / p2, 3)},
    }


def run(names, n, steps, period, rule, torch):
    from jssenv_b200 import JssVecEnv
    from jssenv_b200.instances import load_instance
    if len(names) == 1:
        env = JssVecEnv(n, {"instance_path": names[0]}, auto_reset=True, seed=1234)
        inst_of = np.zeros(n, np.int64)
    else:
        inst_of = np.arange(n) % len(names)
        env = JssVecEnv(n, {"instance_paths": names, "env_to_instance": inst_of}, auto_reset=True, seed=2)
    tabs = [load_instance(s) for s in names]
    env.reset()
    acts = preroll(env, rule, period, torch)
    tallies = {}
    done0 = env.export_state()["flags"].numpy() & 1            # JSS_FLAG_DONE
    for _ in range(steps):
        *_, acts = env.step_sample(acts, rule)
        st = {k: v.numpy().copy() for k, v in env.export_state().items()}
        for e in range(n):
            if done0[e]:                                      # this step reset the env: no check ran
                continue
            mach, dur = tabs[inst_of[e]]
            J, M = mach.shape
            KJ = lane_kj(J)
            T = tallies.setdefault(KJ, Tally())
            noop = replay(T, mach, dur, KJ, int(st["t"][e]), st["todo"][e, :J], st["tufco"][e, :J], st["tuam"][e, :M],
                   st["legal"][e, :J], st["blocked"][e, :J], int(dur.max()))
            assert noop == bool((st["flags"][e] >> 8) & 4), (e, noop)   # JSS_FLAG_NOOP_LEGAL: the replay is the check
        done0 = st["flags"] & 1
    env.close()
    return {f"{KJ}_jobs_per_lane": report(T, KJ) for KJ, T in sorted(tallies.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--workloads", default="ta80,ta01,cfg5")
    args = ap.parse_args()

    import torch
    from tests.emu.emu_backend import use_emulation

    out = {}
    with use_emulation():
        for w in args.workloads.split(","):
            if w == "cfg5":
                names = ["ta%02d" % (k + 1) for k in range(80)]
                res = run(names, args.envs, args.steps, TA80_EPISODE, "RANDOM", torch)
                desc = f"mixed ta01..ta80 N={args.envs}, masked-random, pre-rolled (i*7919) mod {TA80_EPISODE}"
            else:
                from jssenv_b200.instances import load_instance
                J, M = load_instance(w)[0].shape
                period = TA80_EPISODE if J * M >= 2000 else int(1.13 * J * M)
                res = run([w], args.envs, args.steps, period, "RANDOM", torch)
                desc = f"{w} N={args.envs}, masked-random auto-reset, pre-rolled (i*7919) mod {period}"
            out[w] = {"workload": desc + f", {args.steps} steps, host emulation", **res}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
