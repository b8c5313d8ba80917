"""Times stochastic beam search for a policy that reads observations (ObsBeamSearch(stochastic=True) over
jss_stochastic_beam_step) against the deterministic search and against sampling with replacement, and compares what
the two sampling paths decode.

The policy is the fixed, seeded linear score of the 7 real_obs columns of each job that tools/bench_beam_step.py uses,
divided by a temperature.  Paths, per search of G groups of width W on the same N = G*W envs:
  (a) ObsBeamSearch(stochastic=True): start(), then per round policy -> step() (one jss_stochastic_beam_step launch per
      lane class): W distinct episodes per group;
  (b) ObsBeamSearch (deterministic), to show what the noise costs;
  (c) step_logits of the policy, one call per round of (a): sampling with replacement, the floor.
Before timing, a bit-for-bit check: rows gathered from a logit table at each slot's todo must give
sample_without_replacement of that table on a G-env batch with the same seed, ids and counter, in every group (the
groups start from different states after the random walk).  Timing: one untimed run, then three alternating rounds
(CUDA events around work that ends in a device synchronise); ms per search, median and range.  Quality: the mean over
groups of the best makespan and the number of repeated schedules per search, of (a) and of (c) run to the end, at
temperatures 1 and 0.05.  Prints the GPU's name, power limit and clocks in the same run.
Usage: python tools/bench_stochastic_beam_step.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jssenv_b200 import JssVecEnv  # noqa: E402
from jssenv_b200.beam import ObsBeamSearch  # noqa: E402

W_POLICY = torch.tensor(np.random.default_rng(0).normal(size=7), dtype=torch.float32)


def policy(temp=1.0):
    """(N, J+1) logits: the linear score of each job's real_obs row over `temp`; the no-op column -inf (never read by
    the searches; step_logits takes the no-op only when it is the one legal action)."""
    def rows(env):
        x = (env.real_obs @ W_POLICY.to(env.device)) / temp
        return torch.cat([x, torch.full_like(x[:, :1], float("-inf"))], 1)
    return rows


def make(name, G, W, walk):
    """G groups of W envs of `name` (env_id_base 0, seed 1); with walk > 0 group g starts where env g of a G-env batch
    is after `walk` random decisions (every group from its own state).  Returns the env, the start snapshot and the
    G-env batch in the groups' start states."""
    base = JssVecEnv(G, {"instance_path": name}, auto_reset=False, seed=1)
    base.reset()
    for _ in range(walk):
        base.step(base.policy("RANDOM"))
    env = JssVecEnv(G * W, {"instance_path": name}, auto_reset=False, seed=1)
    env.reset()
    env.import_state({k: v.clone().repeat_interleave(W, 0) for k, v in base.export_state().items()})
    return env, {k: v.clone() for k, v in env.export_state().items()}, base


def gathered(env, table, W):
    """Each slot's row: its group's table entry at each job's current operation (NaN in the no-op column)."""
    J, M = env.jobs, env.machines
    todo = env.export_state()["todo"].long().clamp(0, M - 1)
    vals = table.repeat_interleave(W, 0).gather(2, todo[:, :, None]).squeeze(2)
    return torch.cat([vals, torch.full_like(vals[:, :1], float("nan"))], 1)


def check_table(env, snap, base, W):
    """Groups (of G) in which the search driven by gathered table rows equals sample_without_replacement bit for bit:
    makespan, score / log_prob and key."""
    G = base.num_envs
    table = torch.randn((G, env.jobs, env.machines), generator=torch.Generator(device=env.device).manual_seed(5),
                        device=env.device)
    env.import_state(snap)
    s = ObsBeamSearch(env, W, stochastic=True).start()
    while not s.done:
        s.step(gathered(env, table, W))
    got = s.result()
    base._step_index = s._counter
    want = base.sample_without_replacement(table, W)
    same = (got["makespan"] == want["makespan"]).all(1)
    for a, b in (("score", "log_prob"), ("key", "key")):
        same &= (got[a].view(torch.int32) == want[b].view(torch.int32)).all(1)
    return int(same.sum())


def run_search(env, W, stochastic, pol):
    s = ObsBeamSearch(env, W, stochastic=stochastic).start()
    n = 0
    while not s.done:
        s.step(pol(env))
        n += 1
    return s, n


def run_c(env, rounds, pol):
    for _ in range(rounds):
        env.step_logits(pol(env))


def sample_to_end(env, W, pol):
    """(c) to the end: every env steps by step_logits until done.  Returns the makespans (G, W) and, per env, its
    job sequence as a tuple (for repeats)."""
    J, n = env.jobs, env.num_envs
    seq = []
    while not bool(env.done.all()):
        alive = ~env.done
        a = env.step_logits(pol(env))[4]["actions"]
        seq.append(torch.where(alive & (a < J), a, -1))
    seqs = torch.stack(seq, 1).cpu().numpy() if seq else np.zeros((n, 0), np.int32)
    return env.current_time_step.view(-1, W).cpu().numpy(), [tuple(r[r >= 0]) for r in seqs]


def quality(env, snap, W, temp):
    """Mean best makespan and repeats (W minus distinct schedules, summed over groups) of (a) and of (c) to the end."""
    G = env.num_envs // W
    env.import_state(snap)
    s, _ = run_search(env, W, True, policy(temp))
    out = s.result(all_orders=True)
    ms = out["makespan"].cpu().numpy()
    orders = out["orders"].cpu().numpy().reshape(G, W, -1)
    rep_a = sum(W - len({o.tobytes() for o, m in zip(orders[g], ms[g]) if m >= 0}) for g in range(G))
    best_a = np.where(ms >= 0, ms, np.iinfo(np.int32).max).min(1)
    env.import_state(snap)
    ms_c, seqs = sample_to_end(env, W, policy(temp))
    rep_c = sum(W - len(set(seqs[g * W:(g + 1) * W])) for g in range(G))
    return {"T": temp, "a_mean_best": round(float(best_a.mean()), 1), "a_repeats": int(rep_a),
            "a_complete": int((ms >= 0).sum()), "c_mean_best": round(float(ms_c.min(1).mean()), 1),
            "c_repeats": int(rep_c)}


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the query is informational only
        q = f"unavailable ({e})"
    return q


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_stochastic_beam_step: needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, G, W, walk in (("ta80", 256, 16, 0), ("ta80", 256, 16, 500), ("ta01", 4096, 8, 0)):
        env, snap, base = make(name, G, W, walk)
        equal = check_table(env, snap, base, W)
        env.import_state(snap)
        _, rounds = run_search(env, W, True, policy())
        pol = policy()
        fns = {"a": lambda: run_search(env, W, True, pol), "b": lambda: run_search(env, W, False, pol),
               "c": lambda: run_c(env, rounds, pol)}
        for fn in fns.values():                           # untimed
            env.import_state(snap)
            fn()
        times = {k: [] for k in fns}
        for _ in range(3):
            for k, fn in fns.items():
                env.import_state(snap)
                times[k].append(timed(fn))
        res = {"workload": f"{name} G={G} W={W} walk={walk}", "rounds": rounds,
               "groups_equal_to_table_swor": f"{equal}/{G}"}
        for k, v in times.items():
            v = sorted(v)
            res[k] = {"ms_per_search": round(v[1], 2), "range_ms": [round(v[0], 2), round(v[2], 2)],
                      "us_per_round": round(1000 * v[1] / max(rounds, 1), 2)}
        res["quality"] = [quality(env, snap, W, t) for t in (1.0, 0.05)]
        print(json.dumps(res), flush=True)
        env.close()
        base.close()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
