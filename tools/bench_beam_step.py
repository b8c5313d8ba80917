"""Times beam search for a policy that reads observations (ObsBeamSearch over jss_beam_step) against the torch loop it
replaces, and against step_greedy on the same N*W batch as the floor.

The policy is a fixed, seeded linear score of the 7 real_obs columns of each job, computed in torch (a genuine
observation-based policy whose network costs next to nothing).  Paths, per search of G groups of width W:
  (a) ObsBeamSearch: start(), then per round policy -> step() (one jss_beam_step launch per lane class);
  (b) the torch loop on the same N*W envs: export_state, log-softmax over the legal jobs, top-W in the same total order
      (score descending, then parent slot, then job), import_state of the parents, step, forced no-ops;
  (c) step_greedy of the policy on the N*W batch, one call per round.
Before timing, (a) and (b) are run once and the groups whose final makespan rows agree are counted (near-ties in the
scores may order candidates differently in fp32).  Reports ms per search and us per round, median and range of three
alternating rounds (CUDA events), with the GPU's power limit and clocks.  Usage: python tools/bench_beam_step.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jssenv_b200 import JssVecEnv  # noqa: E402
from jssenv_b200 import _native as N  # noqa: E402
from jssenv_b200.beam import ObsBeamSearch  # noqa: E402

W_POLICY = torch.tensor(np.random.default_rng(0).normal(size=7), dtype=torch.float32)


def policy(env):
    """(N, J+1) logits: the linear score of each job's real_obs row; the no-op column -inf (never read)."""
    x = env.real_obs @ W_POLICY.to(env.device)
    return torch.cat([x, torch.full_like(x[:, :1], float("-inf"))], 1)


def make(name, G, W, walk):
    """G groups of W envs of `name`; with walk > 0 every group's slot 0 (and the rest) after `walk` random decisions of
    one env, copied to every slot.  Returns the env and the start snapshot."""
    env = JssVecEnv(G * W, {"instance_path": name}, auto_reset=False, seed=1)
    env.reset()
    if walk:
        base = JssVecEnv(G, {"instance_path": name}, auto_reset=False, seed=1)
        base.reset()
        for _ in range(walk):
            base.step(base.policy("RANDOM"))
        snap = {k: v.clone().repeat_interleave(W, 0) for k, v in base.export_state().items()}
        env.import_state(snap)
    return env, {k: v.clone() for k, v in env.export_state().items()}


def run_a(env, W):
    s = ObsBeamSearch(env, W).start()
    n = 0
    while not s.done:
        s.step(policy(env))
        n += 1
    return s.result()["makespan"], n


def run_b(env, W):
    """The torch loop: returns the final makespan rows (G, W) and the rounds."""
    n, J, dev = env.num_envs, env.jobs, env.device
    G = n // W
    score = torch.full((G, W), float("-inf"), device=dev)
    score[:, 0] = 0.0
    skip = torch.full((n,), N.ACTION_SKIP, dtype=torch.int32, device=dev)
    rounds = 0

    def forced():
        while True:
            m = env.action_mask
            need = ~m[:, :J].any(1) & m[:, J] & torch.isfinite(score.view(-1)) & ~env.done
            if not bool(need.any()):
                return
            env.step(torch.where(need, J, skip))

    forced()
    while True:
        live = torch.isfinite(score.view(-1)) & ~env.done & env.action_mask[:, :J].any(1)
        if not bool(live.any()):
            break
        x = {k: v.clone() for k, v in env.export_state().items()}
        legal = env.action_mask[:, :J] & live[:, None]
        z = torch.where(legal, policy(env)[:, :J], float("-inf"))
        lp = z - torch.logsumexp(z, 1, keepdim=True)
        cand = torch.where(legal, score.view(-1)[:, None] + lp, float("-inf")).view(G, W * J)
        top, idx = torch.sort(cand, dim=1, descending=True, stable=True)
        top, idx = top[:, :W], idx[:, :W]
        ok = top > float("-inf")
        parent, job = idx // J, idx % J
        rows = (torch.arange(G, device=dev)[:, None] * W + parent).view(-1)
        env.import_state({k: v[rows] for k, v in x.items()})
        env.step(torch.where(ok.view(-1), job.view(-1).to(torch.int32), skip))
        score = torch.where(ok, top, float("-inf"))
        forced()
        rounds += 1
    ms = torch.where(torch.isfinite(score) & env.done.view(G, W), env.current_time_step.view(G, W), -1)
    return ms, rounds


def run_c(env, rounds):
    for _ in range(rounds):
        env.step_greedy(policy(env))


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
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, G, W, walk in (("ta80", 256, 16, 0), ("ta80", 256, 16, 500), ("ta01", 4096, 8, 0)):
        env, snap = make(name, G, W, walk)
        env.import_state(snap)
        a, rounds = run_a(env, W)
        env.import_state(snap)
        b, rb = run_b(env, W)
        match = int((a == b).all(1).sum())
        times = {"a": [], "b": [], "c": []}
        for _ in range(3):
            for k, fn in (("a", lambda: run_a(env, W)), ("b", lambda: run_b(env, W)), ("c", lambda: run_c(env, rounds))):
                env.import_state(snap)
                times[k].append(timed(fn))
        res = {"workload": f"{name} G={G} W={W} walk={walk}", "rounds": rounds, "rounds_torch": rb,
               "rows_matching": f"{match}/{G}"}
        for k, v in times.items():
            v = sorted(v)
            res[k] = {"ms_per_search": round(v[1], 2), "range_ms": [round(v[0], 2), round(v[2], 2)],
                      "us_per_round": round(1000 * v[1] / max(rounds, 1), 2)}
        print(json.dumps(res), flush=True)
        env.close()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
