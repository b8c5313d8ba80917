#!/usr/bin/env python
"""Counts the bytes a fused ta80 step moves per env-step, and how many of the written ones it actually changes, on the
host emulation of the kernels (tests/emu): no GPU needed, and no time is measured.

Workload: bench.py's headline at a reduced N -- auto-reset, masked-random (step_sample "RANDOM"), env i pre-rolled
(i * 7919) mod 2236 transitions.  Around each of --steps steps the observation rows (real_obs) and the state blocks
(re-encoded from export_state() with the layout of jss_block_geom / jss_pack_job, envs at their device offsets) are
diffed at ABSOLUTE 32-byte sector granularity: a sector is dirty when one of its bytes changed.  Reported per env-step
and per region (obs, w0, w1, w2, tail): the bytes written today (every changed env rewrites its whole row and block),
the bytes written when only dirty sectors are stored (the tail -- tuam, job bits, header -- always), and the number of
contiguous dirty runs (one bulk store each).  The block tail is counted as always written, so its header fields that
export_state() does not return (episode steps and return) need not be re-encoded.  `state_block_sector_store` is what the
uniform step kernels store of a block: every sector that holds a changed byte of w0 / w1 / w2, every sector of the
tail and the block's first sector, each with the block's bytes in it; `per_env_step_total` sets it against whole
blocks with the changed row sectors (`dirty_rows`) and with whole rows (`today`).

  python tools/count_step_bytes.py [--envs N] [--steps S] [--instance ta80]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import TA80_EPISODE, preroll   # noqa: E402

SECTOR = 32


def lane_slots(J):
    kj = 1 if J <= 32 else 2 if J <= 64 else 4 if J <= 128 else 8
    return max(4, kj)


def block_geom(J, M):
    """jss_block_geom (csrc/jss_types.h), in bytes: w0, w1, w2 and tail offsets, block size."""
    slots = lane_slots(J)
    Jc = (J + slots - 1) & ~(slots - 1)
    Mc = (M + 3) & ~3
    tail = 2 * Jc + ((Jc + 7) & ~7) // 2
    words = tail + Mc + 2 * slots + 4
    return {"Jc": Jc, "w0": 0, "w1": 4 * Jc, "w2": 8 * Jc, "tail": 4 * tail, "size": 4 * words}


def encode_jobs(st, J, g):
    """The job records of every block (w0 | w1 | w2 regions, jss_pack_job), (N, tail bytes) uint8; padding slots hold
    a finished job (todo == M, the rest 0), as env_store_to writes them."""
    n = st["todo"].shape[0]
    Jc = g["Jc"]
    todo = st["todo"].astype(np.uint32)
    w0 = todo | (st["tufco"].astype(np.uint32) << 6) | (st["col4"].astype(np.uint32) << 17)
    ti = st["total_idle"].astype(np.uint32)
    w1 = st["idle_last"].astype(np.uint32) | (ti << 24)
    w2 = (ti >> 8).astype(np.uint16)
    out = np.zeros((n, g["tail"]), np.uint8)
    W0 = np.zeros((n, Jc), np.uint32)
    W0[:, :] = st["M"]
    W0[:, :J] = w0
    W1 = np.zeros((n, Jc), np.uint32)
    W1[:, :J] = w1
    W2 = np.zeros((n, (g["tail"] - g["w2"]) // 2), np.uint16)
    W2[:, :J] = w2
    out[:, g["w0"]:g["w1"]] = W0.view(np.uint8)
    out[:, g["w1"]:g["w2"]] = W1.view(np.uint8)
    out[:, g["w2"]:g["tail"]] = W2.view(np.uint8)
    return out


def dirty_sectors(old, new, base, stride):
    """old / new: (N, B) byte rows stored at absolute byte base + i * stride.  Returns the (N, n_sectors) bool of
    dirty sectors, counted from the sector that holds each row's first byte, and each row's offset into that sector."""
    n, B = old.shape
    lead = (base + np.arange(n, dtype=np.int64) * stride) % SECTOR          # bytes of the first sector before the row
    ns = (int(lead.max()) + B + SECTOR - 1) // SECTOR
    diff = old != new
    pad = np.zeros((n, ns * SECTOR), bool)
    idx = lead[:, None] + np.arange(B)[None, :]
    np.put_along_axis(pad, idx, diff, axis=1)
    return pad.reshape(n, ns, SECTOR).any(axis=2), lead


def sector_bytes(mask, lead, lo, hi):
    """Bytes stored when the dirty sectors of `mask` are written, clipped to row bytes [lo, hi): per env."""
    n, ns = mask.shape
    s0 = np.arange(ns)[None, :] * SECTOR - lead[:, None]                  # row byte where each sector starts
    a = np.clip(s0, lo, hi)
    b = np.clip(s0 + SECTOR, lo, hi)
    return ((b - a) * mask).sum(axis=1)


def runs(mask):
    """Contiguous runs of dirty sectors per env."""
    m = mask.astype(np.int8)
    return ((m[:, 1:] == 1) & (m[:, :-1] == 0)).sum(axis=1) + m[:, 0]


def region_mask(mask, lead, lo, hi):
    """The dirty sectors that overlap row bytes [lo, hi)."""
    n, ns = mask.shape
    s0 = np.arange(ns)[None, :] * SECTOR - lead[:, None]
    return mask & (s0 + SECTOR > lo) & (s0 < hi)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--instance", default="ta80")
    args = ap.parse_args()

    import torch
    from jssenv_b200 import JssVecEnv
    from tests.emu.emu_backend import use_emulation

    with use_emulation():
        env = JssVecEnv(args.envs, {"instance_path": args.instance}, auto_reset=True, seed=1234)
        n, J, M = env.num_envs, env.jobs, env.machines
        g = block_geom(J, M)
        env.reset()
        acts = preroll(env, "RANDOM", TA80_EPISODE if J * M >= 2000 else int(1.13 * J * M), torch)

        def snap():
            st = {k: v.numpy().copy() for k, v in env.export_state().items() if k in
                  ("todo", "tufco", "idle_last", "total_idle", "col4")}
            st["M"] = M
            return encode_jobs(st, J, g), env.real_obs.numpy().reshape(n, J * 7).view(np.uint8).copy()

        regions = {"w0": (g["w0"], g["w1"]), "w1": (g["w1"], g["w2"]), "w2": (g["w2"], g["tail"])}
        tail_bytes = g["size"] - g["tail"]
        tot = {k: 0.0 for k in ("obs", "w0", "w1", "w2")}
        full_runs = {"obs": 0.0, "block": 0.0}
        block_store = 0.0
        blk0, obs0 = snap()
        for _ in range(args.steps):
            *_, acts = env.step_sample(acts, "RANDOM")
            blk1, obs1 = snap()
            om, olead = dirty_sectors(obs0, obs1, 0, J * 28)
            bm, blead = dirty_sectors(blk0, blk1, 0, g["size"])
            tot["obs"] += sector_bytes(om, olead, 0, J * 28).sum()
            for k, (lo, hi) in regions.items():
                tot[k] += sector_bytes(region_mask(bm, blead, lo, hi), blead, lo, hi).sum()
            # the tail is always stored, from the start of its first sector; block runs end in it
            ns = bm.shape[1]
            s0 = np.arange(ns)[None, :] * SECTOR - blead[:, None]
            bm_t = bm | (s0 + SECTOR > g["tail"]) & (s0 < g["size"])
            # the sector store: bm covers the job records only, so widen it to the whole block first
            nsb = (int(blead.max()) + g["size"] + SECTOR - 1) // SECTOR
            sb = np.arange(nsb)[None, :] * SECTOR - blead[:, None]
            stored = np.zeros((n, nsb), bool)
            stored[:, :ns] = bm
            stored |= (sb + SECTOR > g["tail"]) & (sb < g["size"]) | (sb <= 0)
            block_store += sector_bytes(stored, blead, 0, g["size"]).sum()
            full_runs["obs"] += runs(om).sum()
            full_runs["block"] += runs(bm_t).sum()
            blk0, obs0 = blk1, obs1
        es = float(args.steps * n)
        per = {k: v / es for k, v in tot.items()}
        today = {"obs": J * 28, "w0": g["w1"] - g["w0"], "w1": g["w2"] - g["w1"], "w2": g["tail"] - g["w2"],
                 "tail": tail_bytes}
        dirty = {**per, "tail": float(tail_bytes)}
        other = 128   # mask row, scalar record, action read, next action written (ta80 geometry)
        read = g["size"] + 4
        w_today = sum(today.values()) + other - 4
        w_dirty = sum(dirty.values()) + other - 4
        w_rows = per["obs"] + g["size"] + other - 4
        w_store = per["obs"] + block_store / es + other - 4
        print(json.dumps({
            "workload": f"{args.instance} N={n} masked-random auto-reset, pre-rolled (i*7919) mod {TA80_EPISODE}, "
                        f"{args.steps} steps, host emulation",
            "bytes_written_today": today, "bytes_written_dirty_sectors": {k: round(v, 1) for k, v in dirty.items()},
            "state_block_read": g["size"], "state_block_sector_store": round(block_store / es, 1),
            "per_env_step_total": {"today": w_today + read, "dirty_sectors": round(w_dirty + read, 1),
                                   "saving": round(w_today - w_dirty, 1),
                                   "saving_frac": round((w_today - w_dirty) / (w_today + read), 4),
                                   "dirty_rows": round(w_rows + read, 1),
                                   "dirty_rows_and_block_sectors": round(w_store + read, 1),
                                   "block_saving_frac": round((w_rows - w_store) / (w_rows + read), 4)},
            "mean_runs_per_env_step": {k: round(v / es, 2) for k, v in full_runs.items()},
        }, indent=1))


if __name__ == "__main__":
    main()
