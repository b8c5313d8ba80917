"""Beam search for a policy that reads the observation at every decision.

``ObsBeamSearch`` drives ``JssVecEnv.beam_step`` (jss_beam_step): the env's N envs are G = N / W searches of width W,
env g*W + b holding slot b of search g, and each round the caller's network reads every slot's ``real_obs`` /
``action_mask`` and emits one logit row per slot::

    search = ObsBeamSearch(venv, width=16)
    search.start()
    while not search.done:
        search.step(policy(venv.real_obs, venv.action_mask))    # (N, >= J+1) logits
    out = search.result(order=True)

With rows gathered from a logit table at each slot's current operation, the result equals ``beam_search()`` of that
table on a G-env batch in the same start state, bit for bit.

With ``stochastic=True`` the search is a stochastic beam search (``JssVecEnv.stochastic_beam_step``): each group's W
slots end as W distinct episodes drawn without replacement from the policy, and with gathered rows the result equals
``sample_without_replacement()`` of the table on a G-env batch with env_id_base / W, the same seed and counter.
"""
import numpy as np

from . import _native as N


class ObsBeamSearch:
    """Beam search of width `width` over each group of `width` consecutive envs of `venv` (a JssVecEnv without
    auto-reset whose groups each run one instance).  The search starts from each group's slot 0 (env g*width) in its
    current state; the other envs of a group are overwritten by the search.  With `stochastic`, the beams are ranked
    by Gumbel-perturbed log-probability (stochastic beam search), so that the slots are distinct samples."""

    def __init__(self, venv, width: int, stochastic: bool = False):
        n = venv.num_envs
        if not 1 <= int(width) <= N.MAX_BEAM_WIDTH or n % int(width):
            raise ValueError(f"ObsBeamSearch: width must be in 1..{N.MAX_BEAM_WIDTH} and divide {n}, got {width!r}")
        self.venv, self.width, self.groups = venv, int(width), n // int(width)
        self.stochastic = bool(stochastic)
        inst = np.asarray(venv.env_to_instance).reshape(self.groups, self.width)
        if (inst != inst[:, :1]).any():
            raise ValueError("ObsBeamSearch: every env of a group must run the same instance")
        self.score = self.key = None
        self._round = self._rounds = 0

    def start(self):
        """Begin a search from each group's slot 0: take the forced no-ops there with ``step`` until slot 0 of every
        group has a legal job or is done, set the scores to [0, -inf, ..., -inf] per group, and allocate the (J*M, N)
        parent / action history on the device.  Refuses an auto-reset env (a completed beam must stay done).
        Stochastic: also set the keys to [0, -inf, ..., -inf] per group, and take the env's RNG counter c for the
        search (round r draws with c + r), advancing it by J*M as sample_without_replacement() does."""
        import torch
        v, W, G = self.venv, self.width, self.groups
        if v.auto_reset:
            raise ValueError("ObsBeamSearch: the env must not auto-reset")
        dev, J, M = v.device, v.jobs, v.machines
        slot0 = torch.arange(G, device=dev) * W
        jobs = torch.as_tensor(np.asarray(v.env_jobs, np.int64), device=dev)
        mach = torch.as_tensor(np.asarray(v.env_machines, np.int64), device=dev)
        own = torch.arange(J + 1, device=dev)[None, :] < jobs[:, None]          # each env's job columns
        while True:
            mask = v.action_mask
            need = (~(mask & own).any(1) & mask.gather(1, jobs[:, None]).squeeze(1) & ~v.done)[slot0]
            if not bool(need.any()):
                break
            act = torch.full((v.num_envs,), N.ACTION_SKIP, dtype=torch.int32, device=dev)
            act[slot0[need]] = jobs[slot0[need]].to(torch.int32)
            v.step(act)
        x = v.export_state()
        left = (mach[:, None] - x["todo"].long() - (x["tufco"] > 0).long()).clamp(min=0) * own[:, :J]
        self._done0 = v.done[slot0].clone()
        rounds = torch.where(self._done0, 0, left.sum(1)[slot0])
        self._rounds = int(rounds.max()) if G else 0
        self._round = 0
        self.score = torch.full((v.num_envs,), float("-inf"), dtype=torch.float32, device=dev)
        self.score[slot0] = 0.0
        if self.stochastic:
            if v.env_id_base % W:
                raise ValueError(f"ObsBeamSearch: env_id_base {v.env_id_base} must be a multiple of width {W}")
            self.key = self.score.clone()
            self._counter = v._step_index
            v._step_index += J * M
        self._parent = torch.empty((J * M, v.num_envs), dtype=torch.int32, device=dev)
        self._action = torch.empty((J * M, v.num_envs), dtype=torch.int32, device=dev)
        self._bad = torch.zeros(G, dtype=torch.int32, device=dev)
        self._slot0, self._mach = slot0, mach
        return self

    @property
    def done(self) -> bool:
        """True once no group can move: after as many rounds as the most operations any group had left at start()
        (every round allocates one operation per beam, so a complete beam is done by then)."""
        return self.score is not None and self._round >= self._rounds

    def step(self, logits):
        """One round (JssVecEnv.beam_step, or stochastic_beam_step at counter c + round) with the (N, >= J+1) logit
        rows of every slot, read at the live, not-done slots' legal jobs.  Records each slot's parent and job in the
        history."""
        if self.score is None or self.done:
            raise RuntimeError("ObsBeamSearch.step: call start() first, and stop once done")
        r = self._round
        if self.stochastic:
            _, _, bad = self.venv.stochastic_beam_step(logits, self.width, self.score, self.key, self._counter + r,
                                                       self._parent[r], self._action[r])
        else:
            _, _, bad = self.venv.beam_step(logits, self.width, self.score, self._parent[r], self._action[r])
        self._bad |= bad
        self._round = r + 1

    def result(self, order: bool = False, all_orders: bool = False):
        """The search's outcome, in JssVecEnv.beam_search()'s encoding, as device tensors: ``"makespan"`` (G, W) int32
        and ``"score"`` (G, W) float32 of the slots (-1 / -inf for a slot without a complete beam; -1 / NaN in every slot
        of a group that ended with no complete beam after a bad row; -1 / 0 in every slot of a group done at start());
        ``"best"`` (G,) int64, the lowest slot of smallest makespan, -1 if none; with `order`, ``"order"`` (G, J, M)
        int32, the round at which the best slot allocates each operation (-1 for operations started before start(),
        and everywhere in a group without a complete beam), so that rollout_priority(-order) replays it from the start
        state; with `all_orders`, ``"orders"`` (G, W, J, M), every slot's (-1 everywhere in a slot without a complete
        beam).  Stochastic: also ``"key"`` (G, W) float32, each slot's key, with the score's -inf / NaN / 0 in the
        same cases, as sample_without_replacement() reports them ("score" is its "log_prob").  The walk back through
        the history runs on the host after one copy of it."""
        import torch
        if self.score is None:
            raise RuntimeError("ObsBeamSearch.result: call start() first")
        v, W, G = self.venv, self.width, self.groups
        sc = self.score.view(G, W)
        complete = v.done.reshape(G, W) & (sc > float("-inf")) & (sc < float("inf"))
        makespan = torch.where(complete, v.current_time_step.reshape(G, W), -1)
        score = torch.where(complete, sc, float("-inf"))
        bad = ~complete.any(1) & (self._bad != 0)
        score = torch.where(bad[:, None], float("nan"), score)
        makespan = torch.where(self._done0[:, None], -1, makespan).to(torch.int32)
        score = torch.where(self._done0[:, None], 0.0, score)
        if self.stochastic:
            key = torch.where(complete, self.key.view(G, W), float("-inf"))
            key = torch.where(bad[:, None], float("nan"), key)
            key = torch.where(self._done0[:, None], 0.0, key)
        ended = makespan >= 0
        best = torch.where(ended, makespan, torch.iinfo(torch.int32).max).argmin(1)
        best = torch.where(ended.any(1), best, -1)
        out = {"makespan": makespan, "score": score, "best": best}
        if self.stochastic:
            out["key"] = key
        if order or all_orders:
            starts = [best[:, None]] if order else []
            if all_orders:
                slots = torch.arange(W, device=best.device)[None, :].expand(G, W)
                starts.append(torch.where(ended, slots, -1))
            walked = self._walk(torch.cat(starts, 1).cpu().numpy())
            if order:
                out["order"] = torch.from_numpy(walked[:, 0]).to(v.device)
            if all_orders:
                out["orders"] = torch.from_numpy(walked[:, -W:]).to(v.device)
        return out

    def _walk(self, at):
        """The orders of the beams ending in slots `at` (G, S) (-1: none) after the rounds so far, walked back through
        one host copy of the history: (G, S, J, M) int32."""
        v, W, R = self.venv, self.width, self._round
        G, S = at.shape
        par, act = self._parent[:R].cpu().numpy(), self._action[:R].cpu().numpy()
        mach = self._mach[self._slot0].cpu().numpy()
        order = np.full((G, S, v.jobs, v.machines), -1, np.int32)
        seen = np.zeros((G, S, v.jobs), np.int64)
        valid = at >= 0
        at = np.where(valid, at, 0)
        rows = np.arange(G)[:, None] * W
        for r in range(R - 1, -1, -1):
            j, p = act[r][rows + at], par[r][rows + at]
            g, s = np.nonzero(valid & (j >= 0))
            jj = j[g, s]
            order[g, s, jj, mach[g] - 1 - seen[g, s, jj]] = r
            seen[g, s, jj] += 1
            at = np.where(valid, p, at)
        return order
