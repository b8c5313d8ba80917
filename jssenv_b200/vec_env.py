"""JssVecEnv -- N independent job-shop environments stepped by the sm_90a kernels.

Batched form of the reference's ``JssEnv`` contract (JSSEnv/envs/jss_env.py):
``reset() -> obs`` (jss_env.py:145), ``step(actions) -> (obs, reward, done,
truncated, info)`` (jss_env.py:403-481) with ``obs = {"real_obs": (N, J, 7) float32,
"action_mask": (N, J+1) bool}`` (jss_env.py:112-119, 130-134).  As in the reference,
the observation entries are LIVE ALIASES of the environment's buffers (here: device
memory owned by the native library), the no-op is action index ``J``, actions are
not validated beyond setting a per-env error bit, and ``truncated`` is always False.
One exception to the live alias: after ``step_logits_record()`` or ``step_greedy_record()``, which write the
observation into the caller's rollout slot instead, ``real_obs`` is stale until the next non-recording call or
``refresh_obs()``.

The gradients of sample_episodes(), order_log_prob() and sample_without_replacement() are replayed from the envs' state
at backward time.  Every call that may change an env's state (reset, the steps and their _record forms, the rollouts,
beam_step, stochastic_beam_step, import_state and the host-buffer steps) counts as a change, whether or not it changed
one in the end, and a backward of such an output made before it raises RuntimeError; so does a backward after close().
"""
import ctypes
import functools
from typing import Any, Dict, Optional, Union

import numpy as np

from . import _native as N
from .instances import DEFAULT_INSTANCE, load_instance


def _instance_list(env_config: Optional[Dict[str, Any]]):
    """`env_config` keeps the reference key ``instance_path`` (jss_env.py:35-39) and adds
    ``instance_paths`` (list) + ``env_to_instance`` (int array) for mixed batches."""
    if env_config is None:
        env_config = {"instance_path": DEFAULT_INSTANCE}
    if "instance_paths" in env_config:
        specs = list(env_config["instance_paths"])
    else:
        specs = [env_config["instance_path"]]
    return [load_instance(s) for s in specs], env_config.get("env_to_instance")


def _rule_id(rule: Union[str, int]) -> int:
    return N.RULES[rule.upper()] if isinstance(rule, str) else int(rule)


def _coin_id(coin: str) -> int:
    return N.COIN_DEVICE if coin == "device" else N.COIN_NEVER


def _ptr(t):
    """Pointer argument of a tensor (None: NULL).  A plain int: ctypes converts it for a c_void_p parameter, and the
    hot methods pass ``t.data_ptr()`` directly for the same reason (no pointer object per call)."""
    return None if t is None else t.data_ptr()


def _table_args(v):
    """The pointer and the three element strides of a table view (JssVecEnv._table_view), as the entry points take
    them.  The caller keeps `v` alive across the call: it may be a converted copy."""
    return (v.data_ptr(), *(int(s) for s in v.stride()))


def _best_slot(makespan):
    """Per row of an (N, k) int32 makespan tensor, the lowest column of smallest makespan among those that ended
    (>= 0), -1 if none: (N,) int64."""
    import torch
    ended = makespan >= 0
    best = torch.where(ended, makespan, torch.iinfo(torch.int32).max).argmin(1)
    return torch.where(ended.any(1), best, -1)


def _host_buffer(shape, dtype):
    """Host staging buffer, page-locked where the backend can pin (DMA target, device-mapped writes); a backend that
    does not declare ``pin_memory`` gets ordinary pageable memory."""
    import torch
    return torch.empty(shape, dtype=dtype, pin_memory=getattr(N.backend, "pin_memory", False))


@functools.lru_cache(maxsize=None)
def _sampled_log_prob():
    """The autograd Function of JssVecEnv.rollout_priority_sample's log_prob (made on first use: torch is imported
    lazily).  Forward runs the call with a gradient buffer; backward weights each env's gradient rows by the incoming
    gradient and sums them over the table's broadcast dimensions.  With `entropy`, forward also returns the entropy and
    stores its gradient rows, and backward adds those weighted by the entropy's incoming gradient."""
    import torch

    class SampledLogProb(torch.autograd.Function):
        @staticmethod
        def forward(ctx, logits, env, n_steps, entropy=False):
            # zero-filled: the kernel leaves the entries past J_i / M_i alone, and a broadcast table sums over them
            shape = (env.num_envs, env.jobs, env.machines)
            grad = torch.zeros(shape, dtype=torch.float32, device=env.device)
            hgrad = torch.zeros(shape, dtype=torch.float32, device=env.device) if entropy else None
            out = env._rollout_priority_sample(logits, n_steps, grad, entropy, hgrad)
            ctx.save_for_backward(grad, hgrad)
            ctx.shape, ctx.dtype = logits.shape, logits.dtype
            return out

        @staticmethod
        def backward(ctx, g, gh=None):
            grad, hgrad = ctx.saved_tensors
            total = g[:, None, None] * grad
            if hgrad is not None:
                total = total + gh[:, None, None] * hgrad
            return total.sum_to_size(ctx.shape).to(ctx.dtype), None, None, None

    return SampledLogProb


@functools.lru_cache(maxsize=None)
def _episodes_log_prob():
    """The autograd Function of JssVecEnv.sample_episodes' log_prob (made on first use).  Forward draws the episodes and
    saves the table, the RNG counter and the envs' state epoch; backward replays the draws (jss_sample_episodes_grad)
    with the incoming (N, k) gradient as weights, sums the chunks and then over the table's broadcast dimensions.  The
    replay starts from the envs' state at backward time, so backward raises RuntimeError, before any launch, if a call
    that may change that state ran after forward, or if the env was closed.  With `entropy`, forward also returns the
    (N, k) entropy, and the one replay takes its incoming gradient as the entropy weights."""
    import torch

    class EpisodesLogProb(torch.autograd.Function):
        @staticmethod
        def forward(ctx, logits, env, k, step_index, entropy=False):
            out = env._sample_episodes(logits, k, step_index, entropy)
            ctx.save_for_backward(logits)              # torch's version counter refuses a table changed in place
            ctx.env, ctx.k, ctx.step_index, ctx.entropy = env, k, step_index, entropy
            ctx.epoch = env._state_epoch
            ctx.mark_non_differentiable(out[0])
            return out

        @staticmethod
        def backward(ctx, _, g, gh=None):
            (logits,) = ctx.saved_tensors
            env = ctx.env
            env._check_replay(ctx.epoch, "sample_episodes")
            split = min(ctx.k, -(-env._warp_slots() // env.num_envs))
            grad = env._sample_episodes_grad(logits, ctx.k, ctx.step_index, g, split, gh)
            return grad.sum(0).sum_to_size(logits.shape).to(logits.dtype), None, None, None, None

    return EpisodesLogProb


@functools.lru_cache(maxsize=None)
def _order_log_prob_fn():
    """The autograd Function of the log_prob of JssVecEnv.order_log_prob and JssVecEnv.sample_without_replacement
    (made on first use; `who` names the call).  Forward runs `run(logits)`, which returns the (N, k) log_prob first,
    the (N, k, J, M) int32 orders last and any other outputs between, and saves the table, the orders and the envs'
    state epoch; backward calls jss_order_log_prob_grad with the incoming (N, k) gradient as weights, sums the chunks
    and then over the table's broadcast dimensions.  The orders are replayed from the envs' state at backward time, so
    backward raises RuntimeError, before any launch, if a call that may change that state ran after forward, or if the
    env was closed.  With `entropy`, `run` returns the (N, k) entropy second, differentiable too, and the one replay
    takes its incoming gradient as the entropy weights."""
    import torch

    class OrderLogProb(torch.autograd.Function):
        @staticmethod
        def forward(ctx, logits, env, run, who, entropy=False):
            outs = run(logits)
            ctx.save_for_backward(logits, outs[-1])    # torch's version counter refuses a table changed in place
            ctx.env, ctx.who, ctx.entropy, ctx.epoch = env, who, entropy, env._state_epoch
            ctx.mark_non_differentiable(*outs[2 if entropy else 1:])
            return outs

        @staticmethod
        def backward(ctx, g, *rest):
            logits, order = ctx.saved_tensors
            env = ctx.env
            env._check_replay(ctx.epoch, ctx.who)
            k = order.shape[1]
            split = min(k, -(-env._warp_slots() // env.num_envs))
            grad = env._order_log_prob_grad(logits, order, g, split, rest[0] if ctx.entropy else None)
            return grad.sum(0).sum_to_size(logits.shape).to(logits.dtype), None, None, None, None

    return OrderLogProb


def _state_views(b, n, J, M, view):
    """The canonical-state arrays of jss_export_state, each made by ``view(ptr, shape, dtype)``."""
    return {"todo": view(b.x_todo, (n, J), np.int32), "tufco": view(b.x_tufco, (n, J), np.int32),
            "idle_last": view(b.x_idle_last, (n, J), np.int32), "total_idle": view(b.x_total_idle, (n, J), np.int32),
            "col4": view(b.x_col4, (n, J), np.int32), "tuam": view(b.x_tuam, (n, M), np.int32),
            "legal": view(b.x_legal, (n, J), np.uint8), "blocked": view(b.x_blocked, (n, J), np.uint8)}


class JssVecEnv:
    def __init__(self, num_envs: int, env_config: Optional[Dict[str, Any]] = None, device: int = 0,
                 auto_reset: bool = False, record_solution: bool = False, env_id_base: int = 0, seed: int = 0,
                 host_mirror: bool = False):
        self._h = ctypes.c_void_p()
        self._L = N.backend.library()
        self.num_envs = int(num_envs)
        self.device_index = int(device)
        self.seed = int(seed)
        self.env_id_base = int(env_id_base)
        self.auto_reset = bool(auto_reset)
        self._step_index = 0
        # bumped by every call that may change an env's state: a replayed gradient refuses to run across a bump
        self._state_epoch = 0
        insts, env_to_inst = _instance_list(env_config)
        self.instances = insts
        flags = ((N.CREATE_AUTO_RESET if auto_reset else 0) | (N.CREATE_RECORD_SOLUTION if record_solution else 0) |
                 (N.CREATE_HOST_MIRROR if host_mirror else 0))
        rc = self._L.jss_create(ctypes.byref(self._h), self.device_index, self.num_envs, flags, self.env_id_base)
        N.check(None, rc, "jss_create")
        # instance tables (jss_env.py:72-95)
        jobs = np.array([m.shape[0] for m, _ in insts], np.int32)
        machines = np.array([m.shape[1] for m, _ in insts], np.int32)
        sizes = jobs.astype(np.int64) * machines
        offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        mach = np.concatenate([m.reshape(-1) for m, _ in insts]).astype(np.int32)
        dur = np.concatenate([d.reshape(-1) for _, d in insts]).astype(np.int32)
        rc = self._L.jss_load_instances(self._h, len(insts), N.as_i32p(jobs), N.as_i32p(machines),
                                        offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                        N.as_i32p(mach), N.as_i32p(dur))
        N.check(self._h, rc, "jss_load_instances")
        if env_to_inst is None:
            env_to_inst = np.arange(self.num_envs) % len(insts)
        self.env_to_instance = np.ascontiguousarray(env_to_inst, dtype=np.int32)
        assert self.env_to_instance.shape == (self.num_envs,)
        rc = self._L.jss_assign(self._h, N.as_i32p(self.env_to_instance))   # also performs the first reset
        N.check(self._h, rc, "jss_assign")
        self.env_jobs = jobs[self.env_to_instance]           # J_i per env (no-op index of env i)
        self.env_machines = machines[self.env_to_instance]
        sc = np.zeros((len(insts), 3), np.int64)
        for k in range(len(insts)):
            N.check(self._h, self._L.jss_instance_scalars(
                self._h, k, sc[k].ctypes.data_as(ctypes.POINTER(ctypes.c_int64))), "jss_instance_scalars")
        self.instance_scalars = sc                           # max_time_op, max_time_jobs, sum_op
        b = N.JssBuffers()
        N.check(self._h, self._L.jss_get_buffers(self._h, ctypes.byref(b)), "jss_get_buffers")
        self._b = b
        self.jobs, self.machines = int(b.jobs_max), int(b.machines_max)
        n, J, M, w = self.num_envs, self.jobs, self.machines, N.backend.wrap
        d = self.device_index
        self.device = N.backend.torch_device(d)
        import torch
        self._mask_u8 = w(b.action_mask, (n, J + 1), np.uint8, d, strides=(b.mask_stride, 1))
        self.action_mask = self._mask_u8.view(torch.bool)
        # stale after step_logits_record() until the next non-recording call or refresh_obs()
        self.real_obs = w(b.real_obs, (n, J, 7), np.float32, d)
        ss = (int(b.scalar_stride),)      # the five scalar outputs are fields of one 16-byte record per env
        self.reward = w(b.reward, (n,), np.float32, d, strides=ss)
        self.reward_raw = w(b.reward_raw, (n,), np.int32, d, strides=ss)
        self.done = w(b.done, (n,), np.uint8, d, strides=ss).view(torch.bool)
        self.current_time_step = w(b.time, (n,), np.int32, d, strides=ss)
        self._flags_done = w(b.flags_done, (n,), np.int32, d, strides=ss)
        self.solution = w(b.solution, (n, J, M), np.int32, d) if b.solution else None
        self.episode_count = w(b.episode_count, (n,), np.int32, d)
        self.last_makespan = w(b.last_makespan, (n,), np.int32, d)
        self.last_return = w(b.last_return, (n,), np.int32, d)
        self._x = _state_views(b, n, J, M, lambda ptr, shape, dt: w(ptr, shape, dt, d))
        self.host = None
        if b.host_mirror:
            # JSS_CREATE_HOST_MIRROR: the same memory seen from the host (pinned, device-mapped): numpy views, no copies
            hv = N.host_view
            self.host = {
                "action_mask": hv(b.action_mask, (n, J + 1), np.uint8, strides=(int(b.mask_stride), 1)),
                "real_obs": hv(b.real_obs, (n, J, 7), np.float32), "scalars": hv(b.reward, (n, 4), np.int32),
                **_state_views(b, n, J, M, hv),
                "actions": hv(b.mirror_actions, (n,), np.int32),
            }
            self._mirror_actions = w(b.mirror_actions, (n,), np.int32, d)
        self._truncated = torch.zeros(n, dtype=torch.bool, device=self.device)
        self._actions = torch.zeros(n, dtype=torch.int32, device=self.device)

    @property
    def flags(self):
        """Per-env JSS_FLAG_* bits (done / error / no-op legal) as an int32 tensor."""
        return self._flags_done >> 8

    # ---------------------------------------------------------------- lifetime
    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.jss_destroy(self._h)
            self._h = ctypes.c_void_p()

    def _check_replay(self, epoch: int, who: str):
        """Refuses the replayed backward of an output of `who` made at state epoch `epoch` once the handle is closed or
        a call that may change an env's state ran since: the replay would call into a destroyed handle, or walk other
        episodes than the ones the output describes."""
        if not self._h.value:
            raise RuntimeError(f"{who}: backward after close(): the gradient is replayed on the envs, so take it before "
                               f"closing them")
        if self._state_epoch != epoch:
            raise RuntimeError(f"{who}: backward after a call that may have changed the envs' state (a step, reset, "
                               f"rollout, beam step or import_state): the gradient is replayed from the current state, "
                               f"so run {who} again from the new state")

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return N.backend.stream(self.device_index)

    def _obs(self):
        return {"real_obs": self.real_obs, "action_mask": self.action_mask}

    def _device_i32(self, actions):
        """`actions` as a contiguous int32 tensor on the env's device (the tensor itself if it already is one)."""
        import torch
        a = torch.as_tensor(actions, device=self.device)
        if a.dtype != torch.int32 or not a.is_contiguous():
            a = a.to(torch.int32).contiguous()
        return a

    def _env_mask(self, mask):
        """Env selection mask (nonzero = selected) as a contiguous uint8 device tensor; None selects every env."""
        if mask is None:
            return None
        import torch
        return torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous()

    # ---------------------------------------------------------------- reference API, batched
    def reset(self, mask=None):
        """reset() of every env (or of the envs where `mask` is nonzero) -> obs (jss_env.py:145-181)."""
        m = self._env_mask(mask)
        self._state_epoch += 1
        N.check(self._h, self._L.jss_reset(self._h, _ptr(m), self._stream()), "jss_reset")
        return self._obs()

    def step(self, actions):
        """actions: int32[N] on the env's device (torch) or anything torch.as_tensor accepts."""
        a = self._device_i32(actions)
        self._state_epoch += 1
        N.check(self._h, self._L.jss_step(self._h, a.data_ptr(), self._stream()), "jss_step")
        return self._obs(), self.reward, self.done, self._truncated, {}

    def step_export_host(self):
        """Host-mirror batches (the single-env facade): apply the actions written to ``self.host["actions"]`` and decode
        the new state into the x_* arrays in ONE launch (jss_step_export), then wait; afterwards every array of
        ``self.host`` is current.  No per-transition copies: the kernels write straight into the pinned block."""
        self._state_epoch += 1
        rc = self._L.jss_step_export(self._h, self._mirror_actions.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_step_export")
        N.backend.synchronize(self.device_index)

    def step_sample(self, actions, rule: Union[str, int] = "RANDOM", coin: str = "device", out=None):
        """step(actions) fused with policy(rule) for the next decision (one launch): returns the usual
        step tuple plus the int32[N] tensor of next actions (`out`, default: in place of `actions`)."""
        a = self._device_i32(actions)
        out = a if out is None else out
        self._state_epoch += 1
        rc = self._L.jss_step_sample(self._h, a.data_ptr(), _rule_id(rule), _coin_id(coin), self.seed,
                                     self._step_index, out.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_step_sample")
        self._step_index += 1
        return self._obs(), self.reward, self.done, self._truncated, {}, out

    def _logits_arg(self, logits, what):
        """`logits` as an (N, >= J+1) float32 device tensor with unit column stride (converted only if needed), and its
        row stride `ld` in elements."""
        import torch
        n, J = self.num_envs, self.jobs
        x = torch.as_tensor(logits, device=self.device)
        if x.dim() != 2 or x.shape[0] != n or x.shape[1] < J + 1:
            raise ValueError(f"{what}: logits must have shape ({n}, >= {J + 1}), got {tuple(x.shape)}")
        if x.dtype != torch.float32 or x.stride(1) != 1 or (n > 1 and x.stride(0) < J + 1):
            x = x.to(torch.float32).contiguous()
        return x, (x.stride(0) if n > 1 else max(x.stride(0), J + 1))

    @staticmethod
    def _epsilon_arg(epsilon, what):
        e = float(epsilon)
        if not 0.0 <= e <= 1.0:                           # NaN included
            raise ValueError(f"{what}: epsilon must be in [0, 1], got {epsilon!r}")
        return e

    def _row_call(self, what, x, ld, pre, acts, logp, slot=()):
        """The native call of the steps that take their action from a row (`what` = step_logits, step_greedy or their
        _record forms): jss_<what>(h, row, ld, *pre, seed, step_index, actions_out, log_prob_out, *slot, stream); then
        the RNG counter advances."""
        self._state_epoch += 1
        rc = getattr(self._L, "jss_" + what)(self._h, x.data_ptr(), int(ld), *pre, self.seed, self._step_index,
                                             acts.data_ptr(), logp.data_ptr(), *slot, self._stream())
        N.check(self._h, rc, "jss_" + what)
        self._step_index += 1

    def _row_step(self, what, rows, pre, actions_out, log_prob_out):
        """step_logits / step_greedy: the row and output checks, the call, and the step tuple."""
        import torch
        n = self.num_envs
        x, ld = self._logits_arg(rows, what)
        if actions_out is None:
            actions_out = torch.empty(n, dtype=torch.int32, device=self.device)
        if log_prob_out is None:
            log_prob_out = torch.empty(n, dtype=torch.float32, device=self.device)
        for t, dt in ((actions_out, torch.int32), (log_prob_out, torch.float32)):
            if t.dtype != dt or t.shape != (n,) or not t.is_contiguous() or t.device != x.device:
                raise ValueError(f"{what}: outputs must be contiguous {dt} tensors of shape ({n},) on {x.device}")
        self._row_call(what, x, ld, pre, actions_out, log_prob_out)
        return self._obs(), self.reward, self.done, self._truncated, {"actions": actions_out, "log_prob": log_prob_out}

    def _row_record(self, what, rows, pre, traj, k):
        """step_logits_record / step_greedy_record: the trajectory and row checks, the call into slot `k`, and the step
        tuple of the slot's views."""
        K = self._check_trajectory(traj, what)
        if not 0 <= k < K:
            raise ValueError(f"{what}: step {k} outside the trajectory's {K} steps")
        x, ld = self._logits_arg(rows, what)
        acts, logp = traj["actions"][k], traj["log_prob"][k]
        slot = (traj["real_obs"][k + 1].data_ptr(), traj["_mask_rows"][k + 1].data_ptr(), traj["_scalars"][k].data_ptr())
        self._row_call(what, x, ld, pre, acts, logp, slot)
        obs = {"real_obs": traj["real_obs"][k + 1], "action_mask": traj["action_mask"][k + 1]}
        return obs, traj["reward"][k], traj["done"][k], self._truncated, {"actions": acts, "log_prob": logp}

    def step_logits(self, logits, actions_out=None, log_prob_out=None):
        """Step every env with an action drawn from policy logits (jss_step_logits, one launch): a masked categorical
        draw (Gumbel-max over the legal actions, RNG counter ``self._step_index``), then the step.  `logits`: (N, >= J+1)
        tensor on the env's device whose columns line up with ``action_mask``; converted to float32 with unit column
        stride only if needed.  Returns the step tuple with ``{"actions": int32 (N,), "log_prob": float32 (N,)}`` as info.
        A done env gets action 0 and log_prob 0, an env whose only legal action is the no-op gets J_i and 0, and an env
        whose legal logits are bad (NaN / +inf, or all -inf) gets the error bit, action JSS_ACTION_SKIP and NaN."""
        return self._row_step("step_logits", logits, (), actions_out, log_prob_out)

    def step_greedy(self, scores, epsilon: float = 0.0, actions_out=None, log_prob_out=None):
        """Step every env with the epsilon-greedy action of its scores (jss_step_greedy, one launch): the legal action
        with the largest score (ties to the lowest index) with probability 1 - epsilon, else a uniformly random legal
        action (RNG counter ``self._step_index``), then the step.  epsilon = 0 is greedy evaluation
        (``deterministic=True``), epsilon > 0 the behaviour policy of a value-based agent.  `scores` (logits or
        Q-values) are taken like step_logits' logits.  Returns the step tuple with ``{"actions", "log_prob"}`` as info;
        log_prob is the action's log-probability under the epsilon-greedy policy (0 at epsilon = 0).  Done, no-op-only
        and bad-score envs are handled as in step_logits()."""
        e = self._epsilon_arg(epsilon, "step_greedy")
        return self._row_step("step_greedy", scores, (e,), actions_out, log_prob_out)

    def logits_trajectory(self, n_steps: int, out: Optional[Dict[str, Any]] = None):
        """Rollout buffers for `n_steps` recorded logits steps (step_logits_record), as device tensors:
        ``real_obs`` (K+1, N, J, 7) f32, ``action_mask`` (K+1, N, J+1) bool, and ``actions``, ``log_prob``, ``reward``,
        ``reward_raw``, ``done``, ``time``, each (K, N).  Allocated zero-filled, or `out` reused when it has K steps;
        either way the current observation and mask are copied into slot 0 (after refresh_obs()), so that
        ``real_obs[k]`` is what the network sees at step k and ``real_obs[K]`` is the bootstrap observation."""
        import torch
        K, n, J, ms = int(n_steps), self.num_envs, self.jobs, int(self._b.mask_stride)
        if out is None or out["actions"].shape[0] != K:
            dev = self.device
            # each observation / mask slot starts 16-byte aligned (jss_step_logits_record), whatever N and J are
            obs_w, mask_w = -(-n * J * 7 // 4) * 4, -(-n * ms // 16) * 16
            out = {"_obs": torch.zeros((K + 1, obs_w), dtype=torch.float32, device=dev),
                   "_mask": torch.zeros((K + 1, mask_w), dtype=torch.uint8, device=dev),
                   "_scalars": torch.zeros((K, n, 4), dtype=torch.int32, device=dev),
                   "actions": torch.zeros((K, n), dtype=torch.int32, device=dev),
                   "log_prob": torch.zeros((K, n), dtype=torch.float32, device=dev)}
            out["real_obs"] = out["_obs"][:, : n * J * 7].view(K + 1, n, J, 7)
            out["_mask_rows"] = out["_mask"][:, : n * ms].view(K + 1, n, ms)
            out["action_mask"] = out["_mask_rows"][:, :, : J + 1].view(torch.bool)
            out["reward"] = out["_scalars"][:, :, 0].view(torch.float32)
            out["reward_raw"] = out["_scalars"][:, :, 1]
            out["time"] = out["_scalars"][:, :, 2]
            out["done"] = out["_scalars"].view(torch.uint8)[:, :, 12].view(torch.bool)   # low byte of flags << 8 | done
        self._check_trajectory(out, "logits_trajectory")
        self.refresh_obs()
        out["real_obs"][0].copy_(self.real_obs)
        out["_mask_rows"][0][:, : J + 1].copy_(self._mask_u8)
        return out

    def _check_trajectory(self, traj, what):
        """The number of steps K of a logits_trajectory() dict, after checking that every buffer the kernel writes has
        this env's layout (a dict made for another env would let it write past the tensors)."""
        import torch
        K, n, J, ms = traj["actions"].shape[0], self.num_envs, self.jobs, int(self._b.mask_stride)
        want = {"real_obs": ((K + 1, n, J, 7), torch.float32), "_mask_rows": ((K + 1, n, ms), torch.uint8),
                "_scalars": ((K, n, 4), torch.int32), "actions": ((K, n), torch.int32),
                "log_prob": ((K, n), torch.float32)}
        for name, (shape, dt) in want.items():
            t = traj[name]
            if tuple(t.shape) != shape or t.dtype != dt or t.device != self.device or not t[0].is_contiguous():
                raise ValueError(f"{what}: trajectory buffer {name!r} is {tuple(t.shape)} {t.dtype} on {t.device}, "
                                 f"this env needs {shape} {dt} on {self.device} (rows contiguous)")
        return K

    def step_logits_record(self, logits, traj: Dict[str, Any], k: int):
        """step_logits() that records transition `k` straight into `traj` (a logits_trajectory() dict) in the same
        launch (jss_step_logits_record): ``actions[k]``, ``log_prob[k]``, ``reward[k]``, ``reward_raw[k]``, ``done[k]``,
        ``time[k]`` and the next observation ``real_obs[k+1]`` / ``action_mask[k+1]``.  An env the step left unchanged
        (frozen done, error bit) records reward 0.  The env's own action_mask, rewards, state and statistics end up
        exactly as after step_logits(); its real_obs is left stale (see refresh_obs()).  Returns the step tuple of the
        slot's views."""
        return self._row_record("step_logits_record", logits, (), traj, k)

    def step_greedy_record(self, scores, traj: Dict[str, Any], k: int, epsilon: float = 0.0):
        """step_greedy() that records transition `k` straight into `traj` (a logits_trajectory() dict) in the same
        launch (jss_step_greedy_record), as step_logits_record() does for step_logits()."""
        e = self._epsilon_arg(epsilon, "step_greedy_record")
        return self._row_record("step_greedy_record", scores, (e,), traj, k)

    def refresh_obs(self):
        """Bring ``real_obs`` up to date after recording steps (jss_refresh_obs; nothing to do otherwise).  Every other
        native call does this by itself, so it is only needed to read ``real_obs`` right after step_logits_record()."""
        N.check(self._h, self._L.jss_refresh_obs(self._h, self._stream()), "jss_refresh_obs")

    def get_legal_actions(self):
        return self.action_mask

    # ---------------------------------------------------------------- policies on device
    def policy(self, rule: Union[str, int] = "RANDOM", coin: str = "device", out=None, step_index=None):
        """Device-side action selection (masked-uniform sampler or a dispatching rule)."""
        r = _rule_id(rule)
        out = self._actions if out is None else out
        if step_index is None:
            step_index = self._step_index
            self._step_index += 1
        rc = self._L.jss_policy(self._h, r, _coin_id(coin), self.seed, int(step_index), out.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_policy")
        return out

    def set_cr_due_date_factor(self, factor: float):
        """CriticalRatio(due_date_factor) of the reference (dispatching.py:337-349) for later CR launches."""
        N.check(self._h, self._L.jss_set_cr_due_date_factor(self._h, float(factor)), "jss_set_cr_due_date_factor")

    def rollout(self, rule: Union[str, int], n_steps: int, write_obs: bool = True):
        """n_steps x (policy -> step) fused on device (DispatchingRule.run_episode, dispatching.py:55-75)."""
        self._state_epoch += 1
        rc = self._L.jss_rollout(self._h, _rule_id(rule), self.seed, self._step_index, int(n_steps),
                                 int(bool(write_obs)), self._stream())
        N.check(self._h, rc, "jss_rollout")
        self._step_index += int(n_steps)
        return self._obs(), self.reward, self.done, self._truncated, {}

    def rollout_priority(self, priorities, n_steps: Optional[int] = None):
        """Run a static priority rule to the end of every env's episode in one launch per lane class
        (jss_rollout_priority): at each decision the legal job whose current operation has the largest priority
        (ties to the lowest job index), the no-op only when no job is legal.  `priorities`: a 3-D tensor on the env's
        device whose shape broadcasts to (N, J, M), J and M the batch maxima: (N, J, 1) gives one priority per job,
        (1, J, M) one table for every env; converted to float32 only if needed.  Each env makes at most `n_steps`
        decisions (default 2*J*M + 1, enough for any episode), never resets, and a done env is left untouched; bad
        priorities (NaN / +inf on a legal current operation, or every legal job at -inf) set the error bit and stop
        that env.  Returns the step tuple; the RNG counter does not advance."""
        J, M = self.jobs, self.machines
        v = self._table_view(self._table_arg(priorities, "rollout_priority", "priorities"))
        if n_steps is None:
            n_steps = 2 * J * M + 1
        self._state_epoch += 1
        rc = self._L.jss_rollout_priority(self._h, *_table_args(v), int(n_steps), self._stream())
        N.check(self._h, rc, "jss_rollout_priority")
        return self._obs(), self.reward, self.done, self._truncated, {}

    def rollout_priority_sample(self, logits, n_steps: Optional[int] = None, entropy: bool = False):
        """Run every env to the end of its episode in one launch per lane class, each decision drawn from the softmax
        over the legal jobs of the entries of their current operations (jss_rollout_priority_sample; the no-op only
        when no job is legal).  `logits` and `n_steps` are taken as rollout_priority's priorities and n_steps.  Decision
        d of the call uses RNG counter ``self._step_index + d`` and equals a step_logits() draw on the gathered row;
        the counter then advances by `n_steps`.  Returns the step tuple with ``{"log_prob": float32 (N,)}`` as info:
        each env's sum of its decisions' log-probabilities in this call (NaN for an env that got the error bit).  When
        `logits` requires grad (and grad mode is on), log_prob is differentiable with respect to it: the kernel also
        writes d log_prob / d table, and broadcast tables such as (1, J, M) get the gradient summed over the envs.
        With `entropy`, info also holds ``"entropy"`` float32 (N,): each env's sum over its decisions in this call of
        the policy's entropy at the decision, H_t = log S - T/S over the legal jobs (jss_rollout_priority_sample_entropy;
        forced no-ops add 0, NaN where log_prob is NaN); everything else is bit for bit what the call without it gives.
        With a table that requires grad, log_prob and entropy are then both differentiable from one stored forward."""
        import torch
        J, M = self.jobs, self.machines
        x = self._table_arg(logits, "rollout_priority_sample", "logits")
        n_steps = 2 * J * M + 1 if n_steps is None else int(n_steps)
        if x.requires_grad and torch.is_grad_enabled():
            out = _sampled_log_prob().apply(x, self, n_steps, True) if entropy else \
                _sampled_log_prob().apply(x, self, n_steps)
        else:
            out = self._rollout_priority_sample(x, n_steps, None, entropy)
        info = {"log_prob": out[0], "entropy": out[1]} if entropy else {"log_prob": out}
        return self._obs(), self.reward, self.done, self._truncated, info

    def _rollout_priority_sample(self, x, n_steps: int, grad_out, entropy: bool = False, entropy_grad_out=None):
        """The native call of rollout_priority_sample on a checked table `x` (read through a detached float32 view,
        strides passed through); writes the gradient to `grad_out` ((N, J, M) float32, or None); advances the RNG
        counter.  Returns log_prob, or with `entropy` (log_prob, entropy) and the entropy's gradient written to
        `entropy_grad_out` (as grad_out)."""
        import torch
        v = self._table_view(x)
        log_prob = torch.empty(self.num_envs, dtype=torch.float32, device=self.device)
        self._state_epoch += 1
        if entropy:
            ent = torch.empty(self.num_envs, dtype=torch.float32, device=self.device)
            rc = self._L.jss_rollout_priority_sample_entropy(self._h, *_table_args(v), self.seed, self._step_index,
                                                             n_steps, log_prob.data_ptr(), ent.data_ptr(),
                                                             _ptr(grad_out), _ptr(entropy_grad_out), self._stream())
            N.check(self._h, rc, "jss_rollout_priority_sample_entropy")
            self._step_index += n_steps
            return log_prob, ent
        rc = self._L.jss_rollout_priority_sample(self._h, *_table_args(v), self.seed, self._step_index, n_steps,
                                                 log_prob.data_ptr(), _ptr(grad_out), self._stream())
        N.check(self._h, rc, "jss_rollout_priority_sample")
        self._step_index += n_steps
        return log_prob

    def lookahead(self, rule: Union[str, int] = "MWR", coin: str = "never", out=None):
        """Value every legal action by a rollout of `rule` to the end of the episode, in one launch per lane class
        (jss_lookahead), leaving the envs untouched: out[i, a] is the makespan env i reaches if it takes action a now
        and then follows `rule` (as policy(rule, coin) with RNG counters ``self._step_index + d``, the same for every
        action of an env), -1 for an action that is not legal, every action of a done env, and a rollout that stops
        before done (only from an imported state).  Returns `out`, an (N, >= J+1) contiguous int32 device tensor;
        by default a fresh (N, J+1) one filled with -1, so that the columns past an env's J_i read -1 too (the call
        writes only columns 0..J_i).  coin="never" makes each value exact and the rollout method (take the argmin,
        repeat) never worse than the rule alone; "device" gives the reference's 10 % wait draw.  The RNG counter
        advances by 2*J*M + 1, the rule decisions a candidate may take."""
        J = self.jobs
        if isinstance(rule, str) and rule.upper() not in N.RULES:
            raise ValueError(f"lookahead: unknown rule {rule!r} (one of {sorted(N.RULES)})")
        if coin not in ("never", "device"):
            raise ValueError(f"lookahead: coin must be 'never' or 'device', got {coin!r}")
        out = self._values_out(out, "lookahead")
        rc = self._L.jss_lookahead(self._h, _rule_id(rule), _coin_id(coin), self.seed, self._step_index,
                                   out.data_ptr(), int(out.shape[1]), self._stream())
        N.check(self._h, rc, "jss_lookahead")
        self._step_index += 2 * J * self.machines + 1
        return out

    def lookahead_priority(self, priorities, out=None):
        """Value every legal action by a greedy rollout of the priority table `priorities` to the end of the episode, in
        one launch per lane class (jss_lookahead_priority), leaving the envs untouched: out[i, a] is the makespan env i
        reaches if it takes action a now and then follows the table as rollout_priority() does (the legal job whose
        current operation has the largest priority, ties to the lowest index, the no-op only when no job is legal); -1
        for an action that is not legal, every action of a done env, and a rollout that stops before done, such as one
        that meets a bad entry (NaN / +inf on a legal current operation, or every legal job at -inf; no error bit is
        set).  `priorities` is taken as by rollout_priority(); a table that requires grad is read detached (the values
        have no gradient).  `out` is taken and returned as by lookahead().  The argmin of the values, taken at every
        decision, is never worse than rollout_priority(priorities) from the same state.  No RNG: the counter does not
        advance."""
        v = self._table_view(self._table_arg(priorities, "lookahead_priority", "priorities"))
        out = self._values_out(out, "lookahead_priority")
        rc = self._L.jss_lookahead_priority(self._h, *_table_args(v), out.data_ptr(), int(out.shape[1]), self._stream())
        N.check(self._h, rc, "jss_lookahead_priority")
        return out

    def lookahead_sample(self, logits, k: int, out=None):
        """Value every legal action by `k` episodes drawn from the logit table `logits` after it, in one launch per lane
        class (jss_lookahead_sample), leaving the envs untouched: the action values Q(s, a) of the table's stochastic
        policy.  With B = 2*J*M + 1, ``"makespan"[i, a, s]`` is the makespan env i reaches if it takes action a now and
        then draws as sample s of sample_episodes(logits, k) would (decision d at RNG counter ``self._step_index +
        s*B + d``), or its end time at once if a ends the episode; -1 for an action that is not legal (the no-op
        unless it is), every action of a done env, and a sample that stops before done, such as one that meets a bad
        entry (no error bit is set).  Every action of an env uses the same counters (common random numbers), so
        differences between actions reflect the action, not the noise.  `logits` is taken as by
        rollout_priority_sample(); a table that requires grad is read detached (the values have no gradient).  `out`:
        a contiguous int32 (N, J+1, k) device tensor; by default a fresh one filled with -1, so that the columns past
        an env's J_i read -1 too (the call writes only columns 0..J_i).  Returns a dict of device tensors: ``"makespan"``
        (`out`); ``"mean"`` (N, J+1) float32, the mean over the samples that ended (computed in float64), NaN where
        none did; ``"min"`` (N, J+1) int32, their best, -1 where none did.  The RNG counter advances by k*B."""
        import torch
        n, J, M = self.num_envs, self.jobs, self.machines
        v = self._table_view(self._table_arg(logits, "lookahead_sample", "logits"))
        if int(k) < 1:
            raise ValueError(f"lookahead_sample: k must be at least 1, got {k!r}")
        k = int(k)
        if out is None:
            out = torch.full((n, J + 1, k), -1, dtype=torch.int32, device=self.device)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.int32 or tuple(out.shape) != (n, J + 1, k)
              or not out.is_contiguous() or out.device != self.device):
            raise ValueError(f"lookahead_sample: out must be a contiguous int32 tensor of shape ({n}, {J + 1}, {k}) "
                             f"on the env's device")
        rc = self._L.jss_lookahead_sample(self._h, *_table_args(v), self.seed, self._step_index, k, out.data_ptr(),
                                          (J + 1) * k, self._stream())
        N.check(self._h, rc, "jss_lookahead_sample")
        self._step_index += k * (2 * J * M + 1)
        ended = out >= 0
        count = ended.sum(2)
        total = torch.where(ended, out, 0).sum(2, dtype=torch.float64)
        mean = torch.where(count > 0, total / count, torch.nan).to(torch.float32)
        best = torch.where(ended, out, torch.iinfo(torch.int32).max).amin(2)
        best = torch.where(count > 0, best, -1)
        return {"makespan": out, "mean": mean, "min": best}

    def sample_episodes(self, logits, k: int, solution: bool = False, entropy: bool = False):
        """Draw `k` whole episodes per env from the logit table `logits`, each from the env's current state, in one
        launch per lane class (jss_sample_episodes), leaving the envs untouched.  With B = 2*J*M + 1, sample s of env i
        is the episode rollout_priority_sample(logits) would draw from this state with the RNG counter at
        ``self._step_index + s*B``; the counter then advances by k*B.  `logits` is taken as by rollout_priority_sample().
        Returns a dict of device tensors: ``"makespan"`` (N, k) int32, the end time of each sample (-1 if it does not
        end done: a bad table entry on its path, or an env done now); ``"log_prob"`` (N, k) float32, each sample's
        log-probability (NaN where it meets a bad entry, 0 for an env done now); ``"best"`` (N,) int64, the lowest-index
        sample of smallest makespan, -1 if none ended; with `solution`, ``"solution"`` (N, J, M) int32, the start times
        of the best sample's operations over this env's solution so far (-1 without record_solution).  When `logits`
        requires grad (and grad mode is on), log_prob is differentiable with respect to it: the backward replays the
        draws from the envs' state, so it raises RuntimeError after a call that may change that state (a step, reset,
        rollout, beam step or import_state) or after close(); draw again instead.  With `entropy`, the dict
        also holds ``"entropy"`` (N, k) float32, each sample's policy entropy as rollout_priority_sample(entropy=True)
        reports it for the same episode (0 for an env done now); with a table that requires grad it is differentiable
        too, and one replay gives the gradient of both."""
        import torch
        J, M = self.jobs, self.machines
        x = self._table_arg(logits, "sample_episodes", "logits")
        if int(k) < 1:
            raise ValueError(f"sample_episodes: k must be at least 1, got {k!r}")
        k, step_index = int(k), self._step_index
        if x.requires_grad and torch.is_grad_enabled():
            res = _episodes_log_prob().apply(x, self, k, step_index, True) if entropy else \
                _episodes_log_prob().apply(x, self, k, step_index)
        else:
            res = self._sample_episodes(x, k, step_index, entropy)
        makespan, log_prob = res[0], res[1]
        self._step_index += k * (2 * J * M + 1)
        best = _best_slot(makespan)
        out = {"makespan": makespan, "log_prob": log_prob, "best": best}
        if entropy:
            out["entropy"] = res[2]
        if solution:
            sol = (self.solution.clone() if self.solution is not None
                   else torch.full((self.num_envs, J, M), -1, dtype=torch.int32, device=self.device))
            v = self._table_view(x)
            b32 = best.to(torch.int32)
            rc = self._L.jss_sample_episodes_solution(self._h, *_table_args(v), self.seed, step_index, b32.data_ptr(),
                                                      sol.data_ptr(), self._stream())
            N.check(self._h, rc, "jss_sample_episodes_solution")
            out["solution"] = sol
        return out

    def beam_search(self, logits, width: int, order: bool = False):
        """Decode the logit table `logits` by beam search from each env's current state, in one launch per lane class
        (jss_beam_search), leaving the envs untouched.  Each round allocates one job per beam: every legal job of every
        beam is a candidate scored by the beam's score plus the job's log-probability under the softmax over the legal
        jobs' current-operation entries (exactly rollout_priority_sample()'s), and the `width` best candidates -- score
        descending, then parent slot, then job index -- are kept.  A beam takes the no-op only when no job is legal and
        it is.  After the last operation every kept beam is complete, and its score is, bit for bit, the log_prob
        rollout_priority_sample() reports for the same episode.  `logits` is taken as by rollout_priority_sample(); a
        table that requires grad is read detached (the search has no gradient).  Deterministic: the RNG counter does
        not advance.  Returns a dict of device tensors: ``"makespan"`` (N, width) int32 and ``"score"`` (N, width)
        float32 of the final slots, best score first (-1 and -inf for a slot without a complete beam, -1 and NaN in
        every slot of an env whose every beam met a bad entry, -1 and 0 for an env done now); ``"best"`` (N,) int64,
        the lowest slot of smallest makespan, -1 if none; with `order`, ``"order"`` (N, J, M) int32, the round at which
        the best slot allocates each operation (-1 for operations started before the call, and everywhere for an env
        without a complete beam).  The best schedule is replayed greedily from the same state by::

            env.rollout_priority(-out["order"])    # ends done at out["makespan"][i, out["best"][i]]
        """
        import torch
        x = self._table_arg(logits, "beam_search", "logits")
        if not 1 <= int(width) <= N.MAX_BEAM_WIDTH:
            raise ValueError(f"beam_search: width must be in 1..{N.MAX_BEAM_WIDTH}, got {width!r}")
        width = int(width)
        v = self._table_view(x)
        makespan = torch.empty((self.num_envs, width), dtype=torch.int32, device=self.device)
        score = torch.empty((self.num_envs, width), dtype=torch.float32, device=self.device)
        ord_ = (torch.full((self.num_envs, self.jobs, self.machines), -1, dtype=torch.int32, device=self.device)
                if order else None)
        rc = self._L.jss_beam_search(self._h, *_table_args(v), width, makespan.data_ptr(), score.data_ptr(), width,
                                     _ptr(ord_), self._stream())
        N.check(self._h, rc, "jss_beam_search")
        out = {"makespan": makespan, "score": score, "best": _best_slot(makespan)}
        if order:
            out["order"] = ord_
        return out

    def beam_step(self, logits, width: int, score, parent_out=None, action_out=None):
        """One round of beam search for a policy that reads the observation at every decision (jss_beam_step, one
        launch per lane class): the envs form groups of `width` consecutive envs, one search each, env g*width + b
        holding slot b of group g; every env of a group must run the same instance.  `score` is the (N,) float32 device
        tensor of the slots' scores, updated in place; a slot is live iff its score is finite (a search starts at
        [0, -inf, ..., -inf] per group).  `logits` (N, >= J+1) gives each slot's row, taken as step_logits() takes it (a
        tensor that requires grad is read detached); only a live, not-done slot's legal columns are read.  Every live,
        not-done slot's legal jobs are candidates scored by its score plus the job's log-softmax over its legal columns
        (as beam_search() computes it); the `width` best per group (score descending, then parent slot, then job) are
        stepped into the group's slots, each then taking the no-op while no job is legal and the no-op is.  A group
        without a live, not-done slot is left untouched.  No statistics, solution, auto-reset or RNG.  Returns
        ``(parent, action, bad)``: int32 (N,) tensors of each slot's parent slot and job (-1 / -1 for an empty slot,
        b / -1 in an untouched group; `parent_out` / `action_out` when given), and int32 (N / width,) bad, 1 where a
        beam of the group met a bad row (NaN / +inf at a legal job, or all legal jobs -inf).  ObsBeamSearch
        (jssenv_b200.beam) drives whole searches with it."""
        return self._beam_step("beam_step", logits, width, score, None, None, parent_out, action_out)

    def stochastic_beam_step(self, logits, width: int, score, key, step_index: int, parent_out=None, action_out=None):
        """One round of stochastic beam search (Kool et al., 2019) for a policy that reads the observation at every
        decision (jss_stochastic_beam_step, one launch per lane class): beam_step() with each candidate's score
        perturbed by top-down Gumbel noise and the `width` best per group ranked by that perturbed log-probability, the
        key.  `key` is the (N,) float32 device tensor of the slots' keys, updated in place like `score` (a search starts
        at key [0, -inf, ..., -inf] per group); `score` stays each slot's log-probability under its rows.  The noise of
        group g is drawn from ``self.seed``, the group's global id env_id_base / width + g (env_id_base must be a
        multiple of width) and the explicit RNG counter `step_index`, one per round; the env's own counter does not
        move.  Over a whole search (ObsBeamSearch(stochastic=True)) the slots of a group are distinct episodes drawn
        without replacement from the policy.  Returns ``(parent, action, bad)`` as beam_step()."""
        return self._beam_step("stochastic_beam_step", logits, width, score, key, int(step_index), parent_out,
                               action_out)

    def _beam_step(self, who, logits, width, score, key, step_index, parent_out, action_out):
        """The checked native call of beam_step (key None) and stochastic_beam_step."""
        import torch
        n = self.num_envs
        if not 1 <= int(width) <= N.MAX_BEAM_WIDTH or n % int(width):
            raise ValueError(f"{who}: width must be in 1..{N.MAX_BEAM_WIDTH} and divide {n}, got {width!r}")
        width = int(width)
        if key is not None and self.env_id_base % width:
            raise ValueError(f"{who}: env_id_base {self.env_id_base} must be a multiple of width {width}")
        x, ld = self._logits_arg(logits.detach() if isinstance(logits, torch.Tensor) else logits, who)
        if parent_out is None:
            parent_out = torch.empty(n, dtype=torch.int32, device=self.device)
        if action_out is None:
            action_out = torch.empty(n, dtype=torch.int32, device=self.device)
        bufs = (("score", score, torch.float32),) + ((("key", key, torch.float32),) if key is not None else ()) + (
            ("parent_out", parent_out, torch.int32), ("action_out", action_out, torch.int32))
        for name, t, dt in bufs:
            if (not isinstance(t, torch.Tensor) or t.dtype != dt or tuple(t.shape) != (n,) or not t.is_contiguous()
                    or t.device != x.device):
                raise ValueError(f"{who}: {name} must be a contiguous {dt} tensor of shape ({n},) on {x.device}")
        bad = torch.empty(n // width, dtype=torch.int32, device=self.device)
        self._state_epoch += 1
        if key is None:
            rc = self._L.jss_beam_step(self._h, x.data_ptr(), int(ld), width, score.data_ptr(), parent_out.data_ptr(),
                                       action_out.data_ptr(), bad.data_ptr(), self._stream())
        else:
            rc = self._L.jss_stochastic_beam_step(self._h, x.data_ptr(), int(ld), width, self.seed, step_index,
                                                  score.data_ptr(), key.data_ptr(), parent_out.data_ptr(),
                                                  action_out.data_ptr(), bad.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_" + who)
        return parent_out, action_out, bad

    def sample_without_replacement(self, logits, k: int, order: bool = False):
        """Draw `k` distinct episodes per env without replacement from the logit table `logits` by stochastic beam
        search (Kool et al., 2019), each from the env's current state, in one launch per lane class
        (jss_sample_without_replacement), leaving the envs untouched.  The distribution is the one
        rollout_priority_sample() draws from; the search is beam_search()'s with each candidate's score perturbed by
        top-down Gumbel noise and the beams ranked by that perturbed log-probability (the key).  `logits` is taken as by
        rollout_priority_sample(); 1 <= k <= MAX_BEAM_WIDTH.  The RNG counter advances by J*M (the batch maxima).
        Returns a dict of device tensors: ``"makespan"`` (N, k) int32, ``"log_prob"`` (N, k) float32 (bit for bit the
        log_prob rollout_priority_sample() reports for the same episode) and ``"key"`` (N, k) float32, key descending
        (-1 / -inf / -inf for a slot without a complete beam, -1 / NaN / NaN in every slot of an env whose every beam
        met a bad entry, -1 / 0 / 0 for an env done now); ``"best"`` (N,) int64, the lowest slot of smallest makespan,
        -1 if none; with `order`, ``"order"`` (N, k, J, M) int32, every slot's allocation round of each operation in
        beam_search()'s format (-1 for operations started before the call, and everywhere in a slot without a complete
        beam).  When `logits` requires grad (and grad mode is on), log_prob is differentiable with respect to it: the
        backward replays the slots' orders (order_log_prob()) from the envs' state, so it raises RuntimeError after a
        call that may change that state, as sample_episodes()' does.  With k + 1 draws, ``key[:, k]`` is the threshold
        of the priority-sampling estimator (INTEGRATION.md)."""
        import torch
        x = self._table_arg(logits, "sample_without_replacement", "logits")
        if not 1 <= int(k) <= N.MAX_BEAM_WIDTH:
            raise ValueError(f"sample_without_replacement: k must be in 1..{N.MAX_BEAM_WIDTH}, got {k!r}")
        k, step_index = int(k), self._step_index
        grad = x.requires_grad and torch.is_grad_enabled()
        run = functools.partial(self._sample_without_replacement, k=k, step_index=step_index, order=order or grad)
        if grad:
            log_prob, makespan, key, ord_ = _order_log_prob_fn().apply(x, self, run, "sample_without_replacement")
        else:
            log_prob, makespan, key, ord_ = run(x)
        self._step_index += self.jobs * self.machines
        out = {"makespan": makespan, "log_prob": log_prob, "key": key, "best": _best_slot(makespan)}
        if order:
            out["order"] = ord_
        return out

    def _sample_without_replacement(self, x, k: int, step_index: int, order: bool):
        """The native call of sample_without_replacement on a checked table `x` at RNG counter `step_index`:
        (log_prob, makespan, key, order), order None unless asked for."""
        import torch
        v = self._table_view(x)
        n = self.num_envs
        makespan = torch.empty((n, k), dtype=torch.int32, device=self.device)
        log_prob = torch.empty((n, k), dtype=torch.float32, device=self.device)
        key = torch.empty((n, k), dtype=torch.float32, device=self.device)
        ord_ = (torch.full((n, k, self.jobs, self.machines), -1, dtype=torch.int32, device=self.device)
                if order else None)
        rc = self._L.jss_sample_without_replacement(self._h, *_table_args(v), self.seed, step_index, k,
                                                    makespan.data_ptr(), log_prob.data_ptr(), key.data_ptr(), k,
                                                    _ptr(ord_), self._stream())
        N.check(self._h, rc, "jss_sample_without_replacement")
        return log_prob, makespan, key, ord_

    def order_log_prob(self, logits, order, entropy: bool = False):
        """The log-likelihood under the logit table `logits` of given operation orders, each from the env's current
        state, in one launch per lane class (jss_order_log_prob), leaving the envs untouched.  `order` is (N, J, M) or
        (N, k, J, M) integer: order s of env i stands for the episode rollout_priority(-order[i, s]) runs from this
        state (the orders of beam_search() and sample_without_replacement() replay their beams).  `logits` is taken as
        by rollout_priority_sample().  Returns ``(log_prob, makespan)``, each (N,) or (N, k): log_prob float32, the sum
        of the decisions' log-probabilities computed as rollout_priority_sample() computes them (forced no-ops add 0;
        NaN where a decision meets a bad entry; 0 for an env done now), makespan int32, the end time (-1 unless the
        episode ends done).  When `logits` requires grad (and grad mode is on), log_prob is differentiable with respect
        to it (jss_order_log_prob_grad): the backward replays the orders from the envs' state, so it raises
        RuntimeError after a call that may change that state, as sample_episodes()' does.
        With `entropy`, returns ``(log_prob, makespan, entropy)``: entropy float32 like log_prob, the sum over the
        episode's decisions of the policy's entropy, bit for bit what rollout_priority_sample(entropy=True) reports for
        an episode drawing the same jobs from this state (0 for an env done now, NaN where log_prob is NaN); with a
        table that requires grad both log_prob and entropy are differentiable, through one replay."""
        import torch
        x = self._table_arg(logits, "order_log_prob", "logits")
        o, single = self._orders_arg(order, "order_log_prob")
        if entropy:
            run = functools.partial(self._order_log_prob, order=o, entropy=True)
            if x.requires_grad and torch.is_grad_enabled():
                log_prob, ent, makespan, _ = _order_log_prob_fn().apply(x, self, run, "order_log_prob", True)
            else:
                log_prob, ent, makespan, _ = run(x)
            return (log_prob[:, 0], makespan[:, 0], ent[:, 0]) if single else (log_prob, makespan, ent)
        run = functools.partial(self._order_log_prob, order=o)
        if x.requires_grad and torch.is_grad_enabled():
            log_prob, makespan, _ = _order_log_prob_fn().apply(x, self, run, "order_log_prob")
        else:
            log_prob, makespan, _ = run(x)
        return (log_prob[:, 0], makespan[:, 0]) if single else (log_prob, makespan)

    def improve_orders(self, order, max_moves: Optional[int] = None):
        """Improve given operation orders by steepest descent on the critical path, each from the env's current state,
        in one launch per lane class (jss_improve_orders), leaving the envs untouched.  `order` is (N, J, M) or
        (N, k, J, M) integer, as order_log_prob() takes it: order s of env i stands for the episode
        rollout_priority(-order[i, s]) runs from this state (the orders of beam_search() and
        sample_without_replacement() replay their beams).  Each order is first replaced by its canonical form, the
        round at which its replay allocates each operation; then each move replays every swap of two adjacent
        operations of a machine block on the critical path (N1 of van Laarhoven, Aarts and Lenstra, 1992) and takes
        the one of smallest makespan (the first on the path from its end on ties) if it is strictly better, until none
        is or after `max_moves` moves (None: no limit).  Neighbours are valued by this env's own replay, so every
        returned order is an episode of it.  No RNG, no table.  Returns a dict of device tensors, shaped like the input
        without (J, M): ``"makespan"`` and ``"start_makespan"`` int32, the final and the input's makespan,
        ``"moves"`` int32, the accepted moves, and ``"order"`` int32 like the input, the final canonical order (-1 /
        -1 / 0 and -1 everywhere for an env done now or an input whose replay does not end done); for (N, k, J, M)
        input also ``"best"`` (N,) int64, the lowest s of smallest makespan, -1 if none.  The improved order is an
        imitation target: ``order_log_prob(logits, out["order"])`` is its differentiable log-likelihood."""
        import torch
        n = self.num_envs
        o, single = self._orders_arg(order, "improve_orders")
        if max_moves is None:
            max_moves = 2 ** 31 - 1
        elif isinstance(max_moves, bool) or not isinstance(max_moves, (int, np.integer)) or not 0 <= max_moves < 2 ** 31:
            raise ValueError(f"improve_orders: max_moves must be None or an integer in [0, 2^31), got {max_moves!r}")
        k = o.shape[1]
        out = {"order": torch.full_like(o, -1)}
        for name in ("makespan", "start_makespan", "moves"):
            out[name] = torch.empty((n, k), dtype=torch.int32, device=self.device)
        rc = self._L.jss_improve_orders(self._h, o.data_ptr(), k, int(max_moves), out["order"].data_ptr(),
                                        out["makespan"].data_ptr(), out["start_makespan"].data_ptr(),
                                        out["moves"].data_ptr(), k, self._stream())
        N.check(self._h, rc, "jss_improve_orders")
        if single:
            return {name: t[:, 0] for name, t in out.items()}
        out["best"] = _best_slot(out["makespan"])
        return out

    def _order_log_prob(self, x, order, entropy: bool = False):
        """The native call of order_log_prob on a checked table `x` and (N, k, J, M) contiguous int32 orders:
        (log_prob, makespan, order), with `entropy` (log_prob, entropy, makespan, order)."""
        import torch
        v = self._table_view(x)
        k = order.shape[1]
        makespan = torch.empty((self.num_envs, k), dtype=torch.int32, device=self.device)
        log_prob = torch.empty((self.num_envs, k), dtype=torch.float32, device=self.device)
        if entropy:
            ent = torch.empty((self.num_envs, k), dtype=torch.float32, device=self.device)
            rc = self._L.jss_order_log_prob_entropy(self._h, *_table_args(v), order.data_ptr(), k, makespan.data_ptr(),
                                                    log_prob.data_ptr(), ent.data_ptr(), k, self._stream())
            N.check(self._h, rc, "jss_order_log_prob_entropy")
            return log_prob, ent, makespan, order
        rc = self._L.jss_order_log_prob(self._h, *_table_args(v), order.data_ptr(), k, makespan.data_ptr(),
                                        log_prob.data_ptr(), k, self._stream())
        N.check(self._h, rc, "jss_order_log_prob")
        return log_prob, makespan, order

    def _order_log_prob_grad(self, x, order, weights, split: int, entropy_weights=None):
        """The native backward of order_log_prob: the (split, N, J, M) float32 chunks of sum_s weights[:, s] *
        d log_prob[:, s] / d table for the (N, k, J, M) int32 orders, replayed from the current state; with
        `entropy_weights`, plus entropy_weights[:, s] * d entropy[:, s] / d table, in the same replay."""
        import torch
        v = self._table_view(x)
        k = order.shape[1]
        w = weights.detach().to(torch.float32).contiguous()
        grad = torch.zeros((split, self.num_envs, self.jobs, self.machines), dtype=torch.float32, device=self.device)
        if entropy_weights is not None:
            u = entropy_weights.detach().to(torch.float32).contiguous()
            rc = self._L.jss_order_log_prob_entropy_grad(self._h, *_table_args(v), order.data_ptr(), k, w.data_ptr(),
                                                         u.data_ptr(), k, int(split), grad.data_ptr(), self._stream())
            N.check(self._h, rc, "jss_order_log_prob_entropy_grad")
            return grad
        rc = self._L.jss_order_log_prob_grad(self._h, *_table_args(v), order.data_ptr(), k, w.data_ptr(), k, int(split),
                                             grad.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_order_log_prob_grad")
        return grad

    def _sample_episodes(self, x, k: int, step_index: int, entropy: bool = False):
        """The native call of sample_episodes on a checked table `x` at RNG counter `step_index`: (makespan, log_prob),
        each (N, k); with `entropy` (makespan, log_prob, entropy)."""
        import torch
        v = self._table_view(x)
        makespan = torch.empty((self.num_envs, k), dtype=torch.int32, device=self.device)
        log_prob = torch.empty((self.num_envs, k), dtype=torch.float32, device=self.device)
        if entropy:
            ent = torch.empty((self.num_envs, k), dtype=torch.float32, device=self.device)
            rc = self._L.jss_sample_episodes_entropy(self._h, *_table_args(v), self.seed, step_index, k,
                                                     makespan.data_ptr(), log_prob.data_ptr(), ent.data_ptr(), k,
                                                     self._stream())
            N.check(self._h, rc, "jss_sample_episodes_entropy")
            return makespan, log_prob, ent
        rc = self._L.jss_sample_episodes(self._h, *_table_args(v), self.seed, step_index, k, makespan.data_ptr(),
                                         log_prob.data_ptr(), k, self._stream())
        N.check(self._h, rc, "jss_sample_episodes")
        return makespan, log_prob

    def _sample_episodes_grad(self, x, k: int, step_index: int, weights, split: int, entropy_weights=None):
        """The native backward of sample_episodes: the (split, N, J, M) float32 chunks of sum_s weights[:, s] *
        d log_prob[:, s] / d table, replayed from the current state at RNG counter `step_index`; with
        `entropy_weights`, plus entropy_weights[:, s] * d entropy[:, s] / d table, in the same replay."""
        import torch
        v = self._table_view(x)
        w = weights.detach().to(torch.float32).contiguous()
        grad = torch.zeros((split, self.num_envs, self.jobs, self.machines), dtype=torch.float32, device=self.device)
        if entropy_weights is not None:
            u = entropy_weights.detach().to(torch.float32).contiguous()
            rc = self._L.jss_sample_episodes_entropy_grad(self._h, *_table_args(v), self.seed, step_index, k,
                                                          w.data_ptr(), u.data_ptr(), k, int(split), grad.data_ptr(),
                                                          self._stream())
            N.check(self._h, rc, "jss_sample_episodes_entropy_grad")
            return grad
        rc = self._L.jss_sample_episodes_grad(self._h, *_table_args(v), self.seed, step_index, k, w.data_ptr(), k,
                                              int(split), grad.data_ptr(), self._stream())
        N.check(self._h, rc, "jss_sample_episodes_grad")
        return grad

    def _warp_slots(self):
        """Resident warps of the env's device (1 for a backend that does not say: one gradient chunk)."""
        slots = getattr(N.backend, "warp_slots", None)
        return slots(self.device_index) if slots is not None else 1

    def _table_arg(self, x, who: str, what: str):
        """A caller's priority / logit table as a tensor on the env's device, refused unless it is 3-D and broadcasts
        to (N, J, M), J and M the batch maxima."""
        import torch
        n, J, M = self.num_envs, self.jobs, self.machines
        x = torch.as_tensor(x, device=self.device)
        if x.dim() != 3 or any(s not in (1, t) for s, t in zip(x.shape, (n, J, M))):
            raise ValueError(f"{who}: {what} must be 3-D and broadcast to ({n}, {J}, {M}), got {tuple(x.shape)}")
        return x

    def _table_view(self, x):
        """The (N, J, M) float32 view the kernels read of a checked table: detached, converted only if needed, and
        expanded so that broadcast dimensions get stride 0 (the strides are passed through)."""
        import torch
        v = x.detach()
        if v.dtype != torch.float32:
            v = v.to(torch.float32)
        return v.expand(self.num_envs, self.jobs, self.machines)

    def _orders_arg(self, order, who: str):
        """Operation orders, (N, J, M) or (N, k, J, M) integer, as an (N, k, J, M) contiguous int32 tensor on the env's
        device, and whether they came without the k dimension."""
        import torch
        n, J, M = self.num_envs, self.jobs, self.machines
        o = torch.as_tensor(order, device=self.device)
        if (o.dim() not in (3, 4) or o.shape[0] != n or tuple(o.shape[-2:]) != (J, M) or o.is_floating_point()
                or o.is_complex() or o.dtype == torch.bool or (o.dim() == 4 and o.shape[1] < 1)):
            raise ValueError(f"{who}: order must be an integer tensor of shape ({n}, {J}, {M}) or "
                             f"({n}, k, {J}, {M}), got {tuple(o.shape)} {o.dtype}")
        return o.reshape(n, -1, J, M).to(torch.int32).contiguous(), o.dim() == 3

    def _values_out(self, out, who: str):
        """The (N, >= J+1) contiguous int32 device table a lookahead writes: `out` once checked, else a fresh (N, J+1)
        one filled with -1."""
        import torch
        n, J = self.num_envs, self.jobs
        if out is None:
            return torch.full((n, J + 1), -1, dtype=torch.int32, device=self.device)
        if (not isinstance(out, torch.Tensor) or out.dtype != torch.int32 or out.dim() != 2 or out.shape[0] != n
                or out.shape[1] < J + 1 or not out.is_contiguous() or out.device != self.device):
            raise ValueError(f"{who}: out must be a contiguous int32 tensor of shape ({n}, >= {J + 1}) on the "
                             f"env's device")
        return out

    def rollout_record(self, rule: Union[str, int], n_steps: int, out: Optional[Dict[str, Any]] = None):
        """n_steps x (policy -> step) fused on device WITH the trajectory recorded (jss_rollout_traj): returns
        {"real_obs": (K, N, J, 7) f32, "action_mask": (K, N, J+1) bool, "reward": (K, N) f32, "done": (K, N) bool,
        "actions": (K, N) i32, ...} as device tensors; pass the dict back as `out` to reuse the buffers."""
        import torch
        r = _rule_id(rule)
        K, n, J, ms = int(n_steps), self.num_envs, self.jobs, int(self._b.mask_stride)
        if out is None or out["_obs"].shape[0] != K:
            dev = self.device
            # zero-filled once: rows of envs with fewer jobs than the batch maximum are only written up to J_i
            out = {"_obs": torch.zeros((K, n, J, 7), dtype=torch.float32, device=dev),
                   "_mask": torch.zeros((K, n, ms), dtype=torch.uint8, device=dev),
                   "_scalars": torch.zeros((K, n, 4), dtype=torch.int32, device=dev),
                   "actions": torch.zeros((K, n), dtype=torch.int32, device=dev)}
            out["real_obs"] = out["_obs"]
            out["action_mask"] = out["_mask"][:, :, : J + 1].view(torch.bool)
            out["reward"] = out["_scalars"][:, :, 0].view(torch.float32)
            out["reward_raw"] = out["_scalars"][:, :, 1]
            out["time"] = out["_scalars"][:, :, 2]
        self._state_epoch += 1
        rc = self._L.jss_rollout_traj(self._h, r, self.seed, self._step_index, K, _ptr(out["_obs"]), _ptr(out["_mask"]),
                                      _ptr(out["_scalars"]), _ptr(out["actions"]), self._stream())
        N.check(self._h, rc, "jss_rollout_traj")
        self._step_index += K
        out["done"] = (out["_scalars"][:, :, 3] & 1).bool()       # lazily evaluated view of the done bit
        return out

    # ---------------------------------------------------------------- host-buffer form
    def step_host(self, actions: np.ndarray, want_obs: bool = True):
        """step() with HOST buffers: H2D of the actions and D2H of the results inside the call."""
        a = np.ascontiguousarray(actions, dtype=np.int32)
        n, J = self.num_envs, self.jobs
        if not hasattr(self, "_host"):
            import torch
            self._host = {"mask": _host_buffer((n, int(self._b.mask_stride)), torch.uint8),
                          "obs": _host_buffer((n, J, 7), torch.float32), "scalars": _host_buffer((n, 4), torch.int32)}
            sc = self._host["scalars"].numpy()
            self._host_views = {
                "mask": self._host["mask"].numpy()[:, : J + 1].view(np.bool_), "obs": self._host["obs"].numpy(),
                "reward": sc.view(np.float32)[:, 0], "done": sc.view(np.uint8)[:, 12].view(np.bool_)}
        hb, hv = self._host, self._host_views
        self._state_epoch += 1
        rc = self._L.jss_step_host(self._h, ctypes.c_void_p(a.ctypes.data), _ptr(hb["mask"]),
                                   _ptr(hb["obs"]) if want_obs else None, _ptr(hb["scalars"]), self._stream())
        N.check(self._h, rc, "jss_step_host")
        obs = {"real_obs": hv["obs"], "action_mask": hv["mask"]}
        return obs, hv["reward"], hv["done"], np.zeros(n, np.bool_), {}

    # pipelined form: begin -> wait_mask -> (choose next actions) -> begin ... ; obs lands in alternating buffers
    def host_step_begin(self, actions: np.ndarray, packed: bool = False, dma_fraction: float = 0.0):
        """Enqueue one host-buffer step and return immediately (see jss_host_step_begin).  Results land
        in this call's slot of two alternating pinned buffer sets; use host_wait_mask()/host_wait_obs().
        packed=True ships the observation as 10-byte integer records per job instead of 28 bytes of fp32
        (jss_host_step_begin_packed); host_wait_obs() then expands them to the exact float observation.
        dma_fraction > 0 (with packed): that share of the envs ships final fp32 rows by DMA instead, so PCIe and the
        host cores each work on their part in parallel (jss_host_step_begin_hybrid).  The step is ordered after the work
        on the current stream, and every later call of this env, on any stream, after the step and its transfers."""
        a = np.ascontiguousarray(actions, dtype=np.int32)
        n, J = self.num_envs, self.jobs
        if not hasattr(self, "_pipe"):
            import torch
            ms = int(self._b.mask_stride)
            ws = int(self._L.jss_host_wire_stride(self._h))
            self._pipe = [{"mask": _host_buffer((n, ms), torch.uint8), "obs": None, "wire": None, "wire_stride": ws,
                           "n_dma": 0, "scalars": _host_buffer((n, 4), torch.int32),
                           "actions": _host_buffer((n,), torch.int32), "packed": False, "expanded": True}
                          for _ in range(2)]
            self._pipe_slot = 0
            self._pipe_inflight = 0
        if self._pipe_inflight >= 2:
            # the slot about to be reused belongs to the begin before the latest one: its transfers must have drained
            N.check(self._h, self._L.jss_host_wait(self._h, N.WAIT_OBS_PREV), "jss_host_wait")
        self._pipe_slot ^= 1
        b = self._pipe[self._pipe_slot]
        if b["obs"] is None:
            import torch
            # fp32 observation buffer: DMA target (pinned) in plain mode, expansion target in packed mode
            b["obs"] = _host_buffer((n, J, 7), torch.float32)
        if packed and b["wire"] is None:
            import torch
            b["wire"] = _host_buffer((n, b["wire_stride"]), torch.uint8)
        b["actions"].numpy()[:] = a                      # pinned copy: the H2D must not race with the caller's array
        b["packed"] = bool(packed)
        b["expanded"] = not packed
        b["n_dma"] = 0
        self._state_epoch += 1
        if packed and dma_fraction > 0.0:
            g = 256 if n >= 4096 else 1
            b["n_dma"] = min(n, int(dma_fraction * n) // g * g)
        if packed and b["n_dma"] > 0:
            rc = self._L.jss_host_step_begin_hybrid(self._h, _ptr(b["actions"]), _ptr(b["mask"]), _ptr(b["wire"]),
                                                    _ptr(b["obs"]), b["n_dma"], _ptr(b["scalars"]), self._stream())
        elif packed:
            rc = self._L.jss_host_step_begin_packed(self._h, _ptr(b["actions"]), _ptr(b["mask"]), _ptr(b["wire"]),
                                                    _ptr(b["scalars"]), self._stream())
        else:
            rc = self._L.jss_host_step_begin(self._h, _ptr(b["actions"]), _ptr(b["mask"]), _ptr(b["obs"]),
                                             _ptr(b["scalars"]), self._stream())
        N.check(self._h, rc, "jss_host_step_begin")
        self._pipe_inflight = min(2, self._pipe_inflight + 1)
        return self._pipe_slot

    def host_wait_mask(self):
        """Block until mask / reward / done of the latest host_step_begin have landed; returns them."""
        N.check(self._h, self._L.jss_host_wait(self._h, N.WAIT_MASK), "jss_host_wait")
        b = self._pipe[self._pipe_slot]
        sc = b["scalars"].numpy()
        return (b["mask"].numpy()[:, : self.jobs + 1].view(np.bool_), sc.view(np.float32)[:, 0],
                sc.view(np.uint8)[:, 12].view(np.bool_))

    def host_wait_obs(self, previous: bool = False):
        """Block until the observation of the latest host_step_begin (or, with previous=True, of the one
        before it, which may be consumed while the latest is still streaming) has landed; returns (N, J, 7)
        float32.  In packed mode the integer rows are expanded here (multi-threaded host helper)."""
        N.check(self._h, self._L.jss_host_wait(self._h, N.WAIT_OBS_PREV if previous else N.WAIT_OBS), "jss_host_wait")
        b = self._pipe[self._pipe_slot ^ (1 if previous else 0)]
        if b["packed"] and not b["expanded"]:
            rc = self._L.jss_host_expand_obs_range(self._h, _ptr(b["wire"]), _ptr(b["scalars"]), _ptr(b["obs"]),
                                                   int(b["n_dma"]), self.num_envs)
            N.check(self._h, rc, "jss_host_expand_obs")
            b["expanded"] = True
        return b["obs"].numpy()

    @staticmethod
    def host_configure(threads: int = 0, bind_numa_of_device: int = -1) -> int:
        """Size / bind the host worker pool (jss_host_configure); call before the first host helper runs."""
        return int(N.backend.library().jss_host_configure(int(threads), int(bind_numa_of_device)))

    @staticmethod
    def host_set_simd(level: int) -> int:
        """Cap the SIMD level of the packed-observation expansion: 0 scalar, 1 AVX2, 2 AVX-512 (the default: best
        available).  The three paths give identical results; this lets tests exercise each one."""
        return int(N.backend.library().jss_host_set_simd(int(level)))

    def host_masked_random(self, mask: np.ndarray, step_index: int) -> np.ndarray:
        """Same draw as policy('RANDOM') but from a host mask (for host-side agents / tests)."""
        m = np.asarray(mask)
        if m.dtype != np.uint8:
            m = m.view(np.uint8) if m.dtype == np.bool_ else m.astype(np.uint8)
        if m.strides[1] != 1:
            m = np.ascontiguousarray(m)
        out = np.empty(m.shape[0], np.int32)
        rc = self._L.jss_host_masked_random(ctypes.c_void_p(m.ctypes.data), m.shape[0], m.shape[1], m.strides[0], self.seed,
                                            self.env_id_base, int(step_index), ctypes.c_void_p(out.ctypes.data))
        if rc != 0:
            raise N.NativeError("jss_host_masked_random failed")
        return out

    # ---------------------------------------------------------------- statistics / state
    def stats(self) -> Dict[str, int]:
        out = np.zeros(len(N.STATS_KEYS), np.int64)
        rc = self._L.jss_stats(self._h, out.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), self._stream())
        N.check(self._h, rc, "jss_stats")
        return dict(zip(N.STATS_KEYS, (int(v) for v in out)))

    def export_state(self) -> Dict[str, Any]:
        """Canonical per-env integer state as device tensors (snapshot); see jss_b200.h."""
        N.check(self._h, self._L.jss_export_state(self._h, self._stream()), "jss_export_state")
        return {**self._x, "t": self.current_time_step, "flags": self._flags_done}

    def import_state(self, state: Dict[str, Any], mask=None):
        """Restore a snapshot taken with export_state() (tensors are copied into the library's buffers)."""
        self._state_epoch += 1
        if getattr(self, "_pipe_inflight", 0):
            # the copies below are torch ops, which the library cannot order after a host_step_begin still writing
            # the time and flags; its own entry points can
            N.check(self._h, self._L.jss_host_wait(self._h, N.WAIT_OBS), "jss_host_wait")
        for k, dst in {**self._x, "t": self.current_time_step, "flags": self._flags_done}.items():
            if state[k].data_ptr() != dst.data_ptr():
                dst.copy_(state[k])
        m = self._env_mask(mask)
        N.check(self._h, self._L.jss_import_state(self._h, _ptr(m), self._stream()), "jss_import_state")

    @property
    def launch_count(self) -> int:
        return int(self._L.jss_launch_count(self._h))

    def synchronize(self):
        N.backend.synchronize(self.device_index)
