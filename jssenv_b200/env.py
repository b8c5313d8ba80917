"""JssEnv -- single-environment facade with the reference's object interface.

Mirrors ``JSSEnv.envs.jss_env.JssEnv`` (JSSEnv/envs/jss_env.py:14-693): same ctor
(``env_config={"instance_path": ...}``, default instance ta80), ``reset() -> obs``,
``step(action) -> (obs, reward, done, False, {})``, ``get_legal_actions()``,
``increase_time_step()`` and the attribute surface that the reference's dispatching
rules and tests read (``todo_time_step_job``, ``machine_legal``, ``next_time_step``,
``solution`` ...).  It is a batch of ONE env on the GPU: every transition runs the
same sm_90a step kernel as ``JssVecEnv``; the attributes are host copies decoded
from the device state after each transition (redundant reference state such as the
event queue or ``illegal_actions[M][J]`` is re-derived, see SURVEY.md section 8 a13).
"""
from typing import Any, Dict, Optional

import numpy as np

from . import _native as N
from .instances import DEFAULT_INSTANCE
from .vec_env import JssVecEnv

try:  # optional: only used to publish gym spaces / register the id
    import gymnasium as _gym
except Exception:  # gymnasium is not installed in the build image
    _gym = None


class _Space:
    """Minimal stand-in for gym.spaces.* when gymnasium is absent."""

    def __init__(self, kind, **kw):
        self.kind = kind
        self.__dict__.update(kw)

    def __repr__(self):
        return f"{self.kind}({ {k: v for k, v in self.__dict__.items() if k != 'kind'} })"


class JssEnv(_gym.Env if _gym is not None else object):
    def __init__(self, env_config: Optional[Dict[str, Any]] = None, device: int = 0):
        if env_config is None:
            env_config = {"instance_path": DEFAULT_INSTANCE}   # jss_env.py:35-38
        # a batch of ONE env whose outputs live in a pinned, device-mapped host block (JSS_CREATE_HOST_MIRROR): a
        # transition is one kernel launch + one stream sync, and the attributes below are numpy reads of that block
        self._vec = JssVecEnv(1, {"instance_path": env_config["instance_path"]}, device=device, host_mirror=True)
        machine, duration = self._vec.instances[0]
        self.jobs, self.machines = int(machine.shape[0]), int(machine.shape[1])
        self.instance_matrix = np.stack([machine, duration], axis=-1).astype(np.int64)   # (J, M, 2), jss_env.py:78
        self._machine_of = machine.astype(np.int64)
        self.jobs_length = duration.sum(axis=1).astype(np.int64)
        self.max_time_op, self.max_time_jobs, self.sum_op = (int(v) for v in self._vec.instance_scalars[0])
        self.last_solution = None
        self.last_time_step = float("inf")
        J = self.jobs
        if _gym is not None:
            self.action_space = _gym.spaces.Discrete(J + 1)
            self.observation_space = _gym.spaces.Dict({
                "action_mask": _gym.spaces.Box(0, 1, shape=(J + 1,)),
                "real_obs": _gym.spaces.Box(low=0.0, high=1.0, shape=(J, 7), dtype=float)})
        else:
            self.action_space = _Space("Discrete", n=J + 1)
            self.observation_space = _Space("Dict", spaces={
                "action_mask": _Space("Box", low=0, high=1, shape=(J + 1,)),
                "real_obs": _Space("Box", low=0.0, high=1.0, shape=(J, 7), dtype=float)})
        self.solution = np.full((self.jobs, self.machines), -1, dtype=np.int64)       # jss_env.py:163
        self._arange = np.arange(J)
        self._vec.export_state()
        self._pull()

    # ------------------------------------------------------------------ state mirror
    def _pull(self):
        """Read the env's decoded state from the host mirror (written by the device kernels) and rebuild the reference's
        primary attributes; the redundant ones (SURVEY.md section 8 a13) are derived lazily, see __getattr__."""
        v = self._vec
        v.synchronize()
        h = v.host
        self.todo_time_step_job = h["todo"][0].astype(np.int64)
        self.time_until_finish_current_op_jobs = h["tufco"][0].astype(np.int64)
        self.time_until_available_machine = h["tuam"][0].astype(np.int64)
        self.idle_time_jobs_last_op = h["idle_last"][0].astype(np.int64)
        self.total_idle_time_jobs = h["total_idle"][0].astype(np.int64)
        self.action_illegal_no_op = h["blocked"][0].astype(bool)
        sc = h["scalars"][0]
        self.current_time_step = int(sc[2])
        self._flags = int(sc[3]) >> 8
        self._reward_raw = int(sc[1])
        legal = np.empty(self.jobs + 1, dtype=bool)
        legal[: self.jobs] = h["legal"][0]
        legal[self.jobs] = bool(self._flags & N.FLAG_NOOP_LEGAL)
        self.legal_actions = legal
        self.state = h["real_obs"][0].astype(np.float64)
        self._derived = {}

    # redundant reference state, re-derived on first access after a transition
    def _derive(self, name):
        J, M = self.jobs, self.machines
        if name == "needed_machine_jobs":
            todo = self.todo_time_step_job
            val = np.where(todo < M, self._machine_of[self._arange, np.minimum(todo, M - 1)], -1).astype(np.int64)
        elif name == "total_perform_op_time_jobs":
            # total_perform = t - total_idle until the job completes (then jobs_length)
            val = np.where(self.todo_time_step_job < M, self.current_time_step - self.total_idle_time_jobs,
                           self.jobs_length).astype(np.int64)
        elif name == "machine_legal":
            val = np.zeros(M, dtype=bool)
            val[self.needed_machine_jobs[self.legal_actions[:J]]] = True    # machine_legal == "some legal job needs it"
        elif name == "nb_machine_legal":
            val = int(self.machine_legal.sum())
        elif name == "nb_legal_actions":
            val = int(self.legal_actions[:J].sum())
        elif name == "illegal_actions":
            val = np.zeros((M, J), dtype=bool)                               # illegal_actions[m][j] == blocked[j] & needed[j]==m
            bj = np.flatnonzero(self.action_illegal_no_op)
            val[self.needed_machine_jobs[bj], bj] = True
        elif name == "next_time_step":
            # event queue == sorted set {t + tuam[m] : tuam[m] > 0} (appendix A.1)
            val = sorted({int(self.current_time_step + d) for d in self.time_until_available_machine if d > 0})
        elif name == "next_jobs":
            tufco = self.time_until_finish_current_op_jobs
            val = [int(np.flatnonzero((tufco > 0) & (self.current_time_step + tufco == e))[0]) for e in self.next_time_step]
        else:
            raise AttributeError(name)
        self._derived[name] = val
        return val

    _DERIVED = ("needed_machine_jobs", "total_perform_op_time_jobs", "machine_legal", "nb_machine_legal",
                "nb_legal_actions", "illegal_actions", "next_time_step", "next_jobs")

    def __getattr__(self, name):
        if name in JssEnv._DERIVED:
            d = self.__dict__.get("_derived")
            if d is None:
                raise AttributeError(name)
            return d[name] if name in d else self._derive(name)
        raise AttributeError(name)

    def _raise_for_error(self, message):
        """The device error bit is sticky; the facade turns it into the reference's IndexError once and
        clears it (state re-imported unchanged) so the env stays usable if the caller catches it."""
        snap = self._vec.export_state()
        snap["flags"].bitwise_and_(~((N.FLAG_ERROR) << 8))
        self._vec.import_state(snap)
        self._vec.export_state()
        self._pull()
        raise IndexError(message)

    def _get_current_state_representation(self):
        return {"real_obs": self.state, "action_mask": self.legal_actions}

    def _transition(self, action: int):
        self._vec.host["actions"][0] = action
        self._vec.step_export_host()          # one launch (step + decode) and one sync
        self._pull()

    # ------------------------------------------------------------------ reference API
    def get_legal_actions(self):
        return self.legal_actions

    def reset(self, *, seed=None, options=None):
        """Returns the observation only, like the reference (jss_env.py:145-181)."""
        self._vec.reset()
        self._vec.export_state()
        self.solution = np.full((self.jobs, self.machines), -1, dtype=np.int64)
        self._pull()
        return self._get_current_state_representation()

    def step(self, action: int):
        a = int(action)
        if not (0 <= a <= self.jobs):
            raise IndexError(f"action {a} out of range")
        t_before = self.current_time_step
        op_before = int(self.todo_time_step_job[a]) if a < self.jobs else -1
        self._transition(a)
        if self._flags & N.FLAG_ERROR:
            # the reference raises IndexError here (jss_env.py:444 / :517) or silently corrupts
            # its counters (illegal job action); the device env sets the sticky error bit
            self._raise_for_error(f"illegal action {a} for the current state")
        if a < self.jobs:
            self.solution[a][op_before] = t_before             # jss_env.py:454
        # float64 quotient like the reference's _reward_scaler (jss_env.py:483-493); the device record holds the
        # exact integer numerator next to its fp32 quotient
        reward = float(self._reward_raw) / float(self.max_time_op)
        done = bool(self._flags & N.FLAG_DONE)
        if done:                                               # jss_env.py:649-652
            self.last_time_step = self.current_time_step
            self.last_solution = self.solution
        return self._get_current_state_representation(), reward, done, False, {}

    def increase_time_step(self) -> int:
        """Raw time advance without the legal-action heuristics (jss_env.py:495-637)."""
        self._transition(N.ACTION_ADVANCE)
        if self._flags & N.FLAG_ERROR:
            self._raise_for_error("pop from empty list")      # what the reference raises (jss_env.py:517)
        return -self._reward_raw

    def set_cr_due_date_factor(self, factor: float):
        self._vec.set_cr_due_date_factor(factor)

    def rule_action(self, rule: str):
        """(action, noop_legal) chosen on device by a dispatching rule, without the 10 % coin."""
        self._vec.policy(rule, coin="never", out=self._vec._mirror_actions)   # lands in the host-mapped action slot
        self._vec.synchronize()
        return int(self._vec.host["actions"][0]), bool(self._flags & N.FLAG_NOOP_LEGAL)

    def render(self, mode: str = "human"):
        """Gantt rows of the current solution (jss_env.py:655-693 builds a plotly figure from the
        same rows; plotting itself is out of scope here)."""
        rows = []
        for job in range(self.jobs):
            for i in range(self.machines):
                if self.solution[job][i] == -1:
                    break
                rows.append({"Task": f"Job {job}", "Start": int(self.solution[job][i]),
                             "Finish": int(self.solution[job][i] + self.instance_matrix[job][i][1]),
                             "Resource": f"Machine {int(self.instance_matrix[job][i][0])}"})
        return rows or None

    def close(self):
        self._vec.close()
