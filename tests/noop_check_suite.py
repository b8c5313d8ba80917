"""The no-op check (env_check_no_op, the reference's _check_no_op at JSSEnv/envs/jss_env.py:256-401) on states built
with import_state, for every lane class (1, 2, 4 and 8 jobs per lane).

The kernel takes every legal job at once and combines them per machine; the reference walks them in ascending job
order and keeps running per-machine minima.  The states here are built around what makes the two agree: several
legal jobs on one machine in decreasing and in increasing duration order (so the lowest-index job's end, which sets
max_horizon, differs from the machine's minimum), exactly 3 legal machines with 4 legal jobs, a legal job that ends
exactly at the next event, and blocked, running, waiting and last-operation jobs around them.  Each env is imported,
stepped by allocating one extra legal job (the check then runs on the designed state with that job running), and then
stepped at random; after every step the mask's no-op byte must equal `reference_no_op` on the exported state."""
import numpy as np
import torch

from tests.backends import native_test
from tests.parity_common import batch_cfg, np_

# job status in a design
LEGAL, BLOCKED, WAITING, RUNNING, DONE = range(5)


def reference_no_op(machine, duration, t, todo, tufco, tuam, legal, blocked, max_time_op):
    """jss_env.py:256-401 on one exported state, in the reference's order."""
    J, M = machine.shape
    lj = [j for j in range(J) if legal[j]]
    machine_legal = {int(machine[j, todo[j]]) for j in lj}
    pending = [int(x) for x in tuam if x > 0]
    if not pending or len(machine_legal) > 3 or len(lj) > 4:
        return False
    next_event = t + min(pending)
    max_horizon = t
    mhm = [t + max_time_op] * M
    for j in lj:
        m, end = int(machine[j, todo[j]]), t + int(duration[j, todo[j]])
        if end < next_event:
            return False
        mhm[m] = min(mhm[m], end)
        max_horizon = max(max_horizon, mhm[m])
    machine_next = set()
    for j in range(J):
        if legal[j]:
            continue
        if tufco[j] > 0 and todo[j] + 1 < M:
            ts, tn = int(todo[j]) + 1, t + int(tufco[j])
        elif not blocked[j] and todo[j] < M:
            ts = int(todo[j])
            tn = t + int(tuam[machine[j, ts]])
        else:
            continue
        while ts < M - 1 and max_horizon > tn:
            m = int(machine[j, ts])
            if mhm[m] > tn and m in machine_legal:
                machine_next.add(m)
                if len(machine_next) == len(machine_legal):
                    return True
            tn += int(duration[j, ts])
            ts += 1
    return False


def design_env(J, M, rng, kind):
    """A (machine, duration) instance, an exported-state row and the trigger job for one env.

    The designed jobs sit at random job indices; the remaining jobs are running, waiting, blocked or done at random.
    The trigger job is legal on a machine no designed legal job needs, so allocating it leaves the design as it is."""
    machine = rng.integers(0, M, size=(J, M))
    duration = rng.integers(1, 60, size=(J, M))
    todo = rng.integers(0, M, size=J)
    status = rng.choice([RUNNING, WAITING, BLOCKED, DONE], size=J, p=[0.3, 0.3, 0.2, 0.2])
    t = int(rng.integers(50, 500))
    jobs = rng.permutation(J)
    m_legal = [int(x) for x in rng.permutation(M)[:3]]
    # (job slot in `jobs`, machine, duration) of the designed legal jobs, in ascending job order once sorted
    if kind == "decreasing":          # one machine, durations falling with the job index: first end > minimum
        legal = [(m_legal[0], d) for d in (50, 30, 20)]
    elif kind == "increasing":        # one machine, durations rising: first end == minimum
        legal = [(m_legal[0], d) for d in (20, 30, 50)]
    elif kind == "three_four":        # exactly 3 legal machines and 4 legal jobs
        legal = [(m_legal[0], 40), (m_legal[1], 25), (m_legal[0], 15), (m_legal[2], 35)]
    elif kind == "end_at_event":      # a legal job ends exactly at the next event
        legal = [(m_legal[0], 12), (m_legal[1], 40)]
    else:                             # random: 1..4 legal jobs on 1..3 machines
        k = int(rng.integers(1, 5))
        legal = [(m_legal[int(rng.integers(0, 3))], int(rng.integers(1, 60))) for _ in range(k)]
    if kind in ("decreasing", "increasing"):
        idx = np.sort(jobs[:len(legal)])  # durations follow the job order
    else:
        idx = jobs[:len(legal)]
    trig = int(jobs[len(legal)])
    free = [m for m in range(M) if m not in m_legal]
    m_trig = free[int(rng.integers(0, len(free)))]
    for j, (m, d) in zip(idx, legal):
        status[j] = LEGAL
        todo[j] = min(todo[j], M - 1)
        machine[j, todo[j]], duration[j, todo[j]] = m, d
    status[trig] = LEGAL
    todo[trig] = min(todo[trig], M - 2)
    machine[trig, todo[trig]] = m_trig
    duration[trig, todo[trig]] = int(rng.integers(12, 80))   # its allocation adds an event after the designed first
    # no other job may be legal: every other job that is not running / done waits on a busy machine or is blocked
    busy = [m for m in range(M) if m not in m_legal and m != m_trig]
    tuam = np.zeros(M, np.int64)
    tufco = np.zeros(J, np.int64)
    for j in range(J):
        if status[j] in (LEGAL, DONE):
            if status[j] == DONE:
                todo[j] = M
            continue
        if status[j] == RUNNING and busy:
            m = busy[int(rng.integers(0, len(busy)))]
            if tuam[m] == 0:                 # one running job per machine
                todo[j] = min(todo[j], M - 1)
                machine[j, todo[j]] = m
                tufco[j] = tuam[m] = int(rng.integers(1, 80))
                continue
            status[j] = WAITING
        if status[j] == RUNNING:
            status[j] = BLOCKED
        todo[j] = min(todo[j], M - 1)
        if status[j] == WAITING and busy:
            machine[j, todo[j]] = busy[int(rng.integers(0, len(busy)))]
        else:
            status[j] = BLOCKED              # on a legal machine or a free one, kept off by a no-op
            machine[j, todo[j]] = m_legal[int(rng.integers(0, 3))]
    for m in busy:                           # every busy machine has an event; a waiting job's machine is busy
        if tuam[m] == 0:
            tuam[m] = int(rng.integers(1, 80))
    if kind != "random":                     # the first event at or before every designed legal job's end
        first = 12 if kind == "end_at_event" else min(d for _, d in legal) // 2 + 1
        tuam[busy] = np.maximum(tuam[busy], first + 1)
        tuam[busy[0]] = first
        for j in range(J):
            if tufco[j] > 0:
                tufco[j] = tuam[machine[j, todo[j]]]
    st = {"todo": todo, "tufco": tufco, "tuam": tuam, "t": t,
          "legal": (status == LEGAL).astype(np.uint8), "blocked": (status == BLOCKED).astype(np.uint8)}
    return (machine.astype(np.int32), duration.astype(np.int32)), st, trig


def run_designs(make_env, J, M, n_envs, seed, n_random_steps):
    rng = np.random.default_rng(seed)
    kinds = ["decreasing", "increasing", "three_four", "end_at_event", "random"]
    designs = [design_env(J, M, rng, kinds[i % len(kinds)]) for i in range(n_envs)]
    insts = [d[0] for d in designs]
    env = make_env(n_envs, batch_cfg(insts, sort=False), seed=seed)
    env.reset()
    x = env.export_state()
    state = {k: np_(v).copy() for k, v in x.items()}
    for i, (_, st, _) in enumerate(designs):
        for k in ("todo", "tufco", "legal", "blocked"):
            state[k][i, :J] = st[k]
        state["tuam"][i, :M] = st["tuam"]
        state["t"][i] = st["t"]
        for k in ("idle_last", "total_idle", "col4"):
            state[k][i] = 0
        state["flags"][i] = 0
    env.import_state({k: torch.as_tensor(v).to(x[k].device) for k, v in state.items()})
    actions = torch.tensor([d[2] for d in designs], dtype=torch.int32, device=x["todo"].device)
    checked = 0
    for step in range(n_random_steps + 1):
        obs, *_ = env.step(actions)
        mask = np_(obs["action_mask"])
        s = {k: np_(v) for k, v in env.export_state().items()}
        for i, ((machine, duration), _, _) in enumerate(designs):
            if s["flags"][i] & 2 << 8:       # JSS_FLAG_ERROR: the step was refused
                raise AssertionError((J, step, i, "error bit"))
            if step > 0 and not alive[i]:
                continue
            want = reference_no_op(machine, duration, int(s["t"][i]), s["todo"][i, :J], s["tufco"][i, :J],
                                   s["tuam"][i, :M], s["legal"][i, :J], s["blocked"][i, :J], int(duration.max()))
            assert bool(mask[i, J]) == want, (J, step, i, designs[i][2])
            checked += 1
        alive = ~(s["flags"] & 1).astype(bool)
        actions = env.policy("RANDOM")
    return checked


@native_test(emu=[(20, 6, 10), (50, 6, 10), (100, 8, 10), (200, 6, 10)],
             gpu=[(20, 6, 400), (50, 6, 400), (100, 8, 400), (200, 6, 400), (100, 20, 400)])
def noop_check_designed_states(make_env, J, M, n_envs):
    """Designed states of J jobs (1, 2, 4, 8 jobs per lane), then 20 random steps each."""
    assert run_designs(make_env, J, M, n_envs, seed=J * 31 + M, n_random_steps=20) >= n_envs
