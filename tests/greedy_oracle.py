"""Float64 restatement of the epsilon-greedy decode of ``jss_step_greedy`` (include/jss_b200.h), for the tests.

Test infrastructure only, like oracle/logits_oracle.py, whose counter hash it uses: the coin and the exploring pick
are replayed on the host from (seed, global env id, step index), the argmax is numpy's over the legal scores, and the
log-probability is computed in float64.
"""
import numpy as np

from oracle.logits_oracle import ACTION_SKIP, hash3, hash_env


def threshold(epsilon):
    """T = floor(epsilon * 2^32): an env explores iff its coin hash is below T."""
    return int(np.floor(float(epsilon) * 2.0 ** 32))


def greedy(scores, legal, done, epsilon, seed, env_id, step_index):
    """One env's decision.  scores: its row (>= J+1 values), legal: bool[J+1] (the action_mask before the step),
    done: whether the env is done.  Returns (action, log_prob, error): `error` tells whether the env gets the sticky
    error bit."""
    legal = np.asarray(legal, dtype=bool)
    J = legal.shape[0] - 1
    if done:
        return 0, 0.0, False
    if not legal[:J].any():
        return (J, 0.0, False) if legal[J] else (ACTION_SKIP, float("nan"), False)
    cand = np.flatnonzero(legal)
    x = np.asarray(scores, dtype=np.float32)[: J + 1][cand]
    if np.isnan(x).any() or np.isposinf(x).any() or np.isneginf(x).all():
        return ACTION_SKIP, float("nan"), True
    g = int(cand[np.argmax(x)])                           # first maximum: the lowest index on ties, -0.0 == +0.0
    T = threshold(epsilon)
    if T == 0:
        return g, 0.0, False
    coin, pick = (int(v) for v in hash_env(hash3(seed, env_id, step_index), np.array([0, 1], dtype=np.uint64)))
    n = len(cand)                                         # the legal actions, a legal no-op included
    a = int(cand[(pick * n) >> 32]) if coin < T else g    # jss_pick over the set bits in ascending order
    e = T * 2.0 ** -32
    return a, float(np.log((1.0 - e if a == g else 0.0) + e / n)), False
