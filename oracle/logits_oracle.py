"""Float64 restatement of the masked categorical draw of ``jss_step_logits`` (include/jss_b200.h), for the tests.

Test infrastructure only.  The uniforms come from the same counter hash as the device (jss_rng.h), so every draw can
be replayed on the host from (seed, global env id, step index, action index); the Gumbel noise, the scores, the argmax
and the log-probability are computed in float64.
"""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
ACTION_SKIP = -1


def _fold32(v):
    v = np.asarray(v, dtype=np.uint64)
    return (v & M32) ^ (((v >> np.uint64(32)) * np.uint64(0x7FEB352D)) & M32)


def _finalise(h):
    h = h ^ (h >> np.uint64(16))
    h = (h * np.uint64(0x85EBCA6B)) & M32
    h = h ^ (h >> np.uint64(13))
    h = (h * np.uint64(0xC2B2AE35)) & M32
    return h ^ (h >> np.uint64(16))


def hash_env(key, env):
    """jss_hash_env(key, env) of jss_rng.h, elementwise over `env`."""
    return _finalise(np.uint64(key) ^ ((_fold32(env) * np.uint64(0x9E3779B1) + np.uint64(0x85EBCA77)) & M32))


def hash3(seed, env, ctr):
    """jss_hash3(seed, env, ctr) of jss_rng.h."""
    key = int(_fold32(seed)) ^ ((int(_fold32(ctr)) * 0xC2B2AE3D + 0x27D4EB2F) & 0xFFFFFFFF)
    return int(hash_env(key, env))


def uniforms(seed, env_id, step_index, n):
    """u[a] = ((jss_hash_env(h_env, a) >> 8) + 0.5) * 2^-24 for a < n, h_env = jss_hash3(seed, env_id, step_index)."""
    h = hash_env(hash3(seed, env_id, step_index), np.arange(n, dtype=np.uint64))
    return ((h >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24


def gumbel(seed, env_id, step_index, n):
    return -np.log(-np.log(uniforms(seed, env_id, step_index, n)))


def draw(logits, legal, done, seed, env_id, step_index):
    """One env's draw.  logits: its row (>= J+1 values), legal: bool[J+1] (the action_mask before the step),
    done: whether the env is done.  Returns (action, log_prob, error, scores): `error` tells whether the env gets the
    sticky error bit, `scores` (float64[J+1], -inf off the candidates) are (logit - mx) + g with mx the largest legal
    logit, or None if there was no draw.  The scores are max-subtracted, as on the device: the same argmax as logit + g
    in exact arithmetic, and in floating point they keep the noise when the logits are large (1e30 + g is 1e30)."""
    legal = np.asarray(legal, dtype=bool)
    J = legal.shape[0] - 1
    if done:
        return 0, 0.0, False, None
    if not legal[:J].any():
        return (J, 0.0, False, None) if legal[J] else (ACTION_SKIP, float("nan"), False, None)
    cand = np.flatnonzero(legal)
    x = np.asarray(logits, dtype=np.float64)[: J + 1][cand]
    if np.isnan(x).any() or np.isposinf(x).any() or np.isneginf(x).all():
        return ACTION_SKIP, float("nan"), True, None
    mx = x.max()
    d = np.full(J + 1, -np.inf)
    d[cand] = x - mx
    scores = d + gumbel(seed, env_id, step_index, J + 1)
    a = int(np.argmax(scores))                            # first maximum: the lowest index on ties
    return a, float(d[a] - np.log(np.exp(d[cand]).sum())), False, scores
