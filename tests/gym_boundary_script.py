"""Runs in a FRESH interpreter (see tests/test_gym_boundary.py) with the TEST-ONLY gymnasium stand-in of
tests/stubs on sys.path, so that the code paths that only exist when `gymnasium` is importable execute:
the `jss-v1` registration (reference: JSSEnv/__init__.py:6-9), `gym.make('jss-v1', env_config=...)`
(README.md:46-65), the gym.Env / gym.spaces publication of the facade (jss_env.py:97, 112-119), the
`gymnasium.vector.VectorEnv` subclass path of JssGymVectorEnv and `create_env` (JSSEnv/utils.py:32-60).
usage: python tests/gym_boundary_script.py emu|gpu"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "stubs"))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402


def main(backend):
    import gymnasium as gym
    assert gym.__version__ == "0.0-stub"
    import jssenv_b200
    from jssenv_b200 import JssEnv, JssGymVectorEnv, create_env
    from jssenv_b200.instances import load_instance
    from oracle.jss_oracle import OracleEnv
    from tests.parity_common import assert_facade_obs_exact, assert_obs_exact, assert_reward_exact
    assert "jss-v1" in gym.envs.registration.registry, "import must register the reference's id"
    assert jssenv_b200.register_gymnasium() is True

    # README.md:43-65 loop through gym.make
    env = gym.make("jss-v1", env_config={"instance_path": "ta01"})
    assert isinstance(env, JssEnv) and isinstance(env, gym.Env)
    assert isinstance(env.action_space, gym.spaces.Discrete) and env.action_space.n == 16
    sp = env.observation_space
    assert isinstance(sp, gym.spaces.Dict) and sp["real_obs"].shape == (15, 7) and sp["action_mask"].shape == (16,)
    o = OracleEnv(*load_instance("ta01"))
    obs, _ = env.reset(), o.reset()
    rng = np.random.default_rng(0)
    done, total, steps = False, 0.0, 0
    while not done:
        assert sp.contains(obs), "observation outside the declared space"
        legal = np.flatnonzero(obs["action_mask"])
        a = int(rng.choice(legal))
        assert env.action_space.contains(a)
        obs, reward, done, truncated, info = env.step(a)
        oo, r2, d2, _, _ = o.step(a)
        assert reward == r2 and isinstance(reward, float), (reward, r2)      # float64 quotient, bit-equal
        assert done == d2 and truncated is False and info == {}
        assert np.array_equal(obs["action_mask"], oo["action_mask"])
        assert_facade_obs_exact(obs["real_obs"], oo["real_obs"], steps)
        total += reward; steps += 1
    assert env.current_time_step == o.current_time_step and env.last_time_step == o.current_time_step
    env.close()
    # default instance of the reference (jss_env.py:35-38) through make without kwargs
    env = gym.make("jss-v1")
    assert (env.jobs, env.machines) == (100, 20)
    env.close()

    # VectorEnv subclass path
    n = 6
    venv = JssGymVectorEnv(n, {"instance_path": "ta01"}, to_numpy=True, seed=3)
    assert isinstance(venv, gym.vector.VectorEnv)
    assert venv.metadata["autoreset_mode"] is gym.vector.AutoresetMode.NEXT_STEP
    assert venv.observation_space["real_obs"].shape == (n, 15, 7) and venv.observation_space["real_obs"].dtype == np.float32
    assert venv.observation_space["action_mask"].shape == (n, 16) and venv.observation_space["action_mask"].dtype == np.int8
    assert venv.action_space.shape == (n,) and venv.single_action_space.n == 16
    obs, info = venv.reset(seed=11)
    oracles = [OracleEnv(*load_instance("ta01")) for _ in range(n)]
    for o in oracles:
        o.reset()
    was_done = np.zeros(n, bool)
    for k in range(700):
        assert venv.observation_space.contains(obs), k
        # a terminal env has an all-zero mask; its next action is ignored (the transition is the autoreset)
        acts = np.array([rng.choice(np.flatnonzero(m)) if m.any() else 0 for m in obs["action_mask"]], np.int64)
        assert venv.action_space.contains(acts)
        obs, rew, term, trunc, info = venv.step(acts)
        assert obs["action_mask"].dtype == np.int8 and rew.dtype == np.float32 and term.dtype == np.bool_
        for i, o in enumerate(oracles):
            if was_done[i]:                                   # next-step autoreset: this transition IS the reset
                o.reset()
                assert rew[i] == 0.0 and not term[i]
                was_done[i] = False
            else:
                _, r, d, _, _ = o.step(int(acts[i]))
                assert_reward_exact(rew[i], r, (k, i))
                assert bool(term[i]) == d
                was_done[i] = d
            assert np.array_equal(obs["action_mask"][i].astype(bool), o.legal_actions)
            assert_obs_exact(obs["real_obs"][i], o.state, (k, i))
        assert not trunc.any()
    assert int(venv.vec.episode_count.min()) >= 2
    venv.close()

    # create_env (JSSEnv/utils.py:32-60)
    e1 = create_env({"env": "jss-v1", "instance_path": "ta01"})
    assert isinstance(e1, JssEnv) and e1.jobs == 15
    e1.close()
    e2 = create_env({"env": "jss-v1", "env_config": {"instance_path": "ta31"}, "num_envs": 4})
    assert isinstance(e2, JssGymVectorEnv) and e2.vec.jobs == 30
    e2.close()
    for bad in ({"env": "nope-v0"}, {"instance_path": "ta01"}):
        try:
            create_env(bad)
            raise AssertionError("create_env must reject " + repr(bad))
        except (NotImplementedError, KeyError):
            pass
    print("gym boundary ok:", backend, "episode steps", steps, "return", total)


if __name__ == "__main__":
    backend = sys.argv[1] if len(sys.argv) > 1 else "gpu"
    if backend == "emu":
        from tests.emu.emu_backend import use_emulation
        with use_emulation():
            main(backend)
    else:
        main(backend)
