"""`gym.make('jss-v1')` / gymnasium.vector.VectorEnv boundary (reference: JSSEnv/__init__.py:6-9, README.md:46).

gymnasium is installed neither in the build image nor on the GPU box, so the code paths guarded by
`import gymnasium` are executed in a fresh interpreter that has the TEST-ONLY stand-in package of
tests/stubs on its path (tests/gym_boundary_script.py), once per backend of tests/backends.py."""
import os
import subprocess
import sys

from tests.backends import collect, native_test

HERE = os.path.dirname(os.path.abspath(__file__))


@native_test(names={"emu": "test_gym_boundary_emulated"})
def gym_boundary(backend):
    r = subprocess.run([sys.executable, os.path.join(HERE, "gym_boundary_script.py"), backend],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "gym boundary ok" in r.stdout


def test_registration_is_optional():
    """Without gymnasium the package still imports and reports that nothing was registered."""
    import jssenv_b200
    try:
        import gymnasium  # noqa: F401
        have = True
    except Exception:
        have = False
    assert jssenv_b200.register_gymnasium() is have


collect(globals(), globals(), "emu", "gpu")
