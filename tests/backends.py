"""The two backends the native checks run on: `emu`, the host emulation of the kernels (tests/emu), in the CPU suite at
CPU-friendly sizes, and `gpu`, the real sm_90a library, with `-m gpu`.

A test is declared once, with `@native_test`, as a function of `make_env` (a JssVecEnv factory), `backend` and its
own parameters; `collect` binds it into a test module once per backend, as `test_<backend>_<name>`.  Each backend
keeps its own module and test ids, and a check is written, sized and parametrized in one place."""
import contextlib
import inspect

import pytest

from tests.emu.emu_backend import use_emulation


def native_test(emu=(), gpu=(), names=None):
    """Declares a test for both backends.  For each backend: a list of parameter sets for the test's own arguments,
    as for pytest.mark.parametrize; () for one test without parameters; a dict for one test with these arguments;
    None to leave the backend out.  `names` maps a backend to a test name other than `test_<backend>_<name>`."""
    def declare(fn):
        fn.native_cases = {"emu": emu, "gpu": gpu}
        fn.native_names = names or {}
        return fn
    return declare


def _bind(fn, backend, cases=None, schedule=None, suffix=""):
    cases = fn.native_cases[backend] if cases is None else cases
    sig = inspect.signature(fn)
    fixed = cases if isinstance(cases, dict) else {}
    own = [p for p in sig.parameters.values()
           if p.name not in ("make_env", "backend") and p.name not in fixed and p.default is p.empty]

    def test(**params):
        from jssenv_b200 import JssVecEnv
        given = {"make_env": JssVecEnv, "backend": backend, **fixed, **params}
        with use_emulation(schedule) if backend == "emu" else contextlib.nullcontext():
            fn(**{a: given[a] for a in sig.parameters if a in given})

    test.__name__ = test.__qualname__ = fn.native_names.get(backend, f"test_{backend}_{fn.__name__}") + suffix
    test.__doc__ = fn.__doc__
    test.__signature__ = sig.replace(parameters=own)      # pytest reads the test's parameters from here
    if isinstance(cases, list):
        test = pytest.mark.parametrize(",".join(p.name for p in own), cases)(test)
    return pytest.mark.gpu(test) if backend == "gpu" else test


def collect(namespace, source, *backends, only=None, schedule=None, suffix=""):
    """Binds every test `source` (a module or a namespace) declares into `namespace`, for each of `backends`.

    `only` binds just the declarations it names: a dict from name to the parameter sets to bind (in native_test's
    form) or None for the declared ones.  `schedule` runs the emu tests under use_emulation(schedule), and `suffix`
    is appended to the tests' names."""
    for fn in list(vars(source).values() if inspect.ismodule(source) else source.values()):
        if only is not None and getattr(fn, "__name__", None) not in only:
            continue
        for backend in backends:
            if getattr(fn, "native_cases", {}).get(backend) is not None:
                test = _bind(fn, backend, None if only is None else only[fn.__name__], schedule, suffix)
                namespace[test.__name__] = test
