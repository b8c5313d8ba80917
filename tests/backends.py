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


def _bind(fn, backend):
    cases = fn.native_cases[backend]
    sig = inspect.signature(fn)
    fixed = cases if isinstance(cases, dict) else {}
    own = [p for p in sig.parameters.values()
           if p.name not in ("make_env", "backend") and p.name not in fixed and p.default is p.empty]

    def test(**params):
        from jssenv_b200 import JssVecEnv
        given = {"make_env": JssVecEnv, "backend": backend, **fixed, **params}
        with use_emulation() if backend == "emu" else contextlib.nullcontext():
            fn(**{a: given[a] for a in sig.parameters if a in given})

    test.__name__ = test.__qualname__ = fn.native_names.get(backend, f"test_{backend}_{fn.__name__}")
    test.__doc__ = fn.__doc__
    test.__signature__ = sig.replace(parameters=own)      # pytest reads the test's parameters from here
    if isinstance(cases, list):
        test = pytest.mark.parametrize(",".join(p.name for p in own), cases)(test)
    return pytest.mark.gpu(test) if backend == "gpu" else test


def collect(namespace, source, *backends):
    """Binds every test `source` (a module or a namespace) declares into `namespace`, for each of `backends`."""
    for fn in list(vars(source).values() if inspect.ismodule(source) else source.values()):
        for backend in backends:
            if getattr(fn, "native_cases", {}).get(backend) is not None:
                test = _bind(fn, backend)
                namespace[test.__name__] = test
