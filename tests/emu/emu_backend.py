"""TEST-ONLY: swaps jssenv_b200._native.backend for the host emulation library
(tests/emu/libjss_emu.so, see README.md).  Used to exercise the Python host layer and
the kernels' logic in the GPU-less build container; never imported by the product."""
import ctypes
import os
import subprocess

from jssenv_b200 import _native

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_LIB = os.path.join(HERE, "libjss_emu.so")


def build(force=False):
    srcs = [os.path.join(HERE, f) for f in ("cuda_shim.h", "emu_runtime.cpp", "emu_selftest.cpp", "build_emu.sh")]
    csrc = os.path.join(HERE, "..", "..", "jssenv_b200", "csrc")
    srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
    srcs.append(os.path.join(HERE, "..", "..", "include", "jss_b200.h"))
    newest = max(os.path.getmtime(s) for s in srcs)
    if force or not os.path.exists(EMU_LIB) or os.path.getmtime(EMU_LIB) < newest:
        subprocess.check_call(["sh", os.path.join(HERE, "build_emu.sh")])
    return EMU_LIB


class EmuBackend:
    name = "emu"
    pin_memory = False

    def __init__(self):
        self._lib = None

    def library(self):
        if self._lib is None:
            build()
            lib = _native._declare(ctypes.CDLL(EMU_LIB))
            lib.jss_emu_set_schedule.restype = ctypes.c_int
            lib.jss_emu_set_schedule.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_int]
            self._lib = lib
        return self._lib

    def torch_device(self, index):
        import torch
        return torch.device("cpu")

    def stream(self, device_index):
        return None

    def wrap(self, ptr, shape, dtype, device_index, strides=None):
        import torch
        return torch.from_numpy(_native.host_view(ptr, shape, dtype, strides))

    def synchronize(self, device_index):
        pass


ASCENDING, DESCENDING, SHUFFLED = 0, 1, 2
DEFAULT_SCHEDULE = (ASCENDING, 0, -1)


class use_emulation:
    """Context manager / pytest helper: `with use_emulation(): env = JssVecEnv(...)`.

    `schedule=(order, seed, poison)` runs the emulated kernels under another legal schedule until the block exits (see
    README.md): order ASCENDING (the default), DESCENDING or SHUFFLED (seeded by `seed`) for the threads of a block and
    the blocks of a launch; poison -1 (the default) or a byte every block's shared memory and every cudaMalloc
    allocation start as.  The default schedule is restored on exit."""

    def __init__(self, schedule=None):
        self._schedule = schedule

    def __enter__(self):
        self._saved = _native.backend
        _native.backend = EmuBackend()
        if self._schedule is not None:
            try:
                self._set(self._schedule)
            except BaseException:
                _native.backend = self._saved
                raise
        return _native.backend

    def __exit__(self, *exc):
        if self._schedule is not None:
            self._set(DEFAULT_SCHEDULE)
        _native.backend = self._saved
        return False

    @staticmethod
    def _set(schedule):
        if _native.backend.library().jss_emu_set_schedule(*schedule) != 0:
            raise ValueError(f"bad emulation schedule {schedule!r}")
