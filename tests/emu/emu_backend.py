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
    srcs = [os.path.join(HERE, f) for f in ("cuda_shim.h", "emu_runtime.cpp")]
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
            self._lib = _native._declare(ctypes.CDLL(EMU_LIB))
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


class use_emulation:
    """Context manager / pytest helper: `with use_emulation(): env = JssVecEnv(...)`."""

    def __enter__(self):
        self._saved = _native.backend
        _native.backend = EmuBackend()
        return _native.backend

    def __exit__(self, *exc):
        _native.backend = self._saved
        return False
