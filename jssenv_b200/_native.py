"""ctypes binding of the C-ABI in include/jss_b200.h (the only native entry point).

The CUDA library ``libjss_b200.so`` is built in-tree by ``__graft_entry__.build()``
(nvcc, sm_90a).  There is no CPU implementation: if the library is missing, or no
H100 (compute capability 9.0) is present, construction fails loudly.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_int, c_int32, c_int64, c_uint8, c_uint32, c_uint64, c_void_p

import numpy as np

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libjss_b200.so")

JSS_ABI_VERSION = 3
ACTION_SKIP, ACTION_ADVANCE = -1, -2
CREATE_AUTO_RESET, CREATE_RECORD_SOLUTION, CREATE_HOST_MIRROR = 1, 2, 4
FLAG_DONE, FLAG_ERROR, FLAG_NOOP_LEGAL = 1, 2, 4
COIN_DEVICE, COIN_NEVER = 0, 1
MAX_BEAM_WIDTH = 32   # JSS_MAX_BEAM_WIDTH
WAIT_MASK, WAIT_OBS, WAIT_OBS_PREV = 1, 2, 3
RULES = {"RANDOM": 0, "SPT": 1, "FIFO": 2, "MWR": 3, "LWR": 4, "MOR": 5, "LOR": 6, "CR": 7}
STATS_KEYS = ("episodes", "steps", "sum_makespan", "min_makespan", "max_makespan", "sum_return",
              "envs_done", "envs_error")


class JssBuffers(ctypes.Structure):
    _fields_ = [
        ("n_envs", c_int32), ("jobs_max", c_int32), ("machines_max", c_int32), ("mask_stride", c_int32),
        ("action_mask", c_void_p), ("real_obs", c_void_p), ("scalar_stride", c_int32), ("host_mirror", c_int32),
        ("reward", c_void_p), ("reward_raw", c_void_p),
        ("done", c_void_p), ("time", c_void_p), ("flags_done", c_void_p), ("solution", c_void_p),
        ("episode_count", c_void_p), ("last_makespan", c_void_p), ("last_return", c_void_p),
        ("x_todo", c_void_p), ("x_tufco", c_void_p), ("x_idle_last", c_void_p), ("x_total_idle", c_void_p),
        ("x_col4", c_void_p), ("x_tuam", c_void_p), ("x_legal", c_void_p), ("x_blocked", c_void_p),
        ("mirror_actions", c_void_p),
    ]


class NativeError(RuntimeError):
    pass


_VP, _I32P, _I64P = c_void_p, POINTER(c_int32), POINTER(c_int64)

# every entry point of include/jss_b200.h: symbol -> (restype, argtypes), in the header's order
SIGNATURES = {
    "jss_create": (c_int, [POINTER(c_void_p), c_int, c_int, c_uint32, c_uint64]),
    "jss_destroy": (None, [_VP]),
    "jss_last_error": (c_char_p, [_VP]),
    "jss_abi_version": (c_int, []),
    "jss_load_instances": (c_int, [_VP, c_int, _I32P, _I32P, _I64P, _I32P, _I32P]),
    "jss_assign": (c_int, [_VP, _I32P]),
    "jss_get_buffers": (c_int, [_VP, POINTER(JssBuffers)]),
    "jss_instance_scalars": (c_int, [_VP, c_int, _I64P]),
    "jss_reset": (c_int, [_VP, _VP, _VP]),
    "jss_step": (c_int, [_VP, _VP, _VP]),
    "jss_step_export": (c_int, [_VP, _VP, _VP]),
    "jss_policy": (c_int, [_VP, c_int, c_int, c_uint64, c_uint64, _VP, _VP]),
    "jss_set_cr_due_date_factor": (c_int, [_VP, c_double]),
    "jss_step_sample": (c_int, [_VP, _VP, c_int, c_int, c_uint64, c_uint64, _VP, _VP]),
    "jss_step_logits": (c_int, [_VP, _VP, c_int64, c_uint64, c_uint64, _VP, _VP, _VP]),
    "jss_step_logits_record": (c_int, [_VP, _VP, c_int64, c_uint64, c_uint64, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_step_greedy": (c_int, [_VP, _VP, c_int64, c_double, c_uint64, c_uint64, _VP, _VP, _VP]),
    "jss_step_greedy_record": (c_int, [_VP, _VP, c_int64, c_double, c_uint64, c_uint64, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_refresh_obs": (c_int, [_VP, _VP]),
    "jss_rollout": (c_int, [_VP, c_int, c_uint64, c_uint64, c_int, c_int, _VP]),
    "jss_rollout_traj": (c_int, [_VP, c_int, c_uint64, c_uint64, c_int, _VP, _VP, _VP, _VP, _VP]),
    "jss_rollout_priority": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_int, _VP]),
    "jss_rollout_priority_sample": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int, _VP, _VP,
                                            _VP]),
    "jss_rollout_priority_sample_entropy": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int,
                                                    _VP, _VP, _VP, _VP, _VP]),
    "jss_lookahead": (c_int, [_VP, c_int, c_int, c_uint64, c_uint64, _VP, c_int64, _VP]),
    "jss_lookahead_priority": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, _VP, c_int64, _VP]),
    "jss_lookahead_sample": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int64, _VP, c_int64,
                                     _VP]),
    "jss_sample_episodes": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int64, _VP, _VP, c_int64,
                                    _VP]),
    "jss_sample_episodes_grad": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int64, _VP, c_int64,
                                         c_int, _VP, _VP]),
    "jss_sample_episodes_entropy": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int64, _VP, _VP,
                                            _VP, c_int64, _VP]),
    "jss_sample_episodes_entropy_grad": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int64, _VP,
                                                 _VP, c_int64, c_int, _VP, _VP]),
    "jss_sample_episodes_solution": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, _VP, _VP, _VP]),
    "jss_beam_search": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_int, _VP, _VP, c_int64, _VP, _VP]),
    "jss_sample_without_replacement": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, c_uint64, c_uint64, c_int, _VP, _VP,
                                               _VP, c_int64, _VP, _VP]),
    "jss_beam_step": (c_int, [_VP, _VP, c_int64, c_int, _VP, _VP, _VP, _VP, _VP]),
    "jss_stochastic_beam_step": (c_int, [_VP, _VP, c_int64, c_int, c_uint64, c_uint64, _VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_order_log_prob": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, _VP, c_int64, _VP, _VP, c_int64, _VP]),
    "jss_order_log_prob_grad": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, _VP, c_int64, _VP, c_int64, c_int, _VP,
                                        _VP]),
    "jss_order_log_prob_entropy": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, _VP, c_int64, _VP, _VP, _VP, c_int64,
                                           _VP]),
    "jss_order_log_prob_entropy_grad": (c_int, [_VP, _VP, c_int64, c_int64, c_int64, _VP, c_int64, _VP, _VP, c_int64,
                                                c_int, _VP, _VP]),
    "jss_improve_orders": (c_int, [_VP, _VP, c_int64, c_int, _VP, _VP, _VP, _VP, c_int64, _VP]),
    "jss_step_host": (c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_host_step_begin": (c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_host_wait": (c_int, [_VP, c_int]),
    "jss_host_step_begin_packed": (c_int, [_VP, _VP, _VP, _VP, _VP, _VP]),
    "jss_host_step_begin_hybrid": (c_int, [_VP, _VP, _VP, _VP, _VP, c_int, _VP, _VP]),
    "jss_host_expand_obs_range": (c_int, [_VP, _VP, _VP, _VP, c_int, c_int]),
    "jss_host_wire_stride": (c_int64, [_VP]),
    "jss_host_expand_obs": (c_int, [_VP, _VP, _VP, _VP]),
    "jss_host_configure": (c_int, [c_int, c_int]),
    "jss_host_threads": (c_int, []),
    "jss_host_set_simd": (c_int, [c_int]),
    "jss_stats": (c_int, [_VP, _I64P, _VP]),
    "jss_export_state": (c_int, [_VP, _VP]),
    "jss_import_state": (c_int, [_VP, _VP, _VP]),
    "jss_host_masked_random": (c_int, [_VP, c_int, c_int, c_int64, c_uint64, c_uint64, c_uint64, _VP]),
    "jss_launch_count": (c_int64, [_VP]),
}
EXPORTED_SYMBOLS = tuple(SIGNATURES)


def _declare(L):
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    return L


class CudaBackend:
    """Device memory / stream plumbing through torch (plumbing only: every kernel is ours)."""

    name = "cuda"
    pin_memory = True        # host staging buffers are page-locked: DMA targets, device-mapped by the kernels

    def __init__(self):
        self._lib = None

    def library(self):
        if self._lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(
                    f"{LIB_PATH} is missing: build the CUDA extension first "
                    "(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback.")
            L = _declare(ctypes.CDLL(LIB_PATH))
            if L.jss_abi_version() != JSS_ABI_VERSION:
                raise NativeError("libjss_b200.so ABI version mismatch; rebuild")
            self._lib = L
        return self._lib

    def torch_device(self, index):
        import torch
        return torch.device("cuda", index)

    def stream(self, device_index):
        import torch
        return c_void_p(torch.cuda.current_stream(device_index).cuda_stream)

    def wrap(self, ptr, shape, dtype, device_index, strides=None):
        """Zero-copy torch view of library-owned device memory."""
        import torch

        class _Holder:
            pass

        h = _Holder()
        npdt = np.dtype(dtype)
        h.__cuda_array_interface__ = {
            "shape": tuple(int(s) for s in shape), "typestr": npdt.str, "data": (int(ptr), False), "version": 3,
            "strides": None if strides is None else tuple(int(s) for s in strides),
        }
        return torch.as_tensor(h, device=torch.device("cuda", device_index))

    def synchronize(self, device_index):
        import torch
        torch.cuda.synchronize(device_index)

    def warp_slots(self, device_index):
        """Warps the device keeps resident at once: SMs x resident threads per SM / 32."""
        import torch
        prop = torch.cuda.get_device_properties(device_index)
        return prop.multi_processor_count * prop.max_threads_per_multi_processor // 32


backend = CudaBackend()   # tests/emu swaps this object; product code never does


def check(handle, rc, what):
    if rc != 0:
        msg = backend.library().jss_last_error(handle)
        raise NativeError(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")


def as_i32p(a):
    return a.ctypes.data_as(POINTER(c_int32))


def host_view(ptr, shape, dtype, strides=None):
    """Zero-copy numpy view of host memory at address `ptr` (byte `strides`; default: C-contiguous)."""
    dt = np.dtype(dtype)
    shape = tuple(int(s) for s in shape)
    nbytes = (int(np.prod(shape)) * dt.itemsize if strides is None
              else sum((sh - 1) * int(st) for sh, st in zip(shape, strides)) + dt.itemsize)
    buf = (ctypes.c_char * max(nbytes, 1)).from_address(int(ptr))
    return np.ndarray(shape, dt, buffer=buf, strides=None if strides is None else tuple(int(s) for s in strides))
