"""The parity tests of tests/parity_suite.py under HOST EMULATION of the CUDA kernels (tests/emu): the same
jss_device.cuh / jss_api.cu compiled with g++, 32 fibers per warp, strict collectives.  Pre-GPU safety net only -- the
authoritative parity tests are the `-m gpu` ones in tests/test_gpu_parity.py, which run the real sm_90a library."""
from tests import parity_suite
from tests.backends import collect

collect(globals(), parity_suite, "emu")
