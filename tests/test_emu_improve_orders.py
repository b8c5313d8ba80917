"""jss_improve_orders (operation orders improved by steepest descent on the critical path, the envs untouched) under
HOST EMULATION of the CUDA kernels (tests/emu): the tests of tests/improve_orders_suite.py at CPU-friendly sizes."""
from tests import improve_orders_suite
from tests.backends import collect

collect(globals(), improve_orders_suite, "emu")
