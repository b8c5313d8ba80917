"""jss_improve_orders (operation orders improved by steepest descent on the critical path, the envs untouched) on the
real sm_90a library: the tests of tests/improve_orders_suite.py at GPU sizes and full-size ta80 and ta01 runs.  Run on
an H100 with `pytest -m gpu`."""
from tests import improve_orders_suite
from tests.backends import collect

collect(globals(), improve_orders_suite, "gpu")
