"""The lane classes and the layout they decide, against closed forms written out here: the lane class of every J, the
state-block geometry of every J x M the kernels accept, and the action mask's row stride."""
import os
import subprocess

import numpy as np
import pytest

from tests.parity_common import synthetic_instance

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

_DRIVER = r"""
#include <stdio.h>
#include "jss_types.h"
int main() {
    for (int J = 1; J <= 256; J++)
        for (int M = 2; M <= 32; M++) {
            const JssBlockGeom g = jss_block_geom(J, M);
            printf("%d %d %d %d %d %d %d %d\n", J, M, jss_lane_class(J), g.Jcap, g.Mcap, g.tail, g.hdr, g.words);
        }
    return 0;
}
"""


def _round(x, m):
    return (x + m - 1) // m * m


def test_lane_class_and_block_geometry(tmp_path):
    src, exe = tmp_path / "geom.cpp", tmp_path / "geom"
    src.write_text(_DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "jssenv_b200", "csrc"), "-o", str(exe),
                           str(src)])
    got = np.loadtxt(subprocess.check_output([str(exe)], text=True).splitlines(), dtype=np.int64)
    assert got.shape == (256 * 31, 8)
    for J, M, cls, Jcap, Mcap, tail, hdr, words in got.tolist():
        # 1, 2, 4, 8 jobs per lane; J padded to 4 slots per lane (8 with 8 jobs per lane), 16-bit bits per lane above 128
        want_cls = 0 if J <= 32 else 1 if J <= 64 else 2 if J <= 128 else 3
        want_Jcap = _round(J, 8) if J > 128 else _round(J, 4)
        want_tail = 2 * want_Jcap + _round(want_Jcap, 8) // 2
        want_hdr = want_tail + _round(M, 4) + (16 if J > 128 else 8)
        assert (cls, Jcap, Mcap, tail, hdr, words) == (want_cls, want_Jcap, _round(M, 4), want_tail, want_hdr,
                                                       want_hdr + 4), (J, M)


@pytest.mark.parametrize("jobs_max", [1, 4, 5, 32, 33, 128, 129, 136, 256])
def test_action_mask_row_stride(jobs_max):
    from jssenv_b200 import JssVecEnv
    from tests.emu.emu_backend import use_emulation
    with use_emulation():
        env = JssVecEnv(2, {"instance_paths": [synthetic_instance(jobs_max, 2, 0)], "env_to_instance": [0, 0]})
        stride = env.action_mask.stride(0)
        env.close()
    assert stride == _round(jobs_max + 1, 8 if jobs_max > 128 else 4)
