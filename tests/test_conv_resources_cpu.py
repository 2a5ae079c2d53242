"""Register budget of the conv engine's kernel (no GPU): every conv_tc_kernel instantiation in the built library fits the
128 registers a 512-thread CTA gets per thread, with no stack frame (no spills to local memory).  A spill in the consumer
warpgroups lands between the k-block's wgmma issue and its wait; in the producers it costs local-memory traffic per
k-block."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bts_b200", "libbts_b200.so")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def _conv_kernel_resources():
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name and "conv_tc_kernel" in name:
            res[name] = (int(m.group(1)), int(m.group(2)))
        name = None
    return res


def test_conv_kernel_fits_registers_without_spills():
    res = _conv_kernel_resources()
    assert len(res) == 24, "expected 24 conv_tc_kernel instantiations, found %d" % len(res)
    bad = {k: v for k, v in res.items() if v[0] > 128 or v[1] != 0}
    assert not bad, "conv_tc_kernel instantiations over 128 registers or with a stack frame (REG, STACK): %s" % bad
