"""Tile plan and register reallocation of the conv engine's wide output tiles (no GPU): n-tiles of up to 128 channels,
equal and multiples of 16; the packed operator sized from them; and every conv_tc_kernel instantiation moving registers
from its producer warpgroups to its consumer warpgroups (setmaxnreg, SASS USETMAXREG)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bts_b200", "libbts_b200.so")


def _lib():
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    from bts_b200 import _lib as L
    return L.lib()


@pytest.mark.parametrize("cout,n_tile", [(16, 16), (64, 64), (80, 80), (96, 96), (128, 128), (192, 96), (200, 112),
                                         (448, 112), (512, 128), (2208, 128)])
def test_n_tile_widths(cout, n_tile):
    assert _lib().bts_conv_n_tile(cout) == n_tile


def test_group_n_tile_of_a_128_window():
    L = _lib()
    assert L.bts_conv_group_n_tile(128) == 128
    assert L.bts_conv_group_n_tile(96) == 96
    assert L.bts_conv_group_n_tile(256) == 128


@pytest.mark.parametrize("rows,kch,k", [(96, 64, 3), (192, 240, 1), (200, 36, 3), (448, 512, 3), (512, 2208, 3),
                                        (2208, 512, 3)])
def test_packed_floats_follow_the_tile_plan(rows, kch, k):
    L = _lib()
    n_tile = L.bts_conv_n_tile(rows)
    n_tiles = -(-rows // n_tile)
    KB = -(-(k * k * -(-kch // 4)) // 8)
    assert L.bts_conv_packed_floats(rows, kch, k, k) == n_tiles * KB * 2 * n_tile * 32


def test_grouped_packed_floats_follow_the_tile_plan():
    L = _lib()
    width, cpg = 256, 8
    kwin = L.bts_conv_group_window(width, cpg)
    assert kwin == 128
    KB = -(-(9 * kwin // 4) // 8)
    assert L.bts_conv_packed_floats_grouped(width, cpg, 3, 3) == (width // 128) * KB * 2 * 128 * 32


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def test_every_conv_kernel_reallocates_registers_to_its_consumers():
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "conv_tc_kernel" in m.group(1) else None
            if name:
                kernels[name] = set()
            continue
        if name:
            m = re.search(r"USETMAXREG\.(\w+)", line)
            if m:
                kernels[name].add(m.group(1))
    assert kernels, "no conv_tc_kernel in the library"
    missing = sorted(k for k, ops in kernels.items() if not {"TRY_ALLOC", "DEALLOC"} <= ops)
    assert not missing, "conv_tc_kernel instantiations without both register reallocations: %s" % missing
