"""Split-K plan of the forward / dgrad engine (bts_conv_fwd_splitk_plan, csrc/conv_tc.cu) and the resources of its reduce
kernel, without a GPU.

The plan is checked over the engine launches of batch-1 inference at the T1 (DenseNet-121, 416 x 544), NYU test
(DenseNet-161, 480 x 640) and KITTI test (DenseNet-161, 352 x 1216) shapes -- the decoder's H/16 and H/8 layers and the
dense layers of blocks 3 and 4 -- on 132 SMs (H100 SXM), 114 (H100 PCIe) and 66 (BTS_B200_SM_LIMIT).  The library reads the
SM count once per process, so each count runs in a subprocess with no visible device (the library then assumes 132) and
the cap in BTS_B200_SM_LIMIT."""
import json
import os
import subprocess
import sys

import pytest

from test_conv_resources_cpu import LIB, ROOT, _cuobjdump

BLOCK_M = 128
MIN_KB = 8           # SPLITK_MIN_KB of csrc/conv_tc.cu
ENCODERS = {"densenet121": dict(f=[64, 64, 128, 256, 1024], growth=32, blocks=(24, 16), c3=512),
            "densenet161": dict(f=[96, 96, 192, 384, 2208], growth=48, blocks=(36, 24), c3=768)}
SHAPES = {"T1": ("densenet121", 416, 544), "NYU": ("densenet161", 480, 640), "KITTI": ("densenet161", 352, 1216)}


def layers(enc, H, W):
    """(name, Hout, Wout, Cin, Cout, k) of the batch-1 eval forward's engine launches at H/32, H/16 and H/8"""
    e = ENCODERS[enc]
    f, gr = e["f"], e["growth"]
    h8, w8, h16, w16 = H // 8, W // 8, H // 16, W // 16
    h32, w32 = h16 // 2, w16 // 2
    out = [("upconv5", h16, w16, f[4], 512, 3), ("conv5", h16, w16, 512 + f[3], 512, 3),
           ("upconv4", h8, w8, 512, 256, 3), ("conv4", h8, w8, 256 + f[2], 256, 3),
           ("daspp_conv", h8, w8, 512 + 256 + 128, 128, 3)]
    for d, cin in ((3, 256), (6, 256 + 128 + f[2]), (12, 512 + f[2]), (18, 512 + 128 + f[2]), (24, 512 + 256 + f[2])):
        out += [("daspp_%d_1x1" % d, h8, w8, cin, 256, 1), ("daspp_%d_3x3" % d, h8, w8, 256, 128, 3)]
    c0 = e["c3"] // 2                                # after transition 2
    for blk, (n, h, w) in enumerate(((e["blocks"][0], h16, w16), (e["blocks"][1], h32, w32)), start=3):
        for i in range(0, n, max(1, n // 4)):        # a few layers of each block: the 1x1 grows with the layer index
            out += [("db%d_%d_conv1" % (blk, i), h, w, c0 + i * gr, 4 * gr, 1),
                    ("db%d_%d_conv2" % (blk, i), h, w, 4 * gr, gr, 3)]
        c0 = (c0 + n * gr) // 2
    return out


def n_tile(Cout):
    n = -(-Cout // 16) * 16
    if n > 128:
        t = -(-n // 128)
        n = -(-(-(-Cout // t)) // 16) * 16
    return n


_PLAN = """
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from bts_b200 import _lib
L = _lib.lib()
res = []
for args in json.loads(sys.argv[2]):
    s, w = ctypes.c_int(args[-1]), ctypes.c_longlong(-1)
    rc = L.bts_conv_fwd_splitk_plan(*args[:-1], ctypes.byref(s), ctypes.byref(w))
    res.append((rc, s.value, w.value))
print(json.dumps(res))
"""


def plan(sms, calls):
    """[(rc, splits, workspace floats)] of bts_conv_fwd_splitk_plan(B, Hout, Wout, kwin, Cin, KH, KW, Cout, splits) on
    `sms` SMs"""
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", BTS_B200_SM_LIMIT=str(sms))
    r = subprocess.run([sys.executable, "-c", _PLAN, ROOT, json.dumps(calls)], env=env, capture_output=True, text=True,
                       check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("sms", [132, 114, 66])
def test_plan_fills_one_wave_with_long_enough_splits(sms):
    rows = [(shape, l) for shape, (enc, H, W) in SHAPES.items() for l in layers(enc, H, W)]
    calls = [[1, h, w, 0, cin, k, k, cout, 0] for _, (_, h, w, cin, cout, k) in rows]
    split_any = 0
    for (shape, (name, h, w, cin, cout, k)), (rc, s, wsf) in zip(rows, plan(sms, calls)):
        where = "%s %s on %d SMs: splits %d" % (shape, name, sms, s)
        assert rc == 0, where
        M = h * w
        tiles = -(-M // BLOCK_M) * -(-cout // n_tile(cout))
        KB = -(-(k * k * -(-cin // 4)) // 8)
        if 2 * tiles > sms:
            assert s == 1 and wsf == 0, where                       # the launch already fills more than half the SMs
            continue
        want = max(1, min(sms // tiles, KB // MIN_KB))
        want = -(-KB // -(-KB // want))                              # no empty split
        assert s == want, where
        if s > 1:
            split_any += 1
            assert tiles * s <= sms, where                          # one wave
            assert -(-KB // s) >= MIN_KB, where                     # k-blocks per split
            assert wsf == s * M * -(-cout // 4) * 4, where          # [splits][M][Cout rounded up to 4]
        else:
            assert wsf == 0, where
    assert split_any >= 10


def test_plan_examples_and_forced_counts():
    # T1 upconv5: 26 x 34 output, 1024 -> 512 (4 n-tiles of 128): 28 tiles, 288 k-blocks -> 4 splits of 72 (112 CTAs).
    # KB = 9 forced to 4: ranges of 3 would leave the fourth empty -> 3; forced beyond KB -> KB; 1 never splits
    # (Cin 32 at 3x3: 72 channel quads = 9 k-blocks)
    calls = [[1, 26, 34, 0, 1024, 3, 3, 512, 0], [1, 26, 34, 0, 1024, 3, 3, 512, 1], [1, 8, 8, 0, 32, 3, 3, 16, 4],
             [1, 8, 8, 0, 32, 3, 3, 16, 50], [1, 8, 8, 0, 32, 3, 3, 16, 3], [1, 26, 34, 0, 1024, 3, 3, 512, -1],
             [0, 26, 34, 0, 1024, 3, 3, 512, 0], [1, 26, 34, 8, 256, 3, 3, 256, 0]]
    r = plan(132, calls)
    assert r[0] == [0, 4, 4 * 26 * 34 * 512]
    assert r[1] == [0, 1, 0]
    assert r[2] == [0, 3, 3 * 64 * 16]
    assert r[3] == [0, 9, 9 * 64 * 16]
    assert r[4] == [0, 3, 3 * 64 * 16]
    assert r[5][0] == -1 and r[6][0] == -1 and r[7][0] == -1           # negative count, B = 0, kwin not a multiple of 16


def test_reduce_kernel_has_no_stack_frame():
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = []
    name = None
    for line in out.splitlines():
        if line.strip().startswith("Function "):
            name = line.split()[1].rstrip(":")
            continue
        if name and "conv_splitk_reduce_kernel" in name and "STACK:" in line:
            found.append(int(line.split("STACK:")[1].split()[0]))
        name = None
    assert found == [0], found
