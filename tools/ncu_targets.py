"""One representative launch of each kernel family, for `ncu --set full` where Nsight Compute is available.
usage: ncu_targets.py conv_db1 | dgrad_db1 | dgrad_pw | fwd_pw | wgrad2_db1 | wgrad2_pw | bn_onepass   [iters]
Shapes are the K16 ones (batch 16, DenseNet-161 block 1 / 2)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bts_b200 import conv, fused  # noqa: E402

what = sys.argv[1]
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
dev = torch.device("cuda", 0)
g = torch.Generator().manual_seed(0)


def nhwc(*shape):
    return torch.randn(*shape, generator=g).to(dev).contiguous(memory_format=torch.channels_last)


if what == "conv_db1":                       # dense-layer conv2 forward: BN+ReLU prologue, 192 -> 48, 3x3 @ 88x176
    x, w = nhwc(16, 192, 88, 176), (torch.randn(48, 192, 3, 3, generator=g) / 41.6).to(dev)
    sc, sh = (torch.rand(192, generator=g) + 0.5).to(dev), (torch.randn(192, generator=g) * 0.3).to(dev)
    for _ in range(iters):
        y = conv.conv2d_tc(x, w, 1, 1, 1, pre_scale=sc, pre_shift=sh, pre_relu=True)
elif what == "dgrad_db1":                    # its dgrad: 48 -> 192 over the transposed, flipped operator
    gy, w = nhwc(16, 48, 88, 176), (torch.randn(48, 192, 3, 3, generator=g) / 41.6).to(dev)
    for _ in range(iters):
        y = conv.conv2d_tc(gy, w, 1, 1, 1, transpose_flip=True)
elif what == "dgrad_pw":                     # dense-layer conv1 dgrad: 1x1, 192 -> 1200 @ 22x44 (short K, 256-wide tiles)
    gy, w = nhwc(16, 192, 22, 44), (torch.randn(192, 1200, 1, 1, generator=g) / 34.6).to(dev)
    for _ in range(iters):
        y = conv.conv2d_tc(gy, w, 1, 0, 1, transpose_flip=True)
elif what == "fwd_pw":                       # dense-layer conv1 forward: BN+ReLU prologue, 1200 -> 192 @ 22x44
    x, w = nhwc(16, 1200, 22, 44), (torch.randn(192, 1200, 1, 1, generator=g) / 34.6).to(dev)
    sc, sh = (torch.rand(1200, generator=g) + 0.5).to(dev), (torch.randn(1200, generator=g) * 0.3).to(dev)
    for _ in range(iters):
        y = conv.conv2d_tc(x, w, 1, 0, 1, pre_scale=sc, pre_shift=sh, pre_relu=True)
elif what == "wgrad2_db1":                   # its wgrad on the shifted-dY kernel (TMA landing ring)
    x, gy = nhwc(16, 192, 88, 176), nhwc(16, 48, 88, 176)
    sc, sh = (torch.rand(192, generator=g) + 0.5).to(dev), (torch.randn(192, generator=g) * 0.3).to(dev)
    for _ in range(iters):
        y = conv.wgrad_tc(x, gy, (48, 192, 3, 3), (1728, 9, 3, 1), 1, 1, 1, pre_scale=sc, pre_shift=sh, pre_relu=True)
elif what == "wgrad2_pw":                    # dense-layer conv1 wgrad (1x1, 336 -> 192) on the same kernel
    x, gy = nhwc(16, 336, 88, 176), nhwc(16, 192, 88, 176)
    sc, sh = (torch.rand(336, generator=g) + 0.5).to(dev), (torch.randn(336, generator=g) * 0.3).to(dev)
    for _ in range(iters):
        y = conv.wgrad_tc(x, gy, (192, 336, 1, 1), (336, 1, 1, 1), 1, 0, 1, pre_scale=sc, pre_shift=sh, pre_relu=True)
elif what == "bn_onepass":                   # one-pass norm1 backward of a block-2 dense layer: 480 channels @ 44x88
    x, gg, G = nhwc(16, 480, 44, 88), nhwc(16, 480, 44, 88), nhwc(16, 480, 44, 88)
    st = [(torch.rand(480, generator=g) + 0.5).to(dev), (torch.randn(480, generator=g) * 0.3).to(dev),
          (torch.randn(480, generator=g) * 0.1).to(dev), (torch.rand(480, generator=g) + 0.5).to(dev)]
    K = torch.zeros(2, 480, device=dev, dtype=torch.float64)
    for _ in range(iters):
        y = fused.bn_relu_backward_onepass(x, gg, st, G, K)
else:
    raise SystemExit("unknown target " + what)
torch.cuda.synchronize()
print("ok", what)
