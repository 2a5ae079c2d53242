"""Per-layer timing of the wgmma conv engine vs cuDNN fp32 on K16 (B=16, 352x704) DenseNet-161 + decoder shapes.
usage: python tools/conv_layers.py [fwd|dgrad|wgrad|all]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from bts_b200 import conv

torch.backends.cudnn.allow_tf32 = False
torch.backends.cudnn.benchmark = True
B = 16
# name, Cin, H, W, Cout, k, dil, upsample
LAYERS = [
    ("db1 1x1 (Cin 240)", 240, 88, 176, 192, 1, 1, 0),
    ("db1 3x3 192->48", 192, 88, 176, 48, 3, 1, 0),
    ("db2 1x1 (Cin 480)", 480, 44, 88, 192, 1, 1, 0),
    ("db2 3x3 192->48", 192, 44, 88, 48, 3, 1, 0),
    ("db3 1x1 (Cin 1200)", 1200, 22, 44, 192, 1, 1, 0),
    ("db3 3x3 192->48", 192, 22, 44, 48, 3, 1, 0),
    ("db4 1x1 (Cin 1632)", 1632, 11, 22, 192, 1, 1, 0),
    ("upconv5 2208->512 up", 2208, 11, 22, 512, 3, 1, 1),
    ("conv5 896->512", 896, 22, 44, 512, 3, 1, 0),
    ("upconv4 512->256 up", 512, 22, 44, 256, 3, 1, 1),
    ("conv4 448->256", 448, 44, 88, 256, 3, 1, 0),
    ("daspp_6 1x1 576->256", 576, 44, 88, 256, 1, 1, 0),
    ("daspp 3x3 d12 256->128", 256, 44, 88, 128, 3, 12, 0),
    ("daspp_conv 896->128", 896, 44, 88, 128, 3, 1, 0),
    ("conv3 225->128", 225, 88, 176, 128, 3, 1, 0),
    ("upconv2 128->64 up", 128, 88, 176, 64, 3, 1, 1),
    ("conv2 161->64", 161, 176, 352, 64, 3, 1, 0),
    ("upconv1 64->32 up", 64, 176, 352, 32, 3, 1, 1),
    ("conv1 36->32", 36, 352, 704, 32, 3, 1, 0),
]

def timeit(fn, n=5):
    fn(); fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

mode = sys.argv[1] if len(sys.argv) > 1 else "fwd"
tc_only = len(sys.argv) > 2 and sys.argv[2] == "tc"      # skip the cuDNN column (A/B sweeps of the engine)
tot_tc = tot_cd = 0.0
print("%-26s %9s %9s %9s %9s" % ("layer", "tc ms", "tc TF/s", "cudnn ms", "cudnn TF/s"))
for name, Cin, H, W, Cout, k, dil, up in LAYERS:
    x = torch.randn(B, Cin, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cout, Cin, k, k, device="cuda") / (Cin * k * k) ** 0.5
    pad = dil * (k // 2)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    flops = 2.0 * B * Ho * Wo * Cout * Cin * k * k
    packed = conv.pack_weights(w)
    if mode == "fwd":
        f_tc = lambda: conv.conv2d_tc(x, w, 1, pad, dil, upsample2=bool(up))
        xu = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
        f_cd = lambda: F.conv2d(xu, w, None, 1, pad, dil)
    elif mode == "dgrad":
        gy = torch.randn(B, Cout, Ho, Wo, device="cuda").contiguous(memory_format=torch.channels_last)
        packedT = conv.pack_weights(w, True)
        f_tc = lambda: conv.conv2d_tc(gy, w, 1, dil * (k - 1) - pad, dil, transpose_flip=True)
        xu = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
        f_cd = lambda: torch.ops.aten.convolution_backward(gy, xu, w, None, [1, 1], [pad, pad], [dil, dil], False, [0, 0], 1, [True, False, False])
    else:
        gy = torch.randn(B, Cout, Ho, Wo, device="cuda").contiguous(memory_format=torch.channels_last)
        f_tc = lambda: conv.wgrad_tc(x, gy, w.shape, w.stride(), 1, pad, dil, upsample2=bool(up))
        xu = F.interpolate(x, scale_factor=2, mode="nearest") if up else x
        f_cd = lambda: torch.ops.aten.convolution_backward(gy, xu, w, None, [1, 1], [pad, pad], [dil, dil], False, [0, 0], 1, [False, True, False])
    t_tc = timeit(f_tc)
    t_cd = float("nan") if tc_only else timeit(f_cd)
    tot_tc += t_tc; tot_cd += t_cd
    print("%-26s %9.3f %9.1f %9.3f %9.1f" % (name, t_tc, flops / t_tc / 1e9, t_cd, flops / t_cd / 1e9))
print("total %.2f ms (tc) vs %.2f ms (cudnn)" % (tot_tc, tot_cd))
