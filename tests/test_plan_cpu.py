"""Host-side planning logic of the conv engine through the C ABI (no GPU, no kernel launches): split-K plans and workspace
sizes of the wgrad kernels on the K16 layer shapes, routing switches, operator-packing sizes, eligibility tables.
Without a device the library plans for 132 SMs (H100 SXM)."""
import ctypes

import pytest

SMS = 132

# (B, H, W, Cin, Cout, K) of DenseNet-161 / decoder layers at the K16 config
LAYERS = [(16, 88, 176, 192, 48, 3), (16, 44, 88, 192, 48, 3), (16, 22, 44, 192, 48, 3), (16, 11, 22, 192, 48, 3),
          (16, 352, 704, 36, 32, 3), (16, 176, 352, 161, 64, 3), (16, 88, 176, 336, 192, 1), (16, 22, 44, 2064, 192, 1),
          (16, 11, 22, 2160, 192, 1), (16, 22, 44, 896, 512, 3), (16, 44, 88, 256, 128, 3), (16, 22, 44, 2112, 1056, 1)]


def _lib():
    from bts_b200 import _lib as L
    return L.lib()


def _plan(L, B, H, W, Cin, Cout, K, stride=1):
    split, ws = ctypes.c_int(0), ctypes.c_longlong(0)
    rc = L.bts_conv_wgrad_plan(B, H, W, Cin, Cout, K, K, stride, ctypes.byref(split), ctypes.byref(ws))
    assert rc == 0
    return split.value, ws.value


@pytest.mark.parametrize("layer", LAYERS)
def test_wgrad_plan_workspace_and_wave_fill(layer):
    L = _lib()
    B, H, W, Cin, Cout, K = layer
    split, ws = _plan(L, *layer)
    assert split >= 1
    assert ws == split * K * K * Cin * Cout                       # [split][taps][Cin][Cout] partials
    L.bts_wgrad2_set_min_pixels(1 << 40)                          # force the tap-in-grid kernel: still a valid plan
    try:
        s2, w2 = _plan(L, *layer)
        assert s2 >= 1 and w2 == s2 * K * K * Cin * Cout
    finally:
        L.bts_wgrad2_set_min_pixels(-1)


def test_narrow_output_routing_fills_one_wave_and_respects_the_switches():
    L = _lib()
    # dense 3x3 192->48 @22x44x16 = 15488 pixels: shifted-dY kernel, 3 input-channel tiles x 3 output-channel groups x
    # split-K CTAs fill whole waves of the SMs
    split, _ = _plan(L, 16, 22, 44, 192, 48, 3)
    ctas = 9 * split
    assert ctas / (-(-ctas // SMS) * SMS) >= 0.98
    # every CTA keeps at least min_kblocks k-blocks of 16 pixels
    assert (15488 // 16) // split >= 8
    L.bts_wgrad2_set_min_kblocks(64)
    try:
        s64, _ = _plan(L, 16, 22, 44, 192, 48, 3)
        assert s64 <= (15488 // 16 + 63) // 64 and s64 < split          # at most ceil(k-blocks / 64) splits
    finally:
        L.bts_wgrad2_set_min_kblocks(0)
    # below the pixel threshold (block 4: 3872 pixels) the tap-in-grid plan is used: same answer with wgrad2 disabled
    a = _plan(L, 16, 11, 22, 192, 48, 3)
    L.bts_wgrad2_set_min_pixels(1 << 40)
    try:
        assert _plan(L, 16, 11, 22, 192, 48, 3) == a
    finally:
        L.bts_wgrad2_set_min_pixels(-1)
    # 1x1 layers with 64 < Cout <= 256 are routed to the same kernel unless switched off (both plans must be valid)
    on = _plan(L, 16, 88, 176, 336, 192, 1)
    L.bts_wgrad2_set_pointwise(0)
    try:
        off = _plan(L, 16, 88, 176, 336, 192, 1)
    finally:
        L.bts_wgrad2_set_pointwise(1)
    assert on[0] >= 1 and off[0] >= 1 and on[1] == on[0] * 336 * 192 and off[1] == off[0] * 336 * 192
    # strided layers never use the shifted-dY kernel (its plan would differ)
    assert _plan(L, 16, 44, 88, 192, 48, 3, stride=2)[0] >= 1


def test_eligibility_tables_of_the_cuda_core_pointwise_kernels():
    L = _lib()
    for cin in (8, 16, 32, 64):
        assert L.bts_conv_pw_fwd_eligible(cin, 1) and L.bts_conv_pw_fwd_eligible(cin, 64)
        assert not L.bts_conv_pw_fwd_eligible(cin, 65) and not L.bts_conv_pw_fwd_eligible(cin, 0)
        assert L.bts_conv_pw_wgrad_eligible(cin, 32) and not L.bts_conv_pw_wgrad_eligible(cin, 33)
    for cin in (4, 12, 24, 128, 192):
        assert not L.bts_conv_pw_fwd_eligible(cin, 16)
        assert not L.bts_conv_pw_wgrad_eligible(cin, 16)


def test_packed_operator_sizes_and_group_windows():
    L = _lib()
    # packed operator: per N tile, per k-block of 32 channels, hi and lo rows of 128 bytes
    for (cout, kch, k) in [(48, 192, 3), (192, 2064, 1), (512, 2208, 3), (32, 36, 3), (1056, 2112, 1)]:
        n = L.bts_conv_packed_floats(cout, kch, k, k)
        assert n > 0 and n % 32 == 0
        assert n >= 2 * cout * ((kch * k * k + 31) // 32 * 32)    # at least hi + lo of every (row, padded K) element
    # ResNeXt grouped 3x3: 32 groups of 4 / 8 / 16 / 32 / 64 channels -> 128-wide block-diagonal windows
    for width, cpg in [(128, 4), (256, 8), (512, 16), (1024, 32), (2048, 64)]:
        assert L.bts_conv_group_window(width, cpg) == 128
    assert L.bts_conv_group_window(96, 3) == 96                   # narrower widths: one window
    assert L.bts_conv_group_window(100, 3) == 0                   # width not a multiple of the group size: refused


def test_conv_fwd_refuses_conflicting_epilogues_before_any_launch():
    """bts_conv_fwd refuses every argument combination its epilogues cannot serve; with fake, 16-byte aligned device
    addresses each call must return before it touches the device"""
    L = _lib()
    EINVAL, EALIGN = -1, -2
    p = ctypes.c_void_p(1 << 20)

    def fwd(stats=(None, None), act=0, bn=(None, None), splits=1, ws=None):
        # a 3x3 32 -> 32 layer on one 8 x 8 image: every geometry argument is valid
        return L.bts_conv_fwd(p, 32, 1, 8, 8, 0, 0, 0, 0, 32, 3, 3, 1, 1, 1, p, 32, None, None, 0, p, 32, act, 0,
                              stats[0], stats[1], bn[0], 32, bn[1], 1, splits, ws, None)

    assert fwd(stats=(p, p), splits=2, ws=p) == EINVAL             # split-K with statistics
    assert fwd(stats=(p, p), bn=(p, p), splits=2, ws=p) == EINVAL  # split-K with the BatchNorm-backward epilogue
    assert fwd(bn=(p, p)) == EINVAL                                # BatchNorm-backward without its sums
    assert fwd(stats=(p, p), bn=(p, p), act=1) == EINVAL           # BatchNorm-backward after an activation
    assert fwd(stats=(p, p), bn=(p, None)) == EINVAL               # half the BatchNorm-backward operands
    assert fwd(stats=(p, p), bn=(None, p)) == EINVAL
    assert fwd(stats=(p, p), act=2) == EINVAL                      # statistics of an activated output
    assert fwd(stats=(p, None)) == EINVAL                          # one of the two statistics pointers
    assert fwd(stats=(None, p)) == EINVAL
    assert fwd(splits=2) == EINVAL                                 # splits without a workspace
    assert fwd(splits=0) == EINVAL
    assert fwd(splits=2, ws=ctypes.c_void_p((1 << 20) + 4)) == EALIGN   # misaligned workspace
