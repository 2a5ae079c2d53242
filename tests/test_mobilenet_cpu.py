"""CPU tests of the MobileNetV2 path (no GPU): the depthwise kernels compile without a stack frame, their entry points
refuse what they do not cover before any launch, and adopt_convs re-classes torchvision's mobilenet_v2 blocks without
touching the state_dict wire format."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from test_conv_resources_cpu import LIB, _cuobjdump


def _dw_kernel_resources():
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
        if m and name and ("dw3x3_" in name or "dw_colsum" in name):
            res[name] = (int(m.group(1)), int(m.group(2)))
        name = None
    return res


def test_depthwise_kernels_have_no_stack_frame():
    res = _dw_kernel_resources()
    # fwd and wgrad: stride {1,2} x prologue {off,on}; the stride-2 dgrad; the two fixed-order column sums
    assert len(res) == 11, "expected 11 depthwise kernel instantiations, found %d: %s" % (len(res), sorted(res))
    bad = {k: v for k, v in res.items() if v[1] != 0}
    assert not bad, "depthwise kernels with a stack frame (REG, STACK): %s" % bad


def _lib():
    from bts_b200 import _lib
    _lib.build()
    return _lib.lib()


def test_depthwise_entry_points_refuse_unsupported_arguments():
    L = _lib()
    EINVAL = -1
    # fake, 16-byte aligned device addresses: every call below must return before it launches anything
    p = ctypes.c_void_p(1 << 20)
    for C, stride in ((30, 1), (6, 2), (32, 3), (32, 0)):
        assert L.bts_dw3x3_fwd_workspace_floats(1, 9, 13, C, stride) == EINVAL
        assert L.bts_dw3x3_wgrad_workspace_floats(1, 9, 13, C, stride) == EINVAL
        assert L.bts_dw3x3_fwd(p, C, 1, 9, 13, C, stride, p, 9, 3, 1, None, None, None, None, p, C, None, None, None,
                               None) == EINVAL
        assert L.bts_dw3x3_dgrad(p, C, 1, 9, 13, C, stride, p, 9, 3, 1, p, C, None) == EINVAL
        assert L.bts_dw3x3_wgrad(p, C, p, C, 1, 9, 13, C, stride, None, None, p, p, 9, 3, 1, None) == EINVAL
    assert L.bts_dw3x3_fwd_workspace_floats(1, 9, 13, 32, 1) > 0
    assert L.bts_dw3x3_wgrad_workspace_floats(2, 9, 13, 96, 2) > 0
    # null pointers
    assert L.bts_dw3x3_fwd(None, 32, 1, 9, 13, 32, 1, p, 9, 3, 1, None, None, None, None, p, 32, None, None, None,
                           None) == EINVAL
    assert L.bts_dw3x3_fwd(p, 32, 1, 9, 13, 32, 1, None, 9, 3, 1, None, None, None, None, p, 32, None, None, None,
                           None) == EINVAL
    assert L.bts_dw3x3_fwd(p, 32, 1, 9, 13, 32, 1, p, 9, 3, 1, p, None, None, None, p, 32, None, None, None,
                           None) == EINVAL                      # half a prologue
    assert L.bts_dw3x3_fwd(p, 32, 1, 9, 13, 32, 1, p, 9, 3, 1, None, None, None, None, p, 32, p, p, None,
                           None) == EINVAL                      # statistics without a workspace
    assert L.bts_dw3x3_dgrad(None, 32, 1, 9, 13, 32, 1, p, 9, 3, 1, p, 32, None) == EINVAL
    assert L.bts_dw3x3_dgrad(p, 32, 1, 9, 13, 32, 1, p, 9, 3, 1, None, 32, None) == EINVAL
    assert L.bts_dw3x3_wgrad(p, 32, None, 32, 1, 9, 13, 32, 1, None, None, p, p, 9, 3, 1, None) == EINVAL
    assert L.bts_dw3x3_wgrad(p, 32, p, 32, 1, 9, 13, 32, 1, None, None, None, p, 9, 3, 1, None) == EINVAL
    # pixel strides that break the 16-byte granules
    assert L.bts_dw3x3_fwd(p, 34, 1, 9, 13, 32, 1, p, 9, 3, 1, None, None, None, None, p, 32, None, None, None,
                           None) == EINVAL
    assert L.bts_bn_add(None, 32, 10, 32, p, p, p, 32, p, 32, None) == EINVAL


def test_adopt_convs_reclasses_mobilenet_v2_and_keeps_the_state_dict():
    import torchvision
    from bts_b200 import model as M
    torch.manual_seed(0)
    ref = torchvision.models.mobilenet_v2().features
    f = torchvision.models.mobilenet_v2().features
    f.load_state_dict(ref.state_dict())
    M.adopt_convs(f)
    names = [type(m).__name__ for m in f.modules()]
    assert names.count("InvertedResidualTC") == 17
    assert names.count("ConvNormReLU6TC") == 2
    assert type(f[0]).__name__ == "ConvNormReLU6TC" and type(f[18]).__name__ == "ConvNormReLU6TC"
    assert all(M._inverted_residual_eligible(m) for m in f.modules() if type(m).__name__ == "InvertedResidualTC")
    a, b = ref.state_dict(), f.state_dict()
    assert list(a) == list(b)
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k
    assert "1.conv.0.0.weight" in b and "2.conv.0.0.weight" in b and "18.1.running_var" in b
    # the 17 depthwise convs are Conv2dTC and eligible for the depthwise kernels
    from bts_b200 import dwconv
    dws = [m for m in f.modules() if isinstance(m, torch.nn.Conv2d) and m.groups > 1]
    assert len(dws) == 17 and all(type(m) is M.Conv2dTC and dwconv.eligible(m) for m in dws)
