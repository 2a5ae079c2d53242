"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the header declares,
and the Python module surface / state_dict wire format matches the reference's (no compute calls here)."""
import ctypes
import os
import re
import types

import pytest
import torch

from conftest import ROOT


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "bts_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(?:int|long long)\s+(bts_\w+)\s*\(", txt)))


def test_library_builds_and_exports_every_declared_symbol():
    from bts_b200 import _lib
    _lib.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    syms = _header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(L, s), "libbts_b200.so does not export %s" % s
    assert sorted(_lib.SIGNATURES) == syms          # ctypes table covers exactly the header
    buf = ctypes.create_string_buffer(128)
    assert L.bts_version(buf, 128) == 90 and b"sm_90a" in buf.value


def test_ops_refuse_cpu_tensors_no_fallback():
    from bts_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.lpg(torch.zeros(1, 4, 2, 2), 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.silog(torch.ones(4), torch.ones(4), torch.ones(4, dtype=torch.bool), 0.85)


def test_module_surface_matches_reference_names():
    import bts
    for n in ("BtsModel", "silog_loss", "weights_init_xavier", "bn_init_as_tf", "encoder", "bts",
              "local_planar_guidance", "reduction_1x1", "atrous_conv", "upconv", "torch", "nn", "math"):
        assert hasattr(bts, n), n


def test_decoder_state_dict_matches_golden_reference_keys(golden):
    import bts
    g = golden("decoder_kitti")
    want = {k[3:]: tuple(v.shape) for k, v in g.items() if k.startswith("sd.")}
    dec = bts.bts(types.SimpleNamespace(max_depth=80.0, dataset="kitti"), [8, 8, 16, 24, 40], 128)
    got = {k: tuple(v.shape) for k, v in dec.state_dict().items()}
    assert got == want
    assert list(got) == [k[3:] for k in g if k.startswith("sd.")]      # same order too


def test_full_model_state_dict_and_freezing_contract():
    """bts_main.set_misc freezes encoder params by substring ('conv0','norm' for DenseNet) and
    builds AdamW groups from model.encoder / model.decoder -- names must stay torchvision's."""
    import bts
    p = types.SimpleNamespace(encoder="densenet161_bts", max_depth=80.0, dataset="kitti", bts_size=512)
    m = bts.BtsModel(p)
    sd = m.state_dict()
    assert len(sd) == 1075                                           # SURVEY Appendix C
    assert sd["decoder.upconv5.conv.weight"].shape == (512, 2208, 3, 3)
    assert sd["decoder.reduc8x8.reduc.inter_128_128.0.weight"].shape == (128, 128, 1, 1)
    assert sd["decoder.reduc1x1.reduc.final.0.weight"].shape == (1, 8, 1, 1)
    assert "encoder.base_model.denseblock1.denselayer1.norm1.weight" in sd
    names = [n for n, _ in m.encoder.named_parameters()]
    assert any("conv0" in n for n in names) and any("norm" in n for n in names)
    m.decoder.apply(bts.weights_init_xavier)                          # must hit our conv modules
    n_params = sum(p.numel() for p in m.parameters())
    assert abs(n_params - 47.0e6) < 0.1e6
