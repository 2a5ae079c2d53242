"""bts_b200 -- GPU-native (H100, sm_90a) implementation of the BTS dense forward/backward hot path.

Public surface = the reference's `bts` module surface (see bts_b200.model and the root-level bts.py);
native boundary = the C ABI in include/bts_b200.h (libbts_b200.so, loaded by bts_b200._lib).
"""
from .model import (BtsModel, atrous_conv, bn_init_as_tf, bts, encoder, local_planar_guidance,  # noqa: F401
                    reduction_1x1, silog_loss, upconv, weights_init_xavier)
from .conv import get_precision, set_precision  # noqa: F401
from .graph import get_eval_graphs, set_eval_graphs  # noqa: F401

__all__ = ["BtsModel", "atrous_conv", "bn_init_as_tf", "bts", "encoder", "local_planar_guidance",
           "reduction_1x1", "silog_loss", "upconv", "weights_init_xavier",
           "set_precision", "get_precision", "set_eval_graphs", "get_eval_graphs"]
