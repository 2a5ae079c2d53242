"""Drop-in replacement for the reference's `pytorch/bts.py` module (the boundary of the hot path).

`bts_main.py` does `from bts import *` / `from bts import BtsModel` (bts_main.py:38,122-133) and
`bts_test.py` imports `<model_name>.py` from the checkpoint directory (bts_test.py:68-74): putting this
file (or a copy named <model_name>.py) on the import path swaps the whole model for the GPU-native one.
The reference module also leaks `torch`, `nn`, `math`, `torch_nn_func` through `import *`; so do we.
"""
import math  # noqa: F401

import torch  # noqa: F401
import torch.nn as nn  # noqa: F401
import torch.nn.functional as torch_nn_func  # noqa: F401

from bts_b200.model import (BtsModel, atrous_conv, bn_init_as_tf, bts, encoder,  # noqa: F401
                            local_planar_guidance, reduction_1x1, silog_loss, upconv, weights_init_xavier)
