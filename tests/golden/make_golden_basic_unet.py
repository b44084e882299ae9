"""Generate tests/golden/basic_unet_tc.npz from the REAL reference (Project-MONAI/MONAI on PYTHONPATH):

    PYTHONPATH=<MONAI source checkout> python tests/golden/make_golden_basic_unet.py

The BasicUNet configurations of basic_unet_cases.py, in the layout of make_golden_tc.py: the reference runs in fp32 (eval mode) on
the fp16-rounded input; the fixture stores a strided sample of the input, a strided sample of the output and its float64 sum.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from basic_unet_cases import BASIC_CASES, FIXTURE  # noqa: E402
from monai.networks.nets import BasicUNet  # noqa: E402
from tc_cases import X_STRIDE, make_input  # noqa: E402
from weights import fill_state_dict  # noqa: E402


def write() -> None:
    out = {}
    for tag, (kw, shape, seed, xseed, s) in BASIC_CASES.items():
        net = BasicUNet(**kw)
        net.load_state_dict(fill_state_dict(net.state_dict(), seed))
        net.eval()
        x = make_input(shape, xseed)
        with torch.no_grad():
            y = net(x.float())
        out[f"{tag}.x_sub"] = x.numpy()[..., ::X_STRIDE, ::X_STRIDE, ::X_STRIDE]
        out[f"{tag}.x_stride"] = np.array(X_STRIDE)
        out[f"{tag}.y_sub"] = y.numpy()[..., ::s, ::s, ::s]
        out[f"{tag}.y_stride"] = np.array(s)
        out[f"{tag}.y_sum"] = np.array(float(y.double().sum()))
    np.savez_compressed(os.path.join(HERE, FIXTURE), **out)
    print(f"wrote {FIXTURE}", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    write()
