"""UNet configurations with residual units of the fp16 tensor-core forward, shared by make_golden_unet_res.py (reference side) and
the tests.

RES_CASES[tag] is a tc_cases.Case; the fixture unet_res_tc.npz has the layout of the other <net>_tc.npz fixtures (a strided sample
of the input, a strided sample of the output and the output's float64 sum)."""
from __future__ import annotations

import os

from tc_cases import Case, make_input

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = "unet_res_tc.npz"

RES_CASES = {
    # A: the spleen CT configuration of MONAI's tutorial and bundle -- 5 levels 16 ... 256, two residual units per level,
    # eval-mode BatchNorm, PReLU, 1 -> 2 channels; two 64^3 windows
    "A": Case(dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64, 128, 256), strides=(2, 2, 2, 2), num_res_units=2,
                   norm="batch"), (2, 1, 64, 64, 64), 20, 21, 4),
    # B: MONAI's default norm (InstanceNorm, PReLU) with two residual units, 4 input modalities, 3 outputs, a non-cubic input
    "B": Case(dict(spatial_dims=3, in_channels=4, out_channels=3, channels=(16, 32, 64, 128), strides=(2, 2, 2), num_res_units=2),
              (1, 4, 48, 64, 32), 22, 23, 4),
    # C: the other branches -- one residual unit, stride-1 levels (a 1x1x1 residual, an identity residual, stride-1 transposed
    # convolutions), affine InstanceNorm, LeakyReLU 0.1 and 20 outputs (the top runs padded to 32 channels)
    "C": Case(dict(spatial_dims=3, in_channels=1, out_channels=20, channels=(16, 32, 32, 64), strides=(2, 1, 1), num_res_units=1,
                   norm=("instance", {"affine": True}), act=("leakyrelu", {"negative_slope": 0.1})), (1, 1, 32, 40, 24), 24, 25, 4),
}


def load_input(tag: str, npz=None):
    """The case's fp16 input (on the CPU) regenerated from its seed, checked against the sample the fixture keeps of the
    reference's input.  `npz`: the loaded fixture, read from unet_res_tc.npz when not given."""
    import numpy as np

    case = RES_CASES[tag]
    g = npz if npz is not None else np.load(os.path.join(HERE, FIXTURE))
    x = make_input(case.shape, case.xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x
