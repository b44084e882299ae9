"""SegResNetDS configurations shared by make_golden_segresnet_ds.py (reference side) and the tests.

FP32_CASES: tiny fp32 cases of the generic forward and the oracle, (constructor kwargs, input shape, weight seed); segresnet_ds.npz
keeps their full input and output.  KEY_CASES: the reference's own test configurations (tests/networks/nets/test_segresnet_ds.py),
whose state_dict keys and shapes segresnet_ds_state_dict_keys.json keeps.  TC_CASES[tag] is a tc_cases.Case of the fp16 tensor-core
forward; segresnet_ds_tc.npz has the layout of the other <net>_tc.npz fixtures (a strided sample of the input, a strided sample of the
output and the output's float64 sum)."""
from __future__ import annotations

import os

from tc_cases import Case, make_input

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = "segresnet_ds.npz"
TC_FIXTURE = "segresnet_ds_tc.npz"
KEYS = "segresnet_ds_state_dict_keys.json"

FP32_CASES = [
    # the reference's defaults (BatchNorm, ReLU, deconv, blocks (1,2,2,4)) at init 8
    (dict(init_filters=8), (1, 1, 16, 16, 16), 100),
    # 2-D, affine instance norm, LeakyReLU, trilinear upsampling with its 1x1 preconv
    (dict(spatial_dims=2, init_filters=8, norm=("instance", {"affine": True}), act="leakyrelu", upsample_mode="nontrainable"), (2, 1, 16, 16), 101),
    # anisotropic levels ([3,3,1] kernels, (2,2,1) strides), "instance_nvfuser", deep-supervision heads, 2 -> 3 channels
    (dict(init_filters=8, in_channels=2, out_channels=3, dsdepth=3, resolution=[1, 1, 5], norm="instance_nvfuser", blocks_down=(1, 2, 2)),
     (1, 2, 16, 16, 8), 102),
    # GroupNorm, trilinear upsampling, a non-cubic input
    (dict(init_filters=8, norm=("group", {"num_groups": 4}), upsample_mode="nontrainable", blocks_down=(1, 2, 2)), (1, 1, 16, 8, 12), 103),
    # no downsampling: the single head of the flat corner case
    (dict(init_filters=8, blocks_down=(2,), out_channels=3), (1, 1, 8, 8, 8), 104),
    # kernels with two axes of size 1 ([3,1,1] at level 1) and (2,1,1) strides
    (dict(init_filters=8, dsdepth=3, resolution=[1, 2, 5], blocks_down=(1, 1, 1, 1)), (1, 1, 16, 8, 8), 105),
]

KEY_CASES = [
    dict(spatial_dims=sd, init_filters=8, act=act, norm=norm, upsample_mode=up)
    for sd in (2, 3) for act in ("relu", "leakyrelu") for norm in ("BATCH", ("instance", {"affine": True})) for up in ("deconv", "nontrainable")
] + [
    dict(init_filters=8, dsdepth=2, resolution=None),
    dict(init_filters=8, dsdepth=3, resolution=None),
    dict(init_filters=8, dsdepth=3, resolution=[1, 1, 5]),
    dict(init_filters=8, dsdepth=3, resolution=[1, 2, 5]),
]

TC_CASES = {
    # A: the reference's defaults (init 32, BatchNorm, ReLU, deconv, blocks (1,2,2,4)) on two 64^3 windows
    "A": Case(dict(), (2, 1, 64, 64, 64), 110, 115, 4),
    # B: Auto3DSeg-style -- init 32, blocks (1,2,2,4,4), "instance_nvfuser", dsdepth 4, resolution (0.8, 0.8, 2.5) (level 0 kernel
    # [3,3,1], stride (2,2,1)), 4 -> 3 channels
    "B": Case(dict(init_filters=32, in_channels=4, out_channels=3, blocks_down=(1, 2, 2, 4, 4), norm="instance_nvfuser", dsdepth=4,
                   resolution=(0.8, 0.8, 2.5)), (1, 4, 64, 64, 32), 111, 116, 4),
    # C: resolution (4, 1, 1) (kernels [1,3,3] at levels 0 and 1), LeakyReLU 0.1, BatchNorm, 20 outputs (the > 16-channel head),
    # one input channel through the channel-padded one-plane stem
    "C": Case(dict(init_filters=16, out_channels=20, resolution=(4, 1, 1), act=("leakyrelu", {"negative_slope": 0.1}), blocks_down=(1, 2, 2)),
              (2, 1, 12, 32, 32), 112, 117, 4),
    # D: trilinear upsampling (1x1 preconv + x2), non-affine instance norm, init 16 on a non-cubic input
    "D": Case(dict(init_filters=16, out_channels=2, norm=("instance", {"affine": False}), upsample_mode="nontrainable"), (1, 1, 32, 48, 32),
              113, 118, 4),
}


def load_input(tag: str, npz=None):
    """The case's fp16 input (on the CPU) regenerated from its seed, checked against the sample the fixture keeps of the
    reference's input.  `npz`: the loaded fixture, read from segresnet_ds_tc.npz when not given."""
    import numpy as np

    case = TC_CASES[tag]
    g = npz if npz is not None else np.load(os.path.join(HERE, TC_FIXTURE))
    x = make_input(case.shape, case.xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x
