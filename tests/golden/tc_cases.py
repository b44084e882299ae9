"""Fixture cases of the fp16 tensor-core forwards, shared by make_golden_tc.py (reference side) and the tests.

TC_CASES[net][tag] is a `Case`.  The input is regenerated from its seed on both sides; the fixture `<net>_tc.npz` keeps a
strided sample of it (to prove the two agree), a strided sample of the output and the output's float64 sum."""
from __future__ import annotations

import os
from typing import NamedTuple

HERE = os.path.dirname(os.path.abspath(__file__))
X_STRIDE = 8   # input sample: x[..., ::8, ::8, ::8]


class Case(NamedTuple):
    kw: dict            # constructor kwargs
    shape: tuple        # input shape
    seed: int           # weight seed (weights.fill_state_dict)
    xseed: int          # input seed (make_input)
    y_stride: int       # output sample: y[..., ::s, ::s, ::s]


TC_CASES = {
    "unetr": {
        # A: the reference's defaults (ViT-B: hidden 768, 12 heads of 64, mlp 3072; feature_size 16) on one 96^3 window, batch 2;
        # 2 x 14 x 12^3 output values
        "A": Case(dict(in_channels=1, out_channels=14, img_size=96), (2, 1, 96, 96, 96), 80, 90, 8),
        # B: the other branches -- several input channels, qkv bias, a second feature size, 6 heads of 64 and a non-cubic
        # 4 x 4 x 3 token grid (48 tokens)
        "B": Case(dict(in_channels=4, out_channels=3, img_size=(64, 64, 48), feature_size=32, hidden_size=384, num_heads=6, mlp_dim=1536,
                       qkv_bias=True), (1, 4, 64, 64, 48), 81, 91, 4),
    },
    "dynunet": {
        # A: the nnU-Net default plan (6 levels, filters 32 ... 320, affine instance norm, LeakyReLU 0.01) on two 64^3 windows;
        # 2 x 3 x 16^3 output values
        "A": Case(dict(spatial_dims=3, in_channels=1, out_channels=3, kernel_size=[3] * 6, strides=[1, 2, 2, 2, 2, 2], upsample_kernel_size=[2] * 5),
                  (2, 1, 64, 64, 64), 30, 40, 4),
        # B: the other branches -- several input channels, residual blocks (strided conv3 + affine norm3), transposed-conv bias,
        # deep-supervision heads (parameters only in eval mode), eps 1e-4, LeakyReLU 0.1 and a non-cubic input
        "B": Case(dict(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[3] * 5, strides=[1, 2, 2, 2, 2], upsample_kernel_size=[2] * 4,
                       filters=[16, 48, 96, 192, 320], res_block=True, trans_bias=True, deep_supervision=True, deep_supr_num=2,
                       norm_name=("instance", {"affine": True, "eps": 1e-4}), act_name=("leakyrelu", {"inplace": True, "negative_slope": 0.1})),
                  (1, 4, 48, 64, 32), 31, 41, 4),
    },
    "segresnet": {
        # A: BraTS-style -- init 16, 4 input modalities, 3 outputs, GroupNorm(8), ReLU, trilinear upsampling, blocks (1,2,2,4) / (1,1,1)
        "A": Case(dict(spatial_dims=3, init_filters=16, in_channels=4, out_channels=3), (2, 4, 32, 32, 32), 50, 60, 4),
        # B: whole-body-CT-style -- init 32, one input channel, 105 outputs (the > 16-channel head), GroupNorm(8), dropout 0.2 (eval);
        # 105 x 7^3 output values
        "B": Case(dict(spatial_dims=3, init_filters=32, in_channels=1, out_channels=105, norm=("GROUP", {"num_groups": 8}), dropout_prob=0.2),
                  (1, 1, 32, 32, 32), 51, 61, 5),
        # C: the other branches -- transposed-convolution upsampling, affine instance norm, LeakyReLU 0.1, two input channels and a
        # non-cubic input
        "C": Case(dict(spatial_dims=3, init_filters=16, in_channels=2, out_channels=4, blocks_down=(1, 2, 2), blocks_up=(1, 1), upsample_mode="deconv",
                       norm=("instance", {"affine": True}), act=("leakyrelu", {"negative_slope": 0.1})),
                  (1, 2, 24, 32, 16), 52, 62, 4),
    },
}


def make_input(shape, seed):
    """The fp16 input of a case: a seeded CPU torch.randn rounded to fp16."""
    import torch

    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).half()


def load_input(net: str, tag: str, npz=None):
    """The case's fp16 input (on the CPU) regenerated from its seed, checked against the sample the fixture keeps of the
    reference's input.  `npz`: the loaded fixture, read from `<net>_tc.npz` when not given."""
    import numpy as np

    case = TC_CASES[net][tag]
    g = npz if npz is not None else np.load(os.path.join(HERE, f"{net}_tc.npz"))
    x = make_input(case.shape, case.xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x
