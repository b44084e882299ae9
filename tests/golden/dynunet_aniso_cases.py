"""Anisotropic DynUNet plans of the fp16 tensor-core forward, shared by make_golden_dynunet_aniso.py (reference side) and the tests.

ANISO_CASES[tag] is a tc_cases.Case; the fixture dynunet_aniso_tc.npz has the layout of the other <net>_tc.npz fixtures (a strided
sample of the input, a strided sample of the output and the output's float64 sum)."""
from __future__ import annotations

import os

from tc_cases import Case, make_input

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = "dynunet_aniso_tc.npz"

ANISO_CASES = {
    # A: an nnU-Net-style anisotropic plan (kernel 1 along D at the two high-resolution levels, no D stride there), default filters
    # 32 ... 320 and affine instance norm, on two thick-slice windows; 2 x 3 x 4 x 16 x 16 output values
    "A": Case(dict(spatial_dims=3, in_channels=1, out_channels=3, kernel_size=[[1, 3, 3], [1, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
                   strides=[[1, 1, 1], [1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2], [1, 2, 2]],
                   upsample_kernel_size=[[1, 2, 2], [1, 2, 2], [2, 2, 2], [2, 2, 2], [1, 2, 2]]),
              (2, 1, 16, 64, 64), 32, 42, 4),
    # B: MONAI-style, kernel 1 along W -- several input channels, residual blocks (strided conv3 + affine norm3), transposed-conv
    # bias, deep-supervision heads (parameters only in eval mode), eps 1e-4, LeakyReLU 0.1
    "B": Case(dict(spatial_dims=3, in_channels=2, out_channels=4, kernel_size=[[3, 3, 1], [3, 3, 1], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
                   strides=[[1, 1, 1], [2, 2, 1], [2, 2, 1], [2, 2, 2], [2, 2, 2]], upsample_kernel_size=[[2, 2, 1], [2, 2, 1], [2, 2, 2], [2, 2, 2]],
                   filters=[16, 32, 64, 128, 256], res_block=True, trans_bias=True, deep_supervision=True, deep_supr_num=2,
                   norm_name=("instance", {"affine": True, "eps": 1e-4}), act_name=("leakyrelu", {"inplace": True, "negative_slope": 0.1})),
              (1, 2, 48, 32, 16), 33, 43, 4),
    # C: kernel 1 along H, stride 1 along H at level 1, residual blocks, non-affine instance norm
    "C": Case(dict(spatial_dims=3, in_channels=1, out_channels=2, kernel_size=[[3, 1, 3], [3, 3, 3], [3, 3, 3], [3, 3, 3]],
                   strides=[[1, 1, 1], [2, 1, 2], [2, 2, 2], [2, 2, 2]], upsample_kernel_size=[[2, 1, 2], [2, 2, 2], [2, 2, 2]],
                   filters=[16, 32, 48, 64], res_block=True, norm_name=("instance", {"affine": False})),
              (1, 1, 32, 16, 32), 34, 44, 4),
}


def load_input(tag: str, npz=None):
    """The case's fp16 input (on the CPU) regenerated from its seed, checked against the sample the fixture keeps of the
    reference's input.  `npz`: the loaded fixture, read from dynunet_aniso_tc.npz when not given."""
    import numpy as np

    case = ANISO_CASES[tag]
    g = npz if npz is not None else np.load(os.path.join(HERE, FIXTURE))
    x = make_input(case.shape, case.xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x
