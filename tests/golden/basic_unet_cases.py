"""BasicUNet configurations of the fp16 tensor-core forward, shared by make_golden_basic_unet.py (reference side) and the tests.

BASIC_CASES[tag] is a tc_cases.Case; the fixture basic_unet_tc.npz has the layout of the other <net>_tc.npz fixtures (a strided
sample of the input, a strided sample of the output and the output's float64 sum)."""
from __future__ import annotations

import os

from tc_cases import Case, make_input

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = "basic_unet_tc.npz"

BASIC_CASES = {
    # A: the reference's defaults (features 32, 32, 64, 128, 256, 32, affine instance norm, LeakyReLU 0.1) on two 64^3 windows
    "A": Case(dict(), (2, 1, 64, 64, 64), 70, 75, 4),
    # B: several input channels, other widths (a 48-channel upcat_1), non-affine instance norm, ReLU, no convolution bias and a
    # non-cubic input
    "B": Case(dict(in_channels=4, out_channels=3, features=(16, 32, 64, 128, 256, 48), norm="instance", act="relu", bias=False),
              (1, 4, 32, 64, 48), 71, 76, 4),
    # C: 20 outputs (the > 16-channel head), dropout 0.1 (eval), LeakyReLU 0.01 and norm eps 1e-4 on one 32^3 window (C1's roi:
    # the bottom level is 2^3)
    "C": Case(dict(out_channels=20, dropout=0.1, act=("leakyrelu", {"negative_slope": 0.01}), norm=("instance", {"affine": True, "eps": 1e-4})),
              (1, 1, 32, 32, 32), 72, 77, 4),
}


def load_input(tag: str, npz=None):
    """The case's fp16 input (on the CPU) regenerated from its seed, checked against the sample the fixture keeps of the
    reference's input.  `npz`: the loaded fixture, read from basic_unet_tc.npz when not given."""
    import numpy as np

    case = BASIC_CASES[tag]
    g = npz if npz is not None else np.load(os.path.join(HERE, FIXTURE))
    x = make_input(case.shape, case.xseed)
    s = int(g[f"{tag}.x_stride"])
    assert np.array_equal(x.numpy()[..., ::s, ::s, ::s], g[f"{tag}.x_sub"]), "regenerated input differs from the reference's"
    return x
