"""Generate tests/golden/<net>_tc.npz from the REAL reference (Project-MONAI/MONAI on PYTHONPATH):

    PYTHONPATH=<MONAI source checkout> python tests/golden/make_golden_tc.py [unetr|dynunet|segresnet ...]   (default: all three)

The configurations of the fp16 tensor-core paths (tc_cases.py).  The input is regenerated from its seed by the tests, so the
fixture stores only a strided sample of it (to prove both sides saw the same values); the reference runs in fp32 on the
fp16-rounded input.  The output is stored subsampled with a per-case stride, plus its float64 sum over the whole volume.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from monai.networks.nets import UNETR, DynUNet, SegResNet  # noqa: E402
from tc_cases import TC_CASES, X_STRIDE, make_input  # noqa: E402
from weights import fill_state_dict  # noqa: E402

NETS = {"unetr": UNETR, "dynunet": DynUNet, "segresnet": SegResNet}


def write(name: str) -> None:
    out = {}
    for tag, (kw, shape, seed, xseed, s) in TC_CASES[name].items():
        net = NETS[name](**kw)
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
    np.savez_compressed(os.path.join(HERE, f"{name}_tc.npz"), **out)
    print(f"wrote {name}_tc.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    for name in sys.argv[1:] or NETS:
        write(name)
