"""Generate tests/golden/dynunet_tc.npz from the REAL reference (Project-MONAI/MONAI on PYTHONPATH):

    PYTHONPATH=<MONAI source checkout> python tests/golden/make_golden_dynunet_tc.py

DynUNet configurations of the fp16 tensor-core path (dynunet_tc_cases.py).  The input is regenerated from its seed by the tests, so
the fixture stores only a strided sample of it (to prove both sides saw the same values); the reference runs in fp32 on the
fp16-rounded input.  The output is stored subsampled with a per-case stride, plus its float64 sum over the whole volume.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from monai.networks.nets import DynUNet  # noqa: E402
from dynunet_tc_cases import DYNUNET_TC_CASES, make_input  # noqa: E402
from weights import fill_state_dict  # noqa: E402

X_STRIDE = 8                 # input sample: x[..., ::8, ::8, ::8]
Y_STRIDE = {"A": 4, "B": 4}  # output sample: y[..., ::s, ::s, ::s] (case A: 2 x 3 x 16^3 values)


def main() -> None:
    out = {}
    for tag, (kw, shape, seed, xseed) in DYNUNET_TC_CASES.items():
        net = DynUNet(**kw)
        net.load_state_dict(fill_state_dict(net.state_dict(), seed))
        net.eval()
        x = make_input(shape, xseed)
        with torch.no_grad():
            y = net(x.float())
        s = Y_STRIDE[tag]
        out[f"{tag}.x_sub"] = x.numpy()[..., ::X_STRIDE, ::X_STRIDE, ::X_STRIDE]
        out[f"{tag}.x_stride"] = np.array(X_STRIDE)
        out[f"{tag}.y_sub"] = y.numpy()[..., ::s, ::s, ::s]
        out[f"{tag}.y_stride"] = np.array(s)
        out[f"{tag}.y_sum"] = np.array(float(y.double().sum()))
    np.savez_compressed(os.path.join(HERE, "dynunet_tc.npz"), **out)
    print("wrote dynunet_tc.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
