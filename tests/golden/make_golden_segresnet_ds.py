"""Generate the SegResNetDS fixtures from the REAL reference (Project-MONAI/MONAI on PYTHONPATH):

    PYTHONPATH=<MONAI source checkout> python tests/golden/make_golden_segresnet_ds.py

segresnet_ds.npz: the full input and eval-mode output of each fp32 case of segresnet_ds_cases.py.  segresnet_ds_state_dict_keys.json:
state_dict keys and shapes of the fp32, key and tensor-core cases.  segresnet_ds_tc.npz: the tensor-core cases in the layout of
make_golden_tc.py (the reference runs in fp32, eval mode, on the fp16-rounded input).  Weights come from weights.fill_state_dict.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from monai.networks.nets import SegResNetDS  # noqa: E402
from segresnet_ds_cases import FIXTURE, FP32_CASES, KEY_CASES, KEYS, TC_CASES, TC_FIXTURE  # noqa: E402
from tc_cases import X_STRIDE, make_input  # noqa: E402
from weights import fill_state_dict  # noqa: E402


def _net(kw, seed=None):
    net = SegResNetDS(**kw)
    if seed is not None:
        net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval()


def _keys(net):
    return {k: list(v.shape) for k, v in net.state_dict().items()}


def write() -> None:
    keys, out = {}, {}
    for i, (kw, shape, seed) in enumerate(FP32_CASES):
        net = _net(kw, seed)
        x = torch.randn(shape, generator=torch.Generator().manual_seed(seed + 1000))
        with torch.no_grad():
            y = net(x)
        out[f"c{i}.x"], out[f"c{i}.y"] = x.numpy(), y.numpy()
        keys[f"c{i}"] = _keys(net)
    np.savez_compressed(os.path.join(HERE, FIXTURE), **out)
    for i, kw in enumerate(KEY_CASES):
        keys[f"k{i}"] = _keys(_net(kw))
    tc = {}
    for tag, (kw, shape, seed, xseed, s) in TC_CASES.items():
        net = _net(kw, seed)
        keys[f"tc{tag}"] = _keys(net)
        x = make_input(shape, xseed)
        with torch.no_grad():
            y = net(x.float())
        tc[f"{tag}.x_sub"] = x.numpy()[..., ::X_STRIDE, ::X_STRIDE, ::X_STRIDE]
        tc[f"{tag}.x_stride"] = np.array(X_STRIDE)
        tc[f"{tag}.y_sub"] = y.numpy()[..., ::s, ::s, ::s]
        tc[f"{tag}.y_stride"] = np.array(s)
        tc[f"{tag}.y_sum"] = np.array(float(y.double().sum()))
    np.savez_compressed(os.path.join(HERE, TC_FIXTURE), **tc)
    with open(os.path.join(HERE, KEYS), "w") as f:
        json.dump(keys, f, separators=(",", ":"))
    print(f"wrote {FIXTURE}, {TC_FIXTURE}, {KEYS}")


if __name__ == "__main__":
    write()
