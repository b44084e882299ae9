"""GPU parity of the monai_b200 networks (CUDA kernels) vs the reference fixtures and the CPU oracle."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from monai_b200.inferers import sliding_window_inference
from monai_b200.networks.nets import BasicUNet, UNet
from oracle import networks as onet
from oracle import sliding_window as osw
from weights import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _build(factory, seed):
    with contextlib.redirect_stdout(io.StringIO()):
        net = factory()
    net.load_state_dict(fill_state_dict(net.state_dict(), seed))
    return net.eval().to(DEV)


@pytest.mark.parametrize(
    "name,seed,args,kw",
    [
        ("unet_tiny.npz", 0, (3, 1, 2, (4, 8, 16), (2, 2)), {}),
        ("unet_c2_32.npz", 1, (3, 1, 2, (16, 32, 64, 128, 256), (2, 2, 2, 2)), {}),
        ("unet_res.npz", 2, (3, 2, 3, (4, 8, 8), (2, 1)), {"num_res_units": 2}),
    ],
)
def test_unet_matches_reference_fixture(golden_dir, name, seed, args, kw):
    g = np.load(os.path.join(golden_dir, name))
    net = _build(lambda: UNet(*args, **kw), seed)
    y = net(torch.from_numpy(g["x"]).to(DEV))
    ref = g["y"]
    err = np.abs(y.cpu().numpy() - ref).max() / max(1e-6, np.abs(ref).max())
    assert err < 1e-3, f"{name}: relative error {err}"  # north-star tolerance for fp32 conv: 1e-3 rel


def test_unet_fp16_close_to_fp32_oracle():
    net = _build(lambda: UNet(3, 1, 2, (16, 32, 64, 128, 256), (2, 2, 2, 2)), 1)
    x = torch.randn(2, 1, 32, 32, 32, generator=torch.Generator().manual_seed(3))
    ref = onet.unet_forward({k: v.float().cpu() for k, v in net.state_dict().items()}, x, (2, 2, 2, 2)).numpy()
    y = net.half()(x.to(DEV).half()).float().cpu().numpy()
    err = np.abs(y - ref).max() / np.abs(ref).max()
    assert err < 3e-2, err  # fp16 storage between layers, fp32 accumulation
    assert (y.argmax(1) == ref.argmax(1)).mean() > 0.98


def test_config_c1_style_sliding_window_unet_fp32_vs_oracle():
    """sliding_window_inference + UNet end to end (C1-shaped: 64^3 fp32, roi 32^3, overlap 0.25) vs the CPU oracle."""
    net = _build(lambda: UNet(3, 1, 2, (8, 16, 32), (2, 2)), 7)
    sd = {k: v.float().cpu() for k, v in net.state_dict().items()}
    x = torch.randn(1, 1, 64, 64, 64, generator=torch.Generator().manual_seed(4))
    want = osw.sliding_window_inference(x.numpy(), (32, 32, 32), 4, lambda a: onet.unet_forward(sd, torch.from_numpy(a), (2, 2)).numpy(), 0.25, "constant")
    got = sliding_window_inference(x.to(DEV), (32, 32, 32), 4, net, 0.25, "constant")
    err = np.abs(got.cpu().numpy() - want).max() / np.abs(want).max()
    assert err < 1e-3, err


def test_basic_unet_matches_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "basic_unet_tiny.npz"))
    net = _build(lambda: BasicUNet(3, 1, 2, features=(4, 4, 8, 8, 16, 4)), 3)
    y = net(torch.from_numpy(g["x"]).to(DEV))
    err = np.abs(y.cpu().numpy() - g["y"]).max() / np.abs(g["y"]).max()
    assert err < 1e-3, err
    # odd input size exercises the replicate-pad branch of UpCat (basic_unet.py:165-170)
    x = torch.randn(1, 1, 36, 40, 44, generator=torch.Generator().manual_seed(9))
    ref = onet.basic_unet_forward({k: v.float().cpu() for k, v in net.state_dict().items()}, x).numpy()
    y = net(x.to(DEV)).cpu().numpy()
    assert np.abs(y - ref).max() / np.abs(ref).max() < 1e-3


def test_unet_tensor_core_path_matches_direct_path(monkeypatch):
    """fp16 UNet (C2 topology): wgmma im2col path (NC8, CUDA-graph replay) vs the CUDA-core NCDHW path."""
    net = _build(lambda: UNet(3, 1, 2, (16, 32, 64, 128, 256), (2, 2, 2, 2)), 1).half()
    x = torch.randn(3, 1, 32, 48, 64, generator=torch.Generator().manual_seed(5)).to(DEV).half()
    assert net._tc_eligible(x)
    a = net(x).float()
    a2 = net(x).float()  # second call replays the captured graph
    torch.testing.assert_close(a, a2, rtol=1e-2, atol=1e-2)  # InstanceNorm sums use float atomics: last-bit differences
    monkeypatch.setenv("MONAI_B200_UNET_TC", "0")
    assert not net._tc_eligible(x)
    b = net(x).float()
    err = float((a - b).abs().max() / b.abs().max())
    assert err < 2e-2, err
    ref = onet.unet_forward({k: v.float().cpu() for k, v in net.state_dict().items()}, x.float().cpu(), (2, 2, 2, 2))
    assert float((a.cpu() - ref).abs().max() / ref.abs().max()) < 3e-2
