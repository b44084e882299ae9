"""SegResNetDS on the CPU: the oracle against fixtures of the real reference, the module tree and state_dict keys of the reference's
configurations, the reference's helpers, the input check and which configurations the fp16 tensor-core forward implements."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
from segresnet_ds_cases import FIXTURE, FP32_CASES, KEY_CASES, KEYS, TC_CASES
from segresnet_ds_oracle import segresnet_ds_forward
from weights import fill_state_dict

from monai_b200.networks.blocks import UpSample
from monai_b200.networks.layers.factories import get_norm_layer
from monai_b200.networks.nets import SegResNetDS
from monai_b200.networks.nets.segresnet_ds import aniso_kernel, scales_for_resolution


def oracle_kw(kw: dict) -> dict:
    """segresnet_ds_forward's arguments for a constructor's kwargs."""
    norm = kw.get("norm", "batch")
    name, nkw = (norm, {}) if isinstance(norm, str) else norm
    name = {"instance_nvfuser": "instance"}.get(name.lower(), name.lower())
    act = kw.get("act", "relu")
    aname, akw = (act, {}) if isinstance(act, str) else act
    slope = None if aname.lower() == "relu" else akw.get("negative_slope", 0.01)
    return dict(blocks_down=kw.get("blocks_down", (1, 2, 2, 4)), norm=name, groups=nkw.get("num_groups", 8), eps=nkw.get("eps", 1e-5),
                slope=slope, upsample_mode=kw.get("upsample_mode", "deconv"), resolution=kw.get("resolution"))


def _keys(net):
    return {k: list(v.shape) for k, v in net.state_dict().items()}


def test_segresnet_ds_oracle_equals_the_reference(golden_dir):
    """The oracle reproduces the reference's fp32 outputs bit for bit (2-D and 3-D, BatchNorm / instance / group norm, deconv and
    trilinear upsampling, anisotropic levels, the flat corner case)."""
    g = np.load(os.path.join(golden_dir, FIXTURE))
    for i, (kw, shape, seed) in enumerate(FP32_CASES):
        net = SegResNetDS(**kw)
        net.load_state_dict(fill_state_dict(net.state_dict(), seed))
        x = torch.from_numpy(g[f"c{i}.x"])
        assert tuple(x.shape) == shape
        with torch.no_grad():
            y = segresnet_ds_forward(net.state_dict(), x, **oracle_kw(kw))
        np.testing.assert_array_equal(y.numpy(), g[f"c{i}.y"], err_msg=str(kw))


@pytest.mark.parametrize("group", ["c", "k", "tc"])
def test_segresnet_ds_module_tree_matches_the_reference(golden_dir, group):
    want = json.load(open(os.path.join(golden_dir, KEYS)))
    cases = {"c": {f"c{i}": c[0] for i, c in enumerate(FP32_CASES)}, "k": {f"k{i}": kw for i, kw in enumerate(KEY_CASES)},
             "tc": {f"tc{t}": c.kw for t, c in TC_CASES.items()}}[group]
    for key, kw in cases.items():
        assert _keys(SegResNetDS(**kw)) == want[key], kw


def test_segresnet_ds_submodules_match_the_reference():
    net = SegResNetDS(init_filters=8, dsdepth=2, resolution=[1, 1, 5])
    assert isinstance(net.encoder.conv_init, nn.Conv3d) and tuple(net.encoder.conv_init.kernel_size) == (3, 3, 1)
    assert tuple(net.encoder.layers[0].downsample.stride) == (2, 2, 1) and isinstance(net.encoder.layers[3].downsample, nn.Identity)
    up = net.up_layers[2].upsample.deconv
    assert (tuple(up.kernel_size), tuple(up.stride), tuple(up.padding), tuple(up.output_padding)) == ((3, 3, 1), (2, 2, 1), (1, 1, 0), (1, 1, 0))
    assert [isinstance(l["head"], nn.Identity) for l in net.up_layers] == [True, False, False]
    blk = net.encoder.layers[0].blocks[0]
    assert isinstance(blk.norm1, nn.BatchNorm3d) and blk.norm1.affine and blk.act1.inplace
    assert not get_norm_layer(("instance", {}), 3, 8).affine and SegResNetDS(norm="instance").encoder.layers[0].blocks[0].norm1.affine
    assert not SegResNetDS(norm=("instance", {"affine": False})).encoder.layers[0].blocks[0].norm1.affine
    assert type(SegResNetDS(norm="instance_nvfuser").encoder.layers[0].blocks[0].norm1) is nn.InstanceNorm3d
    assert type(get_norm_layer("instance_nvfuser", 2, 8)) is nn.InstanceNorm2d
    flat = SegResNetDS(init_filters=8, blocks_down=(1,))
    assert len(flat.up_layers) == 1 and isinstance(flat.up_layers[0]["upsample"], nn.Identity)
    nt = SegResNetDS(init_filters=8, upsample_mode="nontrainable").up_layers[0].upsample
    assert [n for n, _ in nt.named_children()] == ["preconv", "upsample_non_trainable"] and nt.preconv.bias is None


def test_segresnet_upsample_is_unchanged():
    """SegResNet's UpSample (no kernel_size, scalar scale, in == out channels) keeps its module tree."""
    d = UpSample(3, 16, 16, 2, mode="deconv")
    assert (tuple(d.deconv.kernel_size), tuple(d.deconv.stride), tuple(d.deconv.padding), tuple(d.deconv.output_padding)) == ((2,) * 3, (2,) * 3, (0,) * 3, (0,) * 3)
    n = UpSample(3, 16, 16, 2, mode="nontrainable")
    assert [k for k, _ in n.named_children()] == ["upsample_non_trainable"] and n.upsample_non_trainable.scale_factor == 2.0


def test_segresnet_ds_helpers_follow_the_reference():
    # the reference's tests/networks/nets/test_segresnet_ds.py: output sizes of the deep-supervision levels follow these scales
    assert scales_for_resolution([1, 1, 5], 5) == [(2, 2, 1), (2, 2, 1), (2, 2, 2), (2, 2, 2), (2, 2, 2)]
    assert scales_for_resolution([1, 2, 5]) == [(2, 2, 1), (2, 1, 1)]
    assert scales_for_resolution((0.8, 0.8, 2.5), 5)[0] == (2, 2, 1)
    with pytest.raises(ValueError, match="positive"):
        scales_for_resolution([1, 0, 1])
    assert aniso_kernel((2, 2, 1)) == ([3, 3, 1], [1, 1, 0], (2, 2, 1))
    net = SegResNetDS(init_filters=8, resolution=[1, 2, 5])
    assert [int(v) for v in net.shape_factor()] == [8, 4, 2]
    assert SegResNetDS(init_filters=8).shape_factor() == [8, 8, 8]
    assert net.is_valid_shape(torch.zeros(1, 1, 16, 8, 6)) and not net.is_valid_shape(torch.zeros(1, 1, 16, 8, 5))
    with pytest.raises(TypeError, match="tuple"):
        SegResNetDS(resolution=1.0)
    with pytest.raises(ValueError, match="positive"):
        SegResNetDS(resolution=(1.0, -1.0, 1.0))


def test_segresnet_ds_rejects_bad_shapes_before_any_launch():
    """The reference's divisibility check (and its message) and the channel check run before either path touches a kernel."""
    net = SegResNetDS(init_filters=16).eval()
    with pytest.raises(ValueError, match=r"Input spatial dims .* must be divisible by \[8, 8, 8\]"):
        net(torch.zeros(1, 1, 16, 16, 12))
    with pytest.raises(ValueError, match="expects an"):
        net(torch.zeros(1, 2, 16, 16, 16))
    seen = []
    pre = SegResNetDS(init_filters=16, preprocess=lambda t: seen.append(t.shape) or t[..., :12]).eval()
    with pytest.raises(ValueError, match="divisible"):
        pre(torch.zeros(1, 1, 16, 16, 16))
    assert seen == [(1, 1, 16, 16, 16)]   # preprocess runs first
    ds = SegResNetDS(init_filters=16, dsdepth=2, norm="instance").train()
    with pytest.raises(RuntimeError, match="inference-only"):
        ds(torch.zeros(1, 1, 16, 16, 16))


@pytest.mark.parametrize("kw,ok", [
    (TC_CASES["A"].kw, True),                                           # the reference defaults
    (TC_CASES["B"].kw, True),                                           # Auto3DSeg-style, [3,3,1] at level 0
    (TC_CASES["C"].kw, True),                                           # [1,3,3] kernels, LeakyReLU 0.1, BatchNorm, 20 outputs
    (TC_CASES["D"].kw, True),                                           # trilinear, non-affine instance norm
    (dict(norm=("group", {"num_groups": 8})), True),
    (dict(resolution=[1, 1, 5]), True),                                 # [3,3,1] at two levels
    (dict(act=("leakyrelu", {"negative_slope": 1.0})), True),
    (dict(blocks_down=(2,)), True),                                     # no downsampling: blocks and the head
    (dict(resolution=[1, 2, 5]), False),                                # level 1: [3,1,1], two axes of size 1
    (dict(upsample_mode="nontrainable", resolution=[1, 1, 5]), False),  # anisotropic trilinear upsampling
    (dict(init_filters=8), False),
    (dict(init_filters=24), False),
    (dict(spatial_dims=2), False),
    (dict(act="prelu"), False),
    (dict(act="gelu"), False),
    (dict(act=("leakyrelu", {"negative_slope": 1.5})), False),
    (dict(norm=("batch", {"track_running_stats": False})), False),
    (dict(norm=("instance", {"track_running_stats": True})), False),
    (dict(blocks_down=(1, 2, 2), blocks_up=(1, 1, 1)), False),          # blocks_up longer than the decoder
    (dict(upsample_mode="pixelshuffle"), None),                         # not a mode this package builds
])
def test_segresnet_ds_tc_eligibility(kw, ok):
    if ok is None:
        with pytest.raises(NotImplementedError):
            SegResNetDS(**kw)
        return
    assert SegResNetDS(**kw)._tc_ok is ok
