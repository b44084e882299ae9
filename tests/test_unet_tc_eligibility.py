"""Which UNet configurations the fp16 tensor-core forward implements (`_tc_eligible`, the module checks of `_use_tc`), and the
eval-mode BatchNorm fold of the residual forward, in float64 (CPU only)."""
import pytest
import torch
import torch.nn as nn
from unet_res_cases import RES_CASES
from weights import fill_state_dict

from monai_b200.networks.nets import UNet

TC = RES_CASES
SPLEEN = TC["A"][0]
DEFAULT = TC["B"][0]


def _net(kw):
    return UNet(**kw).eval()


@pytest.mark.parametrize("kw,ok", [
    (TC["A"][0], True),                                                  # spleen: BatchNorm (eval), PReLU, 1 -> 2
    (TC["B"][0], True),                                                  # InstanceNorm, 4 -> 3, two residual units
    (TC["C"][0], True),                                                  # one unit, stride-1 levels, affine IN, LeakyReLU, 20 outputs
    (dict(DEFAULT, num_res_units=1, act="relu"), True),
    (dict(DEFAULT, num_res_units=3, dropout=0.2), True),                 # dropout: the identity in eval mode
    (dict(SPLEEN, norm=("batch", {"affine": False})), True),
    (dict(DEFAULT, out_channels=4, norm=("group", {"num_groups": 4})), False),
    (dict(DEFAULT, adn_ordering="ADN"), False),
    (dict(DEFAULT, kernel_size=5), False),
    (dict(DEFAULT, up_kernel_size=5), False),
    (dict(DEFAULT, channels=(16, 24, 64, 128)), False),                  # 24 is not a multiple of 16
    (dict(DEFAULT, strides=(2, 3, 2)), False),
    (dict(DEFAULT, spatial_dims=2), False),
    (dict(DEFAULT, norm=("instance", {"track_running_stats": True})), False),
    (dict(DEFAULT, act="gelu"), False),
    (dict(DEFAULT, norm=None), False),
    (dict(DEFAULT, act=("prelu", {"num_parameters": 16})), False),
])
def test_unet_res_tc_eligibility(kw, ok):
    assert _net(kw)._tc_eligible() is ok


def test_unet_res_tc_eligibility_follows_the_module_modes():
    net = _net(SPLEEN)
    assert net._tc_eligible()
    assert not net.train()._tc_eligible()            # BatchNorm in training mode: the generic path, which rejects it
    drop = _net(dict(DEFAULT, dropout=0.2))
    assert drop._tc_eligible()
    assert not drop.train()._tc_eligible()           # active dropout


@pytest.mark.parametrize("kw,ok", [
    (dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64, 128, 256), strides=(2, 2, 2, 2)), True),   # C2
    (dict(spatial_dims=3, in_channels=2, out_channels=2, channels=(16, 32, 64), strides=(2, 2)), False),
    (dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64), strides=(2, 2), norm="batch"), False),
    (dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64), strides=(2, 2), dropout=0.1), False),
    (dict(spatial_dims=3, in_channels=1, out_channels=2, channels=(16, 32, 64), strides=(2, 2), norm=("instance", {"affine": True})), False),
])
def test_unet_plain_tc_eligibility_is_unchanged(kw, ok):
    assert _net(kw)._tc_eligible() is ok


def _bn_block(net, transposed):
    """A Convolution block with a BatchNorm: the down unit0 of level 0, or the transposed convolution of the top up layer."""
    return net.model[2][0] if transposed else net.model[0].conv.unit0


@pytest.mark.parametrize("transposed", [False, True], ids=["conv", "transposed"])
@pytest.mark.parametrize("affine", [True, False])
def test_unet_bn_fold_matches_conv_then_batchnorm_float64(transposed, affine):
    norm = "batch" if affine else ("batch", {"affine": False})
    net = UNet(**dict(SPLEEN, channels=(16, 32, 64), strides=(2, 2), norm=norm))
    net.load_state_dict(fill_state_dict(net.state_dict(), 5))
    net = net.eval().double()
    blk = _bn_block(net, transposed)
    bn = blk.adn.N
    assert isinstance(bn, nn.BatchNorm3d) and bn.running_var.min() > 0 and bn.running_mean.abs().max() > 0
    if affine:
        assert bn.bias.abs().max() > 0
    m = blk.conv
    x = torch.randn(2, m.in_channels, 6, 7, 5, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    with torch.no_grad():
        ref = bn(m(x))
        w, b = net._folded(blk)
        f = nn.functional.conv_transpose3d if transposed else nn.functional.conv3d
        kw = dict(stride=m.stride, padding=m.padding) | (dict(output_padding=m.output_padding) if transposed else {})
        got = f(x, w.double(), b.double(), **kw)
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), float((got - ref).abs().max())
    # zero-padded output channels carry zero weight and bias
    wp, bp = net._folded(blk, cout_pad=48)
    ax = 1 if transposed else 0
    assert torch.equal(wp.narrow(ax, 0, w.shape[ax]), w) and not wp.narrow(ax, w.shape[ax], 48 - w.shape[ax]).any()
    assert torch.equal(bp[: b.numel()], b) and not bp[b.numel():].any()
