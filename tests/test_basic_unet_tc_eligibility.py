"""Which BasicUNet configurations the fp16 tensor-core forward implements (`_tc_ok`, decided at construction; CPU only)."""
import pytest
from basic_unet_cases import BASIC_CASES

from monai_b200.networks.nets import BasicUNet

TC = BASIC_CASES
FEA = (32, 32, 64, 128, 256, 32)


@pytest.mark.parametrize("kw,ok", [
    (TC["A"][0], True),                                                     # the reference defaults
    (TC["B"][0], True),                                                     # 4 -> 3, non-affine norm, ReLU, no bias
    (TC["C"][0], True),                                                     # 20 outputs, dropout, LeakyReLU 0.01, eps 1e-4
    (dict(in_channels=3, out_channels=40), True),
    (dict(features=(16, 16, 32, 64, 128, 16)), True),
    (dict(act=("leakyrelu", {"negative_slope": 1.0})), True),
    (dict(features=(16, 16, 48, 96, 192, 16)), False),                     # upcat_3's upsampled half would have 24 channels
    (dict(features=(16, 16, 64, 96, 176, 16)), False),                     # upcat_4's: 88
    (dict(features=(24, 32, 64, 128, 256, 32)), False),
    (dict(features=(32, 32, 64, 128, 256, 40)), False),
    (dict(norm="batch"), False),
    (dict(norm=("group", {"num_groups": 8})), False),
    (dict(norm=("instance", {"track_running_stats": True})), False),
    (dict(act="prelu"), False),
    (dict(act=("leakyrelu", {"negative_slope": 1.5})), False),
    (dict(act=("leakyrelu", {"negative_slope": -0.1})), False),
    (dict(act="gelu"), False),
])
def test_basic_unet_tc_eligibility(kw, ok):
    assert BasicUNet(**kw)._tc_ok is ok


def test_basic_unet_dropout_follows_train_and_eval_mode():
    net = BasicUNet(**TC["C"][0])
    assert net._tc_ok
    assert net._dropout_active()
    assert not net.eval()._dropout_active()
    assert net.train()._dropout_active()
    assert not BasicUNet()._dropout_active()   # dropout 0.0 is the identity in either mode


def test_basic_unet_keeps_the_reference_module_tree():
    net = BasicUNet(features=FEA)
    keys = list(net.state_dict())
    assert keys[0] == "conv_0.conv_0.conv.weight" and keys[-1] == "final_conv.bias"
    assert "down_1.convs.conv_1.adn.N.weight" in keys and "upcat_4.upsample.deconv.weight" in keys
    assert not any(k.startswith("_") for k in keys)
