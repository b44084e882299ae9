"""Which SegResNet configurations the fp16 tensor-core forward implements (`_tc_ok`, decided at construction; CPU only)."""
import pytest
from tc_cases import TC_CASES

from monai_b200.networks.nets import SegResNet

TC = TC_CASES["segresnet"]
BRATS = TC["A"][0]


@pytest.mark.parametrize("kw,ok", [
    (TC["A"][0], True),                                                     # BraTS-style
    (TC["B"][0], True),                                                     # whole-body CT: 105 outputs, dropout
    (TC["C"][0], True),                                                     # deconv, affine instance norm, LeakyReLU 0.1
    (dict(BRATS, norm="instance"), True),
    (dict(BRATS, norm=("group", {"num_groups": 4, "affine": False})), True),
    (dict(BRATS, act=("leakyrelu", {"negative_slope": 0.01})), True),
    (dict(BRATS, upsample_mode="deconv"), True),
    (dict(BRATS, use_conv_final=False), True),
    (dict(BRATS, init_filters=48, blocks_down=(1, 2), blocks_up=(1,)), True),
    (dict(), False),                                                        # the reference defaults: init_filters 8
    (dict(BRATS, init_filters=24), False),
    (dict(BRATS, spatial_dims=2), False),
    (dict(BRATS, norm="batch"), False),
    (dict(BRATS, act="prelu"), False),
    (dict(BRATS, act=("leakyrelu", {"negative_slope": 1.5})), False),
    (dict(BRATS, norm=("instance", {"track_running_stats": True})), False),
    (dict(BRATS, blocks_up=(1, 1)), False),                                 # the decoder would not reach level 0
])
def test_segresnet_tc_eligibility(kw, ok):
    assert SegResNet(**kw)._tc_ok is ok


def test_segresnet_dropout_is_inactive_in_eval_mode():
    net = SegResNet(**TC["B"][0])
    assert net._tc_ok
    assert net._dropout_active()
    assert not net.eval()._dropout_active()
    assert not SegResNet(**BRATS)._dropout_active()
