"""Which DynUNet configurations the fp16 tensor-core forward implements (`_tc_ok`, decided at construction; CPU only)."""
import pytest
from dynunet_cases import DYNUNET_CASES as GENERIC
from tc_cases import TC_CASES

from monai_b200.networks.nets import DynUNet

TC = TC_CASES["dynunet"]
DEFAULT = TC["A"][0]


@pytest.mark.parametrize("kw,ok", [
    (TC["A"][0], True),
    (TC["B"][0], True),
    (GENERIC[0][0], True),                                              # affine, 4 levels
    (GENERIC[2][0], True),                                              # non-affine, deep supervision, transposed-conv bias
    (GENERIC[1][0], False),                                             # anisotropic kernels and strides, filters of 8
    (dict(DEFAULT, norm_name="batch"), False),
    (dict(DEFAULT, norm_name=("instance", {"affine": True, "track_running_stats": True})), False),
    (dict(DEFAULT, norm_name=("group", {"num_groups": 4})), False),
    (dict(DEFAULT, act_name="relu"), False),
    (dict(DEFAULT, act_name=("leakyrelu", {"negative_slope": 1.5})), False),
    (dict(DEFAULT, out_channels=17), False),
    (dict(DEFAULT, filters=[24, 48, 96, 192, 320, 320]), False),
    (dict(DEFAULT, kernel_size=[3, 3, 3, 3, 3, 5]), False),
    (dict(DEFAULT, strides=[2, 2, 2, 2, 2, 2]), False),
    (dict(DEFAULT, strides=[1, 2, 2, 2, 2, [2, 2, 1]], upsample_kernel_size=[[2, 2, 1], 2, 2, 2, 2]), False),
    (dict(DEFAULT, spatial_dims=2, kernel_size=[3] * 6), False),
])
def test_dynunet_tc_eligibility(kw, ok):
    assert DynUNet(**kw)._tc_ok is ok


def test_dynunet_dropout_is_inactive_in_eval_mode():
    net = DynUNet(**dict(DEFAULT, dropout=0.2))
    assert net._tc_ok
    assert net._dropout_active()
    assert not net.eval()._dropout_active()
    assert not DynUNet(**dict(DEFAULT, dropout=0.0))._dropout_active()
