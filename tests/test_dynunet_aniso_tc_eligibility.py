"""Which anisotropic DynUNet plans the fp16 tensor-core forward implements (`_tc_ok`, decided at construction; CPU only)."""
import pytest
from dynunet_aniso_cases import ANISO_CASES as ANISO

from monai_b200.networks.nets import DynUNet

A = ANISO["A"].kw


@pytest.mark.parametrize("tag", ["A", "B", "C"])
def test_anisotropic_fixture_plans_are_eligible(tag):
    assert DynUNet(**ANISO[tag].kw)._tc_ok


@pytest.mark.parametrize("kw", [
    dict(A, kernel_size=[[1, 1, 3]] + A["kernel_size"][1:]),                                    # two axes of size 1
    dict(A, kernel_size=A["kernel_size"][:-1] + [[5, 5, 5]]),                                    # kernel 5
    dict(A, kernel_size=A["kernel_size"][:-1] + [[3, 5, 3]]),                                    # kernel 5 on one axis
    dict(A, strides=A["strides"][:-1] + [[1, 3, 3]], upsample_kernel_size=[[1, 3, 3]] + A["upsample_kernel_size"][1:]),   # stride 3
    dict(A, strides=A["strides"][:-1] + [[1, 1, 1]], upsample_kernel_size=[[1, 1, 1]] + A["upsample_kernel_size"][1:]),   # no stride 2
    dict(A, upsample_kernel_size=[[2, 2, 2]] + A["upsample_kernel_size"][1:]),                    # upsample kernel != stride
    dict(A, strides=[[1, 2, 2]] + A["strides"][1:]),                                              # strides[0] != 1 on one axis
], ids=["two-axes-of-1", "kernel-5", "kernel-5-one-axis", "stride-3", "later-stride-1", "upsample-ne-stride", "first-stride-not-1"])
def test_anisotropic_plans_outside_the_kernels_are_ineligible(kw):
    assert not DynUNet(**kw)._tc_ok


def test_level_shapes_follow_the_per_axis_strides():
    net = DynUNet(**A)
    assert net._level_shapes((16, 64, 64)) == [(16, 64, 64), (16, 32, 32), (16, 16, 16), (8, 8, 8), (4, 4, 4), (4, 2, 2)]
