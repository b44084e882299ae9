"""The ctypes mirror of the ABI 7 tensor-core convolution descriptor (include/monai_b200.h); CPU only."""
import ctypes

from monai_b200 import _lib


def test_conv_tc_desc_in_table_sits_in_the_former_padding():
    # ABI 7's in_table takes the 4 bytes of padding between in_slope and res_w: the descriptor keeps its size and every other offset
    assert ctypes.sizeof(_lib.ConvTcDesc) == 128
    assert (_lib.ConvTcDesc.in_slope.offset, _lib.ConvTcDesc.in_table.offset, _lib.ConvTcDesc.res_w.offset) == (56, 60, 64)
    assert (_lib.ConvTcDesc.in_stats.offset, _lib.ConvTcDesc.in_gamma.offset, _lib.ConvTcDesc.add.offset, _lib.ConvTcDesc.add_coff.offset) == (40, 96, 112, 124)
    assert _lib.ABI_VERSION == 7
