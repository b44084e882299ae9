"""DynUNet fixture cases of the fp16 tensor-core path, shared by make_golden_dynunet_tc.py (reference side) and the tests:
(constructor kwargs, input shape, weight seed, input seed)."""
DYNUNET_TC_CASES = {
    # A: the nnU-Net default plan (6 levels, filters 32 ... 320, affine instance norm, LeakyReLU 0.01) on two 64^3 windows
    "A": (dict(spatial_dims=3, in_channels=1, out_channels=3, kernel_size=[3] * 6, strides=[1, 2, 2, 2, 2, 2], upsample_kernel_size=[2] * 5),
          (2, 1, 64, 64, 64), 30, 40),
    # B: the other branches -- several input channels, residual blocks (strided conv3 + affine norm3), transposed-conv bias,
    # deep-supervision heads (parameters only in eval mode), eps 1e-4, LeakyReLU 0.1 and a non-cubic input
    "B": (dict(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[3] * 5, strides=[1, 2, 2, 2, 2], upsample_kernel_size=[2] * 4,
               filters=[16, 48, 96, 192, 320], res_block=True, trans_bias=True, deep_supervision=True, deep_supr_num=2,
               norm_name=("instance", {"affine": True, "eps": 1e-4}), act_name=("leakyrelu", {"inplace": True, "negative_slope": 0.1})),
          (1, 4, 48, 64, 32), 31, 41),
}


def make_input(shape, seed):
    """The fp16 input of a case, regenerated from its seed on both sides (the fixture keeps a strided sample of it to prove the
    two agree): a seeded CPU torch.randn rounded to fp16."""
    import torch

    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).half()
