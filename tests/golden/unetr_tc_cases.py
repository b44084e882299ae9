"""UNETR fixture cases of the fp16 tensor-core path, shared by make_golden_unetr_tc.py (reference side) and the tests:
(constructor kwargs, input shape, weight seed, input seed)."""
UNETR_TC_CASES = {
    # A: the reference's defaults (ViT-B: hidden 768, 12 heads of 64, mlp 3072; feature_size 16) on one 96^3 window, batch 2
    "A": (dict(in_channels=1, out_channels=14, img_size=96), (2, 1, 96, 96, 96), 80, 90),
    # B: the other branches -- several input channels, qkv bias, a second feature size, 6 heads of 64 and a non-cubic
    # 4 x 4 x 3 token grid (48 tokens)
    "B": (dict(in_channels=4, out_channels=3, img_size=(64, 64, 48), feature_size=32, hidden_size=384, num_heads=6, mlp_dim=1536,
               qkv_bias=True), (1, 4, 64, 64, 48), 81, 91),
}


def make_input(shape, seed):
    """The fp16 input of a case, regenerated from its seed on both sides (the fixture keeps a strided sample of it to prove the
    two agree): a seeded CPU torch.randn rounded to fp16."""
    import torch

    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).half()
