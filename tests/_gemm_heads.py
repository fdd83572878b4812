"""UNet configurations whose attention heads are wider than 256 channels (the GEMM-composed attention route), shared by
the route's tests and their fixture generator (tests/golden/make_golden_gemm_heads.py).

Heads are sized by num_heads (num_head_channels=-1, the reference UNetModel default), at the attention level and in the
middle block:
- mid_hd512: mid_pixel with channel_mult (1, 2, 8) and one head of its 512 channels;
- mid_hd1024: channel_mult (1, 2, 16) and one head of 1024 (the DDPM-style single head of a 1024-channel middle block);
- mid_hd336_new: 672 channels (model_channels 32 x 21) over 2 heads of 336 in the new qkv order at a 40x40 image:
  T = 100 tokens at the attention level (not a multiple of 64) and a head width that is not a multiple of 32;
- mid_st_hd384: 768 channels and a SpatialTransformer over 2 heads of 384, in both the self- and the cross-attention
  (context: the 3-channel condition).
Every channel count is a multiple of 32 (GroupNorm-32 and the tensor-core convolutions)."""
from _recipe import UNET_CONFIGS

_MID = UNET_CONFIGS["mid_pixel"]
GEMM_HEAD_CONFIGS = {
    "mid_hd512": dict(_MID, channel_mult=(1, 2, 8), num_heads=1, num_head_channels=-1),
    "mid_hd1024": dict(_MID, channel_mult=(1, 2, 16), num_heads=1, num_head_channels=-1),
    "mid_hd336_new": dict(_MID, image_size=40, model_channels=32, channel_mult=(1, 2, 21), num_heads=2,
                          num_head_channels=-1, use_new_attention_order=True),
    "mid_st_hd384": dict(_MID, channel_mult=(1, 2, 12), num_heads=2, num_head_channels=-1, use_spatial_transformer=True,
                         transformer_depth=1, context_dim=3, condition_key="SpatialRescaler"),
}
GEMM_HEAD_DIMS = {"mid_hd512": 512, "mid_hd1024": 1024, "mid_hd336_new": 336, "mid_st_hd384": 384}
