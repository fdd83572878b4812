"""UNet configurations whose attention heads are wider than 128 channels (multiples of 8 up to 256), shared by the
wide-head tests and their fixture generator (tests/golden/make_golden_wide_heads.py).

Heads are sized by num_heads (num_head_channels=-1, the reference UNetModel default), at the attention level (8x8,
T=64) and in the middle block:
- mid_hd256: mid_pixel with one head of its 256 channels;
- mid_hd136 / mid_hd136_new: 544 channels (model_channels 32 x 17) over 4 heads of 136, a size that is not a multiple
  of 16, in the legacy and the new qkv order;
- mid_st_hd160: 320 channels and a SpatialTransformer over 2 heads of 160, in both the self- and the cross-attention
  (context: the 3-channel condition).
Every channel count is a multiple of 32 (GroupNorm-32 and the tensor-core convolutions)."""
from _recipe import UNET_CONFIGS

_MID544 = dict(UNET_CONFIGS["mid_pixel"], model_channels=32, channel_mult=(1, 2, 17), num_heads=4, num_head_channels=-1)
WIDE_HEAD_CONFIGS = {
    "mid_hd256": dict(UNET_CONFIGS["mid_pixel"], num_heads=1, num_head_channels=-1),
    "mid_hd136": _MID544,
    "mid_hd136_new": dict(_MID544, use_new_attention_order=True),
    "mid_st_hd160": dict(UNET_CONFIGS["mid_pixel"], channel_mult=(1, 2, 5), num_heads=2, num_head_channels=-1,
                         use_spatial_transformer=True, transformer_depth=1, context_dim=3,
                         condition_key="SpatialRescaler"),
}
WIDE_HEAD_DIMS = {"mid_hd256": 256, "mid_hd136": 136, "mid_hd136_new": 136, "mid_st_hd160": 160}
