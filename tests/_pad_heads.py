"""UNet configurations whose attention heads are not a multiple of 8 wide (the padded-head route), shared by the route's
tests and their fixture generator (tests/golden/make_golden_pad_heads.py).

Heads are sized by num_heads (num_head_channels=-1, the reference UNetModel default), at the attention level (8x8,
T=64) and in the middle block; each width lands on one kernel family at d rounded up to 8 (dp):
- mid_hd4: 32 channels over 8 heads of 4 (dp 8, attention_split);
- mid_hd12_new: 96 channels over 8 heads of 12 in the new qkv order (dp 16, attention_split);
- mid_hd20: 160 channels over 8 heads of 20 (dp 24, attention_split);
- mid_hd60: 480 channels over 8 heads of 60 (dp 64, the wgmma attention_tc);
- mid_hd132: 1056 channels over 8 heads of 132 (dp 136, the wide kernels);
- mid_st_hd20 / mid_st_hd36: SpatialTransformers with 8 heads of 20 / 36 (dp 24 / 40) in the self- and the
  cross-attention (context: the 3-channel condition).
Every channel count is a multiple of 32 (GroupNorm-32 and the tensor-core convolutions)."""
from _recipe import UNET_CONFIGS

_MID = dict(UNET_CONFIGS["mid_pixel"], model_channels=32, num_heads=8, num_head_channels=-1)
_ST = dict(use_spatial_transformer=True, transformer_depth=1, context_dim=3, condition_key="SpatialRescaler")
PAD_HEAD_CONFIGS = {
    "mid_hd4": dict(_MID, channel_mult=(1, 2, 1)),
    "mid_hd12_new": dict(_MID, channel_mult=(1, 2, 3), use_new_attention_order=True),
    "mid_hd20": dict(_MID, channel_mult=(1, 2, 5)),
    "mid_hd60": dict(_MID, channel_mult=(1, 2, 15)),
    "mid_hd132": dict(_MID, channel_mult=(1, 2, 33)),
    "mid_st_hd20": dict(_MID, channel_mult=(1, 2, 5), **_ST),
    "mid_st_hd36": dict(_MID, channel_mult=(1, 2, 9), **_ST),
}
PAD_HEAD_DIMS = {"mid_hd4": 4, "mid_hd12_new": 12, "mid_hd20": 20, "mid_hd60": 60, "mid_hd132": 132, "mid_st_hd20": 20,
                 "mid_st_hd36": 36}
