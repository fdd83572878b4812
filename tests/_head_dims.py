"""UNet configurations whose attention head sizes are multiples of 8 but not 16/32/64/128, shared by the head-size
tests and their fixture generator (tests/golden/make_golden_head_dims.py).

Heads are sized by num_heads (num_head_channels=-1, the reference UNetModel default).  The mid_hd* variants of
mid_pixel have 192 channels at the attention level (8x8, T=64) and in the middle block: 8 / 4 / 2 heads give head_dim
24 / 48 / 96.  The mid_st_hd* variants have 320 channels there and a SpatialTransformer: 8 / 4 heads give d_head
40 / 80 in both the self- and the cross-attention."""
from _recipe import UNET_CONFIGS

_MID192 = dict(UNET_CONFIGS["mid_pixel"], channel_mult=(1, 2, 3), num_head_channels=-1)
_MID320_ST = dict(UNET_CONFIGS["mid_pixel"], channel_mult=(1, 2, 5), num_head_channels=-1,
                  use_spatial_transformer=True, transformer_depth=1, context_dim=3, condition_key="SpatialRescaler")
HEAD_DIM_CONFIGS = {
    "mid_hd24": dict(_MID192, num_heads=8),
    "mid_hd48": dict(_MID192, num_heads=4),
    "mid_hd96": dict(_MID192, num_heads=2),
    "mid_st_hd40": dict(_MID320_ST, num_heads=8),
    "mid_st_hd80": dict(_MID320_ST, num_heads=4),
}
HEAD_DIMS = {"mid_hd24": 24, "mid_hd48": 48, "mid_hd96": 96, "mid_st_hd40": 40, "mid_st_hd80": 80}
