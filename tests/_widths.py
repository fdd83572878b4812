"""UNet configurations whose channel counts are multiples of 32 but not all of 64, shared by the channel-width tests
and their fixture generator (tests/golden/make_golden_widths.py).  All are mid_pixel variants at 32x32 images:

  mid_w96      96 / 192 / 384 channels; AttentionBlocks at ds 1 (32x32, 96 channels) and ds 4 (8x8, 384 channels) with
               num_head_channels 32.  The 96-channel convs, the 96+96 and 192+96 concatenations and the 288-channel qkv
               GEMM of the first level miss the 64 rule.
  mid_w224_st  224 / 448 / 672 channels (LDM-4's model_channels 224); SpatialTransformers at ds 1 and 4 with inner widths
               224 and 672, d_head 32, cross-attending to the 3-channel conditioning image.
  mid_w96_rs   mid_w96 with resblock_updown=False: standalone Downsample and Upsample convs at 96 and 192 channels."""
from _recipe import UNET_CONFIGS

_W96 = dict(UNET_CONFIGS["mid_pixel"], model_channels=96, channel_mult=(1, 2, 4), attention_resolutions=(1, 4),
            num_head_channels=32)
WIDTH_CONFIGS = {
    "mid_w96": _W96,
    "mid_w224_st": dict(UNET_CONFIGS["mid_pixel"], model_channels=224, channel_mult=(1, 2, 3),
                        attention_resolutions=(1, 4), num_head_channels=32, use_spatial_transformer=True,
                        transformer_depth=1, context_dim=3, condition_key="SpatialRescaler"),
    "mid_w96_rs": dict(_W96, resblock_updown=False),
}
