"""UNet configurations with attention heads of 128 channels, shared by the head_dim-128 tests and their fixture
generator (tests/golden/make_golden_hd128.py).

Heads are sized by num_heads (num_head_channels=-1, the reference UNetModel default): 256 channels / 2 heads =
head_dim 128 at the attention level (8x8, T=64) and in the middle block.  The _st variant has d_head 128 in both
the SpatialTransformer self- and cross-attention."""
from _recipe import UNET_CONFIGS

HD128_CONFIGS = {"mid_hd128": dict(UNET_CONFIGS["mid_pixel"], num_heads=2, num_head_channels=-1)}
HD128_CONFIGS["mid_st_hd128"] = dict(HD128_CONFIGS["mid_hd128"], use_spatial_transformer=True, transformer_depth=1,
                                     context_dim=3, condition_key="SpatialRescaler")
