"""Autoencoder configurations whose AttnBlocks run at token counts T = H*W that are not multiples of 64, shared by the
ragged-T VQGAN tests and their fixture generator (tests/golden/make_golden_vqgan_ragged.py).

The shrunken LBBDM ddconfig of vq_tc (ch 64, ch_mult (1, 2)) with an attention level at image/2: each encoder and
decoder AttnBlock (the level's and the middle block's) has C = 128 at T = 196, 400 or 784, the token counts of the f16
autoencoder at 224x224 and 320x320 and of the f8 autoencoder at 224x224.  Fixture batch 2, one image size per model."""

VQ_RAGGED_CONFIGS = {
    f"vq_t{(res // 2) ** 2}": dict(embed_dim=3, n_embed=128,
                                  ddconfig=dict(double_z=False, z_channels=3, resolution=res, in_channels=3, out_ch=3,
                                                ch=64, ch_mult=(1, 2), num_res_blocks=1, attn_resolutions=[res // 2],
                                                dropout=0.0))
    for res in (28, 40, 56)
}

# Template-LBBDM-f8 / f16 autoencoders (tests/test_gpu_vqgan.py) and image sizes whose attention level misses T % 64
LBBDM_F8 = dict(embed_dim=4, n_embed=16384,
                ddconfig=dict(double_z=False, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
                              ch_mult=(1, 2, 2, 4), num_res_blocks=2, attn_resolutions=[32], dropout=0.0))
LBBDM_F16 = dict(embed_dim=16, n_embed=16384,
                 ddconfig=dict(double_z=False, z_channels=16, resolution=256, in_channels=3, out_ch=3, ch=128,
                               ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2, attn_resolutions=[16], dropout=0.0))
