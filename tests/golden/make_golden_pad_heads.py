#!/usr/bin/env python
"""Generate the padded-head fixtures (mid_hd4, mid_hd12_new, mid_hd20, mid_hd60, mid_hd132, mid_st_hd20 and
mid_st_hd36 .npz) by running the UNMODIFIED reference, with the same recipe, inputs and outputs as make_golden.py's other UNet fixtures.

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_pad_heads.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from _pad_heads import PAD_HEAD_CONFIGS  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    make_golden.UNET_CONFIGS.update(PAD_HEAD_CONFIGS)    # build_ref looks configurations up by name
    for tag in PAD_HEAD_CONFIGS:
        make_golden.unet_and_psample(tag, 2, tag, with_loop=False)
