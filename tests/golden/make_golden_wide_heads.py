#!/usr/bin/env python
"""Generate the wide-head fixtures (mid_hd256.npz, mid_hd136.npz, mid_hd136_new.npz, mid_st_hd160.npz) by running the
UNMODIFIED reference, with the same recipe, inputs and outputs as make_golden.py's other UNet fixtures.

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_wide_heads.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from _wide_heads import WIDE_HEAD_CONFIGS  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    make_golden.UNET_CONFIGS.update(WIDE_HEAD_CONFIGS)    # build_ref looks configurations up by name
    for tag in WIDE_HEAD_CONFIGS:
        make_golden.unet_and_psample(tag, 2, tag, with_loop=False)
