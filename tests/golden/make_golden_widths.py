#!/usr/bin/env python
"""Generate the channel-width fixtures (mid_w96.npz, mid_w224_st.npz, mid_w96_rs.npz) by running the UNMODIFIED
reference, with the same recipe, inputs and outputs as make_golden.py's other UNet fixtures (8-step loop included).

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_widths.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from _widths import WIDTH_CONFIGS  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    make_golden.UNET_CONFIGS.update(WIDTH_CONFIGS)        # build_ref looks configurations up by name
    for tag in WIDTH_CONFIGS:
        make_golden.unet_and_psample(tag, 2, tag)
