#!/usr/bin/env python
"""Generate the head_dim-128 fixtures (mid_hd128.npz, mid_st_hd128.npz) by running the UNMODIFIED reference, with
the same recipe, inputs and outputs as make_golden.py's other UNet fixtures.

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_hd128.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from _hd128 import HD128_CONFIGS  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    make_golden.UNET_CONFIGS.update(HD128_CONFIGS)       # build_ref looks configurations up by name
    make_golden.unet_and_psample("mid_hd128", 2, "mid_hd128")
    make_golden.unet_and_psample("mid_st_hd128", 2, "mid_st_hd128", with_loop=False)
