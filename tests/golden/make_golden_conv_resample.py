#!/usr/bin/env python
"""Generate mid_resample.npz with the UNMODIFIED reference: the aligned UNet of tests/test_gpu_conv_resample.py
(mid_pixel with resblock_updown=False, i.e. standalone Downsample / Upsample convolutions between the levels).  UNet
output, q_sample / p_losses and two p_sample steps (make_golden.unet_and_psample), plus the gradients of one training
step (p_losses + backward on the same x, y, t, q_noise) of the resampling convs and a few neighbours, as at most 16
output rows each (test_gpu_conv_resample.fixture_rows).

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_conv_resample.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from test_gpu_conv_resample import RS_CONFIGS, fixture_rows, picked_gradients  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    make_golden.UNET_CONFIGS.update(RS_CONFIGS)
    make_golden.unet_and_psample("mid_resample", 2, "mid_resample", with_loop=False)
    path = os.path.join(HERE, "mid_resample.npz")
    data = dict(np.load(path))
    torch.set_grad_enabled(True)
    net = make_golden.build_ref("mid_resample").train()
    x, y, t, nz = (torch.from_numpy(data[k]) for k in ("x", "y", "t", "q_noise"))
    loss, _ = net.p_losses(x, y, y, t, nz)
    loss.backward()
    data["loss"] = np.float32(loss.item())
    for n, p in picked_gradients(net.denoise_fn).items():
        data["grad:" + n] = fixture_rows(p.grad.detach()).contiguous().numpy()
    np.savez_compressed(path, **data)
    print("mid_resample", len(data), "entries", f"{os.path.getsize(path) / 1e3:.0f} kB")
