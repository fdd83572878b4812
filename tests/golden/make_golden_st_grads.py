#!/usr/bin/env python
"""Generate st_grads.npz: one training step (p_losses + backward) of the UNMODIFIED reference on the SpatialTransformer
UNets of tests/test_gpu_transformer_training.py (mid_st_hd128 and its head_dim-64 variant), on mid_st_hd128.npz's
x, y, t, q_noise with y as the cross-attention context.  Stores per configuration the loss and the gradients of every
parameter of the middle block's transformer, the norms of the other transformers and a few ResBlock / stem / head
tensors (large ones as 16 evenly spread output rows, test_gpu_transformer_training.fixture_rows), in the style of
make_golden.py:mid_pixel_gradients.

    BBDM_REFERENCE_CHECKOUT=<upstream BBDM checkout> python tests/golden/make_golden_st_grads.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
from test_gpu_transformer_training import ST_CONFIGS, fixture_rows, picked_gradients  # noqa: E402

if __name__ == "__main__":
    torch = make_golden.torch
    torch.set_num_threads(os.cpu_count())
    torch.set_grad_enabled(True)
    make_golden.UNET_CONFIGS.update(ST_CONFIGS)
    g = np.load(os.path.join(HERE, "mid_st_hd128.npz"))
    x, y, t, nz = (torch.from_numpy(g[k]) for k in ("x", "y", "t", "q_noise"))
    data = {}
    for tag in ST_CONFIGS:
        net = make_golden.build_ref(tag).train()
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        data[f"{tag}:loss"] = np.float32(loss.item())
        for n, p in picked_gradients(net.denoise_fn).items():
            data[f"{tag}:grad:{n}"] = fixture_rows(p.grad.detach()).contiguous().numpy()
    path = os.path.join(HERE, "st_grads.npz")
    np.savez_compressed(path, **data)
    print("st_grads", len(data), "entries", f"{os.path.getsize(path) / 1e6:.1f} MB")
