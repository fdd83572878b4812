#!/usr/bin/env python
"""Where the Winograd forward route stops giving finite results as the activations grow.

V = B^T d B amplifies a 6x6 tile by up to 10 x 10 = 100 (the largest absolute row sum of B^T is 10), and the V planes
are fp16 (largest finite value 65504): max|act| <= 655 is finite for every input.  This sweeps max|act| upwards on a
GroupNorm-normalised random input (reached through gamma, as a model would), runs the chain and reports max|V|, the
deviation from the fp64 conv and the first magnitude whose result is not finite.
    python tools/wino_activation_window.py [B H W C Cout]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from oracle import bbdm_oracle as O  # noqa: E402
from _recipe import rel_dev  # noqa: E402
from test_gpu_winograd import layered_input, rnd, wino_chain  # noqa: E402
from bbdm_b200 import cabi  # noqa: E402


def main():
    B, H, W, C, Cout = (int(v) for v in sys.argv[1:6]) if len(sys.argv) > 5 else (2, 32, 32, 256, 128)
    be = cabi.CudaBackend()
    print(torch.cuda.get_device_name(), f"B={B} H={H} W={W} C={C} Cout={Cout}")
    x1, _, x = layered_input(B, H, W, C, 0, 80)
    w = rnd((Cout, C, 3, 3), 81, 0.02).to("cuda")
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    beta = torch.zeros(C, device="cuda")
    unit = O.op_gn_act(x.double(), mean.double(), rstd.double(), torch.ones(C, device="cuda").double(), beta.double(),
                       None, None, True, 0).abs().max().item()
    first_bad = None
    for target in (64, 128, 256, 512, 655, 1024, 1536, 2048, 4096):
        gamma = torch.full((C,), target / unit, device="cuda")
        act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(), None, None, True, 0)
        out, _, (vh, _, _, _, _, _) = wino_chain(be, x1, None, w, mean=mean, rstd=rstd, gamma=gamma, beta=beta)
        fin = bool(torch.isfinite(out).all())
        vmax = vh.float().abs().max().item()
        d = rel_dev(out, O.op_conv_nhwc(act, w.double(), None)) if fin else float("nan")
        print(f"max|act| {act.abs().max().item():8.1f}  max|V_hi| {vmax:9.1f}  finite {int(fin)}  rel dev {d:.3e}")
        if not fin and first_bad is None:
            first_bad = act.abs().max().item()
    print(f"first non-finite result at max|act| = {first_bad}")


if __name__ == "__main__":
    main()
