#!/usr/bin/env python
"""Time the Winograd transform kernels (and the position GEMM) in isolation for the cfg2 layer shapes.
    python tools/time_wino.py [--once]        # --once: one launch per kernel (for ncu)
    python tools/time_wino.py --output-only   # only the output transform, without / with a same-size residual
    python tools/time_wino.py --pack          # weight packing (max|w| reduction + planes), forward and dgrad
    python tools/time_wino.py --f63-conv1     # the cfg2 conv1s of 128 output or input channels and the pooled
                                              # down-ResBlock conv1: direct route (prep + conv) against the F(6,3) chain
                                              # (convs.wino_channels_ok rests on these figures)"""
import json
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200 import cabi  # noqa: E402

SHAPES = [(16, 64, 64, 1024, 1024), (16, 128, 128, 512, 512), (16, 256, 256, 512, 512), (16, 128, 128, 1536, 512)]


def timeit(fn, n):
    for _ in range(2 if n > 1 else 0):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


# (B, H, W of the source map, c1, c2, Cout, down2, fused 1x1 skip) of the cfg2 ResBlock conv1s below 256 channels on
# one side, and the pooled one: 640 -> 128 and 256 -> 128 at 256x256 (skip concat), 128 -> 512 at 128x128 (kept
# direct), 512 -> 512 pooled to 64x64
F63_CONV1 = [(16, 256, 256, 512, 128, 128, False, True), (16, 256, 256, 128, 128, 128, False, True),
             (16, 128, 128, 128, 0, 512, False, True), (16, 128, 128, 512, 0, 512, True, False)]


def time_f63_conv1(be, dev):
    """Each conv as the ResBlock flow runs it, without the skip GEMM (the same on both routes): GroupNorm-SiLU
    (-> 2x2 pool) operand pass (+ the raw split planes for a fused 1x1 skip) and the direct split-bf16 conv, against
    the F(6,3) input transform (same side outputs), 64 position GEMMs and output transform."""
    from bbdm_b200 import convs
    bf = torch.bfloat16
    for B, H, W, c1, c2, Cout, down2, skip in F63_CONV1:
        C = c1 + c2
        h, w = (H // 2, W // 2) if down2 else (H, W)
        x1 = torch.randn(B, H, W, c1, device=dev)
        x2 = torch.randn(B, H, W, c2, device=dev) if c2 else None
        gkw = dict(groups=32, mean=torch.zeros(B, 32, device=dev), rstd=torch.ones(B, 32, device=dev),
                   gamma=torch.ones(C, device=dev), beta=torch.zeros(C, device=dev), silu=True)
        wt, bias = 0.02 * torch.randn(Cout, C, 3, 3, device=dev), torch.zeros(Cout, device=dev)
        packer = convs.WeightPacker(be, torch.device(dev))
        e = packer.conv("c", wt, bias)
        packer.winograd("c", wt, tile=6)
        a_hi, a_lo = torch.empty((B, h, w, C), dtype=bf, device=dev), torch.empty((B, h, w, C), dtype=bf, device=dev)
        r_hi, r_lo = (torch.empty((B, h, w, C), dtype=bf, device=dev) for _ in range(2)) if skip else (None, None)
        out = torch.empty((B, h, w, Cout), device=dev)
        part = torch.empty((B * be.conv_geometry(h, w)[3], Cout, 2), device=dev)

        def direct():
            be.prep(x1, x2, **gkw, resample=cabi.RESAMPLE_DOWN2 if down2 else cabi.RESAMPLE_NONE, act_hi=a_hi,
                    act_lo=a_lo, raw_hi=r_hi, raw_lo=r_lo)
            be.conv_umma(B=B, H=h, W=w, Cin=C, Cout=Cout, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=e["hi"], w_lo=e["lo"],
                         bias=bias, out=out, passes=3, stats_partial=part)

        pool = convs.FreshBuffers(dev)
        geom = be.wino_geometry(B, h, w, tile=6)
        kw = dict(down2=True) if down2 else dict(raw_hi=r_hi, raw_lo=r_lo)
        chain = lambda: convs.wino_conv(be, pool, geom, x1, x2, cout=Cout, planes=(e["u_hi"], e["u_lo"], e["u_inv"]),
                                        bias=bias, stats=True, tile=6, **gkw, **kw)
        t_d, t_w = timeit(direct, 10), timeit(chain, 10)
        print(json.dumps({"B": B, "H": h, "W": w, "Cin": C, "Cout": Cout, "down2": down2, "direct_ms": t_d,
                          "f63_ms": t_w, "speedup": t_d / t_w}))
        del x1, x2, a_hi, a_lo, r_hi, r_lo, out, part, packer, e
        torch.cuda.empty_cache()
    be.check_fault()


def main():
    once = "--once" in sys.argv
    be = cabi.CudaBackend()
    dev = "cuda"
    rows = []
    if "--f63-conv1" in sys.argv:
        time_f63_conv1(be, dev)
        return
    inv = torch.full((1,), 1.0 / 256, device=dev)        # 1/s of the weight planes (wino_pack_weight writes it)
    if "--pack" in sys.argv:
        for Cout, Cin in ((1024, 1024), (512, 512), (512, 1536), (1024, 1536), (512, 640)):
            w = 0.02 * torch.randn(Cout, Cin, 3, 3, device=dev)
            row = {"Cout": Cout, "Cin": Cin}
            for dgrad in (False, True):
                uh = torch.empty((36, Cin, Cout) if dgrad else (36, Cout, Cin), dtype=torch.float16, device=dev)
                ul = torch.empty_like(uh)
                row["dgrad_ms" if dgrad else "fwd_ms"] = timeit(lambda: be.wino_pack_weight(w, uh, ul, inv, dgrad=dgrad), 50)
            print(json.dumps(row))
        be.check_fault()
        return
    if "--output-only" in sys.argv:
        for B, H, W, Cout in ((16, 128, 128, 512), (16, 64, 64, 1024)):
            th, tw, mt, ok = be.wino_geometry(B, H, W)
            m = torch.randn((36, mt, Cout), device=dev)
            out, res = torch.empty((B, H, W, Cout), device=dev), torch.randn((B, H, W, Cout), device=dev)
            part = torch.empty((B * th, Cout, 2), device=dev)
            t0 = timeit(lambda: be.wino_output(m, inv_wscale=inv, B=B, H=H, W=W, Cout=Cout, out=out, stats_partial=part), 10)
            t1 = timeit(lambda: be.wino_output(m, inv_wscale=inv, B=B, H=H, W=W, Cout=Cout, out=out, stats_partial=part,
                                               residual=res, res_mode=cabi.RES_SAME), 10)
            gb = (36 * mt * Cout * 4 + B * H * W * Cout * 4) / 1e9
            print(json.dumps({"B": B, "H": H, "W": W, "Cout": Cout, "tiles": mt, "wino_output_ms": t0,
                              "wino_output_tbps": gb / t0, "wino_output_residual_ms": t1,
                              "wino_output_residual_tbps": (gb + B * H * W * Cout * 4 / 1e9) / t1}))
        be.check_fault()
        return
    for B, H, W, Cin, Cout in (SHAPES[1:2] if once else SHAPES):
        x = torch.randn(B, H, W, Cin, device=dev)
        mean, rstd = torch.zeros(B, 32, device=dev), torch.ones(B, 32, device=dev)
        gamma, beta = torch.ones(Cin, device=dev), torch.zeros(Cin, device=dev)
        th, tw, mt, ok = be.wino_geometry(B, H, W)
        vh = torch.empty((36, mt, Cin), dtype=torch.float16, device=dev)
        vl = torch.empty_like(vh)
        uh = torch.randn(36, Cout, Cin, device=dev).to(torch.float16)
        ul = (0.001 * torch.randn(36, Cout, Cin, device=dev)).to(torch.float16)
        m = torch.empty((36, mt, Cout), device=dev)
        out = torch.empty((B, H, W, Cout), device=dev)
        part = torch.empty((B * th, Cout, 2), device=dev)
        n = 1 if once else 10
        t_in = timeit(lambda: be.wino_input(x, None, groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True,
                                            v_hi=vh, v_lo=vl), n)
        t_g = timeit(lambda: be.conv_umma(B=36, H=mt // 16, W=16, Cin=Cin, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh,
                                          w_lo=ul, out=m, passes=3, weights_per_image=True, operand_f16=True), n)
        t_o = timeit(lambda: be.wino_output(m, inv_wscale=inv, B=B, H=H, W=W, Cout=Cout, out=out, stats_partial=part), n)
        gb_in = (B * H * W * Cin * 4 + 36 * mt * Cin * 4) / 1e9
        gb_out = (36 * mt * Cout * 4 + B * H * W * Cout * 4) / 1e9
        rows.append({"B": B, "H": H, "W": W, "Cin": Cin, "Cout": Cout, "tiles": mt,
                     "wino_input_ms": t_in, "wino_input_tbps": gb_in / t_in, "gemm_ms": t_g,
                     "gemm_algo_tflops": 2.0 * B * H * W * Cout * 9 * Cin / t_g / 1e9,
                     "wino_output_ms": t_o, "wino_output_tbps": gb_out / t_o})
        print(json.dumps(rows[-1]))
        del x, vh, vl, uh, ul, m, out
        torch.cuda.empty_cache()
    be.check_fault()


if __name__ == "__main__":
    main()
