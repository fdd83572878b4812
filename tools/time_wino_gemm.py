#!/usr/bin/env python
"""Time the Winograd position GEMMs (bbdm_conv_umma, weights_per_image) at every distinct shape of a sampling step.

    python bench.py --dump-convs convs.jsonl ...           # the step's launches; rows with "wino": true
    python tools/time_wino_gemm.py convs.jsonl [--rounds 7] [--passes 1]

Each round times every shape once (CUDA events around --reps back-to-back launches), so slow drift of the clock is
spread over all shapes; the median and the spread (min, max) over the rounds are printed per shape, with the executed
tensor-core rate (2 * passes * positions * M * K * N over the time), the HBM bytes the GEMM must move (the V and U
planes read, M written) and the step's launches of that shape.  The card name, power limit and SM clock (sampled by
nvidia-smi while the rounds run) are printed with the results.

Timing-only diagnostics (both change the results; neither is a default):
    BBDM_WINO_CHUNK=16 python tools/time_wino_gemm.py ...  # promote once per 16 K blocks: what the promotions cost
    python tools/time_wino_gemm.py ... --passes 1           # A_hi . W_hi only: the main loop without the split"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200 import cabi  # noqa: E402


def shapes_of(dump):
    """{(positions, H, W, Cin, Cout): launches per step} of the dump's position-GEMM rows."""
    count = collections.Counter()
    with open(dump) as f:
        for line in f:
            r = json.loads(line)
            if r.get("wino"):
                count[(r["B"], r["H"], r["W"], r["Cin"], r["Cout"])] += 1
    return count


def smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True)
    return [s.strip() for s in r.stdout.strip().split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dump", help="bench.py --dump-convs output")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10, help="launches per timed window")
    ap.add_argument("--passes", type=int, default=3, choices=[1, 3])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_wino_gemm needs a GPU"
    dev = "cuda"
    be = cabi.CudaBackend()
    counts = shapes_of(args.dump)
    assert counts, f"no position-GEMM rows in {args.dump}"
    runs = []
    for (P, H, W, Cin, Cout), n in sorted(counts.items()):
        M = H * W
        g = torch.Generator(device=dev).manual_seed(0)
        vh = torch.randn((P, M, Cin), generator=g, device=dev).half()
        vl = (1e-3 * torch.randn((P, M, Cin), generator=g, device=dev)).half()
        uh = (0.05 * torch.randn((P, Cout, Cin), generator=g, device=dev)).half()
        ul = (5e-5 * torch.randn((P, Cout, Cin), generator=g, device=dev)).half()
        m = torch.empty((P, M, Cout), device=dev)

        def launch(P=P, H=H, W=W, Cin=Cin, Cout=Cout, vh=vh, vl=vl, uh=uh, ul=ul, m=m):
            be.conv_umma(B=P, H=H, W=W, Cin=Cin, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh, w_lo=ul, out=m,
                         passes=args.passes, weights_per_image=True, operand_f16=True)
        launch()
        runs.append(((P, H, W, Cin, Cout), n, launch, []))
    torch.cuda.synchronize()
    be.check_fault()

    sampler = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0",
                                "-lms", "200"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        for _ in range(args.rounds):
            for _shape, _n, launch, times in runs:
                launch()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    launch()
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) / args.reps)
    finally:
        sampler.terminate()
        clocks = [int(s) for s in sampler.communicate()[0].split() if s.strip().isdigit()]
    be.check_fault()

    name, power_limit = smi("name,power.limit")
    print(json.dumps({"gpu": name, "power_limit_w": float(power_limit), "passes": args.passes,
                      "wino_chunk": os.environ.get("BBDM_WINO_CHUNK", "default"),
                      "sm_clock_mhz_median": statistics.median(clocks) if clocks else None,
                      "sm_clock_mhz_min": min(clocks) if clocks else None}))
    step_ms = 0.0
    for (P, H, W, Cin, Cout), n, _launch, times in runs:
        M = H * W
        t = statistics.median(times)
        step_ms += n * t
        hbm = P * M * Cin * 4 + P * Cout * Cin * 4 + P * M * Cout * 4
        print(json.dumps({"positions": P, "M": M, "K": Cin, "N": Cout, "per_step": n, "ms": round(t, 4),
                          "ms_min": round(min(times), 4), "ms_max": round(max(times), 4),
                          "tflops": round(2 * args.passes * P * M * Cin * Cout / t / 1e9, 1),
                          "hbm_mb": round(hbm / 1e6, 1), "hbm_tb_s": round(hbm / t / 1e9, 2)}))
    print(json.dumps({"position_gemm_ms_per_step": round(step_ms, 3)}))


if __name__ == "__main__":
    main()
