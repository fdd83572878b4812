"""The phase-stacked nearest-2x form of the F(6x6,3x3) output transform's tile routine (csrc/winograd.cu,
wino6_output_tile<WINO6_UP_PHASES>: A^T M A + bias stored at the interleaved pixels of the 2x map + the partial sums of
the fused GroupNorm statistics, masked past the low-res h and w) is a __host__ __device__ function: the source the kernel
runs is compiled for the host and executed on the CPU against a direct fp64 evaluation
(tools/host_check_wino6_up2_output.cu).  No GPU involved."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_wino6_up2_output_tile_routine_on_host(tmp_path):
    exe = str(tmp_path / "host_check_wino6_up2_output")
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-o", exe,
                        os.path.join(ROOT, "tools", "host_check_wino6_up2_output.cu"),
                        os.path.join(ROOT, "bbdm_b200", "csrc", "cabi.cu")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    assert r.stdout.count("-> ok") == 3
