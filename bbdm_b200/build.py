"""In-tree build of libbbdm_b200.so (explicit nvcc, sm_90a only).

``python -m bbdm_b200.build`` or ``__graft_entry__.build()``.  The .so and the object files are
build products (git-ignored), rebuilt whenever a source or the header is newer.  No JIT cache, no
torch extension machinery: the library has a plain C ABI (include/bbdm_b200.h) and is loaded with ctypes.
"""
from __future__ import annotations

import os
import shlex
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.environ.get("BBDM_LIB_OUT") or os.path.join(HERE, "libbbdm_b200.so")   # BBDM_LIB_OUT: experiment builds
SOURCES = ["cabi.cu", "elementwise.cu", "groupnorm.cu", "conv_direct.cu", "conv_umma.cu", "attention_split.cu", "attention_split_padded.cu", "attention_split_wide.cu", "attention_tc.cu", "conv_wgrad.cu", "gn_backward.cu", "attention_bwd.cu", "attention_bwd_wide.cu", "attention_pad.cu", "vqgan_ops.cu", "winograd.cu", "optim.cu", "transformer_ops.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# opt-in experiment switches (e.g. BBDM_NVCC_DEFINES="-DBBDM_UNIFORM_ISSUE"); empty for the product build
FLAGS += shlex.split(os.environ.get("BBDM_NVCC_DEFINES", ""))


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(os.path.dirname(HERE), "include", "bbdm_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    objdir = os.path.join(HERE, "build", os.path.splitext(os.path.basename(OUT))[0])
    os.makedirs(objdir, exist_ok=True)

    def cc(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(cc, SOURCES))
    r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
