"""TEST-ONLY: the ragged launch shadow (tests/_launch_shadow_ragged.py) that also checks softmax_rows_split's backward
mode, the score gradient of the GEMM-composed attention's training route (heads wider than 256): with grad given, the
planes must hold ds = scale * p * (grad - sum_j p_j grad_j), p = softmax(scale * src) over the first valid_cols columns,
against fp64 over the whole launch (one image-head's [T, Tkvp] block), as a split pair, +0 past valid_cols.  Launches
without grad get the ragged shadow's references."""
import math

import torch

from _launch_shadow import F64, image_devs, pair_well_formed, planes
from _launch_shadow_ragged import RaggedShadow

# ds of a [T, Tkvp] block against fp64: test_gpu_attention_gemm_heads.py::test_softmax_rows_split_grad (measured on an
# H100 80GB HBM3 up to 6.4e-6 of the block's largest |ds|, the split pair's 16 bits included)
DS_BOUND = 2e-5


class GemmHeadsShadow(RaggedShadow):
    def _form(self, name, a):
        f = super()._form(name, a)
        if name == "softmax_rows_split" and a.get("grad") is not None:
            f += " grad"
        return f

    def _ref_softmax_rows_split(self, idx, form, shapes, c, a, pre):
        if c.get("grad") is None:
            return super()._ref_softmax_rows_split(idx, form, shapes, c, a, pre)
        n = c["src"].shape[-1]
        v = n if c.get("valid_cols") is None else int(c["valid_cols"])
        s, g = c["src"].reshape(-1, n).to(F64), c["grad"].reshape(-1, n).to(F64)
        p = torch.zeros_like(s)
        p[:, :v] = torch.softmax(s[:, :v] * c["scale"], dim=-1)
        ds = c["scale"] * p * (g - (p * g).sum(-1, keepdim=True))
        ds[:, v:] = 0
        hi, lo = a["out_hi"].reshape(-1, n), a["out_lo"].reshape(-1, n)
        self._record(idx, "softmax_rows_split", form, "score gradient hi + lo",
                     image_devs(planes(hi, lo).reshape(1, -1), ds.reshape(1, -1)), DS_BOUND, shapes)
        self._record(idx, "softmax_rows_split", form, "rows split", pair_well_formed(hi, lo), 0.0, shapes)
        pad = torch.cat([hi[:, v:], lo[:, v:]], 1).contiguous().view(torch.int16)
        self._record(idx, "softmax_rows_split", form, "padding columns +0",
                     torch.tensor([0.0 if bool((pad == 0).all()) else math.inf], dtype=F64), 0.0, shapes)
