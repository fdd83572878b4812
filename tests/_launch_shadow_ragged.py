"""TEST-ONLY: the launch shadow (tests/_launch_shadow.py) whose row-softmax reference honours valid_cols, the columns
of each row the VQGAN AttnBlock's softmax covers when its key axis is padded to a multiple of 64: fp64 softmax over
those columns, and exact zeros in both planes past them.  Launches without valid_cols (or with all columns valid) get
the base reference; their form names the valid columns otherwise."""
import math

import torch

from _launch_shadow import F64, Shadow, image_devs, pair_well_formed, planes


class RaggedShadow(Shadow):
    def _form(self, name, a):
        f = super()._form(name, a)
        if name == "softmax_rows_split" and a.get("valid_cols") not in (None, a["src"].shape[-1]):
            f += f" {a['valid_cols']} valid"
        return f

    def _ref_softmax_rows_split(self, idx, form, shapes, c, a, pre):
        s, v = c["src"], c.get("valid_cols")
        n = s.shape[-1]
        if v is None or v == n:
            return super()._ref_softmax_rows_split(idx, form, shapes, c, a, pre)
        hi, lo = a["out_hi"].reshape(-1, n), a["out_lo"].reshape(-1, n)
        want = torch.zeros((hi.shape[0], n), dtype=F64, device=hi.device)
        want[:, :v] = torch.softmax(s.reshape(-1, n)[:, :v].to(F64) * c["scale"], dim=-1)
        self._record(idx, "softmax_rows_split", form, "rows hi + lo", image_devs(planes(hi, lo), want),
                     self.bounds["softmax"], shapes)
        self._record(idx, "softmax_rows_split", form, "rows split", pair_well_formed(hi, lo), 0.0, shapes)
        # +0.0 in both planes past valid_cols (bit patterns: a -0.0 would also be a wrong store)
        pad = torch.cat([hi[:, v:], lo[:, v:]], 1).contiguous().view(torch.int16)
        self._record(idx, "softmax_rows_split", form, "padding columns +0", torch.where(
            (pad == 0).all(1), 0.0, math.inf).to(F64), 0.0, shapes)
