"""TEST-ONLY: the launch shadow of tests/_launch_shadow.py with the reference of prep's head-repack mode (prep(heads=...),
the padded-head attention route): the raw outputs bit for bit against the torch repack (one fp32 multiply per element,
zeros past the head width) and its split.  Every other launch, and prep without heads, keeps the base references."""
import torch

from _emu_backend_pad_heads import pad_heads_ref, unpad_heads_ref
from _launch_shadow import Shadow, image_equal, split_bf16


class PadHeadsShadow(Shadow):
    def _form(self, name, a):
        f = super()._form(name, a)
        return f + " heads" if name == "prep" and a.get("heads") is not None else f

    def _ref_prep(self, idx, form, shapes, c, a, pre):
        if c.get("heads") is None:
            return super()._ref_prep(idx, form, shapes, c, a, pre)
        n, scales, order = c["heads"]
        src = c["src1"]
        out = a["raw_f32"] if a["raw_f32"] is not None else a["raw_hi"]
        ws, wo = src.shape[-1] // (len(scales) * n), out.shape[-1] // (len(scales) * n)
        pad = wo >= ws
        want = pad_heads_ref(src, n, scales, order) if pad else unpad_heads_ref(src, n, scales, order, wo)
        what = "heads pad" if pad else "heads unpad"
        if a["raw_f32"] is not None:
            self._record(idx, "prep", form, what, image_equal(a["raw_f32"], want.reshape(a["raw_f32"].shape)), 0.0,
                         shapes)
        if a["raw_hi"] is not None:
            h, l = split_bf16(want.reshape(a["raw_hi"].shape))
            self._record(idx, "prep", form, what + " planes",
                         torch.maximum(image_equal(a["raw_hi"], h), image_equal(a["raw_lo"], l)), 0.0, shapes)
