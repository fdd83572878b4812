"""TEST-ONLY: the emulation backend (tests/_emu_backend_origin.py) with bbdm_softmax_rows_split's valid_cols: the row
softmax over the first valid_cols columns, exact zeros past them.  A call without valid_cols is the base emulation's, so
the launch traces of every other scenario bind the same arguments."""
import torch

from _emu_backend_origin import EmuBackendOrigin


class EmuBackendRagged(EmuBackendOrigin):
    def softmax_rows_split(self, src, scale, out_hi, out_lo, valid_cols=None):
        if valid_cols is None:
            return super().softmax_rows_split(src, scale, out_hi, out_lo)
        self.calls.append("softmax_rows_split")
        s = src.reshape(out_hi.shape)
        assert 0 < valid_cols <= s.shape[-1] and not torch.isnan(s).any()
        p = torch.zeros_like(s)
        p[..., :valid_cols] = torch.softmax(s[..., :valid_cols] * scale, dim=-1)
        self._write_split(p, out_hi, out_lo)
