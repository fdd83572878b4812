"""TEST-ONLY: the F(6x6,3x3) emulation backend (tests/_emu_backend_f63.py) with CudaBackend's 2x2-pooled input form as
well (wino_input's down2 argument): the transform of avg_pool2(GroupNorm-SiLU(x)), the down-ResBlock conv1's input."""
import torch

from _emu_backend_f63 import EmuBackendF63
from oracle import bbdm_oracle as O


class EmuBackendF63Pool(EmuBackendF63):
    def wino_input(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None, film_scale=None,
                   film_shift=None, film_stride=0, silu=True, v_hi, v_lo, raw_hi=None, raw_lo=None, act_hi=None,
                   act_lo=None, tile=4, down2=False):
        kw = dict(groups=groups, mean=mean, rstd=rstd, gamma=gamma, beta=beta, film_scale=film_scale,
                  film_shift=film_shift, film_stride=film_stride, silu=silu, v_hi=v_hi, v_lo=v_lo, raw_hi=raw_hi,
                  raw_lo=raw_lo, act_hi=act_hi, act_lo=act_lo, tile=tile)
        if not down2:
            return super().wino_input(src1, src2, **kw)
        # activate every full-resolution pixel, pool 2x2 (an odd last row / column is dropped), then transform the
        # pooled map as it is (identity mode of the base form)
        assert tile == 6 and raw_hi is None and act_hi is None and mean is not None
        x = src1 if src2 is None else torch.cat([src1, src2], dim=3)
        a = O.op_gn_act(x, mean, rstd, gamma, beta, film_scale, film_shift, silu, 0)
        h2, w2 = a.shape[1] // 2, a.shape[2] // 2
        a = O.op_resample(a[:, :2 * h2, :2 * w2].contiguous(), 2)
        return super().wino_input(a, None, groups=groups, silu=False, v_hi=v_hi, v_lo=v_lo, tile=6)
