"""TEST-ONLY: the wide emulation backend (tests/_emu_backend_wide.py: CudaBackend's head-size limit of 256, its channel
multiple of 32) that also declares CudaBackend's padded-head route (attn_pad_heads) for head widths that are not a
multiple of 8, with the route's head repack (prep(heads=...)) from a torch reference.  Its attention methods still reject every
width that is not a multiple of 8, so every such head must reach them repacked; attention_tc takes 64 and 128 as the
kernel does.  The base and wide emulations declare no route: on them these heads keep raising in sampling and training
on the stock graph, and their launch traces stay as they are."""
import torch

from _emu_backend_wide import EmuBackendWide, _check
from bbdm_b200 import cabi


def _group_scales(heads, scales, order):
    """[G] fp32 scale of every column group of a row: tensor t of len(scales), order 0 interleaved per head."""
    g = torch.arange(len(scales) * heads)
    return torch.tensor([float(s) for s in scales], dtype=torch.float32)[g // heads if order else g % len(scales)]


def pad_heads_ref(src, heads, scales, order):
    """fp32 [..., G*d] -> [..., G*dp]: every group scaled (one fp32 multiply) and zero-filled from d to dp."""
    G = len(scales) * heads
    d = src.shape[-1] // G
    x = src.reshape(-1, G, d)
    out = torch.zeros(x.shape[0], G, cabi.pad_heads_width(d), dtype=torch.float32, device=src.device)
    out[..., :d] = x * _group_scales(heads, scales, order).to(src.device)[:, None]
    return out.reshape(src.shape[:-1] + (-1,))


def unpad_heads_ref(src, heads, scales, order, d):
    """fp32 [..., G*dp] -> [..., G*d] with the same per-group scales."""
    G = len(scales) * heads
    x = src.reshape(-1, G, cabi.pad_heads_width(d))[..., :d]
    return (x * _group_scales(heads, scales, order).to(src.device)[:, None]).reshape(src.shape[:-1] + (-1,))


class EmuBackendPadHeads(EmuBackendWide):
    attn_pad_heads = True

    def prep(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None, film_scale=None,
             film_shift=None, film_stride=0, silu=True, resample=0, act_f32=None, act_hi=None, act_lo=None,
             raw_f32=None, raw_hi=None, raw_lo=None, heads=None):
        """CudaBackend.prep; with heads the raw outputs take src1's heads re-laid to their own head width (calls records
        'prep heads pad' or 'prep heads unpad')."""
        if heads is None:
            return super().prep(src1, src2, groups=groups, mean=mean, rstd=rstd, gamma=gamma, beta=beta,
                                film_scale=film_scale, film_shift=film_shift, film_stride=film_stride, silu=silu,
                                resample=resample, act_f32=act_f32, act_hi=act_hi, act_lo=act_lo, raw_f32=raw_f32,
                                raw_hi=raw_hi, raw_lo=raw_lo)
        assert src2 is None and mean is None and act_f32 is None and act_hi is None and resample == 0
        assert not torch.isnan(src1).any()
        n, scales, order = heads
        assert 1 <= len(scales) <= 3
        out = raw_f32 if raw_f32 is not None else raw_hi
        ws, wo = src1.shape[-1] // (len(scales) * n), out.shape[-1] // (len(scales) * n)
        assert max(ws, wo) == cabi.pad_heads_width(min(ws, wo))
        if wo >= ws:
            self.calls.append("prep heads pad")
            y = pad_heads_ref(src1, n, scales, order)
        else:
            self.calls.append("prep heads unpad")
            y = unpad_heads_ref(src1, n, scales, order, wo)
        if raw_f32 is not None:
            raw_f32.copy_(y.reshape(raw_f32.shape))
        if raw_hi is not None:
            self._write_split(y.reshape(raw_hi.shape), raw_hi, raw_lo)

    def attention_tc(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        assert qkv_hi.shape[2] // 3 // heads in cabi.ATTN_TC_HEAD_DIMS
        _check(qkv_hi.shape[-1] // 3, heads)
        self.calls.append("attention_tc")
        self.attention(self._planes(qkv_hi, qkv_lo), heads, order, out_f32, out_hi, out_lo)
