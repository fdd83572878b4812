"""TEST-ONLY: the wide emulation backend (tests/_emu_backend_wide.py: CudaBackend's head-size limit of 256, its channel
multiple of 32) that also declares CudaBackend's GEMM-composed attention route (attn_gemm_route) for wider heads, with
the backward mode of softmax_rows_split (grad=: the planes of the score gradient) from an fp64 oracle.  Its
flash-attention methods still reject heads wider than 256, so every such head must reach the route.  The base and wide emulations declare no route: on them these heads keep raising in sampling and
training on the stock graph, and their launch traces stay as they are."""
import torch

from _emu_backend_wide import EmuBackendWide


def softmax_rows_bwd64(s, dp, scale, valid_cols):
    """fp64 (p, ds) of a [rows, cols] score block: p = softmax(scale * s) over the first valid_cols columns,
    ds = scale * p * (dp - sum_j p_j dp_j), both zero past valid_cols."""
    s, dp = s.double(), dp.double()
    p = torch.zeros_like(s)
    p[..., :valid_cols] = torch.softmax(s[..., :valid_cols] * scale, dim=-1)
    ds = scale * p * (dp - (p * dp).sum(-1, keepdim=True))
    ds[..., valid_cols:] = 0
    return p, ds


class EmuBackendGemmHeads(EmuBackendWide):
    attn_gemm_route = True

    def __init__(self):
        super().__init__()
        self.softmax_grads = 0          # softmax_rows_split launches in the backward mode

    def softmax_rows_split(self, src, scale, out_hi, out_lo, valid_cols=None, grad=None):
        if grad is None:
            return super().softmax_rows_split(src, scale, out_hi, out_lo, valid_cols)
        self.calls.append("softmax_rows_split")
        self.softmax_grads += 1
        n = src.shape[-1]
        v = n if valid_cols is None else int(valid_cols)
        assert 0 < v <= n and n % 4 == 0 and scale > 0 and grad.shape == src.shape
        s2, dp2 = src.reshape(-1, n), grad.reshape(-1, n)
        assert not torch.isnan(s2[:, :v]).any() and not torch.isnan(dp2[:, :v]).any()
        _, ds = softmax_rows_bwd64(s2, dp2, scale, v)
        self._write_split(ds.float().reshape(out_hi.shape), out_hi, out_lo)
