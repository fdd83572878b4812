"""Derived conv weights (host-side, at cache-refresh time only).

``upsample_phase_weights``: nearest-2x upsampling followed by a 3x3 'same' conv
(reference openaimodel.py:118 + :207, i.e. ResBlock(up=True).in_layers, :212-214) equals, per
output phase (a, b) = (y % 2, x % 2), a 2x2 conv on the LOW-RES input whose taps are sums of the
3x3 taps:

    upsampled row 2i+a+dy comes from source row i + floor((a+dy)/2),  dy in {-1,0,1}
      a = 0:  source rows (i-1, i)   get  (w[-1],        w[0] + w[1])
      a = 1:  source rows (i,  i+1)  get  (w[-1] + w[0], w[1])
    (same along x).  Out-of-image source rows are zero in both formulations.

4 phases x 4 taps = 16 [Cout, Cin] matrices -> 2.25x fewer MACs than 9 taps on 4x the pixels.
"""
import torch


def upsample_phase_weights(w: torch.Tensor) -> torch.Tensor:
    """w [Cout, Cin, 3, 3] -> [Cout, Cin, 16], index phase*4 + r*2 + c with phase = a*2 + b."""
    assert w.dim() == 4 and w.shape[2] == 3 and w.shape[3] == 3
    # row-combination matrices R[a][r, dy]: which 3x3 rows feed source row r of phase a
    # (filled on the device rather than copied from a host list: a host-to-device copy cannot be captured into the
    # training step's CUDA graph)
    R = torch.zeros(2, 2, 3, dtype=w.dtype, device=w.device)
    R[0, 0, 0] = R[0, 1, 1] = R[0, 1, 2] = 1.0           # a = 0: r=0 <- dy=-1 ; r=1 <- dy=0,+1
    R[1, 0, 0] = R[1, 0, 1] = R[1, 1, 2] = 1.0           # a = 1: r=0 <- dy=-1,0 ; r=1 <- dy=+1
    # out[o,i,a,b,r,c] = sum_{dy,dx} R[a,r,dy] * R[b,c,dx] * w[o,i,dy,dx]
    out = torch.einsum("ary,bcx,oiyx->oiabrc", R, R, w)
    return out.reshape(w.shape[0], w.shape[1], 16).contiguous()


# ---- the UNet Downsample: 3x3 conv, stride 2, padding 1 (openaimodel.py:137-163) ---------------------------------
# On the space-to-depth operand x'[i] = (x[2i], x[2i+1]) (phase a = 0, 1; bbdm_s2d_split) it is a 2x2-tap conv:
#     y[i] = sum_k w[k] x[2i+k-1] = sum_{o in {-1,0}, a} w[2o+a+1] x'[i+o][a]
# (per axis; the pair o = -1, a = 0 would need k = -1 and is zero).  The window sits at offsets -1..0 (conv
# window_origin -1).  _S2[o+1, a, k] = 1 where k = 2o + a + 1.
def _s2_select(dtype, device):
    s = torch.zeros(2, 2, 3, dtype=dtype, device=device)
    s[0, 1, 0] = s[1, 0, 1] = s[1, 1, 2] = 1.0
    return s


def stride2_s2d_weights(w: torch.Tensor) -> torch.Tensor:
    """w [Cout, Cin, 3, 3] of the stride-2 conv -> [Cout, 4*Cin, 4] (pack_weight_split_taps input): channel
    (a*2 + b)*Cin + ci of the space-to-depth operand, tap (oy+1)*2 + (ox+1) of the 2x2 window at origin -1."""
    co, ci = w.shape[0], w.shape[1]
    S = _s2_select(w.dtype, w.device)
    out = torch.einsum("yak,xbl,oikl->oabiyx", S, S, w)
    return out.reshape(co, 4 * ci, 4).contiguous()


def stride2_dgrad_weights(w: torch.Tensor) -> torch.Tensor:
    """The data gradient of the stride-2 conv with respect to the space-to-depth operand: the transposed 2x2 conv at
    offsets t = -o in {0, +1} (window_origin 0) over dY.  w [Cout, Cin, 3, 3] -> [4*Cin, Cout, 4]: output channel
    (a*2 + b)*Cin + ci, input channel co, tap ty*2 + tx."""
    co, ci = w.shape[0], w.shape[1]
    S = _s2_select(w.dtype, w.device).flip(0)                      # t = 0 <-> o = 0, t = 1 <-> o = -1
    out = torch.einsum("yak,xbl,oikl->abioyx", S, S, w)
    return out.reshape(4 * ci, co, 4).contiguous()


def stride2_fold_wgrad(g: torch.Tensor) -> torch.Tensor:
    """Weight gradient of the 2x2 window conv on the space-to-depth operand, g [Cout, 4*Cin, 2, 2] (conv_wgrad,
    taps 4, origin -1) -> dW [Cout, Cin, 3, 3] of the stride-2 conv: every 3x3 tap is exactly one (tap, phase)."""
    co, ci = g.shape[0], g.shape[1] // 4
    S = _s2_select(g.dtype, g.device)
    return torch.einsum("yak,xbl,oabiyx->oikl", S, S, g.reshape(co, 2, 2, ci, 2, 2)).contiguous()


# ---- nearest-2x followed by a 3x3 'same' conv (Upsample(use_conv), openaimodel.py:93-121), backward --------------
# Per axis the forward is y[2i+p] = sum_k w[k] x[i + f(p,k)], f(p,k) = floor((p+k-1)/2) in {-1, 0, 1}.  With dY' the
# space-to-depth of dY (4*Cout phase-major channels on the low-res grid):
#   dX[j]   = sum_{p, off} (sum_{k: f(p,k) = off} w[k]^T) dY'[j - off][p]   a stride-1 3x3 conv, tap -off
#   dW[k]   = sum_p V[f(p,k)][p],  V[off][p] = sum_i dY'[i][p] x[i + off]^T  the 3x3 weight gradient of (x, dY')
# so neither gradient materialises the upsampled tensor.  _UP[off+1, p, k] = 1 where f(p,k) = off.
def _up_select(dtype, device):
    s = torch.zeros(3, 2, 3, dtype=dtype, device=device)
    for p in range(2):
        for k in range(3):
            s[(p + k - 1) // 2 + 1, p, k] = 1.0
    return s


def upsample_dgrad_weights(w: torch.Tensor) -> torch.Tensor:
    """w [Cout, Cin, 3, 3] -> [Cin, 4*Cout, 9] (pack_weight_split_taps input) of the data-gradient conv over dY':
    output channel ci, input channel (py*2 + px)*Cout + co, tap (dy+1)*3 + (dx+1) reading dY' at offset (dy, dx)."""
    co, ci = w.shape[0], w.shape[1]
    T = _up_select(w.dtype, w.device).flip(0)                      # tap d = -off
    out = torch.einsum("ypk,xql,oikl->ipqoyx", T, T, w)
    return out.reshape(ci, 4 * co, 9).contiguous()


def upsample_fold_wgrad(v: torch.Tensor) -> torch.Tensor:
    """V [4*Cout, Cin, 3, 3] (conv_wgrad, taps 9, over (x, dY')) -> dW [Cout, Cin, 3, 3] of the nearest-2x conv."""
    co, ci = v.shape[0] // 4, v.shape[1]
    U = _up_select(v.dtype, v.device)
    return torch.einsum("ypk,xql,pqoiyx->oikl", U, U, v.reshape(2, 2, co, ci, 3, 3)).contiguous()
