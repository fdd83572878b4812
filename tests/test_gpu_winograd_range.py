"""-m gpu: the Winograd path away from the N(0, 0.02) weights and unit-scale activations the rest of the suite uses.

Its operands are split-fp16 planes, and fp16 has 5 exponent bits: weights far below or above the scale the weight
planes are packed at fall into fp16's subnormal range or overflow, and the input transform amplifies a 6x6 tile by up
to 100x.  These tests sweep the weight magnitude through the packing and the whole chain, report the chain's deviation
beside the direct split-bf16 kernel's on the same operands, and pin the activation magnitude the forward route
takes."""
import pytest
import torch

from _recipe import rel_dev
from oracle import bbdm_oracle as O
from test_gpu_winograd import (CHAIN_BOUND_BIASED, DEV, be, film_rows, layered_input, pack, rnd,  # noqa: F401
                               wino_chain, wino_u_ref)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dgrad", [False, True])
@pytest.mark.parametrize("wmax", [1e-4, 1e-3, 2e-2, 3.0, 100.0])
def test_wino_pack_weight_magnitudes(be, wmax, dgrad):
    """hi + lo of the packed planes equal s * G g G^T (s: the power of two the kernel reports) to 22 bits of the
    tensor's largest entry, at every weight magnitude; no plane overflows; packing is deterministic."""
    Cout, Cin = 128, 192
    w = rnd((Cout, Cin, 3, 3), 60)
    w = (w * (wmax / float(w.abs().max()))).to(DEV)
    uh, ul, inv = pack(be, w, dgrad)
    torch.cuda.synchronize()
    be.check_fault()
    s = 1.0 / float(inv)
    assert s > 0 and s == 2.0 ** round(torch.log2(torch.tensor(s)).item()), s
    assert not (torch.isinf(uh).any() or torch.isinf(ul).any() or torch.isnan(uh).any() or torch.isnan(ul).any())
    want = wino_u_ref(w, dgrad) * s
    d = rel_dev(uh.double() + ul.double(), want)
    print(f"\n[wino pack max|w| {wmax:g} dgrad {int(dgrad)}] scale 2^{round(torch.log2(torch.tensor(s)).item())} "
          f"rel dev {d:.3e}")
    assert d < 2e-7, d
    uh2, ul2, inv2 = pack(be, w, dgrad)
    assert torch.equal(uh, uh2) and torch.equal(ul, ul2) and torch.equal(inv, inv2)


def test_wino_pack_weight_zero_tensor(be):
    """An all-zero weight (zero_module output convs) packs to zero planes at the default scale 2^8."""
    uh, ul, inv = pack(be, torch.zeros((64, 128, 3, 3), device=DEV))
    torch.cuda.synchronize()
    assert float(inv) == 2.0 ** -8
    assert not bool(uh.any()) and not bool(ul.any())


def direct_conv(be, x, w, *, mean, rstd, gamma, beta, film=None):
    """The same GN-affine(+FiLM)+SiLU -> 3x3 conv on the direct split-bf16 wgmma kernel (bbdm_prep_operand +
    bbdm_conv_umma, 9 taps, passes 3)."""
    B, H, W, C = x.shape
    Cout = w.shape[0]
    a_hi = torch.empty((B, H, W, C), dtype=torch.bfloat16, device=DEV)
    a_lo = torch.empty_like(a_hi)
    fkw = {} if film is None else dict(film_scale=film[0], film_shift=film[1], film_stride=film[2])
    be.prep(x, None, groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True, act_hi=a_hi, act_lo=a_lo,
            **fkw)
    w_hi = torch.empty((9, Cout, C), dtype=torch.bfloat16, device=DEV)
    w_lo = torch.empty_like(w_hi)
    be.pack_weight_split(w, w_hi, w_lo)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    be.conv_umma(B=B, H=H, W=W, Cin=C, Cout=Cout, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo, out=out, passes=3)
    torch.cuda.synchronize()
    be.check_fault()
    return out


SWEEP_CASES = [  # B, H, W, Cin, Cout
    (2, 32, 32, 256, 128),    # 4 K-blocks, promotion every 2
    (2, 32, 32, 576, 64),     # 9 K-blocks, promotion every 4 with a tail of 1
]


_SWEEP = {}


def _sweep_devs(be, case, std):
    """(Winograd, direct split-bf16) deviation from the fp64 conv of the same activation and weights."""
    if (case, std) not in _SWEEP:
        _SWEEP[case, std] = _chain_and_direct(be, case, std)
    return _SWEEP[case, std]


@pytest.mark.parametrize("std", [2e-2, 4e-3, 1e-3, 1e-4])
@pytest.mark.parametrize("case", SWEEP_CASES)
def test_wino_chain_weight_magnitude_sweep(be, case, std):
    """The whole chain at weight std 2e-2 (the training init) down to 1e-4: within the chain bound of the fp64 conv,
    and no further from it than at std 2e-2 -- as the direct split-bf16 kernel, whose deviation does not depend on
    the weight magnitude.  (With a fixed 2^8 scale the lo planes of small weights became fp16 subnormals: 2.5e-5 at
    std 1e-3, 2.2e-4 at 1e-4.)"""
    dw, dd = _sweep_devs(be, case, std)
    d0, _ = _sweep_devs(be, case, 2e-2)
    print(f"\n[wino weight std {std:g} {case}] winograd {dw:.3e}  direct split-bf16 {dd:.3e}")
    assert dw < CHAIN_BOUND_BIASED, dw
    assert dw <= 1.5 * d0, (dw, d0)


def _chain_and_direct(be, case, std):
    B, H, W, C, Cout = case
    x1, _, x = layered_input(B, H, W, C, 0, 61)
    w = rnd((Cout, C, 3, 3), 62, std).to(DEV)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = (1.0 + 0.1 * rnd((C,), 63)).to(DEV), (0.1 * rnd((C,), 64)).to(DEV)
    act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(), None, None, True, 0)
    want = O.op_conv_nhwc(act, w.double(), None)
    out, _, _ = wino_chain(be, x1, None, w, mean=mean, rstd=rstd, gamma=gamma, beta=beta)
    assert torch.isfinite(out).all()
    return rel_dev(out, want), rel_dev(direct_conv(be, x, w, mean=mean, rstd=rstd, gamma=gamma, beta=beta), want)


def test_wino_chain_activation_window(be):
    """Activations up to |act| ~ 64, reached through gamma and the FiLM scale as a model would (x itself is
    normalised): the fp16 V planes stay finite and the chain stays within its bound.  The input transform amplifies a
    tile by up to 100x, so the fp16 range (65504) ends the window a little above this (see bbdm_wino_input)."""
    B, H, W, C, Cout = 2, 32, 32, 256, 128
    x1, _, x = layered_input(B, H, W, C, 0, 70)
    w = rnd((Cout, C, 3, 3), 71, 0.02).to(DEV)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = (4.0 + 0.1 * rnd((C,), 72)).to(DEV), (0.1 * rnd((C,), 73)).to(DEV)
    fs, fb, fstride = film_rows(B, C, 74)
    fs += 3.0                                  # (1 + scale) ~ 4: GroupNorm output x 16
    act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(), fs.double(),
                      fb.double(), True, 0)
    amax = float(act.abs().max())
    assert 48 <= amax <= 96, amax
    want = O.op_conv_nhwc(act, w.double(), None)
    out, _, (vh, vl, _, _, _, _) = wino_chain(be, x1, None, w, mean=mean, rstd=rstd, gamma=gamma, beta=beta,
                                              film=(fs, fb, fstride))
    vmax = float(vh.float().abs().max())
    d = rel_dev(out, want)
    print(f"\n[wino max|act| {amax:.1f}] max|V| {vmax:.0f}, rel dev vs fp64 conv {d:.3e}")
    assert torch.isfinite(out).all() and torch.isfinite(vh).all() and torch.isfinite(vl).all()
    assert d < CHAIN_BOUND_BIASED, d
