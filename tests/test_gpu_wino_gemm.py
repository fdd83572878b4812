"""-m gpu: the Winograd position GEMMs (bbdm_conv_umma with weights_per_image and a plain fp32 store, the wino_gemm
kernel) against an fp64 evaluation of the same split products, at the cfg2 shapes (rows scaled down where the fp64
reference would be large) and at the edges of the kernel's tiling: ragged last M tiles, 64-wide N tiles, K-block counts
that the promotion chunk does not divide, grids smaller than the SM count, and the 4096 phase-stacked columns of the
up-ResBlock convs.  The GEMM is also checked bit for bit against the general conv_umma kernel, and run once under the
launch guard."""
import pytest
import torch

from _launch_guard import Guard
from _recipe import rel_dev

pytestmark = pytest.mark.gpu
DEV = "cuda"
GEMM_BOUND = 3e-6              # the position-GEMM bound of test_gpu_winograd.py

# (positions, rows per position, Cin, Cout)
CASES = [
    (64, 1936, 1024, 1024),    # 64x64 at batch 16: 121 F(6,3) tiles per image, last M tile 16 rows of 128
    (64, 512, 2048, 1024),     # 64x64 conv1 of the skip concat: K = 2048
    (64, 1024, 512, 512),      # 128x128
    (64, 1024, 640, 512),      # 640 input channels: 10 K blocks, chunks of 4 with a tail of 2
    (64, 512, 1536, 512),      # 128x128 conv1 of the skip concat
    (64, 1024, 256, 128),      # 256x256: K = 256, chunks of 2
    (64, 1024, 640, 128),      # 256x256 conv1 of the skip concat: 10 K blocks at chunks of 4
    (64, 512, 384, 192),       # Cout % 128 == 64: 64-wide N tiles
    (64, 256, 192, 64),        # 3 K blocks at chunks of 2: a 1-block tail; one N tile of 64
    (8, 128, 256, 64),         # 8 tiles: a grid far below the SM count
    (64, 512, 1024, 4096),     # the phase-stacked up-ResBlock conv: 4 x 1024 columns
]


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def planes(shape, seed, scale):
    """fp16 hi / lo planes of a N(0, scale) tensor (the split the Winograd transforms write)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = scale * torch.randn(shape, generator=g, device=DEV)
    hi = x.half()
    return hi, (x - hi.float()).half()


def operands(P, M, Cin, Cout, seed=0):
    vh, vl = planes((P, M, Cin), seed + 1, 1.0)
    uh, ul = planes((P, Cout, Cin), seed + 2, 0.05)
    return vh, vl, uh, ul


def gemm(be, P, M, Cin, Cout, vh, vl, uh, ul, bias=None, residual=None):
    m = torch.full((P, M, Cout), float("nan"), device=DEV)
    be.conv_umma(B=P, H=M // 16, W=16, Cin=Cin, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh, w_lo=ul, bias=bias,
                 residual=residual, res_mode=0 if residual is None else 1, out=m, passes=3, weights_per_image=True,
                 operand_f16=True)
    torch.cuda.synchronize()
    be.check_fault()
    return m


def reference(vh, vl, uh, ul, bias=None):
    want = torch.bmm(vh.double() + vl.double(), (uh.double() + ul.double()).transpose(1, 2))
    return want if bias is None else want + bias.double()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
def test_position_gemm_vs_fp64(be, case):
    P, M, Cin, Cout = case
    ops = operands(P, M, Cin, Cout)
    m = gemm(be, P, M, Cin, Cout, *ops)
    assert not torch.isnan(m).any()
    d = rel_dev(m, reference(*ops))
    print(f"\n[position GEMM {case}] rel dev vs fp64 {d:.3e}")
    assert d < GEMM_BOUND, d


@pytest.mark.parametrize("case", [(64, 1936, 640, 512), (64, 256, 384, 192)], ids=lambda c: "x".join(map(str, c)))
def test_position_gemm_bias_bits_match_general_kernel(be, case):
    """A zero residual sends the same GEMM through the general conv_umma kernel (adding +0 leaves every value's bits
    as they are): both kernels issue the same products in the same chunks and fold them in the same order."""
    P, M, Cin, Cout = case
    ops = operands(P, M, Cin, Cout, seed=10)
    bias = 0.1 * torch.randn(Cout, generator=torch.Generator(device=DEV).manual_seed(13), device=DEV)
    got = gemm(be, P, M, Cin, Cout, *ops, bias=bias)
    general = gemm(be, P, M, Cin, Cout, *ops, bias=bias, residual=torch.zeros(P, M, Cout, device=DEV))
    assert torch.equal(got.view(torch.int32), general.view(torch.int32))
    assert rel_dev(got, reference(*ops, bias=bias)) < GEMM_BOUND


def test_position_gemm_under_launch_guard(be):
    """Ragged last M tiles (1936 rows) on guarded, NaN-poisoned copies: every output element written, nothing outside
    it touched."""
    from bbdm_b200 import cabi
    g = Guard(cabi.CudaBackend())
    P, M, Cin, Cout = 64, 1936, 640, 192
    ops = operands(P, M, Cin, Cout, seed=20)
    m = gemm(g, P, M, Cin, Cout, *ops)
    print("\n" + g.summary("position GEMM"))
    assert not g.findings, g.summary()
    assert g.launches == ["conv_umma"]
    assert rel_dev(m, reference(*ops)) < GEMM_BOUND
