"""Host dispatch plans of the tensor-core convolution (bbdm_conv_umma) and weight gradient (bbdm_conv_wgrad).

Restates the host arithmetic of csrc/conv_umma.cu and csrc/conv_wgrad.cu, so that tests can say which kernel
instantiation, tile plan and promotion-chunk layout a case runs on a given card.  The N-tile rule and the grid rule
depend on the SM count: the same shape can run a different instantiation on a 114-SM H100 PCIe than on a 132-SM
H100 SXM.  test_conv_cases_cover_dispatch_regimes checks the tile geometry and the split count against the library.
"""
import math

UM_BM, UM_BK = 128, 64       # conv: pixels per M tile, input channels per K block
WG_BM, WG_BK = 128, 64       # wgrad: couts per M tile, pixels per K block
WG_KB_PER_CHUNK = 4


def num_sms(dev=None):
    import torch
    return torch.cuda.get_device_properties(dev if dev is not None else torch.cuda.current_device()).multi_processor_count


def _pow2_floor(x):
    p = 1
    while p * 2 <= x:
        p *= 2
    return p


def _pow2_ceil(x):
    p = 1
    while p < x:
        p *= 2
    return p


def conv_geometry(H, W):
    """(TW, TH, TB): the 128-pixel box of one M tile (tile_geometry in conv_umma.cu)."""
    TW = min(_pow2_floor(W), 16)
    TH = min(_pow2_ceil(H), UM_BM // TW)
    return TW, TH, UM_BM // (TW * TH)


def conv_plan(B, H, W, Cin, Cout, taps, Cin2=0, up2=False, passes=3, wpi=False, sms=None):
    """Plan of one bbdm_conv_umma call (H, W: the conv input grid; taps 4 with up2 for the fused upsample)."""
    sms = num_sms() if sms is None else sms
    TW, TH, TB = conv_geometry(H, W)
    m_tiles = math.ceil(W / TW) * math.ceil(H / TH) * math.ceil(B / TB) * (4 if up2 else 1)
    BN = 128 if Cout % 128 == 0 else 64
    if BN > 64 and m_tiles * (Cout // BN) < int(0.7 * sms):
        BN = 64
    KB = taps * (Cin // UM_BK) + Cin2 // UM_BK
    kb_per_chunk = ((4 if Cin >= 512 else 2) if wpi else (4 if passes == 3 else 8))
    tiles = m_tiles * (Cout // BN)
    grid = min(tiles, sms)
    return dict(TW=TW, TH=TH, TB=TB, BN=BN, KB=KB, kb_per_chunk=kb_per_chunk, kb_tail=KB % kb_per_chunk,
                tiles=tiles, grid=grid, tiles_per_cta=math.ceil(tiles / grid))


def wgrad_plan(B, H, W, Cin, Cout, taps, sms=None):
    """Plan of one bbdm_conv_wgrad call.  splits_ws is the split count the workspace is sized for
    (bbdm_conv_wgrad_workspace); the kernel drops empty splits, so splits <= splits_ws."""
    sms = num_sms() if sms is None else sms
    kblocks = B * H * W // WG_BK
    BN = 128 if Cin % 128 == 0 else 64
    n_co, n_ci = math.ceil(Cout / WG_BM), Cin // BN
    tiles = taps * n_co * n_ci
    sp = min(max(min(math.ceil(3 * sms / tiles), kblocks // 8), 1), 64)
    kb_per_split = math.ceil(kblocks / sp)
    splits = math.ceil(kblocks / kb_per_split)
    items = splits * tiles
    grid = min(items, sms)
    return dict(BN=BN, n_co=n_co, n_ci=n_ci, splits_ws=sp, workspace=sp * taps * Cout * Cin, splits=splits,
                kb_per_split=kb_per_split, kb_last_split=kblocks - (splits - 1) * kb_per_split,
                kb_tail=kb_per_split % WG_KB_PER_CHUNK, items=items, grid=grid, items_per_cta=math.ceil(items / grid))
