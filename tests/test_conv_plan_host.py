"""The dispatch-plan restatement (tests/_conv_plan.py) on the two H100 SM counts: 114 (PCIe) and 132 (SXM).
The GPU suite checks the tile geometry and split counts against the library on the card it runs on."""
import pytest

from _conv_plan import conv_geometry, conv_plan, wgrad_plan


@pytest.mark.parametrize("case,BN,KB,tail,tiles,per_cta", [
    # (B, H, W, Cin, Cout, taps, Cin2, up2), tiles per CTA on (114, 132) SMs
    ((4, 64, 64, 128, 256, 9, 0, False), 128, 18, 2, 256, (3, 2)),
    ((1, 256, 256, 128, 128, 9, 0, False), 128, 18, 2, 512, (5, 4)),
    ((4, 64, 64, 256, 256, 9, 128, False), 128, 38, 2, 256, (3, 2)),
    ((8, 32, 32, 512, 512, 9, 0, False), 128, 72, 0, 256, (3, 2)),
    ((4, 64, 64, 64, 256, 1, 0, False), 128, 1, 1, 256, (3, 2)),
    ((4, 32, 32, 1024, 1024, 9, 0, False), 128, 144, 0, 256, (3, 2)),
    ((4, 64, 64, 128, 192, 9, 0, False), 64, 18, 2, 384, (4, 3)),
    ((4, 32, 32, 256, 256, 4, 0, True), 128, 16, 0, 256, (3, 2)),
    ((2, 16, 16, 128, 128, 9, 0, False), 64, 18, 2, 8, (1, 1)),
])
def test_conv_plan_is_the_same_on_114_and_132_sms(case, BN, KB, tail, tiles, per_cta):
    B, H, W, Cin, Cout, taps, Cin2, up2 = case
    for sms, n in zip((114, 132), per_cta):
        p = conv_plan(B, H, W, Cin, Cout, taps, Cin2, up2=up2, sms=sms)
        assert (p["BN"], p["KB"], p["kb_tail"], p["tiles"], p["tiles_per_cta"]) == (BN, KB, tail, tiles, n), (sms, p)


def test_conv_plan_n_tile_threshold_depends_on_the_card():
    # 10 M tiles x 8 N tiles of 128 = 80: at least int(0.7 * 114) = 79, below int(0.7 * 132) = 92
    assert conv_plan(5, 16, 16, 1024, 1024, 9, sms=114)["BN"] == 128
    p = conv_plan(5, 16, 16, 1024, 1024, 9, sms=132)
    assert p["BN"] == 64 and p["tiles"] == 160 and p["tiles_per_cta"] == 2


def test_conv_plan_chunk_lengths():
    assert conv_plan(1, 16, 16, 64, 64, 9, passes=3, sms=132)["kb_per_chunk"] == 4
    assert conv_plan(1, 16, 16, 64, 64, 9, passes=1, sms=132)["kb_per_chunk"] == 8
    assert conv_plan(36, 8, 16, 256, 256, 1, wpi=True, sms=132)["kb_per_chunk"] == 2
    assert conv_plan(36, 8, 16, 512, 256, 1, wpi=True, sms=132)["kb_per_chunk"] == 4


def test_conv_geometry():
    assert conv_geometry(64, 64) == (16, 8, 1)
    assert conv_geometry(8, 8) == (8, 8, 2)
    assert conv_geometry(4, 4) == (4, 4, 8)
    assert conv_geometry(12, 20) == (16, 8, 1)


def test_wgrad_plan():
    p = wgrad_plan(2, 256, 256, 128, 128, 9, sms=132)
    assert (p["BN"], p["splits_ws"], p["splits"], p["kb_per_split"], p["kb_last_split"], p["kb_tail"]) == \
        (128, 44, 44, 47, 27, 3)
    assert (p["items"], p["items_per_cta"]) == (396, 3)
    p = wgrad_plan(2, 256, 256, 128, 128, 9, sms=114)
    assert (p["splits"], p["kb_per_split"], p["kb_tail"], p["items_per_cta"]) == (38, 54, 2, 3)
    for sms in (114, 132):
        p = wgrad_plan(16, 16, 16, 512, 320, 9, sms=sms)
        assert (p["n_co"], p["splits"], p["kb_per_split"], p["items_per_cta"]) == (3, 4, 16, 4)
        p = wgrad_plan(4, 32, 32, 1024, 1024, 9, sms=sms)
        assert (p["splits"], p["kb_per_split"]) == (1, 64)
        p = wgrad_plan(2, 64, 64, 64, 192, 9, sms=sms)
        assert (p["BN"], p["splits"], p["items_per_cta"]) == (64, 16, 3)
    assert wgrad_plan(1, 32, 32, 512, 512, 9, sms=132)["workspace"] == 2 * 9 * 512 * 512
