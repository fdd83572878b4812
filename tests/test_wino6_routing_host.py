"""Which Winograd tile size the UNet sampling executor packs and runs each 3x3 ResBlock conv at (no GPU): F(6x6,3x3)
on the maps of 48x48 and more, F(4x4,3x3) at 32x32 and below; the VQGAN executor and the training Functions keep
F(4x4,3x3)."""
import pytest

from _emu_backend import EmuBackend
from _recipe import UNET_CONFIGS
from bbdm_b200 import convs
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel


@pytest.mark.parametrize("side,tile", [(256, 6), (128, 6), (64, 6), (48, 6), (32, 4), (16, 4), (8, 4)])
def test_wino_tile_rule(side, tile):
    assert convs.wino_tile(side, side) == tile


class PackRecorder(EmuBackend):
    """Emulation backend that offers both tile sizes and records the Winograd packing calls (the other weight packs
    are skipped: only the routing is checked here)."""
    wino_tiles = (4, 6)

    def __init__(self):
        super().__init__()
        self.wino_packs = []

    def pack_weight_split(self, w, hi, lo):
        pass

    def pack_weight_split_taps(self, w, hi, lo):
        pass

    def pack_weight_f32(self, w, out):
        pass

    def wino_geometry(self, B, H, W, tile=4):
        if tile == 4:
            return super().wino_geometry(B, H, W)
        th, tw = -(-H // 6), -(-W // 6)
        return th, tw, max(128, -(-B * th * tw // 16) * 16), True

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None, tile=4):
        assert u_hi.shape[0] == (tile + 2) ** 2 and u_lo.shape == u_hi.shape
        self.wino_packs.append(tile)


def packed_tiles(cfg):
    net = UNetModel(**UNET_CONFIGS[cfg]).eval()
    eng = UNetEngine(net, backend=PackRecorder())
    eng.refresh_weights()
    sizes = eng._resblock_sizes()
    got = {}
    for name, ent in eng._w.items():
        if isinstance(ent, dict) and "u_tile" in ent:
            got[name] = (sizes[name.rsplit(".", 2)[0]], ent["u_tile"])
    return eng, got


def test_cfg2_maps_take_f63():
    eng, got = packed_tiles("cfg2")               # UNet at 256x256: levels 256, 128, 64
    assert got and {side for side, _ in got.values()} == {256, 128, 64}
    assert all(tile == 6 for _, tile in got.values()), got
    assert eng.be.wino_packs.count(6) == len(got)
    # the geometry the forward uses for a packed F(6,3) conv
    th, tw, tot, ok = eng._wino_geometry(1, 64, 64, 6)
    assert (th, tw, tot, ok) == (11, 11, 128, True)


def test_small_maps_keep_f43():
    eng, got = packed_tiles("cfg1")               # UNet at 64x64: Winograd convs at 32x32 and 16x16, and the up
    assert got                                    # ResBlock's second conv back at 64x64
    for name, (side, tile) in got.items():
        assert tile == (6 if side >= 48 else 4), (name, side, tile)
    assert {side for side, _ in got.values()} >= {32, 16}


def test_backend_without_f63_packs_f43():
    net = UNetModel(**UNET_CONFIGS["cfg2"]).eval()

    class F43Only(PackRecorder):
        wino_tiles = (4,)

    eng = UNetEngine(net, backend=F43Only())
    eng.refresh_weights()
    assert eng.be.wino_packs and set(eng.be.wino_packs) == {4}


@pytest.mark.parametrize("cfg", ["cfg2", "cfg1"])
def test_routing_does_not_depend_on_batch_size(cfg):
    """On maps of at least 128 F(4,3) tiles' worth of pixels (2048) every packed conv takes the Winograd path at every
    batch size (batch-independent, bit-identical results): the size rule counts output pixels, and the F(6,3) tile
    count is padded to a full M block.  Every F(6,3) conv is on such a map.  Smaller maps keep the batch-dependent
    rule (min_tiles over the whole batch)."""
    eng, got = packed_tiles(cfg)
    for name, (side, tile) in got.items():
        ok = [eng._wino_ok(eng._w[name], B, side, side) for B in (1, 3, 4, 5, 16)]
        if side * side >= 2048:
            assert all(ok), (name, side, tile, ok)
        else:
            assert tile == 4, (name, side)
    assert any(tile == 6 for _, tile in got.values())


def test_f63_needs_64_channel_chunks_in_each_input():
    eng, got = packed_tiles("cfg2")
    name = next(n for n, (side, tile) in got.items() if tile == 6 and n.endswith("in_layers.2"))
    ent = eng._w[name]
    assert eng._wino_ok(ent, 1, 64, 64, c1=ent["cin"] - 64 if ent["cin"] > 64 else None)
    assert not eng._wino_ok(ent, 1, 64, 64, c1=ent["cin"] - 32)
