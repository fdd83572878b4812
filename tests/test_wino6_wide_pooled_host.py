"""The F(6x6,3x3) channel rule of the UNet sampling executor and the pooled input form of the down-ResBlock conv1 (no
GPU): which convs get F(6,3) planes, that the F(4,3)-only backend, the VQGAN executor and training keep their rule,
the emulated pooled chain against fp64 on a ragged map, and a cfg2-architecture forward against the direct route."""
import pytest
import torch
import torch.nn.functional as F

from _emu_backend_f63_pool import EmuBackendF63Pool
from _recipe import UNET_CONFIGS, fill_state_dict, rel_dev
from bbdm_b200 import cabi, convs, train
from bbdm_b200.engine import KernelExecutor, UNetEngine
from bbdm_b200.unet import UNetModel


class PackOnly(EmuBackendF63Pool):
    """Skips the weight arithmetic: only which planes get packed is checked."""

    def pack_weight_split(self, w, hi, lo):
        pass

    def pack_weight_split_taps(self, w, hi, lo):
        pass

    def pack_weight_f32(self, w, out):
        pass

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None, tile=4):
        assert u_hi.shape == ((tile + 2) ** 2, w.shape[0], w.shape[1])


def packed(cfg, backend=PackOnly, **over):
    net = UNetModel(**(UNET_CONFIGS[cfg] | over)).eval()
    eng = UNetEngine(net, backend=backend())
    eng.refresh_weights()
    return eng, {k: v["u_tile"] for k, v in eng._w.items() if isinstance(v, dict) and "u_tile" in v}


@pytest.mark.parametrize("cin,cout,ok", [(640, 128, True), (256, 128, True), (128, 512, False), (512, 512, True),
                                         (128, 128, False), (64, 512, False), (192, 128, False), (384, 128, True),
                                         (160, 512, False)])
def test_f63_channel_rule(cin, cout, ok):
    assert convs.wino_channels_ok(cin, cout, 256, tile=6) == ok
    assert convs.wino_channels_ok(cin, cout, 256) == (min(cin, cout) >= 256 and cin % 64 == 0 and cout % 64 == 0)


# ResBlock conv1s that the F(6,3) rule adds in cfg2: the wide-input 256x256 conv1s and the 2x2-pooled down-ResBlock
# conv1 at 64x64
CFG2_NEW = {"output_blocks.6.0.in_layers.2", "output_blocks.7.0.in_layers.2", "output_blocks.8.0.in_layers.2",
            "input_blocks.6.0.in_layers.2"}


def test_cfg2_packs_f63_planes_for_the_wide_and_pooled_conv1s():
    eng, got = packed("cfg2")
    assert CFG2_NEW <= set(got) and all(got[n] == 6 for n in CFG2_NEW)
    assert "input_blocks.4.0.in_layers.2" not in got          # 128 -> 512 at 128x128: slower on F(6,3)
    # 128 -> 128 convs stay direct: the 256x256 and 128x128 ResBlocks of 128 channels, both convs, the 128-channel conv2s
    # of the wide-input blocks, and the 128x128 down-ResBlock
    for n, m in eng.unet.named_modules():
        if hasattr(m, "out_layers") and m.out_channels == 128:
            assert n + ".out_layers.3" not in got, n
            if m.channels == 128:
                assert n + ".in_layers.2" not in got, n
    assert "input_blocks.3.0.in_layers.2" not in got


def test_cfg1_packs_f63_planes_for_its_64x64_wide_conv1s_only():
    eng, got = packed("cfg1")
    new = {"output_blocks.6.0.in_layers.2", "output_blocks.7.0.in_layers.2", "output_blocks.8.0.in_layers.2"}
    assert new <= set(got) and all(got[n] == 6 for n in new)
    # 128 -> 512 at 32x32 and the down-ResBlocks at 32x32 and 16x16 take F(4,3) tiles: the F(4,3) rule keeps them direct
    assert not {"input_blocks.4.0.in_layers.2", "input_blocks.3.0.in_layers.2", "input_blocks.6.0.in_layers.2"} & set(got)


def test_backend_without_f63_keeps_the_f43_rule():
    class F43Only(PackOnly):
        wino_tiles = (4,)

    eng, got = packed("cfg2", F43Only)
    assert got and set(got.values()) == {4}
    assert not CFG2_NEW & set(got)
    for name in got:
        assert min(eng._w[name]["cin"], eng._w[name]["cout"]) >= 256


def test_vqgan_and_training_keep_the_f43_rule():
    from _recipe import VQGAN_CONFIGS, vqgan_namespace
    from bbdm_b200.vqgan import VQModel
    from bbdm_b200.vqgan_engine import VQGANEngine
    cfg = VQGAN_CONFIGS["vq_tc"]
    # 128 <-> 256-channel ResnetBlocks on 64x64 maps: what the F(6,3) rule would admit
    cfg = cfg | dict(ddconfig=cfg["ddconfig"] | dict(ch=128, ch_mult=(1, 2), resolution=128))
    vq = VQModel(**vqgan_namespace(cfg)).eval()
    eng = VQGANEngine(vq, backend=PackOnly())
    eng.refresh_weights()
    wide = [v for v in eng._w.values() if isinstance(v, dict) and v.get("k") == 3 and {v["cin"], v["cout"]} == {128, 256}]
    assert wide and not any("u_hi" in v for v in wide)
    assert all(v["u_tile"] == 4 for v in eng._w.values() if isinstance(v, dict) and "u_tile" in v)
    be = PackOnly()
    assert not train._wino_ok(be, 16, 256, 256, 640, 128, 3)
    assert not train._wino_ok(be, 16, 64, 64, 256, 128, 3)


def _act(x, mean, rstd, gamma, beta):
    B, H, W, C = x.shape
    xg = x.double().reshape(B, H, W, 32, C // 32)
    a = ((xg - mean.double()[:, None, None, :, None]) * rstd.double()[:, None, None, :, None]).reshape(B, H, W, C)
    return F.silu(a * gamma.double() + beta.double())


@pytest.mark.parametrize("h,w", [(26, 26), (27, 31)])
def test_emulated_pooled_chain_matches_fp64_conv_of_pooled_activation(h, w):
    """GroupNorm + SiLU -> 2x2 average pool inside the F(6,3) input transform -> 64 position GEMMs -> output
    transform, against conv2d(avg_pool2(act)) in fp64, on maps whose pooled size (13x13, 13x15) leaves ragged edge
    tiles and an odd tile count (3x3 per image); the second has odd source sides (the last row / column is not
    pooled)."""
    B, cin, cout = 2, 128, 64
    g = torch.Generator().manual_seed(h * w)
    x = torch.randn(B, h, w, cin, generator=g)
    wt, bias = 0.05 * torch.randn(cout, cin, 3, 3, generator=g), torch.randn(cout, generator=g)
    gamma, beta = 1.0 + 0.2 * torch.randn(cin, generator=g), 0.2 * torch.randn(cin, generator=g)
    mean, rstd = 0.3 * torch.randn(B, 32, generator=g), 0.5 + torch.rand(B, 32, generator=g)
    be = EmuBackendF63Pool()
    packer = convs.WeightPacker(be, torch.device("cpu"))
    packer.conv("c", wt, bias)
    packer.winograd("c", wt, tile=6)
    e = packer.w["c"]
    ho, wo = h // 2, w // 2
    geom = be.wino_geometry(B, ho, wo, 6)
    assert (geom[0] * geom[1]) % 2 == 1
    out = convs.wino_conv(be, convs.FreshBuffers("cpu"), geom, x, None, cout=cout,
                          planes=(e["u_hi"], e["u_lo"], e["u_inv"]), bias=bias, stats=True, tile=6, down2=True,
                          groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True)
    a = _act(x, mean, rstd, gamma, beta).permute(0, 3, 1, 2)
    ref = F.conv2d(F.avg_pool2d(a, 2), wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape == (B, ho, wo, cout)
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 2e-5
    part, rows = out._gn
    assert rows == geom[0] and part.shape == (B * rows, cout, 2)
    torch.testing.assert_close(part.view(B, rows, cout, 2).sum(1).double()[..., 0], ref.sum(dim=(1, 2)),
                               rtol=1e-4, atol=1e-3)


def _resblock(cin, cout, seed=0):
    g = torch.Generator().manual_seed(seed)
    conv1, conv2 = torch.nn.Conv2d(cin, cout, 3, padding=1), torch.nn.Conv2d(cout, cout, 3, padding=1)
    norm1, norm2 = torch.nn.GroupNorm(32, cin), torch.nn.GroupNorm(32, cout)
    with torch.no_grad():
        for p in (*conv1.parameters(), *conv2.parameters()):
            p.copy_(0.05 * torch.randn(p.shape, generator=g))
        for p in (*norm1.parameters(), *norm2.parameters()):
            p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
    return conv1, conv2, norm1, norm2


class Emu6(EmuBackendF63Pool):
    """Records the down2 flag of each F(6,3) input transform."""

    def __init__(self):
        super().__init__()
        self.down2_inputs = []

    def wino_input(self, src1, src2, **kw):
        if kw.get("tile", 4) == 6:
            self.down2_inputs.append(bool(kw.get("down2")))
        return super().wino_input(src1, src2, **kw)


@pytest.mark.parametrize("B", [1, 3])
def test_down_resblock_pooled_route_matches_the_direct_route(B):
    """A down-ResBlock whose pooled map takes F(6,3) runs its conv1 on the pooled input form (conv2 on F(6,3) with the
    2x2-averaged residual), at every batch size, and gives what the prep + direct conv route gives."""
    C = 256
    conv1, conv2, norm1, norm2 = _resblock(C, C)
    be = Emu6()
    ex = KernelExecutor(backend=be)
    packer = convs.WeightPacker(be, torch.device("cpu"))
    e1 = packer.conv("c1", conv1.weight, conv1.bias)
    packer.winograd("c1", conv1.weight, tile=6)
    e2 = packer.conv("c2", conv2.weight, conv2.bias)
    packer.winograd("c2", conv2.weight, tile=6)
    x = torch.randn(B, 96, 96, C, generator=torch.Generator().manual_seed(B))
    film = (0.1 * torch.randn(B, C), 0.1 * torch.randn(B, C))
    run = lambda ent: ex._resblock_flow(ex._pool(torch.device("cpu"), ("t", B)), x, None, norm1, norm2, ent, e2, None,
                                        cabi.RESAMPLE_DOWN2, film=film).clone()
    y6 = run(e1)
    assert be.down2_inputs == [True, False]
    yd = run({k: v for k, v in e1.items() if k not in ("u_hi", "u_lo", "u_inv", "u_tile")})
    assert be.down2_inputs == [True, False, False]
    assert y6.shape == (B, 48, 48, C)
    assert (y6 - yd).abs().max() <= 1e-4 * yd.abs().max()


def test_cfg2_architecture_forward_matches_the_direct_route():
    """The cfg2 UNet (channels, blocks, attention) at image_size 192, where its levels sit at 192, 96 and 48 and every
    conv the F(6,3) rule adds takes it: the forward through the F(6,3) emulation against the same engine with those
    convs' planes dropped (the direct route)."""
    net = UNetModel(**(UNET_CONFIGS["cfg2"] | dict(image_size=192))).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(fill_state_dict(shapes, seed=1234))
    g = torch.Generator().manual_seed(7)
    x, y = torch.randn(1, 3, 192, 192, generator=g), torch.randn(1, 3, 192, 192, generator=g)
    t = torch.tensor([321])
    be = Emu6()
    eng = UNetEngine(net, backend=be)
    eng.refresh_weights()
    assert all(eng._w[n].get("u_tile") == 6 for n in CFG2_NEW)
    out = eng.forward(x, t, y)
    assert be.down2_inputs.count(True) == 1
    direct = UNetEngine(net, backend=EmuBackendF63Pool())
    direct.refresh_weights()
    for n in CFG2_NEW:
        for k in ("u_hi", "u_lo", "u_inv", "u_tile"):
            direct._w[n].pop(k, None)
    ref = direct.forward(x, t, y, assume_fresh_weights=True)
    assert not torch.isnan(out).any()
    assert rel_dev(out, ref) < 5e-5
