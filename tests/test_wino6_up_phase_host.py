"""The phase-stacked F(6x6,3x3) route of the up-ResBlocks' nearest-2x convs (no GPU): which convs get the planes, that
the route does not depend on the batch size, and the emulated chain against conv2d(nearest2x(act)) in fp64."""
import pytest
import torch
import torch.nn.functional as F

from _emu_backend_f63 import EmuBackendF63
from _recipe import UNET_CONFIGS
from bbdm_b200 import cabi, convs
from bbdm_b200.engine import KernelExecutor, UNetEngine
from bbdm_b200.unet import UNetModel


class Emu6(EmuBackendF63):
    """Records the up2_phases flag of each output transform."""

    def __init__(self):
        super().__init__()
        self.up2_outputs = []

    def wino_output(self, m, **kw):
        self.up2_outputs.append(bool(kw.get("up2_phases")))
        return super().wino_output(m, **kw)


class PackOnly(Emu6):
    """Skips the weight arithmetic: only which planes get packed is checked."""

    def pack_weight_split(self, w, hi, lo):
        pass

    def pack_weight_split_taps(self, w, hi, lo):
        pass

    def pack_weight_f32(self, w, out):
        pass

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None, tile=4):
        assert u_hi.shape == ((tile + 2) ** 2, w.shape[0], w.shape[1])


def up6_entries(cfg):
    net = UNetModel(**UNET_CONFIGS[cfg]).eval()
    eng = UNetEngine(net, backend=PackOnly())
    eng.refresh_weights()
    return eng, {k: v for k, v in eng._w.items() if isinstance(v, dict) and "up6" in v}


def test_cfg2_packs_phase_stacked_planes_for_its_two_up_resblocks():
    eng, got = up6_entries("cfg2")
    sizes = eng._resblock_sizes()
    ups = {n for n, m in eng.unet.named_modules() if getattr(m, "up", False) is True}
    assert len(ups) == 2 and {n + ".in_layers.2" for n in ups} == set(got)
    assert sorted(sizes[n] for n in ups) == [128, 256]
    for name, ent in got.items():
        u = ent["up6"]
        assert u is eng._w[name + "#up6"] and u["u_tile"] == 6 and "u_hi" not in ent
        assert u["u_hi"].shape == (64, 4 * ent["cout"], ent["cin"]) and u["cout"] == 4 * ent["cout"]


@pytest.mark.parametrize("cfg", ["cfg1", "lbbdm_f4", "mid_pixel"])
def test_small_maps_pack_none(cfg):
    eng, got = up6_entries(cfg)
    assert not got and not any(k.endswith("#up6") for k in eng._w)


def test_no_phase_stacked_planes_without_winograd():
    net = UNetModel(**UNET_CONFIGS["cfg2"]).eval()
    eng = UNetEngine(net, backend=PackOnly(), precision="bf16")
    eng.refresh_weights()
    assert not any(k.endswith("#up6") for k in eng._w)


def _up_resblock(cin, cout, seed=0):
    g = torch.Generator().manual_seed(seed)
    conv1, conv2 = torch.nn.Conv2d(cin, cout, 3, padding=1), torch.nn.Conv2d(cout, cout, 3, padding=1)
    norm1, norm2 = torch.nn.GroupNorm(32, cin), torch.nn.GroupNorm(32, cout)
    with torch.no_grad():
        for p in (*conv1.parameters(), *conv2.parameters()):
            p.copy_(0.05 * torch.randn(p.shape, generator=g))
        for p in (*norm1.parameters(), *norm2.parameters()):
            p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
    return conv1, conv2, norm1, norm2


@pytest.mark.parametrize("B", [1, 3, 16])
def test_up_resblock_route_does_not_depend_on_batch_size(B):
    """An up-ResBlock at a 48x48 low-res map takes the phase-stacked route at every batch size, and gives what the
    16-phase-tap route gives."""
    conv1, conv2, norm1, norm2 = _up_resblock(64, 64)
    be = Emu6()
    ex = KernelExecutor(backend=be)
    packer = convs.WeightPacker(be, torch.device("cpu"))
    e1 = packer.conv("c1", conv1.weight, conv1.bias)
    packer.up_phase("c1", conv1.weight)
    packer.up_phase_winograd("c1", conv1.weight)
    e2 = packer.conv("c2", conv2.weight, conv2.bias)
    x = torch.randn(B, 48, 48, 64, generator=torch.Generator().manual_seed(B))
    film = (0.1 * torch.randn(B, 64), 0.1 * torch.randn(B, 64))
    run = lambda ent: ex._resblock_flow(ex._pool(torch.device("cpu"), ("t", B)), x, None, norm1, norm2, ent, e2, None,
                                        cabi.RESAMPLE_UP2, film=film).clone()
    y6 = run(e1)
    assert be.up2_outputs == [True]
    y16 = run({k: v for k, v in e1.items() if k != "up6"})
    assert be.up2_outputs == [True]                      # the phase-tap route has no output transform
    assert y6.shape == (B, 96, 96, 64)
    assert (y6 - y16).abs().max() <= 1e-4 * y16.abs().max()


@pytest.mark.parametrize("h,w,cin,cout", [(13, 10, 64, 64), (6, 12, 128, 64)])
def test_emulated_up_phase_chain_matches_conv_of_upsampled_activation(h, w, cin, cout):
    """GroupNorm + SiLU -> wino6 input on the low-res map -> 64 position GEMMs with 4*cout outputs -> up-phase output
    transform, against conv2d(nearest2x(act), W) in fp64 on a ragged map (edge tiles past h, w)."""
    B = 2
    g = torch.Generator().manual_seed(h * w)
    x = torch.randn(B, h, w, cin, generator=g)
    wt, bias = 0.05 * torch.randn(cout, cin, 3, 3, generator=g), torch.randn(cout, generator=g)
    gamma, beta = 1.0 + 0.2 * torch.randn(cin, generator=g), 0.2 * torch.randn(cin, generator=g)
    be = Emu6()
    packer = convs.WeightPacker(be, torch.device("cpu"))
    packer.conv("c", wt, bias)
    packer.up_phase_winograd("c", wt)
    u = packer.w["c#up6"]
    mean = x.double().view(B, -1, 32, cin // 32).mean(dim=(1, 3)).float()
    rstd = (x.double().view(B, -1, 32, cin // 32).var(dim=(1, 3), unbiased=False) + 1e-5).rsqrt().float()
    out = convs.wino_conv(be, convs.FreshBuffers("cpu"), be.wino_geometry(B, h, w, 6), x, None, cout=cout,
                          planes=(u["u_hi"], u["u_lo"], u["u_inv"]), bias=bias, stats=True, tile=6, up2_phases=True,
                          groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True)
    xg = x.double().view(B, h * w, 32, cin // 32)
    a = ((xg - xg.mean(dim=(1, 3), keepdim=True)) * rstd.double().view(B, 1, 32, 1)).view(B, h, w, cin)
    a = F.silu(a * gamma.double() + beta.double()).permute(0, 3, 1, 2)
    ref = F.conv2d(F.interpolate(a, scale_factor=2, mode="nearest"), wt.double(), bias.double(), padding=1)
    ref = ref.permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 2e-5
    part, rows = out._gn
    assert rows == 4 * -(-h // 6) and part.shape == (B * rows, cout, 2)
    torch.testing.assert_close(part.view(B, rows, cout, 2).sum(1).double()[..., 0], ref.sum(dim=(1, 2)),
                               rtol=1e-4, atol=1e-3)
