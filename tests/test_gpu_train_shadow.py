"""-m gpu: every kernel launch of the benchmarked training micro-step at batch 32 -- q_sample, the UNet training forward,
the backward, two FusedAdam steps -- against an fp64 recomputation of that launch (tests/_launch_shadow.py), for
tools/bench_train.py's cfg3 (LBBDM-f4) and tools/bench_train_st.py's SpatialTransformer variant of it; and every
parameter gradient of the cfg3 step against fp64 autograd of a float64 copy of the UNet.

At batch 32 the training routes differ from the small-batch tests: the 16x16 / 1024-channel level and the middle
block take the Winograd forward and data gradient (512 F(4,3) tiles), the weight gradients run over 131072-pixel K
chains, the GroupNorm backward over 2048-channel concat inputs, the attention backward over 512 (image, head) pairs,
and adam_multi over the UNet's whole parameter list."""
import contextlib
import copy
import math
import time

import pytest
import torch

from _launch_shadow import ST_TRAIN_FORMS, TRAIN_FORMS, Shadow, missing_forms
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, rel_dev, synth_images

pytestmark = pytest.mark.gpu

B = 32
# tools/bench_train_st.py's UNet: cfg3's with the middle block's transformer attending over the 3-channel context
ST_UNET = dict(UNET_CONFIGS["lbbdm_f4"], in_channels=6, use_spatial_transformer=True, context_dim=3,
               condition_key="SpatialRescaler")
LR = 1e-4                    # the benchmarks' learning rate
GRAD_BOUND = 1e-4            # every parameter gradient of the cfg3 step against fp64, per tensor (rel_dev)
REF_CHUNK = 4                # images per fp64 reference pass


def _model(unet):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(unet)).train()
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=1234))
    return net.cuda()


def _inputs():
    """synth_images latents and context, seeded noise; timesteps spread over 0..999, both ends included."""
    x, y = synth_images((B, 3, 64, 64), 1).cuda(), synth_images((B, 3, 64, 64), 2).cuda()
    nz = torch.randn((B, 3, 64, 64), generator=torch.Generator().manual_seed(3)).cuda()
    t = torch.linspace(0, 999, B).round().long().cuda()
    return x, y, nz, t


@contextlib.contextmanager
def _shadowed(monkeypatch):
    """The shadow installed through the product's hooks: the training Functions' backend, the bridge's and
    FusedAdam's backend factories."""
    from bbdm_b200 import cabi, train
    from bbdm_b200.bridge import BridgeOps
    from bbdm_b200.optim import FusedAdam
    sh = Shadow(cabi.CudaBackend())
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
    monkeypatch.setattr(FusedAdam, "backend_factory", staticmethod(lambda: sh))
    old = train._BACKEND
    train.set_backend(sh)
    try:
        yield sh
    finally:
        train.set_backend(old)


def _attention_fp64(self, qkv):
    """AttentionBlock's stock attention core without its fp32 softmax: the whole reference stays in fp64."""
    bs, width, length = qkv.shape
    ch = width // (3 * self.num_heads)
    if self.new_order:
        q, k, v = (z.reshape(bs * self.num_heads, ch, length) for z in qkv.chunk(3, dim=1))
    else:
        q, k, v = qkv.reshape(bs * self.num_heads, ch * 3, length).split(ch, dim=1)
    w = torch.softmax(torch.einsum("bct,bcs->bts", q, k) / math.sqrt(ch), dim=-1)
    return torch.einsum("bts,bcs->bct", w, v).reshape(bs, -1, length)


def _fp64_step(u64, x_t, t, objective, monkeypatch):
    """fp64 autograd of a float64 copy of the UNet on the stock graph, REF_CHUNK images at a time (GroupNorm and
    attention are per image and the parameter gradients are sums over images, so chunking is exact in fp64 and keeps
    the device memory bounded).  The loss gradient is the L1 loss's, -sign(objective - pred64) / N, in fp32 -- what
    the native graph then receives too: the L1 derivative jumps, so the two graphs must not take it from their own
    predictions.  u64: the float64 copy.  Returns (loss gradient, {name: fp64 gradient})."""
    import bbdm_b200.unet as U
    emb = U.timestep_embedding
    with monkeypatch.context() as mp:
        mp.setattr(U, "NATIVE_TRAIN_CONV", False)
        mp.setattr(U.GroupNorm32, "forward", torch.nn.GroupNorm.forward)              # no fp32 round trip
        mp.setattr(U, "timestep_embedding", lambda *a, **k: emb(*a, **k).double())     # the model's fp32 features
        mp.setattr(U.AttentionBlock, "_attention_torch", _attention_fp64)
        dys = []
        for b0 in range(0, B, REF_CHUNK):
            sl = slice(b0, b0 + REF_CHUNK)
            pred = u64(x_t[sl].double(), timesteps=t[sl], context=None)
            dy = (-torch.sign(objective[sl].double() - pred.detach()) / objective.numel()).float()
            pred.backward(dy.double())
            dys.append(dy)
            del pred
    grads = {n: p.grad for n, p in u64.named_parameters()}
    torch.cuda.empty_cache()
    return torch.cat(dys), grads


def _report(sh, title, t0):
    fails = sh.failures()
    print(f"\n{sh.table(title)}\n  wall time {time.time() - t0:.1f} s")
    for f in fails[:40]:
        print("  FAIL", f)
    return fails


def test_cfg3_training_step_every_launch_and_gradient_against_fp64(monkeypatch):
    t0 = time.time()
    net = _model(UNET_CONFIGS["lbbdm_f4"])
    assert net.loss_type == "l1" and net.condition_key == "nocond"
    u64 = copy.deepcopy(net.denoise_fn).double()          # before the bridge attaches its executor to the UNet
    x, y, nz, t = _inputs()
    with _shadowed(monkeypatch) as sh:
        from bbdm_b200.optim import FusedAdam
        opt = FusedAdam(net.get_parameters(), lr=LR)
        with torch.no_grad():
            x_t, objective = net.q_sample(x, y, t, nz)
        dy, want = _fp64_step(u64, x_t, t, objective, monkeypatch)
        del u64
        pred = net.denoise_fn(x_t, timesteps=t, context=None)
        pred.backward(dy)
        got = {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()}
        del pred
        opt.step()                      # bias correction of step 1 ...
        opt.step()                      # ... and step 2 (same gradients)
    fails = _report(sh, f"cfg3 training micro-step (lbbdm_f4, 64x64, B={B})", t0)
    assert not missing_forms(sh, TRAIN_FORMS), missing_forms(sh, TRAIN_FORMS)
    assert not fails, fails[:10]
    devs = {n: rel_dev(got[n], want[n]) for n in want}
    worst = sorted(devs, key=devs.get, reverse=True)
    print(f"  parameter gradients vs fp64 autograd ({len(devs)} tensors), worst ten:")
    for n in worst[:10]:
        print(f"    {n:60s} {devs[n]:.3e}")
    assert len(devs) == len(list(net.denoise_fn.parameters()))
    assert devs[worst[0]] < GRAD_BOUND, (worst[0], devs[worst[0]])


def test_st_training_step_every_launch_against_fp64(monkeypatch):
    """tools/bench_train_st.py's configuration: p_losses with y as the context, backward, two FusedAdam steps."""
    t0 = time.time()
    net = _model(ST_UNET)
    x, y, nz, t = _inputs()
    with _shadowed(monkeypatch) as sh:
        from bbdm_b200.optim import FusedAdam
        opt = FusedAdam(net.get_parameters(), lr=LR)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        opt.step()
        opt.step()
    fails = _report(sh, f"bench_train_st configuration (lbbdm_f4 + SpatialTransformer, 64x64, B={B})", t0)
    assert torch.isfinite(loss)
    assert not missing_forms(sh, ST_TRAIN_FORMS), missing_forms(sh, ST_TRAIN_FORMS)
    assert not fails, fails[:10]
