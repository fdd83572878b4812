"""UNetModel(use_checkpoint=True) on the native training Functions, host side (kernels emulated): every ResBlock,
AttentionBlock and transformer block recomputes its forward in the backward, the loss and every parameter gradient are
bit-identical to the un-checkpointed step, dropout masks are reproduced, the activations kept for the backward shrink,
and two gloo DDP ranks match one process."""
import os
import sys
from collections import Counter

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, synth_images
from test_transformer_training_host import EmuBackend          # with the SpatialTransformer backward entry points

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture()
def emu(monkeypatch):
    from bbdm_b200 import train
    from bbdm_b200.bridge import BridgeOps
    be = EmuBackend()
    train.set_backend(be)
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: be))          # q_sample
    yield be
    train.set_backend(None)


def _net(cfg, **kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(dict(UNET_CONFIGS[cfg], **kw))).train()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net


def _inputs(net, B, S):
    C = 3
    x, y = synth_images((B, C, S, S), seed=11), synth_images((B, C, S, S), seed=12)
    t = torch.tensor([(17 + 311 * i) % 1000 for i in range(B)], dtype=torch.long)
    nz = torch.randn((B, C, S, S), generator=torch.Generator().manual_seed(77))
    return x, y, t, nz


def _step(net, inputs, seed=0):
    x, y, t, nz = inputs
    net.zero_grad(set_to_none=True)
    torch.manual_seed(seed)                      # dropout masks
    loss, _ = net.p_losses(x, y, y, t, nz)
    loss.backward()
    return loss.detach(), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()}


def _same(a, b):
    assert torch.equal(a[0], b[0]), (float(a[0]), float(b[0]))
    assert a[1].keys() == b[1].keys()
    bad = [n for n in a[1] if not torch.equal(a[1][n], b[1][n])]
    assert not bad, bad[:5]


def test_flag_is_stored_and_reaches_every_block():
    from bbdm_b200 import transformer as T
    from bbdm_b200 import unet as U
    kinds = (U.ResBlock, U.AttentionBlock, T.BasicTransformerBlock)
    for cfg in ("mid_pixel", "tiny_st"):
        plain, ck = _net(cfg).denoise_fn, _net(cfg, use_checkpoint=True).denoise_fn
        assert plain.use_checkpoint is False and ck.use_checkpoint is True
        blocks = [m for m in ck.modules() if isinstance(m, kinds)]
        assert blocks and all(m.use_checkpoint for m in blocks)
        assert not any(m.use_checkpoint for m in plain.modules() if isinstance(m, kinds))
        assert list(plain.state_dict()) == list(ck.state_dict())             # the parameter tree is unchanged
        ck.use_checkpoint = False
        assert not any(m.use_checkpoint for m in blocks)


CASES = [("mid_pixel", {}, 2, 32), ("mid_pixel", dict(image_size=48), 3, 48), ("tiny_st", {}, 2, 16),
         ("tiny_variant", {}, 2, 16), ("mid_pixel_winograd", {}, 2, 32)]
ATTENTION = ("attention", "attention_tc", "attention_split", "attention_cross")


@pytest.mark.parametrize("cfg,kw,B,S", CASES, ids=["mid_pixel", "mid_pixel_48_b3", "tiny_st", "tiny_variant",
                                                   "mid_pixel_winograd"])
def test_checkpointed_step_is_bit_identical(emu, monkeypatch, cfg, kw, B, S):
    """The plain step, the trimmed recompute and the whole-block recompute: the same loss and gradients, every block
    kind recomputed, and the trimmed recompute reducing no GroupNorm statistics and skipping GEMMs."""
    from bbdm_b200 import train
    if cfg == "mid_pixel_winograd":               # the 3x3 convs on the Winograd route, whose recompute prep replaces
        cfg = "mid_pixel"
        monkeypatch.setattr(train, "WINO_MIN_C", 1)
        monkeypatch.setattr(train, "WINO_MIN_TILES", 1)
    net = _net(cfg, **kw)
    inputs = _inputs(net, B, S)
    res, calls = {}, {}
    for name, ck, trim in (("plain", False, True), ("trimmed", True, True), ("whole", True, False)):
        net.denoise_fn.use_checkpoint = ck
        monkeypatch.setattr(train, "RECOMPUTE_TRIM", trim)
        emu.calls.clear()
        res[name] = _step(net, inputs)
        calls[name] = Counter(emu.calls)
    _same(res["plain"], res["trimmed"])
    _same(res["plain"], res["whole"])
    n = lambda name, kinds: sum(calls[name][k] for k in kinds)
    for name in ("trimmed", "whole"):
        assert n(name, ATTENTION) == 2 * n("plain", ATTENTION) > 0                  # attention / transformer blocks
    if cfg == "tiny_st":
        assert calls["trimmed"]["layernorm_split"] == 2 * calls["plain"]["layernorm_split"] > 0
    assert calls["whole"]["gn_stats"] > calls["plain"]["gn_stats"] == calls["trimmed"]["gn_stats"]
    gemms = ("conv_umma", "wino_output")
    assert n("plain", gemms) < n("trimmed", gemms) < n("whole", gemms)
    if train.WINO_MIN_C == 1:
        assert calls["plain"]["wino_input"] > 0


def test_dropout_masks_are_reproduced(emu):
    net = _net("tiny_variant", dropout=0.1)
    inputs = _inputs(net, 2, 16)
    plain = _step(net, inputs, seed=5)
    net.denoise_fn.use_checkpoint = True
    _same(plain, _step(net, inputs, seed=5))
    assert not torch.equal(plain[0], _step(net, inputs, seed=6)[0])        # the masks do depend on the seed


def _kept_bytes(net, inputs):
    """Bytes of the distinct storages the training forward keeps for the backward, parameters excluded: what the
    autograd nodes save (saved_tensors_hooks) and the inputs of checkpointed blocks."""
    params = {p.untyped_storage().data_ptr() for p in net.parameters()}
    seen = {}

    def keep(t):
        s = t.untyped_storage()
        if s.data_ptr() not in params:
            seen[s.data_ptr()] = s.nbytes()

    def pack(t):
        keep(t)
        return t

    real = torch.utils.checkpoint.checkpoint

    def spy(fn, *args, **kw):
        for a in args:
            if isinstance(a, torch.Tensor):
                keep(a)
        return real(fn, *args, **kw)

    x, y, t, nz = inputs
    torch.utils.checkpoint.checkpoint = spy
    try:
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            loss, _ = net.p_losses(x, y, y, t, nz)
    finally:
        torch.utils.checkpoint.checkpoint = real
    del loss
    return sum(seen.values())


def test_cfg2_kept_activations_fall_at_least_5x(emu):
    net = _net("cfg2", image_size=32)
    inputs = _inputs(net, 1, 32)
    plain = _kept_bytes(net, inputs)
    net.denoise_fn.use_checkpoint = True
    ck = _kept_bytes(net, inputs)
    assert ck * 5 <= plain, (plain, ck)


# ---- two gloo ranks through the reference's DDP(net) ------------------------------------------------------------------
STEPS, GLOBAL_BATCH = 2, 4


def _train(wrap, rows, use_checkpoint):
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    from test_ddp_training_gloo import _batch, _Step
    from bbdm_b200 import optim, train
    from bbdm_b200.bridge import BridgeOps
    be = EmuBackend()
    BridgeOps.backend_factory = staticmethod(lambda: be)
    optim.FusedAdam.backend_factory = staticmethod(lambda: be)
    train.set_backend(be)
    net = _net("mid_pixel", use_checkpoint=use_checkpoint)
    step_mod = wrap(_Step(net))
    opt = optim.FusedAdam(net.get_parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-3)
    for s in range(STEPS):
        x, y, t, nz = (a[rows] for a in _batch(s))
        opt.zero_grad()
        step_mod(x, y, t, nz).backward()
        opt.step()
    assert "adam_multi" in be.calls and "conv_wgrad" in be.calls
    return {n: p.detach().clone() for n, p in net.denoise_fn.named_parameters()}


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    per = GLOBAL_BATCH // world
    params = _train(lambda m: torch.nn.parallel.DistributedDataParallel(m), slice(rank * per, (rank + 1) * per), True)
    q.put((rank, {k: v.numpy() for k, v in params.items()}))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_ddp_with_checkpointing_matches_single_process(monkeypatch):
    from bbdm_b200 import optim, train
    from bbdm_b200.bridge import BridgeOps
    monkeypatch.setattr(BridgeOps, "backend_factory", BridgeOps.__dict__["backend_factory"])
    monkeypatch.setattr(optim.FusedAdam, "backend_factory", optim.FusedAdam.__dict__["backend_factory"])
    monkeypatch.setattr(train, "_BACKEND", train._BACKEND)
    threads = torch.get_num_threads()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 500
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    for _ in procs:
        rank, res = q.get(timeout=600)
        got[rank] = res
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for k in got[0]:
        assert (got[0][k] == got[1][k]).all(), f"ranks diverged: {k}"
    torch.set_num_threads(2)
    try:
        want = _train(lambda m: m, slice(0, GLOBAL_BATCH), False)        # one process, no checkpointing
    finally:
        torch.set_num_threads(threads)
    worst = max(float((torch.from_numpy(got[0][k]) - w).abs().max()) for k, w in want.items())
    assert worst < 2e-6, worst
