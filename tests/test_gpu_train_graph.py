"""-m gpu: the UNet's training forward and backward on CUDA-graph replays (bbdm_b200/train_graph.py) against the eager
graph, and FusedAdam(capturable=True) against the host-scalar FusedAdam.

Every comparison is bit for bit: the replays run the same kernels on the same operands as the eager graph, the
randomness (timesteps, noise) is drawn eagerly in both, and the step counter and learning rate of the capturable
optimizer form the same fp32 scalars on the device as on the host."""
import argparse
import copy
import json
import os

import pytest
import torch

from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, latent_state_dict, synth_images

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 8
# mid_pixel at the LBBDM-f16 template's latent size and depth: 16x16 maps, two ResBlocks per level
CFG = dict(UNET_CONFIGS["mid_pixel"], image_size=16, num_res_blocks=2)


def _model(graph, cfg=CFG):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(cfg))
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    net = net.to(DEV).train()
    net.denoise_fn.train_graph = graph
    return net


def _opt(net, **kw):
    from bbdm_b200.optim import FusedAdam
    return FusedAdam(net.get_parameters(), lr=1e-4, **kw)


def _batches(n, b=B, size=16, seed=0):
    return [(synth_images((b, 3, size, size), seed + 2 * i).to(DEV), synth_images((b, 3, size, size), seed + 2 * i + 1).to(DEV))
            for i in range(n)]


def _step(net, opt, batches, seed, params=None):
    """One optimizer step over len(batches) micro-batches (the runner's accumulate_grad_batches loop): losses, the
    accumulated gradients before the update, the parameters after it."""
    params = list(net.get_parameters()) if params is None else params
    opt.zero_grad(set_to_none=True)
    losses = []
    for k, (x, y) in enumerate(batches):
        torch.manual_seed(1000 * seed + k)          # timesteps and noise: the same draws on both sides
        loss, _ = net(x, y)
        loss.backward()
        losses.append(loss.detach().clone())
    grads = [p.grad.clone() for p in params]
    opt.step()
    return losses, grads, [p.detach().clone() for p in params]


def _same(a, b, what):
    la, ga, pa = a
    lb, gb, pb = b
    assert all(torch.equal(x, y) for x, y in zip(la, lb)), (what, "loss", la, lb)
    bad = [i for i, (x, y) in enumerate(zip(ga, gb)) if not torch.equal(x, y)]
    assert not bad, (what, "grad", bad[:5])
    bad = [i for i, (x, y) in enumerate(zip(pa, pb)) if not torch.equal(x, y)]
    assert not bad, (what, "param", bad[:5])


def _same_shadow(a, b):
    """EMA shadows equal tensor by tensor (the flat buffers' alignment padding is never written)."""
    return list(a.shadow) == list(b.shadow) and all(torch.equal(a.shadow[n], b.shadow[n]) for n in a.shadow)


def _captures():
    from bbdm_b200 import train_graph
    return train_graph.CAPTURES["n"]


def _check_fault():
    from bbdm_b200 import cabi
    torch.cuda.synchronize()
    cabi.CudaBackend().check_fault()


@pytest.mark.parametrize("micro", [1, 4], ids=["one_batch", "accumulate4"])
def test_replay_matches_eager_bit_for_bit(micro):
    """3 optimizer steps through graph replays against 3 eager ones; micro=4 accumulates 4 micro-batches per step as
    Template-LBBDM-f16.yaml does -- a gradient that aliased the graph's static buffers would be overwritten by the next
    micro-batch's replay."""
    eager, graphed = _model(False), _model(True)
    oe, og = _opt(eager), _opt(graphed)
    n0 = _captures()
    for s in range(3):
        batches = _batches(micro, seed=10 * s)
        _same(_step(eager, oe, batches, s), _step(graphed, og, batches, s), f"step {s}")
    assert _captures() - n0 == 1
    _check_fault()


def _ema_round_trip(net, opt, ema):
    ema.apply_shadow(net)
    ema.restore(net)
    return 0


def _ema_step_under_shadow(net, opt, ema):
    ema.apply_shadow(net)                        # new parameter addresses: one capture
    _step(net, opt, _batches(1, seed=77), 77)
    ema.restore(net)                             # back to the old addresses: one more
    return 2


def _load_state_dict(net, opt, ema):
    sd = {k: v * 0.5 for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(sd)           # copied in place: same addresses, no capture, new values replayed
    opt.load_state_dict(copy.deepcopy(opt.state_dict()))
    return 0


def _batch_size(net, opt, ema):
    _step(net, opt, _batches(1, b=4, seed=55), 55)
    return 2                                     # B=4, then back to B=8 (one live graph)


def _train_eval(net, opt, ema):
    net.eval()
    _step(net, opt, _batches(1, seed=66), 66)
    net.train()
    return 2


@pytest.mark.parametrize("change", [_ema_round_trip, _ema_step_under_shadow, _load_state_dict, _batch_size, _train_eval],
                         ids=lambda f: f.__name__.lstrip("_"))
def test_key_changes_recapture_and_replay_fresh_state(change):
    from bbdm_b200.optim import FusedEMA
    nets = [_model(False), _model(True)]
    opts = [_opt(n) for n in nets]
    emas = []
    for n in nets:
        e = FusedEMA(0.9)
        e.register(n)
        emas.append(e)
    res = [[], []]
    for s in range(2):
        for i in range(2):
            if s == 1:
                n_before = _captures()
                want = change(nets[i], opts[i], emas[i])
                if i == 0:
                    assert _captures() == n_before                      # the eager model never captures
            res[i].append(_step(nets[i], opts[i], _batches(1, seed=10 * s), s))
            emas[i].update(nets[i])
            if s == 1 and i == 1:
                assert _captures() - n_before == want, (change.__name__, _captures() - n_before, want)
    for s in range(2):
        _same(res[0][s], res[1][s], f"{change.__name__} step {s}")
    assert _same_shadow(emas[0], emas[1])
    _check_fault()


def _namespace(d):
    return argparse.Namespace(**{k: _namespace(v) if isinstance(v, dict) else v for k, v in d.items()})


def test_context_that_requires_grad_spatial_rescaler():
    """LatentBrownianBridgeModel with a trainable SpatialRescaler: the context enters the graph with requires_grad, and
    the rescaler's channel_mapper gradient comes back through the replayed backward."""
    import model.BrownianBridge.LatentBrownianBridgeModel as L
    with open(os.path.join(os.path.dirname(__file__), "golden", "latent_model.json")) as f:
        ns = _namespace(json.load(f)["SpatialRescaler"])
    nets = []
    for graph in (False, True):
        torch.manual_seed(0)
        m = L.LatentBrownianBridgeModel(ns)
        m.load_state_dict(latent_state_dict(m.state_dict()))
        m = m.to(DEV).train()
        m.denoise_fn.train_graph = graph
        nets.append(m)
    opts = [_opt(m) for m in nets]
    n0 = _captures()
    for s in range(2):
        batches = [(synth_images((4, 3, 32, 32), 40 + s).to(DEV), synth_images((4, 3, 32, 32), 50 + s).to(DEV))]
        r = [_step(m, o, batches, s) for m, o in zip(nets, opts)]
        _same(r[0], r[1], f"latent step {s}")
    assert nets[1].cond_stage_model.channel_mapper.weight.grad is not None
    assert torch.equal(nets[0].cond_stage_model.channel_mapper.weight.grad,
                       nets[1].cond_stage_model.channel_mapper.weight.grad)
    assert _captures() - n0 == 1
    _check_fault()


@pytest.mark.parametrize("case", ["autocast", "dropout", "switch_off"])
def test_fallbacks_run_eagerly(case, monkeypatch):
    if case == "autocast":
        # reduced precision is a stock-PyTorch graph (the native Functions are fp32); deterministic cuDNN algorithms so
        # that the two eager runs agree bit for bit
        import bbdm_b200.unet as U
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", False)
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    cfg = dict(CFG, num_res_blocks=1, dropout=0.1 if case == "dropout" else 0)
    net = _model(case != "switch_off", cfg)
    ref = _model(False, cfg)
    n0 = _captures()
    x, y = _batches(1)[0]
    outs = []
    for m in (ref, net):
        torch.manual_seed(3)
        if case == "autocast":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss, _ = m(x, y)
        else:
            loss, _ = m(x, y)
        loss.backward()
        outs.append((loss.detach(), [p.grad for p in m.get_parameters()]))
    assert _captures() == n0
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))


# ---- FusedAdam(capturable=True) -----------------------------------------------------------------------------------
def _adam_params(seed=0):
    g = torch.Generator().manual_seed(seed)
    shapes = [(256, 128, 3, 3), (256,), (4097,), (64, 64), (3,)]
    return [torch.nn.Parameter(torch.randn(s, generator=g).to(DEV)) for s in shapes]


def _set_grads(params, seed):
    g = torch.Generator().manual_seed(seed)
    for p in params:
        gr = (1e-3 * torch.randn(p.shape, generator=g)).to(DEV)
        if p.grad is None:
            p.grad = gr
        else:
            p.grad.copy_(gr)


def test_capturable_adam_matches_host_scalar_adam_5_steps():
    """The device-side bias corrections (CUDA's fp64 pow) give the same fp32 scalars as the host's: bit-identical."""
    from bbdm_b200.optim import FusedAdam
    pa, pb = _adam_params(), _adam_params()
    oa = FusedAdam(pa, lr=1e-3, weight_decay=1e-2)
    ob = FusedAdam(pb, lr=1e-3, weight_decay=1e-2, capturable=True)
    for s in range(5):
        _set_grads(pa, s)
        _set_grads(pb, s)
        oa.param_groups[0]["lr"] = ob.param_groups[0]["lr"] = 1e-3 * (0.7 ** s)     # a scheduler between steps
        oa.step()
        ob.step()
        assert all(torch.equal(a, b) for a, b in zip(pa, pb)), s
    assert ob.state[pb[0]]["step"].is_cuda and float(ob.state[pb[0]]["step"]) == 5.0
    _check_fault()


def test_capturable_adam_step_with_ema_in_a_graph():
    """optimizer.step(ema=..., ema_update=True) captured once and replayed 5 times against 5 eager steps."""
    from bbdm_b200.optim import FusedAdam, FusedEMA
    nets = []
    for _ in range(2):
        m = torch.nn.Module()
        for i, p in enumerate(_adam_params()):
            m.register_parameter(f"p{i}", p)
        nets.append(m)
    oa, ob = FusedAdam(nets[0].parameters(), lr=1e-3, capturable=True), FusedAdam(nets[1].parameters(), lr=1e-3, capturable=True)
    ea, eb = FusedEMA(0.9), FusedEMA(0.9)
    ea.register(nets[0])
    eb.register(nets[1])
    pa, pb = list(nets[0].parameters()), list(nets[1].parameters())
    # one eager step each creates the optimizer state (the warm-up of a whole-step capture)
    for p_, o, e, s in ((pa, oa, ea, 0), (pb, ob, eb, 0)):
        _set_grads(p_, s)
        o.step(ema=e, ema_update=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        ob.step(ema=eb, ema_update=True)
    for s in range(1, 6):
        _set_grads(pa, s)
        _set_grads(pb, s)
        oa.step(ema=ea, ema_update=True)
        graph.replay()
        assert all(torch.equal(a, b) for a, b in zip(pa, pb)), s
        assert _same_shadow(ea, eb), s
    assert float(ob.state[pb[0]]["step"]) == 6.0
    _check_fault()


def test_capturable_adam_state_dict_round_trips_with_torch_adam():
    from bbdm_b200.optim import FusedAdam
    pa, pb = _adam_params(), _adam_params()
    ta = torch.optim.Adam(pa, lr=1e-3)
    fb = FusedAdam(pb, lr=1e-3, capturable=True)
    for s in range(3):
        _set_grads(pa, s)
        _set_grads(pb, s)
        ta.step()
        fb.step()
        if s == 1:                                    # swap checkpoints in both directions
            sa, sb = copy.deepcopy(ta.state_dict()), copy.deepcopy(fb.state_dict())
            assert set(sa["state"][0]) == set(sb["state"][0]) == {"step", "exp_avg", "exp_avg_sq"}
            ta.load_state_dict(sb)
            fb.load_state_dict(sa)
            assert fb.param_groups[0]["capturable"] is True
    for a, b in zip(pa, pb):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-8)
    assert float(fb.state_dict()["state"][0]["step"]) == 3.0
    assert float(ta.state_dict()["state"][0]["step"]) == 3.0


# ---- DDP ----------------------------------------------------------------------------------------------------------
def _ddp_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        res = []
        for graph in (False, True):
            net = _model(graph)
            ddp = torch.nn.parallel.DistributedDataParallel(net, device_ids=[rank])
            opt = _opt(net)
            steps = []
            for s in range(3):
                batches = _batches(1, seed=100 * rank + 10 * s)
                steps.append(_step(ddp, opt, batches, 10 * rank + s, params=list(net.get_parameters())))
            res.append(steps)
        for s in range(3):
            _same(res[0][s], res[1][s], f"rank {rank} step {s}")
        torch.save(True, os.path.join(out, f"ok{rank}"))
    finally:
        dist.destroy_process_group()


def test_ddp_two_ranks_replay_matches_eager(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("the 2-rank NCCL run needs two GPUs; this machine has one")
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_ddp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert all(os.path.exists(tmp_path / f"ok{r}") for r in range(2))
