"""The UNet's training forward and backward as two CUDA-graph replays (opt-in: ``UNetModel.train_graph``, default from
``BBDM_TRAIN_GRAPH``).

At the map sizes of the latent templates (16x16 to 64x64 latents) each kernel of an eager training step runs for
microseconds, and the step is paced by the host: every autograd Function goes through Python and ctypes, repacks its
weights and issues its launches one at a time.  Here the whole UNet forward (``UNetModel._forward_emb``) is captured
once into a forward graph and its backward into a backward graph, in one private memory pool, following
``torch.cuda.make_graphed_callables``; a training call then copies its inputs into static buffers and replays.

To autograd the pair is one Function (``_Replay``) whose inputs are x, the timestep embedding, the context and every
parameter that requires a gradient; its backward copies ``grad_output`` in, replays the backward graph and returns the
gradients.  ``AccumulateGrad``, DDP's reducer hooks and ``zero_grad`` therefore see ordinary gradients.  Those are
copied out of the graph's static buffers into fresh storage on every backward: a returned tensor that aliased a static
buffer could become ``param.grad``, and the next replay would overwrite a gradient that is being accumulated over
micro-batches.

What stays eager: the timestep draw, the noise and ``q_sample`` (the reference's RNG order is unchanged), the
sinusoidal timestep embedding, the loss and everything after it.  Each replay re-reads the parameters at their
addresses and repacks the weights inside the graph, so in-place optimizer updates and ``load_state_dict`` need no
re-capture.  A change of anything the captured work depends on (``cache_key``) captures anew; one graph is kept per
model, because its pool holds a full step's activations.

The eager graph runs instead, without a warning, under autocast, with a ``Dropout`` of p > 0 in training mode, for CPU
inputs, while another stream capture is in progress and on any backend but ``cabi.CudaBackend`` (``fallback_reason``).
"""
from __future__ import annotations

import weakref

import torch

from . import cabi, train

# captures so far (tests count them: every key change must cost exactly one)
CAPTURES = {"n": 0}
WARMUP_ITERS = 2

_STATES = weakref.WeakKeyDictionary()          # UNetModel -> _GraphState (at most one live graph per model)


def fallback_reason(unet, x, emb, context):
    """Why this training call runs on the eager graph, or None when it can be graphed."""
    if torch.is_autocast_enabled("cuda") or torch.is_autocast_enabled("cpu"):
        return "autocast"
    if any(isinstance(m, torch.nn.Dropout) and m.p > 0 and m.training for m in unet.modules()):
        return "active dropout"
    if not all(t.is_cuda for t in (x, emb) + (() if context is None else (context,))):
        return "CPU input"
    if torch.cuda.is_current_stream_capturing():
        return "stream capture in progress"
    if not isinstance(train.backend(), cabi.CudaBackend):
        return "backend"
    return None


def _trainable(unet):
    return [p for p in unet.parameters() if p.requires_grad]


def cache_key(unet, x, emb, context):
    """Everything the captured work depends on besides the values of its inputs and parameters."""
    from . import unet as unet_mod

    def desc(t):
        return None if t is None else (tuple(t.shape), tuple(t.stride()), t.dtype, t.device, t.requires_grad)

    params = list(unet.parameters())
    # the blocks' own checkpoint switches (UNetModel.use_checkpoint sets them all): the backward graph holds the recompute
    ckpt = tuple(m.use_checkpoint for m in unet.modules() if isinstance(getattr(m, "use_checkpoint", None), bool))
    return (desc(x), desc(emb), desc(context),
            tuple(p.data_ptr() for p in params), tuple(p.requires_grad for p in params),
            unet.training, unet_mod.NATIVE_TRAIN_CONV, train.WINO_TRAIN, train.WINO_MIN_C, train.WINO_MIN_TILES, ckpt,
            train.RECOMPUTE_TRIM)


class _GraphState:
    """Static inputs / output / gradients and the two graphs of one capture."""

    def __init__(self, key):
        self.key = key
        self.generation = 0            # forward replays so far: a backward must belong to the latest one


def _capture(unet, x, emb, context, key):
    dev = x.device
    st = _GraphState(key)
    st.x = x.detach().clone().requires_grad_(x.requires_grad)
    st.emb = emb.detach().clone().requires_grad_(emb.requires_grad)
    st.ctx = None if context is None else context.detach().clone().requires_grad_(context.requires_grad)
    st.params = _trainable(unet)
    st.inputs = [t for t in (st.x, st.emb, st.ctx) if t is not None and t.requires_grad]
    diff = st.inputs + st.params

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        # warm-up outside the capture (module loading, library handles, allocator state); autograd.grad leaves .grad
        # alone.  Zero output gradients keep the warm-up finite.
        for _ in range(WARMUP_ITERS):
            out = unet._forward_emb(st.x, st.emb, st.ctx)
            torch.autograd.grad(out, diff, grad_outputs=torch.zeros_like(out), allow_unused=True)
        del out
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)

    pool = torch.cuda.graph_pool_handle()
    st.fwd, st.bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    # an explicit capture stream on the tensors' device (torch.cuda.graph's default stream is created once per process
    # on whatever device was current then)
    with cabi.collector_paused():
        with torch.cuda.graph(st.fwd, pool=pool, stream=side):
            st.out = unet._forward_emb(st.x, st.emb, st.ctx)
        st.gout = torch.zeros_like(st.out)
        with torch.cuda.graph(st.bwd, pool=pool, stream=side):
            grads = torch.autograd.grad(st.out, diff, grad_outputs=st.gout, allow_unused=True)
    st.grads = list(grads)
    # the parameter gradients are copied out into one flat buffer per backward (one multi-tensor copy); its layout
    st.pidx = [i for i, g in enumerate(st.grads[len(st.inputs):]) if g is not None]
    st.numel = [st.grads[len(st.inputs) + i].numel() for i in st.pidx]
    CAPTURES["n"] += 1
    return st


class _Replay(torch.autograd.Function):
    @staticmethod
    def forward(ctx, st, x, emb, context, *params):
        st.x.copy_(x)
        st.emb.copy_(emb)
        if context is not None:
            st.ctx.copy_(context)
        st.fwd.replay()
        st.generation += 1
        ctx.st, ctx.generation = st, st.generation
        ctx.has_ctx = context is not None
        return st.out.clone()         # the next replay rewrites st.out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        st = ctx.st
        if ctx.generation != st.generation:
            raise RuntimeError("graphed UNet training step: backward of a forward whose activations a later forward "
                               "replay has overwritten; run each backward before the next forward")
        st.gout.copy_(gout)
        st.bwd.replay()
        n_in = len(st.inputs)
        # fresh storage for every returned gradient (see the module docstring: never the static buffers)
        pgrads = [None] * len(st.params)
        if st.pidx:
            flat = torch.empty(sum(st.numel), dtype=torch.float32, device=gout.device)
            views = [v.view(st.grads[n_in + i].shape) for v, i in zip(flat.split(st.numel), st.pidx)]
            torch._foreach_copy_(views, [st.grads[n_in + i] for i in st.pidx])
            for v, i in zip(views, st.pidx):
                pgrads[i] = v
        igrads = {id(t): (None if g is None else g.clone()) for t, g in zip(st.inputs, st.grads[:n_in])}
        out = [None]
        for t in (st.x, st.emb, st.ctx if ctx.has_ctx else None):
            out.append(igrads.get(id(t)) if t is not None else None)
        return tuple(out + pgrads)


def forward(unet, x, emb, context):
    """The UNet output on graph replays, or None when this call has to run on the eager graph
    (fallback_reason)."""
    if fallback_reason(unet, x, emb, context) is not None:
        return None
    key = cache_key(unet, x, emb, context)
    st = _STATES.get(unet)
    if st is None or st.key != key:
        _STATES.pop(unet, None)                  # frees the old graphs and their pool before the new capture
        with torch.cuda.device(x.device):
            st = _capture(unet, x, emb, context, key)
        _STATES[unet] = st
    return _apply(st, x, emb, context)


def _apply(st, x, emb, context):
    return _Replay.apply(st, x, emb, context, *st.params)


def release(unet):
    """Drop the model's captured graphs and the memory their pool holds."""
    _STATES.pop(unet, None)
