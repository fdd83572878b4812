"""Host side of the Brownian-bridge q_sample / p_sample path: picks timesteps and per-step
scalars on the host (bit-exact indexing), launches the fused elementwise kernels and the UNet
engine, and drives the sampling loop.

Mirrors BrownianBridgeModel.{q_sample,p_sample,p_sample_loop} of the reference
(model/BrownianBridge/BrownianBridgeModel.py:128-146,171-221).
"""
from __future__ import annotations

import torch

from . import cabi
from .schedule import step_coefficients


class BridgeOps:
    # the product backend; tests/ may substitute an emulation to exercise this host logic on CPU
    backend_factory = staticmethod(lambda: cabi.CudaBackend())

    def __init__(self, model):
        self.__dict__["model"] = model
        self._be = None
        self._coef = None
        self._coef_key = None
        self.noise_source = None     # optional callable(like) -> noise tensor (tests: reference noise)
        self.use_cuda_graph = True   # replay one captured step graph in p_sample_loop (CUDA backend only)
        self._graphs = {}

    def backend(self):
        if self._be is None:
            self._be = self.backend_factory()
            # the UNet engine must use the same backend object
            eng = self.model.denoise_fn._engine
            if eng is None:
                from .engine import UNetEngine
                object.__setattr__(self.model.denoise_fn, "_engine",
                                   UNetEngine(self.model.denoise_fn, backend=self._be))
        return self._be

    def _require_device(self, t):
        if not t.is_cuda and getattr(self.backend(), "requires_cuda", True):
            raise RuntimeError("bbdm_b200: q_sample/p_sample run only on a CUDA sm_90a device "
                               "(kernels behind libbbdm_b200.so); there is no CPU fallback.")

    # ------------------------------------------------------------------------------ q_sample
    def q_sample(self, x0, y, t, noise):
        m = self.model
        self._require_device(x0)
        be = self.backend()
        x0c, yc, nz = (z.detach().contiguous().float() for z in (x0, y, noise))
        x_t, obj = torch.empty_like(x0c), torch.empty_like(x0c)
        be.q_sample(x0c, yc, nz, t.to(torch.int64).contiguous(), m.m_t, m.variance_t, m.objective, x_t, obj)
        return x_t, obj

    # ------------------------------------------------------------------------------ p_sample
    def coef_table(self):
        m = self.model
        key = (m.m_t.data_ptr(), m.m_t._version, m.variance_t.data_ptr(), m.variance_t._version,
               id(m.steps), float(m.eta))
        if key != self._coef_key:
            self._coef = step_coefficients(m.m_t, m.variance_t, m.steps, m.eta)
            self._coef_key = key
        return self._coef

    def _step_index(self, i):
        m = self.model
        step = m.steps[i]
        t_val = int(step)                       # torch.full(..., dtype=long) truncates like this
        if not (0 <= t_val < m.num_timesteps):
            # the reference reaches a.gather(-1, t) with this value (model/utils.py:6)
            raise RuntimeError(f"index {t_val} is out of bounds for dimension 0 with size {m.num_timesteps}")
        return t_val, bool(step == 0)

    def p_sample(self, x_t, y, context, i, clip_denoised=False, noise=None, _fresh=False):
        m = self.model
        self._require_device(x_t)
        be = self.backend()
        t_val, is_last = self._step_index(i)
        B = x_t.shape[0]
        x_t = x_t.contiguous().float()
        y = y.contiguous().float()
        t = torch.full((B,), t_val, device=x_t.device, dtype=torch.long)
        eng = m.denoise_fn.engine()
        eng.num_timesteps = max(eng.num_timesteps, m.num_timesteps)
        eps = eng.forward(x_t, t, context, assume_fresh_weights=_fresh)
        if not is_last and noise is None:
            noise = self.noise_source(x_t) if self.noise_source is not None else torch.randn_like(x_t)
        out, x0 = torch.empty_like(x_t), torch.empty_like(x_t)
        be.p_sample(x_t, y, eps, None if is_last else noise.contiguous().float(), self.coef_table()[i].tolist(),
                    m.objective, bool(clip_denoised), is_last, out, x0)
        if is_last:
            return x0, x0
        return out, x0

    def p_sample_loop(self, y, context, clip_denoised, sample_mid_step, progress):
        m = self.model
        self._require_device(y)
        self.backend()
        m.denoise_fn.engine().refresh_weights()       # once per loop, not per step
        n = len(m.steps)
        it = progress(range(n), desc='sampling loop time step', total=n)
        if sample_mid_step:
            imgs, one_step_imgs = [y], []
            for i in it:
                img, x0_recon = self.p_sample(imgs[-1], y, context, i, clip_denoised, _fresh=True)
                imgs.append(img)
                one_step_imgs.append(x0_recon)
            return imgs, one_step_imgs
        if self.use_cuda_graph and y.is_cuda and getattr(self.backend(), "requires_cuda", False):
            with torch.cuda.device(y.device):         # capture/replay on the tensors' device, not the process default
                return self._graphed_loop(y, context, clip_denoised, it)
        img = y
        for i in it:
            img, _ = self.p_sample(img, y, context, i, clip_denoised, _fresh=True)
        return img

    # ------------------------------------------------------------------------------ CUDA-graph loop
    def _step_graph(self, y, context, clip):
        """Capture (UNet forward + fused bridge update + x <- x_next) once per
        (shape, clip, weight-address generation); every non-final step replays it with only the
        timestep vector, 7 coefficient floats and the noise buffer rewritten."""
        m = self.model
        be = self.backend()
        eng = m.denoise_fn.engine()
        ctx_is_y = context is y or context is None
        key = (tuple(y.shape), y.device, bool(clip), eng.generation, m.objective,
               None if context is None else tuple(context.shape), ctx_is_y,
               eng.pool_serial(y.device, (y.shape[0], y.shape[2], y.shape[3])))
        g = self._graphs.get(key)
        if g is not None:
            return g
        self._graphs.clear()                          # one live graph: frees the old static buffers
        dev = y.device
        st = {"x": torch.empty_like(y), "y": torch.empty_like(y), "noise": torch.empty_like(y),
              "eps": torch.empty_like(y), "out": torch.empty_like(y), "x0": torch.empty_like(y),
              "t": torch.zeros((y.shape[0],), dtype=torch.int64, device=dev),
              "coef": torch.zeros((7,), dtype=torch.float32, device=dev),
              "ctx": None}
        if context is not None:
            st["ctx"] = st["y"] if ctx_is_y else torch.empty_like(context)

        def step():
            eng.forward(st["x"], st["t"], st["ctx"], assume_fresh_weights=True, out=st["eps"])
            be.p_sample_dev(st["x"], st["y"], st["eps"], st["noise"], st["coef"], m.objective, clip, False,
                            st["out"], st["x0"])
            st["x"].copy_(st["out"])

        st["x"].copy_(y)
        st["y"].copy_(y)
        st["noise"].zero_()
        if st["ctx"] is not None and not ctx_is_y:
            st["ctx"].copy_(context)
        st["coef"].copy_(self.coef_table()[0].to(dev))
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            step()                                    # warm-up: fills the buffer pool, sets func attributes
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        # explicit capture stream on THIS device: torch.cuda.graph's default capture stream is created once per
        # process on whatever device was current then (a model on cuda:1 after one on cuda:0 captured nothing)
        with cabi.collector_paused(), torch.cuda.graph(graph, stream=side):
            step()
        st["graph"] = graph
        self._graphs[key] = st
        return st

    def _graphed_loop(self, y, context, clip_denoised, it):
        m = self.model
        y = y.contiguous().float()
        st = self._step_graph(y, context, bool(clip_denoised))
        dev = y.device
        coef_dev = self.coef_table().to(dev)
        steps_dev = m.steps.to(device=dev, dtype=torch.int64)
        st["x"].copy_(y)
        st["y"].copy_(y)
        if st["ctx"] is not None and st["ctx"] is not st["y"]:
            st["ctx"].copy_(context)
        img = None
        for i in it:
            t_val, is_last = self._step_index(i)
            if is_last:
                img, _ = self.p_sample(st["x"], st["y"], st["ctx"], i, clip_denoised, _fresh=True)
                break
            st["t"].copy_(steps_dev[i].expand_as(st["t"]))
            st["coef"].copy_(coef_dev[i])
            if self.noise_source is not None:
                st["noise"].copy_(self.noise_source(st["x"]))
            else:
                st["noise"].normal_()                 # same Philox consumption as torch.randn_like
            st["graph"].replay()
        if img is None:                               # schedule without a t == 0 step
            img = st["x"].clone()
        return img
