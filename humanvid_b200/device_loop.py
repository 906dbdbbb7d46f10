"""The denoising loop of ``Pose2VideoPipeline.__call__`` (src/pipelines/pipeline_pose2vid_long.py:454-563) with every
per-timestep operation on the device (SURVEY 8f-2):

    for t in timesteps:                                   one CUDA graph, replayed per timestep
        for window in context_windows:                    (context.py:15-42; 1 window at 24 frames, 3 at 48)
            x   = latents[:, :, window].repeat(2)         hv_op_window_gather
            eps = denoising_unet(x, t, ehs, cond[window]) hv_unet3d_forward, t read from a device table
        latents = DDIM(CFG(mean over windows of eps))     hv_op_cfg_ddim_step (accumulate, /counter, CFG mix, DDIM in one kernel)
        step   += 1                                       hv_op_advance_index

The step-invariant PoseGuider / CameraPoseEncoder features are computed once per window before the loop (the reference
recomputes them every step, :526-537).  Nothing in the loop touches the host: the timestep and the DDIM coefficients
come from device tables indexed by a device-resident step counter, which is what makes one captured step replayable.

With ``units`` (humanvid_b200.distributed) the UNet work of a step is split into (window x CFG-half) units over ranks;
the predictions are exchanged with one all-gather per step and every rank runs the glue kernel redundantly.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional, Sequence

import torch

from . import _native as N


def window_inverse_map(windows: Sequence[Sequence[int]], num_frames: int) -> torch.Tensor:
    """[num_frames][K] int32: the (window * Fw + position) slots that hold each frame, -1 padded (the ``counter`` of
    pipeline_pose2vid_long.py:550-552 is the number of valid entries of a row)."""
    fw = len(windows[0])
    slots: List[List[int]] = [[] for _ in range(num_frames)]
    for w, win in enumerate(windows):
        if len(win) != fw:
            raise ValueError("all context windows must have the same length")
        for i, f in enumerate(win):
            slots[f].append(w * fw + i)
    if any(len(s) == 0 for s in slots):
        raise ValueError("context windows do not cover every frame")
    k = max(len(s) for s in slots)
    return torch.tensor([s + [-1] * (k - len(s)) for s in slots], dtype=torch.int32)


class DeviceDenoiseLoop:
    """Owns the static buffers of one clip's denoising loop and runs it step by step (eagerly or as a replayed CUDA graph)."""

    def __init__(self, unet, scheduler, latents: torch.Tensor, windows: Sequence[Sequence[int]], encoder_hidden_states: torch.Tensor,
                 cond_features: Sequence[Optional[torch.Tensor]], guidance_scale: float, cfg_on: bool,
                 exchange: Optional[Callable] = None, my_units: Optional[Sequence] = None, all_units: Optional[Sequence] = None):
        if not latents.is_cuda:
            raise RuntimeError("DeviceDenoiseLoop needs CUDA tensors (humanvid_b200 has no CPU path)")
        self.unet, self.scheduler = unet, scheduler
        self.cfg_on, self.guidance = bool(cfg_on), float(guidance_scale)
        self.latents = latents.to(torch.float16).contiguous().clone()
        self.Bl, self.Cl, self.F, self.H, self.W = self.latents.shape
        self.windows = [list(w) for w in windows]
        self.Fw = len(self.windows[0])
        dev = latents.device
        self.win_idx = [torch.tensor(w, dtype=torch.int32, device=dev) for w in self.windows]
        inv = window_inverse_map(self.windows, self.F)
        self.K = inv.shape[1]
        self.inv = inv.to(dev).contiguous()
        self.ehs = encoder_hidden_states.to(torch.float16).contiguous()
        self.cond = [None if c is None else c.to(torch.float16).contiguous() for c in cond_features]
        self.coef = scheduler.coef_table().to(dev).contiguous()                      # [steps][4] fp32
        self._ts_host = [int(t) for t in scheduler._host_timesteps]
        self.ts = torch.tensor(self._ts_host, dtype=torch.int64, device=dev)
        self.step_index = torch.zeros(1, dtype=torch.int32, device=dev)
        self.pred_type = {"v_prediction": 0, "epsilon": 1}[scheduler.config.prediction_type]
        self.exchange, self.my_units, self.all_units = exchange, my_units, all_units
        if exchange is not None and hasattr(exchange, "prime"):   # ranks that own no unit still take part in the all-gather
            exchange.prime((self.Bl, self.Cl, self.Fw, self.H, self.W), dev, torch.float16)
        self._graph = None
        self._h = unet._sync_native()
        self._epoch = unet._epoch   # a rebuilt handle (weights, dtype, FP8 mode) may reuse the old one's address
        N.check(N.lib().hv_set_timestep_source(self._h, C.c_void_p(self.ts.data_ptr()), C.c_void_p(self.step_index.data_ptr())), self._h)

    def close(self):
        if self._h is not None and self.unet._handle is not None:
            N.lib().hv_set_timestep_source(self.unet._handle, None, None)
        self._h = None
        self._graph = None

    # ---- reuse for the next clip of the same shape: the captured graph stays valid because every buffer it touches is static ------
    def signature(self):
        return (tuple(self.latents.shape), tuple(tuple(w) for w in self.windows), self.cfg_on, self.guidance, tuple(self.scheduler._host_timesteps),
                self.pred_type, tuple(None if c is None else tuple(c.shape) for c in self.cond), tuple(self.ehs.shape))

    def matches(self, unet, scheduler, latents, windows, encoder_hidden_states, cond_features, guidance_scale, cfg_on) -> bool:
        return (self._h is not None and unet is self.unet and unet._handle is not None and unet._sync_native().value == self._h.value
                and unet._epoch == self._epoch
                and self.exchange is None and tuple(latents.shape) == tuple(self.latents.shape)
                and [list(w) for w in windows] == self.windows and bool(cfg_on) == self.cfg_on and float(guidance_scale) == self.guidance
                and [int(t) for t in scheduler._host_timesteps] == self._ts_host and tuple(encoder_hidden_states.shape) == tuple(self.ehs.shape)
                and [None if c is None else tuple(c.shape) for c in cond_features] == [None if c is None else tuple(c.shape) for c in self.cond])

    def reload(self, latents, encoder_hidden_states, cond_features):
        """New clip, same shapes: copy the inputs into the static buffers the captured step reads, rewind the step counter and hand the
        (new) reference banks to the handle -- inside the graph the bank pointers are the handle's own buffers, which stay put."""
        self.latents.copy_(latents.to(torch.float16))
        self.ehs.copy_(encoder_hidden_states.to(torch.float16))
        for dst, src in zip(self.cond, cond_features):
            if dst is not None:
                dst.copy_(src.to(torch.float16))
        self.step_index.zero_()
        self.unet._push_banks(self._h)
        N.check(N.lib().hv_set_timestep_source(self._h, C.c_void_p(self.ts.data_ptr()), C.c_void_p(self.step_index.data_ptr())), self._h)

    def detach(self):
        """Between clips: the UNet takes its timestep from the host argument again; buffers and the captured graph are kept."""
        if self._h is not None and self.unet._handle is not None:
            N.lib().hv_set_timestep_source(self.unet._handle, None, None)

    # ---- one timestep ---------------------------------------------------------------------------------------------
    def _gather(self, w: int, repeat: int) -> torch.Tensor:
        out = torch.empty((repeat * self.Bl, self.Cl, self.Fw, self.H, self.W), device=self.latents.device, dtype=torch.float16)
        N.check(N.lib().hv_op_window_gather(N.ptr(self.latents), N.ptr(self.win_idx[w]), N.ptr(out), N.i64(self.Bl), N.i64(self.Cl), N.i64(self.F),
                                            N.i64(self.Fw), N.i64(self.H * self.W), N.i32(repeat), N.stream()))
        return out

    def _predict_windows(self):
        """-> (uncond[w], cond[w]) tensors of shape (Bl, C, Fw, H, W)."""
        un, co = [], []
        if self.exchange is None:
            rep = 2 if self.cfg_on else 1
            for w in range(len(self.windows)):
                x = self._gather(w, rep)
                pred = self.unet(x, 0, self.ehs[: x.shape[0]], pose_cond_fea=self.cond[w], return_dict=False)[0]
                un.append(pred[: self.Bl])
                co.append(pred[self.Bl:] if self.cfg_on else None)
            return un, co
        # multi-GPU: this rank runs its (window, half) units at batch Bl with the one-half flags, then one all-gather
        mine = []
        for (w, half) in self.my_units:
            x = self._gather(w, 1)
            self.unet._forward_flags = 4 if half == 1 else 2           # HV_FLAG_COND_ONLY / HV_FLAG_UNCOND_ONLY
            try:
                e = self.ehs[half * self.Bl:(half + 1) * self.Bl] if self.cfg_on else self.ehs[: self.Bl]
                c = self.cond[w]
                c = None if c is None else c[: self.Bl]
                mine.append(self.unet(x, 0, e, pose_cond_fea=c, return_dict=False)[0])
            finally:
                self.unet._forward_flags = None
        preds = self.exchange(mine)                                     # {unit: tensor} for all units
        for w in range(len(self.windows)):
            un.append(preds[(w, 0)])
            co.append(preds[(w, 1)] if self.cfg_on else None)
        return un, co

    def _one_step(self):
        un, co = self._predict_windows()
        n = len(un)
        pu = (C.c_void_p * n)(*[t.data_ptr() for t in un])
        pc = (C.c_void_p * n)(*[t.data_ptr() for t in co]) if self.cfg_on else None
        N.check(N.lib().hv_op_cfg_ddim_step(pu, pc, N.i32(n), N.ptr(self.inv), N.i32(self.K), N.ptr(self.coef), N.ptr(self.step_index),
                                            N.ptr(self.latents), N.i64(self.Bl), N.i64(self.Cl), N.i64(self.F), N.i64(self.Fw), N.i64(self.H * self.W),
                                            C.c_float(self.guidance), N.i32(self.pred_type), N.stream()))
        N.check(N.lib().hv_op_advance_index(N.ptr(self.step_index), N.stream()))
        self._keep = (un, co)   # the prediction buffers must outlive the asynchronous launch

    # ---- the loop -------------------------------------------------------------------------------------------------
    def run(self, num_steps: Optional[int] = None, use_graph: bool = True, steps_per_graph: int = 1) -> torch.Tensor:
        n = len(self.scheduler._host_timesteps) if num_steps is None else int(num_steps)
        if self.exchange is not None:
            use_graph = False   # the NCCL all-gather of the unit split stays outside graphs (one collective per step)
        if not use_graph:
            for _ in range(n):
                self._one_step()
            return self.latents
        if n % steps_per_graph:
            raise ValueError("num_steps must be a multiple of steps_per_graph")
        if self._graph is None or self._graph[1] != steps_per_graph:
            # warm-up outside capture (lazy kernel attributes, workspace reservation), then restore the loop state
            saved = self.latents.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._one_step()
            torch.cuda.current_stream().wait_stream(side)
            self.latents.copy_(saved)
            self.step_index.zero_()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(steps_per_graph):
                    self._one_step()
            self._graph = (g, steps_per_graph)
        for _ in range(n // steps_per_graph):
            self._graph[0].replay()
        return self.latents
