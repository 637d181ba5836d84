"""Public training API: one call per step, gradients exchanged by DeepReduce.

``Trainer.step(x, y)`` consumes device-resident inputs; ``Trainer.step_host(x, y)``
is the end-to-end form: pinned host batch → (async H2D on a copy stream,
double-buffered) → optional uint8→bf16 normalisation kernel → forward/backward →
fused gradient exchange overlapped with backward → optimizer → loss read back to
pinned host memory.  This mirrors what the reference's trainers
(grace-benchmarks ``trainer_grace.py`` / ``ncf_grace.py``, reference
run_deepreduce.sh:33,47) do around ``grc.step``.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .parallel.ddp import DeepReduceDDP


class Trainer:
    def __init__(self, model: nn.Module, params: dict, *, lr: float = 0.1, momentum: float = 0.9,
                 weight_decay: float = 1e-4, amp_dtype: Optional[torch.dtype] = torch.bfloat16,
                 channels_last: bool = False, loss_fn: Optional[Callable] = None, optimizer=None,
                 overlap: bool = True, bucket_cap_mb: float = 1e9, background_thread: bool = True,
                 blocks_per_sm: int = 2, u8_input: bool = False, accum_steps: int = 1, nvtx: bool = False,
                 check_every: int = 100, overlap_grid: Optional[int] = None):
        self.model = model
        self.device = next(model.parameters()).device
        self.is_cuda = self.device.type == "cuda"
        self.amp_dtype = amp_dtype if self.is_cuda else None
        self.channels_last = channels_last and self.is_cuda
        if self.channels_last:
            self.model = self.model.to(memory_format=torch.channels_last)
        self.loss_fn = loss_fn or F.cross_entropy
        self.ddp = DeepReduceDDP(self.model, params, overlap=overlap, bucket_cap_mb=bucket_cap_mb,
                                 background_thread=background_thread, blocks_per_sm=blocks_per_sm,
                                 overlap_grid=overlap_grid)
        if optimizer is None:
            # 'memory': 'dgc' accumulates the momentum before the exchange (momentum correction): the optimizer then
            # runs without one, whatever ``momentum`` says.  A user optimizer must do the same.  With 'weight_decay'
            # in the dict the memory adds the decay ahead of that momentum, and the dict's value replaces
            # ``weight_decay`` here: the optimizer runs without it ('weight_decay_exclude' and 'nesterov' live in the
            # memory as well).
            if params.get('memory') == 'dgc':
                momentum = 0.0
                if 'weight_decay' in params:
                    weight_decay = 0.0
            kw = dict(lr=lr, momentum=momentum, weight_decay=weight_decay)
            if self.is_cuda:
                kw["fused"] = True
            optimizer = torch.optim.SGD(self.model.parameters(), **kw)
        self.opt = optimizer
        self.u8_input = u8_input
        self.accum_steps = max(1, int(accum_steps))     # reference trainers' --grads_accumulated
        self._micro = 0
        # failure detection: the kernels' watchdogs (peer-flag wait, grid barrier, TMA, stage-2 overflow) set a device
        # status word instead of hanging; it is read back every `check_every` optimisation steps (0 = never)
        self.check_every = max(0, int(check_every))
        self._opt_steps = 0
        self.nvtx = nvtx and self.is_cuda
        self._copy_stream = torch.cuda.Stream(device=self.device) if self.is_cuda else None
        self._staged = None
        self._loss_host = torch.zeros(1, dtype=torch.float32).pin_memory() if self.is_cuda else torch.zeros(1)
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    # ---- device-resident step ------------------------------------------------
    def _prep(self, x):
        if self.u8_input and x.dtype == torch.uint8:
            from . import ops
            x = ops.u8_to_nhwc_norm(x).permute(0, 3, 1, 2)      # NHWC storage == channels_last NCHW view
        elif self.channels_last and x.dim() == 4:
            x = x.contiguous(memory_format=torch.channels_last)
        return x

    def _range(self, name):
        import contextlib
        return torch.cuda.nvtx.range(name) if self.nvtx else contextlib.nullcontext()

    def step(self, *inputs, target) -> torch.Tensor:
        """One optimisation step on device tensors; returns the loss (device scalar).  With
        ``accum_steps > 1`` gradients accumulate locally and are exchanged every ``accum_steps`` calls."""
        first = self._micro == 0
        last = self._micro == self.accum_steps - 1
        if first:
            self.ddp.zero_grad()
        self.ddp.set_exchange_enabled(last)
        inputs = tuple(self._prep(x) for x in inputs)
        with self._range("forward"):
            if self.amp_dtype is not None:
                with torch.autocast(device_type="cuda", dtype=self.amp_dtype):
                    out = self.model(*inputs)
            else:
                out = self.model(*inputs)
            loss = self.loss_fn(out.float() if torch.is_tensor(out) and out.is_floating_point() else out, target)
        with self._range("backward+exchange"):
            (loss / self.accum_steps if self.accum_steps > 1 else loss).backward()
        self._micro = (self._micro + 1) % self.accum_steps
        if last:
            with self._range("finish+optimizer"):
                self.ddp.finish()
                self.opt.step()
            self._opt_steps += 1
            if self.is_cuda:
                self.ddp.check_async()            # every step, no host sync: raises one step after a watchdog fired
            if self.check_every and self._opt_steps % self.check_every == 0:
                self.ddp.check()                  # raises with rank / bucket / watchdog name
        return loss.detach()

    # ---- end-to-end step (host in, host out) -----------------------------------
    def _stage(self, host_inputs, host_target):
        with torch.cuda.stream(self._copy_stream):
            dev = tuple(t.to(self.device, non_blocking=True) for t in host_inputs)
            tgt = host_target.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in host_inputs) + host_target.numel() * host_target.element_size()
        return dev, tgt, ev

    def step_host(self, host_inputs, host_target, next_batch=None) -> float:
        """``host_inputs``/``host_target`` are pinned CPU tensors for THIS step;
        ``next_batch`` (optional) is prefetched while this step computes."""
        if not self.is_cuda:
            return float(self.step(*host_inputs, target=host_target))
        if self._staged is None:
            self._staged = self._stage(host_inputs, host_target)
        dev, tgt, ev = self._staged
        torch.cuda.current_stream().wait_event(ev)
        self._staged = self._stage(*next_batch) if next_batch is not None else None
        loss = self.step(*dev, target=tgt)
        self._loss_host.copy_(loss.reshape(1), non_blocking=True)
        self.d2h_bytes = 4
        torch.cuda.current_stream().synchronize()
        for t in dev:
            t.record_stream(torch.cuda.current_stream())
        return float(self._loss_host[0])

    def close(self):
        self.ddp.close()
