"""DDP communication hook: the fused DeepReduce exchange on torch ``DistributedDataParallel``'s gradient buckets.

For users who keep torch DDP (``no_sync()``, ``find_unused_parameters``, ``static_graph``, its bucket sizing, their
training loop) and add compression through its hook API, the way torch's PowerSGD hook ships::

    ddp = DDP(model, device_ids=[rank])
    state = register_deepreduce_hook(ddp, params)          # params: the dict DeepReduceDDP takes

Routing is ``DeepReduceDDP``'s:

CUDA bucket + ``fused_path(params)``   -> fused engine (one persistent kernel per bucket)
``'compressor': 'none'``                 -> torch's default all-reduce (mean, or sum with ``'average': False``)
anything else (CPU/gloo, other codecs) -> GRACE per-tensor path (``grc.step`` on the bucket's gradient views)

DDP packs a bucket's gradients back to back, unpadded, at arbitrary offsets; the engine wants every tensor on a
32-element boundary, large tensors chunked (``parallel/plan.py``).  Each bucket layout gets its own plan, engine and
segment table, built the first time the hook meets it; ``bucket_pack`` / ``bucket_unpack`` (``ops/csrc/repack.cu``)
move the whole bucket in one launch each way.  DDP rebuilds its buckets after the first iteration, so a run meets two
layouts: the residual of every parameter is carried from the old engine into the new one (DESIGN.md, "DDP
communication hook"), and with ``'memory': 'dgc'`` its momentum too.  That memory holds the momentum, so the optimizer
stepping the DDP model must run without one (e.g. ``torch.optim.SGD(..., momentum=0)``).  With ``'weight_decay'`` in
the dict the memory adds the decay ahead of its momentum, reading the parameters of each bucket, so that optimizer also
runs with ``weight_decay=0``.  The parameters are read in the order of their gradients in the bucket, i.e. in their
storage order, which DDP gives a dense parameter's gradient; their layouts must not change after DDP built its buckets.
``'clip_norm'`` clips each parameter's gradient inside the memory, in both routes, because the hook runs inside backward
and no user code can clip in between; the norm is per parameter, summed in the gradient's order in the bucket.
``'nesterov'`` and ``'weight_decay_exclude'`` apply in both routes too; the patterns match the module's parameter
names, the names the checkpoint is keyed by, and a pattern that matches none of them raises.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from .ddp import (BUCKET_DTYPES, engine_split_numel, fused_path, grace_state_dict, load_grace_state_dict, make_engine,
                  make_grc, stage_plans)
from ..grace.memory import check_exclude_patterns
from .engine import BucketEngine, StatusPoller, total_stats
from .plan import BucketPlan, split_large

# the checkpoint key of each engine memory buffer (``BucketEngine.memory_buffers``), a map by parameter name
MEMORY_KEYS = {"resid": "residuals", "mom": "momentum"}


# ---------------------------------------------------------------------------
# segment tables and the torch reference of the repack
# ---------------------------------------------------------------------------
def bucket_segments(bucket) -> List[Tuple[int, int]]:
    """(element offset in ``bucket.buffer()``, numel) of every gradient of a DDP ``GradBucket``, in bucket order."""
    buf = bucket.buffer()
    base, es = buf.data_ptr(), buf.element_size()
    return [((g.data_ptr() - base) // es, g.numel()) for g in bucket.gradients()]


def segment_table(segments: Sequence[Tuple[int, int]], plan: BucketPlan, owner: Sequence[int]) -> torch.Tensor:
    """Host int64 [n, 3] rows ``{ddp_off, eng_off, numel}``: parameter i of the bucket is the DDP range ``segments[i]``
    and starts at its first plan tensor in the engine's buffer (a split parameter's chunks are whole tiles, hence
    contiguous there).  ``owner[j]``: the parameter plan tensor j belongs to (``split_large``)."""
    first: Dict[int, int] = {}
    for j, o in enumerate(owner):
        first.setdefault(o, plan.tensors[j].elem_off)
    rows = [[int(d), first[i], int(n)] for i, (d, n) in enumerate(segments)]
    return torch.tensor(rows, dtype=torch.int64).reshape(-1, 3)


def pack_reference(ddp_buf: torch.Tensor, eng_buf: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """torch indexing version of ``bucket_pack``: every segment copied from the DDP buffer into the engine's, in place."""
    for d, e, n in table.tolist():
        eng_buf[e:e + n].copy_(ddp_buf[d:d + n])
    return eng_buf


def unpack_reference(eng_buf: torch.Tensor, ddp_buf: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """torch indexing version of ``bucket_unpack``: every segment copied from the engine buffer back into DDP's."""
    for d, e, n in table.tolist():
        ddp_buf[d:d + n].copy_(eng_buf[e:e + n])
    return ddp_buf


class _Layout:
    """One DDP bucket layout on the fused path: plan, engine, segment table and repack object."""

    def __init__(self, key, index, params, names, segments, plan, engine, table, repack):
        self.key, self.index = key, index
        self.params, self.names, self.segments = params, names, segments
        self.plan, self.engine, self.table, self.repack = plan, engine, table, repack
        self.eng_off = [int(r[1]) for r in table.tolist()]
        self.slot = {id(p): i for i, p in enumerate(params)}
        self.live = len(params)          # parameters whose residual still lives in this engine

    def memory_of(self, p) -> Dict[str, torch.Tensor]:
        """The parameter's slice of each of the engine's memory buffers, by buffer name."""
        i = self.slot[id(p)]
        lo, hi = self.eng_off[i], self.eng_off[i] + self.segments[i][1]
        return {k: t[lo:hi] for k, t in self.engine.memory_buffers().items()}

    def resid_of(self, p) -> torch.Tensor:
        return self.memory_of(p)["resid"]

    def mom_of(self, p) -> torch.Tensor:
        return self.memory_of(p)["mom"]


# ---------------------------------------------------------------------------
# state + hook
# ---------------------------------------------------------------------------
class DeepReduceHookState:
    """State of :func:`deepreduce_hook` for one DDP model: the engines of the bucket layouts met so far, the side stream
    the fused buckets run on, and the GRACE compressor of the per-tensor path.

    ``params`` is the dict ``DeepReduceDDP`` takes.  ``module`` is the model (or the DDP wrapper around it): its
    parameter names key the checkpoint.  ``blocks_per_sm``, ``use_history`` and ``overlap_grid`` mean what they mean for
    ``DeepReduceDDP``."""

    def __init__(self, params: dict, module: nn.Module, process_group=None, *, blocks_per_sm: int = 2,
                 use_history: bool = True, overlap_grid: Optional[int] = None):
        if isinstance(module, nn.parallel.DistributedDataParallel):
            module = module.module
        self.params = dict(params)
        self.module = module
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.blocks_per_sm, self.use_history = int(blocks_per_sm), bool(use_history)
        self.overlap_grid_cap = int(overlap_grid if overlap_grid is not None else (self.params.get('overlap_grid', 0) or 0))
        self.average = bool(self.params.get('average', True))
        self.dense = self.params.get('compressor', 'none') in ('none', None)
        self.fused_params = not self.dense and fused_path(self.params)
        from ..config import warmup_from_params
        self.warmup = warmup_from_params(self.params)   # sparsity warm-up: stages counted in exchanges (hook calls)
        self._names: Dict[int, str] = {id(p): n for n, p in module.named_parameters()}
        if self.params.get('memory') == 'dgc':     # a pattern that matches nothing is a typo: refuse it
            # over the parameters DDP exchanges (those that require a gradient), as DeepReduceDDP checks them
            check_exclude_patterns(self.params.get('weight_decay_exclude'),
                                   [n for n, p in module.named_parameters() if p.requires_grad])
        self._layouts: List[_Layout] = []            # every engine not yet closed
        self._by_index: Dict[int, _Layout] = {}      # the layout a bucket index had last
        self._owner: Dict[int, _Layout] = {}         # id(parameter) -> the layout holding its residual
        # the loaded memory of parameters no engine holds yet, by buffer name ('dgc' engines add the momentum)
        buffers = ("resid", "mom") if self.params.get('memory') == 'dgc' else ("resid",)
        self._pending: Dict[str, Dict[str, torch.Tensor]] = {k: {} for k in buffers}
        self._pending_epoch = 0
        self._plans: Dict[tuple, list] = {}          # warm-up: every stage's plan of a layout, built when first met
        self._stream: Optional[torch.cuda.Stream] = None
        self.grc = None
        self.step_count = 0
        self._status = StatusPoller()

    # ---- routing ------------------------------------------------------------------
    def path(self, buffer: torch.Tensor) -> str:
        """'fused', 'dense' or 'grace': where a bucket with this buffer goes."""
        if self.dense:
            return "dense"
        if buffer.is_cuda and self.fused_params:
            return "fused"
        return "grace"

    def _name(self, p) -> str:
        n = self._names.get(id(p))
        if n is None:
            raise ValueError("a bucket holds a parameter that is not one of the module's (pass the model DDP wraps)")
        return n

    def _run(self, bucket) -> torch.futures.Future:
        buf = bucket.buffer()
        path = self.path(buf)
        if path == "fused":
            if buf.dtype not in BUCKET_DTYPES:
                raise ValueError(f"bucket {bucket.index()} is {buf.dtype}: the fused engine takes fp32 or bf16 buckets")
            fut = self._fused(bucket, buf)
        elif path == "dense":
            fut = self._dense(bucket, buf)
        else:
            fut = self._grace(bucket, buf)
        if bucket.is_last():
            self.step_count += 1
        return fut

    def _dense(self, bucket, buf):
        if self.average:
            from torch.distributed.algorithms.ddp_comm_hooks.default_hooks import allreduce_hook
            return allreduce_hook(self.group, bucket)
        work = dist.all_reduce(buf, group=self.group, async_op=True)
        return work.get_future().then(lambda f: f.value()[0])

    def _make_grc(self):
        # bucket.gradients() are plain reshapes of the flat bucket, which holds every gradient in its parameter's
        # storage order: a memory that reads the parameters reads them in that order too
        self.grc = make_grc(self.params, self.module.named_parameters(), storage_order=True)

    def _grace(self, bucket, buf):
        if self.grc is None:
            self._make_grc()
        for p, g in zip(bucket.parameters(), bucket.gradients()):
            out = self.grc.step(g, self._name(p))
            g.copy_(out.view_as(g))
        fut = torch.futures.Future(devices=[buf.device]) if buf.is_cuda else torch.futures.Future()
        fut.set_result(buf)
        return fut

    # ---- fused path -------------------------------------------------------------
    def _side_stream(self, dev) -> torch.cuda.Stream:
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=dev, priority=-1)
        return self._stream

    def _fused(self, bucket, buf):
        dev = buf.device
        side = self._side_stream(dev)
        # every bucket runs on ONE side stream, in the order DDP hands them over (bucket index order, the same on every
        # rank): the persistent kernels of two buckets can never be ordered differently on two ranks, which is the
        # cross-rank inversion DeepReduceDDP's launch thread has to guard against
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.device(dev), torch.cuda.stream(side):
            lay = self._layout_for(bucket, buf)
            eng = lay.engine
            lay.repack.pack(buf, eng.grad)
            # the engine's own step counter, never reset: peer flags carry the epoch (see DeepReduceDDP._launch_bucket)
            eng.epoch = eng.epoch + 1
            # buckets that arrive while backward is still running get a capped grid, so that the persistent kernel does
            # not take every SM from cuDNN / cuBLAS; the last bucket (nothing left to overlap with) gets the whole GPU
            last = bucket.is_last()
            eng.ctx.set_grid_cap(0 if last or self.overlap_grid_cap <= 0 else self.overlap_grid_cap)
            eng.step(eng.epoch)
            lay.repack.unpack(eng.grad, buf)
            # CUDA-aware future completed on the side stream: DDP's consumer stream waits on its event, not the host
            fut = torch.futures.Future(devices=[dev])
            fut.set_result(buf)
        return fut

    def _layout_for(self, bucket, buf) -> _Layout:
        params = bucket.parameters()
        segments = bucket_segments(bucket)
        # the warm-up stage is part of the layout: a new stage builds the stage's engine and carries the state into it
        stage = 0 if self.warmup is None else self.warmup.stage(self.step_count)
        key = (bucket.index(), tuple(id(p) for p in params), tuple(segments), buf.numel(), buf.dtype, stage)
        lay = self._by_index.get(bucket.index())
        if lay is not None and lay.key == key:
            return lay
        return self._new_layout(key, bucket.index(), params, segments, buf, stage)

    def _new_layout(self, key, index, params, segments, buf, stage=0) -> _Layout:
        """Plan, engine and segment table of a layout met for the first time, with the residuals carried over.

        Collective at W > 1 (IPC handle exchange and barriers in ``BucketEngine``, the partition calibration's exchange
        steps, and ``BucketEngine.close`` of a superseded engine), here inside a DDP hook.  That is safe only because
        every rank meets the same layouts in the same order: DDP calls the hook in bucket-index order, and its bucket
        rebuild broadcasts rank 0's order, so every rank builds and closes the same engines at the same point.  A
        sparsity warm-up stage switch meets every bucket again, on the same exchange on every rank (each counts the same
        hook calls).  Every stage's plan of a layout is built when the layout is first met (and kept), so a stage a plan
        refuses raises on the first exchange."""
        from .. import ops
        names = [self._name(p) for p in params]
        numels = [n for _, n in segments]
        shapes = [tuple(p.shape) for p in params]
        numels, pnames, shapes, owner = split_large(numels, names, shapes,
                                                     engine_split_numel(self.params, self.blocks_per_sm))
        plans = self._plans.get(key[:-1])
        if plans is None:
            plans = stage_plans(numels, pnames, shapes, self.params, self.warmup)
            if self.warmup is not None:
                self._plans[key[:-1]] = plans
        plan = plans[stage]
        # 'weight_decay': the engine reads every parameter in storage order, where the bucket holds its gradient (DDP
        # lays a dense parameter's gradient out with the parameter's strides; bind_parameters refuses any other).  The
        # parameters' layouts are recorded here and must stay as DDP found them: a later change raises at the next step
        # calibration (inside make_engine) resets the residual: it runs before the carry below
        eng = make_engine(plan, self.params, device=buf.device, group=self.group, use_history=self.use_history,
                          blocks_per_sm=self.blocks_per_sm, grad_dtype=buf.dtype, parameters=list(params), owner=owner,
                          names=names)
        table = segment_table(segments, plan, owner)
        repack = ops.cuda_module().Repack(table, buf.numel(), plan.total_elems, eng.grad)
        lay = _Layout(key, index, list(params), names, list(segments), plan, eng, table, repack)
        # carry every parameter's memory, by parameter identity and in storage order, from the engine that held it;
        # an engine closes once none of its parameters is left in it
        for p, n in zip(params, names):
            dst = lay.memory_of(p)
            old = self._owner.get(id(p))
            if old is not None:
                for k, t in old.memory_of(p).items():
                    dst[k].copy_(t)
                if self.warmup is not None:
                    # a warm-up run's engines only move their epochs forward, across stage switches and DDP's rebuild
                    # alike; without the keys a new layout keeps its own count, as it always has (its arena is new
                    # and zeroed, so no stale flag can match)
                    eng.epoch = max(eng.epoch, old.engine.epoch)
                old.live -= 1
                if old.live == 0:
                    self._close_layout(old)
            else:
                for k, pending in self._pending.items():
                    if n in pending:
                        dst[k].copy_(pending.pop(n).to(eng.device, torch.float32).reshape(-1))
            self._owner[id(p)] = lay
        eng.epoch = max(eng.epoch, self._pending_epoch)
        self._by_index[index] = lay
        self._layouts.append(lay)
        return lay

    def _close_layout(self, lay: _Layout):
        lay.engine.close()
        self._layouts.remove(lay)
        for i in [i for i, l in self._by_index.items() if l is lay]:
            del self._by_index[i]

    @property
    def engines(self) -> List[BucketEngine]:
        """The live engines, oldest layout first."""
        return [l.engine for l in self._layouts]

    # ---- checks -----------------------------------------------------------------
    def check(self):
        """Read the engines' device status words (one small D2H each); raises with rank and bucket on a watchdog."""
        for lay in self._layouts:
            try:
                lay.engine.check_status()
            except RuntimeError as err:
                raise RuntimeError(f"[rank {self.rank}/{self.world}] DDP bucket {lay.index} "
                                   f"({len(lay.params)} tensors, step {self.step_count}): {err}") from err

    def check_async(self):
        """Per-step failure detection without a host sync (as ``DeepReduceDDP.check_async``): copy the status words to
        pinned memory on the current stream, and inspect the copy the previous call enqueued once it has landed."""
        bad = self._status.poll([(lay.index, lay.engine) for lay in self._layouts])
        if bad is not None:
            raise RuntimeError(f"[rank {self.rank}/{self.world}] DDP bucket {bad[0]} (step {self.step_count}): {bad[1]}")

    # ---- accounting ---------------------------------------------------------------
    def dense_bytes(self) -> int:
        return sum(p.numel() * p.element_size() for p in self.module.parameters() if p.requires_grad)

    def wire_bytes_per_step(self) -> int:
        if self._layouts:
            return sum(l.plan.wire_bytes() for l in self._layouts)
        if self.dense:
            return self.dense_bytes()
        if self.grc is not None:
            return int(self.grc.bytes_sent / max(self.step_count, 1))
        return 0

    def exchange_stats(self) -> dict:
        """Device-side counters of the last exchanged step, summed over the live engines (fused path); synchronises."""
        if not self._layouts:
            return {"wire_bytes": self.wire_bytes_per_step(), "dense_bytes": self.dense_bytes()}
        return total_stats(self.engines)

    # ---- checkpoint / resume ----------------------------------------------------------
    def _held_memory(self) -> Dict[str, Dict[str, torch.Tensor]]:
        """By parameter name, ``_Layout.memory_of`` of every parameter in the engine that holds it."""
        return {n: lay.memory_of(p) for lay in self._layouts for p, n in zip(lay.params, lay.names)
                if self._owner.get(id(p)) is lay}

    def state_dict(self) -> dict:
        """Keyed by parameter name, so that a checkpoint loads into a run with other buckets: the residual of every
        parameter (fused path, flat in storage order; with 'dgc' its momentum too, under ``"momentum"``) or the GRACE
        memory (per-tensor path)."""
        if self._layouts:
            torch.cuda.synchronize(self._layouts[0].engine.device)
        memory = {k: {n: t.clone() for n, t in pending.items()} for k, pending in self._pending.items()}
        for n, held in self._held_memory().items():
            for k, t in held.items():
                memory[k][n] = t.detach().cpu().clone()
        out = {"step": self.step_count, "epoch": max([self._pending_epoch] + [e.epoch for e in self.engines])}
        out.update((MEMORY_KEYS[k], m) for k, m in memory.items())
        if self.grc is not None:
            out.update(grace_state_dict(self.grc, self.warmup))
        return out

    def load_state_dict(self, state: dict):
        self.step_count = int(state.get("step", 0))
        # engine epochs only move forward (BucketEngine.load_state_dict): peer flags carry epochs already used
        self._pending_epoch = max(self._pending_epoch, int(state.get("epoch", 0)))
        for e in self.engines:
            e.epoch = max(e.epoch, self._pending_epoch)
        held = self._held_memory()
        if ("mom" in self._pending) != ("momentum" in state) and state.get("residuals"):
            raise ValueError("hook state of another memory: 'dgc' states carry a 'momentum' map, other states do not")
        self._pending = {k: {} for k in self._pending}
        for k, pending in self._pending.items():
            for n, t in state.get(MEMORY_KEYS[k], {}).items():
                if n in held:
                    held[n][k].copy_(t.to(held[n][k].device, torch.float32).reshape(-1))
                else:
                    pending[n] = t.detach().cpu().clone()
        if "memory" in state:
            if self.grc is None:
                self._make_grc()
            load_grace_state_dict(self.grc, state, self.warmup, next(self.module.parameters()).device)

    def close(self):
        """Release the engines and their arenas (collective at W > 1)."""
        for lay in list(self._layouts):
            self._close_layout(lay)
        self._owner.clear()
        self._by_index.clear()


def deepreduce_hook(state: DeepReduceHookState, bucket: dist.GradBucket) -> torch.futures.Future[torch.Tensor]:
    """DDP communication hook: ``ddp.register_comm_hook(state, deepreduce_hook)``.  The future's value is
    ``bucket.buffer()`` holding the aggregate (the mean over ranks unless ``'average': False``)."""
    return state._run(bucket)


def register_deepreduce_hook(ddp_model: nn.parallel.DistributedDataParallel, params: dict, **kw) -> DeepReduceHookState:
    """Build a :class:`DeepReduceHookState` for ``ddp_model`` (its process group unless ``process_group`` is given),
    register :func:`deepreduce_hook` and return the state."""
    group = kw.pop("process_group", getattr(ddp_model, "process_group", None))
    state = DeepReduceHookState(params, ddp_model.module, group, **kw)
    ddp_model.register_comm_hook(state, deepreduce_hook)
    return state
