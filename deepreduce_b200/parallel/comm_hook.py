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
"""
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from ..grace.helper import sparsifier_of
from .ddp import BUCKET_DTYPES, engine_split_numel, fused_path, make_engine, stage_plans
from .engine import STATUS_NAMES, BucketEngine
from .plan import BucketPlan, split_large


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

    def resid_of(self, p) -> torch.Tensor:
        i = self.slot[id(p)]
        return self.engine.resid[self.eng_off[i]:self.eng_off[i] + self.segments[i][1]]

    def mom_of(self, p) -> torch.Tensor:
        """The parameter's 'dgc' momentum in this engine (same place as its residual)."""
        i = self.slot[id(p)]
        return self.engine.mom[self.eng_off[i]:self.eng_off[i] + self.segments[i][1]]


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
        self._layouts: List[_Layout] = []            # every engine not yet closed
        self._by_index: Dict[int, _Layout] = {}      # the layout a bucket index had last
        self._owner: Dict[int, _Layout] = {}         # id(parameter) -> the layout holding its residual
        self._pending: Dict[str, torch.Tensor] = {}  # loaded residuals of parameters no engine holds yet
        self._pending_mom: Dict[str, torch.Tensor] = {}  # ... and their loaded 'dgc' momenta
        self.dgc = self.params.get('memory') == 'dgc'
        self._pending_epoch = 0
        self._plans: Dict[tuple, list] = {}          # warm-up: every stage's plan of a layout, built when first met
        self._stream: Optional[torch.cuda.Stream] = None
        self.grc = None
        self.step_count = 0
        self._status_host = None
        self._status_event = None

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
        from ..wrappers import deepreduce_from_params
        self.grc = deepreduce_from_params(self.params)
        if hasattr(self.grc.memory, "bind_parameters"):           # 'dgc' weight decay reads the parameters
            # bucket.gradients() are plain reshapes of the flat bucket, which holds every gradient in its
            # parameter's storage order: the memory reads the parameters in that order too
            self.grc.memory.bind_parameters(self.module.named_parameters(), storage_order=True)

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
                          blocks_per_sm=self.blocks_per_sm, grad_dtype=buf.dtype, parameters=list(params), owner=owner)
        table = segment_table(segments, plan, owner)
        repack = ops.cuda_module().Repack(table, buf.numel(), plan.total_elems, eng.grad)
        lay = _Layout(key, index, list(params), names, list(segments), plan, eng, table, repack)
        # carry every parameter's residual, by parameter identity and in storage order, from the engine that held it;
        # an engine closes once none of its parameters is left in it
        for p, n in zip(params, names):
            dst = lay.resid_of(p)
            old = self._owner.get(id(p))
            if old is not None:
                dst.copy_(old.resid_of(p))
                if self.dgc:
                    lay.mom_of(p).copy_(old.mom_of(p))
                if self.warmup is not None:
                    # a warm-up run's engines only move their epochs forward, across stage switches and DDP's rebuild
                    # alike; without the keys a new layout keeps its own count, as it always has (its arena is new
                    # and zeroed, so no stale flag can match)
                    eng.epoch = max(eng.epoch, old.engine.epoch)
                old.live -= 1
                if old.live == 0:
                    self._close_layout(old)
            else:
                if n in self._pending:
                    dst.copy_(self._pending.pop(n).to(dst.device, torch.float32).reshape(-1))
                if self.dgc and n in self._pending_mom:
                    lay.mom_of(p).copy_(self._pending_mom.pop(n).to(dst.device, torch.float32).reshape(-1))
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
        if self._status_host is not None and self._status_event.query():
            st, idx = self._status_host
            for b in range(len(idx)):
                if int(st[b, 0]) != 0:
                    raise RuntimeError(f"[rank {self.rank}/{self.world}] DDP bucket {idx[b]} (step {self.step_count}): "
                                       f"deepreduce engine error: {STATUS_NAMES.get(int(st[b, 0]), int(st[b, 0]))} "
                                       f"(aux={int(st[b, 1])})")
        if not self._layouts:
            return
        st = torch.zeros(len(self._layouts), 8, dtype=torch.int32).pin_memory()
        for b, lay in enumerate(self._layouts):
            st[b].copy_(lay.engine.status, non_blocking=True)
        self._status_host = (st, [lay.index for lay in self._layouts])
        self._status_event = torch.cuda.Event()
        self._status_event.record()

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
        torch.cuda.synchronize(self._layouts[0].engine.device)
        tot: dict = {}
        for e in self.engines:
            for k, v in e.stats()["total"].items():
                tot[k] = tot.get(k, 0) + v
        tot["relative_volume"] = tot["wire_bytes"] / max(1, tot["dense_bytes"])
        return tot

    # ---- checkpoint / resume ----------------------------------------------------------
    def state_dict(self) -> dict:
        """Keyed by parameter name, so that a checkpoint loads into a run with other buckets: the residual of every
        parameter (fused path, flat in storage order; with 'dgc' its momentum too, under ``"momentum"``) or the GRACE
        memory (per-tensor path)."""
        if self._layouts:
            torch.cuda.synchronize(self._layouts[0].engine.device)
        resid = {n: t.clone() for n, t in self._pending.items()}
        mom = {n: t.clone() for n, t in self._pending_mom.items()}
        for lay in self._layouts:
            for p, n in zip(lay.params, lay.names):
                if self._owner.get(id(p)) is lay:
                    resid[n] = lay.resid_of(p).detach().cpu().clone()
                    if self.dgc:
                        mom[n] = lay.mom_of(p).detach().cpu().clone()
        out = {"step": self.step_count, "residuals": resid,
               "epoch": max([self._pending_epoch] + [e.epoch for e in self.engines])}
        if self.dgc:
            out["momentum"] = mom
        if self.grc is not None:
            out["memory"] = self.grc.memory.state_dict()
            if self.warmup is not None:               # the per-name exchange counts of the warm-up
                out["sparsifier"] = sparsifier_of(self.grc).state_dict()
        return out

    def load_state_dict(self, state: dict):
        self.step_count = int(state.get("step", 0))
        # engine epochs only move forward (BucketEngine.load_state_dict): peer flags carry epochs already used
        self._pending_epoch = max(self._pending_epoch, int(state.get("epoch", 0)))
        for e in self.engines:
            e.epoch = max(e.epoch, self._pending_epoch)
        by_name = {}
        for lay in self._layouts:
            for p, n in zip(lay.params, lay.names):
                if self._owner.get(id(p)) is lay:
                    by_name[n] = lay
        if self.dgc != ("momentum" in state) and state.get("residuals"):
            raise ValueError("hook state of another memory: 'dgc' states carry a 'momentum' map, other states do not")
        self._pending, self._pending_mom = {}, {}
        for key, pending, view in (("residuals", self._pending, _Layout.resid_of),
                                   ("momentum", self._pending_mom, _Layout.mom_of)):
            for n, t in state.get(key, {}).items():
                lay = by_name.get(n)
                if lay is None:
                    pending[n] = t.detach().cpu().clone()
                else:
                    p = next(q for q, m in zip(lay.params, lay.names) if m == n)
                    view(lay, p).copy_(t.to(lay.engine.device, torch.float32).reshape(-1))
        if "memory" in state:
            if self.grc is None:
                self._make_grc()
            dev = next(self.module.parameters()).device
            self.grc.memory.load_state_dict(state["memory"], device=dev)
            if self.warmup is not None:               # a checkpoint from before the warm-up: every count at 0
                sparsifier_of(self.grc).load_state_dict(state.get("sparsifier", {}))

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
