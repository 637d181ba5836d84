"""Bucketed, overlapped data-parallel wrapper — the new entry point next to the
per-tensor ``grc.step(grad, name)`` (SURVEY §7.1).

The reference runs strictly after backward, one Python call and 2-3 NCCL
all_gathers per tensor (SURVEY §3.2, C1).  Here parameters are laid out in flat
fp32 or bf16 buckets, one dtype per bucket (``p.grad`` are views), autograd post-accumulate hooks mark
buckets ready during backward, and each ready bucket is handed to a C++
background thread that launches the fused exchange kernel on a high-priority
side stream; ``finish()`` makes the optimizer's stream wait on the done events.

CUDA + ('topk' [+ 'index': 'bloom' | plain])  -> fused engine (one kernel/bucket)
CUDA + 'both' + 'rle' + 'fused_rle_values'    -> fused engine, value codec over the run-length index
CUDA + 'index'/'both' + 'elias_fano'          -> fused engine, Elias-Fano index (fp32 or any fused value codec)
CUDA + 'dexp' values + 'fused_dexp'           -> fused engine, double-exponential values (plain, bloom or rle index)
CUDA + 'bf16' values                          -> fused engine, 16-bit values (plain, bloom or rle index, or 'randomk')
CUDA + 'sign' values                          -> fused engine, 1-bit scaled-sign values (wherever bf16 values are)
CUDA + 'fp8' values                           -> fused engine, E4M3 values with a scale per 32 (wherever sign values are)
CUDA + 'randomk' [+ QSGD, bf16, sign or fp8 values] -> fused engine, values only on the wire (shared-seed index)
CUDA + 'none'/'allreduce'                     -> dense NCCL all-reduce of the flat bucket
anything else (CPU/gloo, other codecs)        -> GRACE-compatible per-tensor path
"""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.distributed as dist
import torch.nn as nn

from .. import spec
from ..grace.helper import sparsifier_of
from ..grace.memory import check_exclude_patterns, decay_excluded, is_dense
from ..wrappers import deepreduce_from_params
from .engine import BucketEngine, StatusPoller, total_stats
from .plan import BucketPlan


def _fused_supported(params: dict) -> bool:
    """Which top-k / threshold ``params`` dicts the fused bucket engine serves with a per-rank index (everything else
    takes the GRACE-compatible per-tensor path, unless ``_fused_randomk_supported`` takes it).  Covers every recipe of
    the reference's launch script (run_deepreduce.sh:35-107): top-k or threshold sparsifier x {no codec, index (bloom
    leftmost / random / p0, run-length), value (polyfit, QSGD int8/int16), both}, and bf16 values (``'value': 'bf16'``)
    over the plain, bloom or run-length index, with no opt-in key: no earlier dict names 'bf16'.  Scaled-sign values
    (``'value': 'sign'``, 512-value buckets) and fp8 values (``'value': 'fp8'``, 32-value blocks) take every route bf16
    values take, with no opt-in key either.
    Bloom policy 'conflict_sets' (P2) is fused only with top-k and ``'p2_pick_mask': True``: the sender then ships its pick as a
    bitmask over the positives, a different wire from the reference's, where every receiver redraws the pick.
    'both' with the run-length index is fused only with ``'fused_rle_values': True``: without the key that dict keeps
    the per-tensor route it always had (and its checkpoint format).
    Double-exponential values ('dexp') are fused only with ``'fused_dexp': True``, for the same reason: 'value', or
    'both' over the bloom or run-length index.
    The Elias-Fano index ('elias_fano') is fused wherever the run-length index is, with every value codec and no
    opt-in key: no earlier dict names it.
    Not fused: 'conflict_sets' without that key (per-tensor GPU kernel), host codecs (Huffman, Deflate, the integer
    family), dexp without 'fused_dexp', non-512 QSGD buckets."""
    if params.get('compressor') not in ('topk', 'threshold') or params.get('communicator', 'allgather') != 'allgather':
        return False
    dr = params.get('deepreduce', None)
    if dr is None:
        return True
    from ..codecs.bloom import canonical_policy
    policy = canonical_policy(params.get('policy', 'leftmost'))
    # P2 needs top-k: under 'threshold' K is the slot capacity, so the draw would keep every positive
    p2_ok = policy == 'conflict_sets' and params.get('p2_pick_mask') is True and params.get('compressor') == 'topk'
    pol_ok = policy in ('leftmost', 'random', 'p0') or p2_ok
    value_ok = (params.get('value', 'polyfit') in ('polyfit', 'bf16', 'sign', 'fp8')
                or (params.get('value') == 'qsgd' and 1 <= int(params.get('quantum_num', 127)) <= 32767
                    and int(params.get('bucket_size', 512)) == 512))
    # the same index rule whether the index is shipped ('both') or not ('value'), as the config check has it
    index = params.get('index', 'bloom')
    dexp_ok = (params.get('value') in ('dexp', 'double_exp') and params.get('fused_dexp') is True
               and ((index == 'bloom' and pol_ok) or (index == 'rle' and policy != 'conflict_sets')))
    if dr == 'index' and params.get('index', 'bloom') == 'bloom':
        return pol_ok
    if dr == 'index' and params.get('index') == 'rle':
        return True                      # lossless tile-local run coding inside the fused kernel
    if dr == 'index' and params.get('index') == 'elias_fano':
        return policy != 'conflict_sets'  # lossless tile-local Elias-Fano; the fused plan refuses P2 outside bloom
    if dr == 'value':
        return value_ok or dexp_ok       # coded values + plain indices
    if dr == 'both' and params.get('index', 'bloom') == 'bloom':
        return pol_ok and (value_ok or dexp_ok)
    if dr == 'both' and params.get('index') == 'rle':
        # the bloom policies do not apply to a lossless index; the fused plan refuses 'conflict_sets' outside bloom
        # bf16, sign and fp8 values need no key, and 'fused_rle_values' keeps its meaning: it refuses them
        rv, keyless = params.get('fused_rle_values') is True, params.get('value') in ('bf16', 'sign', 'fp8')
        return ((rv and value_ok and not keyless) or dexp_ok or (keyless and not rv)) and policy != 'conflict_sets'
    if dr == 'both' and params.get('index') == 'elias_fano':
        # every value codec the run-length index fuses, with no opt-in key: no earlier dict names this index
        return (value_ok or params.get('value') in ('dexp', 'double_exp')) and policy != 'conflict_sets'
    return False


def _fused_randomk_supported(params: dict) -> bool:
    """Which 'randomk' ``params`` dicts the fused engine serves in its shared-index mode (``kModeShared``): every rank
    draws the same index set from (step, tensor), so only values travel and the allgather and allreduce communicators
    give the same aggregate.  With no codec, with QSGD values (``'deepreduce': 'value', 'value': 'qsgd'``, bucket
    512), with bf16 values (``'value': 'bf16'``), with scaled-sign values (``'value': 'sign'``) or with fp8 values
    (``'value': 'fp8'``).  Not fused:
    'randomk' with an index codec, 'both', or polyfit values."""
    if params.get('compressor') != 'randomk' or params.get('communicator', 'allgather') not in ('allgather', 'allreduce'):
        return False
    dr = params.get('deepreduce', None)
    v = params.get('value', 'polyfit')
    return dr is None or (dr == 'value' and (v in ('bf16', 'sign', 'fp8')
                                             or (v == 'qsgd' and 1 <= int(params.get('quantum_num', 127)) <= 32767
                                                 and int(params.get('bucket_size', 512)) == 512)))


BUCKET_DTYPES = (torch.float32, torch.bfloat16)


def group_buckets(named, cap_mb: float) -> list:
    """Cut the ``(name, parameter)`` list into flat buckets, in reverse order (roughly the order gradients become
    ready).  A bucket holds one dtype: fp32 parameters and bf16 parameters each fill their own buckets, in the order the
    dtype first appears, cut at ``cap_mb`` MiB of that dtype.  An all-fp32 list gives the buckets it always gave.
    Other dtypes raise ``ValueError``."""
    order = list(reversed(named))
    dtypes = []
    for n, p in order:
        if p.dtype not in BUCKET_DTYPES:
            raise ValueError(f"parameter {n!r} is {p.dtype}: flat buckets hold fp32 or bf16 gradients")
        if p.dtype not in dtypes:
            dtypes.append(p.dtype)
    buckets = []
    for dt in dtypes:
        cap = int(cap_mb * 1024 * 1024 / (4 if dt == torch.float32 else 2))
        cur, cur_n = [], 0
        for n, p in order:
            if p.dtype != dt:
                continue
            if cur and cur_n + p.numel() > cap:
                buckets.append(cur)
                cur, cur_n = [], 0
            cur.append((n, p))
            cur_n += p.numel()
        if cur:
            buckets.append(cur)
    return buckets


def fused_path(params: dict) -> bool:
    """True if ``DeepReduceDDP`` on CUDA runs ``params`` through the fused bucket engine."""
    return _fused_supported(params) or _fused_randomk_supported(params)


def plan_kwargs_from_params(params: dict) -> dict:
    """``params`` dict (the reference's ``--grace_config``) -> BucketPlan keyword arguments."""
    from ..codecs.bloom import canonical_policy
    dr = params.get('deepreduce')
    v = params.get('value', 'polyfit')
    kw = dict(compress_ratio=params.get('compress_ratio', 0.01),
              index=(params.get('index', 'bloom') if dr in ('index', 'both') else None),
              value=({'double_exp': 'dexp'}.get(v, v) if dr in ('value', 'both') else None),
              quantum_num=int(params.get('quantum_num', 127)),
              poly_degree=int(params.get('poly_degree', 5)),
              fpr=params.get('fpr', None),
              policy=canonical_policy(params.get('policy', 'leftmost')),
              min_numel=int(params.get('min_numel', spec.SMALL_TENSOR_NUMEL)),
              hint=bool(params.get('hint', True)))
    if kw['value'] == 'dexp':
        from ..codecs.dexp import MIN_NUMEL
        kw['dexp_min_numel'] = int(params.get('dexp_min_numel', MIN_NUMEL))
    if params.get('compressor') == 'threshold':
        kw.update(sparsifier='threshold', threshold=float(params.get('threshold', 0.0)),
                  capacity_ratio=params.get('threshold_capacity', None))
    elif params.get('compressor') == 'randomk':
        kw.update(sparsifier='randomk')
    return kw


def engine_split_numel(params: dict, blocks_per_sm: int) -> int:
    """Chunk size of the fused plan for ``params``: tensors whose bloom filter would not fit the kernel's SMEM staging
    buffer enter the plan as tile-aligned chunks with their own top-k / filter ('split_numel': 'auto', the default; an
    int pins the chunk size, 0 / None keeps every tensor whole and lets oversize filters be probed from L2)."""
    sn = params.get('split_numel', 'auto')
    if sn == 'auto':
        uses_bloom = params.get('deepreduce') in ('index', 'both') and params.get('index', 'bloom') == 'bloom'
        from .plan import auto_split_numel
        sn = auto_split_numel(params.get('compress_ratio', 0.01), params.get('fpr', None),
                              (160 if blocks_per_sm < 2 else 80) * 1024) if uses_bloom and params.get('compressor') == 'topk' else 0
    return int(sn or 0)


def engine_kwargs(params: dict, names=None) -> dict:
    """The ``BucketEngine`` memory arguments for ``params``: beta, gamma, momentum, Nesterov, weight decay, clipping and
    averaging.  They follow the per-tensor memory GRACE builds for the same dict: only ``ResidualMemory`` scales the
    gradient by gamma, so 'none' and 'dgc' memory run with gamma = 1 ('dgc' accepts no other), and without a residual
    beta is 0.  With ``'weight_decay_exclude'``, ``names`` are the bucket's parameter names, one per parameter: those
    that match a pattern get a decay factor of 0 (``weight_decays``)."""
    memory = params.get('memory', 'none')
    kw = dict(beta=float(params.get('beta', 1.0)) if memory in ('residual', 'dgc') else 0.0,
              gamma=float(params.get('gamma', 1.0)) if memory == 'residual' else 1.0,
              average=params.get('average', True),
              momentum=float(params.get('momentum', 0.9)) if memory == 'dgc' else None,
              weight_decay=float(params.get('weight_decay', 0.0)) if memory == 'dgc' else 0.0,
              clip_norm=float(params['clip_norm']) if memory == 'dgc' and 'clip_norm' in params else None,
              nesterov=memory == 'dgc' and params.get('nesterov', False) is True)
    if memory == 'dgc' and params.get('weight_decay_exclude'):
        if names is None:
            raise ValueError("'weight_decay_exclude' matches parameter names: engine_kwargs needs the bucket's names")
        wd = kw.pop('weight_decay')
        kw['weight_decays'] = [0.0 if decay_excluded(n, params['weight_decay_exclude']) else wd for n in names]
    return kw


def stage_plans(numels, names, shapes, params: dict, warmup) -> List[BucketPlan]:
    """The ``BucketPlan`` of every sparsity warm-up stage (``spec.Warmup``) of one bucket, over the same list of plan
    tensors, the last one at ``'compress_ratio'``; without a warm-up, the one plan of ``params``.  The chunking
    (``engine_split_numel``) follows the final ratio, so the tile offsets and ``total_elems`` are those of the final
    plan in every stage and only K, the filter sizes and the slot layout change.  Built up front: a stage a plan
    refuses (e.g. P2's positive limit at a dense ratio) raises before the first exchange."""
    kw = plan_kwargs_from_params(params)
    if warmup is None:
        return [BucketPlan(numels, names, shapes, **kw)]
    return [BucketPlan(numels, names, shapes, **{**kw, 'compress_ratio': warmup.ratio(s)})
            for s in range(warmup.n_stages)]


def switch_engine(old: BucketEngine, build) -> BucketEngine:
    """A sparsity warm-up stage switch of one bucket: ``build(grad)`` makes the new stage's engine adopting ``grad``, the
    old engine's gradient buffer (``make_engine(..., grad=grad)``; collective at W > 1, like everything here), so
    ``p.grad`` keeps viewing it.  The buffer's aggregate is saved across the build, whose partition calibration writes
    it; the stages share one layout, so the residual and the 'dgc' momentum carry over as whole buffers, bit for bit;
    the select history does not (the selection is exact without it); the epoch only moves forward; the old engine is
    closed.  Returns the new engine."""
    agg = old.grad.clone()
    new = build(old.grad)
    new.grad.copy_(agg)
    buffers = new.memory_buffers()
    for k, t in old.memory_buffers().items():
        buffers[k].copy_(t)
    new.epoch = max(new.epoch, old.epoch)
    old.close()
    return new


def make_engine(plan: BucketPlan, params: dict, *, device, group, use_history: bool, blocks_per_sm: int,
                grad_dtype: torch.dtype, parameters=None, owner=None, grad=None, names=None) -> BucketEngine:
    """The ``BucketEngine`` of one bucket for ``params`` (memory arguments from ``engine_kwargs``), with its tile
    partitions calibrated unless ``'calibrate_partition': False``.  ``parameters`` / ``owner``: the bucket's parameters
    and the plan tensors' owners (``split_large``), bound when the engine applies weight decay; ``owner`` also makes
    the chunks of a split parameter one tensor for ``'clip_norm'``.  ``grad``: the flat gradient buffer to adopt
    (``BucketEngine``); the calibration overwrites it.  ``names``: the parameters' names, which
    ``'weight_decay_exclude'`` matches (``engine_kwargs``).  Collective at W > 1."""
    eng = BucketEngine(plan, device=device, group=group, use_history=use_history, blocks_per_sm=blocks_per_sm,
                       grad_dtype=grad_dtype, owner=owner, grad=grad, **engine_kwargs(params, names))
    if eng.reads_parameters:
        if parameters is None:
            raise ValueError("'weight_decay' reads the parameters: make_engine needs the bucket's parameters")
        eng.bind_parameters(parameters, owner)
    # re-cut the kernel's tile partitions from measured per-CTA phase times (collective; ~12 exchange steps
    # on synthetic gradients, state reset afterwards) — 'calibrate_partition': False keeps the static cut
    if params.get('calibrate_partition', True) and eng.cuts is not None:
        try:
            eng.calibrate_partition()
        except (ValueError, ArithmeticError, IndexError) as e:      # host-side arithmetic only: the static
            import warnings                                      # per-phase cut is a complete fallback
            warnings.warn(f"deepreduce_b200: partition calibration skipped ({e!r}); using the static cut")
            eng.cta_speeds = None
            eng._set_cuts()
            eng.reset_state()
    return eng


def make_grc(params: dict, named_parameters, storage_order: bool = False):
    """The GRACE communicator of the per-tensor path for ``params``; a memory that reads the parameters ('dgc' weight
    decay) is bound to the ``(name, parameter)`` pairs (``storage_order``: see ``DgcMemory.bind_parameters``)."""
    grc = deepreduce_from_params(params)
    if hasattr(grc.memory, "bind_parameters"):
        grc.memory.bind_parameters(named_parameters, storage_order=storage_order)
    return grc


def grace_state_dict(grc, warmup) -> dict:
    """The per-tensor path's checkpoint: the GRACE ``memory``, plus the warm-up's per-name ``sparsifier`` counts."""
    out = {"memory": grc.memory.state_dict()}
    if warmup is not None:
        out["sparsifier"] = sparsifier_of(grc).state_dict()
    return out


def load_grace_state_dict(grc, state: dict, warmup, device):
    """Restore what ``grace_state_dict`` saved.  A checkpoint from before the warm-up restores every count to 0."""
    if "memory" in state:
        grc.memory.load_state_dict(state["memory"], device=device)
    if warmup is not None:
        sparsifier_of(grc).load_state_dict(state.get("sparsifier", {}))


class DeepReduceDDP:
    def __init__(self, module: nn.Module, params: dict, *, bucket_cap_mb: float = 1e9, overlap: bool = True,
                 group=None, blocks_per_sm: int = 2, use_history: bool = True, background_thread: bool = True,
                 broadcast_parameters: bool = True, overlap_grid: int | None = None):
        self.module = module
        self.params = dict(params)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if self.params.get('memory') == 'dgc':     # a pattern that matches nothing is a typo: refuse it
            check_exclude_patterns(self.params.get('weight_decay_exclude'), [n for n, _ in self.named])
        self.device = self.named[0][1].device
        self.is_cuda = self.device.type == "cuda"
        self.dense = self.params.get('compressor', 'none') in ('none', None)
        self.fused = self.is_cuda and not self.dense and fused_path(self.params)
        self.overlap = overlap and self.is_cuda
        self.step_count = 0
        self.engines: List[BucketEngine] = []
        self.flat: List[torch.Tensor] = []
        self.bucket_of: Dict[int, int] = {}
        self.pending: List[int] = []
        self.sched = None
        self.grc = None
        self._handles = []
        self._exchange = True
        self._grad_views: Dict[int, torch.Tensor] = {}
        self._status = StatusPoller()
        self.overlap_grid_cap = int(overlap_grid if overlap_grid is not None else (self.params.get('overlap_grid', 0) or 0))
        from ..config import warmup_from_params
        self.warmup = warmup_from_params(self.params)        # sparsity warm-up: stages counted in exchanges (finish())
        self.stage = 0
        if self.world > 1 and broadcast_parameters:
            # replicas must start from the same weights: rank 0's parameters and buffers win (torch DDP does the same)
            with torch.no_grad():
                for t in list(module.parameters()) + list(module.buffers()):
                    dist.broadcast(t.data, 0, group=group)
        if self.fused or (self.dense and self.is_cuda):
            self._build_buckets(bucket_cap_mb, blocks_per_sm, use_history)
            if (self.fused and self.overlap and background_thread
                    and all(e.transport == "p2p" for e in self.engines)):     # the NCCL transport is issued from Python
                from .. import ops
                self.sched = ops.cuda_module().Scheduler(len(self.buckets))
            if self.overlap:
                self._install_hooks()
        else:
            self.grc = make_grc(self.params, self.named)

    # ---- bucket construction ------------------------------------------------
    def _build_buckets(self, cap_mb, blocks_per_sm, use_history):
        self.buckets: List[List] = group_buckets(self.named, cap_mb)
        self._plans: List[List[BucketPlan]] = []           # fused: [bucket][warm-up stage]
        self._engine_args: List[dict] = []
        for b, items in enumerate(self.buckets):
            dtype = items[0][1].dtype
            numels = [p.numel() for _, p in items]
            names = [n for n, _ in items]
            shapes = [tuple(p.shape) for _, p in items]
            owner = list(range(len(items)))
            if self.fused:
                sn = engine_split_numel(self.params, blocks_per_sm)
                if sn:
                    from .plan import split_large
                    numels, names, shapes, owner = split_large(numels, names, shapes, int(sn))
            if self.fused:
                self._plans.append(stage_plans(numels, names, shapes, self.params, self.warmup))
                self._engine_args.append(dict(device=self.device, group=self.group, use_history=use_history,
                                              blocks_per_sm=blocks_per_sm, grad_dtype=dtype,
                                              parameters=[p for _, p in items], owner=owner,
                                              names=[n for n, _ in items]))
                plan = self._plans[b][self.stage]
                eng = make_engine(plan, self.params, **self._engine_args[b])
                self.engines.append(eng)
                flat, views = eng.grad, eng.grad_views
            else:
                plan = BucketPlan(numels, names, shapes, index=None)
                flat = torch.zeros(plan.total_elems, dtype=dtype, device=self.device)
                views = plan.views(flat)
            self.flat.append(flat)
            first = {}
            for j, o in enumerate(owner):
                first.setdefault(o, plan.tensors[j])                # the first chunk of every parameter
            for i, (n, p) in enumerate(items):
                t = first[i]
                seg = flat[t.elem_off:t.elem_off + p.numel()]        # chunks are tile multiples: contiguous
                # the gradient view mirrors the parameter's own (dense) layout — e.g. channels_last conv
                # weights — so fused optimizers see identical strides; the bucket is in storage order
                p.grad = seg.as_strided(p.size(), p.stride()) if is_dense(p) else seg.view(p.shape)
                self._grad_views[id(p)] = p.grad
                self.bucket_of[id(p)] = b
        self._in_backward = False
        self._ready_count = [0] * len(self.buckets)
        self._launched = [False] * len(self.buckets)
        self._bucket_size = [len(it) for it in self.buckets]

    def _install_hooks(self):
        for n, p in self.named:
            self._handles.append(p.register_post_accumulate_grad_hook(self._hook))

    def set_exchange_enabled(self, on: bool):
        """Gradient accumulation: hooks only launch the exchange on the last micro-step."""
        self._exchange = bool(on)

    def _hook(self, p):
        if not self._exchange:
            return
        b = self.bucket_of[id(p)]
        self._ready_count[b] += 1
        if self._ready_count[b] == self._bucket_size[b]:
            self._in_backward = True
            try:
                self._launch_bucket(b)
            finally:
                self._in_backward = False

    def _launch_bucket(self, b):
        self._ready_count[b] = 0
        self._launched[b] = True
        if self.fused:
            eng = self.engines[b]
            eng.refresh_parameters()          # weight decay: follow a parameter whose storage moved (p.data = ...)
            # the engine's own step counter, never reset: peer flags carry the epoch, so an epoch that was already used
            # (e.g. by calibrate_partition's synthetic steps, or by a self-check step between training steps) would
            # let the flag waits pass before the peers have written their slots
            eng.epoch = eng.epoch + 1
            # buckets that become ready while backward is still running are launched with a capped grid so that the
            # persistent exchange kernel does not take every SM from cuDNN / cuBLAS; the bucket launched from
            # finish() (nothing left to overlap with) gets the whole GPU
            more_to_come = not all(self._launched)
            if self.sched is not None and more_to_come:
                # backward is still running: hand the bucket to the C++ launch thread (high-priority side stream), with a
                # capped grid so that the persistent kernel does not take every SM from cuDNN / cuBLAS
                eng.ctx.set_grid_cap(self.overlap_grid_cap if self.overlap_grid_cap > 0 else 0)
                self.sched.submit(b, eng.ctx, eng.epoch)
            else:
                # the LAST bucket (or the only one): nothing is left to overlap with, so every microsecond until the
                # kernel starts is exposed — launch inline on the current stream with the whole GPU instead of paying
                # the thread hand-off + event round trip
                eng.ctx.set_grid_cap(0)
                if self.sched is not None and len(self.buckets) > 1 and self.world > 1:
                    # cross-rank ordering: every rank must run its bucket kernels in the same order — a full-grid
                    # kernel that spins on peer flags would otherwise keep this rank's earlier (side-stream) buckets
                    # from starting while the peers wait for exactly those (deadlock until the peer watchdog fires).
                    # Make this stream wait for everything handed to the launch thread first.
                    self.sched.wait_all()
                eng.step(eng.epoch)
        else:
            if self.world > 1:
                self.pending.append(dist.all_reduce(self.flat[b], group=self.group, async_op=True))

    # ---- per-step API ---------------------------------------------------------
    def zero_grad(self):
        if self.flat:
            for f in self.flat:
                f.zero_()
        else:
            for _, p in self.named:
                p.grad = None

    def finish(self):
        """Call after backward, before optimizer.step(): gradients become the
        cross-rank aggregate."""
        if self.grc is not None:
            for n, p in self.named:
                if p.grad is not None:
                    p.grad = self.grc.step(p.grad, n).view_as(p)
        elif self.fused:
            self._check_grad_views()
            for b in range(len(self.buckets)):        # not overlapped, or a parameter received no gradient this step
                if not self._launched[b]:
                    self._launch_bucket(b)
            if self.sched is not None:
                self.sched.wait_all()
            self._launched = [False] * len(self.buckets)
        else:
            self._check_grad_views()
            for b in range(len(self.buckets)):
                if not self._launched[b]:
                    self._launch_bucket(b)
            self._launched = [False] * len(self.buckets)
            for w in self.pending:
                w.wait()
            self.pending = []
            if self.world > 1 and self.params.get('average', True):
                for f in self.flat:
                    f.div_(self.world)
        self.step_count += 1
        if self.fused and self.warmup is not None and self.warmup.stage(self.step_count) != self.stage:
            self._switch_stage(self.warmup.stage(self.step_count))

    def _switch_stage(self, stage: int):
        """Move every bucket to the engine of warm-up ``stage`` between two exchanges (``switch_engine``; collective at
        W > 1: every rank counts the same exchanges, so all switch after the same ``finish()``).  ``p.grad`` still
        holds this exchange's aggregate for the optimizer step."""
        for b, old in enumerate(self.engines):
            plan, args = self._plans[b][stage], self._engine_args[b]
            self.engines[b] = switch_engine(old, lambda grad: make_engine(plan, self.params, grad=grad, **args))
        self.stage = stage

    def _check_grad_views(self):
        """``p.grad`` must still be the view into the flat bucket: ``optimizer.zero_grad(set_to_none=True)`` (torch's
        default) or ``p.grad = None`` detaches it, autograd then allocates a fresh gradient and the exchange would
        silently run on stale bucket contents.  Re-attach: copy what autograd produced into the bucket and point
        ``p.grad`` back at the view."""
        for _, p in self.named:
            v = self._grad_views.get(id(p))
            if v is None or p.grad is v:
                continue
            if p.grad is None:
                v.zero_()                              # no gradient this step: the bucket slice must not keep old data
            elif p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
            p.grad = v

    def check_async(self):
        """Per-step failure detection without a host sync (``StatusPoller``): raises like :meth:`check` one step after
        a watchdog fired."""
        bad = self._status.poll(list(enumerate(self.engines)))
        if bad is not None:
            raise RuntimeError(f"[rank {self.rank}/{self.world}] bucket {bad[0]} (step {self.step_count}): {bad[1]}")

    def check(self):
        """Read the engines' device status words (one small D2H each); raises with rank and bucket on a watchdog."""
        for b, e in enumerate(self.engines):
            try:
                e.check_status()
            except RuntimeError as err:
                raise RuntimeError(f"[rank {self.rank}/{self.world}] bucket {b} "
                                   f"({len(self.buckets[b])} tensors, step {self.step_count}): {err}") from err

    # ---- accounting -------------------------------------------------------------
    def wire_bytes_per_step(self) -> int:
        if self.fused:
            return sum(e.plan.wire_bytes() for e in self.engines)
        if self.dense:
            return sum(f.numel() * f.element_size() for f in self.flat)
        return int(self.grc.bytes_sent / max(self.step_count, 1))

    def stage2_bytes_per_step(self) -> int:
        """Sharded decode (W > 1): bytes of the second in-kernel exchange this rank sent last step — its decoded slice
        as (index, value) pairs to each of the W-1 peers — read from the live entry count in the stage-2 header.
        Together with ``wire_bytes_per_step`` this is everything a rank puts on NVLink per step."""
        if not self.fused or self.world == 1:
            return 0
        torch.cuda.synchronize(self.device)
        return sum(e.stage2_bytes() for e in self.engines)

    def dense_bytes(self) -> int:
        return sum(p.numel() * p.element_size() for _, p in self.named)

    def exchange_stats(self) -> dict:
        """Device-side counters of the last exchanged step, summed over the buckets (fused path): shipped
        coordinates, bloom positives / false positives, value / index / header bytes (``BucketEngine.stats``).
        Call it after ``finish()`` (i.e. after a training step); it synchronises the device, so every N steps."""
        if not self.fused:
            return {"wire_bytes": self.wire_bytes_per_step(), "dense_bytes": self.dense_bytes()}
        return total_stats(self.engines)

    # ---- checkpoint / resume (SURVEY §5) -------------------------------------------
    def state_dict(self):
        if self.fused:
            return {"step": self.step_count, "engines": [e.state_dict() for e in self.engines]}
        if self.grc is not None:
            return {"step": self.step_count, **grace_state_dict(self.grc, self.warmup)}
        return {"step": self.step_count}

    def load_state_dict(self, state):
        self.step_count = int(state.get("step", 0))
        if self.fused:
            if self.warmup is not None and self.warmup.stage(self.step_count) != self.stage:
                self._switch_stage(self.warmup.stage(self.step_count))
            for e, s in zip(self.engines, state["engines"]):
                e.load_state_dict(s)
        elif self.grc is not None:
            load_grace_state_dict(self.grc, state, self.warmup, self.device)

    def close(self):
        for h in self._handles:
            h.remove()
        if self.sched is not None:
            self.sched.shutdown()
            self.sched = None
        for e in self.engines:
            e.close()
