"""Validated, frozen view of the GRACE / DeepReduce ``params`` dict.

The reference threads one mutable dict through every layer and also uses it as a
side channel (``params['dense_tensor']`` pytorch/deepreduce.py:117,
``params['hash_table']`` :33,44; the TF half adds derived keys ``m, k, N, K,
X_train, num_of_segments`` tensorflow/deepreduce.py:312,385,392,412,454,481).
Here the dict stays the front door (API compatibility: reference README.md:30-48,
run_deepreduce.sh ``--grace_config``), but it is parsed once into
:class:`DeepReduceConfig` — typed, range-checked, immutable — and nothing is ever
written back into the user's dict.  Unknown keys are reported (typos such as
``'compres_ratio'`` silently fall back to defaults in the reference).
"""
from __future__ import annotations

import math
import warnings
from dataclasses import asdict, dataclass
from typing import Optional, Tuple

from . import spec

COMPRESSORS = ("none", "topk", "threshold", "randomk")
OUT_OF_SCOPE_COMPRESSORS = ("SKCompressCPU", "SKCompressGPU", "sketch")        # comparison baselines of a GRACE fork
MEMORIES = ("none", "residual", "dgc")
COMMUNICATORS = ("allgather", "allreduce")
MODES = (None, "value", "index", "both")
POLICIES = ("leftmost", "leftmostK", "random", "randomK", "p0", "policy_zero", "conflict_sets", "p2")

# keys the PyTorch side reads (reference pytorch/deepreduce.py:36,57,106,384-385,512-513,857-858) + the ones this
# framework adds; the TF-side keys are handled by tf_compat and only listed so they do not trigger the typo warning
KNOWN_KEYS = frozenset({
    "compressor", "memory", "communicator", "compress_ratio", "threshold", "deepreduce", "value", "index", "fpr",
    "policy", "sort", "poly_degree", "quantum_num", "bucket_size", "micro-benchmark", "world_size", "average",
    "beta", "gamma", "seed", "code", "hint", "min_numel", "dense_tensor", "hash_table", "split_numel", "pack_mapping",
    "qsgd_seed", "gzip_level", "dexp_min_numel", "overlap_grid", "capacity_ratio", "calibrate_partition",
    "p2_pick_mask", "fused_rle_values", "fused_dexp", "momentum", "gradient_clipping", "weight_decay",
    "clip_norm", "warmup_ratios", "warmup_steps", "nesterov", "weight_decay_exclude",
    # TF-side (tensorflow/deepreduce.py:34-36,57-59,282,307-343,361-369,458-490)
    "use_memory", "horovod_size", "bloom_fpr", "bloom_on", "threshold_val", "bloom_false_positives_aware",
    "bloom_policy", "bloom_logs_path", "gradient_id", "bloom_verbosity_frequency", "bloom_verbosity", "mem_mode",
    "suffix", "model_name", "approximation_mode", "polynomial_degree", "tensor_name", "step", "rank",
})


class ConfigError(ValueError):
    pass


@dataclass(frozen=True)
class DeepReduceConfig:
    compressor: str = "none"
    memory: str = "none"
    communicator: str = "allreduce"
    compress_ratio: float = 0.01
    threshold: float = 0.0
    deepreduce: Optional[str] = None
    value: str = "polyfit"
    index: str = "bloom"
    fpr: Optional[float] = None
    policy: str = "leftmost"
    poly_degree: int = 5
    quantum_num: int = 127
    bucket_size: int = 512
    micro_benchmark: bool = False
    average: bool = True
    beta: float = 1.0
    gamma: float = 1.0
    world_size: Optional[int] = None
    hint: bool = True
    min_numel: int = 1000
    warmup_ratios: Optional[Tuple[float, ...]] = None
    warmup_steps: Optional[int] = None

    # ------------------------------------------------------------------
    @classmethod
    def from_params(cls, params: dict, *, strict: bool = False) -> "DeepReduceConfig":
        """Parse + validate.  ``strict`` turns the unknown-key warning into an error."""
        if not isinstance(params, dict):
            raise ConfigError(f"params must be a dict (got {type(params).__name__})")
        unknown = sorted(k for k in params if k not in KNOWN_KEYS)
        if unknown:
            msg = f"unknown params key(s) {unknown}; known keys: {sorted(KNOWN_KEYS)}"
            if strict:
                raise ConfigError(msg)
            warnings.warn(msg, stacklevel=3)
        g = params.get
        comp = g("compressor", "none") or "none"
        if comp in OUT_OF_SCOPE_COMPRESSORS:
            raise NotImplementedError(
                f"compressor '{comp}' is a comparison baseline from a GRACE fork and is out of scope (SURVEY §2.5)")
        cfg = cls(
            compressor=comp, memory=g("memory", "none") or "none", communicator=g("communicator", "allreduce"),
            compress_ratio=float(g("compress_ratio", 0.01)), threshold=float(g("threshold", 0.0)),
            deepreduce=g("deepreduce", None) or None, value=g("value", "polyfit"), index=g("index", "bloom"),
            fpr=None if g("fpr", None) is None else float(g("fpr")), policy=g("policy", "leftmost"),
            poly_degree=int(g("poly_degree", 5)), quantum_num=int(g("quantum_num", 127)),
            bucket_size=int(g("bucket_size", 512)), micro_benchmark=bool(g("micro-benchmark", False)),
            average=bool(g("average", True)), beta=float(g("beta", 1.0)), gamma=float(g("gamma", 1.0)),
            world_size=None if g("world_size", None) is None else int(g("world_size")),
            hint=bool(g("hint", True)), min_numel=int(g("min_numel", 1000)))
        cfg.validate()
        wu = warmup_from_params(params)
        if wu is not None:
            object.__setattr__(cfg, "warmup_ratios", wu.ratios)
            object.__setattr__(cfg, "warmup_steps", wu.steps)
        # 'dgc' memory (momentum correction + momentum factor masking, Lin et al. 2018): the momentum factor rides in
        # 'momentum'; it replaces the optimizer's momentum, and the residual it keeps is the plain one (beta = gamma = 1)
        if "momentum" in params:
            m = params["momentum"]
            if cfg.memory != "dgc":
                raise ConfigError(f"'momentum' applies to 'memory': 'dgc' (got memory={cfg.memory!r})")
            if isinstance(m, bool) or not isinstance(m, (int, float)) or not 0.0 <= float(m) < 1.0:
                raise ConfigError(f"'momentum' must be a number in [0, 1) (got {m!r})")
        # ... and weight decay, added to the gradient ahead of that momentum as momentum SGD adds it: 'weight_decay' then
        # replaces the optimizer's weight decay too
        if "weight_decay" in params:
            wd = params["weight_decay"]
            if cfg.memory != "dgc":
                raise ConfigError(f"'weight_decay' applies to 'memory': 'dgc' (got memory={cfg.memory!r})")
            if (isinstance(wd, bool) or not isinstance(wd, (int, float)) or not math.isfinite(float(wd))
                    or float(wd) < 0.0):
                raise ConfigError(f"'weight_decay' must be a finite number >= 0 (got {wd!r})")
        # ... except on the parameters whose names match a pattern: the param group with weight_decay=0 that recipes
        # give BatchNorm weights and biases
        if "weight_decay_exclude" in params:
            pats = params["weight_decay_exclude"]
            if cfg.memory != "dgc":
                raise ConfigError(f"'weight_decay_exclude' applies to 'memory': 'dgc' (got memory={cfg.memory!r})")
            if not isinstance(pats, (list, tuple)) or not all(isinstance(p, str) for p in pats):
                raise ConfigError(f"'weight_decay_exclude' must be a list of fnmatch patterns (strings) over parameter "
                                  f"names (got {pats!r})")
            if not float(params.get("weight_decay", 0.0)) > 0.0:
                raise ConfigError("'weight_decay_exclude' excludes parameters from 'weight_decay': it needs "
                                  "'weight_decay' > 0")
        # ... and Nesterov momentum, as torch's SGD(nesterov=True) takes it
        if "nesterov" in params:
            nv = params["nesterov"]
            if cfg.memory != "dgc":
                raise ConfigError(f"'nesterov' applies to 'memory': 'dgc' (got memory={cfg.memory!r})")
            if not isinstance(nv, bool):
                raise ConfigError(f"'nesterov' must be True or False (got {nv!r})")
            if nv and float(params.get("momentum", 0.9)) == 0.0:
                raise ConfigError("'nesterov': True needs a momentum > 0 (got 'momentum': 0)")
        # ... and DGC's local gradient clipping: each tensor's gradient is scaled down to norm c / sqrt(W) before it
        # enters the momentum, inside the memory, because no user code runs between backward and the exchange
        if "clip_norm" in params:
            c = params["clip_norm"]
            if cfg.memory != "dgc":
                raise ConfigError(f"'clip_norm' applies to 'memory': 'dgc' (got memory={cfg.memory!r})")
            if (isinstance(c, bool) or not isinstance(c, (int, float)) or not math.isfinite(float(c))
                    or float(c) <= 0.0):
                raise ConfigError(f"'clip_norm' must be a finite number > 0 (got {c!r})")
        if cfg.memory == "dgc":
            if cfg.compressor == "none":
                raise ConfigError("'memory': 'dgc' needs a sparsifier: set 'compressor' to topk/threshold/randomk")
            if cfg.beta != 1.0 or cfg.gamma != 1.0:
                raise ConfigError(f"'memory': 'dgc' keeps the residual with beta = gamma = 1 (got beta={cfg.beta}, "
                                  f"gamma={cfg.gamma})")
        # GRACE's DGC clamps each gradient element-wise to a norm reduced across ranks; not supported
        if g("gradient_clipping", False) not in (False, None):
            raise ConfigError("'gradient_clipping' (GRACE's element-wise clamp to the norm reduced across ranks) is not "
                              "supported; for DGC's per-tensor norm clipping use 'memory': 'dgc' with 'clip_norm': c")
        # opt-in wire of the fused engine's conflict_sets policy: the sender ships its pick as a bitmask over the positives
        p2 = g("p2_pick_mask", False)
        if not isinstance(p2, bool):
            raise ConfigError(f"'p2_pick_mask' must be True or False (got {p2!r})")
        if p2 and not (cfg.compressor == "topk" and cfg.deepreduce in ("index", "both") and cfg.index == "bloom"
                       and cfg.policy in ("conflict_sets", "p2")):
            raise ConfigError("'p2_pick_mask' applies to the top-k sparsifier with the bloom index and policy "
                              f"'conflict_sets' (got compressor={cfg.compressor!r}, deepreduce={cfg.deepreduce!r}, "
                              f"index={cfg.index!r}, policy={cfg.policy!r})")
        # scaled-sign values code fixed 512-value buckets, in the fused engine and per tensor alike
        if cfg.deepreduce in ("value", "both") and cfg.value == "sign" and cfg.bucket_size != 512:
            raise ConfigError(f"'value': 'sign' codes buckets of 512 values; 'bucket_size' must be 512 or left out "
                              f"(got {cfg.bucket_size})")
        # fp8 values code fixed 32-value blocks (one warp each); 'bucket_size' may name that size or be left out
        if (cfg.deepreduce in ("value", "both") and cfg.value == "fp8" and "bucket_size" in params
                and params["bucket_size"] != 32):
            raise ConfigError(f"'value': 'fp8' codes blocks of 32 values; 'bucket_size' must be 32 or left out "
                              f"(got {params['bucket_size']!r})")
        # opt-in route of 'both' + run-length index through the fused engine (the value codec rides behind the index);
        # without it that combination keeps the per-tensor path and its checkpoints
        rv = g("fused_rle_values", False)
        if not isinstance(rv, bool):
            raise ConfigError(f"'fused_rle_values' must be True or False (got {rv!r})")
        if rv and not (cfg.compressor in ("topk", "threshold") and cfg.communicator == "allgather"
                       and cfg.deepreduce == "both" and cfg.index == "rle"
                       and (cfg.value == "polyfit" or (cfg.value == "qsgd" and cfg.bucket_size == 512))):
            raise ConfigError("'fused_rle_values' applies to the top-k or threshold sparsifier with 'deepreduce': 'both', "
                              "'index': 'rle' and 'value' 'polyfit' or 'qsgd' (bucket_size 512) over 'allgather' (got "
                              f"compressor={cfg.compressor!r}, communicator={cfg.communicator!r}, "
                              f"deepreduce={cfg.deepreduce!r}, index={cfg.index!r}, value={cfg.value!r}, "
                              f"bucket_size={cfg.bucket_size})")
        # opt-in route of double-exponential values through the fused engine (two curves per tensor, one per sign run,
        # over the fused rank map); without it 'dexp' keeps the per-tensor path, its wire and its checkpoints
        fd = g("fused_dexp", False)
        if not isinstance(fd, bool):
            raise ConfigError(f"'fused_dexp' must be True or False (got {fd!r})")
        if fd and not (cfg.compressor in ("topk", "threshold") and cfg.communicator == "allgather"
                       and cfg.deepreduce in ("value", "both") and cfg.value in ("dexp", "double_exp")
                       and ((cfg.index == "bloom" and (cfg.policy in ("leftmost", "leftmostK", "random", "randomK", "p0",
                                                                      "policy_zero") or p2))
                            or (cfg.index == "rle" and cfg.policy not in ("conflict_sets", "p2")))):
            raise ConfigError("'fused_dexp' applies to the top-k or threshold sparsifier with 'deepreduce': 'value' or "
                              "'both', 'value': 'dexp' and 'index' 'bloom' (policy leftmost, random, p0, or conflict_sets "
                              "with 'p2_pick_mask') or 'rle', over 'allgather' (got "
                              f"compressor={cfg.compressor!r}, communicator={cfg.communicator!r}, "
                              f"deepreduce={cfg.deepreduce!r}, value={cfg.value!r}, index={cfg.index!r}, "
                              f"policy={cfg.policy!r})")
        return cfg

    def validate(self) -> None:
        from .codecs import compressor as registry

        def need(cond, msg):
            if not cond:
                raise ConfigError(msg)

        need(self.compressor in COMPRESSORS, f"'compressor' must be one of {COMPRESSORS} (got {self.compressor!r})")
        need(self.memory in MEMORIES, f"'memory' must be one of {MEMORIES} (got {self.memory!r})")
        need(self.communicator in COMMUNICATORS,
             f"'communicator' must be one of {COMMUNICATORS} (got {self.communicator!r})")
        need(self.deepreduce in MODES, f"'deepreduce' must be one of {MODES} (got {self.deepreduce!r})")
        need(0.0 < self.compress_ratio <= 1.0, f"'compress_ratio' must be in (0, 1] (got {self.compress_ratio})")
        need(self.threshold >= 0.0, f"'threshold' must be >= 0 (got {self.threshold})")
        need(self.fpr is None or 0.0 < self.fpr < 1.0, f"'fpr' must be in (0, 1) (got {self.fpr})")
        need(self.policy in POLICIES, f"'policy' must be one of {POLICIES} (got {self.policy!r})")
        need(1 <= self.poly_degree <= 7, f"'poly_degree' must be in [1, 7] (got {self.poly_degree})")
        need(1 <= self.quantum_num <= 32767, f"'quantum_num' must be in [1, 32767] (got {self.quantum_num})")
        need(self.bucket_size >= 1, f"'bucket_size' must be >= 1 (got {self.bucket_size})")
        need(self.world_size is None or self.world_size >= 1, f"'world_size' must be >= 1 (got {self.world_size})")
        if self.deepreduce in ("value", "both"):
            need(self.value in registry, f"unknown value codec {self.value!r}; registered: {sorted(registry)}")
        if self.deepreduce in ("index", "both"):
            need(self.index in registry, f"unknown index codec {self.index!r}; registered: {sorted(registry)}")
        if self.deepreduce is not None:
            need(self.compressor != "none", "'deepreduce' needs a sparsifier: set 'compressor' to topk/threshold/randomk")
            need(self.communicator == "allgather",
                 "sparse payloads differ per rank: 'deepreduce' requires 'communicator': 'allgather'")
        if self.compressor in ("topk", "threshold"):         # randomk with a shared seed is all-reducible, like GRACE
            need(self.communicator == "allgather",
                 f"compressor {self.compressor!r} produces per-rank index sets: use 'communicator': 'allgather'")

    def ratio_at(self, exchange: int) -> float:
        """Compress ratio of the 0-based ``exchange`` (``spec.Warmup``; ``compress_ratio`` without a warm-up)."""
        if self.warmup_ratios is None:
            return self.compress_ratio
        return spec.Warmup(self.warmup_ratios, self.warmup_steps, self.compress_ratio).ratio_at(exchange)

    def to_params(self) -> dict:
        """Back to the dict form the codecs/wrappers take (a fresh dict; the 'micro-benchmark' key keeps its dash)."""
        d = asdict(self)
        d["micro-benchmark"] = d.pop("micro_benchmark")
        return {k: v for k, v in d.items() if v is not None}


def warmup_from_params(params: dict) -> Optional[spec.Warmup]:
    """The sparsity warm-up of ``params`` (``'warmup_ratios'``: a non-empty list of compress ratios in (0, 1],
    ``'warmup_steps'``: exchanges per stage, an int >= 1), validated; None when neither key is given."""
    has_r, has_s = "warmup_ratios" in params, "warmup_steps" in params
    if not (has_r or has_s):
        return None
    if has_r != has_s:
        raise ConfigError("'warmup_ratios' and 'warmup_steps' go together: give both or neither")
    comp = params.get("compressor", "none") or "none"
    if comp not in ("topk", "randomk"):
        raise ConfigError(f"the sparsity warm-up schedules the compress ratio of 'topk' or 'randomk' (got "
                          f"compressor={comp!r})")
    rs, n = params["warmup_ratios"], params["warmup_steps"]
    if not isinstance(rs, (list, tuple)) or not rs:
        raise ConfigError(f"'warmup_ratios' must be a non-empty list of numbers in (0, 1] (got {rs!r})")
    for r in rs:
        if isinstance(r, bool) or not isinstance(r, (int, float)) or not 0.0 < float(r) <= 1.0:
            raise ConfigError(f"'warmup_ratios' must be a non-empty list of numbers in (0, 1] (got {rs!r})")
    if isinstance(n, bool) or not isinstance(n, int) or n < 1:
        raise ConfigError(f"'warmup_steps' must be an int >= 1 (got {n!r})")
    return spec.Warmup(tuple(float(r) for r in rs), int(n), float(params.get("compress_ratio", 0.01)))


def validate_params(params: dict, *, strict: bool = False) -> DeepReduceConfig:
    return DeepReduceConfig.from_params(params, strict=strict)
