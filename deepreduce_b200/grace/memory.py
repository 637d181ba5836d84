"""Error-feedback memories (GRACE ``memory`` key).

``ResidualMemory``: ``compensate: g <- beta*r + gamma*g`` and
``update: r <- g - decompress(compress(g))`` (SURVEY §2.5; TF twin in
reference tensorflow/deepreduce.py:31-52).  Unlike GRACE the residual state is
checkpointable (``state_dict``), see SURVEY §5.

``DgcMemory``: momentum correction, momentum factor masking and local gradient
clipping of Deep Gradient Compression (Lin et al., ICLR 2018).  The momentum is
accumulated locally, before the selection, and cleared wherever this rank's own
decoded contribution is non-zero.
"""
from __future__ import annotations

import fnmatch
import math

import torch

from .base import Memory


def is_dense(t: torch.Tensor) -> bool:
    """True if t's strides describe a permutation of a contiguous layout (contiguous, channels_last, ...): the layouts
    in which DDP keeps a parameter's gradient with the parameter's strides."""
    expect = 1
    for st, sz in sorted(zip(t.stride(), t.size())):
        if sz == 1:
            continue
        if st != expect:
            return False
        expect *= sz
    return True


def pairwise_sumsq(flat: torch.Tensor) -> float:
    """The sum of fl64(x_i)^2 over the 1-D tensor ``flat`` (each square is exact in fp64), in the one order the fused
    engine uses: zero-padded to 4096 * 2^ceil(log2 ceil(n / 4096)) elements and added by adjacent pairs,
    ``x = x[0::2] + x[1::2]``, until one value is left (per 4096-element tile, then over the tiles)."""
    n = flat.numel()
    tiles = max(1, -(-n // 4096))
    x = torch.zeros(4096 << (tiles - 1).bit_length(), dtype=torch.float64, device=flat.device)
    x[:n] = flat.detach().double()
    x = x * x
    while x.numel() > 1:
        x = x[0::2] + x[1::2]
    return float(x.item())


def decay_excluded(name: str, patterns) -> bool:
    """True if the parameter name matches one of the ``fnmatch`` patterns of ``'weight_decay_exclude'`` (matched case
    sensitively on every platform)."""
    return any(fnmatch.fnmatchcase(name, p) for p in patterns or ())


def check_exclude_patterns(patterns, names) -> None:
    """Raise ``ValueError`` naming every pattern of ``'weight_decay_exclude'`` that matches none of ``names``: a typo
    must not silently keep the decay."""
    names = list(names)
    dead = [p for p in patterns or () if not any(fnmatch.fnmatchcase(n, p) for n in names)]
    if dead:
        raise ValueError(f"'weight_decay_exclude': pattern(s) {dead} match none of the model's parameters")


def clip_factor(sumsq: float, thr: float):
    """DGC's local gradient clipping of one tensor with squared norm ``sumsq`` (``pairwise_sumsq``) at ``thr`` =
    c / sqrt(W): the fp32 factor fl32(thr / nrm) where nrm = sqrt(sumsq) is finite and > thr, else None (the gradient
    stays as it is: NaN is never > thr, and an infinite element leaves it alone too)."""
    nrm = math.sqrt(sumsq)
    if math.isfinite(nrm) and nrm > thr:
        return torch.tensor(thr / nrm, dtype=torch.float32)
    return None


class NoneMemory(Memory):
    def compensate(self, tensor, name):
        return tensor

    def update(self, tensor, name, compressor, tensor_compressed, ctx):
        pass


class ResidualMemory(Memory):
    def __init__(self, beta: float = 1.0, gamma: float = 1.0):
        self.residuals: dict[str, torch.Tensor] = {}
        self.beta = beta
        self.gamma = gamma

    def compensate(self, tensor, name):
        if name in self.residuals:
            tensor = self.beta * self.residuals[name] + self.gamma * tensor
        elif self.gamma != 1.0:
            tensor = self.gamma * tensor
        return tensor

    def update(self, tensor, name, compressor, tensor_compressed, ctx):
        tensor_decompressed = compressor.decompress(tensor_compressed, ctx)
        self.residuals[name] = tensor - tensor_decompressed.view_as(tensor)

    def state_dict(self):
        return {"beta": self.beta, "gamma": self.gamma,
                "residuals": {k: v.detach().cpu().clone() for k, v in self.residuals.items()}}

    def load_state_dict(self, state, device=None):
        self.beta = state.get("beta", self.beta)
        self.gamma = state.get("gamma", self.gamma)
        self.residuals = {k: (v.to(device) if device is not None else v.clone())
                          for k, v in state.get("residuals", {}).items()}


class DgcMemory(Memory):
    """Per tensor, with ``m = momentum``::

        u <- fl(fl(m * u) + g)          # two roundings, never a fused multiply-add
        v <- fl(v + u)                  # v: the residual, as ResidualMemory with beta = gamma = 1
        ... v is selected, encoded and shipped ...
        v <- v - own(v)                 # own(v): what the receivers rebuild from this rank's message
        u[i] <- 0 where own(v)[i] != 0  # momentum factor masking (-0.0 counts as zero)

    A tensor not seen before starts with ``u = v = g`` (no additions, so ``-0.0`` stays intact).  With ``m = 0`` and
    finite gradients it computes bit for bit what ``ResidualMemory()`` computes.  The momentum lives here, so the
    optimizer that follows must not add its own (e.g. ``SGD(momentum=0)``).

    ``weight_decay = wd > 0``: g is first replaced by ``fl(g + fl(wd * w))``, w the parameter ``bind_parameters`` bound
    to the tensor's name, as torch's momentum SGD puts the decay through its momentum buffer; the optimizer then runs
    without weight decay too.  With ``wd = 0`` nothing is read or added.

    ``clip_norm = c``: DGC's local gradient clipping, ahead of the weight decay.  Each tensor's g is replaced by
    ``fl32(g * fl32(thr / nrm))`` where its norm ``nrm`` (fp64, ``pairwise_sumsq`` over g in storage order, the order
    it has in a flat gradient bucket) is finite and > ``thr = c / sqrt(world_size)``.  Per tensor: the chunks of a
    split parameter are one tensor here anyway.  With no ``clip_norm`` nothing is computed.

    ``weight_decay_exclude``: ``fnmatch`` patterns; a tensor whose name matches one gets no weight decay (its parameter
    is not read, so it need not be bound), as a param group with ``weight_decay=0`` would in torch's SGD.

    ``nesterov=True``: Nesterov momentum.  The residual adds ``v = fl(d + fl(m * u))`` with the new u instead of u
    (d: g after clipping and decay); u itself is torch's ``momentum_buffer``.  Torch's CPU step rounds ``d + m * u``
    once (a fused multiply-add); here it is two roundings, as every other op of this memory.  A tensor's first step
    starts from ``u = d``, so its residual starts from ``fl(d + fl(m * d))``."""

    def __init__(self, momentum: float = 0.9, weight_decay: float = 0.0, clip_norm=None, world_size: int = 1,
                 nesterov: bool = False, weight_decay_exclude=()):
        self.momentum = float(momentum)
        self.weight_decay = float(weight_decay)
        self.nesterov = bool(nesterov)
        if self.nesterov and self.momentum == 0.0:
            raise ValueError("Nesterov momentum needs a momentum > 0")
        self.weight_decay_exclude = tuple(weight_decay_exclude or ())
        self.clip_norm = None if clip_norm is None else float(clip_norm)
        self.world_size = int(world_size)
        self.clip_thr = None if clip_norm is None else self.clip_norm / math.sqrt(self.world_size)
        self.momenta: dict[str, torch.Tensor] = {}
        self.residuals: dict[str, torch.Tensor] = {}
        self.parameters: dict[str, torch.Tensor] = {}
        self._storage_layout: dict[str, tuple] = {}   # storage-order names -> the parameter's strides when bound

    def bind_parameters(self, named_parameters, storage_order: bool = False):
        """``(name, parameter)`` pairs: the values the weight decay reads for the gradient of that name.

        ``storage_order=True``: the gradients of these names arrive as plain reshapes of a flat buffer that holds
        them in their parameters' storage order, as torch DDP's gradient buckets do (a dense parameter's gradient is
        laid out with the parameter's strides, e.g. channels_last).  w is then read in storage order too, so that
        element i of w belongs to element i of the gradient.  The parameter's layout must stay the one it had when it
        was bound: a change of strides raises."""
        for n, p in named_parameters:
            self.parameters[n] = p
            if storage_order:
                self._storage_layout[n] = tuple(p.stride())
            else:
                self._storage_layout.pop(n, None)

    def _weights(self, name, shape, dtype):
        w = self.parameters.get(name)
        if w is None:
            raise KeyError(f"'dgc' weight decay: no parameter is bound to {name!r} (bind_parameters)")
        w = w.detach()
        layout = self._storage_layout.get(name)
        if layout is not None:
            if tuple(w.stride()) != layout:
                raise ValueError(f"'dgc' weight decay: parameter {name!r} changed its layout from strides {layout} "
                                 f"to {tuple(w.stride())} after it was bound; its gradient keeps the old order")
            if is_dense(w):
                w = w.as_strided((w.numel(),), (1,))              # storage order
        return w.reshape(shape).to(dtype)

    def _clip(self, tensor):
        flat = tensor.as_strided((tensor.numel(),), (1,)) if is_dense(tensor) else tensor.reshape(-1)
        f = clip_factor(pairwise_sumsq(flat), self.clip_thr)
        if f is None:
            return tensor
        return (tensor.float() * f.to(tensor.device)).to(tensor.dtype)

    def compensate(self, tensor, name):
        if self.clip_thr is not None:
            tensor = self._clip(tensor)
        if self.weight_decay != 0.0 and not decay_excluded(name, self.weight_decay_exclude):
            tensor = tensor + (self.weight_decay * self._weights(name, tensor.shape, tensor.dtype))
        d = tensor
        u = self.momentum * self.momenta[name] + d if name in self.momenta else d
        v = d + (self.momentum * u) if self.nesterov else u
        tensor = self.residuals[name] + v if name in self.momenta else v
        self.momenta[name] = u
        return tensor

    def update(self, tensor, name, compressor, tensor_compressed, ctx):
        own = compressor.decompress(tensor_compressed, ctx).view_as(tensor)
        self.residuals[name] = tensor - own
        u = self.momenta[name]
        self.momenta[name] = torch.where(own != 0, torch.zeros_like(u), u)

    def state_dict(self):
        return {"momentum": self.momentum,
                "momenta": {k: v.detach().cpu().clone() for k, v in self.momenta.items()},
                "residuals": {k: v.detach().cpu().clone() for k, v in self.residuals.items()}}

    def load_state_dict(self, state, device=None):
        if "momenta" not in state:
            raise ValueError("not a 'dgc' memory state (no 'momenta'): it was saved with another memory")
        self.momentum = state.get("momentum", self.momentum)
        self.momenta = {k: (v.to(device) if device is not None else v.clone()) for k, v in state["momenta"].items()}
        self.residuals = {k: (v.to(device) if device is not None else v.clone())
                          for k, v in state.get("residuals", {}).items()}
