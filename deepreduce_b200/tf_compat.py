"""TensorFlow-side API of the reference, re-hosted on PyTorch tensors.

The reference's TF half (tensorflow/deepreduce.py, 557 LoC, TF1 graph mode + Horovod)
exposes whole-GRACE-TF compressors with ``compress(tensor, params)`` /
``decompress(tensors, ctx, params)`` static methods, a class-level residual store and the
custom CPU ops.  TensorFlow/Horovod are not installable here, and a GPU-first framework has
one tensor runtime, so the same classes / parameter keys / wire formats are provided over
torch tensors:

* ``Compressor`` (memory_compensate / memory_update / aggregate)        reference :16-61
* ``Values_Approximation_Helper`` (double-exp fit, bases, knots, tables)  reference :64-253
* ``BloomFilterCompressor`` (single int8 blob, TF-op layout)              reference :256-373
* ``DoubleExpCompressor`` ("Fit-DExp")                                    reference :376-442
* ``PolySegCompressor`` ("Fit-Poly", static or data-driven breakpoints)   reference :445-557
"""
from __future__ import annotations

import json
import os
from typing import Dict

import torch

from . import spec
from .codecs import dexp as _dexp
from .codecs.bloom_cpu import bloom_compress_blob, bloom_decompress_blob
from .codecs.polyfit import gram_basis

_TABLES = None


def _tables():
    global _TABLES
    if _TABLES is None:
        with open(os.path.join(os.path.dirname(__file__), "data", "tf_break_tables.json")) as f:
            _TABLES = {k: {int(n): v for n, v in t.items()} for k, t in json.load(f).items() if not k.startswith("_")}
    return _TABLES


class Compressor(object):
    """Interface + error-feedback memory shared by the TF-style compressors."""

    residuals: Dict[str, torch.Tensor] = {}
    global_step = 0

    @staticmethod
    def compress(tensor, params):
        raise NotImplementedError

    @staticmethod
    def decompress(tensors, ctx, params):
        raise NotImplementedError

    @classmethod
    def memory_compensate(cls, tensor, params, name="t"):
        if params.get('use_memory', False):
            res = cls.residuals.setdefault(name, torch.zeros_like(tensor))
            tensor = params.get('beta', 1.0) * res + params.get('gamma', 1.0) * tensor
        return tensor

    @classmethod
    def memory_update(cls, tensor, tensor_compensate, tensor_compressed, ctx, params, name="t"):
        if params.get('use_memory', False):
            cls.residuals[name] = tensor_compensate - cls.decompress(tensor_compressed, ctx, params).view_as(tensor_compensate)
        return []

    @staticmethod
    def aggregate(tensors, params):
        agg = sum(tensors)
        return agg / params["horovod_size"] if params.get('average', True) else agg


class Values_Approximation_Helper(Compressor):
    double_exponential_fit = staticmethod(lambda X_, Y_, K=None: _dexp.double_exponential_fit(Y_))

    @staticmethod
    def logit_basis(X, a, N):
        return (a * torch.log(X / ((N + 1) - X))).double()

    @staticmethod
    def exp_basis(X, b, c):
        return (b * torch.exp(c * X)).double()

    @staticmethod
    def polynomial_basis(X, a):
        return torch.pow(X, a).double()

    @staticmethod
    def GetInputMatrix_Polynomial(xcol, x):
        x = x.double().flatten()
        return torch.stack([x ** i for i in range(xcol)], dim=1)

    @staticmethod
    def find_breaks(y_train, num_of_segments, N=None):
        """Greedy max-distance-from-chord knots (reference :167-180)."""
        y = y_train.double().flatten()
        N = y.numel() if N is None else int(N)
        b, pts = 0, [0]
        for _ in range(num_of_segments - 1):
            seg = y[b:N]
            if seg.numel() < 3:
                break
            line = torch.linspace(float(seg[0]), float(seg[-1]), seg.numel(), dtype=torch.float64, device=seg.device)
            b = b + int(torch.argmax((line - seg).abs()))
            pts.append(b)
        pts.append(N)
        pts = sorted(set(pts))
        return pts, [hi - lo for lo, hi in zip(pts[:-1], pts[1:])]

    @staticmethod
    def get_breaks(model, N):
        return _tables()[model][int(N)]

    @staticmethod
    def is_convolutional(model, N):
        return int(N) in _tables().get(model, {})

    @staticmethod
    def get_num_of_segments(model, N):
        return len(_tables()[model][int(N)]) - 1

    @staticmethod
    def LeastSquares(X, y):
        X = X.double()
        return torch.linalg.lstsq(X, y.double().reshape(-1, 1)).solution


class BloomFilterCompressor(Compressor):
    """``compress`` → one int8 blob ``[m:i32][h:i32][values][filter bytes]``; "Bloom on CPU"."""

    bloom_configuration = staticmethod(spec.bloom_configuration)

    @staticmethod
    def topk_indices(tensor, K):
        return torch.topk(tensor.abs().flatten(), K, sorted=False).indices.sort().values

    @staticmethod
    def threshold_indices(tensor, params):
        flat = tensor.flatten()
        thr = min(float(params["threshold_val"]), float(flat.abs().max()))
        return torch.nonzero(flat.abs() >= thr).flatten()

    @staticmethod
    def randomk_indices(tensor_name, N, K, device=None):
        seed = spec.policy_seed(BloomFilterCompressor.global_step, sum(str(tensor_name).encode()))
        BloomFilterCompressor.global_step += 1
        ar = torch.arange(N, device=device)
        keys = spec.policy_hash(ar, seed)
        comp = (keys << 31) | ar
        return torch.sort(torch.sort(comp).values[:K] & 0x7FFFFFFF).values

    @staticmethod
    def compress(tensor, params):
        flat = tensor.flatten()
        n = flat.numel()
        k = max(1, int(n * params["compress_ratio"]))
        assert params.get("bloom_fpr") is not None, "False Positive Rate is None"
        params['m'], params['k'] = spec.bloom_configuration(k, params["bloom_fpr"])
        on = params.get('bloom_on', 'topk')
        if on == "topk":
            idx = BloomFilterCompressor.topk_indices(flat, k)
        elif on == "randomk":
            idx = BloomFilterCompressor.randomk_indices(params.get('tensor_name', 't'), n, k, device=flat.device)
        else:
            idx = BloomFilterCompressor.threshold_indices(flat, params)
        step = int(params.get('step', 0))
        blob = bloom_compress_blob(flat[idx], idx, flat, step=step,
                                   false_positives_aware=params.get('bloom_false_positives_aware', True),
                                   policy=params.get('bloom_policy', 'conflict_sets'), fpr=params["bloom_fpr"])
        if params.get('bloom_verbosity_frequency', 0) and step % params['bloom_verbosity_frequency'] == 0 \
                and params.get('bloom_logs_path'):
            from .utils.metrics import log_compressor
            dense = bloom_decompress_blob(blob, n, step=step, policy=params.get('bloom_policy', 'conflict_sets'))
            log_compressor(params['bloom_logs_path'], params.get('rank', 0), step, params.get('gradient_id', 0), N=n,
                           K=k, true_indices=idx, selected_indices=dense.nonzero().flatten(),
                           bloom_bytes=int(blob[:4].view(torch.int32)), policy=params.get('bloom_policy', 'conflict_sets'),
                           verbosity=params.get('bloom_verbosity', 1))
        params['tensors_size_are_same'] = False
        # the op itself is a host op upstream too ("Bloom on CPU", tensorflow/deepreduce.py:256, DEVICE_CPU kernels); the
        # blob is handed back on the gradient's device so that the collective and the caller never see a device change
        return blob.to(tensor.device), tensor.shape

    @staticmethod
    def decompress(compressed_tensor, ctx, params):
        n = 1
        for s in ctx:
            n *= int(s)
        out = bloom_decompress_blob(compressed_tensor.cpu(), n, step=int(params.get('step', 0)),
                                    policy=params.get('bloom_policy', 'conflict_sets'))
        return out.view(tuple(ctx)).to(compressed_tensor.device)


class DoubleExpCompressor(Compressor):
    @staticmethod
    def compress(tensor, params):
        flat = tensor.flatten()
        n = flat.numel()
        k = max(1, int(n * params["compress_ratio"]))
        params['N'], params['K'] = n, k
        idx = torch.topk(flat.abs(), k).indices
        vals = flat[idx]
        if n > 9000:
            coef, signed_idx, _ = _dexp.DoubleExp.compress((vals, idx, torch.Size([n])), {})
            compressed = (signed_idx, coef.double())
        else:
            compressed = (idx.to(torch.int32), vals)
        params['tensors_size_are_same'] = True
        return compressed, (tensor.shape, n)

    @staticmethod
    def decompress(tensor_compressed, ctx, params):
        shape, n = ctx
        a, b = tensor_compressed
        if n > 9000:
            vals, idx, _ = _dexp.DoubleExp.decompress((b.float(), a, torch.Size([n])), {})
        else:
            idx, vals = a.long(), b
        out = torch.zeros(n, dtype=torch.float32, device=vals.device)      # stays on the gradient's device (GPU upstream, :422-442)
        out[idx] = vals.float()
        return out.view(tuple(shape))


class PolySegCompressor(Compressor):
    """Per-segment LS fit of |values| sorted ascending; sign folded into the index; wire =
    ``float64[sizes | coefficients | signed indices]`` (reference :511-513)."""

    @staticmethod
    def _breaks(values, params, N):
        model = params.get('model_name')
        if model and Values_Approximation_Helper.is_convolutional(model, N) and values.numel() == N:
            return Values_Approximation_Helper.get_breaks(model, N)
        nseg = int(params.get('num_of_segments', 4))
        pts, _ = Values_Approximation_Helper.find_breaks(values, nseg, values.numel())
        return pts

    @staticmethod
    def compress(tensor, params):
        flat = tensor.flatten()
        N = flat.numel()
        deg = int(params.get('polynomial_degree', 5))
        params['N'] = N
        eligible = params.get('model_name') is None or Values_Approximation_Helper.is_convolutional(params['model_name'], N)
        if not eligible:
            return tensor, tensor.shape
        absv = flat.abs()
        if params.get('approximation_mode', 'topk') == "topk":
            K = max(1, int(N * params["compress_ratio"]))
            top, mapping = torch.topk(absv, K, sorted=False)
            order = torch.argsort(top)
            values, mapping = top[order], mapping[order]
        else:
            K = N
            values, mapping = torch.sort(absv)
        params['K'] = K
        sign = torch.where(flat[mapping] < 0, -1, 1)
        signed = (mapping + 1) * sign
        pts = PolySegCompressor._breaks(values, params, N)
        sizes = [hi - lo for lo, hi in zip(pts[:-1], pts[1:])]
        params['num_of_segments'] = len(sizes)
        coefs = []
        for lo, hi in zip(pts[:-1], pts[1:]):
            n = hi - lo
            P = gram_basis(n, deg - 1, device=flat.device)   # `polynomial_degree` counts columns in the reference (:490)
            num = P.T @ values[lo:hi].double()
            den = (P * P).sum(0)
            coefs.append(torch.where(den > 0, num / den.clamp_min(1e-300), torch.zeros_like(num)))
        wire = torch.cat([torch.tensor(sizes, dtype=torch.float64, device=flat.device), torch.cat(coefs), signed.double()])
        params['tensors_size_are_same'] = True
        return wire, tensor.shape

    @staticmethod
    def decompress(tensor_compressed, ctx, params):
        N = params['N']
        eligible = params.get('model_name') is None or Values_Approximation_Helper.is_convolutional(params['model_name'], N)
        if not eligible:
            return tensor_compressed
        nseg, deg, K = params['num_of_segments'], int(params.get('polynomial_degree', 5)), params['K']
        sizes, coefs, signed = torch.split(tensor_compressed, [nseg, deg * nseg, K])
        sizes = sizes.long().tolist()
        coefs = coefs.view(nseg, deg)
        vals = torch.cat([gram_basis(n, deg - 1, device=coefs.device) @ coefs[i] for i, n in enumerate(sizes) if n > 0])
        signed = signed.long()
        idx = signed.abs() - 1
        out = torch.zeros(N, dtype=torch.float32, device=tensor_compressed.device)
        out[idx] = (vals * torch.sign(signed).double()).float()
        return out.view(tuple(ctx))
