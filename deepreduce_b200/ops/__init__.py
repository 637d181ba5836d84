"""Native op loader + thin Python wrappers over the sm_90a kernels.

``_dr_cuda.so`` / ``_dr_cpu.so`` are built in-tree by ``ops/build.py``
(``__graft_entry__.build()``).  On a box with a GPU a missing CUDA extension is a
hard error (``require()``) — there is no silent PyTorch fallback for CUDA
tensors; the ``*_oracle`` functions in ``codecs/`` are only used for CPU tensors
and as the numerics reference in tests.
"""
from __future__ import annotations

import importlib
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

from .. import spec

_HERE = os.path.dirname(os.path.abspath(__file__))
_cuda_mod = None
_cpu_mod = None
_cuda_err = None
_cpu_err = None


def _load(name):
    if _HERE not in sys.path:
        sys.path.insert(0, _HERE)
    return importlib.import_module(name)


def _try_load_all():
    global _cuda_mod, _cpu_mod, _cuda_err, _cpu_err
    if _cpu_mod is None and _cpu_err is None:
        try:
            _cpu_mod = _load("_dr_cpu")
        except Exception as e:  # noqa: BLE001
            _cpu_err = e
    if _cuda_mod is None and _cuda_err is None:
        try:
            _cuda_mod = _load("_dr_cuda")
        except Exception as e:  # noqa: BLE001
            _cuda_err = e


_try_load_all()


def has_cpu_native() -> bool:
    return _cpu_mod is not None


def has_cuda_native() -> bool:
    return _cuda_mod is not None


def available() -> bool:
    return _cuda_mod is not None and torch.cuda.is_available()


def require() -> bool:
    """True if the CUDA kernels are usable; raises if a GPU is present but the
    extension is not (never fall back silently on a GPU box)."""
    if _cuda_mod is None:
        raise RuntimeError(
            "deepreduce_b200: CUDA tensor given but the sm_90a extension is not built/loadable "
            f"({_cuda_err!r}). Run `python -c 'import __graft_entry__ as g; g.build()'`.")
    return True


def cuda_module():
    require()
    return _cuda_mod


def launch_count() -> int:
    return int(_cuda_mod.launch_count()) if _cuda_mod is not None else 0


# ---------------------------------------------------------------------------
# host native namespace (numpy in / numpy out)
# ---------------------------------------------------------------------------
def _mk_cpu():
    if _cpu_mod is None:
        return None
    m = _cpu_mod

    def conflict_sets(positives, K, k, m_bits, seed, pseed):
        arr = positives.numpy() if torch.is_tensor(positives) else np.asarray(positives, dtype=np.int64)
        return torch.from_numpy(m.conflict_sets(arr, int(K), int(k), int(m_bits), int(seed) & spec.MASK32,
                                                int(pseed) & spec.MASK32))

    return SimpleNamespace(
        bloom_insert=lambda idx, k, m_bits, seed: m.bloom_insert(np.ascontiguousarray(idx, dtype=np.int64), int(k),
                                                                 int(m_bits), int(seed) & spec.MASK32),
        bloom_select=lambda words, d, K, k, m_bits, seed, policy, pseed: m.bloom_select(
            np.ascontiguousarray(words, dtype=np.uint32), int(d), int(K), int(k), int(m_bits),
            int(seed) & spec.MASK32, int(policy), int(pseed) & spec.MASK32),
        conflict_sets=conflict_sets,
        int_encode=lambda cid, a: m.int_encode(int(cid), np.ascontiguousarray(a, dtype=np.uint32)),
        int_decode=lambda cid, w, n: m.int_decode(int(cid), np.ascontiguousarray(w, dtype=np.uint32), int(n)),
        write_csv=lambda path, v: m.write_csv(str(path), np.ascontiguousarray(v, dtype=np.float64)),
        BloomFilter=m.BloomFilter,      # insert / query / words / num_bytes / num_hashes / hash / compute_false_positives
    )


cpu = _mk_cpu()


# ---------------------------------------------------------------------------
# CUDA per-tensor ops (GRACE-compatible path)
# ---------------------------------------------------------------------------
def bloom_insert(idxs: torch.Tensor, k: int, m_bits: int, seed: int = spec.DEFAULT_SEED) -> torch.Tensor:
    return cuda_module().bloom_insert(idxs.long().contiguous(), int(k), int(m_bits), int(seed))


def bloom_select(words, d, K, k, m_bits, policy, pseed=42, seed=spec.DEFAULT_SEED):
    mod = cuda_module()
    words = words.contiguous()
    if policy == "p0":
        return mod.bloom_select(words, int(d), -1, int(k), int(m_bits), int(seed))
    if policy == "leftmost":
        return mod.bloom_select(words, int(d), int(K), int(k), int(m_bits), int(seed))
    if policy == "random":
        from ..codecs.bloom import apply_policy_oracle
        pos = mod.bloom_select(words, int(d), -1, int(k), int(m_bits), int(seed))
        return apply_policy_oracle(pos, K, "random", pseed, k, m_bits, seed)
    raise ValueError(policy)


def topk_select(flat: torch.Tensor, k: int):
    """Exact top-k by |x| through the engine's radix-select (raw mode)."""
    from ..parallel.engine import topk_select_cuda
    return topk_select_cuda(flat, k)


def qsgd_encode(vals, q, bucket, seed):
    lvl, norms = cuda_module().qsgd_encode(vals.contiguous(), int(q), int(bucket), int(seed))
    return lvl, norms


def qsgd_decode(lvl, norms, q, bucket):
    return cuda_module().qsgd_decode(lvl.contiguous(), norms.contiguous(), int(q), int(bucket))


def sign_encode(vals):
    """Scaled-sign code of fp32 ``vals`` in 512-value buckets: (bits int32[ceil(K/32)], scales fp32[ceil(K/512)]);
    torch oracle: codecs.sign.sign_encode_oracle."""
    bits, scales = cuda_module().sign_encode(vals.float().contiguous())
    return bits, scales


def sign_decode(bits, scales, K):
    return cuda_module().sign_decode(bits.contiguous(), scales.contiguous(), int(K))


def fp8_encode(vals):
    """E4M3 code of fp32 ``vals`` with a scale byte per 32-value block: (scale words int32[ceil(ceil(K/32)/4)], element
    words int32[ceil(K/4)]), four bytes per word; torch oracle: codecs.fp8.fp8_encode_oracle."""
    scales, elems = cuda_module().fp8_encode(vals.float().contiguous())
    return scales, elems


def fp8_decode(scales, elems, K):
    return cuda_module().fp8_decode(scales.contiguous(), elems.contiguous(), int(K))


def pack_bits(vals, bits):
    return cuda_module().pack_bits(vals.contiguous(), int(bits))


def unpack_bits(buf, n, bits):
    return cuda_module().unpack_bits(buf.contiguous(), int(n), int(bits))


def _seg_tensors(segments, device):
    lens = torch.tensor(list(segments), dtype=torch.int32)
    offs = torch.cumsum(lens, 0, dtype=torch.int32) - lens
    return offs.to(device), lens.to(device)


def polyfit_fit(y_sorted, segments, degree):
    from ..codecs.polyfit import MAX_SEGMENTS
    offs, lens = _seg_tensors(segments, y_sorted.device)
    return cuda_module().polyfit_fit(y_sorted.float().contiguous(), offs, lens, int(degree), MAX_SEGMENTS)


def polyfit_eval(coeffs, segments, degree, total):
    offs, lens = _seg_tensors(segments, coeffs.device)
    return cuda_module().polyfit_eval(coeffs.float().contiguous(), offs, lens, int(degree), int(total))


def dexp_fit(y_ascending):
    """(a, b, p, q) float64[4] of the double-exponential fit of ascending |values| — one-CTA sm_90a kernel
    (scans + moment sums + both small solves); torch oracle: codecs.dexp.double_exponential_fit."""
    return cuda_module().dexp_fit(y_ascending.contiguous())


def delta_bp128_encode(idxs):
    return cuda_module().delta_bp128_encode(idxs.long().contiguous())


def delta_bp128_decode(payload, n):
    return cuda_module().delta_bp128_decode(payload.to(torch.int32).contiguous(), int(n))


def rle_runs(idxs, d):
    return cuda_module().rle_runs(idxs.long().contiguous(), int(d))


def rle_indices(runs, n):
    return cuda_module().rle_indices(runs.long().contiguous())


def u8_to_nhwc_norm(x_u8, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
    return cuda_module().u8_to_nhwc_norm(x_u8.contiguous(), list(mean), list(std))
