"""Relative data volume of every DeepReduce variant on the paper's model shapes (CPU, synthetic gradients),
next to the numbers the reference publishes (BASELINE.md §1: paper Table 2 / Table 5 / §6.1 / Fig. 8a).

    python scripts/volume_table.py > profiles/volume_table.md

"Relative volume" = bits on the wire / (32 · d), summed over all parameter tensors of the model, exactly what the
reference prints under 'micro-benchmark' (pytorch/deepreduce.py:93-95,148-150,297-299).  Indices of the plain Top-r
row are counted at 32 bits like the paper does (GRACE ships int64).  Gradients are N(0,1) draws of the parameter
shapes — volumes of bloom/QSGD/top-k do not depend on the values; the curve-fit rows depend only on K."""
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepreduce_b200 import deepreduce_from_params  # noqa: E402
from deepreduce_b200.grace import tensor_bits  # noqa: E402
from deepreduce_b200.models import resnet20  # noqa: E402
from deepreduce_b200.models.zoo import MobileNet, NextWordLSTM  # noqa: E402


def model_volume(model, params):
    grc = deepreduce_from_params(params)
    gen = torch.Generator().manual_seed(0)
    bits = dense = 0
    for name, p in model.named_parameters():
        g = torch.randn(p.shape, generator=gen)
        tensors, _ = grc.compressor.compress(g, name)
        tensors = tensors if isinstance(tensors, (list, tuple)) else [tensors]
        bits += tensor_bits([t for t in tensors if torch.is_tensor(t)])
        dense += 32 * p.numel()
    return bits / dense


def topr_paper(model, ratio):
    d = sum(p.numel() for p in model.parameters())
    k = sum(max(1, int(p.numel() * ratio)) for p in model.parameters())
    return 64.0 * k / (32.0 * d)


def main():
    base = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather'}
    rows = []
    # --- federated configs of the paper: Top-r 10 % (Table 2: LSTM / StackOverflow, Table 5: MobileNet / CIFAR-10)
    for label, model, pub in (("NextWordLSTM (4 053 428 params), Top-r 10 %", NextWordLSTM(),
                               {"Top-r": 0.2033, "BF-P0": 0.1425, "Fit-Poly": 0.1039, "BF-P0 + QSGD": 0.0621}),
                              ("MobileNet / CIFAR-10, Top-r 10 %", MobileNet(),
                               {"Top-r": 0.2069, "BF-P0": 0.1475, "Fit-Poly": 0.1087, "BF-P0 + QSGD": 0.0713})):
        r = 0.1
        cfgs = {"Top-r": None,
                "BF-P0": {**base, 'compress_ratio': r, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'p0', 'fpr': 0.001},
                "Fit-Poly": {**base, 'compress_ratio': r, 'deepreduce': 'value', 'value': 'polyfit'},
                "BF-P0 + QSGD": {**base, 'compress_ratio': r, 'deepreduce': 'both', 'index': 'bloom', 'policy': 'p0',
                                 'fpr': 0.001, 'value': 'qsgd', 'quantum_num': 127, 'bucket_size': 512}}
        for name, cfg in cfgs.items():
            ours = topr_paper(model, r) if cfg is None else model_volume(model, cfg)
            rows.append((label, name, pub[name], ours))
    # --- ResNet-20, Top-r 1 % (paper §6.1 / Fig. 4-5: BF-P0 with FPR 1e-3 is 33 % below Top-r; Fit-Poly ~40 %, Fit-DExp ~50 %)
    m = resnet20()
    top = topr_paper(m, 0.01)
    for name, cfg, pub in (("Top-r", None, None),
                           ("BF-P0 (fpr 1e-3)", {**base, 'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'bloom',
                                                 'policy': 'p0', 'fpr': 0.001}, top * (1 - 0.33)),
                           ("Fit-Poly", {**base, 'compress_ratio': 0.01, 'deepreduce': 'value', 'value': 'polyfit'}, top * 0.6),
                           ("Fit-DExp", {**base, 'compress_ratio': 0.01, 'deepreduce': 'value', 'value': 'dexp'}, top * 0.5),
                           ("BF (leftmost) + Fit-Poly ('both')", {**base, 'compress_ratio': 0.01, 'deepreduce': 'both',
                                                                  'index': 'bloom', 'value': 'polyfit'}, None),
                           ("RLE index", {**base, 'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'rle'}, None),
                           ("Elias-Fano index", {**base, 'compress_ratio': 0.01, 'deepreduce': 'index',
                                                 'index': 'elias_fano'}, None),
                           ("Elias-Fano index + sign values", {**base, 'compress_ratio': 0.01, 'deepreduce': 'both',
                                                               'index': 'elias_fano', 'value': 'sign'}, None),
                           ("Elias-Fano index + fp8 values", {**base, 'compress_ratio': 0.01, 'deepreduce': 'both',
                                                              'index': 'elias_fano', 'value': 'fp8'}, None),
                           ("delta + bp128 index", {**base, 'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'integer'}, None),
                           ("Huffman index", {**base, 'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'huffman'}, None)):
        ours = top if cfg is None else model_volume(m, cfg)
        rows.append(("ResNet-20 (269 722 params), Top-r 1 %", name, pub, ours))
    print("# Relative data volume vs the reference's published numbers (CPU run of `scripts/volume_table.py`)\n")
    print("Bits on the wire / (32·d) over all parameter tensors, through the GRACE-compatible per-tensor API "
          "(`deepreduce_from_params(...).compressor.compress`).  Published = paper Table 2 / Table 5 / §6.1 (BASELINE.md §1); "
          "for ResNet-20 the paper gives reductions relative to Top-r (33 % / ≈40 % / ≈50 %), converted here.  "
          "Tensors ≤ 1000 elements bypass the codecs (reference `:68,84,114`), like upstream.\n")
    print("| model / sparsifier | variant | published | ours | ours ÷ published |")
    print("|---|---|---|---|---|")
    for label, name, pub, ours in rows:
        print(f"| {label} | {name} | {'—' if pub is None else f'{pub:.4f}'} | {ours:.4f} | "
              f"{'—' if pub is None else f'{ours / pub:.2f}'} |")
    print("""
Notes.  (i) Keys travel as int32, coefficient tables are sized by K (`codecs/polyfit.py::seg_rows`), and an
order-preserving value codec (QSGD, Deflate) ships no reorder mapping in 'both' mode — with the reference's int64 keys,
always-present int64 mapping and our earlier fixed 22-row table the Fit-Poly and BF+QSGD rows were 1.7–2.4× the published
values.  (ii) BF-P0 on ResNet-20: fp32 values for K + 0.001·d positives plus 14.4 bit/key of filter give 0.0155 before the
P0 count word; the paper's "33 % less data than Top-r" (0.0135) is quoted from its plot.  (iii) Fit-DExp fits only tensors
with more than 9000 elements like the reference (`tensorflow/deepreduce.py:396,426`); smaller ones ship plain pairs.
(iv) The fused engine's own wire (bucketed, `BucketPlan.wire_bytes`) is reported by `bench.py` as `relative_volume`:
1.6 % (bloom + hint), 1.1 % ('both'), 0.15 % (NCF, top-k 0.1 % + run-length index).""")


if __name__ == "__main__":
    main()
