"""deepreduce_b200 — an H100-native (Hopper, sm_90a) sparse-gradient communication framework with
the capabilities and API of hangxu0304/DeepReduce (see SURVEY.md, DESIGN.md).

Front door (GRACE-compatible, reference README.md:30-48)::

    from deepreduce_b200 import deepreduce_from_params
    grc = deepreduce_from_params({'compressor': 'topk', 'memory': 'residual',
                                  'communicator': 'allgather', 'compress_ratio': 0.01,
                                  'deepreduce': 'index', 'index': 'bloom'})
    new_grad = grc.step(grad, name)

Fast path (fused, bucketed, P2P over NVLink): ``deepreduce_b200.parallel``.
"""
from . import spec
from .codecs import SparseCompressor, compressor, register
from .grace import (Allgather, Allreduce, Communicator, Compressor, Memory, NoneCompressor, NoneMemory,
                    RandomKCompressor, ResidualMemory, ThresholdCompressor, TopKCompressor, grace_from_params,
                    tensor_bits)
from .wrappers import (DeepReduce, IndexCompressor, ValueCompressor, deepreduce_from_params, deepreduce_wrapper,
                       from_params)

__version__ = "0.1.0"

__all__ = ["spec", "SparseCompressor", "compressor", "register", "Allgather", "Allreduce", "Communicator",
           "Compressor", "Memory", "NoneCompressor", "NoneMemory", "RandomKCompressor", "ResidualMemory",
           "ThresholdCompressor", "TopKCompressor", "grace_from_params", "tensor_bits", "DeepReduce",
           "IndexCompressor", "ValueCompressor", "deepreduce_from_params", "deepreduce_wrapper", "from_params"]
