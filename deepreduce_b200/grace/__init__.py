from .base import Communicator, Compressor, Memory
from .communicators import Allgather, Allreduce
from .helper import grace_from_params, tensor_bits
from .memory import DgcMemory, NoneMemory, ResidualMemory
from .sparsifiers import NoneCompressor, RandomKCompressor, ThresholdCompressor, TopKCompressor

__all__ = ["Communicator", "Compressor", "Memory", "Allgather", "Allreduce", "grace_from_params",
           "tensor_bits", "NoneMemory", "ResidualMemory", "DgcMemory", "NoneCompressor", "RandomKCompressor",
           "ThresholdCompressor", "TopKCompressor"]
