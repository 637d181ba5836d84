"""Sparse codecs + registry (reference pytorch/deepreduce.py:913-922)."""
from .base import SparseCompressor, compressor, register
from . import bitpack
from .bf16 import BF16
from .bloom import Bloom, Bloomfilter, get_BFconfig
from .bloom_cpu import BloomCPU, bloom_compress_blob, bloom_decompress_blob
from .dexp import DoubleExp
from .elias_fano import EliasFano
from .fp8 import FP8
from .integer import IntegerIndex
from .lossless import Gzip, Huffman
from .polyfit import PolyFit, PolyFitCPU, get_segments
from .qsgd import QSGD
from .rle import RunLength
from .sign import Sign

__all__ = ["SparseCompressor", "compressor", "register", "bitpack", "BF16", "Bloom", "Bloomfilter", "get_BFconfig",
           "BloomCPU", "bloom_compress_blob", "bloom_decompress_blob", "DoubleExp", "EliasFano", "FP8", "IntegerIndex",
           "Gzip", "Huffman", "PolyFit", "PolyFitCPU", "get_segments", "QSGD", "RunLength", "Sign"]
