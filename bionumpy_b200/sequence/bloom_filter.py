"""BloomFilter over k-mer hashes (mirror of bionumpy/sequence/bloom_filter.py:15-42): hash function i is
``kmer ^ offset_i``, reduced mod the mask size; the mask is one byte per position like the reference's bool array.
Insert and membership run as one kernel each over all values and all hash functions (bnpk_bloom_insert / _query)."""
import numpy as np
import torch

from .. import _native as nv
from .. import ops
from ..encoded_array import EncodedArray
from ..ragged import RaggedArray


def _values(x):
    if isinstance(x, RaggedArray):
        x = x.raw().ravel() if hasattr(x, "encoding") else x.ravel()
    if isinstance(x, EncodedArray):
        x = x.raw()
    if not isinstance(x, torch.Tensor):
        x = torch.as_tensor(np.asarray(x, dtype=np.int64))
    if not x.is_cuda:
        from .. import config
        dev = config.default_device()
        if dev.type != "cuda":
            raise nv.NativeLibraryError("BloomFilter needs a CUDA device: bionumpy_b200 has no CPU fallback")
        x = x.to(dev)
    return x.to(torch.int64).contiguous()


class BloomFilter:
    def __init__(self, mask_size, offsets, device=None):
        from .. import config
        dev = torch.device(device) if device is not None else config.default_device()
        if dev.type != "cuda":
            raise nv.NativeLibraryError("BloomFilter needs a CUDA device: bionumpy_b200 has no CPU fallback")
        self._offsets = torch.as_tensor(np.asarray(offsets, dtype=np.int64)).to(dev)
        self._mask = torch.zeros(int(mask_size), dtype=torch.uint8, device=dev)

    @classmethod
    def from_m_and_k(cls, m, k, seed=12345):
        """bloom_filter.py:26-29: k hash functions with random offsets below m."""
        return cls(m, np.random.RandomState(seed).randint(0, m, k))

    @classmethod
    def from_hash_functions_and_seqeuences(cls, offsets, sequence, mask_size):
        """bloom_filter.py:31-35 (the reference's spelling kept)."""
        f = cls(mask_size, offsets)
        f.insert(sequence)
        return f

    def insert(self, sequences):
        """bloom_filter.py:37-39."""
        ops.bloom_insert(_values(sequences).reshape(-1), self._offsets, self._mask)

    def __getitem__(self, idx):
        """bloom_filter.py:41-42: membership of every value (bool tensor of the same shape)."""
        v = _values(idx)
        return ops.bloom_query(v.reshape(-1), self._offsets, self._mask).to(torch.bool).reshape(v.shape)
