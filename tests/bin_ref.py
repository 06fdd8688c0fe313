"""numpy statement of bin row storage (DESIGN.md §3d): which f32 values a bin row accepts, the stored byte layout (one byte per
4-element chunk, element 4c + k in bit k of byte c, high nibble zero), and the Hamming distance the squared L2 of 0/1 rows equals."""
import numpy as np


def refused(x):
    """Per element: True unless the value is +0.0, -0.0 or 1.0 (bit patterns, so NaN payloads and subnormals are refused too)."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((b & 0x7FFFFFFF) != 0) & (b != 0x3F800000)


def pack(x):
    """Accepted rows (n x dim) -> the stored bytes (n x ceil(dim / 4))."""
    x = np.asarray(x, np.float32)
    n, dim = x.shape
    nchunks = (dim + 3) // 4
    bits = np.zeros((n, nchunks * 4), np.uint8)
    bits[:, :dim] = x == 1.0
    return (bits.reshape(n, nchunks, 4) << np.arange(4, dtype=np.uint8)).sum(axis=2, dtype=np.uint8)


def unpack(codes, dim):
    """Stored bytes -> the 0/1 f32 rows they widen to."""
    codes = np.asarray(codes, np.uint8)
    bits = (codes[:, :, None] >> np.arange(4, dtype=np.uint8)) & 1
    return bits.reshape(codes.shape[0], -1)[:, :dim].astype(np.float32)


def hamming(q, x):
    """Integer Hamming distances between 0/1 rows: q (nq x dim) against x (n x dim), through packed bits and popcounts."""
    qp = np.packbits(np.asarray(q, np.float32) != 0, axis=1)
    xp = np.packbits(np.asarray(x, np.float32) != 0, axis=1)
    return np.unpackbits(qp[:, None, :] ^ xp[None, :, :], axis=2).sum(axis=2, dtype=np.int64)


def binarise(x, ref=None):
    """Each element 1 where it is above the median of its column in `ref` (default: x itself), else 0 (the benchmark's and the
    tests' 0/1 data: queries take the points' medians)."""
    x = np.asarray(x, np.float32)
    return (x > np.median(x if ref is None else ref, axis=0)).astype(np.float32)
