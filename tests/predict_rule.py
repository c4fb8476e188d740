"""Host restatements for the prediction store tests (not a test module).

``top_k`` is the ranking of ddfa_predict_store (csrc/predict.cu) written the reference's way: Python's stable
``sorted(..., reverse=True)`` over the numbers, then the NaNs in node order.  ``top_k_by_keys`` restates the kernel's own
selection (the j-th largest 64-bit (score, node) key) in NumPy.
"""
import math

import numpy as np


def top_k(scores, k: int):
    """(indices int32 [k], scores fp32 [k]) of one function: ranks past its node count hold -1 and NaN."""
    s = np.asarray(scores, dtype=np.float32)
    ids = [i for i in range(len(s)) if not math.isnan(float(s[i]))]
    order = sorted(ids, key=lambda i: float(s[i]), reverse=True) + [i for i in range(len(s)) if math.isnan(float(s[i]))]
    idx = np.full(k, -1, np.int32)
    sc = np.full(k, np.nan, np.float32)
    take = order[:k]
    idx[:len(take)] = take
    sc[:len(take)] = s[take]
    return idx, sc


def _keys(scores):
    s = np.asarray(scores, dtype=np.float32).copy()
    s[s == 0] = 0.0                                           # -0.0 ties +0.0
    u = s.view(np.uint32).astype(np.uint64)
    hi = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    hi = np.where(np.isnan(s), 0, hi).astype(np.uint64)
    lo = (0xFFFFFFFF - np.arange(len(s), dtype=np.uint64)).astype(np.uint64)
    return (hi << np.uint64(32)) | lo


def top_k_by_keys(scores, k: int):
    keys = _keys(scores)
    order = np.argsort(keys)[::-1][:k]
    idx = np.full(k, -1, np.int32)
    sc = np.full(k, np.nan, np.float32)
    idx[:len(order)] = order
    sc[:len(order)] = np.asarray(scores, dtype=np.float32)[order]
    return idx, sc


def store(scores, bnn, k: int):
    """(indices [F, k], scores [F, k]) of every function of a batch (batch_num_nodes ``bnn``)."""
    out_i, out_s = [], []
    n0 = 0
    for n in np.asarray(bnn).tolist():
        i, s = top_k(np.asarray(scores, dtype=np.float32)[n0:n0 + n], k)
        out_i.append(i)
        out_s.append(s)
        n0 += n
    return np.stack(out_i) if out_i else np.zeros((0, k), np.int32), np.stack(out_s) if out_s else np.zeros((0, k), np.float32)


def same_bits(a, b) -> bool:
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def same_floats(a, b) -> bool:
    """Bit for bit, except that any NaN equals any NaN."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and same_bits(np.where(na, 0, a), np.where(nb, 0, b))
