"""Shared helpers for the test-suite (oracle access lives here, never in the product)."""
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def rel_row_err(a, b):
    """max over rows of |a-b|_2 / |b|_2 -- the 'relative error on per-point features' of the north star."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float((np.linalg.norm(a - b, axis=1) / (np.linalg.norm(b, axis=1) + 1e-30)).max())


def kmap_triples(maps):
    """oracle kernel map (list over k of (in_rows, out_rows)) -> set of (k, i, o)."""
    s = set()
    for k, (ii, oo) in enumerate(maps):
        s.update(zip([k] * len(ii), ii.tolist(), oo.tolist()))
    return s


def digest(a):
    """SHA-256 of an array's shape and values (integers as int64, floats as float64 bits, strings joined by newlines): an
    exact comparison that stores 64 characters."""
    a = np.asarray(a)
    if a.dtype.kind in 'US':
        data = '\n'.join(a.reshape(-1).tolist()).encode()
    else:
        data = np.ascontiguousarray(a, dtype=np.float64 if a.dtype.kind == 'f' else np.int64).tobytes()
    return hashlib.sha256(str(a.shape).encode() + data).hexdigest()
