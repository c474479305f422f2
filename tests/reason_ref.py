"""Reference ranking of per-row reason codes (sb_model_reason_codes).

A row's list positions j rank by a key: d for "raise", -d for "lower", |d| for "magnitude" (d the fp32 delta of
sb_model_sensitivity), a larger key first; keys compare as floats (-0 == +0), a NaN key ranks after every other key,
and equal keys rank by the smaller position.  The order is total, so the top k of a row is unique, and the top k of
the union of any blocks' top-k lists is the top k of the whole row: that is how the library merges a row's pieces."""
import numpy as np

ORDERS = ("raise", "lower", "magnitude")


def keys(d, order):
    """the float32 ranking keys of fp32 deltas"""
    d = np.asarray(d, np.float32)
    return {"raise": d, "lower": -d, "magnitude": np.abs(d)}[order]


def rank(d, order, pos=None):
    """[..., n] deltas (with their list positions, default 0 .. n-1) -> the indices along the last axis, best first: a
    stable lexsort on (NaN last, key descending, position)"""
    key = keys(d, order).astype(np.float64)
    pos = np.broadcast_to(np.arange(key.shape[-1]) if pos is None else np.asarray(pos), key.shape)
    nan = np.isnan(key)
    return np.lexsort((pos, np.where(nan, 0.0, -key), nan), axis=-1)


def topk(d, k, order, pos=None):
    """[rows, n] deltas -> (positions [rows, k], their deltas [rows, k]); pos: each delta's list position (default
    0 .. n-1 along the last axis)"""
    d = np.asarray(d, np.float32)
    p = np.broadcast_to(np.arange(d.shape[-1]) if pos is None else np.asarray(pos), d.shape)
    i = rank(d, order, p)[..., :k]
    return np.take_along_axis(p, i, -1).astype(np.int32), np.take_along_axis(d, i, -1)


def merged_topk(d, k, order, bounds):
    """the top k of each row merged block by block, as the library merges a row's pieces: the running list starts
    empty and after each block [b0, b1) becomes the top k of (running list | the block's deltas)"""
    d = np.asarray(d, np.float32)
    rp = np.zeros((d.shape[0], 0), np.int32)
    rd = np.zeros((d.shape[0], 0), np.float32)
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        bp = np.broadcast_to(np.arange(b0, b1, dtype=np.int32), (d.shape[0], b1 - b0))
        rp, rd = topk(np.concatenate([rd, d[:, b0:b1]], 1), k, order, np.concatenate([rp, bp], 1))
    return rp, rd
