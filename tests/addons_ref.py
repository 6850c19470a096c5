"""Oracles for PAD, MIN / MAX, ARGMAX / ARGMIN and REDUCE_ISNAN: numpy restatements of the reference's CPU_REF loops
(cmd/pad/ccv_nnc_pad_cpu_ref.c, cmd/compare/ccv_nnc_{min,max}_cpu_ref.c, cmd/reduce/ccv_nnc_arg{max,min}_cpu_ref.c,
cmd/isnan/ccv_nnc_reduce_isnan_cpu_ref.c), pinned to CPU_REF by tests/golden/cpuref_addons.npz.

None of these commands does arithmetic, so the oracles work on raw element bits: fp32 tensors travel as float32 arrays (numpy copies
them bit for bit, NaN payloads included), 16-bit tensors as uint16 arrays of their bits.  Values are widened to fp32 only to be
compared, which is exact, so a 16-bit result is CPU_REF's on the widened values."""
import numpy as np

ZERO, REPLICATE = 0, 1  # CCV_NNC_PAD_ZERO / _REPLICATE
FP32, BF16, FP16 = "fp32", "bf16", "fp16"
ONE_BITS = {BF16: np.uint16(0x3f80), FP16: np.uint16(0x3c00)}


def widen(bits, kind):
    """the fp32 values of raw element bits of `kind`"""
    bits = np.asarray(bits)
    if kind == FP32:
        return bits.astype(np.float32, copy=False)
    if kind == BF16:
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.view(np.float16).astype(np.float32)


def one(kind):
    return np.float32(1) if kind == FP32 else ONE_BITS[kind]


def _sides(nd, begin, end):
    begin = list(begin)[:nd] + [0] * max(0, nd - len(begin))
    end = list(end)[:nd] + [0] * max(0, nd - len(end))
    return begin, end


def pad_forward(a, begin, end, pad_type):
    """b has dims a + begin + end per axis; zero: 0 outside a; replicate: a at min(adim - 1, max(0, i - begin)) on every axis"""
    begin, end = _sides(a.ndim, begin, end)
    idx, inside = [], np.ones([a.shape[k] + begin[k] + end[k] for k in range(a.ndim)], bool)
    for k in range(a.ndim):
        j = np.arange(a.shape[k] + begin[k] + end[k]) - begin[k]
        shape = [1] * a.ndim
        shape[k] = -1
        inside &= ((j >= 0) & (j < a.shape[k])).reshape(shape)
        idx.append(np.clip(j, 0, max(a.shape[k] - 1, 0)).reshape(shape))
    b = a[tuple(idx)]
    if pad_type == ZERO:
        b = np.where(inside, b, np.zeros((), a.dtype))
    return np.ascontiguousarray(b)


def pad_backward(g, begin, hshape):
    """h = g[begin : begin + hdim] for both pad types: CPU_REF does not add the replicated border into the edge elements"""
    begin, _ = _sides(g.ndim, begin, ())
    return np.ascontiguousarray(g[tuple(slice(begin[k], begin[k] + hshape[k]) for k in range(g.ndim))])


def cmp_forward(a, b, kind, is_min):
    """c = a < b ? a : b (MIN) / a > b ? a : b (MAX): ccv_min / ccv_max, so a NaN or a tie (±0) gives b's bits"""
    wa, wb = widen(a, kind), widen(b, kind)
    return np.where(wa < wb if is_min else wa > wb, a, b)


def cmp_backward(g, a, b, kind, is_min):
    """(ha, hb): g (1 without g) to the winner and 0 to the loser; both get g on a tie or a NaN"""
    wa, wb = widen(a, kind), widen(b, kind)
    a_wins, b_wins = (wa < wb, wb < wa) if is_min else (wa > wb, wb > wa)
    gv = np.full(a.shape, one(kind), a.dtype) if g is None else g
    zero = np.zeros((), a.dtype)
    return np.where(b_wins, zero, gv), np.where(a_wins, zero, gv)


def argext(x, axis, is_min):
    """CPU_REF's loop: max = x[0]; for k >= 1 a strict > (<) takes k.  x holds (widened) values; returns int32 with `axis` kept as 1"""
    x = np.moveaxis(np.asarray(x, np.float32), axis, 0)
    best, idx = x[0].copy(), np.zeros(x.shape[1:], np.int32)
    for k in range(1, x.shape[0]):
        take = x[k] < best if is_min else x[k] > best
        best = np.where(take, x[k], best)
        idx = np.where(take, np.int32(k), idx)
    return np.expand_dims(idx, axis)


def reduce_isnan(x, bshape):
    """b (int32, broadcast onto x; its unit axes are the reduced ones) = 1 where an element mapping to it is NaN, else 0"""
    x = np.asarray(x, np.float32)
    shape = tuple(bshape)
    bshape = (1,) * (x.ndim - len(shape)) + shape
    axes = tuple(k for k in range(x.ndim) if bshape[k] == 1 and x.shape[k] != 1)
    b = np.isnan(x).any(axis=axes, keepdims=True) if axes else np.isnan(x)
    return b.astype(np.int32).reshape(shape)
