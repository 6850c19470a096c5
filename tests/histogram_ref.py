"""numpy restatement of HISTOGRAM_FORWARD and EWPROD forward / backward as CPU_REF computes them (histogram/ccv_nnc_histogram_cpu_ref.c,
ew/ccv_nnc_ew_cpu_ref.c:235-480 of the reference; DESIGN.md §2).  Float32 arithmetic step by step, sums accumulated in float64 in element
order (np.cumsum, which is sequential, not np.sum, which is pairwise), min / max by the scan definition.  Values arrive as the view's
elements in row-major order; 16-bit tensors are widened to float32 first.

`defect` names a plausible kernel mistake the CPU tests show the fixture rejects."""
import ctypes as C

import numpy as np

from ccv_b200 import abi

f32 = np.float32
EVEN, LOG, BINS = abi.CCV_NNC_HISTOGRAM_EVEN, abi.CCV_NNC_HISTOGRAM_LOGARITHMIC, abi.CCV_NNC_HISTOGRAM_BINS
INT_MIN = -2 ** 31

_libm = C.CDLL("libm.so.6")
_libm.logf.restype, _libm.logf.argtypes = C.c_float, [C.c_float]


def host_logf(x):
    """the host's own logf (what CPU_REF calls), element by element"""
    return np.array([_libm.logf(float(v)) for v in np.ravel(x)], f32).reshape(np.shape(x))


def cr_logf(x):
    """the correctly rounded float logarithm (float64 log rounded once)"""
    return np.log(np.asarray(x, np.float64)).astype(f32)


def cvtt(t):
    """x86-64 cvttss2si: truncate toward zero, INT_MIN for NaN and anything outside int range"""
    t = np.asarray(t, f32)
    ok = (t >= f32(-2147483648.0)) & (t < f32(2147483648.0))
    return np.where(ok, np.trunc(np.where(ok, t, 0)).astype(np.int64), INT_MIN)


def wrap32(x):
    return ((np.asarray(x, np.int64) + 2 ** 31) % 2 ** 32) - 2 ** 31


def log_params(lo, hi, rate):
    """(log_base, u, min_inv) as the reference's host code computes them"""
    log_base = f32(1.0 / float(host_logf(f32(rate))))
    u = int(np.ceil(f32(host_logf(f32(f32(hi) / f32(lo))) * log_base)))
    min_inv = f32(1.0 / float(f32(lo)))
    return log_base, u, min_inv


def bin_count(type_, bins=0, lo=0.0, hi=0.0, rate=0.0, nbounds=0):
    if type_ == EVEN:
        return bins + 3
    if type_ == BINS:
        return nbounds + 2
    return 2 * log_params(lo, hi, rate)[1] + 2


def upper_bound(v, bounds, defect=None):
    """CPU_REF's _upper_bound for every element of v at once: the same midpoints, the same `v < bounds[mid]`"""
    v = np.asarray(v, f32)
    bounds = np.asarray(bounds, f32)
    hi = np.full(v.shape, len(bounds), np.int64)
    lo = np.full(v.shape, -1, np.int64)
    live = lo + 1 < hi
    while live.any():
        mid = ((hi - lo) >> 1) + lo
        bm = bounds[np.where(live, mid, 0)]
        left = (v <= bm) if defect == "le_search" else (v < bm)
        hi = np.where(live & left, mid, hi)
        lo = np.where(live & ~left, mid, lo)
        live = lo + 1 < hi
    return hi


def bin_index(v, type_, bins=0, lo=0.0, hi=0.0, rate=0.0, bounds=None, logf=cr_logf, defect=None):
    """the bin of every element of v (float32, 1-d)"""
    v = np.asarray(v, f32)
    nan = np.isnan(v)
    with np.errstate(all="ignore"):
        if type_ == EVEN:
            lo, hi = f32(lo), f32(hi)
            rng = f32(f32(bins) / f32(hi - lo))
            if defect == "fused_even":
                t = ((v.astype(np.float64) - float(lo)) * float(rng)).astype(f32)
            else:
                t = f32(v - lo) * rng
            i = np.clip(wrap32(cvtt(t) + 1), 1, bins)
            i = np.where(v >= hi, bins + 1, i)
            i = np.where(v < lo, 0, i)
            return np.where(nan, bins + 2, i)
        if type_ == LOG:
            lo, hi = f32(lo), f32(hi)
            log_base, u, min_inv = log_params(lo, hi, rate)
            mid = ~nan & (v < hi) & (v > -hi) & ~((v < lo) & (v > -lo))
            y = np.where(mid, np.abs(v) * min_inv, f32(1))
            idx = cvtt(np.ceil(logf(y) * log_base))
            i = np.clip(wrap32(np.where(v > 0, u + idx, u - idx)), 0, 2 * u)
            i = np.where((v < lo) & (v > -lo), u, i)
            i = np.where(v <= -hi, 0, i)
            i = np.where(v >= hi, 2 * u, i)
            return np.where(nan, 2 * u + 1, i)
        n = len(bounds)
        return np.where(nan, n + 1, upper_bound(np.where(nan, 0, v), bounds, defect))


def scan_extremes(v, defect=None):
    """(min, max) of m = m < v ? m : v and m = m > v ? m : v from v[0], as float32 with the selected element's bits"""
    v = np.asarray(v, f32)
    if defect == "fminf":
        return f32(np.fmin.reduce(v)), f32(np.fmax.reduce(v))
    nan = np.flatnonzero(np.isnan(v))
    last = nan[-1] if len(nan) else -1
    if last == len(v) - 1:
        return v[-1], v[-1]
    tail = v[last + 1:]
    # of equal values the later element wins: the last index holding the extreme
    lo, hi = tail.min(), tail.max()
    return tail[np.flatnonzero(tail == lo)[-1]], tail[np.flatnonzero(tail == hi)[-1]]


def sums(v, defect=None):
    """(float)sum and (float)sum of squares: double accumulations of v and of (float)(v * v) in element order"""
    v = np.asarray(v, f32)
    with np.errstate(all="ignore"):
        sq = (v * v).astype(np.float64)
    if defect == "pairwise":
        return f32(np.sum(v.astype(np.float64))), f32(np.sum(sq))
    return f32(np.cumsum(v.astype(np.float64))[-1]), f32(np.cumsum(sq)[-1])


def histogram(v, type_, bins=0, lo=0.0, hi=0.0, rate=0.0, bounds=None, nb=None, logf=cr_logf, defect=None):
    """-> (b int32 of nb counts (the rule's count by default), s float32[4]) for the float32 values v in the view's row-major order"""
    v = np.asarray(v, f32).ravel()
    need = bin_count(type_, bins, lo, hi, rate, 0 if bounds is None else len(bounds))
    idx = bin_index(v, type_, bins, lo, hi, rate, bounds, logf, defect)
    b = np.bincount(idx, minlength=nb or need).astype(np.int32)
    mn, mx = scan_extremes(v, defect)
    s, sq = sums(v, defect)
    return b, np.array([mn, mx, s, sq], f32)


def sum_bound(v):
    """|double sum - exact sum| <= count 2^-53 sum |x|, for the sum and for the sum of squares"""
    v = np.asarray(v, np.float64)
    with np.errstate(all="ignore"):
        sq = (np.asarray(v, f32) * np.asarray(v, f32)).astype(np.float64)
    n = len(v)
    return n * 2.0 ** -53 * np.abs(v).sum(), n * 2.0 ** -53 * np.abs(sq).sum()


def ewsum_order(ptrs, out):
    """EWSUM's / EWPROD's operand order: the first operand z >= 1 that is the output's storage goes first"""
    k = next((z for z in range(1, len(ptrs)) if ptrs[z] == out), 0)
    return [k] + [z for z in range(len(ptrs)) if z != k]


def ewprod(arrays, alias=None, defect=None):
    """c = product in CPU_REF's order; alias: the input index whose storage c is (None: none)"""
    order = list(range(len(arrays))) if defect == "plain_order" or alias is None else ewsum_order(list(range(len(arrays))), alias)
    acc = np.asarray(arrays[order[0]], f32).copy()
    with np.errstate(all="ignore"):
        for z in order[1:]:
            acc = acc * np.asarray(arrays[z], f32)
    return acc


def ewprod_back(g, a_list, b):
    """h_i = g * b / a_i (b / a_i without g), each operation rounded"""
    with np.errstate(all="ignore"):
        num = np.asarray(b, f32) if g is None else np.asarray(g, f32) * np.asarray(b, f32)
        return [num / np.asarray(a, f32) for a in a_list]
