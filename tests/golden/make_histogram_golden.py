"""Writes tests/golden/cpuref_histogram.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on HISTOGRAM_FORWARD
and EWPROD forward / backward, so that tests/test_histogram_cpu.py pins the restatement of tests/histogram_ref.py to CPU_REF without the
reference present.

HISTOGRAM cases (key h_<name>_*: x the view's values in row-major order, p = (type, bins, min, max, rate), bounds, b counts, s stats):
  - all three types on normal, wide-range and uniform data;
  - values exactly at EVEN edges (min + k (max - min) / bins and their neighbours) and at min rate^k for LOG;
  - NaN first, last and in the middle, and NaN-only tensors;
  - +-0 ties, +-Inf and subnormals;
  - unsorted, repeated and NaN BINS bounds;
  - views of rank 1 to 6 (CPU_REF's view recursion);
  - a LOG b longer than the rule's count (the tail stays zero).
EWPROD cases (key e_*): forward with 1, 2, 3 and 9 operands, in place on each operand position; backward with and without g.

  python tests/golden/make_histogram_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import abi, nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests import histogram_ref as R  # noqa: E402

f32 = np.float32
NAN, INF = f32(np.nan), f32(np.inf)


def cmd_of(p):
    t, bins, lo, hi, rate = p
    if t == R.EVEN:
        return nnc.CMD_HISTOGRAM_EVEN(int(bins), lo, hi, backend=abi.CCV_NNC_BACKEND_CPU_REF)
    if t == R.LOG:
        return nnc.CMD_HISTOGRAM_LOG(lo, hi, rate, backend=abi.CCV_NNC_BACKEND_CPU_REF)
    return nnc.CMD_HISTOGRAM_BINS(backend=abi.CCV_NNC_BACKEND_CPU_REF)


def cpu_histogram(base, p, bounds=None, view=None, extra=0):
    """CPU_REF on base (float32) or on a view (dims, ofs, stride) of it -> (row-major values, b, s)"""
    t = int(p[0])
    nb = R.bin_count(t, int(p[1]), p[2], p[3], p[4], 0 if bounds is None else len(bounds)) + extra
    b = np.full(nb, 7, np.int32)  # CPU_REF zeroes b first
    s = np.full(4, -1, f32)
    ta = ref.RefTensor(base)
    a = ta if view is None else ta.view(*view)
    ins = [a] + ([ref.RefTensor(bounds)] if bounds is not None else [])
    outs = [ref.RefTensor(b), ref.RefTensor(s)]
    st = ref.cmd_exec(cmd_of(p), None, 0, ins, outs)
    assert st == 0, st
    for x in ins[1:] + outs + ([a] if view is not None else []) + [ta]:
        x.free()
    if view is None:
        vals = base.ravel()
    else:
        dims, ofs, stride = view
        nd = sum(1 for d in dims if d > 0)
        dims = dims[:nd]
        off = sum(o * s_ for o, s_ in zip(ofs[:nd], stride[:nd]))
        vals = np.lib.stride_tricks.as_strided(base.ravel()[off:], dims, [s_ * 4 for s_ in stride[:nd]]).ravel().copy()
    return vals, b, s


def cases():
    r = np.random.RandomState(11)
    out = {}

    def add(name, base, p, bounds=None, view=None, extra=0):
        vals, b, s = cpu_histogram(np.ascontiguousarray(base, f32), p, bounds, view, extra)
        out["h_%s_x" % name], out["h_%s_p" % name], out["h_%s_b" % name], out["h_%s_s" % name] = vals, np.array(p, np.float64), b, s
        out["h_%s_bounds" % name] = np.zeros(0, f32) if bounds is None else bounds

    even = (R.EVEN, 10, -2.0, 3.0, 0.0)
    log = (R.LOG, 0, 1e-12, 1e20, 1.1)
    log2 = (R.LOG, 0, 0.5, 1000.0, 1.7)
    normal = r.standard_normal(5000).astype(f32) * f32(2)
    wide = (r.standard_normal(5000) * 10.0 ** r.uniform(-14, 22, 5000)).astype(f32)
    add("even_normal", normal, even)
    add("even_many", r.uniform(-5, 5, 20000).astype(f32), (R.EVEN, 1000, -4.0, 4.5, 0.0))
    add("even_odd_range", r.uniform(0, 1, 3000).astype(f32), (R.EVEN, 7, 0.1, 0.7, 0.0))
    edges = np.float32(-2.0) + np.arange(11, dtype=f32) * f32(0.5)
    add("even_edges", np.concatenate([edges, np.nextafter(edges, f32(-10)), np.nextafter(edges, f32(10))]), even)
    for bins, lo, hi in ((997, -1.1, 1.3), (300, -0.3, 0.9)):
        e = (f32(lo) + np.arange(bins + 1, dtype=f32) * f32((hi - lo) / bins)).astype(f32)
        add("even_edges_%d" % bins, np.concatenate([e, np.nextafter(e, f32(-9)), np.nextafter(e, f32(9))]), (R.EVEN, bins, lo, hi, 0.0))
    add("even_extreme", np.array([3e38, -3e38, 1e-45, -0.0, 0.0, INF, -INF, 2.9999998, -2.0, NAN], f32), (R.EVEN, 5, -3e38, 3e38, 0.0))
    add("even_tiny_range", np.array([1.0, 1.0000001, 1.0000002, 0.9999999], f32), (R.EVEN, 1000, 1.0, 1.0000002, 0.0))
    add("log_wide", wide, log)
    add("log_normal", normal, log2)
    k = np.arange(-2, 40)
    rates = (f32(0.5) * f32(1.7) ** k.astype(f32)).astype(f32)
    add("log_edges", np.concatenate([rates, -rates, np.nextafter(rates, f32(0)), np.nextafter(rates, f32(1e30))]), log2)
    rates = (np.float64(1e-12) * 1.1 ** np.arange(0, 770)).astype(f32)
    add("log_edges_default", np.concatenate([rates, -rates]), log)
    add("log_specials", np.array([0.0, -0.0, 1e-45, -1e-45, 1e-12, -1e-12, 9.999999e-13, 1e20, -1e20, INF, -INF, NAN, 3e38], f32), log)
    add("log_long_b", normal[:100], log2, extra=5)
    bounds = np.sort(r.uniform(-3, 3, 37)).astype(f32)
    add("bins_sorted", normal, (R.BINS, 0, 0, 0, 0), bounds)
    add("bins_at_bounds", np.concatenate([bounds, np.nextafter(bounds, f32(-9)), [NAN, INF, -INF]]).astype(f32), (R.BINS, 0, 0, 0, 0), bounds)
    add("bins_unsorted", normal, (R.BINS, 0, 0, 0, 0), r.uniform(-3, 3, 21).astype(f32))
    add("bins_repeated", normal, (R.BINS, 0, 0, 0, 0), np.array([-1, -1, -1, 0, 0, 1, 1, 1, 1, 2], f32))
    add("bins_nan_bound", normal, (R.BINS, 0, 0, 0, 0), np.array([-1, 0, NAN, 1, 2], f32))
    add("bins_one", normal, (R.BINS, 0, 0, 0, 0), np.array([0.25], f32))
    # NaN placement and the scans
    for where, idx in (("first", [0]), ("last", [-1]), ("middle", [2500]), ("several", [3, 1700, 4998])):
        x = normal.copy()
        x[idx] = NAN
        add("nan_" + where, x, even)
    add("nan_only", np.full(9, NAN, f32), even)
    add("zero_ties", np.array([0.0, -0.0, 1.0, 0.0, -0.0, -1.0, 1.0, -1.0, 0.0, -0.0], f32), even)
    add("zero_ties_after_nan", np.array([5.0, NAN, -0.0, 0.0, 0.0, -0.0], f32), even)
    add("inf", np.array([1.0, INF, -INF, 2.0, INF], f32), log)
    add("subnormal", np.array([1e-45, -1e-45, 1e-40, -3e-39, 0.0], f32), log)
    add("big_squares", np.array([1e19, 2e19, -3e19, 1.0], f32), even)
    add("single", np.array([0.5], f32), even)
    # views of rank 1..6 (CPU_REF's recursion; a row-major view of a larger buffer)
    base = r.standard_normal(8192).astype(f32)
    base[[17, 900]] = NAN
    for nd in range(1, 7):
        dims = [3, 2, 4, 3, 2, 5][:nd]
        stride, st = [], 1
        for d in reversed(dims):
            stride.insert(0, st * 1)
            st *= d + 1
        ofs = [1] * nd
        view = (dims + [0] * (12 - nd), ofs + [0] * (12 - nd), stride + [0] * (12 - nd))
        add("view%d_even" % nd, base, even, view=view)
        add("view%d_bins" % nd, base, (R.BINS, 0, 0, 0, 0), bounds, view=view)
        add("view%d_log" % nd, base, log2, view=view)
    return out


def ewprod_cases():
    r = np.random.RandomState(12)
    out = {}
    CPU = abi.CCV_NNC_BACKEND_CPU_REF
    for n in (1, 2, 3, 9):
        ops = [r.uniform(-2, 2, 1000).astype(f32) for _ in range(n)]
        for alias in [None] + list(range(n)):
            arrays = [o.copy() for o in ops]
            c = np.full(1000, 3, f32) if alias is None else arrays[alias]
            ts = [ref.RefTensor(a) for a in arrays]
            tc = ref.RefTensor(c) if alias is None else ts[alias]
            assert ref.cmd_exec(nnc.CMD_EWPROD_FORWARD(backend=CPU), None, 0, ts, [tc]) == 0
            for t in ts + ([tc] if alias is None else []):
                t.free()
            name = "e_f%d_%s" % (n, "none" if alias is None else alias)
            out[name + "_in"], out[name + "_c"] = np.stack(ops), c.copy()
    for withg in (0, 1):
        g, b = r.uniform(-2, 2, 1000).astype(f32), r.uniform(-2, 2, 1000).astype(f32)
        a = [r.uniform(-2, 2, 1000).astype(f32) for _ in range(3)]
        a[1][:5] = 0
        h = [np.zeros(1000, f32) for _ in range(3)]
        ins = [ref.RefTensor(g) if withg else None] + [ref.RefTensor(x) for x in a] + [ref.RefTensor(b)]
        outs = [ref.RefTensor(x) for x in h]
        assert ref.cmd_exec(nnc.CMD_EWPROD_BACKWARD(backend=CPU), None, 0, ins, outs) == 0
        for t in [x for x in ins if x is not None] + outs:
            t.free()
        name = "e_b%d" % withg
        out[name + "_g"], out[name + "_a"], out[name + "_b"], out[name + "_h"] = g, np.stack(a), b, np.stack(h)
    return out


def main():
    if not ref.available():
        sys.exit("oracle/_ref/libccv_ref.so is missing: build it first (make -C oracle)")
    z = cases()
    z.update(ewprod_cases())
    path = os.path.join(ROOT, "tests", "golden", "cpuref_histogram.npz")
    np.savez_compressed(path, **z)
    print("wrote %s (%d arrays)" % (path, len(z)))


if __name__ == "__main__":
    main()
