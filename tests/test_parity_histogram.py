"""HISTOGRAM and EWPROD on the GPU against the restatement of tests/histogram_ref.py (itself pinned to CPU_REF by
tests/test_histogram_cpu.py) and against CPU_REF live where oracle/_ref is present.  Counts and min / max bits must be equal; the sum
and sum of squares may differ from the element-order double sums only where the stored float rounds the other way (one float step).
Cases: every type x dtype, sizes from 1 element to 2^26, ResNet-50's flat parameter buffer, all values in one bin, bins and bounds
beyond the shared-memory limit, packed / misaligned / strided views, repeatability, refusals, and EWPROD in place."""
import numpy as np
import pytest

from ccv_b200 import abi
from tests import histogram_ref as R
from tests.util import pack16, unpack16

pytestmark = pytest.mark.gpu

f32 = np.float32
KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
TYPES = {"even": (R.EVEN, 50, -3.0, 4.0, 0.0), "log": (R.LOG, 0, 1e-12, 1e20, 1.1), "log2": (R.LOG, 0, 0.01, 100.0, 1.3), "bins": (R.BINS, 0, 0, 0, 0)}
BOUNDS = np.sort(np.random.RandomState(3).uniform(-3, 3, 100)).astype(f32)
INVALID = abi.CCV_NNC_EXEC_INVALID
RESNET50_PARAMS = 25557032


def _cmd(nnc, p):
    t, bins, lo, hi, rate = p
    if t == R.EVEN:
        return nnc.CMD_HISTOGRAM_EVEN(int(bins), lo, hi)
    if t == R.LOG:
        return nnc.CMD_HISTOGRAM_LOG(lo, hi, rate)
    return nnc.CMD_HISTOGRAM_BINS()


def _held(x, kind):
    """the fp32 values a tensor of this kind holds, and its host array"""
    if kind == abi.CCV_32F:
        return np.asarray(x, f32), np.asarray(x, f32)
    h = pack16(x, kind)
    return unpack16(h, kind), h


class _Run(object):
    def __init__(self, nnc):
        self.nnc, self.owned = nnc, []

    def tensor(self, host, kind, off=0):
        """a GPU tensor of host's elements (flat) at element offset `off` of a larger allocation"""
        n = host.size
        big = self.nnc.gpu_tensor([n + off + 8], abi.CCV_TENSOR_FORMAT_NHWC, kind)
        buf = np.zeros(n + off + 8, host.dtype)
        buf[off:off + n] = host.ravel()
        big.upload(buf)
        self.owned.append(big)
        if off == 0:
            t = self.nnc.gpu_tensor([n], abi.CCV_TENSOR_FORMAT_NHWC, kind, ptr=big.data_ptr)
        else:
            t = self.nnc.gpu_tensor([n], abi.CCV_TENSOR_FORMAT_NHWC, kind, ptr=big.data_ptr + off * abi.DTYPE_SIZE[kind])
        self.owned.append(t)
        return t

    def out(self, n, kind, fill):
        t = self.nnc.gpu_tensor([n], abi.CCV_TENSOR_FORMAT_NHWC, kind)
        t.upload(np.full(n, fill, np.int32 if kind == abi.CCV_32S else f32))
        self.owned.append(t)
        return t

    def free(self):
        for t in reversed(self.owned):
            t.free()
        self.owned = []


def _gpu(nnc, a, p, bounds=None, nb=None, with_s=True, extra=0):
    """run HISTOGRAM on tensor a (already made by a _Run) -> (status, launches, b, s)"""
    r = _Run(nnc)
    try:
        need = R.bin_count(int(p[0]), int(p[1]), p[2], p[3], p[4], 0 if bounds is None else len(bounds))
        b = r.out(nb or need + extra, abi.CCV_32S, 7)
        s = r.out(4, abi.CCV_32F, -5.0) if with_s else None
        ins = [a] + ([r.tensor(np.asarray(bounds, f32), abi.CCV_32F)] if bounds is not None else [])
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(_cmd(nnc, p), None, 0, ins, [b] + ([s] if with_s else []))
        launches = nnc.launch_count() - l0
        return st, launches, b.download(), (s.download() if with_s else None)
    finally:
        r.free()


def _check(nnc, x, kind, p, bounds=None, off=0, what=""):
    held, host = _held(x, kind)
    if int(p[0]) == R.BINS and bounds is None:
        bounds = BOUNDS
    r = _Run(nnc)
    try:
        a = r.tensor(host, kind, off)
        st, launches, b, s = _gpu(nnc, a, p, bounds)
        st2, _, b2, s2 = _gpu(nnc, a, p, bounds)
    finally:
        r.free()
    assert st == 0 and launches == 3, (what, st, launches, nnc.lib().ccv_nnc_sm100_last_error())
    assert st2 == 0 and np.array_equal(b, b2) and np.array_equal(s.view(np.uint32), s2.view(np.uint32)), what + ": two runs differ"
    _compare(held, p, bounds, b, s, what, kind)
    return b, s


def _compare(held, p, bounds, b, s, what, kind=abi.CCV_32F):
    """fp16 NaNs widen to the device's canonical NaN, so of a NaN min / max from an fp16 tensor only its NaN-ness is compared"""
    wb, ws = R.histogram(held, int(p[0]), int(p[1]), p[2], p[3], p[4], bounds, nb=len(b))
    assert np.array_equal(b, wb), "%s: counts differ in %d bins" % (what, int((b != wb).sum()))
    if kind == abi.CCV_16F and np.isnan(ws[0]):
        assert np.isnan(s[:2]).all(), (what, s[:2], ws[:2])
    else:
        assert np.array_equal(s[:2].view(np.uint32), ws[:2].view(np.uint32)), (what, s[:2], ws[:2])
    for i in (2, 3):
        g, w = float(s[i]), float(ws[i])
        assert g == w or (np.isnan(g) and np.isnan(w)) or abs(g - w) <= np.spacing(np.float32(abs(w))), (what, i, g, w)


def _data(n, seed, kind="normal"):
    r = np.random.default_rng(seed)
    if kind == "normal":
        return (r.standard_normal(n, dtype=np.float32) * f32(2))
    if kind == "wide":
        return (r.standard_normal(n) * 10.0 ** r.uniform(-10, 10, n)).astype(f32)
    x = r.standard_normal(n, dtype=np.float32)
    x[r.integers(0, n, max(1, n // 1000))] = np.nan
    return x


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("typ", list(TYPES))
@pytest.mark.parametrize("n", [1, 7, 4099, 1 << 20])
def test_every_type_and_dtype(gpu, kind, typ, n):
    for dist in ("normal", "wide", "nan"):
        x = _data(n, n + len(typ) + len(kind), dist)
        _check(gpu, x, KINDS[kind], TYPES[typ], what="%s %s %d %s" % (kind, typ, n, dist))


@pytest.mark.parametrize("kind", list(KINDS))
def test_misaligned_bases(gpu, kind):
    x = _data(100003, 5, "nan")
    for off in (1, 3, 5):
        for typ in ("even", "log2", "bins"):
            _check(gpu, x, KINDS[kind], TYPES[typ], off=off, what="off %d %s" % (off, typ))


@pytest.mark.parametrize("kind", list(KINDS))
def test_strided_views(gpu, kind):
    """views of rank 2..5 of a larger tensor, walked in the view's row-major order"""
    k = KINDS[kind]
    base = _data(6 * 7 * 9 * 11, 9, "nan").reshape(6, 7, 9, 11)
    held, host = _held(base, k)
    for nd, (dims, ofs) in {2: ([5, 9], [1, 2]), 3: ([4, 5, 8], [1, 1, 1]), 4: ([5, 6, 7, 10], [1, 0, 2, 1]), 5: ([2, 3, 4, 5, 7], [0, 0, 1, 0, 1])}.items():
        shape = base.shape if nd == 4 else ((6, 7, 99) if nd == 3 else ((42, 99) if nd == 2 else (2, 3, 7, 9, 11)))
        h = held.reshape(shape)
        strides = [int(np.prod(shape[i + 1:])) for i in range(nd)]
        sl = tuple(slice(o, o + d) for o, d in zip(ofs, dims))
        want = np.ascontiguousarray(h[sl]).ravel()
        r = _Run(gpu)
        try:
            t = gpu.gpu_tensor(list(shape), abi.CCV_TENSOR_FORMAT_NHWC, k)
            t.upload(host.reshape(shape))
            r.owned.append(t)
            v = gpu.tensor_view_new(t, dims + [0] * (12 - nd), ofs + [0] * (12 - nd), strides + [0] * (12 - nd))
            r.owned.append(v)
            for typ in ("even", "log2", "bins"):
                p = TYPES[typ]
                bounds = BOUNDS if typ == "bins" else None
                st, launches, b, s = _gpu(gpu, v, p, bounds)
                assert st == 0, gpu.lib().ccv_nnc_sm100_last_error()
                _compare(want, p, bounds, b, s, "view %d-d %s" % (nd, typ), k)
        finally:
            r.free()


def test_large_and_resnet50_parameters(gpu):
    x = (np.random.default_rng(1).standard_normal(RESNET50_PARAMS, dtype=np.float32) * f32(0.05))
    for typ in ("even", "log", "bins"):
        _check(gpu, x, abi.CCV_32F, TYPES[typ], what="resnet50 " + typ)
    x = _data(1 << 26, 2, "wide")
    _check(gpu, x, abi.CCV_32F, TYPES["log"], what="2^26 log")
    _check(gpu, x, abi.CCV_16BF, TYPES["even"], what="2^26 bf16 even")


def test_one_bin_and_bins_beyond_shared_memory(gpu):
    x = np.full(1 << 22, 0.5, f32)
    for typ in ("even", "log", "bins"):
        _check(gpu, x, abi.CCV_32F, TYPES[typ], what="one bin " + typ)
    y = _data(1 << 20, 4, "nan")
    _check(gpu, y, abi.CCV_32F, (R.EVEN, 30000, -4.0, 4.0, 0.0), what="30000 even bins")
    _check(gpu, y, abi.CCV_16F, (R.BINS, 0, 0, 0, 0), bounds=np.sort(np.random.RandomState(8).uniform(-4, 4, 20000)).astype(f32), what="20000 bounds")
    _check(gpu, y, abi.CCV_32F, (R.BINS, 0, 0, 0, 0), bounds=np.sort(np.random.RandomState(8).uniform(-4, 4, 9000)).astype(f32), what="9000 bounds")
    _check(gpu, y, abi.CCV_32F, (R.LOG, 0, 1e-3, 1e3, 1.0005), what="log beyond shared memory")


def test_bins_at_the_shared_memory_limit(gpu):
    """counts plus bounds of exactly 12 032 words stay in shared memory; one word more goes to global memory.  Both launch and agree."""
    y = _data(1 << 18, 14, "nan")
    rs = np.random.RandomState(9)
    _check(gpu, y, abi.CCV_32F, (R.EVEN, 12029, -4.0, 4.0, 0.0), what="EVEN 12029 bins (12 032 shared counts)")
    _check(gpu, y, abi.CCV_32F, (R.EVEN, 12030, -4.0, 4.0, 0.0), what="EVEN 12030 bins (global counts)")
    _check(gpu, y, abi.CCV_16BF, (R.EVEN, 12200, -4.0, 4.0, 0.0), what="EVEN 12200 bins")
    _check(gpu, y, abi.CCV_32F, (R.BINS, 0, 0, 0, 0), bounds=np.sort(rs.uniform(-4, 4, 6015)).astype(f32), what="BINS 6015 (both shared)")
    _check(gpu, y, abi.CCV_32F, (R.BINS, 0, 0, 0, 0), bounds=np.sort(rs.uniform(-4, 4, 6100)).astype(f32), what="BINS 6100")
    _check(gpu, y, abi.CCV_16F, (R.BINS, 0, 0, 0, 0), bounds=np.sort(rs.uniform(-4, 4, 12030)).astype(f32), what="BINS 12030")
    # LOG with u = 6015 (12 032 counts, shared), u = 6016 (12 034, global) and u = 6094
    for rate, u in ((1.0022995471954346, 6015), (1.002299189567566, 6016), (1.00227, 6094)):
        assert R.log_params(1e-3, 1e3, rate)[1] == u
        _check(gpu, y * f32(100), abi.CCV_32F, (R.LOG, 0, 1e-3, 1e3, rate), what="LOG u = %d" % u)


def test_log_counts_equal_bins_counts_with_the_log_edges(gpu):
    """the reference's histogram.tests.c: with the LOG edges (1e-12 * 1.1^i, rounded to float, mirrored) as BINS bounds, the two
    histograms of 3000 x 2000 uniform values in (-1000, 1000] plus specials agree within its tolerance, and their statistics are equal"""
    h = np.zeros(774 * 2, f32)
    v, i = 1e-12, 0
    while v < 1e20:
        h[i + 774], h[774 - i - 1] = v, -v
        i, v = i + 1, v * 1.1
    a = (np.random.default_rng(1).random(3000 * 2000) * 2000 - 1000).astype(f32)
    a[:8] = [np.nan, -np.finfo(f32).max, np.finfo(f32).max, 0, 1e-20, -1e-20, 1e20 - 1e18, -1e20 + 1e18]
    bl, sl = _check(gpu, a, abi.CCV_32F, TYPES["log"], what="identity LOG")
    bb, sb = _check(gpu, a, abi.CCV_32F, (R.BINS, 0, 0, 0, 0), bounds=h, what="identity BINS")
    assert len(bl) == len(bb) == 775 * 2
    tot = bb.astype(np.int64) + bl
    diff = np.abs(bl.astype(np.int64) - bb)
    tol = np.where(tot > 10, diff / np.maximum(tot, 1), diff)
    assert (tol < 0.1).all(), np.flatnonzero(tol >= 0.1)
    for b in (bl, bb):
        assert (b[0], b[774 * 2], b[775 * 2 - 1], b[774 * 2 - 1], b[1], b[774]) == (1, 1, 1, 1, 1, 3)
    assert sl[0] == -np.finfo(f32).max and sl[1] == np.finfo(f32).max and np.isnan(sl[2:]).all()
    assert np.array_equal(sl.view(np.uint32), sb.view(np.uint32))


def test_captured_graph_gives_the_same_bits(gpu):
    """HISTOGRAM (LOG with statistics, BINS, EVEN without) and EWPROD forward / backward as nodes of a graph: run eagerly, through
    the graph, and as a captured CUDA graph replayed, with the same bits"""
    nnc = gpu
    x = _data(300001, 15, "nan")
    ops = [np.random.default_rng(20 + i).uniform(-1.5, 1.5, 4099).astype(f32) for i in range(3)]
    up = lambda a: nnc.gpu_tensor([a.size]).upload(a)
    ta, tbounds = up(x), up(BOUNDS)
    tops = [up(o) for o in ops]
    tc, tg = up(np.zeros(4099, f32)), up(ops[0] * f32(0.5))
    th = [up(np.zeros(4099, f32)) for _ in range(3)]
    nl, nbins = R.bin_count(R.LOG, 0, 0.01, 100.0, 1.3), len(BOUNDS) + 2
    bl, sl = nnc.gpu_tensor([nl], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_32S), nnc.gpu_tensor([4])
    bb, be = nnc.gpu_tensor([nbins], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_32S), nnc.gpu_tensor([53], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_32S)
    nodes = [(_cmd(nnc, TYPES["log2"]), [ta], [bl, sl]), (nnc.CMD_HISTOGRAM_BINS(), [ta, tbounds], [bb]),
             (_cmd(nnc, TYPES["even"]), [ta], [be]), (nnc.CMD_EWPROD_FORWARD(), tops, [tc]),
             (nnc.CMD_EWPROD_BACKWARD(), [tg] + tops + [tc], th)]
    outs = [bl, sl, bb, be, tc] + th

    def clear():
        for t in outs:
            t.upload(np.zeros(t.count, np.int32 if t.params.datatype == abi.CCV_32S else f32))
    owned = [ta, tbounds, tg] + tops + outs
    try:
        for cmd, ins, os_ in nodes:
            assert nnc.cmd_exec(cmd, None, 0, ins, os_) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        eager = [t.download().view(np.uint32).copy() for t in outs]
        wb, ws = R.histogram(x, R.LOG, 0, 0.01, 100.0, 1.3)
        assert np.array_equal(eager[0].view(np.int32), wb)
        stream = nnc.Stream(0)
        graph = nnc.Graph()
        for cmd, ins, os_ in nodes:
            graph.exec_new(cmd, None, 0, ins, os_)
        clear()
        assert graph.run(stream) == 0
        stream.wait()
        assert all(np.array_equal(t.download().view(np.uint32), e) for t, e in zip(outs, eager))
        cid = graph.capture(stream)
        for _ in range(2):
            clear()
            assert graph.replay(cid, stream) == 0
            stream.wait()
            for k, (t, e) in enumerate(zip(outs, eager)):
                assert np.array_equal(t.download().view(np.uint32), e), k
        graph.free()
        stream.free()
    finally:
        for t in owned:
            t.free()


def test_edges_and_specials(gpu):
    log = TYPES["log2"]
    _, _, rate = log[2], log[3], log[4]
    k = np.arange(-2, 40).astype(f32)
    edges = (f32(0.01) * f32(rate) ** k).astype(f32)
    x = np.concatenate([edges, -edges, np.nextafter(edges, f32(0)), np.nextafter(edges, f32(1e30)), [0.0, -0.0, 1e-45, np.inf, -np.inf, np.nan, 5.0]]).astype(f32)
    _check(gpu, x, abi.CCV_32F, log, what="log edges")
    ev = TYPES["even"]
    e = (f32(-3.0) + np.arange(51, dtype=f32) * f32(7.0 / 50)).astype(f32)
    _check(gpu, np.concatenate([e, np.nextafter(e, f32(-9)), np.nextafter(e, f32(9))]), abi.CCV_32F, ev, what="even edges")
    _check(gpu, np.array([0.0, -0.0, 1.0, 0.0, -0.0, -1.0, 1.0, -1.0, 0.0, -0.0], f32), abi.CCV_32F, ev, what="zero ties")
    _check(gpu, np.array([3e38, -3e38, 1e-45, np.inf, -np.inf, np.nan], f32), abi.CCV_32F, (R.EVEN, 5, -3e38, 3e38, 0.0), what="even overflow")
    _check(gpu, np.array([1e19, 2e19, -3e19, 1.0], f32), abi.CCV_32F, ev, what="inf sum of squares")
    for bounds in (np.array([-1, -1, 0, 0, 1, 1, 1], f32), np.random.RandomState(2).uniform(-3, 3, 21).astype(f32), np.array([-1, 0, np.nan, 1], f32)):
        _check(gpu, _data(5000, 6, "nan"), abi.CCV_32F, TYPES["bins"], bounds=bounds, what="odd bounds")
    for pos in (0, 4999, 2500):
        x = _data(5000, 7)
        x[pos] = np.nan
        _check(gpu, x, abi.CCV_32F, ev, what="nan at %d" % pos)


def test_without_statistics_and_long_log_b(gpu):
    x = _data(10000, 10, "nan")
    r = _Run(gpu)
    try:
        a = r.tensor(x, abi.CCV_32F)
        st, launches, b, _ = _gpu(gpu, a, TYPES["log2"], with_s=False, extra=6)
        assert st == 0 and launches == 2
        wb, _ = R.histogram(x, R.LOG, 0, 0.01, 100.0, 1.3, nb=len(b))
        assert np.array_equal(b, wb) and b[-6:].tolist() == [0] * 6
    finally:
        r.free()


def test_refusals_leave_outputs_untouched(gpu):
    x = _data(1000, 12)
    r = _Run(gpu)
    try:
        a = r.tensor(x, abi.CCV_32F)
        ai = r.tensor(np.arange(1000, dtype=np.int32), abi.CCV_32S)
        ev = TYPES["even"]
        cases = [
            (ai, ev, None, 53),                       # int32 a
            (a, (R.EVEN, 50, 4.0, 4.0, 0.0), None, 53),  # max <= min
            (a, (R.EVEN, 0, -1.0, 1.0, 0.0), None, 3),   # bins < 1
            (a, ev, None, 52),                        # short b
            (a, ev, None, 54),                        # long EVEN b
            (a, (R.LOG, 0, 0.0, 1.0, 1.1), None, 8),     # min <= 0
            (a, (R.LOG, 0, 1.0, 10.0, 1.0), None, 8),    # rate <= 1
            (a, (R.LOG, 0, 0.01, 100.0, 1.3), None, 10),  # short LOG b
            (a, TYPES["bins"], None, 102),            # BINS without bounds
        ]
        for i, (t, p, bounds, nb) in enumerate(cases):
            b = r.out(nb, abi.CCV_32S, 7)
            s = r.out(4, abi.CCV_32F, -5.0)
            l0 = gpu.launch_count()
            assert gpu.cmd_exec(_cmd(gpu, p), None, 0, [t], [b, s]) == INVALID, i
            assert gpu.launch_count() == l0, i
            assert (b.download() == 7).all() and (s.download() == -5.0).all(), i
        b = r.out(53, abi.CCV_32S, 7)
        s3 = r.out(3, abi.CCV_32F, -5.0)
        assert gpu.cmd_exec(_cmd(gpu, ev), None, 0, [a], [b, s3]) == INVALID and (b.download() == 7).all()
        assert gpu.cmd_exec(gpu.CMD_HISTOGRAM_EVEN(50, -3.0, 4.0), None, 0, [a], [b]) == 0
        back = gpu.CMD_HISTOGRAM_EVEN(50, -3.0, 4.0)
        back.cmd = abi.CCV_NNC_HISTOGRAM_BACKWARD
        assert gpu.cmd_exec(back, None, 0, [a], [b]) == INVALID
    finally:
        r.free()


def test_matches_cpu_ref_live(gpu, ref):
    from tests.golden.make_histogram_golden import cpu_histogram
    from tests.test_histogram_cpu import host_logf_moves
    for typ in ("even", "log", "log2", "bins"):
        p = TYPES[typ]
        x = _data(200003, 13, "nan") * f32(3)
        bounds = BOUNDS if typ == "bins" else None
        _, cb, cs = cpu_histogram(x, p, bounds)
        gb, gs = _check(gpu, x, abi.CCV_32F, p, bounds, what="live " + typ)
        moved = int(host_logf_moves(x, p).sum())
        assert np.abs(gb.astype(np.int64) - cb).sum() <= 2 * moved, typ
        assert np.array_equal(gs[:2].view(np.uint32), cs[:2].view(np.uint32)), typ


# ---- EWPROD ------------------------------------------------------------------------------------------------------------------------
def _ewprod_gpu(nnc, ops, kind, alias=None, n_out=None):
    r = _Run(nnc)
    try:
        ts = [r.tensor(_held(o, kind)[1], kind, 0) for o in ops]
        c = ts[alias] if alias is not None else r.tensor(_held(np.zeros_like(ops[0]), kind)[1], kind)
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(nnc.CMD_EWPROD_FORWARD(), None, 0, ts, [c])
        out = c.download()
        return st, nnc.launch_count() - l0, (out if kind == abi.CCV_32F else unpack16(out, kind))
    finally:
        r.free()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("n", [1, 2, 3, 8, 9, 20])
def test_ewprod_forward_in_place_every_position(gpu, kind, n):
    k = KINDS[kind]
    if k != abi.CCV_32F and n > 8:
        st, _, _ = _ewprod_gpu(gpu, [_data(100, i) for i in range(n)], k)
        assert st == INVALID
        return
    ops = [np.random.default_rng(i).uniform(-1.5, 1.5, 10007).astype(f32) for i in range(n)]
    held = [_held(o, k)[0] for o in ops]
    for alias in [None] + list(range(n)):
        st, launches, got = _ewprod_gpu(gpu, ops, k, alias)
        assert st == 0, gpu.lib().ccv_nnc_sm100_last_error()
        want = R.ewprod(held, alias)
        if k != abi.CCV_32F:
            want = _held(want, k)[0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (kind, n, alias)


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("withg", [0, 1])
def test_ewprod_backward(gpu, kind, withg):
    k = KINDS[kind]
    rng = np.random.default_rng(withg)
    g, b = rng.uniform(-2, 2, 5003).astype(f32), rng.uniform(-2, 2, 5003).astype(f32)
    a = [rng.uniform(-2, 2, 5003).astype(f32) for _ in range(3)]
    a[1][:4] = 0
    hg, hb, ha = _held(g, k)[0], _held(b, k)[0], [_held(x, k)[0] for x in a]
    want = [x if k == abi.CCV_32F else _held(x, k)[0] for x in R.ewprod_back(hg if withg else None, ha, hb)]
    for inplace in (False, True):
        r = _Run(gpu)
        try:
            tg = r.tensor(_held(g, k)[1], k) if withg else None
            ta = [r.tensor(_held(x, k)[1], k) for x in a]
            tb = r.tensor(_held(b, k)[1], k)
            th = [ta[2], tb, ta[0]] if inplace else [r.tensor(_held(np.zeros_like(x), k)[1], k) for x in a]
            l0 = gpu.launch_count()
            assert gpu.cmd_exec(gpu.CMD_EWPROD_BACKWARD(), None, 0, [tg] + ta + [tb], th) == 0
            assert gpu.launch_count() - l0 == 1
            got = [t.download() for t in th]
            got = [x if k == abi.CCV_32F else unpack16(x, k) for x in got]
        finally:
            r.free()
        for z in range(3):
            assert np.array_equal(got[z].view(np.uint32), want[z].view(np.uint32)), (kind, withg, inplace, z)


def test_ewprod_matches_cpu_ref_live(gpu, ref):
    from tests.util import ref_exec
    ops = [np.random.default_rng(40 + i).uniform(-1.5, 1.5, 4099).astype(f32) for i in range(11)]
    c = np.zeros(4099, f32)
    st, (c,) = ref_exec(ref, gpu.CMD_EWPROD_FORWARD(backend=abi.CCV_NNC_BACKEND_CPU_REF), None, 0, [o.copy() for o in ops], [c])
    assert st == 0
    st, _, got = _ewprod_gpu(gpu, ops, abi.CCV_32F)
    assert st == 0 and np.array_equal(got.view(np.uint32), c.view(np.uint32))
