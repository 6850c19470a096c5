"""ROI_ALIGN and NMS (forward / backward) on CCV_NNC_BACKEND_GPU_SM100 against the oracles of tests/detection_ref.py, which are pinned to
the reference's CPU_REF by tests/golden/cpuref_detection.npz.

ROI_ALIGN's kernels round every product and sum on their own in CPU_REF's source order, and NMS only compares, so fp32 results are
compared bit for bit, and 16-bit ROI_ALIGN results bit for bit against the oracle on the widened inputs, rounded once."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi
from tests import detection_ref as R
from tests.util import NCHW, NHWC, pack16, round16, seeded

KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_detection.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DETECTION = ("ROI_ALIGN", "NMS")


def same(x, y):
    """bitwise equality (float32 / uint16 / int32)"""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    if x.dtype == np.float32:
        x = x.view(np.uint32)
    if y.dtype == np.float32:
        y = y.view(np.uint32)
    return x.shape == y.shape and np.array_equal(x, y)


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_detection.npz missing")
    return np.load(GOLDEN)


# ---- CPU: the oracles against CPU_REF's fixture, and against defects ----------------------------------------------------------
def test_roi_align_oracle_matches_cpu_ref_fixture():
    """bit for bit: CPU_REF is compiled with -ffast-math, but gcc keeps these loops' operations (SSE2, no FMA, no reassociation of the
    per-element sums across k), and the fixture shows it"""
    from tests.golden.make_detection_golden import ROI_CASES
    z = _golden()
    for name, shape, rows, (ph, pw) in ROI_CASES:
        a, b, g = z["roi_a_" + name], z["roi_b_" + name], z["roi_g_" + name]
        assert same(R.roi_align_forward(a, b, ph, pw), z["roi_c_" + name]), name
        assert same(R.roi_align_backward(g, b, shape), z["roi_h_" + name]), name


def test_nms_oracle_matches_cpu_ref_fixture():
    from tests.golden.make_detection_golden import NMS_THRESHOLDS
    z = _golden()
    for t in NMS_THRESHOLDS:
        b, c = R.nms_forward(z["nms_a"], t)
        assert same(b, z["nms_b_%g" % t]) and same(c, z["nms_c_%g" % t]), t
        assert same(R.nms_backward(z["nms_g_%g" % t], c), z["nms_h_%g" % t]), t
    # the fixture holds chained suppression (row 2 survives because row 1 is suppressed), and thresholds 0 and 1 differ from 0.5
    assert (z["nms_c_0.5"] >= 0).sum(1).tolist() != (z["nms_c_0"] >= 0).sum(1).tolist()
    assert ((z["nms_c_1"] >= 0).sum(1) > (z["nms_c_0.5"] >= 0).sum(1)).all()


def test_oracles_reject_plausible_kernel_defects():
    """a swapped corner, a clamp off by one and a forward without CPU_REF's row shift all disagree with CPU_REF's fixture"""
    from tests.golden.make_detection_golden import ROI_CASES
    z = _golden()
    name, shape, rows, (ph, pw) = ROI_CASES[0]
    a, b, want = z["roi_a_" + name], z["roi_b_" + name], z["roi_c_" + name]
    orig = R._corner_weights
    try:
        R._corner_weights = lambda ry, rx: (lambda c: (c[1], c[0], c[2], c[3]))(orig(ry, rx))
        assert not same(R.roi_align_forward(a, b, ph, pw), want)
    finally:
        R._corner_weights = orig
    orig_axis = R._axis
    try:
        def off_by_one(v, vs, size, pool):
            r = orig_axis(v, vs, size, pool)
            return None if r is None else (r[0], r[1], np.clip(r[2], 0, size - 2), r[3], r[4])
        R._axis = off_by_one
        assert not same(R.roi_align_forward(a, b, ph, pw), want)
    finally:
        R._axis = orig_axis
    # no row shift: an oracle that writes bin row i to output row i disagrees on the ROI that starts above the map
    name1, shape1, rows1, (ph1, pw1) = ROI_CASES[3]
    a1, b1, want1 = z["roi_a_" + name1], z["roi_b_" + name1], z["roi_c_" + name1]
    assert R._range(R._coeffs(b1[0], shape1[0], shape1[1], ph1, pw1)[2])[0] > 0
    orig_row = R._out_row
    try:
        R._out_row = lambda i, start_h: i
        assert not same(R.roi_align_forward(a1, b1, ph1, pw1), want1)
    finally:
        R._out_row = orig_row
    assert same(R.roi_align_forward(a1, b1, ph1, pw1), want1)


def test_nms_oracle_rejects_an_unstable_sort():
    """CPU_REF's fixture has no ties (its quicksort is unstable on them), so ties are checked against a hand-derived result: rows 0 and 4
    tie at 0.9 and overlap (IoU 0.6), so the first in input order is kept and suppresses the other; rows 1, 3 tie at 0.5 apart from all.
    The oracle gives that result, and the same oracle with tied rows taken in another order does not."""
    t = np.array([[0.9, 0, 0, 10, 10], [0.5, 40, 40, 2, 2], [0.25, 80, 80, 2, 2], [0.5, 60, 60, 2, 2], [0.9, 2.5, 0, 10, 10]], np.float32)
    want_c = [0, 1, 3, 2, -1]
    b, c = R.nms_forward(t, 0.5)
    assert c.tolist() == want_c and same(b[:4], t[want_c[:4]])
    orig = R._order
    try:
        # descending by key, ties in reverse input order (what an unstable sort may give)
        R._order = lambda s: np.lexsort((-np.arange(len(s)), -R.score_key(s).astype(np.int64)))
        _, c2 = R.nms_forward(t, 0.5)
        assert c2.tolist() != want_c
    finally:
        R._order = orig


def test_forward_sums_before_scaling():
    """the forward multiplies the bin's sum by inv once; scaling each term instead gives other bits on the fixture"""
    from tests.golden.make_detection_golden import ROI_CASES
    z = _golden()
    name, shape, rows, (ph, pw) = ROI_CASES[0]
    a, b, want = z["roi_a_" + name], z["roi_b_" + name], z["roi_c_" + name]
    H, W, Cc = a.shape
    alt = np.zeros_like(want)
    for n in range(len(b)):
        co = R._coeffs(b[n], H, W, ph, pw)
        if co is None:
            continue
        (bh, iy0, iy1, ry, ly), (bw, ix0, ix1, rx, lx), cy, cx = co
        sh, eh = R._range(cy)
        sw, ew = R._range(cx)
        for i in range(sh, eh):
            for j in range(sw, ew):
                inv = np.float32(1.0 / float(int(cy[i]) * int(cx[j])))
                acc = np.zeros(Cc, np.float32)
                for y in [y for y in range(i * bh, (i + 1) * bh) if ly[y]]:
                    for x in [x for x in range(j * bw, (j + 1) * bw) if lx[x]]:
                        c00, c01, c10, c11 = R._corner_weights(ry[y], rx[x])
                        s = a[iy0[y], ix0[x]] * c00 + a[iy0[y], ix1[x]] * c01 + a[iy1[y], ix0[x]] * c10 + a[iy1[y], ix1[x]] * c11
                        acc = acc + s * inv
                alt[n, i - sh, j] = acc
    assert not same(alt, want)


def test_nms_arm_sits_at_the_reference_offset():
    """iou_threshold at byte 48 of ccv_nnc_cmd_param_t (after size.dim[12], lib/nnc/ccv_nnc.h:249-251); the block stays 120 bytes"""
    assert abi.CmdParam.u.offset + abi._CmdUnion.nms.offset + abi._Nms.iou_threshold.offset == 48
    assert C.sizeof(abi.CmdParam) == 120
    from ccv_b200 import nnc
    c = nnc.CMD_NMS_FORWARD(0.375)
    assert c.cmd == abi.CCV_NNC_NMS_FORWARD and c.info.nms.iou_threshold == 0.375
    r = nnc.CMD_ROI_ALIGN_BACKWARD(7, 5)
    assert r.cmd == abi.CCV_NNC_ROI_ALIGN_BACKWARD and list(r.info.size.dim[:4]) == [7, 5, 1, 0]


def _lists():
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    first = re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_COMMANDS(X)"):header.index("#define CCV_SM100_DECLARE_REGISTER")])
    second = re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_DETECTION_COMMANDS(X)"):header.index("CCV_NNC_SM100_DETECTION_COMMANDS(CCV_SM100_DECLARE_REGISTER)")])
    return first, second


def test_both_registration_lists_hold_122_distinct_commands():
    first, second = _lists()
    assert len(first) == 118 and len(second) == 4
    assert len(set(first + second)) == 122
    assert sorted(second) == sorted("CCV_NNC_%s_%s" % (n, d) for n in DETECTION for d in ("FORWARD", "BACKWARD"))
    inc = open(os.path.join(ROOT, "integration", "ccv_nnc_cmd_sm100_init.inc")).read()
    for c in second:
        assert inc.count("_register_command_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % c) == 2, c


class _Registry(C.Structure):
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


def test_every_new_symbol_is_exported_and_fills_its_record():
    from ccv_b200 import nnc
    lib = nnc.lib()
    for name in DETECTION:
        for d in ("FORWARD", "BACKWARD"):
            fn = getattr(lib, "_register_command_CCV_NNC_%s_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % (name, d))
            r = _Registry()
            fn(C.byref(r))
            assert r.exec and r.tensor_memory == abi.CCV_TENSOR_GPU_MEMORY and r.algorithms == 1, (name, d)
            assert r.tensor_formats & abi.CCV_TENSOR_FORMAT_NHWC and r.tensor_formats & abi.CCV_TENSOR_FORMAT_NCHW
            assert r.tensor_datatypes & abi.CCV_32F
            assert lib.ccv_nnc_cmd_ok(getattr(abi, "CCV_NNC_%s_%s" % (name, d)), abi.CCV_NNC_BACKEND_GPU_SM100) == 1


@pytest.mark.ref
def test_constructors_run_cpu_ref_to_the_fixture(ref):
    from ccv_b200 import nnc
    from tests.golden.make_detection_golden import NMS_THRESHOLDS, ROI_CASES
    from tests.util import ref_exec
    z = _golden()
    for name, shape, rows, (ph, pw) in ROI_CASES:
        want = z["roi_c_" + name]
        st, (got,) = ref_exec(ref, nnc.CMD_ROI_ALIGN_FORWARD(ph, pw), None, 0, [z["roi_a_" + name], z["roi_b_" + name]], [np.zeros_like(want)])
        assert st == 0 and same(got, want), name
    for t in NMS_THRESHOLDS:
        st, (b, c) = ref_exec(ref, nnc.CMD_NMS_FORWARD(t), None, 0, [z["nms_a"]], [np.zeros_like(z["nms_a"]), np.zeros(z["nms_a"].shape[:2], np.int32)])
        assert st == 0 and same(b, z["nms_b_%g" % t]) and same(c, z["nms_c_%g" % t]), t


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
class _Dev(object):
    """GPU tensors; everything made here is freed by free()"""

    def __init__(self, nnc):
        self.nnc, self.owned = nnc, []

    def up(self, x, kname="fp32", fmt=NHWC):
        """x: float32 values (rounded to kname when 16-bit) or int32"""
        if x.dtype == np.int32:
            t = self.nnc.gpu_tensor(list(x.shape), fmt, abi.CCV_32S)
            t.upload(x)
        else:
            t = self.nnc.gpu_tensor(list(x.shape), fmt, KINDS[kname])
            t.upload(x if kname == "fp32" else pack16(x, KINDS[kname]))
        self.owned.append(t)
        return t

    def view(self, base, dims, ofs, stride):
        v = self.nnc.tensor_view_new(base, list(dims), list(ofs) + [0] * (12 - len(ofs)), list(stride) + [0] * (12 - len(stride)))
        self.owned.append(v)
        return v

    @staticmethod
    def raw(t):
        x = t.download()
        return x.view(np.uint16) if x.dtype == np.float16 else x

    def run(self, cmd, ins, outs, flags=0):
        l0 = self.nnc.launch_count()
        st = self.nnc.cmd_exec(cmd, None, flags, ins, outs)
        return st, self.nnc.launch_count() - l0

    def free(self):
        for t in reversed(self.owned):
            t.free()
        self.owned = []


@pytest.fixture
def dev(gpu):
    d = _Dev(gpu)
    yield d
    d.free()


def _bits(x, kname):
    """the bits a kname tensor holds for fp32 values x (round to nearest even once)"""
    x = np.asarray(x, np.float32)
    return x.copy() if kname == "fp32" else np.ascontiguousarray(pack16(x, KINDS[kname])).view(np.uint16)


def _rois(k, seed, lo=0.05, hi=0.6, outside=True):
    r = np.random.RandomState(seed)
    xy = r.uniform(-0.2 if outside else 0.0, 0.9, (k, 2))
    wh = r.uniform(lo, hi, (k, 2))
    return np.concatenate([xy, wh], 1).astype(np.float32)


def _roi_case(dev, kname, fmt, shape, rois, ph, pw, b_view=False, seed=0):
    """forward and backward of one case; returns (c, o) raw bits from the GPU and the oracle's"""
    nnc = dev.nnc
    a = seeded(shape, 100 + seed, -1, 1)
    aw = a if kname == "fp32" else round16(a, KINDS[kname])
    n = max(shape[0] if len(shape) == 4 else 1, len(rois) if rois.ndim == 2 else 1)
    cshape = (n, ph, pw, shape[-1]) if len(shape) == 4 or rois.ndim == 2 else (ph, pw, shape[-1])
    g = seeded(cshape, 200 + seed, -1, 1)
    gw = g if kname == "fp32" else round16(g, KINDS[kname])
    want_c = _bits(R.roi_align_forward(aw, rois, ph, pw), kname)
    want_o = _bits(R.roi_align_backward(gw, rois, shape), kname)
    to_fmt = (lambda x: np.moveaxis(x, -1, -3).copy()) if fmt == NCHW else (lambda x: x)
    from_fmt = (lambda x: np.moveaxis(x, -3, -1).copy()) if fmt == NCHW else (lambda x: x)
    ta, tg = dev.up(to_fmt(a), kname, fmt), dev.up(to_fmt(g), kname, fmt)
    tc, to = dev.up(to_fmt(np.full(cshape, 7, np.float32)), kname, fmt), dev.up(to_fmt(np.full(shape, 7, np.float32)), kname, fmt)
    if b_view:
        # the ROIs as columns 1..4 of NMS-shaped rows (score, x, y, w, h): a view with row stride 5
        rows = np.concatenate([np.full((len(rois), 1), 0.5, np.float32), rois], 1)
        base = dev.up(rows)
        tb = dev.view(base, [len(rois), 4], [0, 1], [5, 1])
    else:
        tb = dev.up(rois)
    st, n1 = dev.run(nnc.CMD_ROI_ALIGN_FORWARD(ph, pw), [ta, tb], [tc])
    assert (st, n1) == (0, 1), nnc.lib().ccv_nnc_sm100_last_error()
    st, n2 = dev.run(nnc.CMD_ROI_ALIGN_BACKWARD(ph, pw), [tg, None, tb], [to])
    assert (st, n2) == (0, 1), nnc.lib().ccv_nnc_sm100_last_error()
    return from_fmt(dev.raw(tc)), from_fmt(dev.raw(to)), want_c, want_o, (ta, tb, tc, tg, to)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
@pytest.mark.parametrize("fmt", [NHWC, NCHW], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("ch", [3, 130, 256])
def test_roi_align_equals_the_oracle(dev, kname, fmt, ch):
    """two maps and five ROIs (partly outside, below one pixel), pool 7x7: forward and backward give the oracle's bits"""
    rois = np.concatenate([_rois(4, ch), np.array([[0.3, 0.4, 0.01, 0.02]], np.float32)])
    got_c, got_o, want_c, want_o, _ = _roi_case(dev, kname, fmt, (2, 13, 17, ch), rois, 7, 7, seed=ch)
    assert same(got_c, want_c) and same(got_o, want_o)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_roi_align_batch_forms_pools_and_strided_rois(dev, kname):
    """one map and k ROIs as a stride-5 view, k maps and one ROI (pool 1x1), one ROI above the map (CPU_REF's row shift, pool 14x14)"""
    got_c, got_o, want_c, want_o, _ = _roi_case(dev, kname, NHWC, (20, 24, 32), _rois(9, 1), 7, 7, b_view=True, seed=1)
    assert same(got_c, want_c) and same(got_o, want_o)
    got_c, got_o, want_c, want_o, _ = _roi_case(dev, kname, NHWC, (3, 20, 24, 32), _rois(1, 2)[0], 1, 1, seed=2)
    assert same(got_c, want_c) and same(got_o, want_o)
    got_c, got_o, want_c, want_o, _ = _roi_case(dev, kname, NHWC, (20, 24, 16), np.array([-0.2, -0.3, 0.9, 0.8], np.float32), 14, 14, seed=3)
    assert same(got_c, want_c) and same(got_o, want_o)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_roi_align_1000_overlapping_rois_is_exact_and_deterministic(dev, kname):
    """1000 overlapping ROIs on one map: the oracle's bits, and a second run of the backward gives the same bits"""
    nnc = dev.nnc
    got_c, got_o, want_c, want_o, (ta, tb, tc, tg, to) = _roi_case(dev, kname, NHWC, (1, 40, 48, 24), _rois(1000, 7, 0.2, 0.7), 7, 7, seed=4)
    assert same(got_c, want_c) and same(got_o, want_o)
    assert dev.run(nnc.CMD_ROI_ALIGN_BACKWARD(7, 7), [tg, None, tb], [to]) == (0, 1)
    assert same(dev.raw(to), got_o)


@pytest.mark.gpu
def test_roi_align_bad_coordinates_read_as_empty_rois(dev):
    """NaN, Inf, huge and negative coordinates: SUCCESS, zeros for those ROIs, the oracle's bits for the others"""
    bad = np.array([[np.nan, 0.1, 0.2, 0.2], [0.1, np.inf, 0.2, 0.2], [0.1, 0.1, 1e30, 0.2], [0.1, 0.1, 0.2, -np.inf],
                    [1e30, -1e30, 0.2, 0.2], [0.2, 0.2, 0.3, 0.3], [0.1, 0.1, 5.0, 0.2]], np.float32)
    got_c, got_o, want_c, want_o, _ = _roi_case(dev, "fp32", NHWC, (1, 16, 16, 8), bad, 7, 7, seed=5)
    assert same(got_c, want_c) and same(got_o, want_o)
    assert not got_c[:5].any() and got_c[5].any()


def _nms_data(n, m, seed, ties=False):
    """rows (score, x, y, w, h) with IoUs kept away from 0.5 except at exactly representable values: boxes on an integer grid of
    power-of-two sizes"""
    r = np.random.RandomState(seed)
    a = np.empty((n, m, 5), np.float32)
    a[..., 0] = r.permutation(n * m).reshape(n, m) / np.float32(n * m) if not ties else r.randint(0, 8, (n, m)) / np.float32(8)
    a[..., 1:3] = r.randint(0, 64, (n, m, 2)) * 2
    a[..., 3:5] = 2.0 ** r.randint(1, 5, (n, m, 2))
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 63, 64, 65, 1000, 4097, 12000])
def test_nms_equals_the_oracle(dev, m):
    nnc = dev.nnc
    a = _nms_data(1, m, m)[0]
    want_b, want_c = R.nms_forward(a, 0.5)
    ta, tb, tc = dev.up(a), dev.up(np.full_like(a, 7)), dev.up(np.full((m,), 5, np.int32))
    st, n = dev.run(nnc.CMD_NMS_FORWARD(0.5), [ta], [tb, tc])
    assert (st, n) == (0, 3), nnc.lib().ccv_nnc_sm100_last_error()
    assert same(dev.raw(tb), want_b) and same(dev.raw(tc), want_c)
    g = seeded(a.shape, m, -1, 1)
    th = dev.up(np.full_like(a, 7))
    assert dev.run(nnc.CMD_NMS_BACKWARD(0.5), [dev.up(g), None, None, None, tc], [th]) == (0, 1)
    assert same(dev.raw(th), R.nms_backward(g, want_c))


@pytest.mark.gpu
@pytest.mark.parametrize("m", [65, 1000])
def test_nms_batch_of_8_as_a_strided_view(dev, m):
    """[8, m, 5] inside a larger buffer (batch stride m * 5 + 15), outputs as views too; every item equals the oracle"""
    nnc = dev.nnc
    a = _nms_data(8, m, 3 * m)
    want_b, want_c = R.nms_forward(a, 0.5)
    pad = np.zeros((8, m * 5 + 15), np.float32)
    pad[:, :m * 5] = a.reshape(8, -1)
    base_a, base_b = dev.up(pad), dev.up(np.full_like(pad, 7))
    base_c = dev.up(np.full((8, m + 3), 5, np.int32))
    va = dev.view(base_a, [8, m, 5], [0, 0, 0], [m * 5 + 15, 5, 1])
    vb = dev.view(base_b, [8, m, 5], [0, 0, 0], [m * 5 + 15, 5, 1])
    vc = dev.view(base_c, [8, m], [0, 0], [m + 3, 1])
    assert dev.run(nnc.CMD_NMS_FORWARD(0.5), [va], [vb, vc]) == (0, 3), nnc.lib().ccv_nnc_sm100_last_error()
    got_b = dev.raw(base_b)[:, :m * 5].reshape(8, m, 5)
    got_c = dev.raw(base_c)[:, :m]
    assert same(got_b, want_b) and same(got_c, want_c)
    assert (dev.raw(base_b)[:, m * 5:] == 7).all() and (dev.raw(base_c)[:, m:] == 5).all()


@pytest.mark.gpu
def test_nms_ties_flt_max_and_zero_area(dev):
    """tied scores keep input order; -FLT_MAX scores are never kept and never suppress; zero-area boxes (IoU 0 / 0) never suppress;
    thresholds 0 and 1"""
    nnc = dev.nnc
    a = _nms_data(1, 300, 11, ties=True)[0]
    a[::7, 0] = -R.FLT_MAX
    a[5::11, 3] = 0.0
    a[5::11, 1:3] = a[6::11, 1:3][:len(a[5::11])] if len(a[6::11]) >= len(a[5::11]) else a[5::11, 1:3]
    for thr in (0.5, 0.0, 1.0):
        want_b, want_c = R.nms_forward(a, thr)
        tb, tc = dev.up(np.full_like(a, 7)), dev.up(np.full((300,), 5, np.int32))
        assert dev.run(nnc.CMD_NMS_FORWARD(thr), [dev.up(a)], [tb, tc])[0] == 0
        assert same(dev.raw(tb), want_b) and same(dev.raw(tc), want_c), thr
        kept = want_c[want_c >= 0]
        assert not (a[kept, 0] == -R.FLT_MAX).any()
    ties = R.nms_forward(a, 1.0)[1]
    k = ties[ties >= 0]
    s = a[k, 0]
    assert all(k[i] < k[i + 1] for i in range(len(k) - 1) if s[i] == s[i + 1])


@pytest.mark.gpu
def test_nms_nan_scores_and_determinism(dev):
    """NaN scores: SUCCESS, and c's kept prefix holds distinct valid row indices followed by -1 only; two runs give the same bits"""
    nnc = dev.nnc
    a = _nms_data(1, 2000, 13)[0]
    a[::9, 0] = np.nan
    a[3::17, 0] = -np.nan
    ta = dev.up(a)
    outs = []
    for _ in range(2):
        tb, tc = dev.up(np.full_like(a, 7)), dev.up(np.full((2000,), 5, np.int32))
        assert dev.run(nnc.CMD_NMS_FORWARD(0.5), [ta], [tb, tc]) == (0, 3)
        outs.append((dev.raw(tb), dev.raw(tc)))
    assert same(outs[0][0], outs[1][0]) and same(outs[0][1], outs[1][1])
    c = outs[0][1]
    k = int((c >= 0).sum())
    assert (c[:k] >= 0).all() and (c[k:] == -1).all() and len(set(c[:k].tolist())) == k and c[:k].max() < 2000
    want_b, want_c = R.nms_forward(a, 0.5)
    assert same(outs[0][0], want_b) and same(c, want_c)


@pytest.mark.gpu
def test_refusals(dev):
    """INVALID with no kernel launched and every output untouched"""
    nnc = dev.nnc

    def refused(cmd, ins, outs):
        st, n = dev.run(cmd, ins, outs)
        assert st == INVALID and n == 0, (hex(cmd.cmd), st, n)
        for t in outs:
            x = dev.raw(t)
            assert (x == 5).all() if x.dtype == np.int32 else (x == _bits(np.full(x.shape, 7, np.float32), "fp32" if x.dtype == np.float32 else "bf16")).all()
    f = lambda *s: dev.up(seeded(s, 1))
    sent = lambda *s: dev.up(np.full(s, 7, np.float32))
    h16 = lambda *s: dev.up(np.full(s, 7, np.float32), "bf16")
    i32 = lambda *s: dev.up(np.full(s, 5, np.int32))
    roi, roib = nnc.CMD_ROI_ALIGN_FORWARD(4, 4), nnc.CMD_ROI_ALIGN_BACKWARD(4, 4)
    b = dev.up(np.array([0.1, 0.1, 0.5, 0.5], np.float32))
    refused(roi, [f(8, 8, 3), dev.up(np.array([0.1, 0.1, 0.5, 0.5], np.float32), "bf16")], [sent(4, 4, 3)])  # 16-bit ROIs
    refused(roi, [f(8, 8, 3), b], [sent(4, 4, 5)])                   # channel mismatch
    refused(roi, [f(2, 8, 8, 3), dev.up(seeded((3, 4), 2))], [sent(2, 4, 4, 3)])  # n != max(a_n, b_n)
    refused(roi, [f(8, 8, 3), dev.up(seeded((2, 5), 2))], [sent(2, 4, 4, 3)])     # ROI rows of 5
    refused(roi, [f(8, 8, 3), b], [h16(4, 4, 3)])                    # mixed feature types
    refused(roib, [f(4, 4, 3), None, b], [sent(8, 8, 5)])
    refused(roib, [f(4, 4, 3), None, None], [sent(8, 8, 3)])
    nms, nmsb = nnc.CMD_NMS_FORWARD(0.5), nnc.CMD_NMS_BACKWARD(0.5)
    refused(nms, [f(10, 4)], [sent(10, 4), i32(10)])                 # d != 5
    refused(nms, [f(10, 6)], [sent(10, 6), i32(10)])
    refused(nms, [f(10, 5)], [sent(10, 5), i32(9)])                  # index shape
    refused(nms, [f(10, 5)], [sent(11, 5), i32(10)])
    refused(nms, [f(2, 10, 5)], [sent(2, 10, 5), i32(10)])
    refused(nms, [f(10, 5)], [h16(10, 5), i32(10)])                  # 16-bit
    refused(nmsb, [f(10, 4), None, None, None, i32(10)], [sent(10, 4)])
    refused(nmsb, [f(10, 5), None, None, None, None], [sent(10, 5)])
    q = nnc.gpu_palettized_tensor([8, 8, 8], abi.CCV_32F, 4, 8)
    q.upload(np.zeros(q.nbytes, np.uint8))
    dev.owned.append(q)
    refused(roi, [q, b], [sent(4, 4, 8)])
    q2 = nnc.gpu_palettized_tensor([10, 5], abi.CCV_32F, 4, 5)
    q2.upload(np.zeros(q2.nbytes, np.uint8))
    dev.owned.append(q2)
    refused(nms, [q2], [sent(10, 5), i32(10)])


@pytest.mark.gpu
def test_reference_detection_programs_pass_on_the_dropin_build(gpu, tmp_path):
    """all 8 cases of int.roi_align and both of int.nms, through integration/run_reference_tests.py: they pass and none is skipped"""
    import json
    import subprocess
    import sys
    build = os.path.join(ROOT, "integration", "_build")
    progs = ("int.roi_align", "int.nms")
    if not os.path.exists(os.path.join(build, "libccv_dropin.so")) or not all(os.path.exists(os.path.join(build, p + ".tests")) for p in progs):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    out = str(tmp_path / "report.json")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_reference_tests.py"), "--only", ",".join(progs), "--budget-s", "300",
                        "--case-timeout", "60", "--out", out], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=400)
    assert p.returncode == 0, p.stdout.decode()[-2000:]
    rep = json.load(open(out))["programs"]
    for prog, count in (("int.roi_align.tests", 8), ("int.nms.tests", 2)):
        r = rep[prog]
        assert len(r["passed"]) == count and not r["skipped"] and not r["failed"] and not r["crashed"], r


# ---- a detector head through ccv_nnc_cmd_exec against CPU_REF -----------------------------------------------------------------
# fp32: the convolution's bound of the fp32 chain tests (1e-3 of max|ref|: one-pass TF32 products, 2^-11 each, in sums of 72 and 784
# terms; ROI_ALIGN and NMS add no error of their own).  bf16: the bound of the 16-bit chain tests (3e-2 of max|ref|): every command output
# is rounded to bf16 once, on a path of five (feature map, pooled, head output, pooled gradient, map gradient), CPU_REF runs fp32 on the
# same rounded inputs, and the sums over 784 and 40 terms can cancel.
CHAIN_BOUND = {"fp32": 1e-3, "bf16": 3e-2}


def _proposals(m, seed):
    """m proposal rows (score, x, y, w, h), normalised, distinct scores, clustered so that NMS suppresses about half of them"""
    r = np.random.RandomState(seed)
    centres = r.uniform(0.2, 0.7, (6, 2))
    a = np.empty((m, 5), np.float32)
    a[:, 0] = r.permutation(m) / np.float32(m)
    a[:, 1:3] = centres[r.randint(0, 6, m)] + r.uniform(-0.08, 0.08, (m, 2))
    a[:, 3:5] = r.uniform(0.1, 0.3, (m, 2))
    return a


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_detector_head_chain(gpu, ref, kname):
    """3x3 CONVOLUTION (pad 1) -> feature map; NMS (IoU 0.5) over 40 proposals -> b, c; ROI_ALIGN 7x7 of the feature map over a stride-5
    view of b's coordinate columns (the kept rows first, then the tail, whose coordinates are the sorted rows'); GEMM of the pooled
    [40, 7 * 7 * 16] rows with a [10, 784] weight; then GEMM_BACKWARD -> ROI_ALIGN_BACKWARD -> CONVOLUTION_BACKWARD.  On the GPU and on
    CPU_REF (fp32 on the same rounded inputs; the ROIs as a packed copy of the same columns).  NMS's b and c equal CPU_REF's exactly."""
    from tests.util import ref_exec, unpack16
    nnc, kind = gpu, KINDS[kname]
    H, W, C, K, m, F, P = 24, 32, 8, 16, 40, 10, 7
    r16 = (lambda v: v) if kname == "fp32" else (lambda v: round16(v, kind))
    z = lambda *s: np.zeros(s, np.float32)
    x = r16(seeded((1, H, W, C), 301, -1, 1))
    w = r16((seeded((K, 3, 3, C), 302, -1, 1) / np.sqrt(9 * C)).astype(np.float32))
    bias = r16(seeded((K,), 303, -0.1, 0.1))
    props = _proposals(m, 304)
    wh = r16((seeded((F, P * P * K), 305, -1, 1) / np.sqrt(P * P * K)).astype(np.float32))
    gh = r16(seeded((m, F), 306, -1, 1))
    hint = nnc.hint((1, 1), (1, 1))
    conv_f, conv_b = nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C), nnc.CMD_CONVOLUTION_BACKWARD(1, K, 3, 3, C)
    nms = nnc.CMD_NMS_FORWARD(0.5)
    roi_f, roi_b = nnc.CMD_ROI_ALIGN_FORWARD(P, P), nnc.CMD_ROI_ALIGN_BACKWARD(P, P)
    gemm, gemm_b = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1)), nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))

    def cpu(cmd, ins, outs, h=None):
        st, res = ref_exec(ref, cmd, h, 0, ins, outs)
        assert st == 0, hex(cmd.cmd)
        return res
    (y,) = cpu(conv_f, [x, w, bias], [z(1, H, W, K)], hint)
    nb, nc = cpu(nms, [props], [z(m, 5), np.zeros((m,), np.int32)])
    kept = int((nc >= 0).sum())
    assert 0 < kept < m and (nb[kept:, 0] == -R.FLT_MAX).all()
    rois = np.ascontiguousarray(nb[:, 1:5])
    (pooled,) = cpu(roi_f, [y, rois], [z(m, P, P, K)])
    (out,) = cpu(gemm, [pooled.reshape(m, -1), wh], [z(m, F)])
    dpooled, dwh = cpu(gemm_b, [gh, pooled.reshape(m, -1), wh], [z(m, P * P * K), z(F, P * P * K)])
    (dy,) = cpu(roi_b, [dpooled.reshape(m, P, P, K), None, rois], [z(1, H, W, K)])
    dx, dw, db = cpu(conv_b, [dy, x, w], [z(1, H, W, C), z(K, 3, 3, C), z(K)], hint)
    want = dict(y=y, pooled=pooled, out=out, dpooled=dpooled.reshape(m, P, P, K), dwh=dwh, dy=dy, dx=dx, dw=dw, db=db)

    owned, stream = [], nnc.Stream(0)

    def new(shape, dt=kind):
        t = nnc.gpu_tensor(list(shape), NHWC, dt)
        owned.append(t)
        return t

    def up(arr, dt=kind):
        return new(arr.shape, dt).upload(arr if dt != kind or kname == "fp32" else pack16(arr, kind))

    def view(base, dims, ofs, stride):
        v = nnc.tensor_view_new(base, list(dims), list(ofs) + [0] * (12 - len(ofs)), list(stride) + [0] * (12 - len(stride)))
        owned.append(v)
        return v

    def run(cmd, ins, outs, h=None):
        assert nnc.cmd_exec(cmd, h, 0, ins, outs, stream) == 0, (hex(cmd.cmd), nnc.lib().ccv_nnc_sm100_last_error())

    def down(t):
        stream.wait()
        d = t.download()
        return d if (t.params.datatype & 0xFF000) in (abi.CCV_32F, abi.CCV_32S) else unpack16(d, kind)
    try:
        xg, wg, bg, whg, ghg = up(x), up(w), up(bias), up(wh), up(gh)
        pg = up(props, abi.CCV_32F)
        yg, nbg, ncg = new((1, H, W, K)), new((m, 5), abi.CCV_32F), new((m,), abi.CCV_32S)
        run(conv_f, [xg, wg, bg], [yg], hint)
        run(nms, [pg], [nbg, ncg])
        roi_view = view(nbg, [m, 4], [0, 1], [5, 1])
        # the pooled rows are one [m, 784] tensor for the GEMMs, which ROI_ALIGN writes (and its backward reads) through a 4-d view
        pooledg, dpooledg = new((m, P * P * K)), new((m, P * P * K))
        as4 = lambda t: view(t, [m, P, P, K], [0, 0, 0, 0], [P * P * K, P * K, K, 1])
        run(roi_f, [yg, roi_view], [as4(pooledg)])
        outg, dwhg = new((m, F)), new((F, P * P * K))
        run(gemm, [pooledg, whg], [outg])
        run(gemm_b, [ghg, pooledg, whg], [dpooledg, dwhg])
        dyg = new((1, H, W, K))
        run(roi_b, [as4(dpooledg), None, roi_view], [dyg])
        dxg, dwg, dbg = new((1, H, W, C)), new((K, 3, 3, C)), new((K,))
        run(conv_b, [dyg, xg, wg], [dxg, dwg, dbg], hint)
        got = dict(y=down(yg), pooled=down(pooledg).reshape(m, P, P, K), out=down(outg), dpooled=down(dpooledg).reshape(m, P, P, K),
                   dwh=down(dwhg), dy=down(dyg), dx=down(dxg), dw=down(dwg), db=down(dbg))
        got_nb, got_nc = down(nbg), down(ncg)
    finally:
        stream.wait()
        for t in reversed(owned):
            t.free()
        stream.free()
    assert same(got_nb, nb) and same(got_nc, nc)
    tol = CHAIN_BOUND[kname]
    errs = dict((k, float(np.abs(got[k].astype(np.float64) - want[k]).max() / max(np.abs(want[k]).max(), 1e-30))) for k in want)
    print("detector head chain %s (%d of %d rows kept): max error / max|ref| %s" % (kname, kept, m, ", ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    for k, e in errs.items():
        assert np.isfinite(got[k]).all() and e <= tol, (kname, k, errs)
