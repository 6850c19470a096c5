"""The commands that only move or resample data on CCV_NNC_BACKEND_GPU_SM100, launch path by launch path, against the exact oracles
of tests/move_ref.py (pinned to the reference's CPU_REF by tests/golden/cpuref_move.npz): DATA_TRANSFER, FORMAT_TRANSFORM, TRANSPOSE,
DATATYPE_CONVERSION, INDEX_SELECT and UPSAMPLE.

Every result is compared bit for bit: these commands copy, convert or resample with the reference's own arithmetic, so there is no
rounding to allow for.  Outputs that are views live inside a larger buffer whose other elements must stay untouched; refusals must
launch nothing and leave their outputs as they were.  The CPU tests show that the comparisons reject the defects these paths
plausibly have."""
import os

import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests import move_ref as R
from tests.test_parity_feeder_paths import free_device_bytes
from tests.util import pack16, seeded

NHWC, NCHW, CHWN = abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_TENSOR_FORMAT_NCHW, abi.CCV_TENSOR_FORMAT_CHWN
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_move.npz")
NP = {abi.CCV_8U: np.uint8, abi.CCV_16F: np.float16, abi.CCV_16BF: np.uint16, abi.CCV_32F: np.float32, abi.CCV_32S: np.int32, abi.CCV_64F: np.float64}
BITS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
ALL_TYPES = [abi.CCV_8U, abi.CCV_16F, abi.CCV_16BF, abi.CCV_32F, abi.CCV_32S, abi.CCV_64F]
NAMES = {abi.CCV_8U: "8U", abi.CCV_16F: "16F", abi.CCV_16BF: "16BF", abi.CCV_32F: "32F", abi.CCV_32S: "32S", abi.CCV_64F: "64F"}

# upsample geometries (H, W, OH, OW): 1x, 2x, 1.5x, and scales where (i + 0.5) * H / OH is an integer that float(H / OH) misses
# (6 -> 19 at i = 9, 8 -> 25 at i = 12, 10 -> 23 at i = 11), and 1 -> k
UP_CASES = [(5, 7, 5, 7), (4, 6, 8, 12), (6, 4, 9, 6), (6, 8, 19, 25), (10, 1, 23, 4), (1, 3, 5, 7), (8, 10, 25, 23)]
# index-select lerp: integer-valued indices, the last row (j1 clamps to it), fractions
LERP_IDX = np.array([0.0, 1.0, 2.5, 6.0, 6.75, 5.999, 0.125, 3.3333333, 4.5, 1e-7], np.float32)


# ---- data ---------------------------------------------------------------------------------------------------------------------------
def random_bits(shape, dt, seed):
    """arbitrary bit patterns of the type (NaNs and infinities included): the copies must move bits, not values"""
    r = np.random.RandomState(seed)
    size = np.dtype(NP[dt]).itemsize
    n = int(np.prod(shape))
    return np.frombuffer(r.bytes(n * size), NP[dt]).reshape(shape).copy()


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view(BITS[x.dtype.itemsize])


def same_bits(got, want, what=""):
    got, want = bits(got), bits(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got.ravel() != want.ravel())
    assert bad.size == 0, "%s: %d of %d differ, first at %s: %s != %s" % (what, bad.size, got.size, np.unravel_index(bad[0], got.shape), hex(int(got.ravel()[bad[0]])), hex(int(want.ravel()[bad[0]])))


def cstrides(shape):
    s, acc = [], 1
    for d in reversed(shape):
        s.insert(0, acc)
        acc *= d
    return s


def padded_layout(shape):
    """a view's layout inside a larger buffer: every axis padded (the last by 2) and the base moved by one element"""
    pshape = [d + (2 if i == len(shape) - 1 else 1) for i, d in enumerate(shape)]
    return cstrides(pshape), 1, int(np.prod(pshape)) + 1


class Dev(object):
    """numpy arrays as GPU (or host) tensors, packed or as views inside a guarded buffer"""

    def __init__(self, nnc):
        self.nnc, self.owned, self.layout = nnc, [], {}

    def put(self, a, dt, fmt=NHWC, strided=False, host=False, strides=None):
        nnc = self.nnc
        shape = list(a.shape)
        if not strided:
            t = (nnc.cpu_tensor if host else nnc.gpu_tensor)(shape, fmt, dt)
            t.upload(a)
            self.owned.append(t)
            return t
        st, off, size = padded_layout(shape) if strides is None else strides
        # a guard pattern whose bits must survive wherever the command does not write
        buf = np.full(size * np.dtype(NP[dt]).itemsize, 0x5A, np.uint8).view(NP[dt])
        np.lib.stride_tricks.as_strided(buf[off:], shape=tuple(shape), strides=tuple(s * buf.itemsize for s in st))[...] = a
        parent = (nnc.cpu_tensor if host else nnc.gpu_tensor)([size], fmt, dt)
        parent.upload(buf)
        k = int(np.argmin(st))
        assert off % st[k] == 0
        ofs = [0] * len(shape)
        ofs[k] = off // st[k]
        v = nnc.tensor_view_new(parent, shape, ofs, st)
        self.owned += [v, parent]
        self.layout[id(v)] = (parent, buf, st, off, shape)
        return v

    def get(self, t):
        """a tensor's logical content; for a view, also asserts the rest of its buffer is untouched"""
        if id(t) not in self.layout:
            return t.download()
        parent, before, st, off, shape = self.layout[id(t)]
        after = parent.download()
        inside = np.zeros(after.size, bool)
        idx = np.lib.stride_tricks.as_strided(np.arange(after.size)[off:], shape=tuple(shape), strides=tuple(s * 8 for s in st))
        inside[idx.ravel()] = True
        same_bits(after[~inside], before[~inside], "outside the view")
        return np.ascontiguousarray(R.view(after, off, shape, st))

    def free(self):
        for t in self.owned:
            t.free()
        self.owned = []


def run(nnc, cmd, ins, outs, stream=None):
    """ins / outs: (array, datatype, dict of Dev.put options); -> (status, output arrays, launches)"""
    dev = Dev(nnc)
    try:
        ti = [None if a is None else dev.put(a[0], a[1], **(a[2] if len(a) > 2 else {})) for a in ins]
        to = [None if a is None else dev.put(a[0], a[1], **(a[2] if len(a) > 2 else {})) for a in outs]
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(cmd, None, 0, ti, to, stream)
        if stream is not None:
            stream.wait()
        launches = nnc.launch_count() - l0
        return st, [None if t is None else dev.get(t) for t in to], launches
    finally:
        dev.free()


def refused(nnc, cmd, ins, outs):
    """the call returns INVALID, launches nothing and leaves every output as it was"""
    st, got, launches = run(nnc, cmd, ins, outs)
    assert (st, launches) == (INVALID, 0)
    for g, o in zip(got, outs):
        if o is not None:
            same_bits(g, o[0], "refused output")


def upsample_cmd(bwd, bilinear, align, H, W, OH, OW):
    c = _nnc._simple(abi.CCV_NNC_UPSAMPLE_BACKWARD if bwd else abi.CCV_NNC_UPSAMPLE_FORWARD, (2, 2, 1))
    u = c.info.upsample
    u.type = abi.CCV_NNC_UPSAMPLE_BILINEAR if bilinear else abi.CCV_NNC_UPSAMPLE_NEAREST
    u.width_scale, u.height_scale, u.align_corners = OW / W, OH / H, align
    return c


def up_shape(N, C, H, W, nchw, nd=4):
    s = (N, C, H, W) if nchw else (N, H, W, C)
    return s if nd == 4 else s[1:]


def up_data(shape, seed):
    return seeded(shape, seed, -1, 1)


# ---- CPU: the oracles are CPU_REF ----------------------------------------------------------------------------------------------------
def _golden():
    return np.load(GOLDEN)


def test_conversion_oracle_matches_cpu_ref_fixture():
    g = _golden()
    same_bits(R.f32_to_f16(g["f2h_x"]), g["f2h_h"], "f32 -> f16")
    same_bits(R.f64_to_f16(g["d2h_x"]), g["d2h_h"], "f64 -> f16")
    codes = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    f = R.f16_to_f32(codes)
    fin = ~np.isnan(f)
    same_bits(f[fin], g["h2f_f"][fin], "f16 -> f32")
    assert np.isnan(g["h2f_f"][~fin]).all()
    # the table truncates: 65520 (Inf under round-to-nearest) stays the largest half, 65536 is Inf, and a NaN with only low payload
    # bits becomes Inf
    h = R.f32_to_f16(np.array([65519.0, 65520.0, 65536.0], np.float32))
    assert [int(v) for v in h] == [0x7BFF, 0x7BFF, 0x7C00]
    assert R.f32_to_f16(np.array([0x7F801FFF], np.uint32).view(np.float32))[0] == 0x7C00


@pytest.mark.parametrize("H,W,OH,OW", UP_CASES)
@pytest.mark.parametrize("bilinear", [0, 1])
@pytest.mark.parametrize("align", [0, 1])
@pytest.mark.parametrize("nchw", [0, 1])
def test_upsample_oracle_matches_cpu_ref_fixture(H, W, OH, OW, bilinear, align, nchw):
    g = _golden()
    key = "up_%d_%d_%d_%d_%d_%d_%d_" % (H, W, OH, OW, bilinear, align, nchw)
    a, y = g[key + "a"], g[key + "g"]
    same_bits(R.upsample_forward(a, OH, OW, bilinear, align, nchw), g[key + "b"], "forward")
    same_bits(R.upsample_backward(y, H, W, bilinear, align, nchw), g[key + "h"], "backward")


def test_index_select_oracle_matches_cpu_ref_fixture():
    g = _golden()
    same_bits(R.index_select_lerp(g["is_a"], LERP_IDX), g["is_lerp"], "lerp")
    same_bits(R.index_select(g["is_a"], g["is_idx"]), g["is_b"], "copy")
    same_bits(R.index_select_back(g["is_g"], g["is_idx"], g["is_a"].shape[0]), g["is_h"], "backward")


def test_fixture_holds_the_mismatching_scales():
    """the fixture's nearest cases include outputs where float arithmetic picks another source pixel than CPU_REF"""
    hits = 0
    for H, W, OH, OW in UP_CASES:
        for align in (0, 1):
            for i, o in ((H, OH), (W, OW)):
                hits += int((R.nearest_index(i, o, align) != R.nearest_index(i, o, align, double=False)).sum())
    assert hits >= 3


# ---- CPU: the comparisons reject plausible defects -----------------------------------------------------------------------------------
def _rejects(got, want):
    with pytest.raises(AssertionError):
        same_bits(got, want)


def test_float_nearest_index_is_rejected():
    a = up_data(up_shape(2, 3, 6, 8, 1), 1)
    want = R.upsample_forward(a, 19, 25, 0, 0, 1)
    bad = a[:, :, R.nearest_index(6, 19, 0, double=False)][:, :, :, R.nearest_index(8, 25, 0, double=False)]
    _rejects(bad, want)


def test_round_to_nearest_f16_is_rejected():
    x = R.f16_specials()
    fin = np.isfinite(x)
    with np.errstate(over="ignore"):
        _rejects(x[fin].astype(np.float16).view(np.uint16), R.f32_to_f16(x[fin]))


def test_swapped_transpose_axes_are_rejected():
    a = random_bits((2, 3, 4, 5), abi.CCV_32F, 1)
    _rejects(R.transpose(a, 1, 2).reshape(-1)[:60].reshape(3, 4, 5), R.transpose(a, 1, 3).reshape(-1)[:60].reshape(3, 4, 5))
    _rejects(np.ascontiguousarray(np.transpose(a, (0, 2, 1, 3))).reshape(2, 3, 4, 5), R.transpose(a, 0, 1).reshape(2, 3, 4, 5))


def test_ignored_view_stride_is_rejected():
    a = random_bits((3, 4, 5), abi.CCV_32F, 2)
    st, off, size = padded_layout(a.shape)
    buf = np.zeros(size, np.float32)
    np.lib.stride_tricks.as_strided(buf[off:], shape=a.shape, strides=tuple(s * 4 for s in st))[...] = a
    _rejects(buf[off:off + a.size].reshape(a.shape), a)


def test_reordered_bilinear_backward_is_rejected():
    y = up_data(up_shape(2, 3, 19, 25, 0), 3)
    want = R.upsample_backward(y, 6, 8, 1, 0, 0)
    order = np.random.RandomState(4).permutation(19 * 25)
    _rejects(R.upsample_backward(y, 6, 8, 1, 0, 0, order=order), want)


# ---- GPU: DATA_TRANSFER --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", [("gpu", "gpu"), ("host", "gpu"), ("gpu", "host")])
@pytest.mark.parametrize("dt", ALL_TYPES, ids=lambda d: NAMES[d])
def test_transfer_packed(gpu, src, dst, dt):
    a = random_bits((3, 5, 7), dt, 10)
    st, (b,), _ = run(gpu, gpu.CMD_DATA_TRANSFER_FORWARD(), [(a, dt, dict(host=src == "host"))], [(np.zeros_like(a), dt, dict(host=dst == "host"))])
    assert st == 0
    same_bits(b, a)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ALL_TYPES, ids=lambda d: NAMES[d])
@pytest.mark.parametrize("shape", [(37,), (5, 9), (3, 4, 7), (2, 3, 5, 6)])
@pytest.mark.parametrize("views", ["a", "b", "ab"])
def test_transfer_views(gpu, dt, shape, views):
    a = random_bits(shape, dt, 11)
    st, (b,), launches = run(gpu, gpu.CMD_DATA_TRANSFER_FORWARD(), [(a, dt, dict(strided="a" in views))], [(np.zeros_like(a), dt, dict(strided="b" in views))])
    assert st == 0
    same_bits(b, a)


@pytest.mark.gpu
def test_transfer_permuted_view_strides(gpu):
    """a view whose strides are not in decreasing order (copy_strided reorders the axes by the output's strides)"""
    a = random_bits((4, 6, 5), abi.CCV_32F, 12)
    lay = ([1, 4 * 5 + 3, 4], 0, 6 * 23 + 4 * 5 + 8)  # axis 0 fastest, then axis 2, then axis 1
    st, (b,), _ = run(gpu, gpu.CMD_DATA_TRANSFER_FORWARD(), [(a, abi.CCV_32F, dict(strided=True, strides=lay))], [(np.zeros_like(a), abi.CCV_32F)])
    assert st == 0
    same_bits(b, a)
    st, (b,), _ = run(gpu, gpu.CMD_DATA_TRANSFER_FORWARD(), [(a, abi.CCV_32F)], [(np.zeros_like(a), abi.CCV_32F, dict(strided=True, strides=lay))])
    assert st == 0
    same_bits(b, a)


@pytest.mark.gpu
def test_transfer_several_pairs_and_self(gpu):
    a0, a1 = random_bits((4, 5), abi.CCV_32F, 13), random_bits((6,), abi.CCV_16F, 14)
    st, (b0, b1), _ = run(gpu, gpu.CMD_DATA_TRANSFER_FORWARD(), [(a0, abi.CCV_32F), (a1, abi.CCV_16F, dict(strided=True))],
                          [(np.zeros_like(a0), abi.CCV_32F, dict(strided=True)), (np.zeros_like(a1), abi.CCV_16F)])
    assert st == 0
    same_bits(b0, a0), same_bits(b1, a1)
    nnc = gpu
    t = nnc.gpu_tensor([4, 5])
    try:
        t.upload(a0)
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [t], [t]) == 0
        assert nnc.launch_count() == l0
        same_bits(t.download(), a0)
    finally:
        t.free()


@pytest.mark.gpu
def test_transfer_without_stream_is_blocking(gpu):
    """without a stream context the copy to a host tensor has finished when the call returns"""
    nnc = gpu
    a = random_bits((1 << 20,), abi.CCV_32F, 15)
    ta, tb = nnc.gpu_tensor([a.size]), nnc.cpu_tensor([a.size])
    try:
        ta.upload(a)
        assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [ta], [tb]) == 0
        same_bits(tb.download(), a)
    finally:
        ta.free(), tb.free()


@pytest.mark.gpu
def test_transfer_refusals(gpu):
    a = random_bits((3, 4, 5), abi.CCV_32F, 16)
    cmd = gpu.CMD_DATA_TRANSFER_FORWARD()
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(strided=True, host=True))], [(np.zeros_like(a), abi.CCV_32F)])
    refused(gpu, cmd, [(a, abi.CCV_32F)], [(np.zeros_like(a), abi.CCV_32F, dict(strided=True, host=True))])
    a5 = random_bits((2, 2, 3, 2, 2), abi.CCV_32F, 17)
    refused(gpu, cmd, [(a5, abi.CCV_32F, dict(strided=True))], [(np.zeros_like(a5), abi.CCV_32F)])
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(strided=True))], [(np.zeros((3, 5, 4), np.float32), abi.CCV_32F)])


# ---- GPU: FORMAT_TRANSFORM -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ALL_TYPES, ids=lambda d: NAMES[d])
@pytest.mark.parametrize("nd", [3, 4])
@pytest.mark.parametrize("to_nchw", [1, 0])
@pytest.mark.parametrize("views", ["", "a", "b", "ab"])
def test_format_transform(gpu, dt, nd, to_nchw, views):
    shape = (2, 5, 6, 7)[4 - nd:]
    a = random_bits(shape, dt, 20)
    want = R.nhwc_to_nchw(a) if to_nchw else R.nchw_to_nhwc(a)
    fa, fb = (NHWC, NCHW) if to_nchw else (NCHW, NHWC)
    st, (b,), launches = run(gpu, gpu.CMD_FORMAT_TRANSFORM_FORWARD(), [(a, dt, dict(fmt=fa, strided="a" in views))],
                             [(np.zeros_like(want), dt, dict(fmt=fb, strided="b" in views))])
    assert st == 0
    same_bits(b, want)


@pytest.mark.gpu
def test_format_transform_plain_copies_and_skips(gpu):
    cmd = gpu.CMD_FORMAT_TRANSFORM_FORWARD()
    a = random_bits((2, 3, 4, 5), abi.CCV_16BF, 21)
    st, (b,), _ = run(gpu, cmd, [(a, abi.CCV_16BF, dict(fmt=NCHW, strided=True))], [(np.zeros_like(a), abi.CCV_16BF, dict(fmt=NCHW))])
    assert st == 0
    same_bits(b, a)
    for shape in ((9,), (4, 6)):
        a = random_bits(shape, abi.CCV_32F, 22)
        st, (b,), _ = run(gpu, cmd, [(a, abi.CCV_32F, dict(fmt=NCHW))], [(np.zeros_like(a), abi.CCV_32F, dict(fmt=NHWC))])
        assert st == 0
        same_bits(b, a)
    # dim[0] == 0: nothing to do
    nnc = gpu
    ta, tb = nnc.gpu_tensor([2, 3, 4, 5], NHWC), nnc.gpu_tensor([2, 5, 3, 4], NCHW)
    try:
        ta.struct.info.dim[0] = tb.struct.info.dim[0] = 0
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(cmd, None, 0, [ta], [tb]) == 0
        assert nnc.launch_count() == l0
    finally:
        ta.free(), tb.free()


@pytest.mark.gpu
def test_format_transform_refusals(gpu):
    cmd = gpu.CMD_FORMAT_TRANSFORM_FORWARD()
    a = random_bits((2, 5, 6, 7), abi.CCV_32F, 23)
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(fmt=NHWC))], [(np.zeros((7, 5, 6, 2), np.float32), abi.CCV_32F, dict(fmt=CHWN))])
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(fmt=NHWC))], [(np.zeros((2, 7, 5, 6), np.int32), abi.CCV_32S, dict(fmt=NCHW))])
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(fmt=NHWC))], [(np.zeros((2, 7, 6, 5), np.float32), abi.CCV_32F, dict(fmt=NCHW))])


# ---- GPU: TRANSPOSE ------------------------------------------------------------------------------------------------------------------
TRANSPOSE_SHAPES = {2: (7, 9), 3: (3, 1, 5), 4: (2, 3, 5, 7)}


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [abi.CCV_32F, abi.CCV_16BF, abi.CCV_16F], ids=lambda d: NAMES[d])
@pytest.mark.parametrize("nd", [2, 3, 4])
@pytest.mark.parametrize("views", ["", "ab"])
def test_transpose_every_axis_pair(gpu, dt, nd, views):
    a = random_bits(TRANSPOSE_SHAPES[nd], dt, 30 + nd)
    for ax0 in range(nd):
        for ax1 in range(nd):
            want = R.transpose(a, ax0, ax1)
            st, (b,), launches = run(gpu, gpu.CMD_TRANSPOSE_FORWARD(ax0, ax1), [(a, dt, dict(strided="a" in views))],
                                     [(np.zeros_like(want), dt, dict(strided="b" in views))])
            assert st == 0, (ax0, ax1)
            same_bits(b, want, "axes %d, %d" % (ax0, ax1))


@pytest.mark.gpu
def test_transpose_refusals(gpu):
    a = random_bits((3, 4, 5), abi.CCV_32F, 35)
    refused(gpu, gpu.CMD_TRANSPOSE_FORWARD(0, 3), [(a, abi.CCV_32F)], [(np.zeros((3, 4, 5), np.float32), abi.CCV_32F)])
    refused(gpu, gpu.CMD_TRANSPOSE_FORWARD(0, 1), [(a, abi.CCV_32F)], [(np.zeros((4, 15), np.float32), abi.CCV_32F)])
    refused(gpu, gpu.CMD_TRANSPOSE_FORWARD(0, 1), [(a, abi.CCV_32F)], [(np.zeros((4, 3, 5), np.float16), abi.CCV_16F)])
    refused(gpu, gpu.CMD_TRANSPOSE_FORWARD(0, 1), [(a, abi.CCV_32F)], [(np.zeros((3, 4, 5), np.float32), abi.CCV_32F)])


# ---- GPU: DATATYPE_CONVERSION --------------------------------------------------------------------------------------------------------
def convert(nnc, x, dt_a, dt_b, out_np):
    st, (y,), _ = run(nnc, nnc.CMD_DATATYPE_CONVERSION_FORWARD(), [(x, dt_a)], [(np.zeros(x.shape, out_np), dt_b)])
    assert st == 0
    return y


def f32_inputs():
    r = np.random.RandomState(40)
    return np.concatenate([R.f16_specials(), r.randint(0, 2 ** 32, size=1 << 20, dtype=np.uint64).astype(np.uint32).view(np.float32)])


@pytest.mark.gpu
def test_conversion_from_f16_is_exact_for_every_code(gpu):
    h = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)
    want = R.f16_to_f32(h.view(np.uint16))
    nan = np.isnan(want)
    for dt_b, out_np in ((abi.CCV_32F, np.float32), (abi.CCV_64F, np.float64)):
        y = convert(gpu, h, abi.CCV_16F, dt_b, out_np)
        same_bits(y[~nan], want[~nan].astype(out_np), "f16 -> " + NAMES[dt_b])
        assert np.isnan(y[nan]).all()


@pytest.mark.gpu
def test_conversion_to_f16_truncates_like_the_reference(gpu):
    x = f32_inputs()
    same_bits(convert(gpu, x, abi.CCV_32F, abi.CCV_16F, np.float16), R.f32_to_f16(x), "f32 -> f16")
    r = np.random.RandomState(41)
    d = np.concatenate([R.f16_specials().astype(np.float64), [65519.99999999, 65520.000001, 2.0 ** -25 * (1 + 2.0 ** -30), 1 + 2.0 ** -24 + 2.0 ** -40, 1e300, -1e300, 1e-300],
                        r.uniform(-70000, 70000, 1 << 16), r.standard_normal(1 << 16) * 1e-5])
    same_bits(convert(gpu, d, abi.CCV_64F, abi.CCV_16F, np.float16), R.f64_to_f16(d), "f64 -> f16")


@pytest.mark.gpu
def test_conversion_bf16_f64_f32(gpu):
    x = f32_inputs()
    nan = np.isnan(x)
    y = convert(gpu, x, abi.CCV_32F, abi.CCV_16BF, np.uint16)
    same_bits(y[~nan], R.f32_to_bf16(x[~nan]), "f32 -> bf16")
    assert np.isnan(R.bf16_to_f32(y[nan])).all()
    codes = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    want = R.bf16_to_f32(codes)
    y = convert(gpu, codes, abi.CCV_16BF, abi.CCV_32F, np.float32)
    same_bits(y[~np.isnan(want)], want[~np.isnan(want)], "bf16 -> f32")
    assert np.isnan(y[np.isnan(want)]).all()
    y = convert(gpu, x, abi.CCV_32F, abi.CCV_64F, np.float64)
    same_bits(y[~nan], x[~nan].astype(np.float64), "f32 -> f64")
    assert np.isnan(y[nan]).all()
    r = np.random.RandomState(42)
    d = np.concatenate([x.astype(np.float64), r.standard_normal(1 << 16) * 10.0 ** r.randint(-50, 50, 1 << 16), [1e300, -1e300, 1e-300, 3.4028235677973366e38]])
    with np.errstate(over="ignore"):
        want = d.astype(np.float32)
    y = convert(gpu, d, abi.CCV_64F, abi.CCV_32F, np.float32)
    same_bits(y[~np.isnan(d)], want[~np.isnan(d)], "f64 -> f32")
    assert np.isnan(y[np.isnan(d)]).all()


@pytest.mark.gpu
def test_conversion_same_type_view(gpu):
    a = random_bits((4, 6, 5), abi.CCV_32F, 43)
    st, (b,), _ = run(gpu, gpu.CMD_DATATYPE_CONVERSION_FORWARD(), [(a, abi.CCV_32F, dict(strided=True))], [(np.zeros_like(a), abi.CCV_32F)])
    assert st == 0
    same_bits(b, a)


@pytest.mark.gpu
def test_conversion_refusals(gpu):
    """the directions without a kernel (16F <-> 16BF, 16BF <-> 64F), non-contiguous operands and a count mismatch are refused on purpose"""
    cmd = gpu.CMD_DATATYPE_CONVERSION_FORWARD()
    h = random_bits((64,), abi.CCV_16F, 44)
    bf = random_bits((64,), abi.CCV_16BF, 45)
    d = seeded((64,), 46).astype(np.float64)
    refused(gpu, cmd, [(h, abi.CCV_16F)], [(np.zeros(64, np.uint16), abi.CCV_16BF)])
    refused(gpu, cmd, [(bf, abi.CCV_16BF)], [(np.zeros(64, np.float16), abi.CCV_16F)])
    refused(gpu, cmd, [(bf, abi.CCV_16BF)], [(np.zeros(64, np.float64), abi.CCV_64F)])
    refused(gpu, cmd, [(d, abi.CCV_64F)], [(np.zeros(64, np.uint16), abi.CCV_16BF)])
    a = seeded((4, 16), 47)
    refused(gpu, cmd, [(a, abi.CCV_32F, dict(strided=True))], [(np.zeros((4, 16), np.float16), abi.CCV_16F)])
    refused(gpu, cmd, [(a, abi.CCV_32F)], [(np.zeros((4, 16), np.float16), abi.CCV_16F, dict(strided=True))])
    refused(gpu, cmd, [(a, abi.CCV_32F)], [(np.zeros((4, 15), np.float16), abi.CCV_16F)])


# ---- GPU: INDEX_SELECT ---------------------------------------------------------------------------------------------------------------
def row_view(shape):
    """a row-strided view: each row padded by 3 elements, the base moved by one"""
    cols = shape[1] if len(shape) > 1 else 1
    if len(shape) == 1:
        return ([cols + 3], 1, shape[0] * (cols + 3) + 1)
    return ([cols + 3, 1], 1, shape[0] * (cols + 3) + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [abi.CCV_32F, abi.CCV_32S, abi.CCV_16F, abi.CCV_16BF], ids=lambda d: NAMES[d])
@pytest.mark.parametrize("width,views", [(0, "")] + [(w, v) for w in (1, 31, 64, 257) for v in ("", "a", "b", "ab")])
def test_index_select_forward(gpu, dt, width, views):
    """width 0: a 1-d tensor (whose view stride the reference ignores, so only packed).  Indices -1 and rows are out of range: their
    rows of b stay as they were"""
    rows = 11
    ashape = (rows,) if width == 0 else (rows, width)
    a = random_bits(ashape, dt, 50)
    idx = np.array([3, 0, 10, 3, -1, 7, rows, 10, 5], np.int32)
    bshape = (len(idx),) + ashape[1:]
    b0 = random_bits(bshape, dt, 51)
    want = R.index_select(a, idx, b0)
    st, (b,), launches = run(gpu, gpu.CMD_INDEX_SELECT_FORWARD(), [(a, dt, dict(strided="a" in views, strides=row_view(ashape) if "a" in views else None)), (idx, abi.CCV_32S)],
                             [(b0, dt, dict(strided="b" in views, strides=row_view(bshape) if "b" in views else None))])
    assert st == 0
    same_bits(b, want)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 31, 257])
def test_index_select_lerp(gpu, width):
    a = seeded((7, width), 52, -2, 2)
    st, (b,), _ = run(gpu, gpu.CMD_INDEX_SELECT_FORWARD(), [(a, abi.CCV_32F), (LERP_IDX, abi.CCV_32F)], [(np.zeros((len(LERP_IDX), width), np.float32), abi.CCV_32F)])
    assert st == 0
    same_bits(b, R.index_select_lerp(a, LERP_IDX))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [abi.CCV_32F, abi.CCV_16F, abi.CCV_16BF], ids=lambda d: NAMES[d])
@pytest.mark.parametrize("width", [1, 64, 257])
@pytest.mark.parametrize("views", ["", "gh"])
def test_index_select_backward(gpu, dt, width, views):
    """repeated indices sum in increasing order in fp32; a 16-bit gradient is rounded once; the index gradient is zeroed"""
    rows = 6
    idx = np.array([2, 5, 2, 0, 2, 5, 1, 2], np.int32)
    g = seeded((len(idx), width), 53, -1, 1) * np.float32(1000) ** seeded((len(idx), 1), 54, -1, 1)
    g = g.astype(np.float32)
    if dt != abi.CCV_32F:
        g = pack16(g, dt)
    g32 = g.astype(np.float32) if dt == abi.CCV_16F else (R.bf16_to_f32(g) if dt == abi.CCV_16BF else g)
    h32 = R.index_select_back(g32, idx, rows)
    want = h32 if dt == abi.CCV_32F else pack16(h32, dt)
    h0 = random_bits((rows, width), dt, 55)
    di = np.full(len(idx), 7, np.int32)
    outs = None
    for _ in range(2):
        st, got, _ = run(gpu, gpu.CMD_INDEX_SELECT_BACKWARD(), [(g, dt, dict(strided="g" in views, strides=row_view(g.shape) if views else None)), None, (idx, abi.CCV_32S)],
                         [(h0, dt, dict(strided="h" in views, strides=row_view(h0.shape) if views else None)), (di, abi.CCV_32S)])
        assert st == 0
        same_bits(got[0], want)
        assert (got[1] == 0).all()
        if outs is not None:
            same_bits(got[0], outs[0], "two runs")
        outs = got


# ---- GPU: UPSAMPLE -------------------------------------------------------------------------------------------------------------------
def _up16(x, dt):
    """a float32 result as the 16-bit tensor holds it (rounded once to nearest even), as bits"""
    return pack16(x, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [abi.CCV_32F, abi.CCV_16BF, abi.CCV_16F], ids=lambda d: NAMES[d])
@pytest.mark.parametrize("bilinear", [0, 1])
@pytest.mark.parametrize("align", [0, 1])
@pytest.mark.parametrize("nchw", [0, 1])
def test_upsample(gpu, dt, bilinear, align, nchw):
    """forward and backward at every geometry of UP_CASES, 4-d and 3-d; the backward twice, with the same bits"""
    fmt = NCHW if nchw else NHWC
    for k, (H, W, OH, OW) in enumerate(UP_CASES):
        for nd in (4, 3):
            ishape, oshape = up_shape(2, 3, H, W, nchw, nd), up_shape(2, 3, OH, OW, nchw, nd)
            a, y = up_data(ishape, 60 + k), up_data(oshape, 70 + k)
            if dt != abi.CCV_32F:
                a16, y16 = pack16(a, dt), pack16(y, dt)
                a = a16.astype(np.float32) if dt == abi.CCV_16F else R.bf16_to_f32(a16)
                y = y16.astype(np.float32) if dt == abi.CCV_16F else R.bf16_to_f32(y16)
            else:
                a16, y16 = a, y
            what = "%dx%d -> %dx%d, %d-d" % (H, W, OH, OW, nd)
            want_b = R.upsample_forward(a, OH, OW, bilinear, align, nchw)
            want_h = R.upsample_backward(y, H, W, bilinear, align, nchw)
            if dt != abi.CCV_32F:
                want_b, want_h = _up16(want_b, dt), _up16(want_h, dt)
            st, (b,), _ = run(gpu, upsample_cmd(0, bilinear, align, H, W, OH, OW), [(a16, dt, dict(fmt=fmt))], [(np.zeros(oshape, NP[dt]), dt, dict(fmt=fmt))])
            assert st == 0, what
            same_bits(b, want_b, "forward " + what)
            first = None
            for _ in range(2):
                st, (h,), _ = run(gpu, upsample_cmd(1, bilinear, align, H, W, OH, OW), [(y16, dt, dict(fmt=fmt))], [(random_bits(ishape, dt, 80), dt, dict(fmt=fmt))])
                assert st == 0, what
                if first is not None:
                    same_bits(h, first, "backward run to run " + what)
                first = h
            same_bits(h, want_h, "backward " + what)


@pytest.mark.gpu
def test_upsample_refusals(gpu):
    a = up_data((2, 6, 8, 3), 90)
    refused(gpu, upsample_cmd(0, 0, 0, 6, 8, 3, 4), [(a, abi.CCV_32F)], [(np.zeros((2, 3, 4, 3), np.float32), abi.CCV_32F)])
    refused(gpu, upsample_cmd(0, 1, 0, 6, 8, 12, 16), [(a, abi.CCV_32F, dict(fmt=NHWC))], [(np.zeros((2, 3, 12, 16), np.float32), abi.CCV_32F, dict(fmt=NCHW))])
    y = up_data((2, 12, 16, 3), 91)
    refused(gpu, upsample_cmd(1, 0, 0, 13, 8, 12, 16), [(y, abi.CCV_32F)], [(np.zeros((2, 13, 8, 3), np.float32), abi.CCV_32F)])


# ---- GPU: 64-bit index space ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_transfer_64bit_index(gpu):
    """one copy_strided transfer of a 1-byte view of more than 2^31 elements (3 x 2^15 x 2^15 inside rows of 2^15 + 64); the
    destination's last 4099 bytes are checked"""
    nnc = gpu
    D, P = 1 << 15, (1 << 15) + 64
    shape = (3, D, D)
    total = 3 * D * D
    assert total > 2 ** 31
    need = 3 * D * P + total + (1 << 30)
    if free_device_bytes() < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 2 ** 30))
    big_a = nnc.gpu_tensor([3 * D, P], datatype=abi.CCV_8U)  # a tensor extent is an int: no axis beyond 2^31
    big_b = nnc.gpu_tensor(list(shape), datatype=abi.CCV_8U)
    owned = [big_b, big_a]
    try:
        tail = 4099
        # the last D * 2 elements of the view: its last two rows
        rows = np.random.RandomState(95).randint(0, 256, size=(2, D)).astype(np.uint8)
        src = nnc.gpu_tensor([2, P], datatype=abi.CCV_8U, ptr=big_a.data_ptr + (3 * D - 2) * P)
        owned.insert(0, src)
        host = np.zeros((2, P), np.uint8)
        host[:, :D] = rows
        src.upload(host)
        va = nnc.tensor_view_new(big_a, list(shape), [0, 0, 0], [D * P, P, 1])
        owned.insert(0, va)
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [va], [big_b]) == 0
        assert nnc.launch_count() - l0 == 1
        lb = nnc.gpu_tensor([tail], datatype=abi.CCV_8U, ptr=big_b.data_ptr + total - tail)
        owned.insert(0, lb)
        same_bits(lb.download(), rows.reshape(-1)[-tail:])
    finally:
        for t in owned:
            t.free()
