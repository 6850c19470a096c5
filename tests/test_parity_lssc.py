"""COMPRESSION_LSSC on the GPU, bit for bit against the restatement of tests/lssc_ref.py (itself pinned to CPU_REF by
tests/test_lssc_cpu.py) and against CPU_REF where oracle/_ref is present: every kernel form (NCHW band runs, NHWC 8-channel vectors,
the per-channel form), aligned and misaligned bases, ragged H and W, 3-d and 4-d tensors, the reference's int-test shapes, ResNet-50
activation shapes, multi-pair calls, refusals, and a flat graph (convolution -> LSSC forward -> LSSC backward -> convolution backward)
run fused and captured against the same commands run eagerly."""
import numpy as np
import pytest

from ccv_b200 import abi
from tests import lssc_ref as R
from tests.util import pack16

pytestmark = pytest.mark.gpu

FMT = {R.NCHW: abi.CCV_TENSOR_FORMAT_NCHW, R.NHWC: abi.CCV_TENSOR_FORMAT_NHWC}
INVALID = abi.CCV_NNC_EXEC_INVALID


class _Dev(object):
    """fp16 GPU tensors, each at element offset `off` of a larger buffer (off 0: 16-byte aligned); freed by free()"""

    def __init__(self, nnc):
        self.nnc, self.owned = nnc, []

    def tensor(self, dims, fmt, bits=None, off=0, fill=0x5a5a):
        n = int(np.prod(dims))
        big = self.nnc.gpu_tensor([n + off + 8], FMT[fmt], abi.CCV_16F)
        host = np.full(n + off + 8, fill, np.uint16)
        if bits is not None:
            host[off:off + n] = np.asarray(bits, np.uint16).ravel()
        big.upload(host.view(np.float16))
        t = self.nnc.gpu_tensor(list(dims), FMT[fmt], abi.CCV_16F, ptr=big.data_ptr + 2 * off)
        self.owned += [t, big]
        return t

    def run(self, cmd, ins, outs):
        l0 = self.nnc.launch_count()
        st = self.nnc.cmd_exec(cmd, None, 0, ins, outs)
        return st, self.nnc.launch_count() - l0

    @staticmethod
    def down(t):
        return np.ascontiguousarray(t.download()).view(np.uint16)

    def free(self):
        for t in reversed(self.owned):
            t.free()
        self.owned = []


def _x(shape, seed, scale=4.0):
    """fp16 bits of normal values"""
    return R.f16_bits(np.random.default_rng(seed).standard_normal(shape, dtype=np.float32) * np.float32(scale))


def _roundtrip(nnc, x, fmt, off_x=0, off_y=0):
    """-> (status forward, launches, compressed bits, status backward, launches, decompressed bits)"""
    d = _Dev(nnc)
    try:
        cshape = R.compressed_shape(x.shape, fmt)
        tx, ty = d.tensor(x.shape, fmt, x, off_x), d.tensor(cshape, fmt, None, off_y)
        tz = d.tensor(x.shape, fmt, None, off_x)
        sf, lf = d.run(nnc.CMD_COMPRESSION_LSSC_FORWARD(), [tx], [ty])
        y = d.down(ty)
        sb, lb = d.run(nnc.CMD_COMPRESSION_LSSC_BACKWARD(), [ty], [tz])
        return sf, lf, y, sb, lb, d.down(tz)
    finally:
        d.free()


def _check(nnc, x, fmt, off_x=0, off_y=0, ref=None):
    sf, lf, y, sb, lb, z = _roundtrip(nnc, x, fmt, off_x, off_y)
    assert (sf, lf, sb, lb) == (0, 1, 0, 1), nnc.lib().ccv_nnc_sm100_last_error()
    want_y = R.forward(x, fmt)
    assert np.array_equal(y, want_y), "forward %s %s: %d halves differ" % (fmt, x.shape, int((y != want_y).sum()))
    want_z = R.backward(want_y, x.shape, fmt)
    assert np.array_equal(z, want_z), "backward %s %s: %d halves differ" % (fmt, x.shape, int((z != want_z).sum()))
    if ref is not None:
        ry, rz = _cpu_ref(ref, x, fmt)
        assert np.array_equal(y, ry) and np.array_equal(z, rz)
    return y, z


def _cpu_ref(ref, x, fmt):
    """CPU_REF (NCHW only) forward and backward; NHWC through the NCHW transpose"""
    from ccv_b200 import nnc
    from tests.util import ref_exec
    NCHW = abi.CCV_TENSOR_FORMAT_NCHW
    perm = None if fmt == R.NCHW else ((0, 3, 1, 2) if x.ndim == 4 else (2, 0, 1))
    xn = np.ascontiguousarray(x if perm is None else x.transpose(perm))
    y = np.zeros(nnc.lssc_compressed_dims(xn.shape, NCHW), np.float16)
    st, (y,) = ref_exec(ref, nnc.CMD_COMPRESSION_LSSC_FORWARD(), None, 0, [xn.view(np.float16)], [y], fmt=NCHW)
    assert st == 0
    z = np.zeros(xn.shape, np.float16)
    st, (z,) = ref_exec(ref, nnc.CMD_COMPRESSION_LSSC_BACKWARD(), None, 0, [y], [z], fmt=NCHW)
    assert st == 0
    y, z = y.view(np.uint16), z.view(np.uint16)
    if perm is not None:
        inv = tuple(np.argsort(perm))
        y, z = np.ascontiguousarray(y.transpose(inv)), np.ascontiguousarray(z.transpose(inv))
    return y, z


# ---- every kernel form ------------------------------------------------------------------------------------------------------------
SIZES = (1, 3, 4, 5, 7, 13, 14)


@pytest.mark.parametrize("fmt", [R.NCHW, R.NHWC])
@pytest.mark.parametrize("H", SIZES)
def test_ragged_shapes_both_formats(gpu, H, fmt):
    """every W of SIZES; NCHW as band runs, NHWC with 16 channels (vectors) and 3 channels (per channel); 3-d and 4-d"""
    for W in SIZES:
        c = 16 if (H + W) % 2 else 3
        shape4 = (2, 3, H, W) if fmt == R.NCHW else (2, H, W, c)
        shape3 = (3, H, W) if fmt == R.NCHW else (H, W, c)
        _check(gpu, _x(shape4, H * 100 + W), fmt)
        _check(gpu, _x(shape3, H * 100 + W + 50), fmt)


@pytest.mark.parametrize("off_x,off_y", [(0, 0), (1, 0), (0, 3), (5, 7), (8, 8)])
@pytest.mark.parametrize("shape", [(4, 8, 13, 14), (2, 5, 7, 8), (1, 3, 4, 1), (2, 2, 9, 33)])
def test_nchw_band_form_aligned_and_misaligned(gpu, ref, shape, off_x, off_y):
    """16-byte copies between scalar heads and tails, whatever W and the bases' alignment"""
    _check(gpu, _x(shape, sum(shape) + off_x), R.NCHW, off_x, off_y, ref)


@pytest.mark.parametrize("off_x,off_y", [(0, 0), (1, 0), (0, 1), (8, 8)])
@pytest.mark.parametrize("shape", [(2, 7, 13, 16), (1, 14, 14, 64), (3, 5, 6, 24), (2, 7, 9, 12), (2, 4, 5, 3)])
def test_nhwc_vector_and_per_channel_forms(gpu, ref, shape, off_x, off_y):
    """C % 8 == 0 with 16-byte aligned bases runs 8 channels per thread; C = 12 or 3, or a base off by 2 bytes, runs per channel"""
    _check(gpu, _x(shape, sum(shape) + 2 * off_x), R.NHWC, off_x, off_y, ref)


def test_nchw_wider_than_a_band_runs_per_block(gpu, ref):
    _check(gpu, _x((1, 2, 6, 2051), 9), R.NCHW, ref=ref)
    _check(gpu, _x((3, 5, 4100), 10), R.NCHW, 1, 0, ref)


def test_special_blocks(gpu, ref):
    """the fixture's blocks (NaN in cell 0 and elsewhere, +-Inf, +-0 ties, subnormal ranges, +-65504), as NCHW planes and as NHWC
    channels, and arbitrary compressed tensors (random and NaN / Inf levels) decoded"""
    from tests.golden.make_lssc_golden import level_pairs, nan_level_pairs, special_blocks
    sp = special_blocks()
    planes = sp.reshape(-1, 4, 4)
    _check(gpu, planes, R.NCHW, ref=ref)
    _check(gpu, np.ascontiguousarray(planes[:, :3, :3]), R.NCHW, ref=ref)
    _check(gpu, np.ascontiguousarray(planes[:40].transpose(1, 2, 0)), R.NHWC, ref=ref)  # 40 channels: vectors
    _check(gpu, np.ascontiguousarray(planes[:, :3, :3].transpose(1, 2, 0)), R.NHWC, ref=ref)  # 42 channels: per channel
    d = _Dev(gpu)
    try:
        for q in (level_pairs(np.random.RandomState(4), 4096), nan_level_pairs()):
            for fmt, cshape, shape in ((R.NCHW, (q.shape[0], 1, 4), (q.shape[0], 4, 4)), (R.NHWC, (1, 4, q.shape[0]), (4, 4, q.shape[0]))):
                y = q.reshape(-1, 1, 4) if fmt == R.NCHW else np.ascontiguousarray(q.reshape(-1, 1, 4).transpose(1, 2, 0))
                ty, tz = d.tensor(cshape, fmt, y), d.tensor(shape, fmt)
                assert d.run(gpu.CMD_COMPRESSION_LSSC_BACKWARD(), [ty], [tz]) == (0, 1)
                assert np.array_equal(d.down(tz), R.backward(y, shape, fmt)), fmt
    finally:
        d.free()


# ---- the reference's int-test shapes and ResNet-50 activations ---------------------------------------------------------------------
INT_SHAPES = [(128, 512, 7, 7), (128, 512, 14, 14), (128, 64, 113, 114), (128, 256, 28, 28)]


@pytest.mark.parametrize("shape", INT_SHAPES)
def test_reference_int_test_shapes(gpu, ref, shape):
    """whole tensors against CPU_REF (in slices of 16 images), the first 4 images against the restatement"""
    x = _x(shape, 11)
    sf, lf, y, sb, lb, z = _roundtrip(gpu, x, R.NCHW)
    assert (sf, lf, sb, lb) == (0, 1, 0, 1)
    assert np.array_equal(y[:4], R.forward(x[:4])) and np.array_equal(z[:4], R.backward(y[:4], x[:4].shape))
    for n in range(0, shape[0], 16):
        ry, rz = _cpu_ref(ref, x[n:n + 16], R.NCHW)
        assert np.array_equal(y[n:n + 16], ry) and np.array_equal(z[n:n + 16], rz), n


RESNET50 = [(4, 112, 112, 64), (4, 56, 56, 64), (4, 56, 56, 256), (4, 28, 28, 128), (4, 28, 28, 512), (4, 14, 14, 256),
            (4, 14, 14, 1024), (4, 7, 7, 512), (4, 7, 7, 2048)]


@pytest.mark.parametrize("shape", RESNET50)
def test_resnet50_activation_shapes_nhwc(gpu, shape):
    x = _x(shape, shape[1] + shape[3])
    _check(gpu, x, R.NHWC)


@pytest.mark.parametrize("shape", [(4, 64, 56, 56), (4, 512, 7, 7)])
def test_resnet50_activation_shapes_nchw(gpu, shape):
    _check(gpu, _x(shape, shape[1]), R.NCHW)


# ---- multi-pair calls and refusals ------------------------------------------------------------------------------------------------
def test_multi_pair_call_mixing_formats(gpu):
    """one launch per pair; backward may carry more inputs than outputs"""
    d = _Dev(gpu)
    try:
        cases = [((2, 3, 7, 13), R.NCHW, 0), ((2, 5, 6, 16), R.NHWC, 0), ((9, 10, 3), R.NHWC, 1), ((4, 5, 5), R.NCHW, 3)]
        xs = [_x(s, i) for i, (s, _, _) in enumerate(cases)]
        tx = [d.tensor(s, f, x, o) for (s, f, o), x in zip(cases, xs)]
        ty = [d.tensor(R.compressed_shape(s, f), f, None, o) for s, f, o in cases]
        assert d.run(gpu.CMD_COMPRESSION_LSSC_FORWARD(), tx, ty) == (0, 4)
        for t, (s, f, _), x in zip(ty, cases, xs):
            assert np.array_equal(d.down(t), R.forward(x, f))
        tz = [d.tensor(s, f, None, o) for s, f, o in cases[:3]]
        assert d.run(gpu.CMD_COMPRESSION_LSSC_BACKWARD(), ty, tz) == (0, 3)
        for t, (s, f, _), x in zip(tz, cases, xs):
            assert np.array_equal(d.down(t), R.backward(R.forward(x, f), s, f))
    finally:
        d.free()


def test_refusals_launch_nothing_and_leave_outputs_untouched(gpu):
    nnc = gpu
    d = _Dev(nnc)
    try:
        shape, cshape = (2, 3, 7, 9), R.compressed_shape((2, 3, 7, 9), R.NCHW)
        x = d.tensor(shape, R.NCHW, _x(shape, 1))
        y = d.tensor(cshape, R.NCHW)
        z = d.tensor(shape, R.NCHW)
        good_y, good_x = d.tensor(cshape, R.NCHW), d.tensor(shape, R.NCHW, _x(shape, 2))
        bf16 = nnc.gpu_tensor(list(shape), abi.CCV_TENSOR_FORMAT_NCHW, abi.CCV_16BF)
        f32 = nnc.gpu_tensor(list(shape), abi.CCV_TENSOR_FORMAT_NCHW, abi.CCV_32F)
        qx = nnc.gpu_palettized_tensor(list(shape), abi.CCV_16F, 4, 126)
        chwn = nnc.gpu_tensor(list(shape), abi.CCV_TENSOR_FORMAT_CHWN, abi.CCV_16F)
        nhwc_y = d.tensor(R.compressed_shape((2, 7, 9, 3), R.NHWC), R.NHWC)
        base = d.tensor((2, 3, 7, 18), R.NCHW)
        strided = nnc.tensor_view_new(base, list(shape), [0] * 12, [3 * 7 * 18, 7 * 18, 18, 1] + [0] * 8)
        flat2 = d.tensor((6 * 7, 9), R.NCHW)
        flat2_y = d.tensor((6 * 7, 12), R.NCHW)
        five = d.tensor((1, 2, 3, 7, 9), R.NCHW)
        five_y = d.tensor((1, 2, 3, 2, 12), R.NCHW)
        wrong_h = d.tensor((2, 3, 3, 12), R.NCHW)
        wrong_w = d.tensor((2, 3, 2, 9), R.NCHW)
        d.owned += [bf16, f32, qx, chwn, strided]
        F, B = nnc.CMD_COMPRESSION_LSSC_FORWARD(), nnc.CMD_COMPRESSION_LSSC_BACKWARD()
        bad = {"bf16": (F, [bf16], [y]), "fp32": (F, [f32], [y]), "palettized": (F, [qx], [y]), "CHWN": (F, [chwn], [y]),
               "formats differ": (F, [x], [nhwc_y]), "non-contiguous view": (F, [strided], [y]), "2-d": (F, [flat2], [flat2_y]),
               "5-d": (F, [five], [five_y]), "compressed H": (F, [x], [wrong_h]), "compressed W": (F, [x], [wrong_w]),
               "NULL input": (F, [None], [y]), "NULL output": (F, [x], [None]), "2 inputs 1 output": (F, [x, good_x], [y]),
               "no operands": (F, [], []), "backward 1 input 2 outputs": (B, [y], [z, good_x]),
               "backward bf16": (B, [y], [bf16]), "backward compressed W": (B, [wrong_w], [z]), "backward view": (B, [y], [strided]),
               "a bad second pair": (F, [good_x, x], [good_y, wrong_h])}
        for name, (cmd, ins, outs) in bad.items():
            assert d.run(cmd, ins, outs) == (INVALID, 0), name
        for t in (y, z, good_y, nhwc_y, wrong_h, wrong_w, flat2_y, five_y):
            assert np.all(d.down(t) == 0x5a5a)
    finally:
        d.free()


# ---- a flat graph: convolution -> LSSC -> LSSC backward -> convolution backward ---------------------------------------------------
def test_graph_fused_and_captured_equals_eager(gpu):
    """the memory-compression pass's shape: the activation a convolution produced is compressed, decompressed just before the
    CONVOLUTION_BACKWARD that reads it.  Run eagerly, then through ccv_nnc_sm100_graph_fuse and a captured CUDA graph: same bits."""
    nnc = gpu
    N, H, W, C, K, K2 = 2, 14, 14, 16, 32, 16
    r = np.random.RandomState(3)
    f16 = lambda a: nnc.gpu_tensor(list(a.shape), abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_16F).upload(pack16(a.astype(np.float32), abi.CCV_16F).view(np.float16))
    x, w, bias = f16(r.randn(N, H, W, C)), f16(r.randn(K, 3, 3, C) / 12), f16(r.randn(K) * 0.1)
    w2, g = f16(r.randn(K2, 3, 3, K) / 17), f16(r.randn(N, H, W, K2))
    z = lambda dims: f16(np.zeros(dims, np.float32))
    y, yc, yd = z((N, H, W, K)), z(nnc.lssc_compressed_dims([N, H, W, K], abi.CCV_TENSOR_FORMAT_NHWC)), z((N, H, W, K))
    h, dw, db = z((N, H, W, K)), z((K2, 3, 3, K)), z((K2,))
    hint = nnc.hint((1, 1), (1, 1))
    nodes = [(nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C), hint, [x, w, bias], [y]),
             (nnc.CMD_COMPRESSION_LSSC_FORWARD(), None, [y], [yc]),
             (nnc.CMD_COMPRESSION_LSSC_BACKWARD(), None, [yc], [yd]),
             (nnc.CMD_CONVOLUTION_BACKWARD(1, K2, 3, 3, K), hint, [g, yd, w2], [h, dw, db])]
    outs = (y, yc, yd, h, dw, db)
    try:
        for cmd, hn, ins, os_ in nodes:
            assert nnc.cmd_exec(cmd, hn, 0, ins, os_) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        eager = [t.download().view(np.uint16).copy() for t in outs]
        assert np.array_equal(eager[1], R.forward(eager[0], R.NHWC))
        assert np.array_equal(eager[2], R.backward(eager[1], (N, H, W, K), R.NHWC))
        stream = nnc.Stream(0)
        graph = nnc.Graph()
        for cmd, hn, ins, os_ in nodes:
            graph.exec_new(cmd, hn, 0, ins, os_)
        graph.fuse()
        for t in outs:
            t.upload(np.zeros(t.count, np.float16))
        assert graph.run(stream) == 0
        stream.wait()
        assert all(np.array_equal(t.download().view(np.uint16), e) for t, e in zip(outs, eager))
        cid = graph.capture(stream)
        for t in outs:
            t.upload(np.zeros(t.count, np.float16))
        assert graph.replay(cid, stream) == 0
        stream.wait()
        for t, e, name in zip(outs, eager, ("y", "compressed", "decompressed", "dgrad", "wgrad", "bias grad")):
            assert np.array_equal(t.download().view(np.uint16), e), name
        graph.free()
        stream.free()
    finally:
        for t in (x, w, bias, w2, g) + outs:
            t.free()


# ---- the reference's own program on the drop-in build -----------------------------------------------------------------------------
def test_reference_compression_program_passes_on_the_dropin_build(gpu, tmp_path):
    from tests.test_dropin import _built, _run
    if not _built(["int.compression"]):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    rep = _run(["int.compression"], 600, tmp_path)
    r = rep["programs"]["int.compression.tests"]
    assert not r["failed"] and not r["crashed"] and r["tally"]["PASS"] == 4 and not r["skipped"], r
