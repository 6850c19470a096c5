"""Graph rewrites (h) and (i) on the device.  (h): the end of a residual block, BATCH_NORM_FORWARD ; EWSUM ; RELU_FORWARD, run as one
pass y = relu(bn(x) + s) must give the bits of the three commands it replaces -- y and all four statistics outputs -- in fp32, bf16
and fp16, on every apply path (the channel-stationary vector kernel ResNet-50's shapes take, the 4-wide kernel, the generic one), with
the batch norm reducing its input itself or reading the statistics its producing convolution's epilogue left (rule (f)).  (i): the
shortcut of a strided block, AVERAGE_POOL_BACKWARD ; EWSUM ; RELU_BACKWARD, as one pass, bit for bit, on the one-pass kernel and on
the fallback for other pool geometries."""
import numpy as np
import pytest

from ccv_b200 import abi
from tests.util import pack16, seeded

pytestmark = pytest.mark.gpu

DTYPES = {"f32": abi.CCV_32F, "bf16": abi.CCV_16BF, "f16": abi.CCV_16F}
# (image side, channels): the four junction shapes of ResNet-50 at 224 x 224, then channel counts that take the 4-wide apply
# kernel (12: C / W does not divide 256) and the generic one (6: not a multiple of 4)
SHAPES = [(56, 256), (28, 512), (14, 1024), (7, 2048), (9, 12), (5, 6)]


def _upload(nnc, a, dt):
    t = nnc.gpu_tensor(list(a.shape), datatype=dt)
    return t.upload(a if dt == abi.CCV_32F else pack16(a, dt))


def _bytes(t):
    return np.ascontiguousarray(t.download()).view(np.uint8).copy()


def _run_junction(nnc, stream, dt, x, short, scale, bias, fuse, conv=None, algorithm=-1):
    """[conv ->] bn -> ewsum(bn output, short) -> relu on fresh tensors; returns the bytes of y and of the four statistics
    outputs, and the fused kinds.  With fuse == "blocked" a trailing node reads the batch norm's output, which keeps rule (h) from
    firing while every other rewrite still applies."""
    N, H, W, C = short.shape
    T = lambda a: _upload(nnc, a, dt)
    F = lambda a: nnc.gpu_tensor(list(a.shape)).upload(a)
    keep = []
    g = nnc.Graph()
    if conv is not None:
        src, w = T(conv[0]), T(conv[1])
        tx = nnc.gpu_tensor([N, H, W, C], datatype=dt)
        g.exec_new(nnc.CMD_CONVOLUTION_FORWARD(1, C, 1, 1, conv[0].shape[-1], algorithm=algorithm), nnc.hint((1, 1), (0, 0)), 0, [src, w], [tx])
        keep += [src, w]
    else:
        tx = T(x)
    ts, tscale, tbias = T(short), F(scale), F(bias)
    mean, var = F(np.zeros((1, 1, 1, C), np.float32)), F(np.ones((1, 1, 1, C), np.float32))
    z, y, junk = (nnc.gpu_tensor([N, H, W, C], datatype=dt) for _ in range(3))
    sm, sis = nnc.gpu_tensor([1, 1, 1, C]), nnc.gpu_tensor([1, 1, 1, C])
    g.exec_new(nnc.CMD_BATCH_NORM_FORWARD(1e-4, 0, 0.9), None, 0, [tx, tscale, tbias, mean, var], [z, mean, var, sm, sis])
    g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [z, ts], [y])
    g.exec_new(nnc.CMD_RELU_FORWARD(), None, 0, [y], [y])
    if fuse == "blocked":
        g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [z, ts], [junk])
    if fuse:
        g.fuse()
    kinds = [(c, k, len(i), len(o)) for c, k, i, o in g.nodes()]
    assert g.run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    out = [_bytes(t) for t in (y, mean, var, sm, sis)]
    if conv is not None:
        # the statistics tensor of a linked convolution says how many partial rows its epilogue produced
        stats = [o[1] for c, k, _, o in g.nodes() if c == abi.CCV_NNC_CONVOLUTION_FORWARD and k == 6]
        out.append(abi.Tensor.from_address(stats[0]).sig if stats else None)
    for t in keep + [tx, ts, tscale, tbias, mean, var, z, y, junk, sm, sis, g]:
        t.free()
    return out, kinds


def _residual_node(kinds):
    # the fused node: a batch norm with the residual addend as a 6th (read-only) output
    return [k for k in kinds if k[0] == abi.CCV_NNC_BATCH_NORM_FORWARD and k[3] == 6]


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("side,C", SHAPES)
def test_fused_junction_matches_the_three_commands_bit_for_bit(gpu, dtype, side, C):
    nnc = gpu
    dt = DTYPES[dtype]
    N = 2
    stream = nnc.Stream(0)
    x = seeded((N, side, side, C), 1, -2, 3)
    short = seeded((N, side, side, C), 2, -1, 1)
    scale, bias = seeded((1, 1, 1, C), 3, 0.5, 1.5), seeded((1, 1, 1, C), 4, -1, 1)
    want, k0 = _run_junction(nnc, stream, dt, x, short, scale, bias, fuse=False)
    got, k1 = _run_junction(nnc, stream, dt, x, short, scale, bias, fuse=True)
    assert len(k0) == 3 and len(k1) == 1 and len(_residual_node(k1)) == 1, k1
    for name, a, b in zip(("y", "running mean", "running var", "saved mean", "saved inv_std"), got, want):
        assert np.array_equal(a, b), "%s differs from the unfused commands" % name
    # the sum is not trivially all-zero or all-positive: the ReLU cut something and let something through
    yv = np.frombuffer(got[0].tobytes(), np.float32 if dt == abi.CCV_32F else np.uint16)
    assert (yv == 0).any() and (yv != 0).any()
    stream.free()


@pytest.mark.parametrize("dtype,algorithm", [("f32", abi.CCV_NNC_SM100_ALGO_TF32), ("f32", abi.CCV_NNC_SM100_ALGO_3XTF32), ("bf16", -1), ("f16", -1)])
@pytest.mark.parametrize("side,C", [(56, 256), (7, 2048)])
def test_fused_junction_reads_the_convolution_statistics(gpu, dtype, algorithm, side, C):
    """conv3 -> bn3 -> sum -> ReLU as in every block: the convolution still hands its epilogue statistics to the batch norm (rule
    (f) on the node rule (h) made), and the result is the bits of the same list with (h) kept from firing."""
    nnc = gpu
    dt = DTYPES[dtype]
    N, Cin = 2, 64
    stream = nnc.Stream(0)
    src = seeded((N, side, side, Cin), 5, -1, 1)
    w = seeded((C, 1, 1, Cin), 6, -1, 1) / Cin ** 0.5
    short = seeded((N, side, side, C), 2, -1, 1)
    scale, bias = seeded((1, 1, 1, C), 3, 0.5, 1.5), seeded((1, 1, 1, C), 4, -1, 1)
    want, k0 = _run_junction(nnc, stream, dt, None, short, scale, bias, fuse="blocked", conv=(src, w), algorithm=algorithm)
    got, k1 = _run_junction(nnc, stream, dt, None, short, scale, bias, fuse=True, conv=(src, w), algorithm=algorithm)
    assert not _residual_node(k0) and len(_residual_node(k1)) == 1, (k0, k1)
    # the convolution still produces the statistics (kind 6) and the fused batch norm reads them (6 inputs, kind 7)
    assert [(k[1], k[2]) for k in k1] == [(6, 2), (7, 6)], k1
    # rows > 0: the batch norm read the epilogue's statistics; 0: that launch path has no statistics epilogue and the batch norm
    # reduced its input itself -- either way the same in both runs
    assert got[5] == want[5], (got[5], want[5])
    for name, a, b in zip(("y", "running mean", "running var", "saved mean", "saved inv_std"), got, want):
        assert np.array_equal(a, b), "%s differs from the list without the residual rewrite" % name
    stream.free()


# (input side, channels, window = stride): the three strided blocks of ResNet-50 at 224 x 224; then a side the 2 x 2 windows do not
# tile (7 = 3 * 2 + 1), which runs the three-step fallback
# and 3 x 3 / 3 windows, where g / 9 is inexact and the 16-bit rounding of the pool gradient before the sum decides bits
POOL_SHAPES = [(56, 256, 2), (28, 512, 2), (14, 1024, 2), (7, 64, 2), (9, 64, 3)]


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("side,C,k", POOL_SHAPES)
def test_fused_pool_junction_matches_the_three_commands_bit_for_bit(gpu, dtype, side, C, k):
    nnc = gpu
    dt = DTYPES[dtype]
    N, P = 2, side // k
    stream = nnc.Stream(0)
    gp = seeded((N, P, P, C), 1, -1, 1)
    gmain = seeded((N, side, side, C), 2, -1, 1)
    y = np.maximum(seeded((N, side, side, C), 3, -1, 1), 0)  # a ReLU output: the mask

    def run(fuse):
        tgp, tmain, ty, ts = _upload(nnc, gp, dt), _upload(nnc, gmain, dt), _upload(nnc, y, dt), nnc.gpu_tensor([N, side, side, C], datatype=dt)
        g = nnc.Graph()
        # as resnet50.Net lays it out: the sum is in place on the main branch's gradient
        g.exec_new(nnc.CMD_AVERAGE_POOL_BACKWARD(k, k), nnc.hint((k, k), (0, 0)), 0, [tgp], [ts])
        g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [tmain, ts], [tmain])
        g.exec_new(nnc.CMD_RELU_BACKWARD(), None, 0, [tmain, None, ty], [tmain])
        if fuse:
            assert g.fuse() == 2 and len(g) == 1
        assert g.run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        out = _bytes(tmain)
        for t in (tgp, tmain, ty, ts, g):
            t.free()
        return out

    want, got = run(False), run(True)
    assert np.array_equal(got, want), "the fused shortcut gradient differs from the three commands"
    stream.free()
