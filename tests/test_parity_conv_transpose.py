"""CONVOLUTION_TRANSPOSE_FORWARD / _BACKWARD on CCV_NNC_BACKEND_GPU_SM100 against a float64 oracle at the rounding-level bounds of
tests/contract_ref.py, against the composition it is built from, and against the reference's CPU_REF.

A transposed convolution y = T(a) (a[N, Hi, Wi, Cin], w[Cin, R, S, Cout / groups], y[N, Ho, Wo, Cout]) is the data gradient of the
"mirrored" convolution that maps y's extent onto a's, plus the bias; pixels of y that no tap reaches hold the bias exactly.  Its
backward is that convolution's forward (da = conv(g, w)) and its weight gradient with the activations swapped (dw = wgrad(grad = a,
x = g)).  K_eff of an output pixel is the number of taps of its residue class that land in range, times Cin / groups."""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from ccv_b200 import abi
from tests import contract_ref as cr
from tests.contract_ref import BF16, FP16, FP32, TF32, X3
from tests.util import assert_close, gpu_exec, gpu_exec16, ref_exec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NHWC, NCHW = abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_TENSOR_FORMAT_NCHW
ALGO = {TF32: abi.CCV_NNC_SM100_ALGO_TF32, X3: abi.CCV_NNC_SM100_ALGO_3XTF32, FP32: abi.CCV_NNC_SM100_ALGO_FFMA, BF16: -1, FP16: -1}
MODES = [TF32, X3, FP32, BF16, FP16]
SENTINEL = {FP32: 0x7FBADBAD, BF16: 0x7FBB, FP16: 0x7DBB}  # NaN patterns


def _kind(mode):
    return {BF16: 1, FP16: 2}.get(mode, 0)


def _out(mode):
    return mode if _kind(mode) else FP32


def _dt(mode):
    return {BF16: abi.CCV_16BF, FP16: abi.CCV_16F}.get(mode, abi.CCV_32F)


# ------------------------------------------------------------------------------------------------ geometry and float64 oracle
def out_extent(Hi, R, stride, pad0, pad1, dil, output_padding):
    """ccv_nnc_hint_tensor_auto of the transposed convolution (cmd/convolution/ccv_nnc_convolution.c:96-101)"""
    return (Hi - 1) * stride + (R - 1) * dil + 1 - pad0 - pad1 + output_padding


class TGeom(object):
    def __init__(self, name, N, Hi, Wi, Cin, Cout, R, S, stride=(1, 1), pad=(0, 0), pad_end=None, dil=(1, 1), output_padding=0, groups=1,
                 bias=1, fmt=NHWC, modes=MODES):
        self.name, self.N, self.Hi, self.Wi, self.Cin, self.Cout, self.R, self.S = name, N, Hi, Wi, Cin, Cout, R, S
        self.st, self.pad, self.dil, self.op, self.groups, self.bias, self.fmt, self.modes = tuple(stride), tuple(pad), tuple(dil), output_padding, groups, bias, fmt, modes
        pe = self.pad if pad_end is None else tuple(pad_end)
        self.pad_end = pe
        self.Ho = out_extent(Hi, R, self.st[0], self.pad[0], pe[0], self.dil[0], output_padding)
        self.Wo = out_extent(Wi, S, self.st[1], self.pad[1], pe[1], self.dil[1], output_padding)

    def __repr__(self):
        return self.name

    def mirror(self):
        """the convolution whose data gradient this is (input = y's extent, output = a's)"""
        return cr.Geom(self.N, self.Ho, self.Wo, self.Cout, self.Cin, self.R, self.S, self.st, self.pad, self.dil, P=self.Hi, Q=self.Wi)

    def hint(self, nnc):
        return nnc.hint(self.st, self.pad, border_end=self.pad_end)

    def taps_1d(self, axis):
        """per output coordinate: number of taps that land on it from an in-range input pixel"""
        n_out, n_in, K = (self.Ho, self.Hi, self.R) if axis == 0 else (self.Wo, self.Wi, self.S)
        st, pad, dil = self.st[axis], self.pad[axis], self.dil[axis]
        c = np.zeros(n_out)
        for i in range(n_in):
            for r in range(K):
                o = i * st - pad + r * dil
                if 0 <= o < n_out:
                    c[o] += 1
        return c

    def keff(self):
        return (self.taps_1d(0)[:, None] * self.taps_1d(1)[None, :] * (self.Cin // self.groups))[:, :, None]

    def shapes(self):
        return dict(a=(self.N, self.Hi, self.Wi, self.Cin), w=(self.Cin, self.R, self.S, self.Cout // self.groups), y=(self.N, self.Ho, self.Wo, self.Cout))


def conv_transpose(g, a, w, bias=None):
    """y[N, Ho, Wo, Cout] = bias + every input pixel scattered through the filter taps (contributions past y's extent dropped)"""
    y = np.zeros((a.shape[0], g.Ho, g.Wo, g.Cout))
    cig, cog = g.Cin // g.groups, g.Cout // g.groups
    for r in range(g.R):
        oh = np.arange(g.Hi) * g.st[0] - g.pad[0] + r * g.dil[0]
        vh = (oh >= 0) & (oh < g.Ho)
        for s in range(g.S):
            ow = np.arange(g.Wi) * g.st[1] - g.pad[1] + s * g.dil[1]
            vw = (ow >= 0) & (ow < g.Wo)
            if not vh.any() or not vw.any():
                continue
            src = a[:, vh][:, :, vw]
            for k in range(g.groups):
                y[:, oh[vh][:, None], ow[vw][None, :], k * cog:(k + 1) * cog] += src[..., k * cig:(k + 1) * cig] @ w[k * cig:(k + 1) * cig, r, s, :]
    return y if bias is None else y + bias


def oracle(g, a, w, bias=None):
    """(y, s): the transposed convolution and its scale on absolute values (float64 operands)"""
    y, s = conv_transpose(g, a, w), conv_transpose(g, np.abs(a), np.abs(w))
    if bias is not None:
        y, s = y + bias, s + np.abs(bias)
    return y, s


def nchw(x):
    return np.ascontiguousarray(np.moveaxis(x, -1, 1)) if x.ndim == 4 else x


def nhwc(x):
    return np.ascontiguousarray(np.moveaxis(x, 1, -1)) if x.ndim == 4 else x


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("g", [
    TGeom("s2", 2, 5, 6, 4, 6, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1),
    TGeom("k2s3", 1, 4, 3, 3, 5, 2, 2, stride=(3, 3)),
    TGeom("dil2", 2, 6, 5, 3, 4, 3, 3, pad=(2, 1), dil=(2, 2)),
    TGeom("s1", 1, 7, 7, 5, 3, 3, 3, pad=(1, 1)),
    TGeom("rgb", 1, 6, 6, 8, 3, 7, 7, stride=(2, 2), pad=(3, 3), pad_end=(2, 2)),
], ids=repr)
def test_oracle_is_the_mirrored_data_gradient_plus_bias(g):
    sh = g.shapes()
    a, w, bias = (cr.operand(sh[k], i, FP32).astype(np.float64) for i, k in enumerate(("a", "w", "y"), 1))
    bias = bias[0, 0, 0]
    h = cr.conv_dgrad(g.mirror(), a, w) + bias
    y = conv_transpose(g, a, w, bias)
    assert y.shape == h.shape == sh["y"]
    np.testing.assert_allclose(y, h, rtol=1e-13, atol=1e-13)
    # pixels no tap reaches hold exactly the bias
    k = np.broadcast_to(g.keff(), y.shape)
    assert np.array_equal(y[k == 0], np.broadcast_to(bias, y.shape)[k == 0])


REF_CASES = [
    TGeom("stride1", 2, 7, 6, 5, 6, 3, 3, pad=(1, 1)),
    TGeom("stride2", 2, 6, 5, 4, 6, 3, 3, stride=(2, 2), pad=(1, 1)),
    TGeom("stride3", 1, 5, 4, 3, 4, 3, 3, stride=(3, 3), pad=(1, 1)),
    TGeom("k2s3_tapless", 2, 4, 5, 4, 3, 2, 2, stride=(3, 3)),
    TGeom("dilation2", 1, 6, 7, 3, 5, 3, 3, pad=(2, 2), dil=(2, 2)),
    TGeom("output_padding1", 2, 5, 5, 4, 4, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1),
    TGeom("groups2", 2, 5, 6, 6, 4, 3, 3, stride=(2, 2), pad=(1, 1), groups=2),
    TGeom("depthwise", 1, 6, 5, 4, 4, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1, groups=4),
    TGeom("nchw", 2, 5, 4, 3, 5, 4, 4, stride=(2, 2), pad=(1, 1), fmt=NCHW),
    TGeom("odd_extents", 1, 7, 3, 5, 7, 5, 3, stride=(2, 3), pad=(2, 1), pad_end=(1, 0)),
]


@pytest.mark.ref
@pytest.mark.parametrize("g", REF_CASES, ids=repr)
def test_oracle_matches_cpu_ref(ref, g):
    from ccv_b200 import nnc
    sh = g.shapes()
    seed = zlib.crc32(g.name.encode()) % 10000
    a, w, bias = cr.operand(sh["a"], seed, FP32), cr.operand(sh["w"], seed + 1, FP32), cr.operand((g.Cout,), seed + 2, FP32)
    cmd = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(g.groups, g.Cout, g.op, g.R, g.S, g.Cin, g.dil, backend=abi.CCV_NNC_BACKEND_CPU_REF)
    if g.fmt == NCHW:
        wn = np.ascontiguousarray(w.transpose(0, 3, 1, 2))  # [Cin, Cout / g, R, S]
        st, (yr,) = ref_exec(ref, cmd, g.hint(nnc), 0, [nchw(a), wn, bias], [np.zeros(nchw(np.zeros(sh["y"])).shape, np.float32)], fmt=NCHW)
        yr = nhwc(yr)
    else:
        st, (yr,) = ref_exec(ref, cmd, g.hint(nnc), 0, [a, w, bias], [np.zeros(sh["y"], np.float32)])
    assert st == 0
    y, s = oracle(g, a.astype(np.float64), w.astype(np.float64), bias.astype(np.float64))
    cr.check(yr, y, s, np.maximum(g.keff(), 1), FP32, FP32, "CPU_REF %s" % g)
    k = np.broadcast_to(g.keff(), y.shape)
    assert np.array_equal(yr[k == 0], np.broadcast_to(bias, y.shape)[k == 0])


def test_factory_fills_the_union_arm_at_the_reference_offsets():
    from ccv_b200 import nnc
    # lib/nnc/ccv_nnc.h:121-126: count, groups, dilation[12], output_padding
    assert abi._ConvolutionTranspose.count.offset == 0 and abi._ConvolutionTranspose.groups.offset == 4
    assert abi._ConvolutionTranspose.dilation.offset == 8 and abi._ConvolutionTranspose.output_padding.offset == 56
    assert abi._CmdUnion.convolution_transpose.offset == 0 and C.sizeof(abi.CmdParam) == 120
    c = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(2, 64, 1, 4, 3, 32, dilation=(2, 3))
    assert c.cmd == 0xd691f78e and nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD(1, 8, 0, 3, 3, 8).cmd == 0xd691f78f
    raw = np.frombuffer(bytes(c.info), np.int32)
    assert list(raw[:3]) == [4, 3, 32]  # size.dim (kh, kw, channels)
    u = raw[12:]
    assert (u[0], u[1], u[2], u[3], u[14]) == (64, 2, 2, 3, 1)
    # count / groups / dilation share their offsets with the convolution arm
    assert (c.info.convolution.count, c.info.convolution.groups, c.info.convolution.dilation[1]) == (64, 2, 3)


def test_both_commands_are_registered_under_gpu_sm100():
    from ccv_b200 import nnc
    nnc.init()
    text = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    for cmd in ("CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD", "CCV_NNC_CONVOLUTION_TRANSPOSE_BACKWARD"):
        assert "X(%s)" % cmd in text
        assert nnc.lib().ccv_nnc_cmd_ok(getattr(abi, cmd), abi.CCV_NNC_BACKEND_GPU_SM100) == 1
        assert nnc.lib().ccv_nnc_cmd_ok(getattr(abi, cmd), abi.CCV_NNC_BACKEND_CPU_REF) == 0
    inc = open(os.path.join(ROOT, "integration", "ccv_nnc_cmd_sm100_init.inc")).read()
    assert "_register_command_CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD_backend_CCV_NNC_BACKEND_GPU_SM100(&(init_map[" in inc


def test_cpu_tensors_get_no_kernel():
    from ccv_b200 import nnc
    nnc.init()
    a, w, y = nnc.cpu_tensor([1, 4, 4, 8]), nnc.cpu_tensor([8, 3, 3, 8]), nnc.cpu_tensor([1, 8, 8, 8])
    try:
        for backend in (abi.CCV_NNC_BACKEND_GPU_SM100, 0):
            cmd = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 8, 1, 3, 3, 8, backend=backend)
            assert nnc.cmd_exec(cmd, nnc.hint((2, 2), (1, 1)), 0, [a, w], [y]) == abi.CCV_NNC_EXEC_NO_KERNEL
    finally:
        for t in (a, w, y):
            t.free()


# ------------------------------------------------------------------------------------------------ GPU: forward at the rounding bound
FWD_CASES = [
    TGeom("unet_2x2s2", 2, 8, 8, 64, 32, 2, 2, stride=(2, 2), bias=1),
    TGeom("dcgan_4x4s2p1", 2, 8, 8, 32, 16, 4, 4, stride=(2, 2), pad=(1, 1), bias=2),
    TGeom("3x3s2p1_op1", 2, 9, 9, 16, 8, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1, bias=0),
    TGeom("rgb_7x7s2", 2, 14, 14, 16, 3, 7, 7, stride=(2, 2), pad=(3, 3), pad_end=(2, 2), bias=1),
    TGeom("2x2s3_tapless", 2, 7, 6, 16, 16, 2, 2, stride=(3, 3), bias=2),
    TGeom("dil2", 2, 9, 9, 16, 24, 3, 3, pad=(2, 2), dil=(2, 2), bias=1),
    TGeom("long_k_1x1", 1, 4, 4, 2048, 64, 1, 1, bias=1),
    TGeom("groups2", 2, 8, 8, 32, 32, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1, groups=2, bias=2),
    TGeom("depthwise", 2, 8, 8, 16, 16, 3, 3, stride=(2, 2), pad=(1, 1), output_padding=1, groups=16, bias=1, modes=[TF32, X3, FP32]),
    TGeom("dcgan_nchw", 2, 8, 8, 32, 16, 4, 4, stride=(2, 2), pad=(1, 1), bias=1, fmt=NCHW),
    TGeom("rgb_nchw", 2, 14, 14, 16, 3, 7, 7, stride=(2, 2), pad=(3, 3), pad_end=(2, 2), bias=2, fmt=NCHW),
    # Cin = 4: the 16-bit kinds take the functional form (the tensor cores need Cin % 8 == 0), staged in NCHW
    TGeom("cin4_nchw", 2, 8, 8, 4, 16, 4, 4, stride=(2, 2), pad=(1, 1), bias=2, fmt=NCHW),
]


def _tensor_core(g, mode):
    """whether the fp32 modes run on the tensor cores (else on the FFMA kernels, which multiply raw fp32 operands)"""
    cig, cog = g.Cin // g.groups, g.Cout // g.groups
    if g.groups > 1:
        return cig % 4 == 0 and cog % 4 == 0 and cig >= 16 and cog >= 16
    return g.Cin % 4 == 0 and g.Cout % 4 == 0


def _seen_mode(g, mode):
    return mode if _kind(mode) or mode == FP32 or _tensor_core(g, mode) else FP32


def operands(g, mode, seed_extra=0):
    sh = g.shapes()
    om = mode if _kind(mode) else FP32
    seed = zlib.crc32(g.name.encode()) % 10000 + seed_extra
    a = cr.operand(sh["a"], seed, om)
    w = cr.operand(sh["w"], seed + 1, om) / np.float32(1 << int(np.log2(g.R * g.S * g.Cin // g.groups)))  # exact scaling: keeps |y| ~ 1
    bias = None
    if g.bias:
        bias = cr.operand((g.Cout,), seed + 2, mode if g.bias == 2 and _kind(mode) else FP32, 0.0, 2.0)
    return a, w, bias


def _bits(a, mode):
    return cr.to_bits16(np.asarray(a, np.float64), mode) if _kind(mode) else np.ascontiguousarray(a, np.float32).view(np.uint32)


def _upload(t, bits, mode):
    t.upload(bits.view(np.float16) if mode == FP16 else bits if mode == BF16 else bits.view(np.float32))


def _values(bits, mode):
    return cr.from_bits16(bits, mode) if _kind(mode) else bits.view(np.float32).astype(np.float64)


class Guarded(object):
    """a dense output tensor at an offset into a sentinel-filled allocation"""

    def __init__(self, nnc, shape, mode, fmt):
        self.mode, self.shape = _out(mode), tuple(shape)
        n, guard = int(np.prod(shape)), 64
        self.host = np.full((n + 2 * guard,), SENTINEL[self.mode], np.uint16 if _kind(mode) else np.uint32)
        self.mask = np.zeros(self.host.shape, bool)
        self.mask[guard:guard + n] = True
        self.base = nnc.gpu_tensor([n + 2 * guard], NHWC, _dt(mode))
        self.t = nnc.gpu_tensor(list(shape), fmt, _dt(mode), ptr=self.base.data_ptr + guard * self.host.itemsize)

    def arm(self):
        _upload(self.base, self.host, self.mode)

    def result(self):
        d = self.base.download()
        got = d.view(np.uint16) if _kind(self.mode) else d.view(np.uint32)
        changed = (got != self.host) & ~self.mask
        assert not changed.any(), "%d guard elements overwritten" % changed.sum()
        return got[self.mask].reshape(self.shape)

    def free(self):
        self.t.free(), self.base.free()


def _input(nnc, x, mode, fmt=NHWC):
    m = _out(mode)
    t = nnc.gpu_tensor(list(x.shape), fmt, _dt(m))
    _upload(t, _bits(x, m), m)
    return t


def _run_forward(nnc, g, mode, a, w, bias):
    """two guarded runs of the forward; returns the output bits (NHWC order)"""
    nc = g.fmt == NCHW
    lay = nchw if nc else (lambda x: x)
    wl = np.ascontiguousarray(w.transpose(0, 3, 1, 2)) if nc else w
    ins = [_input(nnc, lay(a), mode, g.fmt), _input(nnc, wl, mode, g.fmt)]
    if bias is not None:
        ins.append(_input(nnc, bias, mode if g.bias == 2 else FP32))
    yshape = g.shapes()["y"]
    out = Guarded(nnc, nchw(np.zeros(yshape)).shape if nc else yshape, mode, g.fmt)
    kw = dict(algorithm=ALGO[mode]) if ALGO[mode] >= 0 else {}
    cmd = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(g.groups, g.Cout, g.op, g.R, g.S, g.Cin, g.dil, **kw)
    try:
        res = []
        for _ in range(2):
            out.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, g.hint(nnc), 0, ins, [out.t])
            assert st == 0, "%s %s: status %d, %s" % (g, mode, st, nnc.lib().ccv_nnc_sm100_last_error())
            assert nnc.launch_count() > l0
            res.append(out.result())
        assert np.array_equal(res[0], res[1]), "%s %s: two runs differ" % (g, mode)
    finally:
        for t in ins:
            t.free()
        out.free()
    return nhwc(res[0]) if nc else res[0]


FWD_PARAMS = [pytest.param(g, m, id="%s-%s" % (g, m)) for g in FWD_CASES for m in g.modes]


@pytest.mark.gpu
@pytest.mark.parametrize("g,mode", FWD_PARAMS)
def test_forward_at_the_rounding_bound(gpu, g, mode):
    nnc = gpu
    a, w, bias = operands(g, mode)
    bits = _run_forward(nnc, g, mode, a, w, bias)
    sm = _seen_mode(g, mode)
    b64 = None if bias is None else bias.astype(np.float64)
    y, s = oracle(g, cr.seen(a, sm), cr.seen(w, sm), b64)
    keff = g.keff()
    got = _values(bits, _out(mode))
    cr.check(got, y, s, keff, sm, _out(mode), "%s %s" % (g, mode))
    # uncovered pixels: exactly the bias (rounded once to the output type), or zero
    k = np.broadcast_to(keff, y.shape)
    if (k == 0).any():
        want = np.broadcast_to(b64 if b64 is not None else np.zeros(g.Cout), y.shape)[k == 0]
        want = cr.rne16(want, mode) if _kind(mode) else want.astype(np.float32).astype(np.float64)
        assert np.array_equal(got[k == 0], want), "%s %s: uncovered pixels are not the bias" % (g, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("command", ["transpose_forward", "convolution_backward_h"])
def test_large_nchw_functional_form_equals_nhwc(gpu, command):
    """fp16, Cin = 4: the tensor cores decline the data gradient and the widen -> FFMA -> narrow form runs, in fp32 copies of g, w and h
    larger than the split-K scratch (y has 33.5M elements).  NCHW stages its tensors in the same workspace, behind the bound the NCHW layer
    reserves; that bound must count the functional form, or its copies land on the staged tensors.  NCHW must give the NHWC bits."""
    nnc = gpu
    N, Hi, Cin, Cout = 8, 128, 4, 64
    hint = nnc.hint((2, 2), (1, 1))
    r = np.random.RandomState(5)
    a = r.random_sample((N, Hi, Hi, Cin)).astype(np.float32)
    w = (r.random_sample((Cin, 4, 4, Cout)) / 64).astype(np.float32)
    y = np.zeros((N, 2 * Hi, 2 * Hi, Cout), np.float32)
    wn = np.ascontiguousarray(w.transpose(0, 3, 1, 2))
    if command == "transpose_forward":
        cmd = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, Cout, 0, 4, 4, Cin)
        st, (ref,) = gpu_exec16(nnc, cmd, hint, 0, [a, w], [y], abi.CCV_16F)
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        st, (got,) = gpu_exec16(nnc, cmd, hint, 0, [nchw(a), wn], [nchw(y)], abi.CCV_16F, in_fmts=[NCHW, NCHW], out_fmts=[NCHW])
    else:
        cmd = nnc.CMD_CONVOLUTION_BACKWARD(1, Cin, 4, 4, Cout)  # h = the data gradient with a as the incoming gradient
        x = np.zeros_like(y)
        st, (ref,) = gpu_exec16(nnc, cmd, hint, 0, [a, x, w], [y], abi.CCV_16F)
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        x = nchw(x)
        st, (got,) = gpu_exec16(nnc, cmd, hint, 0, [nchw(a), x, wn], [nchw(y)], abi.CCV_16F, in_fmts=[NCHW, NCHW, NCHW], out_fmts=[NCHW])
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.array_equal(nhwc(got).view(np.uint32), ref.view(np.uint32)), "%d elements differ" % (nhwc(got) != ref).sum()


def test_tapless_case_has_uncovered_pixels_and_long_case_splits():
    """the forward matrix holds pixels no tap reaches (they must come out as the bias) and a launch that the planner splits"""
    g = [c for c in FWD_CASES if c.name == "2x2s3_tapless"][0]
    assert (g.keff() == 0).any()
    lk = [c for c in FWD_CASES if c.name == "long_k_1x1"][0]
    m = lk.mirror()
    assert cr.pointwise(m)
    assert cr.plan("dgrad", 0, 132, g=m)["path"] == "split" and cr.plan("dgrad", 1, 132, g=m)["path"] == "split"


# ------------------------------------------------------------------------------------------------ GPU: bit-exact composition
COMPOSE_CASES = [c for c in FWD_CASES if c.name in ("dcgan_4x4s2p1", "2x2s3_tapless", "groups2", "rgb_7x7s2", "long_k_1x1", "dcgan_nchw", "depthwise")]
COMPOSE_PARAMS = [pytest.param(g, m, id="%s-%s" % (g, m)) for g in COMPOSE_CASES for m in g.modes]


def _exec(nnc, mode, cmd, hint, flags, ins, outs, fmt, keep32=()):
    if _kind(mode):
        return gpu_exec16(nnc, cmd, hint, flags, ins, outs, _dt(mode), keep32=keep32, in_fmts=[fmt if x is not None and x.ndim == 4 else NHWC for x in ins],
                          out_fmts=[fmt if x is not None and x.ndim == 4 else NHWC for x in outs])
    return gpu_exec(nnc, cmd, hint, flags, ins, outs, in_fmts=[fmt if x is not None and x.ndim == 4 else NHWC for x in ins],
                    out_fmts=[fmt if x is not None and x.ndim == 4 else NHWC for x in outs])


def _cmds(nnc, g, mode):
    kw = dict(algorithm=ALGO[mode]) if ALGO[mode] >= 0 else {}
    T = lambda f: f(g.groups, g.Cout, g.op, g.R, g.S, g.Cin, g.dil, **kw)
    M = lambda f: f(g.groups, g.Cin, g.R, g.S, g.Cout, g.dil, **kw)  # the mirrored convolution: count = Cin
    return (T(nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD), T(nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD),
            M(nnc.CMD_CONVOLUTION_FORWARD), M(nnc.CMD_CONVOLUTION_BACKWARD))


@pytest.mark.gpu
@pytest.mark.parametrize("g,mode", COMPOSE_PARAMS)
def test_composition_is_bit_exact(gpu, g, mode):
    nnc = gpu
    a, w, _ = operands(g, mode)
    gy = cr.operand(g.shapes()["y"], 7, _out(mode))
    nc = g.fmt == NCHW
    L = nchw if nc else (lambda x: x)
    wl = np.ascontiguousarray(w.transpose(0, 3, 1, 2)) if nc else w
    tf, tb, cf, cb = _cmds(nnc, g, mode)
    hint = g.hint(nnc)
    ysh, ash = L(np.zeros(g.shapes()["y"], np.float32)), L(np.zeros(g.shapes()["a"], np.float32))
    # forward without bias == CONVOLUTION_BACKWARD's h on the mirrored geometry
    st, (y,) = _exec(nnc, mode, tf, hint, 0, [L(a), wl], [ysh.copy()], g.fmt)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (h,) = _exec(nnc, mode, cb, hint, 0, [L(a), ysh.copy(), wl], [ysh.copy()], g.fmt)
    assert st == 0
    assert np.array_equal(y.view(np.uint32), h.view(np.uint32)), "%s %s: forward != mirrored data gradient" % (g, mode)
    # backward (da, dw) == (CONVOLUTION_FORWARD(g, w), CONVOLUTION_BACKWARD's dw with x = g and grad = a)
    st, (da, dw) = _exec(nnc, mode, tb, hint, 0, [L(gy), L(a), wl], [ash.copy(), np.zeros_like(wl)], g.fmt)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (da_c,) = _exec(nnc, mode, cf, hint, 0, [L(gy), wl], [ash.copy()], g.fmt)
    assert st == 0
    st, (_, dw_c) = _exec(nnc, mode, cb, hint, 0, [L(a), L(gy)], [None, np.zeros_like(wl)], g.fmt)
    assert st == 0
    assert np.array_equal(da.view(np.uint32), da_c.view(np.uint32)), "%s %s: da != CONVOLUTION_FORWARD(g, w)" % (g, mode)
    assert np.array_equal(dw.view(np.uint32), dw_c.view(np.uint32)), "%s %s: dw != CONVOLUTION_BACKWARD dw(x = g, grad = a)" % (g, mode)


# ------------------------------------------------------------------------------------------------ GPU: backward against float64
BACK_CASES = [c for c in FWD_CASES if c.name in ("dcgan_4x4s2p1", "2x2s3_tapless", "3x3s2p1_op1", "rgb_7x7s2")]
BACK_PARAMS = [pytest.param(g, m, id="%s-%s" % (g, m)) for g in BACK_CASES for m in (TF32, X3, FP32, BF16)]


@pytest.mark.gpu
@pytest.mark.parametrize("g,mode", BACK_PARAMS)
def test_backward_against_float64(gpu, g, mode):
    nnc = gpu
    a, w, _ = operands(g, mode)
    gy = cr.operand(g.shapes()["y"], 11, _out(mode))
    dw_old = cr.operand(w.shape, 12, _out(mode), -1.0, 1.0)
    db_old = cr.operand((g.Cout,), 13, FP32, -1.0, 1.0)
    _, tb, _, _ = _cmds(nnc, g, mode)
    hint = g.hint(nnc)
    nan_a = np.full(g.shapes()["a"], np.nan, np.float32)
    db_in = db_old.copy()
    st, (da, dw, db) = _exec(nnc, mode, tb, hint, abi.CCV_NNC_ACCUMULATE_OUTPUT, [gy, a, w], [nan_a, dw_old.copy(), db_in], NHWC, keep32=(id(db_in),))
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    sm = mode  # da and dw run on the tensor cores for one group (im2col for 3-channel g), on FFMA for ALGO_FFMA
    m = g.mirror()
    G, A, Wt = cr.seen(gy, sm), cr.seen(a, sm), cr.seen(w, sm)
    # da (overwritten despite ACCUMULATE_OUTPUT) = conv(g, w)
    da_ref, s = cr.with_scale(lambda x, f: cr.conv_fwd(m, x, f), G, Wt)
    cr.check(da, da_ref, s, float(g.R * g.S * g.Cout), sm, _out(mode), "%s %s da" % (g, mode))
    # dw += wgrad(grad = a, x = g); dbias += colsum(g) (fp32 for every kind here)
    old = dw_old.astype(np.float64)
    if _kind(mode) and g.Cout % 8:
        # 16-bit filter gradients of unaligned channels (the im2col GEMM of CONVOLUTION_BACKWARD) round the product to 16 bits, then add
        # the old value and round again: each of the two roundings is held to the bound
        dw_ref, s = cr.with_scale(lambda gr, x: cr.conv_wgrad(m, gr, x), A, G)
        e = cr.bound(s, float(g.N * g.Hi * g.Wi), mode)
        lo, hi = cr.rne16(old + cr.rne16(dw_ref - e, mode), mode), cr.rne16(old + cr.rne16(dw_ref + e, mode), mode)
        assert ((lo <= dw) & (dw <= hi)).all(), "%s %s dw: %d elements outside the twice-rounded bound" % (g, mode, (~((lo <= dw) & (dw <= hi))).sum())
    else:
        dw_ref, s = cr.with_scale(lambda gr, x: cr.conv_wgrad(m, gr, x), A, G, old=old)
        cr.check(dw, dw_ref, s, float(g.N * g.Hi * g.Wi), sm, _out(mode), "%s %s dw" % (g, mode))
    gf = np.asarray(gy, np.float64).reshape(-1, g.Cout)
    db_ref, s = gf.sum(0) + db_old, np.abs(gf).sum(0) + np.abs(db_old)
    cr.check(db, db_ref, s, float(gf.shape[0]), FP32, FP32, "%s %s dbias" % (g, mode))
    # the adjoint identity <T(a), g> = <a, T^T(g)> on the device results, to the accumulated rounding of both sides
    st, (y,) = _exec(nnc, mode, _cmds(nnc, g, mode)[0], hint, 0, [a, w], [np.zeros(g.shapes()["y"], np.float32)], NHWC)
    assert st == 0
    lhs, rhs = float(np.sum(np.float64(y) * gy)), float(np.sum(np.float64(a) * da))
    scale = float(np.sum(np.abs(np.float64(y) * gy)) + np.sum(np.abs(np.float64(a) * da)))
    tol = {FP32: 1e-5, X3: 1e-5, TF32: 2e-3, BF16: 2e-2}[mode]
    assert abs(lhs - rhs) <= tol * scale, "%s %s: <T a, g> = %r, <a, T^T g> = %r" % (g, mode, lhs, rhs)
    # da-only and dw-only calls give the same bits as the full call
    st, (da1,) = _exec(nnc, mode, tb, hint, 0, [gy, None, w], [nan_a.copy()], NHWC)
    assert st == 0 and np.array_equal(da1.view(np.uint32), da.view(np.uint32))
    st, (_, dw1) = _exec(nnc, mode, tb, hint, abi.CCV_NNC_ACCUMULATE_OUTPUT, [gy, a], [None, dw_old.copy()], NHWC)
    assert st == 0 and np.array_equal(dw1.view(np.uint32), dw.view(np.uint32))


# ------------------------------------------------------------------------------------------------ GPU: the reference's own shapes against CPU_REF
@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("variant", ["nhwc", "nchw", "half"])
def test_reference_shapes_against_cpu_ref(gpu, ref, variant):
    """test/int/nnc/cudnn.tests.c:5338-5500 at batch 2: a [N, 112, 112, 96] -> y [N, 224, 224, 3], 7 x 7 filters, hint_auto's stride 2 and
    border (3, 2), bias i / 3; tolerances 2e-4 (fp32) and 5e-3 (half)"""
    nnc = gpu
    N, g = 2, TGeom("ref", 2, 112, 112, 96, 3, 7, 7, stride=(2, 2), pad=(3, 3), pad_end=(2, 2))
    r = np.random.RandomState(0)
    w = (r.random_sample((96, 7, 7, 3)) / (3 * 49)).astype(np.float32)
    a = r.random_sample((N, 112, 112, 96)).astype(np.float32)
    bias = (np.arange(3) / 3.0).astype(np.float32)
    hint = g.hint(nnc)
    yz = np.zeros((N, 224, 224, 3), np.float32)
    cmd_ref = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 3, 0, 7, 7, 96, backend=abi.CCV_NNC_BACKEND_CPU_REF)
    cmd = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 3, 0, 7, 7, 96)
    if variant == "nchw":
        wn = np.ascontiguousarray(w.transpose(0, 3, 1, 2))
        _, (yr,) = ref_exec(ref, cmd_ref, hint, 0, [nchw(a), wn, bias], [nchw(yz)], fmt=NCHW)
        st, (y,) = gpu_exec(nnc, cmd, hint, 0, [nchw(a), wn, bias], [nchw(yz)], in_fmts=[NCHW, NCHW, NHWC], out_fmts=[NCHW])
        tol = 2e-4
    elif variant == "half":
        # the reference rounds a, w and bias to half and compares with CPU_REF on the rounded values
        a, w, bias = (x.astype(np.float16).astype(np.float32) for x in (a, w, bias))
        _, (yr,) = ref_exec(ref, cmd_ref, hint, 0, [a, w, bias], [yz.copy()])
        st, (y,) = gpu_exec16(nnc, cmd, hint, 0, [a, w, bias], [yz.copy()], abi.CCV_16F)
        tol = 5e-3
    else:
        _, (yr,) = ref_exec(ref, cmd_ref, hint, 0, [a, w, bias], [yz.copy()])
        st, (y,) = gpu_exec(nnc, cmd, hint, 0, [a, w, bias], [yz.copy()])
        tol = 2e-4
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert_close(y, yr, tol, "reference shape %s" % variant)


@pytest.fixture(scope="module")
def dropin_report(gpu, tmp_path_factory):
    """int.cudnn's three transposed-convolution cases (test/int/nnc/cudnn.tests.c:5338-5500) run on the drop-in build"""
    build = os.path.join(ROOT, "integration", "_build")
    if not os.path.exists(os.path.join(build, "libccv_dropin.so")) or not os.path.exists(os.path.join(build, "int.cudnn.tests")):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    out = str(tmp_path_factory.mktemp("dropin") / "report.json")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_reference_tests.py"), "--only", "int.cudnn", "--match", "convolution transpose",
                        "--budget-s", "300", "--case-timeout", "120", "--out", out], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=420)
    assert p.returncode == 0, p.stdout.decode()[-2000:]
    import json
    rep = json.load(open(out))["programs"]["int.cudnn.tests"]
    assert not rep["crashed"], rep
    return rep


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cudnn forward convolution transpose", "cudnn forward convolution transpose in half precision",
                                  pytest.param("cudnn forward convolution transpose in nchw format", marks=pytest.mark.xfail(strict=False, reason=(
                                      "open: the case holds each fp32 output (about 3.4, a sum of some 1,500 positive products) to 1e-5 absolute, about the "
                                      "difference between two fp32 summation orders of such a sum (on an H100 80GB HBM3: 3.41631 against CPU_REF's 3.41632); "
                                      "the same shape in NCHW is held to 2e-4 against CPU_REF in test_reference_shapes_against_cpu_ref")))])
def test_reference_program_case_passes_on_the_dropin_build(dropin_report, case):
    assert case in dropin_report["passed"], dropin_report.get("fail_detail", {}).get(case, dropin_report)


# ------------------------------------------------------------------------------------------------ GPU: refusals
@pytest.mark.gpu
def test_mismatched_filter_or_count_is_invalid(gpu):
    nnc = gpu
    hint = nnc.hint((2, 2), (1, 1))
    a, y = np.ones((1, 4, 4, 8), np.float32), np.zeros((1, 8, 8, 16), np.float32)
    good = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 16, 0, 4, 4, 8)
    st, _ = gpu_exec(nnc, good, hint, 0, [a, np.ones((8, 4, 4, 16), np.float32)], [y.copy()])
    assert st == 0
    for cmd, w in ((good, np.ones((8, 4, 4, 12), np.float32)),                                      # filter's Cout != count
                   (good, np.ones((6, 4, 4, 16), np.float32)),                                      # filter's Cin != a's channels
                   (nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 12, 0, 4, 4, 8), np.ones((8, 4, 4, 12), np.float32)),  # count != y's channels
                   (nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, 16, 0, 3, 3, 8), np.ones((8, 4, 4, 16), np.float32))):  # size != filter
        st, _ = gpu_exec(nnc, cmd, hint, 0, [a, w], [y.copy()])
        assert st == abi.CCV_NNC_EXEC_INVALID
    st, _ = gpu_exec(nnc, nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD(1, 16, 0, 4, 4, 8), hint, 0, [y, a, np.ones((8, 4, 4, 12), np.float32)],
                     [np.zeros_like(a), np.zeros((8, 4, 4, 12), np.float32)])
    assert st == abi.CCV_NNC_EXEC_INVALID
