"""bf16 / fp16 grouped convolutions whose groups the tensor cores do not take (depthwise, channel multipliers, C / groups or K / groups
below 16 or unaligned, tensors past 2^31 elements) on the direct CUDA-core kernels of ccv_b200/csrc/sm100_conv_grouped.cu, held to the
16-bit rounding bound of tests/contract_ref.py against a grouped float64 oracle.

Output channel k = i Kg + j reads input channels [i Cg, (i + 1) Cg) through filters w[K, R, S, Cg] (the reference's CPU_REF,
convolution/ccv_nnc_conv_cpu_ref.c:47-65).  K_eff of an element is the number of terms of its reduction: the in-range taps of its window
times Cg (forward), the in-range taps of the input pixel's residue class times Kg (data gradient), N P Q (weight gradient)."""
import zlib

import numpy as np
import pytest

from ccv_b200 import abi
from tests import contract_ref as cr
from tests import palette_ref as pr
from tests.contract_ref import BF16, FP16, FP32
from tests.util import gpu_exec16, ref_exec

NHWC, NCHW = abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_TENSOR_FORMAT_NCHW
MODES = [BF16, FP16]
DT = {BF16: abi.CCV_16BF, FP16: abi.CCV_16F, FP32: abi.CCV_32F}
SENTINEL = {BF16: 0x7FBB, FP16: 0x7DBB, FP32: 0x7FBADBAD}  # NaN patterns


class Case(object):
    def __init__(self, name, N, H, W, C, K, groups, R, S, stride=(1, 1), pad=(0, 0), pad_end=None, dil=(1, 1)):
        self.name, self.groups = name, groups
        self.g = cr.Geom(N, H, W, C, K, R, S, stride, pad, dil, pad_end=pad_end)
        self.Cg, self.Kg = C // groups, K // groups

    def __repr__(self):
        return self.name

    def hint(self, nnc):
        return nnc.hint(self.g.st, self.g.pad, border_end=self.g.pad_end)

    def shapes(self):
        g = self.g
        return dict(x=(g.N, g.H, g.W, g.C), w=(g.K, g.R, g.S, self.Cg), y=(g.N, g.P, g.Q, g.K))

    def fwd_cmd(self, nnc, **kw):
        return nnc.CMD_CONVOLUTION_FORWARD(self.groups, self.g.K, self.g.R, self.g.S, self.Cg, self.g.dil, **kw)

    def back_cmd(self, nnc, **kw):
        return nnc.CMD_CONVOLUTION_BACKWARD(self.groups, self.g.K, self.g.R, self.g.S, self.Cg, self.g.dil, **kw)


CASES = [
    Case("dw3x3_s1", 2, 9, 9, 16, 16, 16, 3, 3, pad=(1, 1)),
    Case("dw3x3_s2", 2, 10, 9, 16, 16, 16, 3, 3, stride=(2, 2), pad=(1, 1)),
    Case("dw5x5_s2", 1, 11, 11, 8, 8, 8, 5, 5, stride=(2, 2), pad=(2, 2)),
    Case("dw7x7_p3", 1, 9, 8, 8, 8, 8, 7, 7, pad=(3, 3)),
    Case("multiplier2", 2, 7, 7, 8, 16, 8, 3, 3, pad=(1, 1)),
    Case("cg4_kg4", 2, 8, 8, 16, 16, 4, 3, 3, pad=(1, 1)),
    Case("cg4_kg8", 1, 9, 9, 16, 32, 4, 3, 3, stride=(2, 2), pad=(1, 1)),
    Case("dil2", 1, 10, 9, 8, 8, 8, 3, 3, pad=(2, 2), dil=(2, 2)),
    Case("odd_extents", 1, 7, 5, 8, 8, 8, 3, 3, stride=(2, 2), pad=(1, 0), pad_end=(0, 1)),
    Case("dw3x3_npq4608", 8, 24, 24, 8, 8, 8, 3, 3, pad=(1, 1)),  # a weight gradient of several pixel chunks
]
GPU_CASES = CASES + [
    Case("cg20_unaligned", 2, 8, 7, 40, 40, 2, 3, 3, pad=(1, 1)),
    Case("c12_depthwise_scalar", 3, 9, 11, 12, 12, 12, 3, 3, stride=(2, 2), pad=(1, 1)),
    Case("c12_scalar_npq3600", 4, 30, 30, 12, 12, 12, 3, 3, pad=(1, 1)),  # the scalar weight gradient over several chunks
    Case("effnet_b0_k5s2_n8", 8, 56, 56, 144, 144, 144, 5, 5, stride=(2, 2), pad=(2, 2)),
]


def _seed(case, extra=0):
    return zlib.crc32(case.name.encode()) % 10000 + extra


# ------------------------------------------------------------------------------------------------ grouped float64 oracle
def _slices(case, i):
    return slice(i * case.Cg, (i + 1) * case.Cg), slice(i * case.Kg, (i + 1) * case.Kg)


def gconv_fwd(case, x, w, taps=None, channel_base=None):
    """y = conv(x, w) group by group; channel_base(k0) replaces the group's first input channel (a defect)"""
    g, out = case.g, []
    for i in range(case.groups):
        cs, ks = _slices(case, i)
        if channel_base is not None:
            out.append(np.concatenate([cr.conv_fwd(g, x[..., channel_base(k):channel_base(k) + case.Cg], w[k:k + 1], taps=taps) for k in range(ks.start, ks.stop)], -1))
        else:
            out.append(cr.conv_fwd(g, x[..., cs], w[ks], taps=taps))
    return np.concatenate(out, -1)


def gconv_dgrad(case, gy, w, taps=None):
    g = case.g
    return np.concatenate([cr.conv_dgrad(g, gy[..., _slices(case, i)[1]], w[_slices(case, i)[1]], taps=taps) for i in range(case.groups)], -1)


def gconv_dgrad_extra_tap(case, gy, w):
    """a data gradient that also gathers one tap outside the pixel's residue class (floor division without the divisibility test), or
    for stride 1 the border tap of a clamped window"""
    g = case.g
    h = gconv_dgrad(case, gy, w)
    N, H, W = g.N, g.H, g.W
    for hh in range(H):
        for ww in range(W):
            extra = None
            for r in range(g.R):
                for s in range(g.S):
                    hn, wn = hh + g.pad[0] - r * g.dil[0], ww + g.pad[1] - s * g.dil[1]
                    if hn < 0 or wn < 0:
                        continue
                    if hn % g.st[0] or wn % g.st[1] or hn // g.st[0] >= g.P or wn // g.st[1] >= g.Q:
                        extra = (r, s, min(hn // g.st[0], g.P - 1), min(wn // g.st[1], g.Q - 1))
                        break
                if extra:
                    break
            if extra:
                r, s, p, q = extra
                for i in range(case.groups):
                    cs, ks = _slices(case, i)
                    h[:, hh, ww, cs] += gy[:, p, q, ks] @ w[ks, r, s, :]
    return h


def gconv_wgrad(case, gy, x, rows=None):
    g = case.g
    return np.concatenate([cr.conv_wgrad(g, gy[..., _slices(case, i)[1]], x[..., _slices(case, i)[0]], rows=rows) for i in range(case.groups)], 0)


def keff_fwd(case):
    g = case.g
    th = np.array([sum(0 <= p * g.st[0] - g.pad[0] + r * g.dil[0] < g.H for r in range(g.R)) for p in range(g.P)], np.float64)
    tw = np.array([sum(0 <= q * g.st[1] - g.pad[1] + s * g.dil[1] < g.W for s in range(g.S)) for q in range(g.Q)], np.float64)
    return (th[:, None] * tw[None, :] * case.Cg)[:, :, None]


def keff_dgrad(case):
    g = case.g

    def taps(n, pad, dil, st, lim, R):
        return np.array([sum((i + pad - r * dil) >= 0 and (i + pad - r * dil) % st == 0 and (i + pad - r * dil) // st < lim for r in range(R)) for i in range(n)], np.float64)
    th, tw = taps(g.H, g.pad[0], g.dil[0], g.st[0], g.P, g.R), taps(g.W, g.pad[1], g.dil[1], g.st[1], g.Q, g.S)
    return (th[:, None] * tw[None, :] * case.Kg)[:, :, None]


def wgrad_plan(case):
    """(chunk, splits): the pixels one CTA of the weight gradient sums and their number (wgrad_plan in sm100_conv_grouped.cu, for
    filters whose slices fit the scratch)"""
    g = case.g
    npq, elems = g.N * g.P * g.Q, g.K * g.R * g.S * case.Cg
    units = elems // 8 if case.groups == g.C == g.K and g.C % 8 == 0 else elems
    ctas_x = -(-units // 256)
    splits = max(1, min(-(-2048 // ctas_x), 512, -(-npq // 512)))
    chunk = -(-npq // splits)
    return chunk, -(-npq // chunk)


def operands(case, mode):
    sh, seed = case.shapes(), _seed(case)
    x = cr.operand(sh["x"], seed, mode)
    # scaled to keep |y| ~ 1; back on the 16-bit grid, since the scaling makes some fp16 values subnormal
    w = cr.operand(sh["w"], seed + 1, mode) / np.float32(1 << int(np.log2(case.g.R * case.g.S * case.Cg)))
    w = cr.rne16(w, mode).astype(np.float32)
    gy = cr.operand(sh["y"], seed + 2, mode)
    return x, w, gy


def _admits_all(y, ref, s, keff, mode):
    return bool(cr.admits(y, ref, s, keff, mode, mode).all())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_grouped_oracle_is_the_per_channel_sum(case):
    """the per-group slices of the oracle are the plain definition: output channel k reads input channels k / Kg * Cg + [0, Cg)"""
    x, w, gy = (a.astype(np.float64) for a in operands(case, BF16))
    g = case.g
    y = gconv_fwd(case, x, w)
    xp = g.pad_input(x)
    k = case.g.K - 1
    c0 = k // case.Kg * case.Cg
    want = sum(xp[:, g._win(r, s)[0], g._win(r, s)[1], c0:c0 + case.Cg] @ w[k, r, s] for r, s in g.taps())
    np.testing.assert_allclose(y[..., k], want, rtol=1e-13, atol=1e-13)
    # the adjoint identities tie the three products together
    h, dw = gconv_dgrad(case, gy, w), gconv_wgrad(case, gy, x)
    np.testing.assert_allclose(np.sum(y * gy), np.sum(x * h), rtol=1e-11)
    np.testing.assert_allclose(np.sum(y * gy), np.sum(w * dw), rtol=1e-11)


@pytest.mark.ref
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_oracle_matches_cpu_ref(ref, case):
    """CPU_REF's grouped NHWC forward and backward on fp32 inputs holding 16-bit values, held to the fp32 bound of the oracle"""
    from ccv_b200 import nnc
    x, w, gy = operands(case, BF16)
    bias = cr.operand((case.g.K,), _seed(case, 3), BF16, 0.0, 2.0)
    sh = case.shapes()
    R = abi.CCV_NNC_BACKEND_CPU_REF
    st, (y,) = ref_exec(ref, case.fwd_cmd(nnc, backend=R), case.hint(nnc), 0, [x, w, bias], [np.zeros(sh["y"], np.float32)])
    assert st == 0
    X, Wt, G = (a.astype(np.float64) for a in (x, w, gy))
    want, s = cr.with_scale(lambda a, f: gconv_fwd(case, a, f), X, Wt, bias=bias.astype(np.float64))
    cr.check(y, want, s, np.maximum(keff_fwd(case), 1), FP32, FP32, "CPU_REF forward %s" % case)
    st, (h, dw, db) = ref_exec(ref, case.back_cmd(nnc, backend=R), case.hint(nnc), 0, [gy, x, w],
                               [np.zeros(sh["x"], np.float32), np.zeros(sh["w"], np.float32), np.zeros(case.g.K, np.float32)])
    assert st == 0
    want, s = cr.with_scale(lambda a, f: gconv_dgrad(case, a, f), G, Wt)
    cr.check(h, want, s, np.maximum(keff_dgrad(case), 1), FP32, FP32, "CPU_REF data gradient %s" % case)
    want, s = cr.with_scale(lambda a, b: gconv_wgrad(case, a, b), G, X)
    cr.check(dw, want, s, float(case.g.N * case.g.P * case.g.Q), FP32, FP32, "CPU_REF weight gradient %s" % case)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_bound_rejects_defects(case, mode):
    """the 16-bit bound (c = C_ACC) admits the correctly rounded oracle and rejects each defect a direct kernel could have"""
    x, w, gy = (a.astype(np.float64) for a in operands(case, mode))
    bias = cr.operand((case.g.K,), _seed(case, 3), mode, 0.0, 2.0).astype(np.float64)
    old = cr.operand(case.shapes()["w"], _seed(case, 4), mode, -1.0, 1.0).astype(np.float64)
    g = case.g
    rnd = lambda v: cr.rne16(v, mode)
    # forward
    y, s = cr.with_scale(lambda a, f: gconv_fwd(case, a, f), x, w, bias=bias)
    kf = keff_fwd(case)
    assert _admits_all(rnd(y), y, s, kf, mode)
    defects = {
        "dropped tap": gconv_fwd(case, x, w, taps=g.taps()[:-1]) + bias,
        "truncated": cr.trunc16(y, mode),
        "bias twice": y + bias,
    }
    if case.Cg > 1 or case.Kg > 1:  # (depthwise with multiplier 1 reads channel k either way)
        defects["channel k instead of k / Kg * Cg"] = gconv_fwd(case, x, w, channel_base=lambda k: min(k, g.C - case.Cg)) + bias
    for what, v in defects.items():
        assert not _admits_all(rnd(v) if what != "truncated" else v, y, s, kf, mode), "forward: %s admitted" % what
    # data gradient
    h, s = cr.with_scale(lambda a, f: gconv_dgrad(case, a, f), gy, w)
    kd = keff_dgrad(case)
    assert _admits_all(rnd(h), h, s, kd, mode)
    for what, v in (("dropped residue-class tap", gconv_dgrad(case, gy, w, taps=g.taps()[1:])), ("extra residue-class tap", gconv_dgrad_extra_tap(case, gy, w)),
                    ("truncated", cr.trunc16(h, mode))):
        assert not _admits_all(rnd(v) if what != "truncated" else v, h, s, kd, mode), "data gradient: %s admitted" % what
    # weight gradient, accumulating into an old value
    npq = g.N * g.P * g.Q
    dw, s = cr.with_scale(lambda a, b: gconv_wgrad(case, a, b), gy, x, old=old)
    assert _admits_all(rnd(dw), dw, s, float(npq), mode)
    # the last of the plan's chunks; where the plan makes one chunk, the last quarter of the pixels (a kernel with smaller chunks)
    chunk, splits = wgrad_plan(case)
    if splits == 1:
        chunk = max(1, npq // 4)
    kept = np.arange(npq) < (npq - 1) // chunk * chunk
    for what, v in (("dropped pixel chunk", gconv_wgrad(case, gy, x, rows=kept) + old), ("ignored old dw", dw - old), ("truncated", cr.trunc16(dw, mode))):
        assert not _admits_all(rnd(v) if what != "truncated" else v, dw, s, float(npq), mode), "weight gradient: %s admitted" % what


def test_weight_gradient_plans_several_chunks():
    """the cases the chunk defect and the GPU runs rely on: the vector and the scalar weight gradient over several pixel chunks, and a
    112 x 112 depthwise layer whose ordered combine adds a few hundred slices, not thousands"""
    by = {c.name: c for c in GPU_CASES}
    assert wgrad_plan(by["dw3x3_npq4608"])[1] > 1 and wgrad_plan(by["c12_scalar_npq3600"])[1] > 1 and wgrad_plan(by["effnet_b0_k5s2_n8"])[1] > 1
    assert wgrad_plan(Case("b1", 128, 112, 112, 32, 32, 32, 3, 3, pad=(1, 1)))[1] <= 512


# ------------------------------------------------------------------------------------------------ GPU helpers
def _bits(a, mode):
    return cr.to_bits16(np.asarray(a, np.float64), mode) if mode != FP32 else np.ascontiguousarray(a, np.float32).view(np.uint32)


def _upload(t, bits, mode):
    t.upload(bits.view(np.float16) if mode == FP16 else bits if mode == BF16 else bits.view(np.float32))


def _values(bits, mode):
    return cr.from_bits16(bits, mode) if mode != FP32 else bits.view(np.float32).astype(np.float64)


class Pitched(object):
    """an NHWC tensor (or a view with channel pitch C + pad) inside a sentinel-filled allocation with guards on both sides; inputs carry
    their values in the view's channels and the sentinel everywhere else"""

    def __init__(self, nnc, shape, mode, pad=0, values=None, guard=64):
        self.mode, self.shape, self.pad = mode, tuple(shape), pad
        full = self.shape[:-1] + (self.shape[-1] + pad,)
        n = int(np.prod(full))
        self.host = np.full((n + 2 * guard,), SENTINEL[mode], np.uint16 if mode != FP32 else np.uint32)
        inner = self.host[guard:guard + n].reshape(full)
        if values is not None:
            inner[..., pad:] = _bits(values, mode)
        self.mask = np.zeros(self.host.shape, bool)
        self.mask[guard:guard + n].reshape(full)[..., pad:] = True
        self.base = nnc.gpu_tensor([n + 2 * guard], NHWC, DT[mode])
        ptr = self.base.data_ptr + guard * self.host.itemsize
        if pad:
            self.dense = nnc.gpu_tensor(list(full), NHWC, DT[mode], ptr=ptr)
            stride = [int(np.prod(full[i + 1:])) for i in range(len(full))]
            self.t = nnc.tensor_view_new(self.dense, list(self.shape), [0] * (len(full) - 1) + [pad], stride)
        else:
            self.dense, self.t = None, nnc.gpu_tensor(list(self.shape), NHWC, DT[mode], ptr=ptr)
        self.arm()

    def arm(self):
        _upload(self.base, self.host, self.mode)

    def result(self):
        d = self.base.download()
        got = d.view(np.uint16) if self.mode != FP32 else d.view(np.uint32)
        changed = (got != self.host) & ~self.mask
        assert not changed.any(), "%d elements outside the tensor overwritten" % changed.sum()
        return _values(got[self.mask].reshape(self.shape), self.mode)

    def free(self):
        self.t.free()
        if self.dense is not None:
            self.dense.free()
        self.base.free()


def _run_twice(nnc, cmd, hint, flags, ins, outs, launches, what):
    """two runs on re-armed outputs: status 0, the declared launch count, the same bits; returns the outputs' values"""
    res = []
    for _ in range(2):
        for o in outs:
            if o is not None:
                o.arm()
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(cmd, hint, flags, [None if i is None else i.t for i in ins], [None if o is None else o.t for o in outs])
        assert st == 0, "%s: status %d, %s" % (what, st, nnc.lib().ccv_nnc_sm100_last_error())
        n = nnc.launch_count() - l0
        assert n == launches, "%s: %d launches, declared %d" % (what, n, launches)
        res.append([None if o is None else o.result() for o in outs])
    for a, b in zip(*res):
        if a is not None:
            assert np.array_equal(a, b, equal_nan=True), "%s: two runs differ" % what
    return res[0]


def _free(*ts):
    for t in ts:
        if t is not None:
            t.free()


GPU_PARAMS = [pytest.param(c, m, id="%s-%s" % (c, m)) for c in GPU_CASES for m in MODES]


# ------------------------------------------------------------------------------------------------ GPU: forward at the rounding bound
@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", GPU_PARAMS)
def test_forward_at_the_rounding_bound(gpu, case, mode):
    nnc = gpu
    x, w, _ = operands(case, mode)
    sh, g = case.shapes(), case.g
    X, Wt = x.astype(np.float64), w.astype(np.float64)
    kf = keff_fwd(case)
    for bias_mode in (FP32, mode, None):
        bias = None if bias_mode is None else cr.operand((g.K,), _seed(case, 3), bias_mode, 0.0, 2.0)
        pad = 8 if bias_mode == mode else 0  # pitched views of x and y
        xt, wt = Pitched(nnc, sh["x"], mode, pad, x, 0), Pitched(nnc, sh["w"], mode, 0, w, 0)
        bt = None if bias is None else Pitched(nnc, (g.K,), bias_mode, 0, bias, 0)
        yt = Pitched(nnc, sh["y"], mode, pad)
        try:
            what = "%s %s forward, bias %s, pitch +%d" % (case, mode, bias_mode, pad)
            (y,) = _run_twice(nnc, case.fwd_cmd(nnc), case.hint(nnc), 0, [xt, wt] + ([bt] if bt else []), [yt], 1, what)
        finally:
            _free(xt, wt, bt, yt)
        b64 = None if bias is None else bias.astype(np.float64)
        want, s = cr.with_scale(lambda a, f: gconv_fwd(case, a, f), X, Wt, bias=b64)
        cr.check(y, want, s, kf, mode, mode, what)
        k = np.broadcast_to(kf, want.shape)
        if (k == 0).any():  # windows wholly in the padding: rne(0 + bias)
            assert np.array_equal(y[k == 0], cr.rne16(np.broadcast_to(b64 if b64 is not None else 0.0, want.shape)[k == 0], mode))


# ------------------------------------------------------------------------------------------------ GPU: backward at the rounding bound
@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", GPU_PARAMS)
def test_backward_at_the_rounding_bound(gpu, case, mode):
    nnc = gpu
    x, w, gy = operands(case, mode)
    sh, g = case.shapes(), case.g
    X, Wt, G = x.astype(np.float64), w.astype(np.float64), gy.astype(np.float64)
    npq = float(g.N * g.P * g.Q)
    hint, cmd = case.hint(nnc), case.back_cmd(nnc)
    h_ref, h_s = cr.with_scale(lambda a, f: gconv_dgrad(case, a, f), G, Wt)
    dw_ref, dw_s = cr.with_scale(lambda a, b: gconv_wgrad(case, a, b), G, X)
    kd = keff_dgrad(case)
    colsum_launches = 1 if g.K % 4 else 2
    gt, xt, wt = Pitched(nnc, sh["y"], mode, 0, gy, 0), Pitched(nnc, sh["x"], mode, 0, x, 0), Pitched(nnc, sh["w"], mode, 0, w, 0)
    try:
        # h only, into a pitched view
        ht = Pitched(nnc, sh["x"], mode, 8)
        (h,) = _run_twice(nnc, cmd, hint, 0, [gt, xt, wt], [ht], 1, "%s %s h" % (case, mode))
        _free(ht)
        cr.check(h, h_ref, h_s, kd, mode, mode, "%s %s h" % (case, mode))
        k = np.broadcast_to(kd, h.shape)
        assert (h[k == 0] == 0).all(), "pixels no tap reaches are not 0"
        # dw only (no filter input needed)
        dwt = Pitched(nnc, sh["w"], mode)
        _, dw = _run_twice(nnc, cmd, hint, 0, [gt, xt, None], [None, dwt], 2, "%s %s dw" % (case, mode))
        _free(dwt)
        cr.check(dw, dw_ref, dw_s, npq, mode, mode, "%s %s dw" % (case, mode))
        # h, dw and dbias, accumulating into old dw / dbias (h is overwritten)
        old = cr.operand(sh["w"], _seed(case, 4), mode, -1.0, 1.0)
        db_old = cr.operand((g.K,), _seed(case, 5), FP32, -1.0, 1.0)
        ht, dwt, dbt = Pitched(nnc, sh["x"], mode), Pitched(nnc, sh["w"], mode, 0, old), Pitched(nnc, (g.K,), FP32, 0, db_old)
        h2, dw2, db = _run_twice(nnc, cmd, hint, abi.CCV_NNC_ACCUMULATE_OUTPUT, [gt, xt, wt], [ht, dwt, dbt], 1 + 2 + colsum_launches, "%s %s h + dw + dbias" % (case, mode))
        _free(ht, dwt, dbt)
        assert np.array_equal(h2, h), "h differs between the h-only and the full call"
        o64 = old.astype(np.float64)
        cr.check(dw2, dw_ref + o64, dw_s + np.abs(o64), npq, mode, mode, "%s %s dw += " % (case, mode))
        gf = G.reshape(-1, g.K)
        cr.check(db, gf.sum(0) + db_old, np.abs(gf).sum(0) + np.abs(db_old), npq, FP32, FP32, "%s %s dbias" % (case, mode))
    finally:
        _free(gt, xt, wt)


# ------------------------------------------------------------------------------------------------ GPU: staged operands
NCHW_CASES = [c for c in GPU_CASES if c.name in ("dw3x3_s2", "cg4_kg8", "c12_depthwise_scalar")]


def _nchw(a):
    return np.ascontiguousarray(np.moveaxis(a, -1, 1))


def _nhwc(a):
    return np.ascontiguousarray(np.moveaxis(a, 1, -1))


@pytest.mark.gpu
@pytest.mark.parametrize("case", NCHW_CASES, ids=repr)
@pytest.mark.parametrize("mode", MODES)
def test_nchw_gives_the_nhwc_bits(gpu, case, mode):
    nnc = gpu
    x, w, gy = operands(case, mode)
    bias = cr.operand((case.g.K,), _seed(case, 3), FP32, 0.0, 2.0)
    sh, hint, dt = case.shapes(), case.hint(nnc), DT[mode]
    wn = np.ascontiguousarray(w.transpose(0, 3, 1, 2))
    st, (y,) = gpu_exec16(nnc, case.fwd_cmd(nnc), hint, 0, [x, w, bias], [np.zeros(sh["y"], np.float32)], dt, keep32=(id(bias),))
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (yn,) = gpu_exec16(nnc, case.fwd_cmd(nnc), hint, 0, [_nchw(x), wn, bias], [_nchw(np.zeros(sh["y"], np.float32))], dt, keep32=(id(bias),),
                           in_fmts=[NCHW, NCHW, NHWC], out_fmts=[NCHW])
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert np.array_equal(_nhwc(yn), y)
    outs = [np.zeros(sh["x"], np.float32), np.zeros(sh["w"], np.float32)]
    st, (h, dw) = gpu_exec16(nnc, case.back_cmd(nnc), hint, 0, [gy, x, w], outs, dt)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (hn, dwn) = gpu_exec16(nnc, case.back_cmd(nnc), hint, 0, [_nchw(gy), _nchw(x), wn], [_nchw(outs[0]), np.zeros(wn.shape, np.float32)], dt,
                               in_fmts=[NCHW] * 3, out_fmts=[NCHW] * 2)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert np.array_equal(_nhwc(hn), h) and np.array_equal(dwn.transpose(0, 2, 3, 1), dw)


@pytest.mark.gpu
def test_palettized_depthwise_filter_gives_the_decoded_bits(gpu):
    nnc = gpu
    case = [c for c in GPU_CASES if c.name == "dw3x3_s2"][0]
    sh, hint = case.shapes(), case.hint(nnc)
    x = cr.operand(sh["x"], 5, FP16).astype(np.float16)
    count = int(np.prod(sh["w"]))
    data, dense = pr.random_palettized(count, 6, 32, np.float16, 9, 0.25)
    w = dense.reshape(sh["w"]).astype(np.float16)
    xt = nnc.gpu_tensor(list(sh["x"]), NHWC, abi.CCV_16F).upload(x)
    wt = nnc.gpu_tensor(list(sh["w"]), NHWC, abi.CCV_16F).upload(w)
    qt = nnc.gpu_palettized_tensor(list(sh["w"]), abi.CCV_16F, 6, 32)
    qt.upload(data[:qt.nbytes])
    res = []
    for filt in (wt, qt):
        yt = nnc.gpu_tensor(list(sh["y"]), NHWC, abi.CCV_16F)
        st = nnc.cmd_exec(case.fwd_cmd(nnc), hint, 0, [xt, filt], [yt])
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        res.append(yt.download())
        yt.free()
    _free(xt, wt, qt)
    assert np.array_equal(res[0].view(np.uint16), res[1].view(np.uint16))


# ------------------------------------------------------------------------------------------------ GPU: transposed convolution
TRANSPOSE_CASES = [c for c in GPU_CASES if c.name in ("dw3x3_s2", "multiplier2", "cg4_kg8", "c12_depthwise_scalar", "dw5x5_s2")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRANSPOSE_CASES, ids=repr)
@pytest.mark.parametrize("mode", MODES)
def test_transpose_equals_the_mirrored_convolution(gpu, case, mode):
    """CONVOLUTION_TRANSPOSE with a[N, P, Q, K] (Cin = K), w[K, R, S, C / groups], y[N, H, W, C]: its forward is CONVOLUTION_BACKWARD's h,
    its backward CONVOLUTION_FORWARD (da) and CONVOLUTION_BACKWARD's dw with x = g and grad = a, bit for bit"""
    nnc = gpu
    g, dt, hint = case.g, DT[mode], case.hint(nnc)
    sh = case.shapes()
    a, w, gy = cr.operand(sh["y"], _seed(case, 6), mode), operands(case, mode)[1], cr.operand(sh["x"], _seed(case, 7), mode)
    tf = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(case.groups, g.C, 0, g.R, g.S, g.K, g.dil)
    tb = nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD(case.groups, g.C, 0, g.R, g.S, g.K, g.dil)
    st, (y,) = gpu_exec16(nnc, tf, hint, 0, [a, w], [np.zeros(sh["x"], np.float32)], dt)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (h,) = gpu_exec16(nnc, case.back_cmd(nnc), hint, 0, [a, np.zeros(sh["x"], np.float32), w], [np.zeros(sh["x"], np.float32)], dt)
    assert st == 0
    assert np.array_equal(y, h), "transposed forward != the mirrored data gradient"
    st, (da, dw) = gpu_exec16(nnc, tb, hint, 0, [gy, a, w], [np.zeros(sh["y"], np.float32), np.zeros(sh["w"], np.float32)], dt)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (da_c,) = gpu_exec16(nnc, case.fwd_cmd(nnc), hint, 0, [gy, w], [np.zeros(sh["y"], np.float32)], dt)
    assert st == 0
    st, (_, dw_c) = gpu_exec16(nnc, case.back_cmd(nnc), hint, 0, [a, gy], [None, np.zeros(sh["w"], np.float32)], dt)
    assert st == 0
    assert np.array_equal(da, da_c) and np.array_equal(dw, dw_c)


# ------------------------------------------------------------------------------------------------ GPU: wide groups past 2^31 elements
@pytest.mark.gpu
def test_wide_groups_past_2_31_elements_run(gpu):
    """Cg = Kg = 16 is wide enough for the tensor cores, but the per-group copies walk int strides, so an input of more than 2^31 elements
    takes the direct kernels (64-bit offsets).  The last image is held to the bound."""
    nnc = gpu
    case = Case("wide_2_31", 1100, 248, 248, 32, 32, 2, 3, 3, stride=(2, 2), pad=(1, 1))
    g, mode = case.g, BF16
    assert g.N * g.H * g.W * g.C > 2 ** 31
    sh = case.shapes()
    img = cr.operand((4,) + sh["x"][1:], 21, mode)
    w = cr.operand(sh["w"], 22, mode) / np.float32(128)
    xb = np.empty(sh["x"], np.uint16)
    ib = _bits(img, mode)
    for n in range(0, g.N, 4):
        xb[n:n + 4] = ib[:g.N - n]
    xt = nnc.gpu_tensor(list(sh["x"]), NHWC, abi.CCV_16BF)
    xt.upload(xb)
    del xb
    wt = nnc.gpu_tensor(list(sh["w"]), NHWC, abi.CCV_16BF).upload(_bits(w, mode))
    yt = nnc.gpu_tensor(list(sh["y"]), NHWC, abi.CCV_16BF)
    try:
        st = nnc.cmd_exec(case.fwd_cmd(nnc), case.hint(nnc), 0, [xt, wt], [yt])
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        y = _values(yt.download()[-1], mode)
    finally:
        _free(xt, wt, yt)
    last = img[(g.N - 1) % 4][None].astype(np.float64)
    one = Case("wide_last", 1, 248, 248, 32, 32, 2, 3, 3, stride=(2, 2), pad=(1, 1))
    want, s = cr.with_scale(lambda a, f: gconv_fwd(one, a, f), last, w.astype(np.float64))
    cr.check(y[None], want, s, keff_fwd(one), mode, mode, "past 2^31 elements, last image")
