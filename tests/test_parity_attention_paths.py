"""Every launch path of SCALED_DOT_PRODUCT_ATTENTION against a float64 oracle at rounding-level bounds (tests/attention_ref.py holds
the oracle, the bounds and the restated planner).

Each case names the path it was written for: the 16-bit flash forward and fused backward, the fp32 path with TF32 or FFMA GEMMs, or
the 16-bit functional form (widen, fp32 path, narrow).  A case fails when the planner restatement puts it elsewhere or when
ccv_nnc_sm100_launch_count() disagrees.  Every output, the log-sum-exp included, lives in a NaN-filled guard buffer and is poisoned
before each call; view cases write outputs with a row pitch wider than H * D and read q / k / v as slices of one packed
[B, S, 3, H, D] buffer.  Guard elements must stay untouched and two runs must agree bit for bit.  The logits come in five regimes:
flat (U(-1, 1) data), peaked (about +-20), rising (every 128-key block raises the row max, so every block rescales), falling (the max
is in the first block and later probabilities underflow, through fp16 subnormals) and extreme (exp2 arguments of several hundred).

The CPU tests pin the oracle to CPU_REF (the committed fixture, and the compiled reference when it is built) and show on every GPU
case shape that the bounds reject each modelled defect of the kernels."""
import functools
import os
import zlib

import numpy as np
import pytest

from ccv_b200 import abi
from tests import attention_ref as ar
from tests import contract_ref as cr
from tests.attention_ref import BF16, FP16, FP32
from tests.util import to_bf16

NHWC = abi.CCV_TENSOR_FORMAT_NHWC
DT = {BF16: abi.CCV_16BF, FP16: abi.CCV_16F, FP32: abi.CCV_32F}
SENTINEL = {FP32: 0x7FBADBAD, BF16: 0x7FBB, FP16: 0x7DBB}  # NaN patterns
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ------------------------------------------------------------------------------------------------ the case table
class Case(object):
    def __init__(self, dtype, B, Sq, Sk, H, Hk, D, causal, regime="flat", scale="rsqrt", Dv=None, mask=None, three_d=False,
                 backward=True, view=False, path=None):
        self.dtype, self.B, self.Sq, self.Sk, self.H, self.Hk, self.D, self.causal = dtype, B, Sq, Sk, H, Hk, D, causal
        self.regime, self.scale_kind, self.Dv, self.mask, self.three_d = regime, scale, Dv or D, mask, three_d
        self.backward, self.view, self.path = backward and mask is None, view, path
        self.scale = float(np.float32({"rsqrt": 1.0 / np.sqrt(D), "one": 1.0, "small": 0.02}[scale]))

    def __repr__(self):
        s = "%s B%d Sq%d Sk%d H%d/%d D%d%s%s %s %s" % (self.dtype, self.B, self.Sq, self.Sk, self.H, self.Hk, self.D, "" if self.Dv == self.D else " Dv%d" % self.Dv,
                                                   " causal" if self.causal else "", self.regime, self.scale_kind)
        if self.mask:
            s += " mask%s" % "x".join(map(str, self.mask))
        return s + (" 3d" if self.three_d else "") + (" view" if self.view else "") + " ->" + self.path

    def plans(self):
        a = (self.dtype, self.B, self.H, self.Hk, self.Sq, self.Sk, self.D, self.Dv)
        fp = ar.plan_forward(*a, mask=self.mask is not None, view=self.view, lse=self.lse)
        bp = ar.plan_backward(*a, saved=False, view=self.view) if self.backward else None
        return fp, bp

    @property
    def lse(self):
        return self.dtype != FP32 and self.mask is None and ar.plan_forward(self.dtype, self.B, self.H, self.Hk, self.Sq, self.Sk, self.D, self.Dv)["path"] == "flash"


C = Case
CASES = [
    # flash forward + fused backward: D in {8, 16, 40, 56, 64, 72, 120, 128}, extents around the 64 / 128 blocks, GQA 1 / 2 / 4 / 8
    C(BF16, 1, 1, 2048, 4, 1, 128, 1, path="flash"),                       # decode: Sq = 1, causal, long Sk, Hk = 1
    C(FP16, 2, 333, 200, 4, 2, 64, 1, "peaked", view=True, path="flash"),  # Sq > Sk causal: fully masked rows
    C(BF16, 1, 65, 1024, 8, 1, 128, 1, "rising", path="flash"),            # Sq < Sk causal, every block rescales, GQA 8
    C(FP16, 1, 129, 129, 2, 2, 8, 0, "flat", "small", path="flash"),
    C(BF16, 2, 127, 63, 2, 1, 16, 1, "flat", "one", view=True, path="flash"),
    C(FP16, 1, 1024, 1024, 2, 2, 40, 1, "falling", path="flash"),          # fp16 P subnormal, then zero
    C(BF16, 1, 200, 333, 4, 4, 56, 0, "extreme", path="flash"),
    C(FP16, 1, 64, 2, 2, 2, 72, 1, view=True, path="flash"),
    C(BF16, 1, 2, 64, 4, 2, 120, 0, "peaked", path="flash"),
    C(FP16, 1, 128, 65, 8, 2, 128, 0, "extreme", path="flash"),
    C(BF16, 1, 2048, 2048, 1, 1, 128, 1, "falling", path="flash"),
    C(FP16, 1, 1, 1, 1, 1, 64, 0, path="flash"),
    C(FP16, 1, 333, 1024, 2, 1, 128, 1, "rising", path="flash"),
    C(BF16, 2, 63, 129, 2, 2, 64, 0, "flat", three_d=False, path="flash"),
    C(FP16, 2, 129, 127, 1, 1, 64, 1, "peaked", three_d=True, path="flash"),
    # functional form: D in {36, 100, 160}, Dv != D, masks of every shape
    C(BF16, 2, 63, 129, 4, 2, 36, 1, path="func"),
    C(FP16, 1, 129, 64, 2, 2, 100, 0, "peaked", path="func"),
    C(BF16, 1, 200, 200, 2, 1, 160, 1, "falling", path="func"),
    C(FP16, 1, 65, 127, 2, 2, 64, 0, Dv=32, path="func"),                  # Sk % 4 != 0: the P GEMMs run on FFMA
    C(BF16, 2, 64, 96, 2, 2, 64, 0, mask=(64, 96), path="func"),
    C(FP16, 2, 64, 96, 2, 2, 64, 1, mask=(1, 2, 64, 96), path="func"),
    C(BF16, 2, 33, 65, 2, 2, 128, 0, "peaked", mask=(2, 1, 33, 65), path="func"),
    C(FP16, 2, 64, 96, 2, 2, 64, 0, mask=(2, 2, 64, 96), path="func"),
    C(BF16, 2, 64, 96, 2, 2, 64, 0, mask=(2, 64, 96), path="func"),
    # fp32: TF32 and FFMA GEMMs
    C(FP32, 2, 128, 200, 4, 2, 64, 1, path="fp32"),
    C(FP32, 1, 65, 333, 2, 1, 36, 0, "peaked", path="fp32"),
    C(FP32, 2, 129, 127, 1, 1, 40, 1, "rising", three_d=True, path="fp32"),
    C(FP32, 1, 200, 64, 2, 2, 64, 0, "extreme", Dv=96, path="fp32"),
    C(FP32, 1, 127, 65, 2, 2, 64, 1, "falling", "rsqrt", path="fp32"),
    C(FP32, 2, 64, 96, 2, 2, 32, 0, mask=(2, 1, 64, 96), path="fp32"),
    C(FP32, 2, 64, 96, 2, 2, 32, 1, mask=(2, 64, 96), path="fp32"),
    C(FP32, 1, 64, 1024, 2, 1, 64, 0, path="fp32"),
]
CASE_IDS = [repr(c) for c in CASES]
CALIBRATION = {}


# ------------------------------------------------------------------------------------------------ operands and oracle
def _grid(x, dtype):
    """float32 values on the dtype's grid (16-bit: the nearest 16-bit value; fp32: no TF32 rounding ties)"""
    if dtype == FP32:
        return cr.untie_tf32(x)
    return cr.rne16(np.asarray(x, np.float64), dtype).astype(np.float32)


@functools.lru_cache(maxsize=None)
def operands(case):
    """q, k, v, dO (and the mask) in the tensors' [B, S, H, D] shapes (3-d cases: [B, S, D]), float32 on the dtype's grid"""
    r = np.random.RandomState(zlib.crc32(repr(case).encode()) % 100000)
    u = lambda shape, lo, hi: (lo + (hi - lo) * r.random_sample(shape)).astype(np.float32)
    B, Sq, Sk, H, Hk, D, Dv = case.B, case.Sq, case.Sk, case.H, case.Hk, case.D, case.Dv
    q, k = u((B, Sq, H, D), -1, 1), u((B, Sk, Hk, D), -1, 1)
    v, do = u((B, Sk, Hk, Dv), -0.5, 1), u((B, Sq, H, Dv), -0.5, 1)  # positive means: a dropped or extra term moves the result
    if case.regime == "peaked":
        q *= 12
    elif case.regime == "extreme":
        q *= 25
        k *= 25
    elif case.regime in ("rising", "falling"):
        # a per-key component of feature 0: the logits move by 32 from the first key to the last
        q[..., 0] = 16.0 / case.scale
        ramp = np.linspace(-1, 1, Sk, dtype=np.float32)
        k[:, :, :, 0] = (ramp if case.regime == "rising" else -ramp)[None, :, None]
    mask = None
    if case.mask:
        mask = (np.where(r.random_sample(case.mask) < 0.3, -1e4, 0.0) + u(case.mask, -3, 3)).astype(np.float32)
    d = dict(q=_grid(q, case.dtype), k=_grid(k, case.dtype), v=_grid(v, case.dtype), do=_grid(do, case.dtype), mask=mask)
    if case.three_d:
        for n in ("q", "k", "v", "do"):
            d[n] = np.ascontiguousarray(d[n][:, :, 0, :])
    return d


def _four(d, three_d):
    return dict((n, ar.as4(d[n], three_d)) for n in ("q", "k", "v", "do"))


def forward_oracle(case, d, plan, defect=None, drop=None):
    x = _four(d, case.three_d)
    model = ar.model_for(case.dtype, plan)
    return ar.Forward(ar.seen_s(x["q"], plan), ar.seen_s(x["k"], plan), ar.seen_p(x["v"], plan), case.scale, case.causal, d["mask"], model, defect, drop)


def backward_oracle(case, d, plan, o16=None, defect=None, fdefect=None, drop=None):
    x = _four(d, case.three_d)
    f = forward_oracle(case, d, plan, fdefect, drop)
    if plan["path"] == "fused":
        return ar.Backward(f, x["do"], o16=ar.as4(o16, case.three_d), defect=defect)
    S, P = (lambda a: ar.seen_s(a, plan)), (lambda a: ar.seen_p(a, plan))
    return ar.Backward(f, S(x["do"]), p_ops=(P(x["v"]), P(x["do"]), P(x["k"]), P(x["q"])), dp_v=S(x["v"]), defect=defect)


def _unthree(a, case):
    return a[:, :, 0, :] if case.three_d else a


# ------------------------------------------------------------------------------------------------ CPU: the oracle pinned to CPU_REF
def _pin_check(i, o, grads):
    d = ar.pin_inputs(i)
    t = d["three_d"]
    x = dict((n, np.asarray(ar.as4(d[n], t), np.float64)) for n in ("q", "k", "v", "do"))
    f = ar.Forward(x["q"], x["k"], x["v"], d["scale"], d["causal"], d["mask"], ar.CPU_MODEL)
    oo, uo, _, _ = f.out()
    ar.check(ar.as4(o, t), oo, uo, FP32, "pin %d: O" % i)
    if grads is not None:
        b = ar.Backward(f, x["do"])
        for got, (want, unit), name in zip(grads, b.out(), ("dq", "dk", "dv")):
            ar.check(ar.as4(got, t), want, unit, FP32, "pin %d: %s" % (i, name))


def test_oracle_reproduces_committed_cpu_ref_attention():
    """tests/golden/cpuref_sdpa.npz: GQA, causal Sq < Sk and Sq > Sk (fully masked rows), Dv != D, 3-d tensors, every mask shape"""
    f = np.load(os.path.join(GOLDEN, "cpuref_sdpa.npz"))
    for i in range(len(ar.PINS)):
        d = ar.pin_inputs(i)
        for n in ("q", "k", "v") + (("do",) if d["backward"] else ()):
            assert np.array_equal(f["%d_%s" % (i, n)], d[n]), "pin %d: the fixture's %s is not the seeded operand" % (i, n)
        _pin_check(i, f["%d_o" % i], [f["%d_%s" % (i, n)] for n in ("dq", "dk", "dv")] if d["backward"] else None)


@pytest.mark.ref
@pytest.mark.parametrize("i", range(len(ar.PINS)))
def test_oracle_matches_compiled_reference_attention(ref, i):
    from ccv_b200 import nnc
    from tests.util import ref_exec
    d = ar.pin_inputs(i)
    q, k, v, do, mask = d["q"], d["k"], d["v"], d["do"], d["mask"]
    fwd = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD)
    fwd.info.scaled_dot_product_attention.scale, fwd.info.scaled_dot_product_attention.is_causal = d["scale"], d["causal"]
    st, (o,) = ref_exec(ref, fwd, None, 0, [q, k, v] + ([mask] if mask is not None else []), [np.zeros(q.shape[:-1] + v.shape[-1:], np.float32)])
    assert st == 0
    grads = None
    if d["backward"]:
        bwd = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD)
        bwd.info.scaled_dot_product_attention.scale, bwd.info.scaled_dot_product_attention.is_causal = d["scale"], d["causal"]
        st, grads = ref_exec(ref, bwd, None, 0, [do, None, None, q, k, v], [np.zeros_like(q), np.zeros_like(k), np.zeros_like(v)])
        assert st == 0
    _pin_check(i, o, grads)


# ------------------------------------------------------------------------------------------------ CPU: the bounds able to fail
def _drops(Sk):
    """keys to drop: the Sk tail, the first key of the third 128-key block (or of the second), the first of a 64-key block"""
    out = [("tail", Sk - 1)]
    if Sk > 128:
        out.append(("128-block", 256 if Sk > 256 else 128))
    if Sk > 64:
        out.append(("64-block", 192 if Sk > 192 else 64))
    return out


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_bounds_reject_defective_results(case):
    """The oracle itself passes; with each defect of the kernels' arithmetic it does not.  The defects are shown on the case's shape
    with flat data (every key carries weight, v and dO have positive means); the missing rescale on rising data."""
    fp, bp = case.plans()
    assert fp["path"] == case.path, (case, fp)
    rnd, brnd = ar.rounding_of(fp["path"], case.dtype), ar.rounding_of(case.path, case.dtype)
    f = forward_oracle(case, operands(case), fp)
    o, uo, lse, ul = f.out()
    ar.check(ar.finish(o, rnd), o, uo, rnd, "correct O")
    if fp["path"] == "flash":
        ar.check_lse(lse, lse, ul, "correct LSE")
    flat = _sub(case, regime="flat")
    d = operands(flat)
    f = forward_oracle(flat, d, fp)
    o, uo, lse, ul = f.out()
    if not f.live.any():
        return

    def rejects(bad, what, ref=o, unit=uo, r=rnd):
        assert not ar.admits(ar.finish(bad, r), ref, unit, r).all(), "%s: the bound admits %s" % (case, what)

    if case.causal and case.Sq > 1:
        rejects(forward_oracle(flat, d, fp, "extra_key").out()[0], "one key past the causal horizon")
    for where, j in _drops(case.Sk):
        if f.vis[..., j].sum(-1).max() >= 64:  # (one key of a few rows is within rounding of O; it shows in dV below)
            rejects(forward_oracle(flat, d, fp, drop=j).out()[0], "key %d dropped (%s)" % (j, where))
    if case.H != case.Hk and case.Hk > 1:
        rejects(forward_oracle(flat, d, fp, "gqa_mod").out()[0], "GQA mapped as h % Hk")
    if fp["path"] == "flash" and case.Sk > FLASH_BLOCK:
        rising = _sub(case, regime="rising")
        fr = forward_oracle(rising, operands(rising), fp)
        bad = forward_oracle(rising, operands(rising), fp, "alpha1").out()[0]
        assert not ar.admits(ar.finish(bad, rnd), fr.out()[0], fr.out()[1], rnd).all(), "%s: the bound admits O not rescaled when the max moves" % case
    # A P rounding defect moves O by about u_P sum_j p v, the bound allows C u_P sqrt(sum_j p^2 v^2): it shows once a row spreads its
    # weight over about (2 C)^2 keys, so from Sk = 1024 on (and only where P is rounded at all: FFMA reads P raw, and the functional
    # form's 16-bit output hides a TF32 P defect)
    if fp["path"] != "func" and fp.get("gemm_p") != "ffma" and case.Sk >= 1024 and case.scale_kind != "small":
        rejects(forward_oracle(flat, d, fp, "p_trunc").out()[0], "P truncated")
        if case.dtype != BF16:  # (bf16 P has no coarser format to pass through)
            rejects(forward_oracle(flat, d, fp, "p_twice").out()[0], "P rounded twice (through bf16)")
    if rnd != FP32 and rnd[0] == "rne" and case.Sk >= 1024:  # (the same count: below it the bound spans more than an output ulp)
        assert not ar.admits(cr.trunc16(o, rnd[1]), o, uo, rnd).all(), "%s: the bound admits a truncated output" % case
    if fp["path"] == "flash" and case.Sk > 1:
        bad = forward_oracle(flat, d, fp, "lse_key").lse
        m = np.isfinite(lse)
        assert not ar.admits(bad[m], lse[m], ul[m], FP32).all(), "%s: the bound admits an LSE missing one key" % case
    if not case.backward:
        return
    o16 = _unthree(ar.finish(o, rnd), case) if bp["path"] == "fused" else None
    (dq, uq), (dk, uk), (dv, uv) = backward_oracle(flat, d, bp, o16).out()
    for y, u, n in ((dq, uq, "dq"), (dk, uk, "dk"), (dv, uv, "dv")):
        ar.check(ar.finish(y, brnd), y, u, brnd, "correct " + n)

    def rej(x, what, which=(0, 1, 2)):
        got = x.out()
        ok = [ar.admits(ar.finish(got[i][0], brnd), y, u, brnd).all() for i, (y, u) in enumerate(((dq, uq), (dk, uk), (dv, uv))) if i in which]
        assert not all(ok), "%s: the bounds admit gradients with %s" % (case, what)

    if case.causal and case.Sq > 1:
        rej(backward_oracle(flat, d, bp, o16, fdefect="extra_key"), "one key past the causal horizon")
    for where, j in _drops(case.Sk):
        if f.vis[..., j].any():
            rej(backward_oracle(flat, d, bp, o16, drop=j), "key %d dropped (%s)" % (j, where), (2,))
    if case.H != case.Hk:
        x = backward_oracle(flat, d, bp, o16, defect="group_head")
        rej(x, "one query head of the group missing from dV", (2,))
        rej(x, "one query head of the group missing from dK", (1,))
    if case.scale != 1.0 and case.Sk > 1:  # (one key: dS = 0)
        x = backward_oracle(flat, d, bp, o16, defect="no_scale")
        rej(x, "dQ without scale", (0,))
        rej(x, "dK without scale", (1,))
    if bp["path"] == "fused" and repr(case) in DELTA_VISIBLE:
        rej(backward_oracle(flat, d, bp, o16, defect="delta_exact"), "delta from the exact O instead of the stored one", (0,))


# cases where delta from the exact O instead of the stored 16-bit O moves dQ past its bound (the two differ by at most half an ulp of
# O per feature, which most shapes' dQ bounds absorb)
DELTA_VISIBLE = ["fp16 B2 Sq333 Sk200 H4/2 D64 causal peaked rsqrt view ->flash", "bf16 B2 Sq127 Sk63 H2/1 D16 causal flat one view ->flash",
                 "bf16 B1 Sq2048 Sk2048 H1/1 D128 causal falling rsqrt ->flash"]
FLASH_BLOCK = 128


def test_planner_restatement_on_hand_worked_shapes():
    assert ar.plan_forward(BF16, 32, 16, 16, 2048, 2048, 128, 128) == dict(path="flash", launches=1)
    assert ar.plan_backward(BF16, 32, 16, 16, 2048, 2048, 128, 128, saved=True) == dict(path="fused", launches=3)
    assert ar.plan_backward(FP16, 1, 2, 1, 40, 24, 64, 64)["launches"] == 4  # the forward runs first when o / lse are not passed
    p = ar.plan_forward(BF16, 2, 4, 2, 63, 129, 36, 36)  # D not a multiple of 8: widen q, k, v + 8 (b, h) x 3 + narrow
    assert p["path"] == "func" and p["launches"] == 28 and p["gemm_s"] == "tf32" and p["gemm_p"] == "ffma"  # Sk = 129: pitch not 16 bytes
    assert ar.plan_forward(BF16, 1, 2, 2, 64, 64, 64, 64, mask=True)["path"] == "func"
    assert ar.plan_forward(BF16, 1, 2, 2, 64, 64, 160, 160, lse=True)["path"] == "refused"
    assert ar.plan_forward(FP16, 1, 2, 2, 64, 64, 64, 32)["path"] == "func"  # Dv != D
    assert ar.plan_backward(BF16, 1, 2, 2, 64, 64, 160, 160, view=True)["path"] == "refused"
    assert ar.plan_backward(BF16, 1, 2, 2, 64, 64, 64, 64, view=True)["path"] == "fused"
    assert ar.plan_backward(FP32, 2, 4, 2, 10, 12, 8, 8) == dict(path="fp32", launches=56, gemm_s="tf32", gemm_p="tf32")
    for c in CASES:
        fp, bp = c.plans()
        assert fp["path"] == c.path and (bp is None or bp["path"] == {"flash": "fused"}.get(c.path, c.path)), (c, fp, bp)


# ------------------------------------------------------------------------------------------------ GPU
def _bits(a, dtype):
    if dtype == FP32:
        return np.ascontiguousarray(a, np.float32).view(np.uint32)
    return cr.to_bits16(np.asarray(a, np.float64), dtype)


def _values(bits, dtype):
    return bits.view(np.float32).astype(np.float64) if dtype == FP32 else cr.from_bits16(bits, dtype)


def _np_bits(dtype):
    return np.uint32 if dtype == FP32 else np.uint16


class Buf(object):
    """A flat NaN-filled allocation holding tensors as (views of) strided windows: add(dims, strides, offset[, bits]) returns the
    tensor; result(tensor) its elements; check_guards() that nothing outside the windows changed."""

    def __init__(self, nnc, total, dtype):
        self.nnc, self.dtype = nnc, dtype
        self.host = np.full((total,), SENTINEL[dtype], _np_bits(dtype))
        self.mask = np.zeros((total,), bool)
        self.base = nnc.gpu_tensor([total], NHWC, DT[dtype])
        self.views, self.idx = [], {}

    def add(self, dims, strides=None, offset=0, bits=None):
        dims = list(dims)
        if strides is None:
            strides = [int(np.prod(dims[i + 1:])) for i in range(len(dims))]
        idx = offset + sum(np.arange(n).reshape([-1] + [1] * (len(dims) - 1 - i)) * s for i, (n, s) in enumerate(zip(dims, strides)))
        packed = strides == [int(np.prod(dims[i + 1:])) for i in range(len(dims))]
        if packed:
            t = self.nnc.gpu_tensor(dims, NHWC, DT[self.dtype], ptr=self.base.data_ptr + offset * self.host.itemsize)
        else:
            t = self.nnc.tensor_view_new(self.base, dims, [0] * (len(dims) - 1) + [offset] + [0] * (12 - len(dims)), list(strides) + [0] * (12 - len(dims)))
        self.mask[idx] = True
        if bits is not None:
            self.host[idx] = bits
        self.views.append(t)
        self.idx[id(t)] = idx
        return t

    def arm(self):
        self.base.upload(self.host.view(np.float16) if self.dtype == FP16 else self.host if self.dtype == BF16 else self.host.view(np.float32))
        return self

    def result(self, t):
        got = self.base.download().view(_np_bits(self.dtype))
        changed = (got != self.host) & ~self.mask
        assert not changed.any(), "%d guard elements overwritten, first at %s" % (changed.sum(), np.argwhere(changed)[0])
        return got[self.idx[id(t)]]

    def free(self):
        for t in self.views:
            t.free()
        self.base.free()


def _layout(dims, extra):
    """strides of a [B, S, (H,) D] tensor whose rows have pitch (H *) D + extra"""
    pitch = int(np.prod(dims[2:])) + extra
    return [dims[1] * pitch, pitch] + ([dims[3], 1] if len(dims) == 4 else [1])


def _out_buf(nnc, dims, dtype, view):
    """an output tensor in its own guard buffer: packed after a 64-element guard, or a view with a wider row pitch"""
    extra = 8 if view else 0
    strides = _layout(dims, extra)
    total = 64 + dims[0] * strides[0] + 64
    b = Buf(nnc, total, dtype)
    return b, b.add(dims, strides, 64)


def _in_tensors(nnc, case, d, names, packed_qkv):
    """input tensors; packed_qkv: q, k, v as slices of one [B, S, 3, H, D] buffer (needs Sq == Sk, H == Hk, D == Dv)"""
    if packed_qkv:
        B, S, H, D = case.B, case.Sq, case.H, case.D
        buf = Buf(nnc, B * S * 3 * H * D, case.dtype)
        st = [S * 3 * H * D, 3 * H * D, D, 1]
        ts = [buf.add([B, S, H, D], st, i * H * D, _bits(d[n], case.dtype)) for i, n in enumerate(("q", "k", "v"))]
        return buf, dict(zip(("q", "k", "v"), ts))
    total = sum(d[n].size for n in names)
    buf = Buf(nnc, total, case.dtype)
    out, off = {}, 0
    for n in names:
        out[n] = buf.add(list(d[n].shape), None, off, _bits(d[n], case.dtype))
        off += d[n].size
    return buf, out


def _cmd(nnc, cmd_id, case):
    c = nnc._simple(cmd_id)
    c.info.scaled_dot_product_attention.scale = case.scale
    c.info.scaled_dot_product_attention.is_causal = case.causal
    c.info.scaled_dot_product_attention.deterministic = 1
    return c


def _shape(case, S, H, D):
    return [case.B, S, D] if case.three_d else [case.B, S, H, D]


def run_forward(nnc, case, d, view=False, packed_qkv=False, lse=True, reps=2):
    """(O bits, LSE or None, launches) of the forward; two runs must agree bit for bit"""
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), packed_qkv)
    tm = nnc.gpu_tensor(list(d["mask"].shape)).upload(d["mask"]) if d["mask"] is not None else None
    ob, to = _out_buf(nnc, _shape(case, case.Sq, case.H, case.Dv), case.dtype, view)
    lb, tl = _out_buf(nnc, [case.B, case.H, case.Sq], FP32, False) if lse else (None, None)
    cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case)
    res = []
    try:
        ib.arm()
        for _ in range(reps):
            ob.arm()
            if lb:
                lb.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, None, 0, [ins["q"], ins["k"], ins["v"]] + ([tm] if tm else []), [to] + ([tl] if tl else []), stream)
            stream.wait()
            assert st == 0, "%s: forward status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
            res.append((ob.result(to), lb.result(tl).view(np.float32).astype(np.float64) if lb else None, nnc.launch_count() - l0))
    finally:
        for x in [ib, ob, lb, tm, stream]:
            if x is not None:
                x.free()
    if reps > 1:
        assert np.array_equal(res[0][0], res[1][0]), "%s: two forward runs differ" % case
        assert res[0][1] is None or np.array_equal(res[0][1].view(np.uint64), res[1][1].view(np.uint64)), "%s: two LSE runs differ" % case
    return res[0]


def run_backward(nnc, case, d, view=False, packed_qkv=False, saved=None, alias_dout_q=False, reps=2):
    """(dq, dk, dv bits, launches); saved = (O bits, LSE) passes the forward's outputs as inputs[9], [10]"""
    stream = nnc.Stream(0)
    names = ("do",) if packed_qkv else ("do", "q", "k", "v")
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), True) if packed_qkv else (None, {})
    db, dins = _in_tensors(nnc, case, d, names if not packed_qkv else ("do",), False)
    ins.update(dins)
    extra = []
    if saved is not None:
        sb = Buf(nnc, saved[0].size, case.dtype)
        so = sb.add(_shape(case, case.Sq, case.H, case.Dv), None, 0, saved[0])
        sl = nnc.gpu_tensor([case.B, case.H, case.Sq]).upload(saved[1].astype(np.float32))
        extra = [None, None, None, so, sl]
    bufs, outs = [], []
    for n, S, H, D in (("q", case.Sq, case.H, case.D), ("k", case.Sk, case.Hk, case.D), ("v", case.Sk, case.Hk, case.Dv)):
        b, t = _out_buf(nnc, _shape(case, S, H, D), case.dtype, view)
        bufs.append(b), outs.append(t)
    cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, case)
    dout = ins["q"] if alias_dout_q else ins["do"]
    res = []
    try:
        for b in [x for x in (ib, db) if x is not None]:
            b.arm()
        if saved is not None:
            sb.arm()
        for _ in range(reps):
            for b in bufs:
                b.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, None, 0, [dout, None, None, ins["q"], ins["k"], ins["v"]] + extra, outs, stream)
            stream.wait()
            assert st == 0, "%s: backward status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
            res.append([b.result(t) for b, t in zip(bufs, outs)] + [nnc.launch_count() - l0])
    finally:
        for x in bufs + [x for x in (ib, db) if x is not None] + ([sb, sl] if saved is not None else []) + [stream]:
            x.free()
    if reps > 1:
        for a, b2, n in zip(res[0][:3], res[1][:3], ("dq", "dk", "dv")):
            assert np.array_equal(a, b2), "%s: two backward runs differ in %s" % (case, n)
    return res[0]


def _record(key, ratio, what=""):
    if ratio > CALIBRATION.get(key, (0.0, ""))[0]:
        CALIBRATION[key] = (ratio, what)


@pytest.fixture(scope="module")
def report(gpu):
    yield
    if CALIBRATION:
        print("\nlargest bound ratio per path (C_ATT = %g):" % ar.C_ATT)
        for k in sorted(CALIBRATION):
            print("  %-28s %.3f  (%s)" % (k, CALIBRATION[k][0], CALIBRATION[k][1]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_attention_path(gpu, report, case):
    nnc = gpu
    d = operands(case)
    fp, bp = case.plans()
    assert fp["path"] == case.path, (case, fp)
    o_bits, lse, launches = run_forward(nnc, case, d, view=case.view, lse=case.lse)
    assert launches == fp["launches"], "%s: %d forward launches, planned %d" % (case, launches, fp["launches"])
    rnd = ar.rounding_of(fp["path"], case.dtype)
    f = forward_oracle(case, d, fp)
    o, uo, lse_ref, ul = f.out()
    y = ar.as4(_values(o_bits, case.dtype), case.three_d)
    _record("%s forward O %s" % (fp["path"], case.dtype), ar.check(y, o, uo, rnd, "%s: O" % case), repr(case))
    dead = ~f.live[..., 0]  # [B, H, Sq]
    if dead.any():
        assert (y.transpose(0, 2, 1, 3)[dead] == 0).all(), "%s: fully masked rows must give O = 0 exactly" % case
    if lse is not None:
        _record("flash forward LSE", ar.check_lse(lse, lse_ref, ul, "%s: LSE" % case), repr(case))
    if not case.backward:
        return
    res = run_backward(nnc, case, d, view=case.view)
    assert res[3] == bp["launches"], "%s: %d backward launches, planned %d" % (case, res[3], bp["launches"])
    b = backward_oracle(case, d, bp, o16=_values(o_bits, case.dtype) if bp["path"] == "fused" else None)
    brnd = ar.rounding_of(bp["path"], case.dtype)
    for bits, (want, unit), n in zip(res[:3], b.out(), ("dq", "dk", "dv")):
        got = ar.as4(_values(bits, case.dtype), case.three_d)
        _record("%s backward %s" % (bp["path"], case.dtype), ar.check(got, want, unit, brnd, "%s: %s" % (case, n)), "%s %s" % (case, n))
        if n == "dq" and dead.any():
            assert (got.transpose(0, 2, 1, 3)[dead] == 0).all(), "%s: fully masked rows must give dQ = 0 exactly" % case
    if bp["path"] == "fused":
        saved = run_backward(nnc, case, d, view=case.view, saved=(o_bits, lse), reps=1)
        assert saved[3] == 3, "%s: with the saved o / lse the fused path is prep + dK/dV + dQ" % case
        for a, s, n in zip(res[:3], saved[:3], ("dq", "dk", "dv")):
            assert np.array_equal(a, s), "%s: %s with the saved o / lse differs from the recomputed one" % (case, n)


# ---- exact identities of the flash / fused kernels ------------------------------------------------------------------------
EXACT = [C(BF16, 2, 200, 200, 4, 2, 64, 1, path="flash"), C(FP16, 2, 129, 129, 2, 1, 128, 0, "peaked", path="flash"),
         C(BF16, 2, 64, 64, 2, 2, 64, 0, mask=(64, 64), backward=False, path="func"), C(FP32, 2, 96, 96, 2, 1, 64, 1, path="fp32")]


def _sub(case, **kw):
    a = dict(dtype=case.dtype, B=case.B, Sq=case.Sq, Sk=case.Sk, H=case.H, Hk=case.Hk, D=case.D, causal=case.causal, regime=case.regime,
             scale=case.scale_kind, Dv=case.Dv, mask=case.mask, three_d=case.three_d, backward=case.backward, view=case.view, path=case.path)
    a.update(kw)
    c = Case(**a)
    c.scale = case.scale
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT, ids=[repr(c) for c in EXACT])
def test_gqa_batch_entry_and_view_identities(gpu, case):
    """GQA = K / V repeated to H heads; one batch entry = a call on that entry alone; q, k, v sliced from a packed QKV buffer = packed
    copies; dout aliasing q = a separate copy of q (the bench's backward)."""
    nnc = gpu
    d = operands(case)
    o, lse, _ = run_forward(nnc, case, d, lse=case.lse, reps=1)
    g = case.H // case.Hk
    if g > 1:
        rep = _sub(case, Hk=case.H)
        rd = dict(d, k=np.repeat(d["k"], g, axis=2), v=np.repeat(d["v"], g, axis=2))
        o2, lse2, _ = run_forward(nnc, rep, rd, lse=case.lse, reps=1)
        assert np.array_equal(o, o2), "%s: GQA forward differs from K / V repeated to H heads" % case
    one = _sub(case, B=1)
    od = dict((n, None if a is None else (a[1:2] if n != "mask" or (a.ndim == 4 and a.shape[0] > 1) else a)) for n, a in d.items())
    o1, lse1, _ = run_forward(nnc, one, od, lse=case.lse, reps=1)
    assert np.array_equal(o[1:2], o1), "%s: batch entry 1 differs from a call on it alone" % case
    if lse is not None:
        assert np.array_equal(lse[1:2], lse1), "%s: batch entry 1's LSE differs" % case
    if not case.backward:
        return
    full = run_backward(nnc, case, d, reps=1)
    part = run_backward(nnc, one, od, reps=1)
    for a, b2, n in zip(full[:3], part[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a[1:2], b2), "%s: batch entry 1's %s differs from a call on it alone" % (case, n)
    alias = run_backward(nnc, case, dict(d, do=d["q"]), alias_dout_q=True, reps=1)
    copy = run_backward(nnc, case, dict(d, do=d["q"].copy()), reps=1)
    for a, b2, n in zip(alias[:3], copy[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2), "%s: %s with dout aliasing q differs from a copy" % (case, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_packed_qkv_views_and_pitched_gradients(gpu, dtype):
    """q, k, v as slices of one [B, S, 3, H, D] buffer and dq / dk / dv with a wider row pitch give the packed results bit for bit,
    and leave every guard element untouched (the fused backward takes views; only the functional form refuses them)."""
    nnc = gpu
    case = C(dtype, 2, 129, 129, 2, 2, 64, 1, "peaked", path="flash")
    d = operands(case)
    o, lse, _ = run_forward(nnc, case, d, reps=1)
    ov, lsev, _ = run_forward(nnc, case, d, view=True, packed_qkv=True, reps=1)
    assert np.array_equal(o, ov) and np.array_equal(lse, lsev), "packed QKV views give another forward result"
    g = run_backward(nnc, case, d, reps=1)
    gv = run_backward(nnc, case, d, view=True, packed_qkv=True, reps=1)
    for a, b2, n in zip(g[:3], gv[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2), "%s from views differs from the packed call" % n
    assert gv[3] == 4
    # the functional form (D = 160) refuses views
    fc = C(dtype, 1, 64, 64, 2, 2, 160, 0, path="func")
    fd = operands(fc)
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, fc, fd, ("q", "k", "v"), True)
    dob, dos = _in_tensors(nnc, fc, fd, ("do",), False)
    outs = [_out_buf(nnc, [1, 64, 2, 160], dtype, True) for _ in range(3)]
    try:
        st = nnc.cmd_exec(_cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, fc), None, 0, [dos["do"], None, None, ins["q"], ins["k"], ins["v"]], [t for _, t in outs], stream)
        assert st == abi.CCV_NNC_EXEC_INVALID
    finally:
        for x in [ib, dob] + [b for b, _ in outs] + [stream]:
            x.free()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_head_dim_64_equals_zero_padded_128(gpu, dtype):
    """The TMA unit zero-fills features D..127 of the 128-wide tiles: D = 64 gives the first 64 columns of the same call with q, k, v
    zero-padded to 128 features, forward and backward, bit for bit."""
    nnc = gpu
    c64 = C(dtype, 1, 200, 333, 4, 2, 64, 1, path="flash")
    d = operands(c64)
    pad = lambda a: np.concatenate([a, np.zeros(a.shape[:-1] + (64,), np.float32)], -1)
    c128 = _sub(c64, D=128, Dv=128)
    c128.scale = c64.scale
    dp = dict(d, q=pad(d["q"]), k=pad(d["k"]), v=pad(d["v"]), do=pad(d["do"]))
    o, lse, _ = run_forward(nnc, c64, d, reps=1)
    o2, lse2, _ = run_forward(nnc, c128, dp, reps=1)
    assert np.array_equal(o, o2[..., :64]) and np.array_equal(lse, lse2)
    assert (_values(o2[..., 64:], dtype) == 0).all()
    g = run_backward(nnc, c64, d, reps=1)
    g2 = run_backward(nnc, c128, dp, reps=1)
    for a, b2, n in zip(g[:3], g2[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2[..., :64]), "%s of D = 64 differs from the zero-padded call" % n


@pytest.mark.gpu
def test_bench_shape_forward_and_backward(gpu, report):
    """bench.py's attention workload (bf16, B = 32, H = 16, S = 2048, D = 128, q = k = v, dout = q, the saved o / lse), causal and
    not: a few (b, h) slices of O, LSE, dQ, dK and dV held to the bound.  The data are seeded U(-1, 1) rather than bench.py's
    i / count ramp: the ramp's neighbouring values are nearly equal, so their rounding errors line up instead of averaging out, which
    the random-walk terms of the bound do not model (test_parity_sdpa.py checks the ramp against CPU_REF)."""
    nnc = gpu
    B, H, S, D = 32, 16, 2048, 128
    bits = to_bf16((np.random.RandomState(11).random_sample((B, S, H, D)).astype(np.float32) * 2 - 1))
    stream = nnc.Stream(0)
    tq = nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF).upload(bits)
    to = nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF)
    tl = nnc.gpu_tensor([B, H, S])
    grads = [nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF) for _ in range(3)]
    slices = ((0, 0), (17, 9), (31, 15))
    try:
        for causal in (0, 1):
            case = C(BF16, 1, S, S, 1, 1, D, causal, path="flash")
            fwd, bwd = (_cmd(nnc, c, case) for c in (abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD))
            assert nnc.cmd_exec(fwd, None, 0, [tq, tq, tq], [to, tl], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
            assert nnc.cmd_exec(bwd, None, 0, [tq, None, None, tq, tq, tq, None, None, None, to, tl], grads, stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
            stream.wait()
            o, lse = to.download(), tl.download()
            gs = [g.download() for g in grads]
            model = ar.Model("flash", BF16)
            for b, h in slices:
                x = cr.from_bits16(bits[b:b + 1, :, h:h + 1, :], BF16)
                f = ar.Forward(x, x, x, case.scale, causal, None, model)
                oo, uo, ll, ul = f.out()
                ob = o[b:b + 1, :, h:h + 1, :].view(np.uint16)
                what = "bench causal=%d (b=%d, h=%d)" % (causal, b, h)
                _record("bench forward O bf16", ar.check(cr.from_bits16(ob, BF16), oo, uo, ("rne", BF16), what + " O"), what)
                _record("bench forward LSE", ar.check_lse(lse[b:b + 1, h:h + 1].astype(np.float64), ll, ul, what + " LSE"), what)
                bk = ar.Backward(f, x, o16=cr.from_bits16(ob, BF16))
                for g, (want, unit), name in zip(gs, bk.out(), ("dq", "dk", "dv")):
                    got = cr.from_bits16(g[b:b + 1, :, h:h + 1, :].view(np.uint16), BF16)
                    _record("bench backward bf16", ar.check(got, want, unit, ("rne", BF16), what + " " + name), what + " " + name)
    finally:
        for t in [tq, to, tl] + grads + [stream]:
            t.free()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [FP32, BF16])
def test_unify_head_projection(gpu, dtype):
    """The fused "unify head" output d = concat_heads(c) w^T + bias: c held to the attention bound, d to contract_ref's GEMM bound with
    the GPU's own c as the operand, so the projection's error is separated from the attention's."""
    nnc = gpu
    case = C(dtype, 2, 96, 128, 2, 2, 64, 0, path="fp32" if dtype == FP32 else "flash")
    d = operands(case)
    B, S, H, D = case.B, case.Sq, case.H, case.D
    r = np.random.RandomState(7)
    w = _grid((r.random_sample((H * D, H * D)) * 0.2 - 0.1).astype(np.float32), dtype)
    bias = cr.untie_tf32((r.random_sample((H * D,)) * 2 - 1).astype(np.float32))
    stream = nnc.Stream(0)
    ts = [nnc.gpu_tensor(list(d[n].shape), NHWC, DT[dtype]) for n in ("q", "k", "v")]
    tw = nnc.gpu_tensor([H * D, H * D], NHWC, DT[dtype])
    for t, a in zip(ts + [tw], [d["q"], d["k"], d["v"], w]):
        bb = _bits(a, dtype)
        t.upload(bb.view(np.float32) if dtype == FP32 else bb)
    tb = nnc.gpu_tensor([H * D]).upload(bias)
    td, tc = nnc.gpu_tensor([B, S, H * D], NHWC, DT[dtype]), nnc.gpu_tensor([B, S, H, D], NHWC, DT[dtype])
    try:
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case)
        assert nnc.cmd_exec(cmd, None, 0, ts + [None, tw, tb], [td, None, tc], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        cb, db = (t.download().view(_np_bits(dtype)) for t in (tc, td))
    finally:
        for t in ts + [tw, tb, td, tc, stream]:
            t.free()
    fp = case.plans()[0]
    o, uo, _, _ = forward_oracle(case, d, fp).out()
    c = _values(cb, dtype)
    ar.check(c, o, uo, ar.rounding_of(fp["path"], dtype), "%s: per-head attention" % case)
    mode = cr.X3 if dtype == FP32 else BF16
    y, s = cr.gemm(c.reshape(B * S, H * D), w.astype(np.float64), 0, 1, bias.astype(np.float64))
    cr.check(_values(db, dtype).reshape(B * S, H * D), y, s, H * D, mode, FP32 if dtype == FP32 else BF16, "unified output")
