"""SCALED_DOT_PRODUCT_ATTENTION_BACKWARD through the unify-head projection: inputs (g, -, -, q, k, v, -, w, [bias], y, [lse], c), outputs
(dq, dk, dv, -, dw, [dbias]), with y = concat_heads(c) w^T + bias the forward's output and c its per-head attention.

The call is GEMM_BACKWARD(transpose_b) on g, c_flat and w -- dc = g w, dw (+)= g^T c_flat, dbias (+)= the column sums of g -- followed by
the backward without weights on dO = dc, O = c and the saved log-sum-exp.  So it is checked for bit identity against exactly those two
commands on the same stream, and against the float64 oracles with the two error sources kept apart: dw and dbias to contract_ref's GEMM
bound on the GPU's own g and c, dq / dk / dv to attention_ref's backward bound on the GPU's own dc.

CPU: the planner (GEMM-backward launches plus the attention backward's) on hand-worked shapes, and the refusal table restated (a record of
the table, which the GPU checks against the library).
GPU: the case table (fp32, bf16, fp16; D 64 / 128 fused, 160 wide under algorithm 1, D = 100 and Dv != D functional, fp32 composed; GQA,
causal, 3-d, ragged S, with and without bias and the saved LSE) with guard buffers, reruns and launch counts; ACCUMULATE_OUTPUT; every
refusal with no launch and its outputs untouched; algorithm 2; autotuning; and integration/cnnp_fused_attention_train on the drop-in build."""
import json
import os
import subprocess

import numpy as np
import pytest

from ccv_b200 import abi
from tests import attention_ref as ar
from tests import contract_ref as cr
from tests.attention_ref import BF16, FP16, FP32
from tests.test_parity_attention_paths import DT, NHWC, SENTINEL, Case, _bits, _np_bits, _values, backward_oracle, operands
from tests.test_parity_attention_wide import add_flush_terms, forward_oracle, plan_backward, wide_blocks

COMPOSED, FLASH, FLASH_MASK = 0, abi.CCV_NNC_SM100_SDPA_ALGO_FLASH, abi.CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK
KIND = {FP32: 0, BF16: 1, FP16: 2}
INVALID, NO_KERNEL = abi.CCV_NNC_EXEC_INVALID, abi.CCV_NNC_EXEC_NO_KERNEL


# ------------------------------------------------------------------------------------------------ planner
def plan(dtype, B, H, Hk, Sq, Sk, D, Dv, bias, saved, algorithm, sms):
    """(path, launches) of one call: GEMM_BACKWARD's (dbias column sums: two passes when n % 4 == 0, dw = g^T c, dc = g w; contract_ref's
    planner gives each GEMM's kernels) plus the attention backward's (test_parity_attention_wide's planner, algorithm 0's outside the wide
    heads).  The fp32 backward takes no saved output, so `saved` does not change its plan."""
    n, rows = H * Dv, B * Sq
    gemm = cr.plan("gemm", KIND[dtype], sms, M=n, N=n, K=rows)["kernels"] + cr.plan("gemm", KIND[dtype], sms, M=rows, N=n, K=n)["kernels"]
    colsum = (2 if n % 4 == 0 else 1) if bias else 0
    a = plan_backward(dtype, B, H, Hk, Sq, Sk, D, Dv, saved=saved and dtype != FP32, algorithm=algorithm)
    return dict(path=a["path"], launches=colsum + gemm + a["launches"])


def test_planner_on_hand_worked_shapes():
    # bf16 B = 4, S = 2048, H = 16, D = 128 on 132 SMs: dc is 1024 tiles (no split), dw 256 tiles over 128 k-iterations (a split does not
    # shorten the two waves), the column sums two passes, the fused backward prep + dK/dV + dQ (+ the forward without the saved LSE)
    assert plan(BF16, 4, 16, 16, 2048, 2048, 128, 128, True, True, COMPOSED, 132) == dict(path="fused", launches=1 + 1 + 2 + 3)
    assert plan(BF16, 4, 16, 16, 2048, 2048, 128, 128, False, False, COMPOSED, 132) == dict(path="fused", launches=1 + 1 + 4)
    # fp32 B = 2, S = 96, H = 2, D = 64: one tile each, 7 launches per (b, h) in the composed backward
    assert plan(FP32, 2, 2, 1, 96, 128, 64, 64, True, False, COMPOSED, 132) == dict(path="fp32", launches=2 + 1 + 1 + 28)
    # D = 160: the wide kernels under algorithm 1, the functional form under algorithm 0
    assert plan(FP16, 1, 2, 2, 64, 96, 160, 160, False, True, FLASH, 132)["path"] == "fused"
    assert plan(FP16, 1, 2, 2, 64, 96, 160, 160, False, False, COMPOSED, 132)["path"] == "func"
    for c in CASES:
        assert c.plan(132)["path"] == c.path, c


# ------------------------------------------------------------------------------------------------ the refusal table
# Each entry changes one thing of a valid call; the backward returns INVALID before any launch.  "view": that operand as a tensor view.
REFUSALS = [
    ("mask", dict(mask=True)),
    ("outputs[3] set", dict(out3=True)),
    ("palettized weights", dict(w_qx=True)),
    ("bias without weights", dict(no_w=True)),
    ("no c", dict(no_c=True)),
    ("dbias without bias", dict(no_bias=True)),
    ("g a view", dict(view="g")),
    ("c a view", dict(view="c")),
    ("w a view", dict(view="w")),
    ("dw a view", dict(view="dw")),
    ("dbias a view", dict(view="dbias")),
    ("w of another type", dict(w_type=BF16)),
    ("dw of another type", dict(dw_type=FP32)),
    ("w [n, n - 8]", dict(w_cols=-8)),
    ("g [B, S, n + 8]", dict(g_cols=8)),
    ("dw [n, n - 8]", dict(dw_cols=-8)),
    ("dbias of n - 8", dict(dbias_cols=-8)),
    ("c with another Sq", dict(c_rows=-1)),
    ("lse of another size", dict(lse_rows=-1)),
]


def refused(spec, dtype=FP16):
    """the restated rules of the unify-head backward for the base call of test_refusals with one change `spec`"""
    if spec.get("mask") or spec.get("out3") or spec.get("w_qx") or spec.get("no_w") or spec.get("no_c") or spec.get("no_bias"):
        return True
    if spec.get("view") in ("g", "c", "w", "dw", "dbias"):
        return True
    if spec.get("w_type", dtype) != dtype or spec.get("dw_type", dtype) != dtype:
        return True
    return any(spec.get(k, 0) != 0 for k in ("w_cols", "g_cols", "dw_cols", "dbias_cols", "c_rows", "lse_rows"))


def test_refusal_table():
    """Documents the table test_refusals runs on the GPU: every entry is one of the restated rules, the base call none.  It checks the
    table, not the library; the library's refusals are checked by test_refusals."""
    assert not refused({})
    for name, spec in REFUSALS:
        assert refused(spec), name


# ------------------------------------------------------------------------------------------------ the case table
class UCase(object):
    def __init__(self, case, algorithm=COMPOSED, bias=True, saved=True, bias_f32=True):
        self.case, self.algorithm, self.bias, self.saved, self.bias_f32 = case, algorithm, bias, saved and case.lse_ok, bias_f32
        self.path = "fused" if case.path == "flash" else case.path

    def __repr__(self):
        return "%r alg%d%s%s" % (self.case, self.algorithm, " bias" + ("32" if self.bias_f32 else "16") if self.bias else "", " saved" if self.saved else "")

    def plan(self, sms):
        c = self.case
        return plan(c.dtype, c.B, c.H, c.Hk, c.Sq, c.Sk, c.D, c.Dv, self.bias, self.saved, self.algorithm, sms)


def _case(*a, **kw):
    c = Case(*a, **kw)
    # the forward gives the log-sum-exp only on the flash kernels (the wide ones under algorithm 1)
    c.lse_ok = c.path == "flash"
    return c


C = _case
CASES = [
    UCase(C(BF16, 2, 128, 128, 4, 4, 64, 0, path="flash")),
    UCase(C(FP16, 2, 100, 160, 2, 1, 128, 1, "peaked", path="flash"), saved=False),           # GQA, causal, ragged S
    UCase(C(BF16, 1, 77, 77, 1, 1, 128, 1, three_d=True, path="flash"), bias=False),          # 3-d
    UCase(C(FP16, 2, 128, 128, 4, 4, 64, 1, path="flash"), bias_f32=False),                    # a 16-bit bias and dbias
    UCase(C(FP16, 1, 64, 96, 2, 2, 160, 0, path="flash"), FLASH),                              # wide
    UCase(C(BF16, 2, 65, 65, 2, 1, 160, 1, path="flash"), FLASH, bias=False, saved=False),    # wide, GQA, causal
    UCase(C(FP16, 1, 63, 129, 2, 2, 100, 0, path="func")),                                     # functional form: D % 8 != 0
    UCase(C(BF16, 2, 64, 64, 2, 2, 64, 1, Dv=32, path="func"), bias=False),                    # functional form: Dv != D
    UCase(C(FP32, 2, 96, 128, 2, 1, 64, 1, path="fp32")),                                      # fp32, GQA, causal
    UCase(C(FP32, 1, 65, 65, 1, 1, 32, 0, three_d=True, path="fp32"), bias=False),             # fp32, 3-d, ragged
]
CASE_IDS = [repr(c) for c in CASES]


def projection_operands(u):
    """g [B, S, n] and w [n, n] on the dtype's grid.  fp32: quarter and eighth integers in [-2, 2], so that every dc = g w is exact in
    TF32 (at most 11 significant bits for n <= 256) and the TF32 operands of the attention backward hold no rounding tie."""
    c = u.case
    n = c.H * c.Dv
    r = np.random.RandomState(n * 131 + c.Sq)
    if c.dtype == FP32:
        g = (r.randint(-2, 3, (c.B, c.Sq, n)) / 4.0).astype(np.float32)
        w = (r.randint(-2, 3, (n, n)) / 8.0).astype(np.float32)
    else:
        g = cr.rne16(r.random_sample((c.B, c.Sq, n)) * 2 - 1, c.dtype).astype(np.float32)
        w = cr.rne16((r.random_sample((n, n)) * 2 - 1) / np.sqrt(n), c.dtype).astype(np.float32)
    bias = (r.random_sample((n,)) * 2 - 1).astype(np.float32)
    bias = cr.untie_tf32(bias) if u.bias_f32 or c.dtype == FP32 else cr.rne16(bias, c.dtype).astype(np.float32)
    return g, w, bias


# ------------------------------------------------------------------------------------------------ GPU helpers
def _cmd(nnc, cmd_id, case, algorithm):
    c = nnc._simple(cmd_id, algorithm=algorithm)
    c.info.scaled_dot_product_attention.scale = case.scale
    c.info.scaled_dot_product_attention.is_causal = case.causal
    c.info.scaled_dot_product_attention.deterministic = 1
    return c


def _shape(case, S, H, D):
    return [case.B, S, D] if case.three_d else [case.B, S, H, D]


class Guarded(object):
    """a tensor inside a sentinel-filled allocation with 64 guard elements on each side"""

    def __init__(self, nnc, dims, dtype, bits=None):
        self.dims, self.dtype, self.count = list(dims), dtype, int(np.prod(dims))
        self.host = np.full((self.count + 128,), SENTINEL[dtype], _np_bits(dtype))
        if bits is not None:
            self.host[64:64 + self.count] = np.asarray(bits).reshape(-1)
        self.base = nnc.gpu_tensor([self.count + 128], NHWC, DT[dtype])
        self.t = nnc.gpu_tensor(self.dims, NHWC, DT[dtype], ptr=self.base.data_ptr + 64 * self.host.itemsize)
        self.arm()

    def arm(self, bits=None):
        if bits is not None:
            self.host[64:64 + self.count] = np.asarray(bits).reshape(-1)
        self.base.upload(self.host.view({FP32: np.float32, FP16: np.float16}.get(self.dtype, np.uint16)))

    def result(self):
        got = self.base.download().view(_np_bits(self.dtype))
        assert np.array_equal(got[:64], self.host[:64]) and np.array_equal(got[64 + self.count:], self.host[64 + self.count:]), "guard elements overwritten"
        return got[64:64 + self.count].reshape(self.dims)

    def alias(self, nnc, dims):
        """another header of the same memory"""
        return nnc.gpu_tensor(list(dims), NHWC, DT[self.dtype], ptr=self.t.data_ptr)

    def free(self):
        self.t.free()
        self.base.free()


class Call(object):
    """operands of one unify-head backward: the forward (with weights) has run on the GPU and left y, lse and c"""

    def __init__(self, nnc, u):
        c, self.nnc, self.u = u.case, nnc, u
        self.d = operands(c)
        self.g, self.w, self.bias = projection_operands(u)
        dt = c.dtype
        self.n, self.rows = c.H * c.Dv, c.B * c.Sq
        self.stream = nnc.Stream(0)
        self.live = []
        T = lambda dims, a, t=dt: self._keep(Guarded(nnc, dims, t, _bits(a, t)))
        self.q, self.k, self.v = (T(list(self.d[x].shape), self.d[x]) for x in ("q", "k", "v"))
        self.gy, self.tw = T([c.B, c.Sq, self.n], self.g), T([self.n, self.n], self.w)
        bdt = FP32 if u.bias_f32 or dt == FP32 else dt
        self.tb = T([self.n], self.bias, bdt) if u.bias else None
        self.y = self._keep(Guarded(nnc, [c.B, c.Sq, self.n], dt))
        self.c = self._keep(Guarded(nnc, _shape(c, c.Sq, c.H, c.Dv), dt))
        self.lse = self._keep(Guarded(nnc, [c.B, c.H, c.Sq], FP32)) if u.saved else None
        fwd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, c, u.algorithm)
        st = nnc.cmd_exec(fwd, None, 0, [self.q.t, self.k.t, self.v.t, None, self.tw.t, self.tb.t if self.tb else None],
                          [self.y.t, self.lse.t if self.lse else None, self.c.t], self.stream)
        self.stream.wait()
        assert st == 0, "%s: forward status %d, %s" % (u, st, nnc.lib().ccv_nnc_sm100_last_error())
        self.c_bits = self.c.result()
        self.outs = [self._keep(Guarded(nnc, _shape(c, S, H, D), dt)) for S, H, D in ((c.Sq, c.H, c.D), (c.Sk, c.Hk, c.D), (c.Sk, c.Hk, c.Dv))]
        self.dw = self._keep(Guarded(nnc, [self.n, self.n], dt))
        self.db = self._keep(Guarded(nnc, [self.n], bdt)) if u.bias else None

    def _keep(self, x):
        self.live.append(x)
        return x

    def inputs(self):
        return [self.gy.t, None, None, self.q.t, self.k.t, self.v.t, None, self.tw.t, self.tb.t if self.tb else None, self.y.t,
                self.lse.t if self.lse else None, self.c.t]

    def outputs(self):
        return [o.t for o in self.outs] + [None, self.dw.t, self.db.t if self.db else None]

    def results(self):
        return [o.result() for o in self.outs + [self.dw] + ([self.db] if self.db else [])]

    def arm_outputs(self, dw_bits=None, db_bits=None):
        for o in self.outs:
            o.arm()
        self.dw.arm(dw_bits)
        if self.db:
            self.db.arm(db_bits)

    def backward(self, algorithm=None, flags=0, inputs=None, outputs=None, cmd=None):
        """(status, launches) of one backward call"""
        u = self.u
        cmd = cmd or _cmd(self.nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, u.case, u.algorithm if algorithm is None else algorithm)
        l0 = self.nnc.launch_count()
        st = self.nnc.cmd_exec(cmd, None, flags, self.inputs() if inputs is None else inputs, self.outputs() if outputs is None else outputs, self.stream)
        self.stream.wait()
        return st, self.nnc.launch_count() - l0

    def sequence(self, flags=0):
        """GEMM_BACKWARD (transpose_b) on (g, c_flat, w) -> (dc, dw, dbias), then the backward without weights on dc; (dc bits, launches).
        ACCUMULATE_OUTPUT goes to the parameter gradients only, as a call of its own (dc is written afresh)."""
        nnc, u, c = self.nnc, self.u, self.u.case
        dc = Guarded(nnc, _shape(c, c.Sq, c.H, c.Dv), c.dtype)
        g2, c2, dc2 = self.gy.alias(nnc, [self.rows, self.n]), self.c.alias(nnc, [self.rows, self.n]), dc.alias(nnc, [self.rows, self.n])
        try:
            gemm = nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
            l0 = nnc.launch_count()
            if flags:
                assert nnc.cmd_exec(gemm, None, flags, [g2, c2, self.tw.t], [None, self.dw.t, self.db.t if self.db else None], self.stream) == 0
                assert nnc.cmd_exec(gemm, None, 0, [g2, c2, self.tw.t], [dc2, None, None], self.stream) == 0
            else:
                assert nnc.cmd_exec(gemm, None, 0, [g2, c2, self.tw.t], [dc2, self.dw.t, self.db.t if self.db else None], self.stream) == 0
            bwd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, c, u.algorithm)
            st = nnc.cmd_exec(bwd, None, 0, [dc.t, None, None, self.q.t, self.k.t, self.v.t, None, None, None, self.c.t, self.lse.t if self.lse else None],
                              [o.t for o in self.outs], self.stream)
            self.stream.wait()
            assert st == 0, "%s: the backward without weights on dc: %d, %s" % (u, st, nnc.lib().ccv_nnc_sm100_last_error())
            return dc.result(), nnc.launch_count() - l0
        finally:
            for t in (g2, c2, dc2):
                t.free()
            dc.free()

    def free(self):
        for x in self.live:
            x.free()
        self.stream.free()


# ------------------------------------------------------------------------------------------------ GPU: the case table
@pytest.mark.gpu
@pytest.mark.parametrize("u", CASES, ids=CASE_IDS)
def test_unify_back_case(gpu, u):
    nnc = gpu
    c = u.case
    p = u.plan(cr.device_sms())
    call = Call(nnc, u)
    try:
        runs = []
        for _ in range(2):
            call.arm_outputs()
            st, launches = call.backward()
            assert st == 0, "%s: status %d, %s" % (u, st, nnc.lib().ccv_nnc_sm100_last_error())
            assert launches == p["launches"], "%s: %d launches, planned %d" % (u, launches, p["launches"])
            runs.append(call.results())
        names = ["dq", "dk", "dv", "dw", "dbias"]
        for a, b, n in zip(runs[0], runs[1], names):
            assert np.array_equal(a, b), "%s: two runs differ in %s" % (u, n)
        call.arm_outputs()
        dc_bits, seq_launches = call.sequence()
        seq = call.results()
        for a, b, n in zip(runs[0], seq, names):
            assert np.array_equal(a, b), "%s: %s differs from GEMM_BACKWARD followed by the backward without weights" % (u, n)
        assert seq_launches == p["launches"], "%s: the two-command sequence took %d launches, the fused call %d" % (u, seq_launches, p["launches"])
        cb = call.c_bits
    finally:
        call.free()
    dt = c.dtype
    # dw, dbias: the GEMM bound on the GPU's own g and c
    g64 = call.g.reshape(call.rows, call.n).astype(np.float64)
    c64 = _values(cb, dt).reshape(call.rows, call.n)
    y, s = cr.gemm(g64, c64, 1, 0)
    cr.check(_values(runs[0][3], dt).reshape(call.n, call.n), y, s, call.rows, cr.X3 if dt == FP32 else dt, dt, "%s: dw" % u)
    if u.bias:
        bdt = FP32 if u.bias_f32 or dt == FP32 else dt
        cr.check(_values(runs[0][4], bdt), g64.sum(0), np.abs(g64).sum(0), call.rows, FP32, bdt, "%s: dbias" % u)
    # dq, dk, dv: the attention backward's bound with dO = the GPU's own dc
    dc = _values(dc_bits, dt).astype(np.float32).reshape(call.d["do"].shape)
    d = dict(call.d, do=dc)
    bp = plan_backward(dt, c.B, c.H, c.Hk, c.Sq, c.Sk, c.D, c.Dv, saved=u.saved, algorithm=u.algorithm)
    o16 = _values(cb, dt) if bp["path"] == "fused" else None
    wide = u.algorithm == FLASH and c.D > 128
    if wide:
        with wide_blocks():
            b = backward_oracle(c, d, bp, o16=o16)
            add_flush_terms(forward_oracle(c, d, bp), b, dc, o16, c.three_d)
    else:
        b = backward_oracle(c, d, bp, o16=o16)
    rnd = ar.rounding_of(bp["path"], dt)
    for bits, (want, unit), n in zip(runs[0][:3], b.out(), ("dq", "dk", "dv")):
        ar.check(ar.as4(_values(bits, dt), c.three_d), want, unit, rnd, "%s: %s" % (u, n))


# ------------------------------------------------------------------------------------------------ GPU: single checks
BASE = UCase(C(FP16, 2, 64, 96, 2, 1, 64, 1, path="flash"))


@pytest.mark.gpu
def test_accumulate_output(gpu):
    """dw and dbias accumulate under CCV_NNC_ACCUMULATE_OUTPUT as GEMM_BACKWARD's do, bit for bit; dq, dk, dv are written as without it"""
    nnc = gpu
    call = Call(nnc, BASE)
    try:
        r = np.random.RandomState(5)
        old_w = _bits(cr.rne16(r.random_sample((call.n, call.n)) - 0.5, FP16), FP16)
        old_b = _bits(cr.untie_tf32(r.random_sample((call.n,)).astype(np.float32) - 0.5), FP32)
        call.arm_outputs()
        assert call.backward()[0] == 0
        plain = call.results()
        call.arm_outputs(old_w, old_b)
        assert call.backward(flags=abi.CCV_NNC_ACCUMULATE_OUTPUT)[0] == 0
        acc = call.results()
        call.arm_outputs(old_w, old_b)
        call.sequence(flags=abi.CCV_NNC_ACCUMULATE_OUTPUT)
        seq = call.results()
    finally:
        call.free()
    for a, b, n in zip(acc, seq, ("dq", "dk", "dv", "dw", "dbias")):
        assert np.array_equal(a, b), "accumulated %s differs from GEMM_BACKWARD's" % n
    for a, b, n in zip(acc[:3], plain[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b), "%s accumulated" % n
    assert not np.array_equal(acc[3], plain[3]) and not np.array_equal(acc[4], plain[4])
    got = _values(acc[4], FP32)
    assert np.allclose(got, _values(plain[4], FP32) + _values(old_b, FP32), rtol=1e-6, atol=1e-6)


@pytest.mark.gpu
def test_refusals(gpu):
    """each entry of the refusal table returns INVALID with no launch, and dq, dk, dv, dw, dbias keep their sentinels"""
    nnc = gpu
    call = Call(nnc, BASE)
    c = BASE.case
    extra = []

    def T(dims, dtype=FP16):
        t = nnc.gpu_tensor(list(dims), NHWC, DT[dtype])
        extra.append(t)
        return t

    try:
        for name, spec in REFUSALS:
            ins, outs = call.inputs(), call.outputs()
            if spec.get("mask"):
                ins[6] = T([c.Sq, c.Sk], FP32)
            if spec.get("out3"):
                outs[3] = T([c.Sq, c.Sk], FP32)
            if spec.get("w_qx"):
                t = nnc.gpu_palettized_tensor([call.n, call.n], abi.CCV_16F, 6, 64)
                extra.append(t)
                ins[7] = t
            if spec.get("no_w"):
                ins[7] = None
            if spec.get("no_c"):
                ins[11] = None
            if spec.get("no_bias"):
                ins[8] = None
            if "view" in spec:
                slot = {"g": (ins, 0), "c": (ins, 11), "w": (ins, 7), "dw": (outs, 4), "dbias": (outs, 5)}[spec["view"]]
                src = slot[0][slot[1]]
                dims = src.dims
                strides = [int(np.prod(dims[i + 1:])) for i in range(len(dims))]
                v = nnc.tensor_view_new(src, dims, [0] * 12, strides + [0] * (12 - len(dims)))
                extra.append(v)
                slot[0][slot[1]] = v
            if "w_type" in spec:
                ins[7] = T([call.n, call.n], spec["w_type"])
            if "dw_type" in spec:
                outs[4] = T([call.n, call.n], spec["dw_type"])
            if spec.get("w_cols"):
                ins[7] = T([call.n, call.n + spec["w_cols"]])
            if spec.get("g_cols"):
                ins[0] = T([c.B, c.Sq, call.n + spec["g_cols"]])
            if spec.get("dw_cols"):
                outs[4] = T([call.n, call.n + spec["dw_cols"]])
            if spec.get("dbias_cols"):
                outs[5] = T([call.n + spec["dbias_cols"]], FP32)
            if spec.get("c_rows"):
                ins[11] = T(_shape(c, c.Sq + spec["c_rows"], c.H, c.Dv))
            if spec.get("lse_rows"):
                ins[10] = T([c.B, c.H, c.Sq + spec["lse_rows"]], FP32)
            call.arm_outputs()
            st, launches = call.backward(inputs=ins, outputs=outs)
            assert st == INVALID and launches == 0, "%s: status %d, %d launches" % (name, st, launches)
            for o in call.outs + [call.dw, call.db]:
                assert np.array_equal(o.result().reshape(-1), o.host[64:64 + o.count]), "%s: an output was written" % name
    finally:
        for t in extra:
            t.free()
        call.free()


@pytest.mark.gpu
def test_algorithm_2_and_autotune(gpu):
    """algorithm 2 is forward only: NO_KERNEL, no launch; ccv_nnc_cmd_autotune returns an algorithm that runs the call, bit-identical to
    running that algorithm directly"""
    nnc = gpu
    call = Call(nnc, BASE)
    try:
        call.arm_outputs()
        assert call.backward(algorithm=FLASH_MASK) == (NO_KERNEL, 0)
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, BASE.case, -1)
        tuned = nnc.cmd_autotune(cmd, None, 0, call.inputs(), call.outputs(), call.stream)
        assert tuned.algorithm in (COMPOSED, FLASH), tuned.algorithm
        call.arm_outputs()
        st, _ = call.backward(cmd=tuned)
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        a = call.results()
        call.arm_outputs()
        assert call.backward(algorithm=tuned.algorithm)[0] == 0
        for x, y in zip(a, call.results()):
            assert np.array_equal(x, y)
    finally:
        call.free()


# ------------------------------------------------------------------------------------------------ GPU: through the reference's model layer
TRAIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "integration", "_build", "cnnp_fused_attention_train")


# The reference's own backward bitmask (scaled_dot_product_attention/ccv_nnc_scaled_dot_product_attention.c:26-37) accepts inputs
# (g, q, k, v, y, lse) whenever dq, dk and dv are among the outputs -- its third clause tests outputs & 7 only -- so its autograd prunes w,
# bias and c from the node although dw and dbias are asked for.  The backward then cannot form dc = g w; it returns INVALID and the weights
# never move.  Strict: this test reports the day the reference's bitmask keeps w and c.
@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="the reference's autograd drops w, bias and c from the fused backward (its bitmask's third clause)")
@pytest.mark.parametrize("dtype", ["32f", "16f"])
def test_cnnp_fused_attention_trains_on_the_dropin_build(gpu, dtype):
    """integration/cnnp_fused_attention_train.c on libccv_dropin.so: the reference's ccv_cnnp_scaled_dot_product_attention with fused,
    trainable unify-head weights and bias, trained with evaluate / backward / apply_gradients.  No command of the graph returns anything
    but success (the graph runner prints "Invalid Status" otherwise), the loss falls, and the step-1 weights gradient matches the unfused
    twin's (attention, reshape, ccv_cnnp_dense from the same weights) within the GEMM bound the program computes."""
    if not os.path.exists(TRAIN):
        pytest.skip("integration/_build is not built")
    p = subprocess.run([TRAIN, "--dtype", dtype, "--steps", "4"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    out = p.stdout.decode(errors="replace")
    assert p.returncode == 0, (out[-1500:], p.stderr.decode(errors="replace")[-1500:])
    assert "Invalid Status" not in out, [line for line in out.splitlines() if "Invalid Status" in line][:5]
    r = json.loads(out.strip().splitlines()[-1])
    assert r["dtype"] == dtype
    losses = r["losses"]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], r
    assert 0 <= r["dw_max_bound_ratio"] <= 1.0, r
