"""SCALED_DOT_PRODUCT_ATTENTION algorithm 1 (CCV_NNC_SM100_SDPA_ALGO_FLASH): 16-bit heads with 128 < D = Dv <= 256 on the wide flash
kernels of ccv_b200/csrc/sm100_fmha_wide.cu, against the float64 oracle and rounding-level bounds of tests/attention_ref.py.

The wide kernels compute as the D <= 128 flash / fused kernels do (P rounded to 16 bits before its MMAs, the fused backward's delta from
the stored O), with 64-key blocks in the forward; the oracle's block count follows that while the wide oracles run.  Every other call
under algorithm 1 (D <= 128, masks, Dv != D, D > 256, D % 8 != 0, fp32) is algorithm 0's, and the planner below says so.

CPU: the planner restated for algorithm 1 on hand-worked shapes, and the bounds rejecting defects of a 256-feature head.
GPU: the case table under algorithm 1 (launch counts as planned, O / LSE / dq / dk / dv within the bounds, two runs bit-identical, the
saved o / lse backward equal to the recomputed one), GQA / batch / aliasing / packed-QKV-view identities, D = 160 against the same call
zero-padded to 256, algorithm 1 at D <= 128 against algorithm 0, autotuning, and one 16384-token causal call."""
import contextlib

import numpy as np
import pytest

from ccv_b200 import abi
from tests import attention_ref as ar
from tests import contract_ref as cr
from tests.attention_ref import BF16, FP16, FP32
from tests.test_parity_attention_paths import (Buf, Case, _in_tensors, _out_buf, _shape, _sub, _values, backward_oracle,
                                               forward_oracle, operands)

FLASH = abi.CCV_NNC_SM100_SDPA_ALGO_FLASH
WIDE_BLOCK = 64  # keys per block of the wide forward


# ------------------------------------------------------------------------------------------------ planner (algorithm 1)
def _wide_ok(dtype, D, Dv, H, Hk, mask, aligned):
    return dtype != FP32 and not mask and 128 < D <= 256 and D % 8 == 0 and Dv == D and H % Hk == 0 and aligned


def plan_forward(dtype, B, H, Hk, Sq, Sk, D, Dv, mask=False, view=False, lse=False, aligned=True, algorithm=FLASH):
    """algorithm 1: the wide flash kernel (one launch) where it applies, otherwise exactly algorithm 0's plan"""
    if algorithm == FLASH and _wide_ok(dtype, D, Dv, H, Hk, mask, aligned):
        return dict(path="flash", launches=1)
    return ar.plan_forward(dtype, B, H, Hk, Sq, Sk, D, Dv, mask=mask, view=view, lse=lse, aligned=aligned)


def plan_backward(dtype, B, H, Hk, Sq, Sk, D, Dv, saved=False, view=False, aligned=True, algorithm=FLASH):
    """algorithm 1: prep + dK/dV + dQ on the wide kernels (+ the wide forward when o / lse are not passed)"""
    if algorithm == FLASH and _wide_ok(dtype, D, Dv, H, Hk, False, aligned):
        return dict(path="fused", launches=3 if saved else 4)
    return ar.plan_backward(dtype, B, H, Hk, Sq, Sk, D, Dv, saved=saved, view=view, aligned=aligned)


@contextlib.contextmanager
def wide_blocks():
    """the oracle's forward block count (rescales of the running max, the alpha1 defect) at the wide kernel's 64-key blocks"""
    saved = ar.FM_BLOCK
    ar.FM_BLOCK = WIDE_BLOCK
    try:
        yield
    finally:
        ar.FM_BLOCK = saved


def test_planner_for_algorithm_1_on_hand_worked_shapes():
    # D = 160 with the log-sum-exp: algorithm 0 refuses it, algorithm 1 runs one wide flash launch
    assert ar.plan_forward(BF16, 1, 2, 2, 64, 64, 160, 160, lse=True)["path"] == "refused"
    assert plan_forward(BF16, 1, 2, 2, 64, 64, 160, 160, lse=True) == dict(path="flash", launches=1)
    assert plan_forward(FP16, 4, 16, 16, 4096, 4096, 256, 256, view=True) == dict(path="flash", launches=1)
    # D = 160 backward on views: fused, prep + dK/dV + dQ with the saved o / lse, the forward first without
    assert ar.plan_backward(BF16, 1, 2, 2, 64, 64, 160, 160, view=True)["path"] == "refused"
    assert plan_backward(BF16, 1, 2, 2, 64, 64, 160, 160, view=True, saved=True) == dict(path="fused", launches=3)
    assert plan_backward(BF16, 1, 2, 2, 64, 64, 160, 160, view=True) == dict(path="fused", launches=4)
    # outside the wide kernels: algorithm 0's plan, call for call
    for a in [(BF16, 1, 2, 2, 64, 64, 264, 264), (FP16, 1, 2, 2, 64, 64, 164, 164), (BF16, 1, 2, 2, 64, 64, 160, 128),
              (FP32, 1, 2, 2, 64, 64, 160, 160), (BF16, 2, 4, 2, 63, 129, 64, 64), (FP16, 1, 2, 2, 64, 64, 128, 128)]:
        assert plan_forward(*a) == ar.plan_forward(*a), a
        assert plan_backward(*a) == ar.plan_backward(*a), a
    assert plan_forward(BF16, 1, 2, 2, 64, 96, 160, 160, mask=True) == ar.plan_forward(BF16, 1, 2, 2, 64, 96, 160, 160, mask=True)
    assert plan_forward(BF16, 1, 2, 2, 64, 64, 264, 264) == dict(path="func", launches=3 + 3 * 2 + 1, gemm_s="tf32", gemm_p="tf32")
    assert plan_forward(BF16, 1, 2, 2, 64, 64, 264, 264, lse=True)["path"] == "refused"
    # algorithm 0 (and the default -1) keep today's plan for the wide heads
    assert plan_forward(BF16, 1, 2, 2, 64, 64, 160, 160, algorithm=0)["path"] == "func"
    for c in WIDE:
        fp, bp = plans(c)
        assert fp["path"] == "flash" and bp["path"] == "fused", c


# ------------------------------------------------------------------------------------------------ the case table
C = Case
WIDE = [
    C(BF16, 1, 1, 1024, 4, 1, 256, 1, path="flash"),                       # decode: Sq = 1, causal, GQA 4
    C(FP16, 2, 333, 200, 4, 2, 160, 1, "peaked", view=True, path="flash"), # Sq > Sk causal: fully masked rows, GQA 2
    C(BF16, 1, 65, 1024, 8, 1, 192, 1, "rising", path="flash"),            # Sq < Sk causal, every block rescales, GQA 8
    C(FP16, 1, 129, 129, 2, 2, 136, 0, "flat", "small", path="flash"),
    C(BF16, 2, 127, 63, 2, 1, 224, 1, "flat", "one", view=True, path="flash"),
    C(FP16, 1, 1024, 1024, 2, 2, 256, 1, "falling", path="flash"),         # fp16 P subnormal, then zero
    C(BF16, 1, 200, 333, 4, 4, 160, 0, "extreme", path="flash"),
    C(FP16, 1, 64, 2, 2, 2, 224, 1, view=True, path="flash"),
    C(BF16, 1, 2, 64, 4, 2, 136, 0, "peaked", path="flash"),
    C(FP16, 1, 128, 65, 8, 2, 256, 0, "extreme", path="flash"),
    C(BF16, 2, 129, 127, 1, 1, 192, 1, "peaked", three_d=True, path="flash"),
    C(FP16, 2, 63, 129, 1, 1, 160, 0, three_d=True, path="flash"),
    C(BF16, 1, 192, 192, 2, 2, 256, 0, "rising", path="flash"),
    C(FP16, 1, 65, 64, 4, 1, 200, 1, path="flash"),
]
WIDE_IDS = [repr(c) for c in WIDE]


def plans(case, saved=False):
    a = (case.dtype, case.B, case.H, case.Hk, case.Sq, case.Sk, case.D, case.Dv)
    return plan_forward(*a, view=case.view, lse=True), plan_backward(*a, saved=saved, view=case.view)


# ------------------------------------------------------------------------------------------------ CPU: the bounds able to fail at D = 256
def _rejects(bad, ref, unit, rnd, what):
    assert not ar.admits(ar.finish(bad, rnd), ref, unit, rnd).all(), "the bound admits %s" % what


@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_bounds_reject_wide_head_defects(dtype):
    """At D = 256 the bounds reject a dropped 64-key block, a dropped 64-feature atom of Q K^T or of V, a wrong GQA head, and (D = 160)
    a store of the padded features 160..255, which lands on the next head's first 96 features of a packed [B, S, H, D] output."""
    case = C(dtype, 1, 200, 200, 4, 2, 256, 0, path="flash")
    d = operands(case)
    fp, _ = plans(case)
    rnd = ar.rounding_of("flash", dtype)
    with wide_blocks():
        f = forward_oracle(case, d, fp)
        o, uo, lse, ul = f.out()
        ar.check(ar.finish(o, rnd), o, uo, rnd, "correct O")
        ar.check_lse(lse, lse, ul, "correct LSE")
        _rejects(forward_oracle(case, d, fp, drop=np.arange(64, 128)).out()[0], o, uo, rnd, "a dropped 64-key block")
        for a in range(4):
            cut = slice(64 * a, 64 * a + 64)
            dq = dict(d, q=d["q"].copy(), k=d["k"].copy())
            dq["q"][..., cut] = 0
            dq["k"][..., cut] = 0
            _rejects(forward_oracle(case, dq, fp).out()[0], o, uo, rnd, "S without feature atom %d" % a)
            bad = o.copy()
            bad[..., cut] = 0
            _rejects(bad, o, uo, rnd, "O without feature atom %d" % a)
        _rejects(forward_oracle(case, d, fp, "gqa_mod").out()[0], o, uo, rnd, "GQA mapped as h % Hk")
        # gradients: a dropped key block shows in dV, a wrong GQA head in dK / dV
        _, bp = plans(case)
        o16 = ar.finish(o, rnd)
        (_, _), (dk, uk), (dv, uv) = backward_oracle(case, d, bp, o16).out()
        _rejects(backward_oracle(case, d, bp, o16, drop=np.arange(64, 128)).out()[2][0], dv, uv, rnd, "dV with a dropped key block")
        _rejects(backward_oracle(case, d, bp, o16, defect="group_head").out()[1][0], dk, uk, rnd, "dK missing a query head")
        # features past D: a 256-wide store of a D = 160 row overwrites features 0..95 of the next head with the padding's zeros
        c160 = C(dtype, 1, 96, 96, 4, 4, 160, 1, path="flash")
        o, uo, _, _ = forward_oracle(c160, operands(c160), plans(c160)[0]).out()
        bad = o.copy()
        bad[:, :, 1:, :96] = 0
        _rejects(bad, o, uo, rnd, "features 160..255 of head h stored over head h + 1")


def add_flush_terms(f, b, do, o16, three_d):
    """ex2.approx.ftz returns 0 for a P below 2^-126, so a key whose P is that small drops out of dS, and with |dP - delta| > 1 its dS
    is not below the format's floor either: the shared bounds model the flush for dV only.  Logits of several hundred over 160+ features
    reach that range; add to the dQ / dK units what the flushed (or, within rounding, nearly flushed) probabilities carry."""
    tiny = (f.p > 0) & (f.p < 2.0 ** -125)
    if not tiny.any():
        return
    dob, ob = ar._bhsd(ar.as4(do, three_d)), ar._bhsd(ar.as4(o16, three_d))
    dp = dob @ np.swapaxes(f.ve, -1, -2)
    dsf = np.where(tiny, np.abs(f.p * (dp - (dob * ob).sum(-1, keepdims=True))), 0.0)
    a = abs(f.scale)
    b.unit_dq = b.unit_dq + a * (dsf @ np.abs(f.ke))
    b.unit_dk = b.unit_dk + a * ar.group_sum(np.swapaxes(dsf, -1, -2) @ np.abs(f.q), f.Hk)


# ------------------------------------------------------------------------------------------------ GPU
def _cmd(nnc, cmd_id, case, algorithm=FLASH):
    c = nnc._simple(cmd_id, algorithm=algorithm)
    c.info.scaled_dot_product_attention.scale = case.scale
    c.info.scaled_dot_product_attention.is_causal = case.causal
    c.info.scaled_dot_product_attention.deterministic = 1
    return c


def run_forward(nnc, case, d, view=False, packed_qkv=False, lse=True, reps=2, algorithm=FLASH):
    """(O bits, LSE or None, launches) under `algorithm`; two runs must agree bit for bit"""
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), packed_qkv)
    ob, to = _out_buf(nnc, _shape(case, case.Sq, case.H, case.Dv), case.dtype, view)
    lb, tl = _out_buf(nnc, [case.B, case.H, case.Sq], FP32, False) if lse else (None, None)
    cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case, algorithm)
    res = []
    try:
        ib.arm()
        for _ in range(reps):
            ob.arm()
            if lb:
                lb.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, None, 0, [ins["q"], ins["k"], ins["v"]], [to] + ([tl] if tl else []), stream)
            stream.wait()
            assert st == 0, "%s: forward status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
            res.append((ob.result(to), lb.result(tl).view(np.float32).astype(np.float64) if lb else None, nnc.launch_count() - l0))
    finally:
        for x in [ib, ob, lb, stream]:
            if x is not None:
                x.free()
    if reps > 1:
        assert np.array_equal(res[0][0], res[1][0]), "%s: two forward runs differ" % case
        assert res[0][1] is None or np.array_equal(res[0][1].view(np.uint64), res[1][1].view(np.uint64)), "%s: two LSE runs differ" % case
    return res[0]


def run_backward(nnc, case, d, view=False, packed_qkv=False, saved=None, alias_dout_q=False, reps=2, algorithm=FLASH):
    """(dq, dk, dv bits, launches) under `algorithm`; saved = (O bits, LSE) passes the forward's outputs as inputs[9], [10]"""
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), True) if packed_qkv else (None, {})
    db, dins = _in_tensors(nnc, case, d, ("do",) if packed_qkv else ("do", "q", "k", "v"), False)
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
    cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, case, algorithm)
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


@pytest.mark.gpu
@pytest.mark.parametrize("case", WIDE, ids=WIDE_IDS)
def test_wide_attention_path(gpu, case):
    nnc = gpu
    d = operands(case)
    fp, bp = plans(case)
    o_bits, lse, launches = run_forward(nnc, case, d, view=case.view)
    assert launches == fp["launches"], "%s: %d forward launches, planned %d" % (case, launches, fp["launches"])
    rnd = ar.rounding_of("flash", case.dtype)
    with wide_blocks():
        f = forward_oracle(case, d, fp)
    o, uo, lse_ref, ul = f.out()
    y = ar.as4(_values(o_bits, case.dtype), case.three_d)
    ar.check(y, o, uo, rnd, "%s: O" % case)
    dead = ~f.live[..., 0]  # [B, H, Sq]
    if dead.any():
        assert (y.transpose(0, 2, 1, 3)[dead] == 0).all(), "%s: fully masked rows must give O = 0 exactly" % case
    ar.check_lse(lse, lse_ref, ul, "%s: LSE" % case)
    res = run_backward(nnc, case, d, view=case.view)
    assert res[3] == bp["launches"], "%s: %d backward launches, planned %d" % (case, res[3], bp["launches"])
    o16 = _values(o_bits, case.dtype)
    with wide_blocks():
        b = backward_oracle(case, d, bp, o16=o16)
        add_flush_terms(forward_oracle(case, d, bp), b, d["do"], o16, case.three_d)
    for bits, (want, unit), n in zip(res[:3], b.out(), ("dq", "dk", "dv")):
        got = ar.as4(_values(bits, case.dtype), case.three_d)
        ar.check(got, want, unit, rnd, "%s: %s" % (case, n))
        if n == "dq" and dead.any():
            assert (got.transpose(0, 2, 1, 3)[dead] == 0).all(), "%s: fully masked rows must give dQ = 0 exactly" % case
    saved = run_backward(nnc, case, d, view=case.view, saved=(o_bits, lse), reps=1)
    assert saved[3] == plans(case, saved=True)[1]["launches"] == 3
    for a, s, n in zip(res[:3], saved[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, s), "%s: %s with the saved o / lse differs from the recomputed one" % (case, n)


EXACT = [C(BF16, 2, 200, 200, 4, 2, 160, 1, path="flash"), C(FP16, 2, 129, 129, 4, 1, 256, 0, "peaked", path="flash")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT, ids=[repr(c) for c in EXACT])
def test_wide_gqa_batch_entry_and_alias_identities(gpu, case):
    """GQA = K / V repeated to H heads; batch entry 1 = a call on it alone; dout aliasing q = a separate copy of q"""
    nnc = gpu
    d = operands(case)
    o, lse, _ = run_forward(nnc, case, d, reps=1)
    g = case.H // case.Hk
    rep = _sub(case, Hk=case.H)
    rd = dict(d, k=np.repeat(d["k"], g, axis=2), v=np.repeat(d["v"], g, axis=2))
    o2, lse2, _ = run_forward(nnc, rep, rd, reps=1)
    assert np.array_equal(o, o2) and np.array_equal(lse, lse2), "%s: GQA forward differs from K / V repeated to H heads" % case
    full = run_backward(nnc, case, d, reps=1)
    reps_ = run_backward(nnc, rep, rd, reps=1)
    assert np.array_equal(full[0], reps_[0]), "%s: GQA dq differs from K / V repeated" % case
    one = _sub(case, B=1)
    od = dict((n, None if a is None else a[1:2]) for n, a in d.items())
    o1, lse1, _ = run_forward(nnc, one, od, reps=1)
    assert np.array_equal(o[1:2], o1) and np.array_equal(lse[1:2], lse1), "%s: batch entry 1 differs from a call on it alone" % case
    part = run_backward(nnc, one, od, reps=1)
    for a, b2, n in zip(full[:3], part[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a[1:2], b2), "%s: batch entry 1's %s differs from a call on it alone" % (case, n)
    alias = run_backward(nnc, case, dict(d, do=d["q"]), alias_dout_q=True, reps=1)
    copy = run_backward(nnc, case, dict(d, do=d["q"].copy()), reps=1)
    for a, b2, n in zip(alias[:3], copy[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2), "%s: %s with dout aliasing q differs from a copy" % (case, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_wide_packed_qkv_views_and_pitched_gradients(gpu, dtype):
    """q, k, v as slices of one [B, S, 3, H, D] buffer and dq / dk / dv with a wider row pitch give the packed results bit for bit, and
    every NaN-filled guard element stays untouched"""
    nnc = gpu
    case = C(dtype, 2, 129, 129, 2, 2, 160, 1, "peaked", path="flash")
    d = operands(case)
    o, lse, _ = run_forward(nnc, case, d, reps=1)
    ov, lsev, _ = run_forward(nnc, case, d, view=True, packed_qkv=True, reps=1)
    assert np.array_equal(o, ov) and np.array_equal(lse, lsev), "packed QKV views give another forward result"
    g = run_backward(nnc, case, d, reps=1)
    gv = run_backward(nnc, case, d, view=True, packed_qkv=True, reps=1)
    for a, b2, n in zip(g[:3], gv[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2), "%s from views differs from the packed call" % n
    assert gv[3] == 4


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_head_dim_160_equals_zero_padded_256(gpu, dtype):
    """The TMA unit zero-fills features D..255 of the 256-wide tiles: D = 160 gives the first 160 columns of the same call with q, k, v
    (and dout) zero-padded to 256 features, forward and backward, bit for bit"""
    nnc = gpu
    c160 = C(dtype, 1, 200, 333, 4, 2, 160, 1, path="flash")
    d = operands(c160)
    pad = lambda a: np.concatenate([a, np.zeros(a.shape[:-1] + (96,), np.float32)], -1)
    c256 = _sub(c160, D=256, Dv=256)
    c256.scale = c160.scale
    dp = dict(d, q=pad(d["q"]), k=pad(d["k"]), v=pad(d["v"]), do=pad(d["do"]))
    o, lse, _ = run_forward(nnc, c160, d, reps=1)
    o2, lse2, _ = run_forward(nnc, c256, dp, reps=1)
    assert np.array_equal(o, o2[..., :160]) and np.array_equal(lse, lse2)
    assert (_values(o2[..., 160:], dtype) == 0).all()
    g = run_backward(nnc, c160, d, reps=1)
    g2 = run_backward(nnc, c256, dp, reps=1)
    for a, b2, n in zip(g[:3], g2[:3], ("dq", "dk", "dv")):
        assert np.array_equal(a, b2[..., :160]), "%s of D = 160 differs from the zero-padded call" % n


NARROW = [C(BF16, 2, 200, 200, 4, 2, 64, 1, path="flash"), C(FP16, 1, 129, 333, 2, 1, 128, 0, "peaked", path="flash"),
          C(BF16, 1, 64, 96, 2, 2, 36, 0, path="func")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", NARROW, ids=[repr(c) for c in NARROW])
def test_algorithm_1_outside_the_wide_heads_equals_algorithm_0(gpu, case):
    """D <= 128 (and shapes no flash kernel takes): algorithm 1 is algorithm 0, bit for bit and launch for launch"""
    nnc = gpu
    d = operands(case)
    lse = case.path == "flash"
    a0 = run_forward(nnc, case, d, lse=lse, reps=1, algorithm=0)
    a1 = run_forward(nnc, case, d, lse=lse, reps=1, algorithm=FLASH)
    assert np.array_equal(a0[0], a1[0]) and a0[2] == a1[2]
    assert not lse or np.array_equal(a0[1], a1[1])
    b0 = run_backward(nnc, case, d, reps=1, algorithm=0)
    b1 = run_backward(nnc, case, d, reps=1, algorithm=FLASH)
    for x, y, n in zip(b0, b1, ("dq", "dk", "dv", "launches")):
        assert np.array_equal(x, y), "%s: algorithm 1 %s differs from algorithm 0" % (case, n)


@pytest.mark.gpu
def test_autotune_picks_flash_for_a_wide_forward_with_lse(gpu):
    """ccv_nnc_cmd_autotune times both algorithms; algorithm 0 refuses a D = 160 forward that asks for the log-sum-exp, so the tuned
    command is algorithm 1, and it runs"""
    nnc = gpu
    case = C(BF16, 1, 256, 256, 2, 2, 160, 1, path="flash")
    d = operands(case)
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), False)
    to = nnc.gpu_tensor([1, 256, 2, 160], datatype=abi.CCV_16BF)
    tl = nnc.gpu_tensor([1, 2, 256])
    try:
        ib.arm()
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case, algorithm=-1)
        assert nnc.cmd_exec(cmd, None, 0, [ins["q"], ins["k"], ins["v"]], [to, tl], stream) == abi.CCV_NNC_EXEC_NO_KERNEL
        tuned = nnc.cmd_autotune(cmd, None, 0, [ins["q"], ins["k"], ins["v"]], [to, tl], stream)
        assert tuned.algorithm == FLASH
        assert nnc.cmd_exec(tuned, None, 0, [ins["q"], ins["k"], ins["v"]], [to, tl], stream) == 0
        stream.wait()
    finally:
        for x in (ib, to, tl, stream):
            x.free()


@pytest.mark.gpu
def test_long_sequence_causal_d256(gpu):
    """B = 1, H = 2, S = 16384, D = 256, causal, bf16 under algorithm 1: the first and the last 128 query rows of O, LSE and dQ, and the
    last 128 keys' dK / dV (seen by those rows alone), held to the bound"""
    nnc = gpu
    B, H, S, D, n = 1, 2, 16384, 256, 128
    case = C(BF16, B, S, S, H, H, D, 1, path="flash")
    r = np.random.RandomState(5)
    d = dict((k, cr.rne16(r.random_sample((B, S, H, D)) * hi - lo, BF16).astype(np.float32)) for k, lo, hi in
             (("q", 1, 2), ("k", 1, 2), ("v", 0.5, 1.5), ("do", 0.5, 1.5)))
    d["mask"] = None
    o_bits, lse, launches = run_forward(nnc, case, d, reps=1)
    assert launches == 1
    g = run_backward(nnc, case, d, saved=(o_bits, lse), reps=1)
    assert g[3] == 3
    model = ar.Model("flash", BF16)
    rnd = ("rne", BF16)
    o16 = _values(o_bits, BF16)
    for q0 in (0, S - n):
        sl = slice(q0, q0 + n)
        x = dict((k, d[k][:, sl].astype(np.float64)) for k in ("q", "do"))
        with wide_blocks():
            f = ar.Forward(x["q"], d["k"][:, :q0 + n], d["v"][:, :q0 + n], case.scale, 1, None, model)
            bk = ar.Backward(f, x["do"], o16=o16[:, sl])
        oo, uo, ll, ul = f.out()
        what = "S = 16384 rows %d..%d" % (q0, q0 + n - 1)
        ar.check(o16[:, sl], oo, uo, rnd, what + " O")
        ar.check_lse(lse[:, :, sl], ll, ul, what + " LSE")
        (dq, uq), (dk, uk), (dv, uv) = bk.out()
        ar.check(_values(g[0], BF16)[:, sl], dq, uq, rnd, what + " dq")
        if q0 == S - n:
            ks = slice(S - n, S)
            ar.check(_values(g[1], BF16)[:, ks], dk[:, ks], uk[:, ks], rnd, what + " dk")
            ar.check(_values(g[2], BF16)[:, ks], dv[:, ks], uv[:, ks], rnd, what + " dv")
