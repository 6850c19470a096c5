"""SCALED_DOT_PRODUCT_ATTENTION algorithm 2 (CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK): 16-bit forwards with an additive mask on one flash launch
(ccv_b200/csrc/sm100_fmha.cu for D <= 128, sm100_fmha_wide.cu for 128 < D <= 256), against the float64 oracle and the flash path's
rounding-level bounds of tests/attention_ref.py with the mask added (its |mask_ij| exponent term).

The kernels form t = fmaf(s, scale, mask) as CPU_REF does, cut the causal / Sk horizon on top, and run the online softmax.  A row whose
visible keys are all -inf gives O = 0 exactly and LSE = -inf (the convention of causal Sq > Sk rows); the oracle below models such rows
that way, and -inf entries of other rows as keys with p = 0.  The mask is staged through shared memory by TMA, so its base and every pitch
must be multiples of 16 bytes; other calls, calls without a mask and fp32 calls return NO_KERNEL under algorithm 2.

CPU: the constants, the planner for algorithm 2, and the bound rejecting four mask defects.
GPU: the case table (bf16 / fp16, D in {64, 128, 160, 192, 256}, fp32 and 16-bit masks of every accepted shape, causal, GQA, ragged
Sq / Sk, 3-d tensors, strided q / k / v / o, row-pitched masks, the LSE, -1e4 entries, all -inf rows) with guard buffers around every
output and the mask, bit-identical reruns and one launch; the same calls under algorithm 0; NO_KERNEL without a mask, for an unaligned
pitch and for the backward; packed QKV views and the unify-head entry; autotuning; a NaN in the mask; the CPU_REF fixture."""
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi
from tests import attention_ref as ar
from tests import contract_ref as cr
from tests.attention_ref import BF16, FP16, FP32
from tests.test_parity_attention_paths import (DT, GOLDEN, NHWC, Buf, Case, _bits, _in_tensors, _out_buf, _shape, _values,
                                               operands)
from tests.test_parity_attention_wide import wide_blocks

FLASH_MASK = abi.CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ccv_nnc_sm100.h")


# ------------------------------------------------------------------------------------------------ planner (algorithm 2)
def mask_pitch_ok(mshape, mdtype, pitch=None):
    """the TMA unit reads the mask: every pitch (row, head, batch) a multiple of 16 bytes"""
    esz = 4 if mdtype == FP32 else 2
    return ((pitch or mshape[-1]) * esz) % 16 == 0


def plan_forward(dtype, B, H, Hk, Sq, Sk, D, Dv, mask=False, mask_ok=True, aligned=True, algorithm=FLASH_MASK):
    """algorithm 2: one flash launch for a 16-bit call with a mask the kernels take; NO_KERNEL ("refused") for everything else"""
    if algorithm != FLASH_MASK:
        return ar.plan_forward(dtype, B, H, Hk, Sq, Sk, D, Dv, mask=mask, aligned=aligned)
    if dtype != FP32 and mask and mask_ok and 8 <= D <= 256 and D % 8 == 0 and Dv == D and H % Hk == 0 and aligned:
        return dict(path="flash", launches=1)
    return dict(path="refused", launches=0)


def test_constants_agree_with_the_header():
    text = open(HEADER).read()
    val = lambda n: int(re.search(r"\b%s\s*=\s*(\d+)" % n, text).group(1))
    assert val("CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK") == abi.CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK == 2
    assert val("CCV_NNC_SM100_SDPA_ALGO_COUNT") == abi.CCV_NNC_SM100_SDPA_ALGO_COUNT == 3
    assert val("CCV_NNC_SM100_SDPA_ALGO_FLASH") == abi.CCV_NNC_SM100_SDPA_ALGO_FLASH == 1


def test_planner_for_algorithm_2_on_hand_worked_shapes():
    # masked 16-bit calls: one launch, with the LSE and on views too (algorithm 0 refuses those, or widens to fp32)
    assert plan_forward(BF16, 2, 4, 2, 333, 200, 64, 64, mask=True) == dict(path="flash", launches=1)
    assert plan_forward(FP16, 1, 2, 2, 64, 96, 256, 256, mask=True) == dict(path="flash", launches=1)
    assert ar.plan_forward(BF16, 1, 2, 2, 64, 96, 160, 160, mask=True, lse=True)["path"] == "refused"
    assert ar.plan_forward(BF16, 1, 2, 2, 64, 96, 64, 64, mask=True)["path"] == "func"
    # NO_KERNEL: no mask, fp32, D > 256, D % 8, Dv != D, a mask pitch of 1332 bytes (fp32, Sk = 333) or 400 + 2 (16-bit, Sk = 201)
    for a, kw in [((BF16, 1, 2, 2, 64, 96, 64, 64), {}), ((FP32, 1, 2, 2, 64, 96, 64, 64), dict(mask=True)),
                  ((BF16, 1, 2, 2, 64, 96, 264, 264), dict(mask=True)), ((FP16, 1, 2, 2, 64, 96, 36, 36), dict(mask=True)),
                  ((BF16, 1, 2, 2, 64, 96, 64, 32), dict(mask=True)),
                  ((BF16, 1, 2, 2, 64, 333, 64, 64), dict(mask=True, mask_ok=mask_pitch_ok((64, 333), FP32))),
                  ((FP16, 1, 2, 2, 64, 201, 64, 64), dict(mask=True, mask_ok=mask_pitch_ok((64, 201), FP16)))]:
        assert plan_forward(*a, **kw) == dict(path="refused", launches=0), (a, kw)
    assert mask_pitch_ok((64, 200), FP16) and mask_pitch_ok((64, 204), FP32) and not mask_pitch_ok((64, 204), BF16)
    for c in MASKED:
        assert plans(c)["path"] == "flash", c


# ------------------------------------------------------------------------------------------------ the case table
class MCase(Case):
    """a Case with an additive mask: shape, element type (FP32 or the case's 16-bit type), a row pitch wider than Sk (a view), and rows
    made entirely -inf"""

    def __init__(self, dtype, B, Sq, Sk, H, Hk, D, causal, regime="flat", mask=None, mdtype=FP32, pitched=False, dead=False, **kw):
        Case.__init__(self, dtype, B, Sq, Sk, H, Hk, D, causal, regime, mask=mask, backward=False, path="flash", **kw)
        self.mdtype, self.pitched, self.dead = mdtype, pitched, dead

    def __repr__(self):
        return Case.__repr__(self) + " %smask%s%s" % ("f32" if self.mdtype == FP32 else "16", " pitched" if self.pitched else "", " dead" if self.dead else "")


M = MCase
MASKED = [
    M(BF16, 2, 333, 200, 4, 2, 64, 1, "peaked", mask=(333, 200), view=True),             # Sq > Sk causal, ragged, GQA 2
    M(FP16, 1, 129, 200, 2, 2, 128, 0, mask=(1, 2, 129, 200), mdtype=FP16),
    M(BF16, 2, 200, 200, 4, 4, 160, 1, mask=(2, 1, 200, 200), view=True),
    M(FP16, 2, 65, 128, 2, 1, 256, 0, "peaked", mask=(2, 2, 65, 128), mdtype=FP16, dead=True),
    M(BF16, 1, 1, 1024, 4, 1, 128, 1, mask=(4, 1, 1024)),                                  # decode; 3-d mask [H, Sq, Sk]
    M(FP16, 2, 127, 64, 1, 1, 64, 0, mask=(127, 64), three_d=True, pitched=True),
    M(BF16, 1, 256, 256, 2, 2, 256, 1, mask=(256, 256), mdtype=BF16, pitched=True, dead=True),
    M(FP16, 1, 333, 200, 2, 1, 160, 1, "peaked", mask=(2, 333, 200), mdtype=FP16),           # Sq > Sk causal on the wide kernel
    M(BF16, 2, 129, 136, 2, 2, 128, 0, "peaked", mask=(1, 1, 129, 136), dead=True),
    M(FP16, 1, 1024, 1024, 2, 2, 64, 1, "rising", mask=(1024, 1024)),
    M(BF16, 1, 200, 512, 2, 2, 192, 1, mask=(1, 2, 200, 512), mdtype=BF16, view=True),
    M(FP16, 2, 96, 96, 1, 1, 136, 0, "extreme", mask=(96, 96), three_d=True, pitched=True, dead=True),
]
MASKED_IDS = [repr(c) for c in MASKED]


def plans(case):
    return plan_forward(case.dtype, case.B, case.H, case.Hk, case.Sq, case.Sk, case.D, case.Dv, mask=True,
                        mask_ok=mask_pitch_ok(case.mask, case.mdtype, case.Sk + 8 if case.pitched else None))


def mask_of(case):
    """the mask's values (float32, on the 16-bit grid for a 16-bit mask): U(-3, 3), 30 % of entries -1e4; `dead` rows all -inf"""
    m = operands(case)["mask"].copy()
    if case.dead:
        m[..., [1, case.Sq // 2], :] = -np.inf
    if case.mdtype != FP32:
        m = cr.rne16(m.astype(np.float64), case.mdtype).astype(np.float32)
    return m


def mask_oracle(case, d, mask, drop=None, **kw):
    """ar.Forward on the 16-bit operands with the mask; -inf entries as -1e30 (p = 0 and no |mask| term), rows whose visible keys are all
    -inf as O = 0 and LSE = -inf exactly.  kw may replace the mask the oracle adds (a defect)."""
    x = dict((n, ar.as4(d[n], case.three_d)) for n in ("q", "k", "v"))
    seen = kw.get("added", mask)
    mo = np.where(np.isneginf(seen), -1e30, seen)
    with wide_blocks() if case.D > 128 else _null():
        f = ar.Forward(x["q"], x["k"], x["v"], case.scale, case.causal, mo, ar.Model("flash", case.dtype), drop=drop)
    m4 = np.broadcast_to(ar.mask4(seen, case.B, case.H), (case.B, case.H, case.Sq, case.Sk))
    vis = ar.visible(case.Sq, case.Sk, case.causal)[None, None]
    dead = ~(vis & ~np.isneginf(m4)).any(-1)
    f.o[dead] = 0
    f.unit_o[dead] = 0
    f.lse[dead] = -np.inf
    f.unit_lse[dead] = 0
    f.live = f.live & ~dead[..., None]
    return f


class _null(object):
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------ CPU: the bound rejects mask defects
def _rejects(bad, ref, unit, rnd, what):
    assert not ar.admits(ar.finish(bad, rnd), ref, unit, rnd).all(), "the bound admits %s" % what


@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_bound_rejects_mask_defects(dtype):
    """the mask multiplied by the scale, broadcast on the batch axis instead of the head axis, read one row off, and ignored on the last
    (partial) key block of Sk = 200"""
    case = M(dtype, 2, 200, 200, 2, 2, 64, 0, mask=(2, 1, 200, 200))
    d = operands(case)
    mask = mask_of(case)
    rnd = ("rne", dtype)
    o, uo, _, _ = mask_oracle(case, d, mask).out()
    ar.check(ar.finish(o, rnd), o, uo, rnd, "correct O")
    _rejects(mask_oracle(case, d, mask, added=mask * case.scale).out()[0], o, uo, rnd, "the mask times the scale")
    _rejects(mask_oracle(case, d, mask, added=mask.reshape(1, 2, 200, 200)).out()[0], o, uo, rnd, "the mask broadcast on the wrong axis")
    shifted = np.concatenate([mask[..., 1:, :], mask[..., -1:, :]], -2)
    _rejects(mask_oracle(case, d, mask, added=shifted).out()[0], o, uo, rnd, "mask rows off by one")
    tail = mask.copy()
    tail[..., 128:] = 0
    _rejects(mask_oracle(case, d, mask, added=tail).out()[0], o, uo, rnd, "the mask ignored on the last key block")


# ------------------------------------------------------------------------------------------------ GPU
def _cmd(nnc, cmd_id, case, algorithm=FLASH_MASK):
    c = nnc._simple(cmd_id, algorithm=algorithm)
    c.info.scaled_dot_product_attention.scale = case.scale
    c.info.scaled_dot_product_attention.is_causal = case.causal
    c.info.scaled_dot_product_attention.deterministic = 1
    return c


def _mask_buf(nnc, case, mask):
    """the mask in a NaN-filled guard buffer; pitched: rows Sk + 8 elements apart, every outer stride to match"""
    mdt = case.mdtype
    dims = list(mask.shape)
    pitch = dims[-1] + 8 if case.pitched else dims[-1]
    strides = [0] * len(dims)
    strides[-1], acc = 1, pitch
    for i in range(len(dims) - 2, -1, -1):
        strides[i] = acc
        acc *= dims[i]
    total = 64 + acc + 64
    b = Buf(nnc, total, mdt)
    t = b.add(dims, strides if case.pitched else None, 64, _bits(mask, mdt))
    return b, t


def forward(nnc, case, d, mask, algorithm=FLASH_MASK, lse=True, view=None, packed_qkv=False, reps=2, use_mask=True):
    """(status, O bits, LSE or None, launches); every guard element of O, the LSE and the mask stays untouched, and two runs agree bit for
    bit"""
    view = case.view if view is None else view
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), packed_qkv)
    mb, tm = _mask_buf(nnc, case, mask) if use_mask else (None, None)
    ob, to = _out_buf(nnc, _shape(case, case.Sq, case.H, case.Dv), case.dtype, view)
    lb, tl = _out_buf(nnc, [case.B, case.H, case.Sq], FP32, False) if lse else (None, None)
    cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case, algorithm)
    res = []
    try:
        ib.arm()
        if mb:
            mb.arm()
        for _ in range(reps):
            ob.arm()
            if lb:
                lb.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, None, 0, [ins["q"], ins["k"], ins["v"]] + ([tm] if tm else []), [to] + ([tl] if tl else []), stream)
            stream.wait()
            res.append((st, ob.result(to), lb.result(tl).view(np.float32).astype(np.float64) if lb else None, nnc.launch_count() - l0))
            if mb:
                mb.result(tm)
    finally:
        for x in [ib, mb, ob, lb, stream]:
            if x is not None:
                x.free()
    if reps > 1 and res[0][0] == 0:
        assert np.array_equal(res[0][1], res[1][1]), "%s: two forward runs differ" % case
        assert res[0][2] is None or np.array_equal(res[0][2].view(np.uint64), res[1][2].view(np.uint64)), "%s: two LSE runs differ" % case
    return res[0]


def check_forward(case, d, mask, o_bits, lse):
    f = mask_oracle(case, d, mask)
    o, uo, lse_ref, ul = f.out()
    rnd = ("rne", case.dtype)
    y = ar.as4(_values(o_bits, case.dtype), case.three_d)
    ar.check(y, o, uo, rnd, "%s: O" % case)
    dead = ~f.live[..., 0]
    if dead.any():
        assert (y.transpose(0, 2, 1, 3)[dead] == 0).all(), "%s: fully masked rows must give O = 0 exactly" % case
    if lse is not None:
        ar.check_lse(lse, lse_ref, ul, "%s: LSE" % case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MASKED, ids=MASKED_IDS)
def test_masked_attention_path(gpu, case):
    nnc = gpu
    d = operands(case)
    mask = mask_of(case)
    st, o_bits, lse, launches = forward(nnc, case, d, mask)
    assert st == 0, "%s: status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
    assert launches == plans(case)["launches"] == 1, "%s: %d launches" % (case, launches)
    check_forward(case, d, mask, o_bits, lse)
    # without the LSE: the same O
    st, o2, _, _ = forward(nnc, case, d, mask, lse=False, reps=1)
    assert st == 0 and np.array_equal(o_bits, o2), "%s: O without the LSE differs" % case
    # algorithm 0 on the same call: the functional form for an fp32 mask (no LSE, no views), INVALID for a 16-bit one
    st, o0, _, launches0 = forward(nnc, case, d, mask, algorithm=0, lse=False, view=False, reps=1)
    if case.mdtype != FP32:
        assert st == abi.CCV_NNC_EXEC_INVALID, "%s: algorithm 0 takes a 16-bit mask" % case
    elif not case.pitched:
        p0 = ar.plan_forward(case.dtype, case.B, case.H, case.Hk, case.Sq, case.Sk, case.D, case.Dv, mask=True)
        assert st == 0 and p0["path"] == "func" and launches0 == p0["launches"], (case, st, launches0, p0)


@pytest.mark.gpu
def test_algorithm_2_returns_no_kernel_outside_masked_16bit_forwards(gpu):
    """no mask, an fp32 call, a mask pitch that is not a multiple of 16 bytes (fp32, Sk = 333), D = 264, and the backward"""
    nnc = gpu
    case = M(BF16, 1, 64, 96, 2, 2, 64, 0, mask=(64, 96))
    d = operands(case)
    mask = mask_of(case)
    assert forward(nnc, case, d, mask, use_mask=False, reps=1)[0] == abi.CCV_NNC_EXEC_NO_KERNEL
    c32 = M(FP32, 1, 64, 96, 2, 2, 64, 0, mask=(64, 96))
    assert forward(nnc, c32, operands(c32), mask_of(c32), lse=False, reps=1)[0] == abi.CCV_NNC_EXEC_NO_KERNEL
    odd = M(FP16, 1, 64, 333, 2, 2, 64, 0, mask=(64, 333))
    st, _, _, launches = forward(nnc, odd, operands(odd), mask_of(odd), reps=1)
    assert st == abi.CCV_NNC_EXEC_NO_KERNEL and launches == 0
    wide = M(BF16, 1, 64, 96, 1, 1, 264, 0, mask=(64, 96))
    assert forward(nnc, wide, operands(wide), mask_of(wide), reps=1)[0] == abi.CCV_NNC_EXEC_NO_KERNEL
    # the backward: algorithm 2 is forward only
    stream = nnc.Stream(0)
    ts = [nnc.gpu_tensor(list(d[n].shape), NHWC, DT[BF16]) for n in ("do", "q", "k", "v")]
    outs = [nnc.gpu_tensor(list(d[n].shape), NHWC, DT[BF16]) for n in ("q", "k", "v")]
    try:
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, case)
        assert nnc.cmd_exec(cmd, None, 0, [ts[0], None, None, ts[1], ts[2], ts[3]], outs, stream) == abi.CCV_NNC_EXEC_NO_KERNEL
    finally:
        for t in ts + outs + [stream]:
            t.free()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF16, FP16])
def test_masked_packed_qkv_views_equal_the_packed_call(gpu, dtype):
    """q, k, v as slices of one [B, S, 3, H, D] buffer with a pitched O give the packed call's O and LSE bit for bit"""
    nnc = gpu
    for D in (128, 160):
        case = M(dtype, 2, 200, 200, 2, 2, D, 1, "peaked", mask=(2, 1, 200, 200), mdtype=dtype, pitched=True)
        d = operands(case)
        mask = mask_of(case)
        a = forward(nnc, case, d, mask, view=False, reps=1)
        b = forward(nnc, case, d, mask, view=True, packed_qkv=True, reps=1)
        assert a[0] == b[0] == 0 and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), case
        check_forward(case, d, mask, a[1], a[2])


@pytest.mark.gpu
def test_masked_nan_propagates(gpu):
    """a NaN in the mask makes its row's O NaN (and the LSE); the other rows keep their values"""
    nnc = gpu
    case = M(BF16, 1, 64, 128, 1, 1, 64, 0, mask=(64, 128))
    d = operands(case)
    mask = mask_of(case)
    bad = mask.copy()
    bad[5, 77] = np.nan
    st, o, lse, _ = forward(nnc, case, d, bad, reps=1)
    assert st == 0
    y = _values(o, BF16)
    assert np.isnan(y[0, 5]).all() and np.isnan(lse[0, 0, 5])
    rest = np.ones(64, bool)
    rest[5] = False
    st, o2, lse2, _ = forward(nnc, case, d, mask, reps=1)
    assert np.array_equal(o[:, rest], o2[:, rest]) and np.array_equal(lse[..., rest], lse2[..., rest])


@pytest.mark.gpu
def test_masked_unify_head_entry(gpu):
    """with unify-head weights the per-head attention (outputs[2]) is the masked flash result, bit for bit"""
    nnc = gpu
    case = M(FP16, 2, 96, 128, 2, 2, 64, 0, mask=(96, 128))
    d = operands(case)
    mask = mask_of(case)
    _, o_ref, _, _ = forward(nnc, case, d, mask, lse=False, reps=1)
    B, S, H, D = case.B, case.Sq, case.H, case.D
    w = cr.rne16(np.random.RandomState(3).random_sample((H * D, H * D)) * 0.2 - 0.1, FP16).astype(np.float32)
    stream = nnc.Stream(0)
    ts = [nnc.gpu_tensor(list(d[n].shape), NHWC, DT[FP16]) for n in ("q", "k", "v")]
    tw = nnc.gpu_tensor([H * D, H * D], NHWC, DT[FP16])
    for t, a in zip(ts + [tw], [d["q"], d["k"], d["v"], w]):
        t.upload(_bits(a, FP16).view(np.float16))
    tm = nnc.gpu_tensor(list(mask.shape)).upload(mask)
    td, tc = nnc.gpu_tensor([B, S, H * D], NHWC, DT[FP16]), nnc.gpu_tensor([B, case.Sq, H, D], NHWC, DT[FP16])
    try:
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case)
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(cmd, None, 0, ts + [tm, tw], [td, None, tc], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        assert nnc.launch_count() - l0 >= 2  # the attention, then the projection
        c = tc.download().view(np.uint16)
    finally:
        for t in ts + [tw, tm, td, tc, stream]:
            t.free()
    assert np.array_equal(c.reshape(o_ref.shape), o_ref)


@pytest.mark.gpu
def test_autotune_picks_flash_mask_for_a_masked_forward_with_lse(gpu):
    """algorithms 0 and 1 refuse a masked forward that asks for the log-sum-exp; the tuned command is algorithm 2, and it runs"""
    nnc = gpu
    case = M(BF16, 1, 256, 256, 2, 2, 160, 1, mask=(256, 256))
    d = operands(case)
    mask = mask_of(case)
    stream = nnc.Stream(0)
    ib, ins = _in_tensors(nnc, case, d, ("q", "k", "v"), False)
    tm = nnc.gpu_tensor(list(mask.shape)).upload(mask)
    to = nnc.gpu_tensor([1, 256, 2, 160], datatype=abi.CCV_16BF)
    tl = nnc.gpu_tensor([1, 2, 256])
    try:
        ib.arm()
        cmd = _cmd(nnc, abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, case, algorithm=-1)
        args = ([ins["q"], ins["k"], ins["v"], tm], [to, tl])
        assert nnc.cmd_exec(cmd, None, 0, *args, stream) == abi.CCV_NNC_EXEC_NO_KERNEL
        tuned = nnc.cmd_autotune(cmd, None, 0, *args, stream)
        assert tuned.algorithm == FLASH_MASK
        assert nnc.cmd_exec(tuned, None, 0, *args, stream) == 0
        stream.wait()
    finally:
        for x in (ib, tm, to, tl, stream):
            x.free()


@pytest.mark.gpu
@pytest.mark.parametrize("i", [4, 5, 6, 7, 8])
def test_masked_flash_against_cpu_ref_fixture(gpu, i):
    """tests/golden/cpuref_sdpa.npz (every mask shape, one causal): the pinned operands rounded to fp16 under algorithm 2 against CPU_REF's
    fp32 output, within the flash bound plus what the rounding of q, k, v moves the exact result"""
    nnc = gpu
    f = np.load(os.path.join(GOLDEN, "cpuref_sdpa.npz"))
    p = ar.pin_inputs(i)
    B, Sq, Sk, H, Hk, D, Dv, causal, mshape, three, _ = ar.PINS[i]
    case = M(FP16, B, Sq, Sk, H, Hk, D, causal, mask=mshape)
    case.scale = p["scale"]
    d = dict((n, cr.rne16(p[n].astype(np.float64), FP16).astype(np.float32)) for n in ("q", "k", "v"))
    d["do"] = None
    st, o_bits, lse, launches = forward(nnc, case, d, p["mask"], reps=1)
    assert st == 0 and launches == 1
    y = _values(o_bits, FP16)
    f16 = mask_oracle(case, d, p["mask"])
    f32 = ar.Forward(p["q"], p["k"], p["v"], p["scale"], causal, p["mask"], ar.Model("flash", FP16))
    o16, u16, _, _ = f16.out()
    o32 = f32.out()[0]
    gold = f["%d_o" % i].astype(np.float64)
    assert np.abs(gold - o32).max() < 1e-5, "pin %d: the oracle does not reproduce CPU_REF" % i
    room = ar.C_ATT * u16 + np.abs(o16 - o32) + 2.0 ** -11 * np.abs(o16) + 2.0 ** -24
    assert (np.abs(y - gold) <= room).all(), "pin %d: %g" % (i, np.abs(y - gold).max())
