"""The element-wise, broadcast and reduction commands on CCV_NNC_BACKEND_GPU_SM100, launch path by launch path, against the float64
oracles of tests/ew_ref.py (pinned to the reference's CPU_REF by tests/golden/cpuref_ew.npz): SIGMOID, TANH, LEAKY_RELU, EWEXP, EWLOG,
EWSQRT, CLAMP, GELU, SWISH, EWDIV, REDUCE_SUM / MEAN / MAX / MIN / NORM2, MASKED_FILL, EWSUM, ADD, MUL and SCALAR_MUL.

Every GPU case checks its launch count against the restated plan through ccv_nnc_sm100_launch_count(); every output lives between NaN
guards that must stay NaN; every call is made twice and must give the same bits; the unaligned (all-scalar) forms must give the bits
of the aligned (vector) ones; non-finite outputs must sit exactly where the oracle's are.  The CPU tests show that the bounds reject
the defects these kernels plausibly have."""
import math
import os

import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests import ew_ref as R
from tests.test_parity_feeder_paths import free_device_bytes, run, run_twice
from tests.util import pack16, round16, seeded, unpack16

F32, BF16, F16 = R.F32, R.BF16, R.F16
DT = {F32: abi.CCV_32F, BF16: abi.CCV_16BF, F16: abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_ew.npz")
NAN, INF = float("nan"), float("inf")


# ---- data -------------------------------------------------------------------------------------------------------------------------
UNARY_ARGS = {"SIGMOID": (), "TANH": (), "EWEXP": (), "EWLOG": (), "EWSQRT": (), "LEAKY_RELU": (0.2,), "CLAMP": (-0.5, 0.75)}
UNARY_RANGE = {"SIGMOID": (-20, 20), "TANH": (-5, 5), "EWEXP": (-10, 12), "EWLOG": (0, 5), "EWSQRT": (0, 5), "LEAKY_RELU": (-2, 2), "CLAMP": (-2, 2)}
ACTS = {"GELU": dict(tanh=0), "GELU_TANH": dict(tanh=1), "SWISH": {}}


def specials(name):
    """values every unary case carries at its head: zeros of both signs, fp32 subnormals, the smallest normal, and per command the
    edges of its domain (fp16 overflow of EWEXP above 11.1, fp32 overflow above 88.7; the open ends of EWLOG / EWSQRT at 0)"""
    s = [0.0, -0.0, 1e-40, 2.0 ** -126, 3e-39]
    if name in ("EWLOG", "EWSQRT"):
        return s
    s += [-1e-40, -2.0 ** -126]
    if name == "EWEXP":
        s += [11.2, 12.0, 89.0, 100.0, -100.0, -87.5]
    if name in ("SIGMOID", "SWISH"):
        s += [-88.0, -100.0, 88.0, 30.0]
    if name in ("GELU", "GELU_TANH"):
        s += [-10.0, -6.0, 6.0, 10.0]
    if name == "CLAMP":
        s += [-0.5, 0.75, -0.75, 0.5]
    return s


def unary_data(name, n, seed, kind=F32):
    lo, hi = UNARY_RANGE.get(name, (-6, 6))
    x = seeded((n,), seed, lo, hi)
    s = np.array(specials(name), np.float32)[:n]
    x[:len(s)] = s
    return x if kind == F32 else round16(x, DT[kind])


def q(x, kind):
    return x if kind == F32 else round16(x, DT[kind])


def fwd_cmd(name):
    return getattr(_nnc, "CMD_%s_FORWARD" % name)(*UNARY_ARGS[name])


def bwd_cmd(name):
    return getattr(_nnc, "CMD_%s_BACKWARD" % name)(*UNARY_ARGS[name])


def unary_oracle(name, x):
    return R.UNARY[name][0](x, *UNARY_ARGS[name])


def unary_bwd_oracle(name, g, a, b):
    return R.UNARY[name][1](g, a, b, *UNARY_ARGS[name])


def act_cmds(name):
    if name == "SWISH":
        return _nnc.CMD_SWISH_FORWARD(), _nnc.CMD_SWISH_BACKWARD()
    return _nnc.CMD_GELU_FORWARD(**ACTS[name]), _nnc.CMD_GELU_BACKWARD(**ACTS[name])


def act_oracle(name, x):
    return R.swish(x) if name == "SWISH" else R.gelu(x, name == "GELU_TANH")


def act_bwd_oracle(name, g, x):
    return R.swish_bwd(g, x) if name == "SWISH" else R.gelu_bwd(g, x, name == "GELU_TANH")


# ---- the comparison: finite values within the bound, non-finite ones exactly where the oracle's are ----------------------------------
RATIOS = {}


def _ends(y_hat, e, kind):
    with np.errstate(invalid="ignore", over="ignore"):
        lo, hi = y_hat - e, y_hat + e
        return (R.f32(lo), R.f32(hi)) if kind == F32 else (R.rne16(lo, kind), R.rne16(hi, kind))


def agree(y, y_hat, e, kind=F32):
    """element-wise: y finite and within the bound where the oracle's interval is finite; y exactly the oracle's non-finite value
    (the same infinity, or NaN) where the oracle's value is not finite or overflows the kind"""
    y = np.asarray(y, np.float64)
    y_hat = np.broadcast_to(np.asarray(y_hat, np.float64), y.shape)
    e = np.broadcast_to(np.asarray(e, np.float64), y.shape)
    lo, hi = _ends(y_hat, e, kind)
    special = ~np.isfinite(y_hat) | (np.isinf(lo) & (lo == hi))
    want = np.where(np.isfinite(y_hat), lo, y_hat)
    same = (np.isnan(y) & np.isnan(want)) | (y == want)
    fin = np.where(special, False, np.isfinite(y))
    ok_fin = np.zeros(y.shape, bool)
    ok_fin[fin] = R.within(y[fin], y_hat[fin], e[fin], kind)
    return np.where(special, same, ok_fin)


def check(fam, what, y, y_hat, e, kind=F32):
    y = np.asarray(y, np.float64)
    y_hat = np.broadcast_to(np.asarray(y_hat, np.float64), y.shape)
    e = np.broadcast_to(np.asarray(e, np.float64), y.shape)
    ok = agree(y, y_hat, e, kind)
    fin = np.isfinite(y) & np.isfinite(y_hat)
    r = R.ratio(y[fin], y_hat[fin], e[fin]) if kind == F32 else 0.0
    if kind == F32 and ok.all():
        RATIOS[(fam, what)] = max(RATIOS.get((fam, what), 0.0), r)
    assert ok.all(), (fam, what, kind, "ratio to bound / C: %.2f" % r, int((~ok).sum()), [(tuple(i), y[tuple(i)], y_hat[tuple(i)]) for i in np.argwhere(~ok)[:4]])


def bits(y):
    return np.ascontiguousarray(y, np.float32).view(np.uint32)


def exact(fam, what, y, y_hat, kind=F32):
    """a selection: the kernel's bits are the oracle's value stored in the kind (NaN where the oracle has NaN)"""
    want = R.store(y_hat, kind).astype(np.float32)
    y = np.asarray(y, np.float32).reshape(want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(y), nan), (fam, what, "NaN positions")
    bad = bits(y)[~nan] != bits(want)[~nan]
    assert not bad.any(), (fam, what, kind, int(bad.sum()), y[~nan][bad][:4], want[~nan][bad][:4])
    RATIOS.setdefault((fam, what), 0.0)


def same_bits(a, b, what):
    assert np.array_equal(bits(a), bits(b)), what


def kinds_all(kind):
    return lambda ins, outs: {id(x): kind for x in ins + outs if x is not None and x.dtype != np.int32}


# ---- CPU: the oracles against CPU_REF's fixture --------------------------------------------------------------------------------------
GOLDEN_N = 105
GOLDEN_REDUCE_SHAPE = (2, 3, 4, 5)
GOLDEN_REDUCE_AXES = [(3,), (2, 3), (1, 2), (0, 2), (0, 1, 2, 3), (0,)]
GOLDEN_BCAST = [("add", (2, 3, 4), (1, 3, 1)), ("mul", (2, 3, 4), (2, 1, 4)), ("mul_b", (1, 3, 1), (2, 3, 4))]
ADD_PQ = (0.5, -1.25)
MUL_P = 1.5
MF_P, MF_Q = 1.4, -7.0


def mf_p(mtype):
    """the fill value p: 1.4 against an int32 mask (compared as (int)(1.4 + 0.5) = 1), 1 against an fp32 mask"""
    return MF_P if mtype == "int32" else 1.0


def reduce_golden_data(mode, seed):
    """[2, 3, 4, 5] data; MAX / MIN on a 1/8 grid (ties), with slice [0, 0] all -inf (+inf for MIN) and slice [1, 2] all NaN; the others
    plain"""
    a = seeded(GOLDEN_REDUCE_SHAPE, seed, -2, 2)
    if mode in ("MAX", "MIN"):
        a = (np.round(a * 2) / 2).astype(np.float32)  # 9 values: ties in most slices
        a[0, 0] = -INF if mode == "MAX" else INF
        a[1, 2] = NAN
    if mode == "NORM2":
        a[a == 0] = 0.5
    return a


def bshape_of(ashape, axes):
    return tuple(1 if i in axes else d for i, d in enumerate(ashape))


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_ew.npz missing")
    return np.load(GOLDEN)


def _pinned(got, want, what, e=None, selection=False):
    """the oracle's value against CPU_REF's: selections bit for bit, the rest within the oracle's own bound (CPU_REF rounds as the
    kernel does, in another order)"""
    want = np.asarray(want, np.float32).reshape(np.shape(got))
    if selection:
        g32 = np.asarray(got, np.float32)
        assert np.array_equal(np.isnan(g32), np.isnan(want)) and np.array_equal(bits(g32)[~np.isnan(want)], bits(want)[~np.isnan(want)]), what
        return
    assert agree(want, got, e).all(), (what, np.argwhere(~agree(want, got, e))[:4].tolist())


@pytest.mark.parametrize("name", sorted(UNARY_ARGS))
def test_unary_oracles_match_cpu_ref_fixture(name):
    z = _golden()
    a, g, b, h = z[name + "_a"], z[name + "_g"], z[name + "_b"], z[name + "_h"]
    sel = name in R.SELECTIONS
    y, e = unary_oracle(name, a)
    _pinned(y, b, name + " forward", e, sel)
    hh, eh = unary_bwd_oracle(name, g, a, b)
    _pinned(hh, h, name + " backward", eh, sel)
    if name == "EWEXP":
        hh, eh = unary_bwd_oracle(name, None, a, b)
        _pinned(hh, z["EWEXP_h_nog"], "EWEXP backward without g", eh)


@pytest.mark.parametrize("name", sorted(ACTS))
def test_activation_oracles_match_cpu_ref_fixture(name):
    z = _golden()
    a, g = z[name + "_a"], z[name + "_g"]
    _pinned(*act_oracle(name, a)[:1], z[name + "_b"], name + " forward", act_oracle(name, a)[1])
    _pinned(act_bwd_oracle(name, g, a)[0], z[name + "_h"], name + " backward", act_bwd_oracle(name, g, a)[1])


def test_ewdiv_oracles_match_cpu_ref_fixture():
    z = _golden()
    a, b, g = z["div_a"], z["div_b"], z["div_g"]
    c, e = R.ewdiv(a, b)
    _pinned(c, z["div_c"], "c", e)
    _pinned(*R.ewdiv(None, b)[:1], z["div_c1"], "1 / b", R.ewdiv(None, b)[1])
    for gg, sfx in ((g, ""), (None, "_nog")):
        ha, e_a = R.ewdiv_bwd(gg, b, z["div_c"], "a")
        hb, e_b = R.ewdiv_bwd(gg, b, z["div_c"], "b")
        _pinned(ha, z["div_ha" + sfx], "ha" + sfx, e_a)
        _pinned(hb, z["div_hb" + sfx], "hb" + sfx, e_b)


@pytest.mark.parametrize("mode", ["SUM", "MEAN", "MAX", "MIN", "NORM2"])
@pytest.mark.parametrize("axes", GOLDEN_REDUCE_AXES, ids=str)
def test_reduce_oracles_match_cpu_ref_fixture(mode, axes):
    z = _golden()
    key = "red_%s_%s_" % (mode, "".join(map(str, axes)))
    a = z["red_%s_a" % mode]
    bs = bshape_of(a.shape, axes)
    b, e = R.reduce_fwd(mode, a, bs)
    _pinned(b, z[key + "b"], key + "b", e, mode in ("MAX", "MIN"))
    bb = z[key + "b"]
    for gg, sfx in ((z[key + "g"], "h"), (None, "h_nog")):
        h, eh = R.reduce_bwd(mode, gg, a, bb, a.shape, axes)
        _pinned(h, z[key + sfx], key + sfx, eh, mode in ("MAX", "MIN", "SUM"))


def test_reduce_identity_is_pinned_by_the_fixture():
    """an oracle built with the old -inf / inf identity is rejected by CPU_REF's fixture, forward and backward"""
    z = _golden()
    for mode, ident in (("MAX", -INF), ("MIN", INF)):
        key = "red_%s_23_" % mode
        a = z["red_%s_a" % mode]
        bs = bshape_of(a.shape, (2, 3))
        old, _ = R.reduce_fwd(mode, a, bs, identity=ident)
        assert not np.array_equal(np.asarray(old, np.float32), z[key + "b"])
        h_old, _ = R.reduce_bwd(mode, z[key + "g"], a, old, a.shape)
        assert not np.array_equal(np.asarray(h_old, np.float32), z[key + "h"])


@pytest.mark.parametrize("mtype", ["int32", "fp32"])
def test_masked_fill_oracle_matches_cpu_ref_fixture(mtype):
    z = _golden()
    a, g = z["mf_a"], z["mf_g"]
    for ax in (0, 1, 2):
        key = "mf_%s_%d_" % (mtype, ax)
        m, p = z[key + "mask"], mf_p(mtype)
        _pinned(R.masked_fill(a, m, p, MF_Q, a.shape)[0], z[key + "c"], key + "c", selection=True)
        _pinned(R.masked_fill(g, m, p, 0.0, a.shape)[0], z[key + "h"], key + "h", selection=True)


def test_ewsum_oracle_matches_cpu_ref_fixture():
    """bit for bit: fp32 left to right, the aliased operand first"""
    z = _golden()
    xs = [z["sum_x%d" % i] for i in range(9)]
    for k, alias in ((3, None), (3, 1), (9, None), (9, 8)):
        y, _ = R.ewsum(xs[:k], alias)
        _pinned(y, z["sum_%d_%s" % (k, alias)], "ewsum %d %s" % (k, alias), selection=True)


@pytest.mark.parametrize("name,ashape,bshape", GOLDEN_BCAST)
def test_broadcast_oracles_match_cpu_ref_fixture(name, ashape, bshape):
    z = _golden()
    a, b, g = z[name + "_a"], z[name + "_b"], z[name + "_g"]
    cs = tuple(max(x, y) for x, y in zip(ashape, bshape))
    if name == "add":
        _pinned(*R.add(a, b, *ADD_PQ, cs)[:1], z[name + "_c"], "add c", R.add(a, b, *ADD_PQ, cs)[1])
        for gg, sfx in ((g, ""), (None, "_nog")):
            for i, (shape, p) in enumerate(((ashape, ADD_PQ[0]), (bshape, ADD_PQ[1]))):
                hh, eh = R.add_bwd(gg, p, shape, cs)
                _pinned(hh, z["%s_h%d%s" % (name, i, sfx)], "add h%d%s" % (i, sfx), eh)
        return
    _pinned(*R.mul(a, b, MUL_P, cs)[:1], z[name + "_c"], name + " c", R.mul(a, b, MUL_P, cs)[1])
    for gg, sfx in ((g, ""), (None, "_nog")):
        for i, (shape, other) in enumerate(((ashape, b), (bshape, a))):
            hh, eh = R.mul_bwd(gg, other, MUL_P, shape, cs)
            _pinned(hh, z["%s_h%d%s" % (name, i, sfx)], "%s h%d%s" % (name, i, sfx), eh)
    _pinned(np.float32(MUL_P) * a, z[name + "_smul"], "scalar mul", selection=True)


def test_golden_pins_every_quirk():
    """the fixture holds the case each restated quirk shows on"""
    z = _golden()
    # MAX / MIN identity: an all -inf (+inf) slice and an all-NaN slice give -FLT_MAX (FLT_MAX), and no gradient reaches them
    for mode, sign in (("MAX", -1), ("MIN", 1)):
        b, h = z["red_%s_23_b" % mode], z["red_%s_23_h" % mode]
        assert b[0, 0, 0, 0] == sign * R.FLT_MAX and b[1, 2, 0, 0] == sign * R.FLT_MAX
        assert (h[0, 0] == 0).all() and (h[1, 2] == 0).all()
        # ties: some slice sends its gradient to more than one element
        hn = z["red_%s_3_h_nog" % mode]
        assert (hn.sum(axis=3) > 1).any()
    # MEAN backward without g: 1 / (h's extents along the command's axes), here axis 0 (1 / 2), while the b passed beside it reduces
    # axes 1 and 3 (count(b) / count(h) = 1 / 15)
    a, b = z["red_MEAN_a"], z["red_MEAN_cmd0_b"]
    assert (z["red_MEAN_cmd0_h_nog"] == np.float32(0.5)).all() and b.size / a.size == 1.0 / 15
    # broadcast ADD / MUL backward: the broadcast operand's gradient is summed (its shape is the operand's)
    assert z["add_h1"].shape == (1, 3, 1) and z["mul_h1"].shape == (2, 1, 4)
    # int32 and fp32 masks; the int32 mask compares against (int)(1.4 + 0.5) = 1
    m = z["mf_int32_0_mask"]
    assert m.dtype == np.int32 and z["mf_fp32_0_mask"].dtype == np.float32
    c = np.broadcast_to(z["mf_int32_0_c"], z["mf_a"].shape)
    assert ((np.broadcast_to(m, c.shape) == 1) == (c == np.float32(MF_Q))).all()
    # EWSUM: the aliased operand comes first, which changes the bits on this data
    assert not np.array_equal(z["sum_9_8"], z["sum_9_None"])
    # GELU backward's pdf carries sqrt(2 / pi): at x = 0 the derivative is 1/2, elsewhere it exceeds the exact one
    a, h, g = z["GELU_a"], z["GELU_h"], z["GELU_g"]
    x = a.astype(np.float64)
    exact_d = 0.5 * (1 + R.erf(x / math.sqrt(2))) + x * np.exp(-x * x / 2) / math.sqrt(2 * math.pi)
    assert not np.allclose(h, g * exact_d, rtol=1e-3)
    # LEAKY_RELU / CLAMP backward test b: a case where a and b disagree in sign / bound is in the fixture
    assert (z["CLAMP_b"] == np.float32(0.75)).any() and (z["CLAMP_b"] == np.float32(-0.5)).any()


# ---- CPU: the launch plan ------------------------------------------------------------------------------------------------------------
def test_declared_paths_are_the_plan():
    assert [R.reduce_path(r) for r in (1, 32, 64, 65, 700, 10 ** 6)] == ["warp", "warp", "warp", "block", "block", "block"]
    assert [R.ewsum_launches(k) for k in (1, 2, 8, 9, 17, 64)] == [0, 1, 1, 2, 3, 8]
    assert R.ewsum_launches(8, BF16) == 1 and R.ewsum_launches(5, "int32") == 1
    assert R.ewdiv_back_launches(1, 0) == 1 and R.ewdiv_back_launches(1, 1) == 2
    assert R.mul_back_launches(True) == 1 and R.mul_back_launches(False) == 2
    assert R.staged_f32_launches(3, 1) == 5 and R.staged_f32_launches(3, 2, inner=4) == 9
    assert R.ew_path(F32) == "vector" and R.ew_path(BF16, aligned=False) == "scalar"
    for shape, axes in RED_CASES:
        bs = bshape_of(shape, axes)
        rc = int(np.prod([shape[i] for i in axes], dtype=np.int64))
        assert rc == int(np.prod(shape)) // int(np.prod(bs))


# ---- CPU: the bounds reject plausible defects -----------------------------------------------------------------------------------------
def _rejects(y_bad, y_hat, e, kind=F32):
    return not agree(y_bad, y_hat, e, kind).all()


@pytest.mark.parametrize("name", ["SIGMOID", "TANH", "EWEXP", "EWSQRT"])
def test_unary_bounds_reject_defects(name):
    """the backward computed from a instead of the saved b; 1 - a^2 for the tanh derivative; the sqrt backward without the 0.5"""
    a = unary_data(name, 4099, 1)[8:]
    a = a[a > 0.05] if name == "EWSQRT" else a
    b = R.f32(unary_oracle(name, a)[0])
    g = seeded(a.shape, 2, -1, 1)
    h, e = unary_bwd_oracle(name, g, a, b)
    assert _rejects(unary_bwd_oracle(name, g, a, a)[0], h, e)
    if name == "TANH":
        assert _rejects(R.f64(g) * (1 - R.f64(a) ** 2), h, e)
    if name == "EWSQRT":
        assert _rejects(R.sqrt_bwd(g, b, half=1.0)[0], h, e)


def test_ewdiv_bounds_reject_defects():
    a, b, g = seeded((4099,), 1, -2, 2), seeded((4099,), 2, 0.5, 2) * np.sign(seeded((4099,), 3, -1, 1)), seeded((4099,), 4, -1, 1)
    c = R.f32(R.ewdiv(a, b)[0])
    hb, e = R.ewdiv_bwd(g, b, c, "b")
    assert _rejects(R.ewdiv_bwd(g, b, c, "b", sign=1.0)[0], hb, e) and _rejects(R.ewdiv_bwd(g, b, c, "b", use_c=False)[0], hb, e)


def test_gelu_forms_swapped_are_rejected():
    x = seeded((4099,), 1, -6, 6)
    g = seeded((4099,), 2, -1, 1)
    for tf in (False, True):
        y, e = R.gelu(x, tf)
        assert _rejects(R.gelu(x, not tf)[0], y, e)
        h, eh = R.gelu_bwd(g, x, tf)
        assert _rejects(R.gelu_bwd(g, x, not tf)[0], h, eh)


@pytest.mark.parametrize("rcount", [33, 65, 700])
def test_reduce_bounds_reject_defects(rcount):
    """a reduction that drops its last partial warp; MEAN over the wrong axes; NORM2 without the root"""
    a = seeded((6, rcount), 1, 0.5, 2)  # positive terms: nothing cancels what the dropped warp held
    for mode in ("SUM", "MEAN", "NORM2"):
        b, e = R.reduce_fwd(mode, a, (6, 1))
        cut = rcount - (rcount % 32 or 32)
        part = R.reduce_fwd(mode, a[:, :cut], (6, 1))[0]
        if mode == "MEAN":
            part = part * cut / rcount
        assert _rejects(part, b, e), mode
    a4 = seeded((3, 4, 5, rcount), 2, -1, 1)
    b, e = R.reduce_fwd("MEAN", a4, (3, 1, 5, 1))
    s = R.f64(a4).sum(axis=(1, 3), keepdims=True)
    assert _rejects(s / (rcount * 5), b, e) and _rejects(s / rcount, b, e)
    b, e = R.reduce_fwd("NORM2", a4, (3, 1, 5, 1))
    assert _rejects(b * b, b, e)
    # the backward of MEAN without g, scaled over all of h instead of the command's axes
    h, eh = R.reduce_bwd("MEAN", None, None, None, (3, 4, 5, rcount), axes=(1, 3))
    assert _rejects(np.full(h.shape, 1.0 / (3 * 4 * 5 * rcount)), h, eh)


@pytest.mark.parametrize("which", ["add", "mul"])
def test_broadcast_bounds_reject_defects(which):
    """gradients not summed over the broadcast axes, or (MUL) p and q swapped: the gradient of a taken from a"""
    cs, bsh = (4, 5, 6, 7), (1, 5, 1, 7)
    a, b, g = seeded(cs, 1, -1, 1), seeded(bsh, 2, 0.5, 2), seeded(cs, 3, -1, 1)
    if which == "add":
        hb, e = R.add_bwd(g, ADD_PQ[1], bsh, cs)
        assert _rejects(R.add_bwd(g, ADD_PQ[1], bsh, cs, summed=False)[0], hb, e)
        assert _rejects(R.add_bwd(g, ADD_PQ[0], bsh, cs)[0], hb, e)
        return
    hb, e = R.mul_bwd(g, a, MUL_P, bsh, cs)
    assert _rejects(R.f64(g)[:1, :, :1] * MUL_P * R.f64(a)[:1, :, :1], hb, e)
    ha, ea = R.mul_bwd(g, b, MUL_P, cs, cs)
    assert _rejects(R.mul_bwd(g, a, MUL_P, cs, cs)[0], ha, ea)


def test_ewsum_bounds_reject_defects():
    """the second chunk of 8 operands overwriting the output instead of adding onto it"""
    xs = [seeded((4099,), i, -1, 1) for i in range(17)]
    y, e = R.ewsum(xs)
    assert _rejects(R.ewsum(xs, chunk_overwrites=True)[0], y, e)


def test_truncated_16bit_stores_are_rejected():
    x = seeded((4099,), 1, -4, 4)
    for kind in (BF16, F16):
        for y, e in (R.sigmoid(x), R.gelu(x), R.reduce_fwd("SUM", seeded((64, 700), 2, -1, 1), (64, 1))):
            y, e = np.asarray(y).ravel(), np.broadcast_to(e, np.shape(y)).ravel()
            t = R.trunc16(y, kind)
            sel = (t != R.rne16(y, kind)) & (R.rne16(y - e, kind) == R.rne16(y + e, kind))
            assert sel.any() and not R.within(t[sel], y[sel], e[sel], kind).any()


# ---- GPU: unary / activation ---------------------------------------------------------------------------------------------------------
def counts(kind):
    w = R.vec_width(kind)
    return [w * 37, w * 37 + 1, w * 37 - 1, w - 1, (1 << 20) + 3]


UNARY_GPU = [(n, k, c) for n in sorted(UNARY_ARGS) for k in (F32, BF16, F16) for c in counts(k)]


def _unary_once(nnc, name, kind, x, g, offset):
    k = kinds_all(kind)
    st, (y,), launches = run_twice(nnc, fwd_cmd(name), lambda: ([x], [np.zeros_like(x)]), k, offset=offset)
    assert st == 0 and launches == R.unary_launches(), nnc.lib().ccv_nnc_sm100_last_error()
    yk = q(y, kind)
    outs = []
    for gg in (g, None):
        st, (h,), launches = run_twice(nnc, bwd_cmd(name), lambda: ([gg, x, yk], [np.zeros_like(x)]), k, offset=offset)
        assert st == 0 and launches == 1
        outs.append(h)
    return y, outs[0], outs[1]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,n", UNARY_GPU)
def test_unary_paths(gpu, name, kind, n):
    nnc = gpu
    x = unary_data(name, n, 11, kind)
    g = q(seeded((n,), 12, -1, 1), kind)
    y, h, h1 = _unary_once(nnc, name, kind, x, g, 0)
    yu, hu, h1u = _unary_once(nnc, name, kind, x, g, 1)
    same_bits(y, yu, "forward: the scalar form differs"), same_bits(h, hu, "backward: the scalar form differs"), same_bits(h1, h1u, "no g")
    sel = name in R.SELECTIONS
    y_hat, e = unary_oracle(name, x)
    exact(name, "forward", y, y_hat, kind) if sel else check(name, "forward", y, y_hat, e, kind)
    yk = q(y, kind)
    for gg, hh, what in ((g, h, "backward"), (None, h1, "backward (no g)")):
        h_hat, eh = unary_bwd_oracle(name, gg, x, yk)
        exact(name, what, hh, h_hat, kind) if sel else check(name, what, hh, h_hat, eh, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("lo,hi", [(NAN, 0.5), (-0.25, NAN), (NAN, NAN), (-0.25, 0.5)])
@pytest.mark.parametrize("kind", [F32, BF16, F16])
def test_clamp_sides(gpu, lo, hi, kind):
    nnc = gpu
    x = q(seeded((4099,), 3, -2, 2), kind)
    x[:4] = [-0.25, 0.5, 0.0, -0.0]
    g = q(seeded((4099,), 4, -1, 1), kind)
    st, (y,), _ = run_twice(nnc, _nnc.CMD_CLAMP_FORWARD(lo, hi), lambda: ([x], [np.zeros_like(x)]), kinds_all(kind))
    assert st == 0
    exact("CLAMP", "forward", y, R.clamp(x, lo, hi)[0], kind)
    st, (h,), _ = run_twice(nnc, _nnc.CMD_CLAMP_BACKWARD(lo, hi), lambda: ([g, x, y], [np.zeros_like(x)]), kinds_all(kind))
    assert st == 0
    exact("CLAMP", "backward", h, R.clamp_bwd(g, y, lo, hi)[0], kind)


ACT_GPU = [(n, k, c) for n in sorted(ACTS) for k in (F32, BF16, F16) for c in counts(k)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,n", ACT_GPU)
def test_activation_paths(gpu, name, kind, n):
    nnc = gpu
    fwd, bwd = act_cmds(name)
    x = unary_data(name, n, 21, kind)
    g = q(seeded((n,), 22, -1, 1), kind)
    k = kinds_all(kind)
    res = []
    for off in (0, 1):
        st, (y,), launches = run_twice(nnc, fwd, lambda: ([x], [np.zeros_like(x)]), k, offset=off)
        assert st == 0 and launches == 1
        st, (h,), launches = run_twice(nnc, bwd, lambda: ([g, x], [np.zeros_like(x)]), k, offset=off)
        assert st == 0 and launches == 1
        res.append((y, h))
    same_bits(res[0][0], res[1][0], "forward: the scalar form differs"), same_bits(res[0][1], res[1][1], "backward: the scalar form differs")
    y, h = res[0]
    check(name, "forward", y, *act_oracle(name, x), kind=kind)
    check(name, "backward", h, *act_bwd_oracle(name, g, x), kind=kind)
    # no gradient: refused before any launch (CPU_REF has no form without g)
    h0 = np.zeros_like(x)  # of the operands' kind: the missing g is the only reason to refuse
    st, _, launches = run(nnc, bwd, [None, x], [h0], k([x], [h0]))
    assert st == INVALID and launches == 0


# ---- GPU: EWDIV -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("n", [4099, 7, 1 << 16])
def test_ewdiv_paths(gpu, kind, n):
    nnc = gpu
    k = kinds_all(kind)
    a = q(seeded((n,), 31, -2, 2), kind)
    b = q(seeded((n,), 32, 0.5, 2) * np.sign(seeded((n,), 33, -1, 1)), kind)
    g = q(seeded((n,), 34, -1, 1), kind)
    b[:2] = [0.0, -0.0]  # division by zero: infinities where the oracle has them
    a[:1] = 0.0  # 0 / 0: NaN
    for off in (0, 1):
        st, (c,), launches = run_twice(nnc, _nnc.CMD_EWDIV_FORWARD(), lambda: ([a, b], [np.zeros_like(a)]), k, offset=off)
        assert st == 0 and launches == 1
        check("ewdiv", "c", c, *R.ewdiv(a, b), kind=kind)
        st, (c1,), _ = run_twice(nnc, _nnc.CMD_EWDIV_FORWARD(), lambda: ([None, b], [np.zeros_like(a)]), k, offset=off)
        assert st == 0
        check("ewdiv", "1 / b", c1, *R.ewdiv(None, b), kind=kind)
    c = q(c, kind)
    bs, cs_ = b[2:], c[2:]  # the backward away from the zeros
    for gg in (g[2:], None):
        for want in ((1, 0), (0, 1), (1, 1)):
            outs = lambda: [np.zeros_like(bs) if want[0] else None, np.zeros_like(bs) if want[1] else None]
            st, (ha, hb), launches = run_twice(nnc, _nnc.CMD_EWDIV_BACKWARD(), lambda: ([gg, None, bs, cs_], outs()), k)
            assert st == 0 and launches == R.ewdiv_back_launches(*want), (want, launches)
            if want[0]:
                check("ewdiv", "ha", ha, *R.ewdiv_bwd(gg, bs, cs_, "a"), kind=kind)
            if want[1]:
                check("ewdiv", "hb", hb, *R.ewdiv_bwd(gg, bs, cs_, "b"), kind=kind)


# ---- GPU: reductions ------------------------------------------------------------------------------------------------------------------
def _subsets(n):
    return [tuple(i for i in range(n) if m >> i & 1) for m in range(1 << n)]


RED_CASES = [((2, 3, 4, 5), ax) for ax in _subsets(4)] + \
            [((32,), (0,)), ((64,), (0,)), ((65,), (0,)), ((100003,), (0,)), ((7, 33), (1,)), ((5, 64), (0,)), ((3, 65), (1,)),
             ((4, 8, 8), (1, 2)), ((4, 5, 13), (1, 2)), ((2, 300000), (1,)), ((3, 1, 7), (1,)), ((6, 5, 4), ())]


def reduce_data(mode, shape, seed, kind):
    a = seeded(shape, seed, -2, 2)
    if mode in ("MAX", "MIN"):
        a = (np.round(a * 8) / 8).astype(np.float32) + np.float32(0)  # ties; + 0 turns -0 into +0 (a tie of signed zeros has no order)
    if mode == "NORM2":
        a[a == 0] = 0.25
    return q(a, kind)


def _reduce_case(nnc, mode, shape, axes, kind, a=None):
    bs = bshape_of(shape, axes)
    a = reduce_data(mode, shape, 41, kind) if a is None else a
    k = kinds_all(kind)
    fwd = getattr(_nnc, "CMD_REDUCE_%s_FORWARD" % mode)(*axes)
    bwd = getattr(_nnc, "CMD_REDUCE_%s_BACKWARD" % mode)(*axes)
    st, (b,), launches = run_twice(nnc, fwd, lambda: ([a], [np.zeros(bs, np.float32)]), k)
    assert st == 0 and launches == 1, nnc.lib().ccv_nnc_sm100_last_error()
    b_hat, e = R.reduce_fwd(mode, a, bs)
    if mode in ("MAX", "MIN"):
        exact("reduce", mode + " forward", b, b_hat, kind)
    else:
        check("reduce", mode + " forward", b, b_hat, e, kind)
    g = q(seeded(bs, 42, -1, 1), kind)
    for gg, what in ((g, "backward"), (None, "backward (no g)")):
        st, (h,), launches = run_twice(nnc, bwd, lambda: ([gg, a, b], [np.zeros(shape, np.float32)]), k)
        assert st == 0 and launches == 1
        h_hat, eh = R.reduce_bwd(mode, gg, a, b, shape, axes)
        if mode in ("MAX", "MIN", "SUM"):
            exact("reduce", mode + " " + what, h, h_hat, kind)
        else:
            check("reduce", mode + " " + what, h, h_hat, eh, kind)
    return a, b


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("mode", ["SUM", "MEAN", "MAX", "MIN", "NORM2"])
@pytest.mark.parametrize("shape,axes", RED_CASES, ids=lambda v: str(v))
def test_reduce_paths(gpu, shape, axes, mode, kind):
    _reduce_case(gpu, mode, shape, axes, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("mode", ["MAX", "MIN"])
@pytest.mark.parametrize("rcount", [20, 700])
def test_reduce_max_min_masked_slices(gpu, mode, kind, rcount):
    """all -inf (+inf for MIN) and all-NaN slices: -FLT_MAX (FLT_MAX), which bf16 / fp16 store as -inf (+inf); the fp32 backward sends
    no gradient there, the 16-bit one (b = -inf = a) sends it to every element, as CPU_REF on the widened values does"""
    shape = (4, 3, rcount)
    a = reduce_data(mode, shape, 43, kind)
    a[0, 1] = -INF if mode == "MAX" else INF
    a[2, 2] = NAN
    a[3, 0, ::2] = NAN  # NaN never wins over a number
    _, b = _reduce_case(gpu, mode, shape, (2,), kind, a=a)
    big = R.FLT_MAX if kind == F32 else INF
    assert b[0, 1, 0] == (-big if mode == "MAX" else big) and b[2, 2, 0] == (-big if mode == "MAX" else big)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["SUM", "MEAN", "MAX", "MIN", "NORM2"])
def test_reduce_strided_view(gpu, mode):
    """the input a slice [.., :10] of a [4, 6, 13] tensor: the packed call's bits"""
    nnc = gpu
    a = reduce_data(mode, (4, 6, 10), 44, F32)
    for axes in ((2,), (0, 2), (1,)):
        _, b0 = _reduce_case(nnc, mode, (4, 6, 10), axes, F32, a=a)
        wide = np.full((4, 6, 13), NAN, np.float32)
        wide[..., :10] = a
        bs = bshape_of(a.shape, axes)
        t = nnc.gpu_tensor([4, 6, 13]).upload(wide)
        v = nnc.tensor_view_new(t, [4, 6, 10], [0] * 12, [78, 13, 1] + [0] * 9)
        o = nnc.gpu_tensor(list(bs)).upload(np.zeros(bs, np.float32))
        try:
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(getattr(nnc, "CMD_REDUCE_%s_FORWARD" % mode)(*axes), None, 0, [v], [o]) == 0
            assert nnc.launch_count() - l0 == 1
            same_bits(o.download(), b0, "the strided view differs from the packed call")
        finally:
            for x in (v, t, o):
                x.free()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
def test_reduce_mean_backward_without_g_scales_by_the_command_axes(gpu, kind):
    """MEAN backward without g: 1 / (h's extents along the command's axes), here axis 0 (1 / 2), whatever b is passed beside it (here
    one that reduces axes 1 and 3, count(b) / count(h) = 1 / 15)"""
    nnc = gpu
    shape = (2, 3, 4, 5)
    a, b = q(seeded(shape, 45, -1, 1), kind), q(seeded((2, 1, 4, 1), 46, -1, 1), kind)
    st, (h,), launches = run_twice(nnc, nnc.CMD_REDUCE_MEAN_BACKWARD(0), lambda: ([None, a, b], [np.zeros(shape, np.float32)]), kinds_all(kind))
    assert st == 0 and launches == 1
    exact("reduce", "MEAN backward (no g, command axes)", h, np.full(shape, R.mean_bwd_scale(shape, None, (0,))), kind)


@pytest.mark.gpu
def test_reduce_refuses_5d(gpu):
    nnc = gpu
    a = seeded((2, 2, 2, 2, 3), 1)
    for mode in ("SUM", "MAX"):
        st, (b,), launches = run(nnc, getattr(nnc, "CMD_REDUCE_%s_FORWARD" % mode)(4), [a], [np.full((2, 2, 2, 2, 1), 7.0, np.float32)])
        assert st == INVALID and launches == 0 and (b == 7.0).all()


# ---- GPU: MASKED_FILL ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("mtype", ["int32", "fp32"])
@pytest.mark.parametrize("axis", [0, 1, 2, 3])
def test_masked_fill_paths(gpu, axis, mtype, kind):
    nnc = gpu
    cs = (3, 4, 5, 6)
    ms = tuple(1 if i == axis else d for i, d in enumerate(cs))
    r = np.random.RandomState(axis)
    m = r.randint(0, 3, size=ms)
    m = m.astype(np.int32) if mtype == "int32" else m.astype(np.float32)
    a, g = q(seeded(cs, 51, -1, 1), kind), q(seeded(cs, 52, -1, 1), kind)
    p = mf_p(mtype)
    k = lambda ins, outs: {id(x): kind for x in ins + outs if x is not None and x is not m}
    st, (c,), launches = run_twice(nnc, _nnc.CMD_MASKED_FILL_FORWARD(p, MF_Q), lambda: ([a, m], [np.zeros(cs, np.float32)]), k)
    assert st == 0 and launches == 1
    exact("masked_fill", "c", c, R.masked_fill(a, m, p, MF_Q, cs)[0], kind)
    st, (h,), launches = run_twice(nnc, _nnc.CMD_MASKED_FILL_BACKWARD(p, MF_Q), lambda: ([g, None, m], [np.zeros(cs, np.float32)]), k)
    assert st == 0 and launches == 1
    exact("masked_fill", "h", h, R.masked_fill(g, m, p, 0.0, cs)[0], kind)


# ---- GPU: EWSUM -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 8, 9, 17, 64])
@pytest.mark.parametrize("alias", ["none", "first", "last"])
@pytest.mark.parametrize("offset", [0, 1])
def test_ewsum_fp32(gpu, k, alias, offset):
    """bit for bit the reference's left-to-right sum (the aliased operand first); chunks of 8 operands; the output may be any operand"""
    nnc = gpu
    n = 4099

    def make():
        xs = [seeded((n,), 60 + i, -1, 1) for i in range(k)]
        out = {"none": np.zeros(n, np.float32), "first": xs[0], "last": xs[-1]}[alias]
        return xs, [out]
    xs0 = make()[0]
    st, (y,), launches = run_twice(nnc, _nnc.CMD_EWSUM_FORWARD(), make, offset=offset)
    assert st == 0 and launches == R.ewsum_launches(k), (launches, k)
    j = {"none": None, "first": 0, "last": k - 1}[alias]
    y_hat, e = R.ewsum(xs0, j if j else None)
    exact("ewsum", "c", y, y_hat)
    check("ewsum", "c (bound)", y, y_hat, e)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [BF16, F16])
@pytest.mark.parametrize("k", [1, 2, 5, 8])
@pytest.mark.parametrize("offset", [0, 1])
def test_ewsum_16bit(gpu, kind, k, offset):
    nnc = gpu
    n = 4099
    xs = [q(seeded((n,), 70 + i, -1, 1), kind) for i in range(k)]
    st, (y,), launches = run_twice(nnc, _nnc.CMD_EWSUM_FORWARD(), lambda: (list(xs), [np.zeros(n, np.float32)]), kinds_all(kind), offset=offset)
    assert st == 0 and launches == R.ewsum_launches(k, kind)
    exact("ewsum", "c (16-bit)", y, R.ewsum(xs)[0], kind)
    # in place onto the last operand
    xi = [x.copy() for x in xs]
    st, (yi,), _ = run(nnc, _nnc.CMD_EWSUM_FORWARD(), xi, [xi[-1]], kinds_all(kind)(xi, []))
    assert st == 0
    exact("ewsum", "c (16-bit, in place)", yi, R.ewsum(xs, k - 1 if k > 1 else None)[0], kind)
    # nine operands: refused before any launch
    x9 = [q(seeded((n,), 80 + i, -1, 1), kind) for i in range(9)]
    o9 = np.full(n, 7.0, np.float32)  # a 16-bit output like the operands: the operand count is the only reason to refuse
    st, (y9,), launches = run(nnc, _nnc.CMD_EWSUM_FORWARD(), x9, [o9], kinds_all(kind)(x9, [o9]))
    assert st == INVALID and launches == 0 and (y9 == 7.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16])
def test_ewsum_backward(gpu, kind):
    """every output receives g bit for bit (ones without g), g itself as an output is left alone"""
    nnc = gpu
    n = 4099
    g = q(seeded((n,), 90, -1, 1), kind)
    k = kinds_all(kind)
    st, (h0, h1), launches = run_twice(nnc, _nnc.CMD_EWSUM_BACKWARD(), lambda: ([g], [np.zeros(n, np.float32), np.zeros(n, np.float32)]), k)
    assert st == 0 and launches == R.ewsum_back_launches(2, True)
    same_bits(h0, g, "h0"), same_bits(h1, g, "h1")
    st, (h0, h1), launches = run_twice(nnc, _nnc.CMD_EWSUM_BACKWARD(), lambda: ([None], [np.zeros(n, np.float32), np.zeros(n, np.float32)]), k)
    assert st == 0 and launches == R.ewsum_back_launches(2, False) and (h0 == 1).all() and (h1 == 1).all()
    gi, h1 = g.copy(), np.zeros(n, np.float32)
    st, (hi, h1), launches = run(nnc, _nnc.CMD_EWSUM_BACKWARD(), [gi], [gi, h1], k([gi], [h1]))
    assert st == 0 and launches == 0
    same_bits(hi, g, "in place"), same_bits(q(h1, kind), g, "h1 beside the in-place output")


# ---- GPU: ADD / MUL / SCALAR_MUL ---------------------------------------------------------------------------------------------------------
CS = (3, 4, 5, 6)
BCAST = [(CS, CS)] + [(CS, tuple(1 if i == ax else d for i, d in enumerate(CS))) for ax in range(4)] + \
        [(tuple(1 if i == ax else d for i, d in enumerate(CS)), CS) for ax in (0, 3)] + [((1, 4, 1, 6), (3, 1, 5, 1))]


def _staged(kind, n16, n16_out, inner=1):
    return inner if kind == F32 else R.staged_f32_launches(n16, n16_out, inner)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("ashape,bshape", BCAST, ids=str)
def test_add_mul_paths(gpu, ashape, bshape, kind):
    nnc = gpu
    cs = tuple(max(x, y) for x, y in zip(ashape, bshape))
    a, b, g = q(seeded(ashape, 101, -1, 1), kind), q(seeded(bshape, 102, -1, 1), kind), q(seeded(cs, 103, -1, 1), kind)
    k = kinds_all(kind)
    same = ashape == bshape
    offs = (0, 1) if same else (0,)
    for off in offs:
        st, (c,), launches = run_twice(nnc, _nnc.CMD_ADD_FORWARD(*ADD_PQ), lambda: ([a, b], [np.zeros(cs, np.float32)]), k, offset=off)
        assert st == 0 and launches == _staged(kind, 3, 1)
        check("add", "c", c, *R.add(a, b, *ADD_PQ, cs), kind=kind)
        st, (c,), launches = run_twice(nnc, _nnc.CMD_MUL_FORWARD(MUL_P), lambda: ([a, b], [np.zeros(cs, np.float32)]), k, offset=off)
        assert st == 0 and launches == _staged(kind, 3, 1)
        check("mul", "c", c, *R.mul(a, b, MUL_P, cs), kind=kind)
    if ashape == cs:
        st, (c,), _ = run_twice(nnc, _nnc.CMD_ADD_FORWARD(*ADD_PQ), lambda: ([a, None], [np.zeros(cs, np.float32)]), k)
        assert st == 0
        check("add", "c (no b)", c, *R.add(a, None, *ADD_PQ, cs), kind=kind)
    for gg in (g, None):
        st, (ha, hb), launches = run_twice(nnc, _nnc.CMD_ADD_BACKWARD(*ADD_PQ), lambda: ([gg], [np.zeros(ashape, np.float32), np.zeros(bshape, np.float32)]), k)
        assert st == 0 and launches == _staged(kind, 3 if gg is not None else 2, 2, 2), launches
        for h, shape, p, what in ((ha, ashape, ADD_PQ[0], "ha"), (hb, bshape, ADD_PQ[1], "hb")):
            if gg is None:
                exact("add", what + " (no g)", h, np.full(shape, float(np.float32(p))), kind)
            else:
                check("add", what, h, *R.add_bwd(gg, p, shape, cs), kind=kind)
        st, (ha, hb), launches = run_twice(nnc, _nnc.CMD_MUL_BACKWARD(MUL_P), lambda: ([gg, a, b], [np.zeros(ashape, np.float32), np.zeros(bshape, np.float32)]), k)
        inner = 2 * R.mul_back_launches(same)  # fused only where a, b (and g) share one shape
        assert st == 0 and launches == _staged(kind, 5 if gg is not None else 4, 2, inner), (launches, inner)
        check("mul", "ha", ha, *R.mul_bwd(gg, b, MUL_P, ashape, cs), kind=kind)
        check("mul", "hb", hb, *R.mul_bwd(gg, a, MUL_P, bshape, cs), kind=kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("offset", [0, 1])
def test_scalar_mul_paths(gpu, kind, offset):
    nnc = gpu
    n = 4099
    a, g = q(seeded((n,), 111, -1, 1), kind), q(seeded((n,), 112, -1, 1), kind)
    k = kinds_all(kind)
    st, (c,), launches = run_twice(nnc, _nnc.CMD_SCALAR_MUL_FORWARD(MUL_P), lambda: ([a], [np.zeros(n, np.float32)]), k, offset=offset)
    assert st == 0 and launches == _staged(kind, 2, 1)
    exact("scalar_mul", "c", c, R.f32(np.float32(MUL_P) * np.asarray(a, np.float32)), kind)
    st, (h,), _ = run_twice(nnc, _nnc.CMD_SCALAR_MUL_BACKWARD(MUL_P), lambda: ([g], [np.zeros(n, np.float32)]), k, offset=offset)
    assert st == 0
    exact("scalar_mul", "h", h, R.f32(np.float32(MUL_P) * np.asarray(g, np.float32)), kind)
    st, (h,), _ = run_twice(nnc, _nnc.CMD_SCALAR_MUL_BACKWARD(MUL_P), lambda: ([None], [np.zeros(n, np.float32)]), k, offset=offset)
    assert st == 0
    exact("scalar_mul", "h (no g)", h, np.full(n, float(np.float32(MUL_P))), kind)


@pytest.mark.gpu
def test_add_mul_strided_view_operand(gpu):
    """b a slice [.., :6] of a [3, 4, 5, 9] tensor: the packed call's bits, forward and MUL backward"""
    nnc = gpu
    a, b = seeded(CS, 121, -1, 1), seeded(CS, 122, -1, 1)
    g = seeded(CS, 123, -1, 1)
    _, (c0,), _ = run(nnc, nnc.CMD_MUL_FORWARD(MUL_P), [a, b], [np.zeros(CS, np.float32)])
    _, (d0,), _ = run(nnc, nnc.CMD_ADD_FORWARD(*ADD_PQ), [a, b], [np.zeros(CS, np.float32)])
    _, (ha0,), _ = run(nnc, nnc.CMD_MUL_BACKWARD(MUL_P), [g, a, b], [np.zeros(CS, np.float32)])
    wide = np.full(CS[:3] + (9,), NAN, np.float32)
    wide[..., :6] = b
    tw = nnc.gpu_tensor(list(wide.shape)).upload(wide)
    v = nnc.tensor_view_new(tw, list(CS), [0] * 12, [4 * 5 * 9, 5 * 9, 9, 1] + [0] * 8)
    ta, tg = nnc.gpu_tensor(list(CS)).upload(a), nnc.gpu_tensor(list(CS)).upload(g)
    out = nnc.gpu_tensor(list(CS)).upload(np.zeros(CS, np.float32))
    try:
        assert nnc.cmd_exec(nnc.CMD_MUL_FORWARD(MUL_P), None, 0, [ta, v], [out]) == 0
        same_bits(out.download(), c0, "MUL with a view operand")
        assert nnc.cmd_exec(nnc.CMD_ADD_FORWARD(*ADD_PQ), None, 0, [ta, v], [out]) == 0
        same_bits(out.download(), d0, "ADD with a view operand")
        assert nnc.cmd_exec(nnc.CMD_MUL_BACKWARD(MUL_P), None, 0, [tg, ta, v], [out]) == 0
        same_bits(out.download(), ha0, "MUL backward with a view operand")
    finally:
        for t in (v, tw, ta, tg, out):
            t.free()


# ---- GPU: the bias-gradient column sum with an fp32 g 8 but not 16 bytes aligned ----------------------------------------------------------
@pytest.mark.gpu
def test_gemm_bias_gradient_fp32_g_at_an_8_byte_offset(gpu):
    """GEMM backward with only dbias requested: fp32 g two elements into its allocation (8-byte aligned), a bf16 bias gradient.  The
    column sum takes the scalar kernel; its value is the column sums of g rounded once"""
    nnc = gpu
    rows, cols = 64, 32
    g = seeded((rows, cols), 131, -1, 1)
    a = seeded((rows, 16), 132, -1, 1)
    big = nnc.gpu_tensor([rows * cols + 2]).upload(np.concatenate([np.zeros(2, np.float32), g.ravel()]))
    tg = nnc.gpu_tensor([rows, cols], ptr=big.data_ptr + 8)
    ta = nnc.gpu_tensor([rows, 16]).upload(a)
    db = nnc.gpu_tensor([cols], datatype=abi.CCV_16BF).upload(pack16(np.zeros(cols, np.float32), abi.CCV_16BF))
    try:
        st = nnc.cmd_exec(nnc.CMD_GEMM_BACKWARD(), None, 0, [tg, ta, None], [None, None, db])
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        got = unpack16(db.download(), abi.CCV_16BF)
        s = R.f64(g).sum(axis=0)
        check("colsum", "dbias (bf16)", got, s, R.sum_bound(rows, np.abs(R.f64(g)).sum(axis=0)), BF16)
    finally:
        for t in (tg, big, ta, db):
            t.free()


# ---- GPU: 64-bit index space -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["unary", "reduce_back"])
def test_ew_64bit_index(gpu, which):
    """more than 2^32 bf16 elements: the unary kernel (SIGMOID forward) and reduce_back_kernel (REDUCE_SUM backward, g broadcast along
    the leading axis).  The tensors are filled on the device; only the last 4099 elements are checked"""
    nnc = gpu
    tail = 4099
    rows = 2 ** 32 // tail + 2  # [rows, tail]: no extent beyond int32, more than 2^32 elements
    total = rows * tail
    assert total > 2 ** 32
    need = (2 if which == "unary" else 1) * total * 2 + (1 << 30)  # the unary case reads a and writes b; the backward writes h only
    if free_device_bytes() < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 2 ** 30))
    dt = DT[BF16]
    big_b = nnc.gpu_tensor([rows, tail], datatype=dt)
    lb = nnc.gpu_tensor([tail], datatype=dt, ptr=big_b.data_ptr + (total - tail) * 2)
    owned = [lb, big_b]
    try:
        if which == "unary":
            big_a = nnc.gpu_tensor([rows, tail], datatype=dt)
            la = nnc.gpu_tensor([tail], datatype=dt, ptr=big_a.data_ptr + (total - tail) * 2)
            owned += [la, big_a]
            assert nnc.cmd_exec(nnc.CMD_SET_FORWARD(0.25), None, 0, [], [big_a]) == 0
            x = round16(seeded((tail,), 5, -6, 6), dt)
            la.upload(pack16(x, dt))
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(nnc.CMD_SIGMOID_FORWARD(), None, 0, [big_a], [big_b]) == 0
            assert nnc.launch_count() - l0 == 1
            check("SIGMOID", "forward (64-bit)", unpack16(lb.download(), dt), *R.sigmoid(x), kind=BF16)
        else:
            g = nnc.gpu_tensor([1, tail], datatype=dt)
            owned.append(g)
            x = round16(seeded((1, tail), 6, -1, 1), dt)
            g.upload(pack16(x, dt))
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(nnc.CMD_REDUCE_SUM_BACKWARD(0), None, 0, [g], [big_b]) == 0
            assert nnc.launch_count() - l0 == 1
            same_bits(unpack16(lb.download(), dt), x.ravel(), "the last row of h")
    finally:
        for t in owned:
            t.free()


@pytest.mark.gpu
def test_zz_report_measured_ratios(gpu):
    """prints the largest |y - y_hat| / (bound / BOUND_C) per family and output over the cases run before it in this session.  Every
    case already asserted its bound (ratio <= BOUND_C); this asserts the margin: no family needs more than half the constant"""
    per = {}
    for (fam, what), r in sorted(RATIOS.items()):
        print("ratio %-12s %-28s %.3f" % (fam, what, r))
        per[fam] = max(per.get(fam, 0.0), r)
    print("largest ratio per family:", ", ".join("%s %.3f" % kv for kv in sorted(per.items())))
    assert all(r <= R.BOUND_C / 2 for r in per.values()), per
