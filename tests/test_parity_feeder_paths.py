"""MAX_POOL / AVERAGE_POOL, SOFTMAX, CATEGORICAL_CROSSENTROPY / SOFTMAX_CROSSENTROPY and SGD_FORWARD (one command and the fused
multi-tensor node) on CCV_NNC_BACKEND_GPU_SM100, launch path by launch path, against the float64 oracles of tests/feeder_ref.py (pinned
to the reference's CPU_REF by tests/golden/cpuref_feeders.npz).

Every GPU case declares the path it takes and is checked against the restated plan through ccv_nnc_sm100_launch_count(); every output
lives between NaN guards that must stay NaN (pools also write through views whose pixel pitch is wider than C); every call is made
twice and must give the same bits.  The CPU tests show that the bounds reject the defects these kernels plausibly have."""
import os

import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests import feeder_ref as R
from tests.contract_ref import trunc16
from tests.util import NCHW, NHWC, pack16, ref_exec, round16, seeded, unpack16

F32, BF16, F16 = R.F32, R.BF16, R.F16
DT = {F32: abi.CCV_32F, BF16: abi.CCV_16BF, F16: abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_feeders.npz")
GUARD = 128
SENTINEL = 7.0


# ---- cases --------------------------------------------------------------------------------------------------------------------------
# (name, N or None for a 3-d tensor, H, W, C, geo = (R, S, stride_h, stride_w, begin_h, begin_w), end border (h, w),
#  declared paths for fp32 and for 16-bit: (forward = max backward, average backward))
POOL_CASES = [
    ("stem", 2, 112, 112, 64, (3, 3, 2, 2, 1, 1), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("avgdown56", 2, 56, 56, 256, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("vector", "tiles")}),
    ("avgdown28", 2, 28, 28, 512, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("vector", "tiles")}),
    ("avgdown14", 2, 14, 14, 1024, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("vector", "tiles")}),
    ("global", 4, 7, 7, 2048, (7, 7, 7, 7, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("vector", "tiles")}),
    ("avg3x3_s1", 2, 14, 14, 32, (3, 3, 1, 1, 1, 1), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("rect", 2, 11, 13, 16, (3, 2, 2, 3, 1, 0), (0, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("gaps", 2, 10, 10, 8, (2, 2, 3, 3, 0, 0), (0, 0), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("leftover", 2, 9, 9, 16, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "shortcut"), BF16: ("vector", "shortcut")}),
    ("clipped_end", 2, 7, 7, 16, (2, 2, 2, 2, 0, 0), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("clipped_end_wide", 3, 13, 5, 64, (2, 2, 2, 2, 0, 0), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("begin_ne_end", 2, 8, 8, 16, (3, 3, 2, 2, 0, 0), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
    ("c1", 2, 9, 9, 1, (3, 3, 2, 2, 1, 1), (1, 1), {F32: ("scalar", "scalar"), BF16: ("scalar", "scalar")}),
    ("c3_clipped", 2, 7, 7, 3, (2, 2, 2, 2, 0, 0), (1, 1), {F32: ("scalar", "scalar"), BF16: ("scalar", "scalar")}),
    ("c5", 2, 9, 9, 5, (3, 3, 2, 2, 1, 1), (1, 1), {F32: ("scalar", "scalar"), BF16: ("scalar", "scalar")}),
    ("c12", 2, 8, 8, 12, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("scalar", "scalar")}),
    ("three_d", None, 8, 8, 8, (2, 2, 2, 2, 0, 0), (0, 0), {F32: ("vector", "tiles"), BF16: ("vector", "tiles")}),
    ("n1", 1, 9, 9, 8, (3, 3, 2, 2, 1, 1), (1, 1), {F32: ("vector", "gather"), BF16: ("vector", "gather")}),
]


def pool_dims(case):
    name, N, H, W, C, geo, end, paths = case
    R_, S, sh, sw, ph, pw = geo
    P, Q = R.out_extent(H, R_, sh, ph, end[0]), R.out_extent(W, S, sw, pw, end[1])
    ashape = (H, W, C) if N is None else (N, H, W, C)
    bshape = (P, Q, C) if N is None else (N, P, Q, C)
    return ashape, bshape, P, Q


def as4(x):
    return x if x.ndim == 4 else x[None]


def pool_data(shape, seed, is_max, kind=F32):
    x = seeded(shape, seed, -1, 1)
    if is_max:
        x = (np.round(x * 8) / 8).astype(np.float32)  # a 1/8 grid: ties are common
    return x if kind == F32 else round16(x, DT[kind])


# ---- CPU: the oracles against CPU_REF's fixture --------------------------------------------------------------------------------------
GOLDEN_POOLS = [("max_stem", "max", (2, 9, 9, 3), (3, 3, 2, 2, 1, 1), (1, 1)), ("avg_clip", "avg", (2, 7, 7, 4), (2, 2, 2, 2, 0, 0), (1, 1)),
                ("avg_3x3", "avg", (2, 6, 6, 3), (3, 3, 1, 1, 1, 1), (1, 1)), ("avg_rect", "avg", (2, 9, 8, 2), (3, 2, 2, 3, 1, 0), (0, 1)),
                ("max_gaps", "max", (1, 9, 9, 2), (2, 2, 3, 3, 0, 0), (0, 0)), ("max_rect", "max", (2, 9, 8, 2), (3, 2, 2, 3, 1, 0), (0, 1))]
GOLDEN_LABELS = ["int", "index", "dist", "range1d"]
GOLDEN_TRIMS = [(0.0, 1.0), (0.01, 0.9)]
GOLDEN_SGD = [("nesterov", 1, 0.0, 0.0005), ("damp", 0, 0.1, 0.0005), ("nodecay", 0, 0.0, 0.0)]
SGD_HP = dict(rate=0.01, scale=1.0 / 128, momentum=0.9)


def pool_hint(geo, end):
    R_, S, sh, sw, ph, pw = geo
    return _nnc.hint((sh, sw), (ph, pw), end)


def golden_labels(which, batch, count, seed):
    """(label array, int_label) for the fixture and the GPU cases"""
    r = np.random.RandomState(seed)
    if which == "int":
        return r.randint(0, count, size=(batch,)).astype(np.int32), True
    if which == "index":  # fp32 indices off the integers, 2.6 -> 3 among them
        lab = (r.randint(0, count - 1, size=(batch,)) + r.choice([0.0, 0.3, 0.6, -0.2], size=batch)).clip(0, count - 1).astype(np.float32)
        lab[0] = 2.6
        return lab, False
    if which == "index2d":
        return golden_labels("index", batch, count, seed)[0].reshape(batch, 1), False
    if which == "dist":
        d = r.random_sample((batch, count)) ** 4
        return (d / d.sum(axis=1, keepdims=True)).astype(np.float32), False
    assert which == "range1d" and batch == 1  # a 1-d fp32 label of batch 1: the range rule makes it a distribution
    d = r.random_sample((count,)) ** 4
    return (d / d.sum()).astype(np.float32), False


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_feeders.npz missing")
    return np.load(GOLDEN)


def _f32_close(got, want, what, ulps=64):
    want = np.asarray(want, np.float64).reshape(np.shape(got))
    tol = ulps * R.U * max(np.abs(want).max(), 1e-30)
    err = np.abs(np.asarray(got, np.float64) - want).max()
    assert err <= tol, (what, err, tol)


@pytest.mark.parametrize("name,kind,shape,geo,end", GOLDEN_POOLS)
def test_pool_oracles_match_cpu_ref_fixture(name, kind, shape, geo, end):
    z = _golden()
    a, g = z[name + "_a"], z[name + "_g"]
    P, Q = g.shape[1:3]
    assert (P, Q) == (R.out_extent(shape[1], geo[0], geo[2], geo[4], end[0]), R.out_extent(shape[2], geo[1], geo[3], geo[5], end[1]))
    if kind == "max":
        b = R.max_pool(a, P, Q, geo)
        assert np.array_equal(b, z[name + "_b"])
        _f32_close(R.max_pool_bwd(g, a, b, geo)[0], z[name + "_h"], name + " h")
    else:
        _f32_close(R.avg_pool(a, P, Q, geo)[0], z[name + "_b"], name + " b")
        _f32_close(R.avg_pool_bwd(g, shape[1], shape[2], geo)[0], z[name + "_h"], name + " h")


@pytest.mark.parametrize("which", GOLDEN_LABELS)
@pytest.mark.parametrize("trims", GOLDEN_TRIMS)
def test_loss_oracles_match_cpu_ref_fixture(which, trims):
    z = _golden()
    if which == "dist" and trims != (0.0, 1.0):
        pytest.skip("a distribution label ignores the trims")
    key = "%s_%g_%g_" % (which, trims[0], trims[1])
    a, lab, g = z["loss_a"], z[key + "label"], z["loss_g"]
    batch, count = (1, a.shape[1]) if which == "range1d" else a.shape
    a2 = a[:batch]
    g1 = g[:batch]
    t = R.targets(lab, batch, count, *trims, int_label=lab.dtype == np.int32)
    y, _ = R.softmax(a2)
    _f32_close(y, (z["softmax_y"][:batch] if which != "range1d" else z["range1d_y"]).reshape(batch, count), "softmax")
    p = (z["softmax_y"][:batch] if which != "range1d" else z["range1d_y"]).reshape(batch, count)
    _f32_close(R.cce(p, t)[0], z[key + "cce_c"], key + "cce c")
    _f32_close(R.cce_bwd(g1, p, t)[0], z[key + "cce_h"], key + "cce h")
    _f32_close(R.cce_bwd(None, p, t)[0], z[key + "cce_h1"], key + "cce h without g")
    (c, _), (d, _) = R.softmax_cce(a2, t)
    _f32_close(c, z[key + "scce_c"], key + "softmax-ce c")
    _f32_close(d, z[key + "scce_d"], key + "softmax-ce d")
    _f32_close(R.softmax_cce_bwd(g1, z[key + "scce_d"].reshape(batch, count), t)[0], z[key + "scce_h"], key + "softmax-ce h")
    _f32_close(R.softmax_cce_bwd(None, z[key + "scce_d"].reshape(batch, count), t)[0], z[key + "scce_h1"], key + "softmax-ce h without g")


def test_softmax_backward_oracle_matches_cpu_ref_fixture():
    z = _golden()
    _f32_close(R.softmax_bwd(z["softmax_g"], z["softmax_y"])[0], z["softmax_h"], "softmax h", ulps=256)


@pytest.mark.parametrize("name,nesterov,dampening,decay", GOLDEN_SGD)
def test_sgd_oracle_matches_cpu_ref_fixture(name, nesterov, dampening, decay):
    z = _golden()
    (b, _), (n, _) = R.sgd(z["sgd_g"], z["sgd_a"], z["sgd_m"], nesterov, decay=decay, dampening=dampening, **SGD_HP)
    _f32_close(b, z["sgd_%s_b" % name], name + " b", ulps=4)
    _f32_close(n, z["sgd_%s_n" % name], name + " n", ulps=4)


def test_golden_pins_every_quirk():
    """the fixture holds the cases each restated quirk shows on: a clipped last window, ties, 2.6 -> 3, the range rule, trims"""
    z = _golden()
    h = z["avg_clip_h"]  # H = 7, P = 4: row 6 belongs to a window of 1 row only
    g = z["avg_clip_g"]
    assert np.isclose(h[0, 6, 0, 0], g[0, 3, 0, 0] / 2) and np.isclose(h[0, 6, 6, 0], g[0, 3, 3, 0])
    a, b = z["max_stem_a"], z["max_stem_b"]
    assert R.max_pool_bwd(np.ones_like(b), a, b, GOLDEN_POOLS[0][3])[0].sum() > b.size  # some window has tied maxima
    assert z["index_0_1_label"][0] == np.float32(2.6) and R.label_range(z["range1d_0_1_label"].shape, 1) > 1
    t = R.targets(z["index_0_1_label"], 5, 37)
    assert t[0, 3] == 1 and t[0].sum() == 1


# ---- CPU: the launch plan ------------------------------------------------------------------------------------------------------------
def test_declared_paths_are_the_plan():
    for case in POOL_CASES:
        name, N, H, W, C, geo, end, paths = case
        ashape, bshape, P, Q = pool_dims(case)
        for kind, (fwd, avg) in paths.items():
            pa, pb = (H * W * C, W * C, C), (P * Q * C, Q * C, C)
            assert R.pool_fwd_path(C, kind, pa + pb) == fwd and R.pool_max_bwd_path(C, kind, pa + pb) == fwd, (name, kind)
            assert R.pool_avg_bwd_path(H, W, P, Q, geo, C, kind, pa + pb) == avg, (name, kind)
    # a pixel pitch of C + 1 or an unaligned base takes the scalar forms
    assert R.pool_fwd_path(16, F32, (9 * 17, 17, 1)) == "scalar" and R.pool_avg_bwd_path(8, 8, 4, 4, (2, 2, 2, 2, 0, 0), 16, F32, (0,), aligned=False) == "scalar"
    assert R.pool_launches("backward", True, nchw=True) == 5 and R.pool_launches("forward", False, nchw=True) == 3
    assert [R.softmax_threads(c) for c in (1, 63, 64, 255, 256, 1023, 1024, 50257)] == [32, 32, 64, 64, 128, 128, 256, 256]
    assert R.sgd_path(4100) == "vec4" and R.sgd_path(4099) == "scalar" and R.sgd_path(8, aligned=False) == "scalar"
    assert R.sgd_multi_plan([(4, True)] * 70) == [list(range(32)), list(range(32, 64)), list(range(64, 70))]
    assert R.sgd_multi_plan([(4, True), (4, True), (5, False), (4, True), (0, True)]) == [[0, 1], [2], [3]]


# ---- CPU: the bounds reject plausible defects -----------------------------------------------------------------------------------------
def _rejects(y_bad, y_hat, e, kind=F32):
    return not R.within(y_bad, y_hat, e, kind).all()


@pytest.mark.parametrize("case", [c for c in POOL_CASES if c[0] in ("clipped_end", "c3_clipped", "avg3x3_s1", "begin_ne_end", "rect", "stem")], ids=lambda c: c[0])
def test_pool_bounds_reject_defects(case):
    name, N, H, W, C, geo, end, paths = case
    ashape, bshape, P, Q = pool_dims(case)
    a4, g4 = as4(pool_data(ashape, 1, False)), as4(seeded(bshape, 2, -1, 1))
    # the average divided by the full window instead of the clipped one, forward and backward
    b, e_b = R.avg_pool(a4, P, Q, geo)
    full = np.zeros_like(b)
    for p, q, h0, h1, w0, w1 in R._windows(H, W, P, Q, geo):
        full[:, p, q] = a4[:, h0:h1, w0:w1].astype(np.float64).sum(axis=(1, 2)) / (geo[0] * geo[1])
    assert _rejects(full, b, e_b)
    h, e_h = R.avg_pool_bwd(g4, H, W, geo)
    assert _rejects(R.avg_pool_bwd(g4, H, W, geo, full_window=True)[0], h, e_h)
    # a window one pixel off at the border (the begin border taken one smaller)
    shifted = (geo[0], geo[1], geo[2], geo[3], max(geo[4] - 1, 0), max(geo[5] - 1, 0)) if geo[4] or geo[5] else (geo[0] - 1 or 1, geo[1], geo[2], geo[3], 0, 0)
    assert _rejects(R.avg_pool(a4, P, Q, shifted)[0], b, e_b)
    # max pool: the gradient only to the first tied maximum
    am = as4(pool_data(ashape, 3, True))
    bm = R.max_pool(am, P, Q, geo)
    hm, e_hm = R.max_pool_bwd(g4, am, bm, geo)
    first = np.zeros_like(hm)
    for p, q, h0, h1, w0, w1 in R._windows(H, W, P, Q, geo):
        win = am[:, h0:h1, w0:w1].reshape(am.shape[0], -1, C)
        k = np.argmax(win == bm[:, p:p + 1, q, None, :].reshape(am.shape[0], 1, C), axis=1)
        ww = w1 - w0
        for n in range(am.shape[0]):
            for c in range(C):
                first[n, h0 + k[n, c] // ww, w0 + k[n, c] % ww, c] += g4[n, p, q, c]
    if name != "gaps":
        assert _rejects(first, hm, e_hm)
    # truncated 16-bit outputs, where the two roundings differ and the bound decides the rounding
    for kind in (BF16, F16):
        t = trunc16(h, kind)
        sel = (t != R.rne16(h, kind)) & (R.rne16(h - e_h, kind) == R.rne16(h + e_h, kind))
        assert sel.any() and not R.within(t[sel], h[sel], e_h[sel], kind).any()


SOFTMAX_COUNTS = [1, 31, 32, 63, 64, 255, 256, 1000, 1023, 1024, 50257, 2 ** 18 + 3]


@pytest.mark.parametrize("count", [c for c in SOFTMAX_COUNTS if c > 1])
def test_softmax_bounds_reject_defects(count):
    batch = 4
    a = seeded((batch, count), 1, -100, 100)  # most exps underflow
    y, e_y = R.softmax(a)
    # without the max shift: exp(a) overflows or loses the row in fp32
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        ex = np.exp(a.astype(np.float32))
        bad = ex / ex.sum(axis=1, keepdims=True, dtype=np.float32)
    assert not np.isfinite(bad).all() or _rejects(bad, y, e_y)
    # a row's last partial warp dropped from the sum
    au = seeded((batch, count), 2, -4, 4)
    yu, e_u = R.softmax(au)
    threads = R.softmax_threads(count)
    tail = count % 32 or min(32, count)
    cut = np.exp(au.astype(np.float64) - au.max(axis=1, keepdims=True))
    s_bad = cut[:, :count - tail].sum(axis=1, keepdims=True)
    if count > tail and count < 2 ** 18:  # beyond ~1e5 elements a few dropped terms are inside 8 u sqrt(K)
        assert _rejects(cut / s_bad, yu, e_u), threads
    # the backward without the sum term
    g = seeded((batch, count), 3, -1, 1)
    h, e_h = R.softmax_bwd(g, yu)
    assert _rejects(g * yu, h, e_h)
    # truncated 16-bit softmax outputs
    for kind in (BF16, F16):
        t = trunc16(yu, kind)
        sel = (t != R.rne16(yu, kind)) & (R.rne16(yu - e_u, kind) == R.rne16(yu + e_u, kind))
        assert not sel.any() or not R.within(t[sel], yu[sel], e_u[sel], kind).any()


@pytest.mark.parametrize("count", [37, 1000, 50257])
def test_loss_bounds_reject_defects(count):
    batch = 37
    a = seeded((batch, count), 1, -4, 4)
    p, _ = R.softmax(a)
    p = p.astype(np.float32)
    lab, _ = golden_labels("index", batch, count, 5)
    lab[1:] = np.floor(lab[1:]) + 0.6  # every fp32 index half-way off its integer
    # labels truncated instead of rounded
    t, t_bad = R.targets(lab, batch, count), R.targets(lab, batch, count, truncate=True)
    c, e_c = R.cce(p, t)
    assert _rejects(R.cce(p, t_bad)[0], c, e_c)
    # trim0 and trim1 swapped
    ts = R.targets(lab, batch, count, 0.1 / (count - 1), 0.9)
    tw = R.targets(lab, batch, count, 0.9, 0.1 / (count - 1))
    c2, e_c2 = R.cce(p, ts)
    assert _rejects(R.cce(p, tw)[0], c2, e_c2)
    (sc, e_sc), (d, e_d) = R.softmax_cce(a, ts)
    assert _rejects(R.softmax_cce(a, tw)[0][0], sc, e_sc)
    # the softmax-CE loss computed from the probabilities instead of the logits (an in-place call that reads d for a)
    assert _rejects(R.softmax_cce(d, ts)[0][0], sc, e_sc)
    # the backward forms: the target left out, the gradient left out
    g = seeded((batch,), 4, 0.5, 1.5)
    h, e_h = R.softmax_cce_bwd(g, d, ts)
    assert _rejects(R.softmax_cce_bwd(g, d, ts * 0)[0], h, e_h) and _rejects(R.softmax_cce_bwd(None, d, ts)[0], h, e_h)
    hc, e_hc = R.cce_bwd(g, p, ts)
    assert _rejects(R.cce_bwd(None, p, ts)[0], hc, e_hc)


def test_sgd_bounds_reject_defects():
    n_ = 4100
    g, a, m = seeded((n_,), 1, -1, 1), seeded((n_,), 2, -1, 1), seeded((n_,), 3, -1, 1)
    hp = dict(rate=0.1, scale=1.0, momentum=0.9)
    (b, e_b), (n, e_n) = R.sgd(g, a, m, 1, decay=0.01, dampening=0.0, **hp)
    # dampening applied under nesterov
    (bd, _), (nd, _) = R.sgd(g, a, m, 0, decay=0.01, dampening=0.5, **hp)
    f = lambda v: float(np.float32(v))
    n_damp = f(0.9) * m.astype(np.float64) + f(0.5) * (g.astype(np.float64) + f(0.01) * a)
    assert _rejects(n_damp, n, e_n)
    # decay added after the scale: scale (g + decay a) instead of scale g + decay a
    hp2 = dict(rate=0.1, scale=1.0 / 128, momentum=0.9)
    (b2, e_b2), (n2, e_n2) = R.sgd(g, a, m, 0, decay=0.01, dampening=0.0, **hp2)
    n_bad = f(0.9) * m.astype(np.float64) + f(1.0 / 128) * (g.astype(np.float64) + f(0.01) * a)
    assert _rejects(n_bad, n2, e_n2) and _rejects(a - f(0.1) * n_bad, b2, e_b2)
    # a fused tensor boundary off by one chunk: the first 4096 elements of tensor 1 updated with tensor 0's gradient
    g1 = seeded((n_,), 4, -1, 1)
    (b1, e_b1), _ = R.sgd(g1, a, m, 0, decay=0.01, dampening=0.0, **hp2)
    g_mix = g1.copy()
    g_mix[:R.SGD_MULTI_CHUNK] = g[:R.SGD_MULTI_CHUNK]
    assert _rejects(R.sgd(g_mix, a, m, 0, decay=0.01, dampening=0.0, **hp2)[0][0], b1, e_b1)


# ---- GPU helpers ---------------------------------------------------------------------------------------------------------------------
class Dev(object):
    """Tensors for one call.  out() tensors sit between GUARD NaN elements (check() wants them untouched); the same numpy object always
    maps to the same tensor (in-place calls).  Integer arrays travel as int32."""

    def __init__(self, nnc):
        self.nnc, self.owned, self.guarded, self.cache = nnc, [], [], {}

    def put(self, a, kind=F32, fmt=NHWC, guard=False, offset=0):
        if a is None:
            return None
        if id(a) in self.cache:
            return self.cache[id(a)]
        if a.dtype == np.int32:
            t = self.nnc.gpu_tensor(list(a.shape), fmt, abi.CCV_32S).upload(a)
            self.owned.append(t)
            self.cache[id(a)] = t
            return t
        dt = DT[kind]
        host = np.ascontiguousarray(a, np.float32) if kind == F32 else pack16(a, dt)
        nan = np.full(GUARD + offset, np.nan, np.float32)
        nan = nan if kind == F32 else pack16(nan, dt)
        tail = nan[:GUARD]
        big = self.nnc.gpu_tensor([host.size + 2 * GUARD + offset], fmt, dt).upload(np.concatenate([nan, host.ravel(), tail]))
        t = self.nnc.gpu_tensor(list(a.shape), fmt, dt, ptr=big.data_ptr + (GUARD + offset) * host.dtype.itemsize)
        if guard:
            self.guarded.append((big, host.size, kind, offset))
        self.owned += [t, big]
        self.cache[id(a)] = t
        return t

    def get(self, t, kind=F32):
        return None if t is None else (t.download() if kind == F32 else unpack16(t.download(), DT[kind]))

    def check(self):
        for big, n, kind, off in self.guarded:
            d = self.get(big, kind)
            assert np.isnan(d[:GUARD + off]).all() and np.isnan(d[GUARD + off + n:]).all(), "a guard element was written"

    def free(self):
        for t in self.owned:
            t.free()


def run(nnc, cmd, ins, outs, kinds=None, fmt=NHWC, hint=None, offset=0):
    """cmd on numpy operands; kinds: {id(array): kind}; outputs guarded; offset: elements every base is moved by (unaligned forms).
    -> (status, outputs, launches)"""
    kinds = kinds or {}
    dev = Dev(nnc)
    try:
        ti = [dev.put(a, kinds.get(id(a), F32), fmt, any(a is o for o in outs), offset) for a in ins]
        to = [dev.put(a, kinds.get(id(a), F32), fmt, True, offset) for a in outs]
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(cmd, hint, 0, ti, to)
        launches = nnc.launch_count() - l0
        res = [dev.get(t, kinds.get(id(a), F32)) for t, a in zip(to, outs)]
        dev.check()
        return st, res, launches
    finally:
        dev.free()


def run_twice(nnc, cmd, make, kinds_of=None, fmt=NHWC, hint=None, offset=0):
    """make() -> (ins, outs) fresh; the call made twice: the same status, launches and bits"""
    first = None
    for _ in range(2):
        ins, outs = make()
        got = run(nnc, cmd, ins, outs, kinds_of(ins, outs) if kinds_of else None, fmt, hint, offset)
        if first is None:
            first = got
        else:
            assert got[0] == first[0] and got[2] == first[2]
            for a, b in zip(got[1], first[1]):
                assert (a is None and b is None) or np.array_equal(a.view(np.uint32), b.view(np.uint32)), "two runs differ"
    return first


RATIOS = {}


def check(fam, what, y, y_hat, e, kind=F32):
    y = np.asarray(y)
    y_hat = np.asarray(y_hat, np.float64).reshape(y.shape)
    e = np.broadcast_to(np.asarray(e, np.float64).reshape(y.shape) if np.size(e) == y.size else e, y.shape)
    assert not np.isnan(y).any(), (fam, what, "NaN")
    ok = R.within(y, y_hat, e, kind)
    if kind == F32 and ok.all():
        RATIOS[(fam, what)] = max(RATIOS.get((fam, what), 0.0), R.ratio(y, y_hat, e))
    assert ok.all(), (fam, what, kind, "ratio to bound / C: %.2f" % R.ratio(y, y_hat, e), int((~ok).sum()), np.argwhere(~ok)[:4].tolist())


# ---- GPU: pools -----------------------------------------------------------------------------------------------------------------
def _pool_case(nnc, case, kind, is_max, fmt=NHWC, offset=0, expect=None):
    name, N, H, W, C, geo, end, paths = case
    ashape, bshape, P, Q = pool_dims(case)
    hint = pool_hint(geo, end)
    R_, S = geo[0], geo[1]
    fwd = (_nnc.CMD_MAX_POOL_FORWARD if is_max else _nnc.CMD_AVERAGE_POOL_FORWARD)(R_, S)
    bwd = (_nnc.CMD_MAX_POOL_BACKWARD if is_max else _nnc.CMD_AVERAGE_POOL_BACKWARD)(R_, S)
    a = pool_data(ashape, 11, is_max, kind)
    g = seeded(bshape, 12, -1, 1)
    g = g if kind == F32 else round16(g, DT[kind])
    k = lambda ins, outs: {id(x): kind for x in ins + outs if x is not None}
    nchw = fmt == NCHW
    tr = (lambda x: np.ascontiguousarray(np.moveaxis(x, -1, -3))) if nchw else (lambda x: x)
    back = (lambda x: np.ascontiguousarray(np.moveaxis(x, -3, -1))) if nchw else (lambda x: x)
    at, gt = tr(a), tr(g)
    st, (b,), n = run_twice(nnc, fwd, lambda: ([at], [np.zeros(at.shape[:-3] + (tr(np.zeros(bshape)).shape[-3:]), np.float32)]), k, fmt, hint, offset)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert n == R.pool_launches("forward", is_max, nchw)
    b = back(b)
    if is_max:
        assert np.array_equal(as4(b), R.max_pool(as4(a), P, Q, geo)), (name, "max forward not exact")
        ins = lambda: ([gt, at, tr(b)], [np.zeros(at.shape, np.float32)])
    else:
        b_hat, e_b = R.avg_pool(as4(a), P, Q, geo)
        check("pool", "avg forward", as4(b), b_hat, e_b, kind)
        ins = lambda: ([gt], [np.zeros(at.shape, np.float32)])
    st, (h,), n = run_twice(nnc, bwd, ins, k, fmt, hint, offset)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert n == R.pool_launches("backward", is_max, nchw)
    h = back(h)
    if is_max:
        h_hat, e_h = R.max_pool_bwd(as4(g), as4(a), as4(b), geo)
    else:
        h_hat, e_h = R.avg_pool_bwd(as4(g), H, W, geo)
    check("pool", ("max" if is_max else "avg") + " backward", as4(h), h_hat, e_h, kind)
    return b, h


POOL_GPU = [(c, k) for c in POOL_CASES for k in (F32, BF16, F16) if not (k == F16 and c[0] not in ("stem", "avgdown56", "clipped_end", "c3_clipped", "c12"))]


@pytest.mark.gpu
@pytest.mark.parametrize("is_max", [1, 0], ids=["max", "avg"])
@pytest.mark.parametrize("case,kind", POOL_GPU, ids=lambda v: v[0] if isinstance(v, tuple) else v)
def test_pool_paths(gpu, case, kind, is_max):
    pk = F32 if kind == F32 else BF16
    name, N, H, W, C, geo, end, paths = case
    ashape, bshape, P, Q = pool_dims(case)
    pa, pb = (H * W * C, W * C, C), (P * Q * C, Q * C, C)
    fwd_path, avg_path = paths[pk]
    assert R.pool_fwd_path(C, kind, pa + pb) == fwd_path and R.pool_avg_bwd_path(H, W, P, Q, geo, C, kind, pa + pb) == avg_path
    _pool_case(gpu, case, kind, is_max)


@pytest.mark.gpu
@pytest.mark.parametrize("is_max", [1, 0], ids=["max", "avg"])
@pytest.mark.parametrize("name", ["clipped_end", "stem", "c5", "rect"])
def test_pool_unaligned_base_and_nchw(gpu, name, is_max):
    """an unaligned base takes the scalar forms; NCHW runs through the layout copies and gives the NHWC bits"""
    case = [c for c in POOL_CASES if c[0] == name][0]
    for kind in (F32, BF16):
        b, h = _pool_case(gpu, case, kind, is_max)
        bu, hu = _pool_case(gpu, case, kind, is_max, offset=1)
        bn, hn = _pool_case(gpu, case, kind, is_max, fmt=NCHW)
        assert np.array_equal(b, bn) and np.array_equal(h, hn), "NCHW differs from NHWC"
        # the scalar forms add the same terms in the same order as the vector ones
        assert np.array_equal(b, bu) and np.array_equal(h, hu), "the scalar form differs"


@pytest.mark.gpu
@pytest.mark.parametrize("is_max", [1, 0], ids=["max", "avg"])
@pytest.mark.parametrize("name", ["stem", "clipped_end", "avgdown28", "leftover"])
def test_pool_views_wider_than_c(gpu, name, is_max):
    """a, b, g, h as views with a pixel pitch of C + 1 inside NaN-filled tensors: the scalar forms, only the view's elements written,
    the bits of the packed call"""
    nnc = gpu
    case = [c for c in POOL_CASES if c[0] == name][0]
    _, N, H, W, C, geo, end, paths = case
    ashape, bshape, P, Q = pool_dims(case)
    b0, h0 = _pool_case(nnc, case, F32, is_max)
    hint = pool_hint(geo, end)
    owned = []

    def wide(x, shape):
        w = np.full(shape[:-1] + (C + 1,), np.nan, np.float32)
        if x is not None:
            w[..., :C] = x
        t = nnc.gpu_tensor(list(w.shape)).upload(w)
        n_, h_, w_ = shape[:3]
        v = nnc.tensor_view_new(t, list(shape), [0] * 12, [h_ * w_ * (C + 1), w_ * (C + 1), C + 1, 1] + [0] * 8)
        owned.extend([v, t])
        return t, v
    try:
        a = pool_data(ashape, 11, is_max)
        g = seeded(bshape, 12, -1, 1)
        (_, av), (bw, bv), (_, gv), (hw, hv) = wide(a, ashape), wide(None, bshape), wide(g, bshape), wide(None, ashape)
        fwd = (nnc.CMD_MAX_POOL_FORWARD if is_max else nnc.CMD_AVERAGE_POOL_FORWARD)(geo[0], geo[1])
        bwd = (nnc.CMD_MAX_POOL_BACKWARD if is_max else nnc.CMD_AVERAGE_POOL_BACKWARD)(geo[0], geo[1])
        assert nnc.cmd_exec(fwd, hint, 0, [av], [bv]) == 0
        wb = bw.download()
        assert np.array_equal(wb[..., :C], b0) and np.isnan(wb[..., C]).all()
        (_, bvin) = wide(b0, bshape)
        assert nnc.cmd_exec(bwd, hint, 0, [gv, av, bvin] if is_max else [gv], [hv]) == 0
        wh = hw.download()
        assert np.array_equal(wh[..., :C], h0) and np.isnan(wh[..., C]).all()
    finally:
        for t in owned:
            t.free()


def free_device_bytes(device=0):
    """free memory of the device through the driver API (cuMemGetInfo in the device's primary context, the one the runtime uses), so
    that the test neither imports another CUDA framework into the process nor leaves a failed allocation's error behind"""
    import ctypes
    cu = ctypes.CDLL("libcuda.so.1")
    dev, ctx = ctypes.c_int(), ctypes.c_void_p()
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), device) == 0
    assert cu.cuDevicePrimaryCtxRetain(ctypes.byref(ctx), dev) == 0
    try:
        assert cu.cuCtxPushCurrent_v2(ctx) == 0
        try:
            assert cu.cuMemGetInfo_v2(ctypes.byref(free), ctypes.byref(total)) == 0
        finally:
            cu.cuCtxPopCurrent_v2(ctypes.byref(ctypes.c_void_p()))
    finally:
        cu.cuDevicePrimaryCtxRelease_v2(dev)
    return free.value


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_pool_64bit_index(gpu, direction):
    """more than 2^32 elements in the kernel's index space (bf16, C = 5: the scalar forms): the 64-bit branch of the index math.  The
    tensors are filled on the device with one value, the last image gets seeded data; only the last image is checked."""
    nnc = gpu
    N, H, W, C = 52429, 128, 128, 5
    total = N * H * W * C
    assert total > 2 ** 32
    need = 2 * total * 2 + (1 << 30)
    if free_device_bytes() < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 2 ** 30))
    geo, end = (2, 2, 1, 1, 0, 0), (1, 1)  # 2 x 2 / 1 with an end border: P = H, the last row and column windows clipped
    hint = pool_hint(geo, end)
    dt = DT[BF16]
    big_a = nnc.gpu_tensor([N, H, W, C], NHWC, dt)
    big_b = nnc.gpu_tensor([N, H, W, C], NHWC, dt)
    img = H * W * C
    last = lambda t: nnc.gpu_tensor([1, H, W, C], NHWC, dt, ptr=t.data_ptr + (total - img) * 2)
    la, lb = last(big_a), last(big_b)
    try:
        assert nnc.cmd_exec(nnc.CMD_SET_FORWARD(0.25), None, 0, [], [big_a]) == 0
        x = round16(seeded((1, H, W, C), 5, -1, 1), dt)
        la.upload(pack16(x, dt))
        if direction == "forward":
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(nnc.CMD_AVERAGE_POOL_FORWARD(2, 2), hint, 0, [big_a], [big_b]) == 0
            assert nnc.launch_count() - l0 == 1
            y = unpack16(lb.download(), dt)
            check("pool", "avg forward (64-bit)", y, *R.avg_pool(x, H, W, geo), kind=BF16)
        else:
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(nnc.CMD_AVERAGE_POOL_BACKWARD(2, 2), hint, 0, [big_a], [big_b]) == 0
            assert nnc.launch_count() - l0 == 1
            y = unpack16(lb.download(), dt)
            check("pool", "avg backward (64-bit)", y, *R.avg_pool_bwd(x, H, W, geo), kind=BF16)
    finally:
        for t in (la, lb, big_a, big_b):
            t.free()


# ---- GPU: softmax ---------------------------------------------------------------------------------------------------------------
def logits(shape, seed, regime):
    a = seeded(shape, seed, -4, 4)
    a2 = a.reshape(R.rows(shape))
    if regime == "peak":
        a2[:, 0] = 30
    elif regime == "wide":
        a2[:] = seeded(a2.shape, seed, -100, 100)
    elif regime == "constant":
        a2[:] = 1.5
    elif regime == "mask":
        a2[:, 1::3] = -1e30
    return a2.reshape(shape)


def _staged(kind, n16, n16_out):
    return 1 if kind == F32 else R.staged_f32_launches(n16, n16_out)


SOFTMAX_GPU = [((3, c), "uniform") for c in SOFTMAX_COUNTS] + [((1, 1000), "uniform"), ((4096, 1000), "uniform"), ((1000,), "uniform"), ((37, 10, 10, 10), "uniform")] + \
              [((37, 1000), r) for r in ("peak", "wide", "constant", "mask")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16, F16])
@pytest.mark.parametrize("shape,regime", SOFTMAX_GPU)
def test_softmax_paths(gpu, shape, regime, kind):
    nnc = gpu
    if kind != F32 and (regime != "uniform" or shape[-1] > 50257 or shape[0] == 4096):
        pytest.skip("16-bit: the functional form on the uniform rows")
    a = logits(shape, 21, regime)
    a = a if kind == F32 or regime == "mask" else round16(a, DT[kind])
    batch, count = R.rows(shape)
    k = lambda i, o: {id(x): kind for x in i + o if x is not None}
    st, (y,), n = run_twice(nnc, nnc.CMD_SOFTMAX_FORWARD(), lambda: ([a], [np.zeros(shape, np.float32)]), k)
    assert st == 0 and n == _staged(kind, 2, 1), n
    y_hat, e_y = R.softmax(a.reshape(batch, count))
    check("softmax", "y", y.reshape(batch, count), y_hat, e_y, kind)
    # in place a -> b
    ai = a.copy()
    st, (yi,), _ = run(nnc, nnc.CMD_SOFTMAX_FORWARD(), [ai], [ai], k([ai], []))
    assert st == 0 and np.array_equal(yi, y)
    g = seeded(shape, 22, -1, 1)
    g = g if kind == F32 else round16(g, DT[kind])
    st, (h,), n = run_twice(nnc, nnc.CMD_SOFTMAX_BACKWARD(), lambda: ([g, None, y], [np.zeros(shape, np.float32)]), k)
    assert st == 0 and n == _staged(kind, 3, 1)
    check("softmax", "h", h.reshape(batch, count), *R.softmax_bwd(g.reshape(batch, count), y.reshape(batch, count)), kind=kind)
    # in place g -> h
    gi = g.copy()
    st, (hi,), _ = run(nnc, nnc.CMD_SOFTMAX_BACKWARD(), [gi, None, y], [gi], k([gi, y], []))
    assert st == 0 and np.array_equal(hi, h)


# ---- GPU: cross-entropy and softmax cross-entropy ----------------------------------------------------------------------------------
LOSS_GPU = [(b, c, lab, trims) for (b, c) in ((37, 1000), (1, 1000), (4096, 1000), (3, 1), (3, 31), (3, 32), (3, 63), (3, 64), (3, 255), (3, 256), (3, 1023), (3, 1024), (3, 50257), (2, 2 ** 18 + 3))
            for lab in ("int", "index", "index2d", "dist") for trims in ((0.0, 1.0), (0.01, 0.9))
            if not (lab == "dist" and trims != (0.0, 1.0)) and (b, c) in ((37, 1000), (4096, 1000)) or (lab == "int" and trims == (0.0, 1.0)) or (lab == "index" and c > 1 and (b, c) == (3, 1023))] + \
           [(1, 1000, "range1d", (0.0, 1.0))]


def _loss_inputs(batch, count, lab, seed, regime="uniform", shape=None):
    shape = shape or (batch, count)
    a = logits(shape, seed, regime)
    label, int_label = golden_labels(lab, batch, count, seed + 1)
    return a, label, int_label


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [F32, BF16])
@pytest.mark.parametrize("batch,count,lab,trims", LOSS_GPU)
def test_cross_entropy_paths(gpu, batch, count, lab, trims, kind):
    nnc = gpu
    if kind != F32 and (count > 1024 or batch > 37):
        pytest.skip("16-bit: the functional form on the small rows")
    shape = (count,) if lab == "range1d" else (batch, count)
    a, label, int_label = _loss_inputs(batch, count, lab, 31, shape=shape)
    a = a if kind == F32 else round16(a, DT[kind])
    t = R.targets(label, batch, count, *trims, int_label=int_label)
    k = lambda i, o: {id(x): kind for x in i + o if x is not None and x.dtype != np.int32 and x is not label}
    n16 = lambda *arrs: sum(1 for x in arrs if x is not None)
    # softmax cross-entropy forward: with c, without c, and in place a -> d
    sf, sb = _nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(*trims), _nnc.CMD_SOFTMAX_CROSSENTROPY_BACKWARD(*trims)
    st, (c, d), n = run_twice(nnc, sf, lambda: ([a, label], [np.zeros((batch,), np.float32), np.zeros(shape, np.float32)]), k)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert n == _staged(kind, 3, 2)
    (c_hat, e_c), (d_hat, e_d) = R.softmax_cce(a.reshape(batch, count), t)
    check("softmax-ce", "c", c, c_hat, e_c, kind)
    check("softmax-ce", "d", d.reshape(batch, count), d_hat, e_d, kind)
    d_out = np.zeros(shape, np.float32)
    st, (none, d1), _ = run(nnc, sf, [a, label], [None, d_out], k([a], [d_out]))
    assert st == 0 and none is None and np.array_equal(d1, d)
    ai = a.copy()
    st, (ci, di), _ = run(nnc, sf, [ai, label], [np.zeros((batch,), np.float32), ai], k([ai], []))
    assert st == 0 and np.array_equal(di, d)
    check("softmax-ce", "c (in place)", ci, c_hat, e_c)  # c is an fp32 tensor in this call
    # softmax cross-entropy backward: with g, without g, in place d -> h
    g = seeded((batch,), 32, 0.5, 1.5)
    g = g if kind == F32 else round16(g, DT[kind])
    st, (h,), n = run_twice(nnc, sb, lambda: ([g, None, None, label, None, d], [np.zeros(shape, np.float32)]), k)
    assert st == 0 and n == _staged(kind, 3, 1)
    check("softmax-ce", "h", h.reshape(batch, count), *R.softmax_cce_bwd(g, d.reshape(batch, count), t), kind=kind)
    h1 = np.zeros(shape, np.float32)
    st, (h1,), _ = run(nnc, sb, [None, None, None, label, None, d], [h1], k([d], [h1]))
    assert st == 0
    check("softmax-ce", "h (no g)", h1.reshape(batch, count), *R.softmax_cce_bwd(None, d.reshape(batch, count), t), kind=kind)
    di = d.copy()
    st, (hi,), _ = run(nnc, sb, [g, None, None, label, None, di], [di], k([g, di], []))
    assert st == 0 and np.array_equal(hi, h)
    # categorical cross-entropy on the probabilities
    p = d
    cf, cb = _nnc.CMD_CATEGORICAL_CROSSENTROPY_FORWARD(*trims), _nnc.CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(*trims)
    st, (cc,), n = run_twice(nnc, cf, lambda: ([p, label], [np.zeros((batch,), np.float32)]), k)
    assert st == 0 and n == _staged(kind, 2, 1)
    check("cce", "c", cc, *R.cce(p.reshape(batch, count), t), kind=kind)
    st, (hc,), n = run_twice(nnc, cb, lambda: ([g, p, label], [np.zeros(shape, np.float32)]), k)
    assert st == 0 and n == _staged(kind, 3, 1)
    check("cce", "h", hc.reshape(batch, count), *R.cce_bwd(g, p.reshape(batch, count), t), kind=kind)
    hc1 = np.zeros(shape, np.float32)
    st, (hc1,), _ = run(nnc, cb, [None, p, label], [hc1], k([p], [hc1]))
    assert st == 0
    check("cce", "h (no g)", hc1.reshape(batch, count), *R.cce_bwd(None, p.reshape(batch, count), t), kind=kind)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["peak", "wide", "constant", "mask"])
@pytest.mark.parametrize("shape", [(37, 1000), (37, 10, 10, 10)])
def test_softmax_cross_entropy_regimes(gpu, regime, shape):
    nnc = gpu
    batch, count = R.rows(shape)
    a = logits(shape, 41, regime)
    label, _ = golden_labels("int", batch, count, 42)
    t = R.targets(label, batch, count, 0.01, 0.9, int_label=True)
    sf = _nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(0.01, 0.9)
    if regime == "mask":  # a masked logit carries weight trim0 > 0 in the loss: keep the mask off the smoothed targets
        t = R.targets(label, batch, count, int_label=True)
        sf = _nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD()
        a.reshape(batch, count)[np.arange(batch), label] = 0.5
    st, (c, d), _ = run_twice(nnc, sf, lambda: ([a, label], [np.zeros((batch,), np.float32), np.zeros(shape, np.float32)]))
    assert st == 0
    (c_hat, e_c), (d_hat, e_d) = R.softmax_cce(a.reshape(batch, count), t)
    check("softmax-ce", "c", c, c_hat, e_c)
    check("softmax-ce", "d", d.reshape(batch, count), d_hat, e_d)


# ---- GPU: SGD -------------------------------------------------------------------------------------------------------------------------
SGD_CASES = [(4100, 0, F32, 1, 0.0, 0.0005), (4100, 0, BF16, 1, 0.0, 0.0005), (4100, 0, F16, 0, 0.1, 0.0005), (4099, 0, F32, 0, 0.1, 0.0),
             (4099, 0, BF16, 1, 0.0, 0.0), (2100, 1, F32, 1, 0.0, 0.0005), (2100, 1, F16, 0, 0.0, 0.01), (1, 0, F32, 0, 0.1, 0.0005), (8192, 0, F32, 0, 0.0, 0.0)]


def _sgd_inputs(count, seed, gkind):
    g, a, m = seeded((count,), seed, -1, 1), seeded((count,), seed + 1, -1, 1), seeded((count,), seed + 2, -1, 1)
    return (g if gkind == F32 else round16(g, DT[gkind])), a, m


@pytest.mark.gpu
@pytest.mark.parametrize("count,offset,gkind,nesterov,dampening,decay", SGD_CASES)
def test_sgd_paths(gpu, count, offset, gkind, nesterov, dampening, decay):
    """offset 1: every operand a contiguous slice at an odd element offset (sgd_kernel<1>); in place (b = a, n = m) as models call it"""
    nnc = gpu
    g, a, m = _sgd_inputs(count, 51, gkind)
    cmd = nnc.CMD_SGD_FORWARD(nesterov, decay=decay, dampening=dampening, **SGD_HP)
    (b_hat, e_b), (n_hat, e_n) = R.sgd(g, a, m, nesterov, decay=decay, dampening=dampening, **SGD_HP)
    kg = lambda i, o: {id(i[0]): gkind}
    assert R.sgd_path(count, aligned=offset == 0) == ("vec4" if count % 4 == 0 and not offset else "scalar")
    st, (b, n), launches = run_twice(nnc, cmd, lambda: ([g, a, m], [np.zeros(count, np.float32), np.zeros(count, np.float32)]), kg, offset=offset)
    assert st == 0 and launches == 1
    check("sgd", "b", b, b_hat, e_b), check("sgd", "n", n, n_hat, e_n)
    ai, mi = a.copy(), m.copy()
    st, (bi, ni), _ = run(nnc, cmd, [g, ai, mi], [ai, mi], {id(g): gkind}, offset=offset)
    assert st == 0 and np.array_equal(bi, b) and np.array_equal(ni, n)
    # 16-bit parameters and momenta: the functional form (widen g, a, m; the fp32 command; narrow b, n), one rounding
    if not offset:
        a16, m16 = round16(a, DT[BF16]), round16(m, DT[BF16])
        (b16_hat, e_b16), (n16_hat, e_n16) = R.sgd(g, a16, m16, nesterov, decay=decay, dampening=dampening, **SGD_HP)
        st, (b16, n16), launches = run(nnc, cmd, [g, a16, m16], [a16, m16], {id(g): gkind, id(a16): BF16, id(m16): BF16})
        assert st == 0 and launches == R.staged_f32_launches(2 + (gkind != F32), 2)
        check("sgd", "b (bf16)", b16, b16_hat, e_b16, BF16), check("sgd", "n (bf16)", n16, n16_hat, e_n16, BF16)


def _fused_sgd(nnc, counts, gkind, nesterov, dampening, decay, odd=(), params16=()):
    """T SGD commands in one graph, fused (expect one node) and run; -> (b, n lists fused, b, n lists of the single commands, launches,
    nodes after fusion).  odd: tensors placed at an odd element offset (cannot take the vector kernel)"""
    cmd = nnc.CMD_SGD_FORWARD(nesterov, decay=decay, dampening=dampening, **SGD_HP)
    data = [_sgd_inputs(c, 100 + 3 * i, gkind) for i, c in enumerate(counts)]
    owned, stream = [], nnc.Stream(0)

    def tensor(x, kind, off=0):
        big = nnc.gpu_tensor([x.size + off + 1], NHWC, DT[kind])
        host = np.concatenate([np.zeros(off, np.float32), x.ravel(), np.zeros(1, np.float32)])
        big.upload(host if kind == F32 else pack16(host, DT[kind]))
        t = nnc.gpu_tensor([x.size], NHWC, DT[kind], ptr=big.data_ptr + off * (4 if kind == F32 else 2))
        owned.extend([t, big])
        return t
    try:
        out = []
        for fuse in (True, False):
            ts = []
            for i, (g, a, m) in enumerate(data):
                off = 1 if i in odd else 0
                pk = BF16 if i in params16 else F32
                ts.append((tensor(g, gkind, off), tensor(a if pk == F32 else round16(a, DT[pk]), pk, off), tensor(m if pk == F32 else round16(m, DT[pk]), pk, off), pk))
            gr = nnc.Graph()
            try:
                for tg, ta, tm, _ in ts:
                    gr.exec_new(cmd, None, 0, [tg, ta, tm], [ta, tm])
                nodes = len(gr)
                if fuse:
                    gr.fuse()
                    nodes = len(gr)
                l0 = nnc.launch_count()
                assert gr.run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
                stream.wait()
                launches = nnc.launch_count() - l0
            finally:
                gr.free()
            get = lambda t, k: t.download() if k == F32 else unpack16(t.download(), DT[k])
            out.append(([get(ta, pk) for _, ta, _, pk in ts], [get(tm, pk) for _, _, tm, pk in ts], launches, nodes))
        return data, out
    finally:
        for t in owned:
            t.free()
        stream.free()


SGD_FUSED = [([4] * 1, ()), ([4096] * 31, ()), ([4100] * 32, ()), ([8188, 8196, 4] * 11, ()), ([4, 4096, 4100, 8188, 8196, 1, 4] * 10, ()),
             ([4096, 4100, 4099, 8192, 8192], (3,)), ([4100] * 70, ())]


@pytest.mark.gpu
@pytest.mark.parametrize("gkind", [F32, BF16])
@pytest.mark.parametrize("counts,odd", SGD_FUSED, ids=lambda v: "T%d" % len(v) if isinstance(v, list) else str(v))
def test_fused_sgd_is_the_unfused_commands(gpu, counts, odd, gkind):
    """the multi-tensor node gives exactly the bits of the single commands; an odd-count or unaligned tensor in the middle of a run
    flushes the batch and runs alone; the launches are the restated plan"""
    nnc = gpu
    for nesterov, dampening, decay in ((1, 0.0, 0.0005), (0, 0.1, 0.0)):
        data, ((bf, nf, lf, nodes_f), (bu, nu, lu, nodes_u)) = _fused_sgd(nnc, counts, gkind, nesterov, dampening, decay, odd)
        assert nodes_f == 1 and nodes_u == len(counts)
        plan = R.sgd_multi_plan([(c, c % 4 == 0 and i not in odd) for i, c in enumerate(counts)])
        assert lf == len(plan) and lu == len(counts), (lf, plan)
        for i, (g, a, m) in enumerate(data):
            assert np.array_equal(bf[i], bu[i]) and np.array_equal(nf[i], nu[i]), "tensor %d: the fused node differs from the command" % i
            (b_hat, e_b), (n_hat, e_n) = R.sgd(g, a, m, nesterov, decay=decay, dampening=dampening, **SGD_HP)
            check("sgd", "b (fused)", bf[i], b_hat, e_b), check("sgd", "n (fused)", nf[i], n_hat, e_n)


@pytest.mark.gpu
def test_fused_sgd_resnet50_parameters(gpu):
    """ResNet-50's own parameter list (161 tensors), weights with decay and the rest without, interleaved as the model lists them"""
    nnc = gpu
    counts = _resnet50_param_counts()
    assert len(counts) == 161 and sum(counts) == 25557032
    data, ((bf, nf, lf, nodes_f), (bu, nu, lu, _)) = _fused_sgd(nnc, counts, F32, 1, 0.0, 0.0005)
    assert nodes_f == 1 and lf == len(R.sgd_multi_plan([(c, c % 4 == 0) for c in counts]))
    for i in range(len(counts)):
        assert np.array_equal(bf[i], bu[i]) and np.array_equal(nf[i], nu[i]), i


def _resnet50_param_counts():
    """the parameter shapes of ResNet-50 (torchvision layout: conv weights, batch-norm scale and bias, the classifier)"""
    counts = [64 * 3 * 7 * 7, 64, 64]
    cin = 64
    for width, blocks in ((64, 3), (128, 4), (256, 6), (512, 3)):
        for b in range(blocks):
            counts += [width * cin, width, width, width * width * 9, width, width, 4 * width * width, 4 * width, 4 * width]
            if b == 0:
                counts += [4 * width * cin, 4 * width, 4 * width]
            cin = 4 * width
    return counts + [1000 * 2048, 1000]


@pytest.mark.gpu
def test_fused_sgd_keeps_16bit_parameters_apart(gpu):
    """SGD nodes with bf16 parameters next to fp32 ones: the fuser leaves the 16-bit ones as single commands (the multi-tensor kernel
    takes fp32 parameters only) and the run gives the unfused bits"""
    nnc = gpu
    counts = [4100, 4096, 4100, 8192]
    data, ((bf, nf, lf, nodes_f), (bu, nu, lu, _)) = _fused_sgd(nnc, counts, F32, 1, 0.0, 0.0005, params16=(1, 2))
    assert nodes_f == 3
    for i in range(len(counts)):
        assert np.array_equal(bf[i], bu[i]) and np.array_equal(nf[i], nu[i]), i


# ---- refusals: CCV_NNC_EXEC_INVALID before any launch, outputs untouched ---------------------------------------------------------------
def _refused(nnc, cmd, ins, outs, kinds=None, hint=None):
    st, res, launches = run(nnc, cmd, ins, outs, kinds, NHWC, hint)
    assert st == INVALID and launches == 0, (st, launches)
    for r in res:
        assert r is None or (r == SENTINEL).all()


@pytest.mark.gpu
def test_refusals(gpu):
    nnc = gpu
    r = lambda *s: seeded(s, 3, 0.1, 0.9)
    s = lambda *shape: np.full(shape, SENTINEL, np.float32)
    lab = np.array([1, 2, 3, 4], np.int32)
    # softmax: mismatched shapes; cross-entropy: a label or loss tensor that does not hold one value per row, g of the wrong count
    _refused(nnc, nnc.CMD_SOFTMAX_FORWARD(), [r(4, 10)], [s(4, 9)])
    _refused(nnc, nnc.CMD_SOFTMAX_BACKWARD(), [r(4, 10), None, r(4, 9)], [s(4, 10)])
    _refused(nnc, nnc.CMD_CATEGORICAL_CROSSENTROPY_FORWARD(), [r(4, 10), lab], [s(2)])
    _refused(nnc, nnc.CMD_CATEGORICAL_CROSSENTROPY_FORWARD(), [r(4, 10), lab[:2]], [s(4)])
    _refused(nnc, nnc.CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(), [r(2), r(4, 10), lab], [s(4, 10)])
    _refused(nnc, nnc.CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(), [None, r(4, 10), r(4, 9)], [s(4, 10)])
    _refused(nnc, nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(), [r(4, 10), lab], [s(2), s(4, 10)])
    _refused(nnc, nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(), [r(4, 10), r(4, 9)], [s(4), s(4, 10)])
    _refused(nnc, nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(), [r(4, 10), lab], [s(4), s(4, 9)])
    _refused(nnc, nnc.CMD_SOFTMAX_CROSSENTROPY_BACKWARD(), [r(3), None, None, lab, None, r(4, 10)], [s(4, 10)])
    _refused(nnc, nnc.CMD_SOFTMAX_CROSSENTROPY_BACKWARD(), [None, None, None, lab[:3], None, r(4, 10)], [s(4, 10)])
    # pools: a max-pool backward whose a does not share h's strides (shape), channel counts that differ
    hint = pool_hint((2, 2, 2, 2, 0, 0), (0, 0))
    _refused(nnc, nnc.CMD_MAX_POOL_BACKWARD(2, 2), [r(1, 4, 4, 8), r(1, 8, 8, 4), r(1, 4, 4, 8)], [s(1, 8, 8, 8)], hint=hint)
    _refused(nnc, nnc.CMD_AVERAGE_POOL_FORWARD(2, 2), [r(1, 8, 8, 8)], [s(1, 4, 4, 4)], hint=hint)
    # SGD: nesterov with dampening, mismatched counts
    cmd = nnc.CMD_SGD_FORWARD(1, decay=0.0, dampening=0.1, **SGD_HP)
    _refused(nnc, cmd, [r(8), r(8), r(8)], [s(8), s(8)])
    _refused(nnc, nnc.CMD_SGD_FORWARD(0, decay=0.0, dampening=0.0, **SGD_HP), [r(8), r(8), r(4)], [s(8), s(8)])
    # views where the softmax kernels assume packed rows
    wide = nnc.gpu_tensor([4, 12]).upload(r(4, 12))
    out = nnc.gpu_tensor([4, 10]).upload(s(4, 10))
    v = nnc.tensor_view_new(wide, [4, 10], [0] * 12, [12, 1] + [0] * 10)
    try:
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(nnc.CMD_SOFTMAX_FORWARD(), None, 0, [v], [out]) == INVALID and nnc.launch_count() == l0
        assert (out.download() == SENTINEL).all()
    finally:
        for t in (v, wide, out):
            t.free()


@pytest.mark.gpu
def test_fused_sgd_refuses_nesterov_with_dampening(gpu):
    """a fused node validates its hyper-parameters as the single command does: refused before any launch, parameters untouched"""
    nnc = gpu
    cmd = nnc.CMD_SGD_FORWARD(1, decay=0.0, dampening=0.1, **SGD_HP)
    ts = [nnc.gpu_tensor([8]).upload(np.full(8, SENTINEL, np.float32)) for _ in range(6)]
    gr, stream = nnc.Graph(), nnc.Stream(0)
    try:
        gr.exec_new(cmd, None, 0, ts[0:3], ts[1:3])
        gr.exec_new(cmd, None, 0, ts[3:6], ts[4:6])
        assert gr.fuse() == 1
        l0 = nnc.launch_count()
        assert gr.run(stream) == INVALID
        stream.wait()
        assert nnc.launch_count() == l0 and all((t.download() == SENTINEL).all() for t in ts)
    finally:
        gr.free(), stream.free()
        for t in ts:
            t.free()


@pytest.mark.gpu
@pytest.mark.ref
def test_against_cpu_ref(gpu, ref):
    """where the compiled reference is present: the clipped-window average-pool backward and the in-place softmax-CE against CPU_REF"""
    nnc = gpu
    a = seeded((1, 7, 7, 16), 61, -1, 1)
    g = seeded((1, 4, 4, 16), 62, -1, 1)
    hint = pool_hint((2, 2, 2, 2, 0, 0), (1, 1))
    bwd = nnc.CMD_AVERAGE_POOL_BACKWARD(2, 2)
    st_r, (h_r,) = ref_exec(ref, bwd, hint, 0, [g[0]], [np.zeros((7, 7, 16), np.float32)])
    st, (h,), _ = run(nnc, bwd, [g], [np.zeros((1, 7, 7, 16), np.float32)], hint=hint)
    assert st_r == 0 and st == 0 and np.abs(h[0] - h_r).max() <= 1e-6
    x = seeded((5, 37), 63, -4, 4)
    lab = np.array([1, 5, 36, 0, 2], np.int32)
    sf = nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD()
    _, (c_r, _) = ref_exec(ref, sf, None, 0, [x.copy(), lab], [np.zeros(5, np.float32), np.zeros_like(x)])
    xi = x.copy()
    st, (c, _), _ = run(nnc, sf, [xi, lab], [np.zeros(5, np.float32), xi])
    assert st == 0 and np.abs(c - c_r).max() <= 1e-5 * np.abs(c_r).max()


@pytest.mark.gpu
def test_zz_report_measured_ratios(gpu):
    """prints the largest |y - y_hat| / (bound / BOUND_C) per family and output over the cases run before it in this session"""
    per = {}
    for (fam, what), r in sorted(RATIOS.items()):
        print("ratio %-10s %-26s %.3f" % (fam, what, r))
        per[fam] = max(per.get(fam, 0.0), r)
    print("largest ratio per family:", ", ".join("%s %.3f" % kv for kv in sorted(per.items())))
    assert all(r <= R.BOUND_C for r in per.values())
