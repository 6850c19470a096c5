"""BINARY_CROSSENTROPY, SIGMOID_BINARY_CROSSENTROPY, MSE and SMOOTH_L1 (forward / backward) on CCV_NNC_BACKEND_GPU_SM100 against the
oracles of tests/loss_ref.py, which are pinned to the reference's CPU_REF by tests/golden/cpuref_loss.npz.

Forward: the kernel's per-row sum is fp32 in a fixed order of its own (sm100_loss.cu), so it is checked against the float64 oracle
with the bound of loss_ref.bound: |y - y_hat| <= C (2^-24 sqrt(K) S + eps_f S), K the row's term count, S the sum of the magnitudes of
its terms (pos_weight times the second BCE sum's), eps_f the per-term error of the accurate fp32 logf / expf / log1pf (a few ulps,
loss_ref.TERM_ULPS).  A 16-bit output y must satisfy rne16(y_hat - e) <= y <= rne16(y_hat + e).  Backward: CPU_REF's fp32
operations in CPU_REF's order, so fp32 gradients equal the oracle (and CPU_REF) bit for bit, 16-bit ones the oracle on the widened
inputs, rounded once to nearest even."""
import os

import numpy as np
import pytest

from ccv_b200 import abi
from tests import loss_ref as L
from tests.util import NHWC, counted, gpu_exec, gpu_exec16, pack16, ref_exec, round16, seeded, unpack16

KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_loss.npz")

# (name, op, parameter): every command and form
FORMS = [("bce", L.BCE, 1.0), ("bce_pw", L.BCE, 2.5), ("sbce", L.SBCE, 1.0), ("sbce_pw", L.SBCE, 2.5),
         ("mse_mean", L.MSE, L.MEAN), ("mse_sum", L.MSE, L.SUM), ("sl1", L.SL1, 1.0)]
SHAPES = [(10, 100), (300,), (6, 1), (6, 7), (5, 1001), (65536, 4), (4096, 1000), (3, 2 ** 20 + 5), (1, 2 ** 22)]


def commands(nnc, op, param):
    if op == L.BCE:
        return nnc.CMD_BINARY_CROSSENTROPY_FORWARD(param), nnc.CMD_BINARY_CROSSENTROPY_BACKWARD(param)
    if op == L.SBCE:
        return nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_FORWARD(param), nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_BACKWARD(param)
    if op == L.MSE:
        return nnc.CMD_MSE_FORWARD(param), nnc.CMD_MSE_BACKWARD(param)
    return nnc.CMD_SMOOTH_L1_FORWARD(param), nnc.CMD_SMOOTH_L1_BACKWARD(param)


def operands(op, shape, seed, kind=abi.CCV_32F, b32=False):
    """(a, b): a in the loss's domain, b labels / targets; values a `kind` tensor holds (b stays fp32 when b32)"""
    a = seeded(shape, seed, 0.02, 0.98) if op == L.BCE else seeded(shape, seed, -4, 4) if op == L.SBCE else seeded(shape, seed, -1, 1)
    if op in (L.BCE, L.SBCE):
        b = (seeded(shape, seed + 1) > 0.5).astype(np.float32)
        b[..., ::3] = seeded(b[..., ::3].shape, seed + 2)  # soft labels too
    elif op == L.MSE:
        b = seeded(shape, seed + 1, -1, 1)
    else:
        # each row far from the switch at beta = 1: even rows sum |b - a| to about 0.3, odd rows to about 3
        r = L.rows(a)
        k = r.shape[1]
        amp = np.where(np.arange(r.shape[0]) % 2 == 0, 0.3, 3.0)[:, None] / k
        b = (r + amp * np.where(seeded(r.shape, seed + 1) > 0.5, 1.0, -1.0) * seeded(r.shape, seed + 2, 0.5, 1.5)).astype(np.float32).reshape(shape)
    if kind != abi.CCV_32F:
        a = round16(a, kind)
        b = b if b32 else round16(b, kind)
    return a, b


def _rne16(x, kind):
    return round16(np.asarray(x, np.float32), kind).astype(np.float64)


def within(y, y_hat, e, kind):
    """y (what the kernel stored) against the oracle y_hat +- e; for 16-bit outputs the interval's ends rounded like the output"""
    y, y_hat, e = (np.asarray(v, np.float64).ravel() for v in (y, y_hat, e))
    if kind == abi.CCV_32F:
        return np.abs(y - y_hat) <= e
    return (_rne16(y_hat - e, kind) <= y) & (y <= _rne16(y_hat + e, kind))


# ---- CPU: the oracles against CPU_REF's fixture, and the bound against defects ------------------------------------------------
def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_loss.npz missing")
    return np.load(GOLDEN)


@pytest.mark.parametrize("name,op,param", FORMS)
def test_forward_oracle_matches_cpu_ref_fixture(name, op, param):
    """CPU_REF's forward (a sequential fp32 sum of double terms) is within the bound of the float64 oracle (its error is of the same
    kind: K roundings of a sum); the sigmoid of SBCE (d) within 1 ulp of the float64 one"""
    z = _golden()
    a, b = z["a_" + op], z["b_" + op]
    y_hat, S = L.forward(op, a, b, param)
    y = z["c_" + name]
    assert within(y, y_hat, L.bound(op, a.shape[1], S), abi.CCV_32F).all(), (name, np.abs(y - y_hat).max())
    if op == L.SBCE:
        d = z["d_" + name]
        assert np.abs(d - L.sigmoid(a)).max() <= np.spacing(np.float32(1)) / 2


@pytest.mark.parametrize("name,op,param", FORMS)
@pytest.mark.parametrize("with_g", [1, 0])
def test_backward_oracle_matches_cpu_ref_fixture(name, op, param, with_g):
    z = _golden()
    a, b, g = z["a_" + op], z["b_" + op], z["g"] if with_g else None
    tag = "%s_g%d" % (name, with_g)
    if op == L.BCE:
        assert np.array_equal(L.bce_backward(g, a, b, param), z["h_" + tag])
        assert np.array_equal(L.bce_backward(g, z["a_clamp"], z["b_clamp"], param), z["hclamp_" + tag])
    elif op == L.SBCE:
        assert np.array_equal(L.sbce_backward(g, b, z["d_" + name], param), z["h_" + tag])
    elif op == L.MSE:
        ha, hb = L.mse_backward(g, a, b, param)
        assert np.array_equal(ha, z["ha_" + tag]) and np.array_equal(hb, z["hb_" + tag])
    else:
        assert np.array_equal(L.sl1_backward(g, a, b, z["c_" + name], param), z["h_" + tag])


def test_fixture_covers_both_smooth_l1_branches_and_the_clamp():
    z = _golden()
    c = z["c_sl1"]
    assert (c < 0.5).any() and (c >= 0.5).any()
    a = z["a_clamp"]
    assert (a == 1).any() and (((1 - a) * a).astype(np.float64) <= 1e-12).any()


MUTATION_SHAPES = [(10, 100), (3, 2 ** 20 + 5), (1, 2 ** 22), (65536, 4), (4096, 1000)]


@pytest.mark.parametrize("shape", MUTATION_SHAPES)
def test_bound_rejects_defects(shape):
    """Each defect a kernel could have moves the loss outside the bound on every row of the shape (16-bit truncation: on rows where
    truncating and rounding differ at all)."""
    count = shape[-1]
    _, _, chunks, _, _ = L.plan(L.MSE, 1, shape[0], count, 4)
    # MSE: a dropped last chunk of a split row, a chunk counted twice, a missing mean scale
    a, b = operands(L.MSE, shape, 3)
    L.rows(b)[:, -5:] += 30.0  # the last chunk of (3, 2^20 + 5) holds 5 elements: give them weight
    y_hat, S = L.mse_forward(a, b, L.MEAN)
    e = L.bound(L.MSE, count, S)
    ra, rb = L.rows(a), L.rows(b)
    scale = L.mse_scale(count, L.MEAN)
    if chunks > 1:
        last = 4 * 2048 * (chunks - 1)
        tail = ((rb[:, last:].astype(np.float64) - ra[:, last:]) ** 2).sum(1) * scale
        first = ((rb[:, :4 * 2048].astype(np.float64) - ra[:, :4 * 2048]) ** 2).sum(1) * scale
        assert not within(y_hat - tail, y_hat, e, abi.CCV_32F).any()
        assert not within(y_hat + first, y_hat, e, abi.CCV_32F).any()
    assert not within(y_hat / scale, y_hat, e, abi.CCV_32F).any()
    # smooth L1: the per-element Huber loss in place of the row switch (the two differ on the rows of the linear branch)
    a, b = operands(L.SL1, (2, count) if len(shape) == 1 or shape[0] == 1 else shape, 5)  # a row of each branch
    y_hat, S = L.sl1_forward(a, b, 1.0)
    bad, _ = L.sl1_forward(a, b, 1.0, huber=True)
    linear = y_hat >= 0.5
    assert linear.any() and not within(bad[linear], y_hat[linear], L.bound(L.SL1, count, S)[linear], abi.CCV_32F).any()
    # BCE: pos_weight on the wrong sum (a below 1/2, so that the two sums do not cancel)
    a = seeded(shape, 7, 0.02, 0.5)
    _, b = operands(L.BCE, shape, 7)
    y_hat, S = L.bce_forward(a, b, 2.5)
    ra, rb = L.rows(a), L.rows(b)
    t1 = ((rb - np.float32(1)).astype(np.float64) * np.log((np.float32(1) - ra).astype(np.float64))).sum(1)
    t2 = (rb.astype(np.float64) * np.log(ra.astype(np.float64))).sum(1)
    assert not within(2.5 * t1 - t2, y_hat, L.bound(L.BCE, count, S), abi.CCV_32F).any()
    # 16-bit outputs truncated instead of rounded to nearest even, on the rows whose rounding the bound determines
    for kind in (abi.CCV_16BF, abi.CCV_16F):
        a, b = operands(L.MSE, shape, 9, kind)
        y_hat, S = L.mse_forward(a, b, L.MEAN)
        e = L.bound(L.MSE, count, S)
        y = np.asarray(y_hat, np.float32)
        if kind == abi.CCV_16BF:
            trunc = (y.view(np.uint32) & 0xFFFF0000).view(np.float32)
        else:
            r = y.astype(np.float16)
            trunc = np.where(np.abs(r.astype(np.float32)) > np.abs(y), np.nextafter(r, np.float16(0)), r).astype(np.float32)
        rows = (trunc != round16(y, kind)) & (_rne16(y_hat - e, kind) == _rne16(y_hat + e, kind))
        assert rows.any() or L.rows(a).shape[0] < 10  # with a few rows, truncation may happen to round correctly
        assert not within(trunc[rows], y_hat[rows], e[rows], kind).any()


def test_bound_rejects_the_naive_softplus():
    """log(1 + expf(-a)) in fp32 overflows to inf at a = -100, where CPU_REF (in double) gives 100 per term"""
    a = np.array([[-100.0, 100.0, -100.0, 3.0]], np.float32)
    b = np.array([[1.0, 0.0, 0.0, 1.0]], np.float32)
    y_hat, S = L.sbce_forward(a, b, 1.0)
    with np.errstate(over="ignore"):
        naive = ((1 - b) * a + np.log1p(np.exp(-a)).astype(np.float32)).astype(np.float64).sum(1)
    assert np.isfinite(y_hat).all() and not within(naive, y_hat, L.bound(L.SBCE, 4, S), abi.CCV_32F).any()


def test_plan():
    """the plan restated in loss_ref against the shapes the kernel's comment describes"""
    assert L.plan(L.SL1, 1, 2 ** 20, 4, 4) == (1, 1, 1, 0, 1)           # box rows: one thread per row, one 16-byte vector
    assert L.plan(L.BCE, 1, 4096, 1000, 4)[1:3] == (32, 1)              # a warp per row
    assert L.plan(L.MSE, 1, 8, 2 ** 21, 4) == (2 ** 19, 256, 256, 8 * 256 * 4, 2)
    assert L.plan(L.SL1, 1, 3, 2 ** 20 + 5, 4)[2:] == (129, 3 * 129 * 2 * 4, 2)  # the last chunk is partial
    assert L.plan(L.SBCE, 1, 1, 2 ** 22, 2, with_c=False)[3:] == (0, 1)  # d only: no partials, one launch


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def _run(nnc, cmd, ins, outs, kind, b32=None, flags=0):
    if kind == abi.CCV_32F:
        return counted(nnc, gpu_exec, cmd, None, flags, ins, outs)
    return counted(nnc, gpu_exec16, cmd, None, flags, ins, outs, kind, keep32=(id(b32),) if b32 is not None else ())


def _fwd_outs(op, batch, shape):
    c = np.zeros((batch,), np.float32)
    return [c, np.zeros(shape, np.float32)] if op == L.SBCE else [c]


CASES = [(n, op, p, s, k) for (n, op, p) in FORMS for s in SHAPES for k in sorted(KINDS)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,op,param,shape,kname", CASES)
def test_forward(gpu, name, op, param, shape, kname):
    nnc, kind = gpu, KINDS[kname]
    b32 = kind != abi.CCV_32F and shape == (10, 100)  # fp32 labels under 16-bit activations
    a, b = operands(op, shape, 11, kind, b32)
    batch, count = L.rows(a).shape
    fwd, _ = commands(nnc, op, param)
    st, outs, launches = _run(nnc, fwd, [a, b], _fwd_outs(op, batch, shape), kind, b if b32 else None)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert launches == L.plan(op, param, batch, count, 4 if kind == abi.CCV_32F else 2)[4]
    y_hat, S = L.forward(op, a, b, param)
    e = L.bound(op, count, S)
    ok = within(outs[0], y_hat, e, kind)
    if kind == abi.CCV_32F:
        print("\nforward %s %s: max |y - y_hat| / (bound / C) = %.3f" % (name, shape, (np.abs(outs[0] - y_hat) / (e / L.BOUND_C)).max()))
    assert ok.all(), (name, shape, kname, np.abs(outs[0] - y_hat).max(), e.max())
    if op == L.SL1:
        assert (L.sl1_margin(a, b) > 100 * e).all()
    if op == L.SBCE:
        d, want = outs[1], L.sigmoid(a)
        if kind == abi.CCV_32F:
            ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
            assert (np.abs(d - want) <= 4 * ulp).all(), np.abs(d - want).max()
        else:
            # the fp32 sigmoid within 4 ulps, then rounded to 16 bits: half a 16-bit ulp more (and the 16-bit subnormal spacing)
            half = np.abs(want) * (2.0 ** -8 if kind == abi.CCV_16BF else 2.0 ** -11) + (1e-40 if kind == abi.CCV_16BF else 2.0 ** -25)
            assert (np.abs(d - want) <= half + 4 * np.spacing(np.abs(want).astype(np.float32))).all()


def _backward(nnc, op, param, a, b, kind, g, b32=False, forms=None):
    """run every backward form of `op` for (g | None, a, b) against the oracle; returns the launch counts"""
    batch, count = L.rows(a).shape
    fwd, bwd = commands(nnc, op, param)
    shape = a.shape
    z = lambda: np.zeros(shape, np.float32)
    bk = b if b32 else None
    r16 = (lambda x: x) if kind == abi.CCV_32F else (lambda x: round16(x, kind))
    launches = []
    if op == L.BCE:
        st, (h,), n = _run(nnc, bwd, [g, a, b], [z()], kind, bk)
        assert st == 0
        assert np.array_equal(h.reshape(L.rows(a).shape), r16(L.bce_backward(g, a, b, param)))
        launches.append(n)
    elif op == L.SBCE:
        d = L.sigmoid(a).astype(np.float32)
        d = r16(d)
        st, (h,), n = _run(nnc, bwd, [g, None, None, b, None, d], [z()], kind, bk)
        assert st == 0
        assert np.array_equal(h.reshape(L.rows(a).shape), r16(L.sbce_backward(g, b, d, param)))
        launches.append(n)
    elif op == L.MSE:
        ha_w, hb_w = L.mse_backward(g, a, b, param)
        for outs in ([z(), z()], [z(), None], [None, z()]):
            st, got, n = _run(nnc, bwd, [g, a, b], outs, kind, bk)
            assert st == 0
            for x, w in zip(got, (ha_w, hb_w)):
                if x is not None:
                    assert np.array_equal(x.reshape(w.shape), r16(w))
            launches.append(n)
    else:
        c_hat, _ = L.sl1_forward(a, b, param)
        c = r16(c_hat.astype(np.float32))
        st, (h,), n = _run(nnc, bwd, [g, a, b, c], [z()], kind, bk)
        assert st == 0
        assert np.array_equal(h.reshape(L.rows(a).shape), r16(L.sl1_backward(g, a, b, c, param)))
        launches.append(n)
    return launches


@pytest.mark.gpu
@pytest.mark.parametrize("name,op,param,shape,kname", CASES)
def test_backward(gpu, name, op, param, shape, kname):
    nnc, kind = gpu, KINDS[kname]
    b32 = kind != abi.CCV_32F and shape == (10, 100)
    a, b = operands(op, shape, 21, kind, b32)
    batch = L.rows(a).shape[0]
    g = seeded((batch,), 23, 0.5, 2)
    g = g if kind == abi.CCV_32F else round16(g, kind)
    for gg in (g, None):
        assert _backward(nnc, op, param, a, b, kind, gg, b32) in ([1], [1, 1, 1])


@pytest.mark.gpu
@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("pw", [1.0, 2.5])
def test_bce_backward_reaches_the_clamp(gpu, kname, pw):
    """a = 1 (and a = 0) make (1 - a) a = 0: CPU_REF divides by 1e-12 in double"""
    nnc, kind = gpu, KINDS[kname]
    a = np.array([[1.0, 0.0, 0.5, 1.0, 0.25, 1.0, 0.0, 0.75]] * 3, np.float32)
    b = np.array([[0.0, 1.0, 1.0, 1.0, 0.0, 0.5, 0.0, 0.0]] * 3, np.float32)
    g = np.array([1.0, 0.5, 2.0], np.float32)
    for gg in (g, None):
        _backward(nnc, L.BCE, pw, a, b, kind, gg)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", sorted(KINDS))
def test_sigmoid_bce_extreme_logits(gpu, kname):
    """logits of +-100: the loss stays finite (100 per term where the label is wrong), d is 0 / 1 within rounding"""
    nnc, kind = gpu, KINDS[kname]
    a = np.tile(np.array([-100.0, 100.0, -100.0, 100.0, 3.0, -3.0, 0.0, 50.0], np.float32), (4, 1))
    b = np.tile(np.array([1.0, 0.0, 0.0, 1.0, 1.0, 0.0, 0.5, 1.0], np.float32), (4, 1))
    a = a if kind == abi.CCV_32F else round16(a, kind)
    fwd, _ = commands(nnc, L.SBCE, 2.0)
    st, (c, d), _ = _run(nnc, fwd, [a, b], [np.zeros(4, np.float32), np.zeros(a.shape, np.float32)], kind)
    assert st == 0
    y_hat, S = L.sbce_forward(a, b, 2.0)
    assert np.isfinite(c).all() and within(c, y_hat, L.bound(L.SBCE, 8, S), kind).all(), (c, y_hat)
    assert np.abs(d - L.sigmoid(a)).max() <= 4e-3


@pytest.mark.gpu
@pytest.mark.parametrize("name,op,param", FORMS)
def test_forward_is_deterministic(gpu, name, op, param):
    nnc = gpu
    shape = (3, 2 ** 20 + 5)
    a, b = operands(op, shape, 31)
    fwd, _ = commands(nnc, op, param)
    runs = [_run(nnc, fwd, [a, b], _fwd_outs(op, 3, shape), abi.CCV_32F)[1] for _ in range(2)]
    for x, y in zip(*runs):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("name,op,param", FORMS)
def test_views_and_guards(gpu, name, op, param, kname):
    """a, b and the element-wise output as row-pitched slices of wider NaN-filled tensors; c as a pitched [batch, 1] view.  Only the
    slices change, and they hold what packed operands give (bit for bit: the plan does not depend on alignment)."""
    nnc, kind = gpu, KINDS[kname]
    batch, count, pitch, ofs = 6, 37, 53, 5
    a, b = operands(op, (batch, count), 41, kind)
    g = seeded((batch,), 43, 0.5, 2)
    g = g if kind == abi.CCV_32F else round16(g, kind)
    fwd, bwd = commands(nnc, op, param)
    up = lambda x: x if kind == abi.CCV_32F else pack16(x, kind)
    down = lambda t: t.download() if kind == abi.CCV_32F else unpack16(t.download(), kind)
    owned = []

    def wide(x, fill):
        w = np.full((batch, pitch), fill, np.float32)
        if x is not None:
            w[:, ofs:ofs + count] = x
        t = nnc.gpu_tensor([batch, pitch], NHWC, kind).upload(up(w))
        v = nnc.tensor_view_new(t, [batch, count], [0, ofs] + [0] * 10, [pitch, 1] + [0] * 10)
        owned.extend([v, t])
        return t, v

    def dense(x):
        t = nnc.gpu_tensor(list(x.shape), NHWC, kind).upload(up(x))
        owned.append(t)
        return t

    try:
        _, av = wide(a, 0.0)
        _, bv = wide(b, 0.0)
        cw = nnc.gpu_tensor([batch, 3], NHWC, kind).upload(up(np.full((batch, 3), np.nan, np.float32)))
        cv = nnc.tensor_view_new(cw, [batch, 1], [0, 1] + [0] * 10, [3, 1] + [0] * 10)
        owned.extend([cv, cw])
        outs = [cv]
        if op == L.SBCE:
            dw, dv = wide(None, np.nan)
            outs.append(dv)
        assert nnc.cmd_exec(fwd, None, 0, [av, bv], outs) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        st, want, _ = _run(nnc, fwd, [a, b], _fwd_outs(op, batch, (batch, count)), kind)
        c_all = down(cw)
        assert np.isnan(c_all[:, [0, 2]]).all() and np.array_equal(c_all[:, 1], want[0])
        if op == L.SBCE:
            d_all = down(dw)
            assert np.isnan(d_all[:, :ofs]).all() and np.isnan(d_all[:, ofs + count:]).all()
            assert np.array_equal(d_all[:, ofs:ofs + count], want[1])
        # backward into a pitched h
        hw, hv = wide(None, np.nan)
        gt = dense(g)
        if op == L.BCE:
            ins, ref_ins = [gt, av, bv], [g, a, b]
        elif op == L.SBCE:
            d = want[1]
            _, ddv = wide(d, 0.0)
            ins, ref_ins = [gt, None, None, bv, None, ddv], [g, None, None, b, None, d]
        elif op == L.MSE:
            ins, ref_ins = [gt, av, bv], [g, a, b]
        else:
            ct = dense(want[0])
            ins, ref_ins = [gt, av, bv, ct], [g, a, b, want[0]]
        assert nnc.cmd_exec(bwd, None, 0, ins, [hv]) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        _, (h_want,), _ = _run(nnc, bwd, ref_ins, [np.zeros((batch, count), np.float32)], kind)
        h_all = down(hw)
        assert np.isnan(h_all[:, :ofs]).all() and np.isnan(h_all[:, ofs + count:]).all()
        assert np.array_equal(h_all[:, ofs:ofs + count], h_want)
    finally:
        for t in owned:
            t.free()


@pytest.mark.gpu
def test_accumulate_output_overwrites(gpu):
    nnc = gpu
    a, b = operands(L.MSE, (4, 64), 51)
    fwd, bwd = commands(nnc, L.MSE, L.MEAN)
    st0, (c0,), _ = _run(nnc, fwd, [a, b], [np.zeros(4, np.float32)], abi.CCV_32F)
    st1, (c1,), _ = _run(nnc, fwd, [a, b], [np.ones(4, np.float32)], abi.CCV_32F, flags=abi.CCV_NNC_ACCUMULATE_OUTPUT)
    assert st0 == 0 and st1 == 0 and np.array_equal(c0, c1)
    g = np.ones(4, np.float32)
    st, (ha,), _ = _run(nnc, bwd, [g, a, b], [np.full((4, 64), 5.0, np.float32)], abi.CCV_32F, flags=abi.CCV_NNC_ACCUMULATE_OUTPUT)
    assert st == 0 and np.array_equal(ha, L.mse_backward(g, a, b, L.MEAN)[0])


SENTINEL = 7.0


def _refused(nnc, cmd, ins, outs):
    st, res, launches = counted(nnc, gpu_exec, cmd, None, 0, ins, outs)
    assert st == INVALID and launches == 0, (st, launches)
    for r in res:
        assert r is None or (r == SENTINEL).all()


@pytest.mark.gpu
def test_refusals(gpu):
    nnc = gpu
    r = lambda *s: seeded(s, 3, 0.1, 0.9)
    s = lambda *shape: np.full(shape, SENTINEL, np.float32)
    bce_f, bce_b = commands(nnc, L.BCE, 1.0)
    mse_f, mse_b = commands(nnc, L.MSE, L.MEAN)
    sl1_f, sl1_b = commands(nnc, L.SL1, 1.0)
    sb_f, sb_b = commands(nnc, L.SBCE, 1.0)
    # more than 2 axes; mismatched a / b; mismatched h; c or g count != batch
    _refused(nnc, bce_f, [r(2, 3, 4), r(2, 3, 4)], [s(2)])
    _refused(nnc, mse_f, [r(4, 8), r(4, 9)], [s(4)])
    _refused(nnc, bce_b, [r(4), r(4, 8), r(4, 8)], [s(4, 9)])
    _refused(nnc, sl1_f, [r(4, 8), r(4, 8)], [s(5)])
    _refused(nnc, mse_b, [r(3), r(4, 8), r(4, 8)], [s(4, 8), None])
    # mixed types other than 16-bit a with fp32 b: fp32 a with 16-bit b; a 16-bit output under fp32 a; an integer operand
    _refused(nnc, mse_f, [r(4, 8), r(4, 8).astype(np.float16)], [s(4)])
    _refused(nnc, mse_b, [r(4), r(4, 8), r(4, 8)], [s(4, 8).astype(np.float16), None])
    _refused(nnc, mse_f, [r(4, 8), (r(4, 8) * 10).astype(np.int32)], [s(4)])
    # missing operands a requested output needs
    _refused(nnc, sl1_b, [r(4), r(4, 8), r(4, 8), None], [s(4, 8)])
    _refused(nnc, sb_b, [r(4), None, None, r(4, 8), None, None], [s(4, 8)])
    _refused(nnc, bce_b, [r(4), None, r(4, 8)], [s(4, 8)])
    _refused(nnc, mse_b, [r(4), r(4, 8), r(4, 8)], [None, None])
    _refused(nnc, sb_f, [r(4, 8), r(4, 8)], [s(4), None])
    # g as a view; a non-contiguous inner axis; a palettized operand
    base = nnc.gpu_tensor([4, 16]).upload(r(4, 16))
    gbase = nnc.gpu_tensor([4, 2]).upload(r(4, 2))
    a, b, h = nnc.gpu_tensor([4, 8]).upload(r(4, 8)), nnc.gpu_tensor([4, 8]).upload(r(4, 8)), nnc.gpu_tensor([4, 8]).upload(s(4, 8))
    c = nnc.gpu_tensor([4]).upload(s(4))
    gv = nnc.tensor_view_new(gbase, [4, 1], [0] * 12, [2, 1] + [0] * 10)
    sv = nnc.tensor_view_new(base, [4, 8], [0] * 12, [16, 2] + [0] * 10)
    q = nnc.gpu_palettized_tensor([4, 8], abi.CCV_32F, 4, 8)
    q.upload(np.zeros(q.nbytes, np.uint8))
    try:
        for cmd, ins, outs in ((bce_b, [gv, a, b], [h]), (mse_f, [sv, b], [c]), (mse_f, [a, q], [c]), (mse_b, [None, q, b], [h, None])):
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(cmd, None, 0, ins, outs) == INVALID and nnc.launch_count() == l0
            assert (h.download() == SENTINEL).all() and (c.download() == SENTINEL).all()
    finally:
        for t in (sv, gv, q, c, h, b, a, gbase, base):
            t.free()


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("name,op,param", FORMS)
def test_against_cpu_ref(gpu, ref, name, op, param):
    """where the compiled reference is present: fp32 gradients equal CPU_REF's, the loss is within the bound of CPU_REF's"""
    nnc = gpu
    a, b = operands(op, (10, 100), 61)
    g = seeded((10,), 63, 0.5, 2)
    fwd, bwd = commands(nnc, op, param)
    st_r, want = ref_exec(ref, fwd, None, 0, [a, b], _fwd_outs(op, 10, (10, 100)))
    st, got, _ = _run(nnc, fwd, [a, b], _fwd_outs(op, 10, (10, 100)), abi.CCV_32F)
    assert st_r == 0 and st == 0
    _, S = L.forward(op, a, b, param)
    assert (np.abs(got[0].astype(np.float64) - want[0]) <= 2 * L.bound(op, 100, S)).all()
    if op == L.BCE:
        ins = [g, a, b]
    elif op == L.SBCE:
        ins = [g, None, None, b, None, want[1]]
    elif op == L.MSE:
        ins = [g, a, b]
    else:
        ins = [g, a, b, want[0]]
    outs = lambda: [np.zeros((10, 100), np.float32)] + ([np.zeros((10, 100), np.float32)] if op == L.MSE else [])
    st_r, hw = ref_exec(ref, bwd, None, 0, ins, outs())
    st, hg, _ = _run(nnc, bwd, ins, outs(), abi.CCV_32F)
    assert st_r == 0 and st == 0
    for x, w in zip(hg, hw):
        assert np.array_equal(x, w)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("shape", [(10, 100), (65536, 4), (3, 2 ** 20 + 5)])
def test_sigmoid_bce_forward_without_c(gpu, kname, shape):
    """(a, b) -> (NULL, d): only d is written, in one launch and without a workspace, also on split rows; d has the bits of the call
    that writes c too"""
    nnc, kind = gpu, KINDS[kname]
    a, b = operands(L.SBCE, shape, 71, kind)
    batch = L.rows(a).shape[0]
    fwd, _ = commands(nnc, L.SBCE, 2.5)
    st, (none, d), launches = _run(nnc, fwd, [a, b], [None, np.zeros(shape, np.float32)], kind)
    assert st == 0 and none is None and launches == 1
    st, (_, d_c), _ = _run(nnc, fwd, [a, b], _fwd_outs(L.SBCE, batch, shape), kind)
    assert st == 0 and np.array_equal(d, d_c)


def _fwd_through_views(nnc, cmd, op, a, b, kind, ofs, pitch):
    """the forward on a and b (and d) held as [batch, count] slices starting at column `ofs` of [batch, pitch] tensors"""
    batch, count = a.shape
    up = lambda x: x if kind == abi.CCV_32F else pack16(x, kind)
    down = lambda t: t.download() if kind == abi.CCV_32F else unpack16(t.download(), kind)
    owned = []

    def view(x):
        w = np.zeros((batch, pitch), np.float32)
        if x is not None:
            w[:, ofs:ofs + count] = x
        t = nnc.gpu_tensor([batch, pitch], NHWC, kind).upload(up(w))
        v = nnc.tensor_view_new(t, [batch, count], [0, ofs] + [0] * 10, [pitch, 1] + [0] * 10)
        owned.extend([v, t])
        return t, v

    try:
        _, av = view(a)
        _, bv = view(b)
        c = nnc.gpu_tensor([batch], NHWC, kind)
        owned.append(c)
        outs = [c]
        if op == L.SBCE:
            dw, dv = view(None)
            outs.append(dv)
        assert nnc.cmd_exec(cmd, None, 0, [av, bv], outs) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        return [down(c)] + ([down(dw)[:, ofs:ofs + count]] if op == L.SBCE else [])
    finally:
        for t in owned:
            t.free()


@pytest.mark.gpu
@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("name,op,param", FORMS)
@pytest.mark.parametrize("count", [64, 4])
def test_forward_load_paths_give_the_same_bits(gpu, name, op, param, count, kname):
    """The forward reads a row as 16-byte vectors (aligned rows of whole vectors), as groups of 4 elements (rows of a multiple of 4 on
    8-byte boundaries: 16-bit boxes) or element by element (anything else).  The summation order is the same in every case, so an
    aligned packed call and calls on the same data at column offsets 4 and 1 of wider tensors give the same bits."""
    nnc, kind = gpu, KINDS[kname]
    a, b = operands(op, (33, count), 81, kind)
    fwd, _ = commands(nnc, op, param)
    st, want, _ = _run(nnc, fwd, [a, b], _fwd_outs(op, 33, (33, count)), kind)
    assert st == 0
    for ofs, pitch in ((4, count + 12), (1, count + 3)):
        got = _fwd_through_views(nnc, fwd, op, a, b, kind, ofs, pitch)
        for x, w in zip(got, want):
            assert np.array_equal(x, w), (name, kname, count, ofs)


# ---- the reference's own loss programs on the drop-in build -----------------------------------------------------------------------
@pytest.mark.gpu
def test_reference_loss_programs_pass_on_the_dropin_build(gpu, tmp_path):
    """int.loss and int.smooth_l1 (test/int/nnc/loss.tests.c, smooth_l1.tests.c) through integration/run_reference_tests.py: every BCE,
    sigmoid-BCE, MSE and smooth-L1 case passes and none is skipped (loss.tests.c holds each BCE and sigmoid-BCE case twice under one
    name; the runner counts names)."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = os.path.join(root, "integration", "_build")
    progs = ("int.loss", "int.smooth_l1")
    if not os.path.exists(os.path.join(build, "libccv_dropin.so")) or not all(os.path.exists(os.path.join(build, p + ".tests")) for p in progs):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    out = str(tmp_path / "report.json")
    p = subprocess.run([sys.executable, os.path.join(root, "integration", "run_reference_tests.py"), "--only", ",".join(progs), "--budget-s", "300",
                        "--case-timeout", "60", "--out", out], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=400)
    assert p.returncode == 0, p.stdout.decode()[-2000:]
    rep = json.load(open(out))["programs"]
    loss, sl1 = rep["int.loss.tests"], rep["int.smooth_l1.tests"]
    family = ("binary cross entropy", "mse")
    mine = lambda names: sorted(n for n in names if any(f in n for f in family))
    assert mine(loss["passed"]) and not mine(loss["skipped"]) and not mine(loss["failed"]) and not loss["crashed"], loss
    # 6 BCE, 8 sigmoid-BCE and 4 MSE case names
    assert len(mine(loss["passed"])) == 18, mine(loss["passed"])
    assert sum("sigmoid" in n for n in mine(loss["passed"])) == 8 and sum(n.startswith("mse") for n in loss["passed"]) == 4
    assert sl1["tally"]["PASS"] == 3 and not sl1["skipped"] and not sl1["failed"] and not sl1["crashed"], sl1


# ---- two small training chains through ccv_nnc_cmd_exec against CPU_REF ----------------------------------------------------------
class _Dev(object):
    """tensors on the GPU for a chain of commands on one stream; `kind` is the element type of the activations"""

    def __init__(self, nnc, kind):
        self.nnc, self.kind, self.owned, self.stream = nnc, kind, [], nnc.Stream(0)

    def new(self, shape, dt=None):
        t = self.nnc.gpu_tensor(list(shape), NHWC, self.kind if dt is None else dt)
        self.owned.append(t)
        return t

    def up(self, arr, dt=None):
        dt = self.kind if dt is None else dt
        t = self.new(arr.shape, dt)
        t.upload(arr if dt == abi.CCV_32F else pack16(arr, dt))
        return t

    def run(self, cmd, ins, outs):
        assert self.nnc.cmd_exec(cmd, None, 0, ins, outs, self.stream) == 0, (hex(cmd.cmd), self.nnc.lib().ccv_nnc_sm100_last_error())
        return outs

    def down(self, t):
        self.stream.wait()
        d = t.download()
        dt = t.params.datatype & 0xFF000
        return d if dt == abi.CCV_32F else unpack16(d, dt)

    def free(self):
        self.stream.wait()
        for t in reversed(self.owned):
            t.free()
        self.stream.free()


def _ref_run(ref, cmd, ins, outs):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def _rel(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max() / max(np.abs(want).max(), 1e-30))


# fp32: the GEMMs are fp32-grade (3xTF32) and the losses within a few ulps per element, so what remains is summation-order noise of
# sums over at most 128 terms, far below 1e-4 of the largest value; 1e-3 leaves room for one-pass TF32 products (2^-11 ~ 5e-4 each).
# bf16: every command output is rounded to bf16 once (relative 2^-9 ~ 2e-3): logits, d, h, then dx / dw of the GEMM backward (4 roundings
# on the longest path, ~8e-3 if they add up) and, for the regression chain, the bf16 copy of the weights each step; sums over 64 rows can
# cancel, which raises an error relative to the largest value by a small factor: 3e-2.
CHAIN_BOUND = {"fp32": 1e-3, "bf16": 3e-2}


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_multilabel_head_chain(gpu, ref, kname):
    """logits = x w^T (GEMM [64, 128] x [32, 128]^T), SIGMOID_BINARY_CROSSENTROPY with pos_weight 2 against fp32 0 / 1 labels -> (c, d),
    its backward -> h, GEMM backward -> (dx, dw); against the same commands on CPU_REF in fp32 on the same (rounded) inputs."""
    nnc, kind = gpu, KINDS[kname]
    N, D, K = 64, 128, 32
    r16 = (lambda v: v) if kind == abi.CCV_32F else (lambda v: round16(v, kind))
    x, w = r16(seeded((N, D), 91, -1, 1)), r16((seeded((K, D), 92, -1, 1) / np.sqrt(D) * 4).astype(np.float32))
    lab = (seeded((N, K), 93) > 0.7).astype(np.float32)
    gemm, gemm_b = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1)), nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
    fwd, bwd = nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_FORWARD(2.0), nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_BACKWARD(2.0)
    z = lambda *s: np.zeros(s, np.float32)
    (lg,) = _ref_run(ref, gemm, [x, w], [z(N, K)])
    c, d = _ref_run(ref, fwd, [lg, lab], [z(N), z(N, K)])
    (h,) = _ref_run(ref, bwd, [None, None, None, lab, None, d], [z(N, K)])
    dx, dw = _ref_run(ref, gemm_b, [h, x, w], [z(N, D), z(K, D)])
    want = dict(c=c, d=d, h=h, dx=dx, dw=dw)
    dev = _Dev(nnc, kind)
    try:
        xg, wg, lg_ = dev.up(x), dev.up(w), dev.up(lab, abi.CCV_32F)
        (lgg,) = dev.run(gemm, [xg, wg], [dev.new((N, K))])
        cg, dg = dev.run(fwd, [lgg, lg_], [dev.new((N,)), dev.new((N, K))])
        (hg,) = dev.run(bwd, [None, None, None, lg_, None, dg], [dev.new((N, K))])
        dxg, dwg = dev.run(gemm_b, [hg, xg, wg], [dev.new((N, D)), dev.new((K, D))])
        got = dict(c=dev.down(cg), d=dev.down(dg), h=dev.down(hg), dx=dev.down(dxg), dw=dev.down(dwg))
    finally:
        dev.free()
    errs = dict((k, _rel(got[k], want[k])) for k in want)
    print("multi-label head %s: max error / max|ref| %s" % (kname, ", ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    for k, e in errs.items():
        assert np.isfinite(got[k]).all() and e <= CHAIN_BOUND[kname], (kname, k, errs)


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_regression_step_chain(gpu, ref, kname):
    """Three SGD steps on a fixed batch: pred = x w^T (GEMM [64, 128] x [16, 128]^T), MSE mean against targets -> c, MSE backward -> dpred,
    GEMM backward -> dw, SGD (rate 0.02) on fp32 master weights (bf16: w is converted to bf16 for the GEMMs each step and dw is bf16).
    The loss (the mean of c) falls at every step, and the losses and the final update w3 - w0 are compared with the same steps on CPU_REF
    in fp32."""
    nnc, kind = gpu, KINDS[kname]
    N, D, K, steps = 64, 128, 16, 3
    r16 = (lambda v: v) if kind == abi.CCV_32F else (lambda v: round16(v, kind))
    x = r16(seeded((N, D), 101, -1, 1))
    w_true = seeded((K, D), 102, -1, 1) / np.sqrt(D)
    y = r16((x @ w_true.T + 0.05 * seeded((N, K), 103, -1, 1)).astype(np.float32))
    w0 = r16((0.1 * seeded((K, D), 104, -1, 1)).astype(np.float32))
    gemm, gemm_b = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1)), nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
    fwd, bwd = nnc.CMD_MSE_FORWARD(abi.CCV_NNC_MSE_REDUCE_MEAN), nnc.CMD_MSE_BACKWARD(abi.CCV_NNC_MSE_REDUCE_MEAN)
    sgd = nnc.CMD_SGD_FORWARD(0, 0.02, 1.0, 0.0, 0.0, 0.0)
    z = lambda *s: np.zeros(s, np.float32)
    w, m, ref_loss = w0.copy(), z(K, D), []
    for _ in range(steps):
        (pred,) = _ref_run(ref, gemm, [x, w], [z(N, K)])
        (c,) = _ref_run(ref, fwd, [pred, y], [z(N)])
        ref_loss.append(float(c.astype(np.float64).mean()))
        (dp,) = _ref_run(ref, bwd, [None, pred, y], [z(N, K)])
        _, dw = _ref_run(ref, gemm_b, [dp, x, w], [z(N, D), z(K, D)])
        _ref_run(ref, sgd, [dw, w, m], [w, m])
    dev = _Dev(nnc, kind)
    loss = []
    try:
        xg, yg = dev.up(x), dev.up(y)
        wg, mg = dev.up(w0, abi.CCV_32F), dev.up(z(K, D), abi.CCV_32F)
        wk = wg if kind == abi.CCV_32F else dev.new((K, D))
        pred, c, dp, dx, dw = dev.new((N, K)), dev.new((N,)), dev.new((N, K)), dev.new((N, D)), dev.new((K, D))
        for _ in range(steps):
            if kind != abi.CCV_32F:
                dev.run(nnc.CMD_DATATYPE_CONVERSION_FORWARD(), [wg], [wk])
            dev.run(gemm, [xg, wk], [pred])
            dev.run(fwd, [pred, yg], [c])
            loss.append(float(dev.down(c).astype(np.float64).mean()))
            dev.run(bwd, [None, pred, yg], [dp, None])
            dev.run(gemm_b, [dp, xg, wk], [dx, dw])
            dev.run(sgd, [dw, wg, mg], [wg, mg])
        w_gpu = dev.down(wg)
    finally:
        dev.free()
    upd = _rel(w_gpu - w0, w - w0)
    errs = [abs(a - b) / ref_loss[0] for a, b in zip(loss, ref_loss)]
    print("regression step %s: losses %s (CPU_REF %s); update error / max|ref update| %.2e" % (kname, loss, ref_loss, upd))
    assert all(b < a for a, b in zip(loss, loss[1:])) and all(b < a for a, b in zip(ref_loss, ref_loss[1:])), (loss, ref_loss)
    assert max(errs) <= CHAIN_BOUND[kname] and upd <= CHAIN_BOUND[kname], (kname, errs, upd)
