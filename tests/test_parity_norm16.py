"""bf16 / fp16 LAYER_NORM, RMSNORM and GROUP_NORM (forward / backward) on CCV_NNC_BACKEND_GPU_SM100, against the float64 oracles of
tests/norm_ref.py evaluated on the widened 16-bit operands.

Datatype rule: the activations (x and y; g, x and h) share one kind K (bf16 or fp16 here); each parameter tensor (scale, bias, dscale,
dbias) is fp32 or K; the two statistics (saved_mean, saved_inv_std) are together fp32 or K.  Anything else is refused before any launch.

Bounds.  The kernels widen every 16-bit operand exactly and compute in fp32 as the fp32 kernels do, so the fp32 bounds of norm_ref hold
for the unrounded result; each output is then rounded to its type once (nearest even).  So every output, stage 1 (statistics, dscale,
dbias) and stage 2 (y, dx) alike, is checked with norm_ref.within(..., kind of that output): rne16(y_hat - e) <= y <= rne16(y_hat + e).
Stage 2 is evaluated with the statistics as the GPU stored them (16-bit statistics widened): with 16-bit statistics the forward computes
y from the stored values, which is what the backward reads.  Every GPU case also checks the NaN guards around each output, that two runs
give the same bits, that the launch count is norm_ref's plan, and that one row alone gives the bits it has inside the batch.

The reported ratio of a 16-bit output is |y - y_hat| / ((e + half a 16-bit ulp of y_hat) / BOUND_C): at most BOUND_C whenever the
output is within its bound, and close to it as soon as one element sits near a rounding midpoint, since the rounding dominates.  The
ratios of the outputs stored in fp32 are the ones that measure the arithmetic."""
import ctypes as C

import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests import norm_ref as R
from tests.contract_ref import rne16, trunc16
from tests.test_parity_norm_paths import (DT, GN_GPU, SENTINEL, _refused, _rejects, gn_shapes, gnorm_cmd, lnorm_cmd, regime, rms_cmd, run,
                                          run_twice)
from tests.util import ref_exec, round16, seeded

F32, BF16, F16 = R.F32, R.BF16, R.F16
KINDS = [BF16, F16]
PARAM_STAT = [(F32, F32), (F32, "K"), ("K", F32), ("K", "K")]  # (parameter kind, statistics kind); "K" = the activations' kind
EPS = 1e-5


def _r(a, kind):
    """the values a tensor of this kind holds"""
    return None if a is None else (np.asarray(a, np.float32) if kind == F32 else round16(a, DT[kind]))


# ---- ratios -------------------------------------------------------------------------------------------------------------------------
RATIOS = {}


def half_ulp16(v, kind):
    """half the spacing of the 16-bit grid at |v|"""
    _, ex = np.frexp(np.abs(R.f64(v)))
    if kind == BF16:
        return np.ldexp(1.0, np.maximum(ex - 1, -126) - 8)
    return np.ldexp(1.0, np.maximum(ex - 1, -14) - 11)


def check(cmd, what, y, y_hat, e, kind):
    """y (stored as `kind`) within the bound of y_hat; records the ratio"""
    y = np.asarray(y, np.float64)
    y_hat = np.asarray(y_hat, np.float64).reshape(y.shape)
    e = np.broadcast_to(np.asarray(e, np.float64).reshape(y.shape) if np.size(e) == y.size else e, y.shape)
    assert np.isfinite(y).all(), (cmd, what, "non-finite")
    ok = R.within(y, y_hat, e, kind)
    r = R.ratio(y, y_hat, e if kind == F32 else e + half_ulp16(y_hat, kind))
    assert ok.all(), (cmd, what, kind, "ratio %.2f" % r, int((~ok).sum()))
    key = (cmd, what if kind == F32 else what + " " + kind)
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)


# ---- CPU: registration and the 16-bit bounds reject defects --------------------------------------------------------------------------
class _Registry(C.Structure):
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


@pytest.mark.parametrize("name", ["LAYER_NORM", "RMSNORM", "GROUP_NORM"])
@pytest.mark.parametrize("d", ["FORWARD", "BACKWARD"])
def test_norms_are_registered_for_16_bit(name, d):
    lib = _nnc.lib()
    r = _Registry()
    getattr(lib, "_register_command_CCV_NNC_%s_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % (name, d))(C.byref(r))
    assert r.exec and r.algorithms == 1
    assert r.tensor_datatypes == abi.CCV_32F | abi.CCV_16F | abi.CCV_16BF


def _row_data(rows, inner, kind, reg="unit"):
    x2 = _r(regime(reg, (rows, 1, inner), 1).reshape(rows, inner) + np.float32(0.25), kind)
    g2 = _r(0.5 * x2 + seeded(x2.shape, 2, -1, 1), kind)
    return x2, g2, _r(seeded((inner,), 3, 0.5, 1.5), kind), _r(seeded((inner,), 4, -1, 1), kind)


@pytest.mark.parametrize("kind", KINDS)
def test_y_from_the_unrounded_statistics_is_rejected(kind):
    x2, _, scale, bias = _row_data(64, 1000, kind)
    (mean, _), (inv_std, _) = R.row_stats(x2, EPS)
    m16, r16 = _r(mean, kind), _r(inv_std, kind)
    y_hat, e = R.row_apply(x2, scale, bias, m16, r16)
    y_bad = rne16(R.row_apply(x2, scale, bias, mean.astype(np.float32), inv_std.astype(np.float32))[0], kind)
    assert R.within(rne16(y_hat, kind), y_hat, e, kind).all()
    assert _rejects(y_bad, y_hat, e, kind)


@pytest.mark.parametrize("kind", KINDS)
def test_a_truncated_output_is_rejected(kind):
    x2, g2, scale, bias = _row_data(64, 1000, kind)
    (mean, _), (inv_std, _) = R.row_stats(x2, EPS)
    m16, r16 = _r(mean, kind), _r(inv_std, kind)
    y_hat, e = R.row_apply(x2, scale, bias, m16, r16)
    assert _rejects(trunc16(y_hat, kind), y_hat, e, kind)
    dx, e_dx = R.row_dx(g2, x2, scale, m16, r16)
    assert _rejects(trunc16(dx, kind), dx, e_dx, kind)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rows", [297, 1000, 5000])
def test_dscale_rounded_per_partial_row_is_rejected(kind, rows):
    x2, _, _, _ = _row_data(rows, 1000, kind)
    g2 = _r(seeded(x2.shape, 5, -1, 1), kind)  # sums that do not grow with the rows, so that the final rounding is fine enough to tell
    (mean, _), (inv_std, _) = R.row_stats(x2, EPS)
    m16, r16 = _r(mean, kind), _r(inv_std, kind)
    (ds, e_ds), (db, e_db) = R.row_dparam(g2, x2, m16, r16)
    assert R.within(rne16(ds, kind), ds, e_ds, kind).all() and R.within(rne16(db, kind), db, e_db, kind).all()
    gy = R.row_dparam_blocks(rows)
    blk = np.arange(rows) % gy
    parts = [R.row_dparam(g2[blk == b], x2[blk == b], m16[blk == b], r16[blk == b]) for b in range(gy)]
    ds_bad = rne16(sum(rne16(p[0][0], kind) for p in parts), kind)
    db_bad = rne16(sum(rne16(p[1][0], kind) for p in parts), kind)
    # Each rounded partial row adds up to half a 16-bit ulp of itself, and the output shows that only where the sum of those errors
    # reaches a fair part of the output's own half ulp.  bf16 shows it for both sums at every row count here.  fp16 has 3 more bits:
    # dbias of 297 rows (partials of one or two 16-bit values of g, nearly exact) and both sums of 5000 rows (17 rows per partial,
    # sums about 70 times wider than a partial) stay within the output's rounding, so no bound at this resolution can tell them.
    if kind == BF16 or rows == 1000:
        assert _rejects(ds_bad, ds, e_ds, kind) and _rejects(db_bad, db, e_db, kind)
    elif rows == 297:
        assert _rejects(ds_bad, ds, e_ds, kind)


@pytest.mark.parametrize("kind", KINDS)
def test_statistics_rounded_before_the_variance_pass_are_rejected(kind):
    x2 = _r(50 + 0.5 * seeded((64, 1000), 6, -1, 1), kind)  # a mean far from zero against a std of about 0.3
    (mean, _), (inv_std, e_inv) = R.row_stats(x2, EPS)
    m16 = R.f64(_r(mean, kind))
    inv_bad = rne16(1.0 / np.sqrt(((R.f64(x2) - m16[:, None]) ** 2).mean(axis=1) + EPS), kind)
    assert R.within(rne16(inv_std, kind), inv_std, e_inv, kind).all()
    assert _rejects(inv_bad, inv_std, e_inv, kind)


# ---- GPU: layer norm / rms norm -----------------------------------------------------------------------------------------------------
def _kinds(ins, outs, pairs):
    return {id(a): k for a, k in pairs if a is not None}


def _row16(nnc, rms, shape, axes, reg, K, pk, sk, affine=1, saved=True):
    inner = int(np.prod([shape[a] for a in axes]))
    rows = int(np.prod(shape)) // inner
    x2 = regime(reg, (rows, 1, inner), 41, K).reshape(rows, inner)
    if reg == "constant":
        x2[0, :] = 3.25
    x = x2.reshape(shape)
    rshape = tuple(1 if i in axes else d for i, d in enumerate(shape))
    pshape = tuple(d if i in axes else 1 for i, d in enumerate(shape))
    scale, bias = (_r(seeded(pshape, 42, 0.5, 1.5), pk), _r(seeded(pshape, 43, -1, 1), pk)) if affine else (None, None)
    name = "rms" if rms else "ln"
    z, zr, zp = (lambda: np.zeros(shape, np.float32)), (lambda: np.zeros(rshape, np.float32)), (lambda: np.zeros(pshape, np.float32))
    params = [(x, K), (scale, pk), (bias, pk)]
    if rms:
        fwd, bwd = rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, EPS, axes), rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, EPS, axes)
        fins = [x, scale]
        fkinds = lambda i, o: _kinds(i, o, params + [(o[0], K), (o[1], sk)])
        st, (y, sis), n = run_twice(nnc, fwd, fins, lambda: (None, [z(), zr()]), fkinds)
        sm = np.zeros(rshape, np.float32)
    else:
        fwd, bwd = lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, EPS, affine, axes), lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, EPS, affine, axes)
        fins = [x, scale, bias] if affine else [x]
        fkinds = lambda i, o: _kinds(i, o, params + [(o[0], K), (o[1], sk), (o[2], sk)])
        st, (y, sm, sis), n = run_twice(nnc, fwd, fins, lambda: (None, [z(), zr(), zr()]), fkinds)
    assert st == 0 and n == R.row_plan("forward"), nnc.lib().ccv_nnc_sm100_last_error()
    (mean, e_mean), (inv_std, e_inv) = R.row_stats(x2, EPS, rms)
    if not rms:
        check(name, "mean", sm.ravel(), mean, e_mean, sk)
    check(name, "inv_std", sis.ravel(), inv_std, e_inv, sk)
    if reg == "constant" and not rms:
        assert sis.ravel()[0] == _r(np.float32(1 / np.sqrt(np.float32(0) + np.float32(EPS))), sk)
    check(name, "y", y.reshape(rows, inner), *R.row_apply(x2, scale, None if rms else bias, sm.ravel(), sis.ravel()), kind=K)
    if not saved:
        # the saved outputs absent: the y of the call with fp32 statistics
        yo = z()
        st, (y2,), _ = run(nnc, fwd, fins, [yo], _kinds(None, None, params + [(yo, K)]))
        y32 = [z(), zr()] if rms else [z(), zr(), zr()]
        st3, got, _ = run(nnc, fwd, fins, y32, _kinds(None, None, params + [(y32[0], K)]))
        assert st == 0 and st3 == 0 and np.array_equal(y2.view(np.uint32), got[0].view(np.uint32))
    if rows > 1:
        one = (1,) * (len(shape) - len(axes)) + tuple(shape[a] for a in axes)
        ax1 = tuple(range(len(one) - len(axes), len(one)))
        c1 = rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, EPS, ax1) if rms else lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, EPS, affine, ax1)
        xr = np.ascontiguousarray(x2[rows - 1]).reshape(one)
        sc1, b1 = (None, None) if scale is None else (scale.reshape(one), bias.reshape(one))
        ins1 = [xr, sc1] if rms else ([xr, sc1, b1] if affine else [xr])
        o1 = [np.zeros(one, np.float32), np.zeros((1,) * len(one), np.float32)] + ([] if rms else [np.zeros((1,) * len(one), np.float32)])
        st, got, _ = run(nnc, c1, ins1, o1, _kinds(None, None, [(xr, K), (sc1, pk), (b1, pk), (o1[0], K)] + [(t, sk) for t in o1[1:]]))
        assert st == 0 and np.array_equal(got[0].ravel().view(np.uint32), y.reshape(rows, inner)[rows - 1].view(np.uint32))
    # backward: all outputs, h only, dscale only
    g2 = _r(0.5 * R.row_apply(x2, None, None, sm.ravel(), sis.ravel())[0] + seeded(x2.shape, 44, -1, 1), K)
    g = g2.reshape(shape)
    if rms:
        ins, all_outs = [g, None, x, scale, None, sis], lambda: (None, [z(), zp()])
    elif affine:
        ins, all_outs = [g, None, None, x, scale, None, None, sm, sis], lambda: (None, [z(), zp(), zp()])
    else:
        ins, all_outs = [g, None, None, x, None, sm, sis], lambda: (None, [z()])
    bparams = params + [(g, K), (sm, sk), (sis, sk)]
    bkinds = lambda i, o: _kinds(i, o, bparams + [(o[0], K)] + [(t, pk) for t in o[1:]])
    st, outs, n = run_twice(nnc, bwd, ins, all_outs, bkinds)
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert n == R.row_plan("backward", dx=True, dparam=bool(affine))
    check(name, "dx", outs[0].reshape(rows, inner), *R.row_dx(g2, x2, scale, sm.ravel(), sis.ravel(), rms), kind=K)
    if affine:
        (ds, e_ds), (db, e_db) = R.row_dparam(g2, x2, sm.ravel(), sis.ravel())
        check(name, "dscale", outs[1].ravel(), ds, e_ds, pk)
        if not rms:
            check(name, "dbias", outs[2].ravel(), db, e_db, pk)
        h_only = [z()] + [None] * (len(outs) - 1)
        st, o1, n1 = run(nnc, bwd, ins, h_only, bkinds(ins, h_only))
        assert st == 0 and n1 == 1 and np.array_equal(o1[0].view(np.uint32), outs[0].view(np.uint32))
        ds_only = [None, zp()] + [None] * (len(outs) - 2)
        st, o2, n2 = run(nnc, bwd, ins, ds_only, _kinds(None, None, bparams + [(ds_only[1], pk)]))
        assert st == 0 and n2 == 2 and np.array_equal(o2[1].view(np.uint32), outs[1].view(np.uint32))


def _ps(K, ps):
    return tuple(K if k == "K" else k for k in ps)


ROW16_INNER = [1, 7, 33, 64, 127, 512, 1000, 2047, 4096, 65536]  # every row_threads step; 1, 7, 33, 127, 2047 take scalar accesses


@pytest.mark.gpu
@pytest.mark.parametrize("ps", PARAM_STAT)
@pytest.mark.parametrize("K", KINDS)
@pytest.mark.parametrize("rms", [0, 1])
@pytest.mark.parametrize("inner", ROW16_INNER)
def test_row_norm16_paths(gpu, inner, rms, K, ps):
    _row16(gpu, rms, (3, inner), (1,), "unit", K, *_ps(K, ps))


@pytest.mark.gpu
@pytest.mark.parametrize("ps", PARAM_STAT)
@pytest.mark.parametrize("K", KINDS)
@pytest.mark.parametrize("rms", [0, 1])
@pytest.mark.parametrize("rows", [1, 295, 296, 297, 5000])
def test_row_norm16_rows(gpu, rows, rms, K, ps):
    """around the 296-row-block cap of the parameter gradients"""
    _row16(gpu, rms, (rows, 64), (1,), "unit", K, *_ps(K, ps))


@pytest.mark.gpu
@pytest.mark.parametrize("ps", [(F32, F32), ("K", "K")])
@pytest.mark.parametrize("K", KINDS)
@pytest.mark.parametrize("rms", [0, 1])
@pytest.mark.parametrize("reg", ["offset", "outlier", "constant", "relu"])
def test_row_norm16_regimes(gpu, reg, rms, K, ps):
    _row16(gpu, rms, (37, 1000), (1,), reg, K, *_ps(K, ps))


@pytest.mark.gpu
@pytest.mark.parametrize("ps", [(F32, "K"), ("K", F32)])
@pytest.mark.parametrize("K", KINDS)
@pytest.mark.parametrize("rms", [0, 1])
@pytest.mark.parametrize("shape,axes,affine,saved", [((4, 3, 5, 40), (1, 2, 3), 1, True), ((6, 1, 10, 1, 64), (2, 4), 1, True), ((6, 10, 64), (2,), 0, True),
                                                     ((5, 7, 96), (1, 2), 1, False), ((5, 7, 96), (1, 2), 0, False)])
def test_row_norm16_forms(gpu, shape, axes, affine, saved, rms, K, ps):
    """multi-axis trailing reductions, axes of extent 1 between reduced ones, affine off (layer norm), saved outputs absent"""
    if rms and not affine:
        pytest.skip("rms norm always has a scale")
    _row16(gpu, rms, shape, axes, "unit", K, *_ps(K, ps), affine=affine, saved=saved)


@pytest.mark.gpu
@pytest.mark.parametrize("K", KINDS)
def test_layer_norm16_mixed_parameter_kinds(gpu, K):
    """each parameter tensor picks its own kind: scale K with bias fp32 forward, dscale fp32 with dbias K backward"""
    nnc = gpu
    rows, inner = 9, 256
    x = _r(seeded((rows, inner), 81, -1, 1), K)
    scale, bias = _r(seeded((1, inner), 82, 0.5, 1.5), K), seeded((1, inner), 83, -1, 1)
    fwd, bwd = lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, EPS, 1, (1,)), lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, EPS, 1, (1,))
    outs = [np.zeros((rows, inner), np.float32), np.zeros((rows, 1), np.float32), np.zeros((rows, 1), np.float32)]
    st, (y, sm, sis), n = run(nnc, fwd, [x, scale, bias], outs, {id(x): K, id(scale): K, id(outs[0]): K})
    assert st == 0 and n == 1
    check("ln", "y", y, *R.row_apply(x, scale, bias, sm.ravel(), sis.ravel()), kind=K)
    g = _r(seeded((rows, inner), 84, -1, 1), K)
    bo = [np.zeros((rows, inner), np.float32), np.zeros((1, inner), np.float32), np.zeros((1, inner), np.float32)]
    st, (h, ds, db), n = run(nnc, bwd, [g, None, None, x, scale, None, None, sm, sis], bo, {id(x): K, id(g): K, id(scale): K, id(bo[0]): K, id(bo[2]): K})
    assert st == 0 and n == 3
    check("ln", "dx", h, *R.row_dx(g, x, scale, sm.ravel(), sis.ravel()), kind=K)
    (dsh, e_ds), (dbh, e_db) = R.row_dparam(g, x, sm.ravel(), sis.ravel())
    check("ln", "dscale", ds.ravel(), dsh, e_ds, F32)
    check("ln", "dbias", db.ravel(), dbh, e_db, K)


# ---- GPU: group norm ------------------------------------------------------------------------------------------------------------------
GN16 = GN_GPU + [("gn_unet_nhwc", (2, 32, 32, 320), 3, 32, (1, 2), 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("ps", PARAM_STAT)
@pytest.mark.parametrize("K", KINDS)
@pytest.mark.parametrize("name,shape,group_axis,groups,reduce_axes,affine", GN16)
def test_group_norm16_paths(gpu, name, shape, group_axis, groups, reduce_axes, affine, K, ps):
    nnc = gpu
    pk, sk = _ps(K, ps)
    x = _r(seeded(shape, 51, -1, 1), K)
    rshape, pshape = gn_shapes(shape, group_axis, groups, reduce_axes)
    scale, bias = (_r(seeded(pshape, 52, 0.5, 1.5), pk), _r(seeded(pshape, 53, -1, 1), pk)) if affine else (None, None)
    fwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, group_axis, groups, 1e-5, affine, reduce_axes)
    bwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_BACKWARD, group_axis, groups, 1e-5, affine, reduce_axes)
    eps = R.gn_epsilon(len(reduce_axes))
    z, zr, zp = (lambda: np.zeros(shape, np.float32)), (lambda: np.zeros(rshape, np.float32)), (lambda: np.zeros(pshape, np.float32))
    params = [(x, K), (scale, pk), (bias, pk)]
    fins = [x, scale, bias] if affine else [x]
    st, (y, sm, sis), n = run_twice(nnc, fwd, fins, lambda: (None, [z(), zr(), zr()]), lambda i, o: _kinds(i, o, params + [(o[0], K), (o[1], sk), (o[2], sk)]))
    assert st == 0 and n == R.gn_plan("forward"), nnc.lib().ccv_nnc_sm100_last_error()
    (mean, e_mean), (inv_std, e_inv) = R.gn_stats(x, rshape, eps)
    check("gn", "mean", sm, mean, e_mean, sk), check("gn", "inv_std", sis, inv_std, e_inv, sk)
    check("gn", "y", y, *R.gn_apply(x, scale, bias, sm, sis), kind=K)
    g = _r(0.5 * R.gn_apply(x, None, None, sm, sis)[0] + seeded(shape, 54, -1, 1), K)
    ins = [g, None, None, x, scale, None, None, sm, sis] if affine else [g, None, None, x, None, sm, sis]
    bparams = params + [(g, K), (sm, sk), (sis, sk)]
    st, outs, n = run_twice(nnc, bwd, ins, lambda: (None, [z(), zp(), zp()] if affine else [z()]),
                            lambda i, o: _kinds(i, o, bparams + [(o[0], K)] + [(t, pk) for t in o[1:]]))
    assert st == 0 and n == R.gn_plan("backward", dx=True, dparam=bool(affine))
    check("gn", "dx", outs[0], *R.gn_dx(g, x, scale, sm, sis), kind=K)
    if affine:
        (ds, e_ds), (db, e_db) = R.gn_dparam(g, x, sm, sis, pshape)
        check("gn", "dscale", outs[1], ds, e_ds, pk), check("gn", "dbias", outs[2], db, e_db, pk)


@pytest.mark.gpu
@pytest.mark.parametrize("K", KINDS)
def test_group_norm16_strided_views(gpu, K):
    """x, y, g and h as slices of wider NaN-filled 16-bit tensors (row pitch 9 for rows of 5): only the slices change, and they hold
    the bits of the packed call"""
    nnc = gpu
    dt = DT[K]
    shape, wide_shape = (2, 16, 6, 5), (2, 16, 6, 9)
    name, _, group_axis, groups, reduce_axes, affine = GN_GPU[0]
    rshape, pshape = gn_shapes(shape, group_axis, groups, reduce_axes)
    x, g = _r(seeded(shape, 61, -1, 1), K), _r(seeded(shape, 62, -1, 1), K)
    scale, bias = _r(seeded(pshape, 63, 0.5, 1.5), K), _r(seeded(pshape, 64, -1, 1), K)
    fwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, group_axis, groups, 1e-5, affine, reduce_axes)
    bwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_BACKWARD, group_axis, groups, 1e-5, affine, reduce_axes)
    zz = lambda s: np.zeros(s, np.float32)
    fo = [zz(shape), zz(rshape), zz(rshape)]
    st, (y, sm, sis), _ = run(nnc, fwd, [x, scale, bias], fo, {id(x): K, id(scale): K, id(bias): K, id(fo[0]): K, id(fo[1]): K, id(fo[2]): K})
    bo = [zz(shape), zz(pshape), zz(pshape)]
    st2, (h, ds, db), _ = run(nnc, bwd, [g, None, None, x, scale, None, None, sm, sis], bo,
                              {id(a): K for a in [g, x, scale, sm, sis] + bo})
    assert st == 0 and st2 == 0
    owned = []
    from tests.util import pack16, unpack16

    def wide(a):
        w = np.full(wide_shape, np.nan, np.float32)
        if a is not None:
            w[..., 2:7] = a
        t = nnc.gpu_tensor(list(wide_shape), abi.CCV_TENSOR_FORMAT_NHWC, dt).upload(pack16(w, dt))
        stride = [16 * 6 * 9, 6 * 9, 9, 1] + [0] * 8
        v = nnc.tensor_view_new(t, list(shape), [0, 0, 0, 2] + [0] * 8, stride)
        owned.extend([v, t])
        return t, v

    def dense(a):
        owned.append(nnc.gpu_tensor(list(a.shape), abi.CCV_TENSOR_FORMAT_NHWC, dt).upload(pack16(a, dt)))
        return owned[-1]
    try:
        (_, xv), (_, gv), (yw, yv), (hw, hv) = wide(x), wide(g), wide(None), wide(None)
        ts, tb, tm, ti, tds, tdb = dense(scale), dense(bias), dense(zz(rshape)), dense(zz(rshape)), dense(zz(pshape)), dense(zz(pshape))
        assert nnc.cmd_exec(fwd, None, 0, [xv, ts, tb], [yv, tm, ti]) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        assert nnc.cmd_exec(bwd, None, 0, [gv, None, None, xv, ts, None, None, tm, ti], [hv, tds, tdb]) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        for w, want in ((unpack16(yw.download(), dt), y), (unpack16(hw.download(), dt), h)):
            assert np.isnan(w[..., :2]).all() and np.isnan(w[..., 7:]).all() and np.array_equal(w[..., 2:7], want)
        for t, want in ((tm, sm), (tds, ds), (tdb, db)):
            assert np.array_equal(unpack16(t.download(), dt), want)
    finally:
        for t in owned:
            t.free()


# ---- refusals -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_norm16_refusals(gpu):
    nnc = gpu
    r = lambda *s: seeded(s, 3, 0.1, 0.9)
    s = lambda *shape: np.full(shape, SENTINEL, np.float32)
    lf, lb = lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, 1e-5, 1, (1,)), lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 1, (1,))
    rf, rb = rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, 1e-5, (1,)), rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, 1e-5, (1,))
    x, g, sc, b, m, i = r(6, 16), r(6, 16), r(1, 16), r(1, 16), r(6, 1), r(6, 1)
    # bf16 x with an fp16 y
    y = s(6, 16)
    _refused(nnc, lf, [x, sc, b], [y, s(6, 1), s(6, 1)], {id(x): BF16, id(y): F16})
    # a bf16 scale under fp16 activations
    y = s(6, 16)
    _refused(nnc, rf, [x, sc], [y, s(6, 1)], {id(x): F16, id(sc): BF16, id(y): F16})
    # fp16 statistics under bf16 activations (forward outputs and backward inputs)
    y, sm, si = s(6, 16), s(6, 1), s(6, 1)
    _refused(nnc, lf, [x, sc, b], [y, sm, si], {id(x): BF16, id(y): BF16, id(sm): F16, id(si): F16})
    h = s(6, 16)
    _refused(nnc, lb, [g, None, None, x, sc, None, None, m, i], [h, s(1, 16), s(1, 16)], {id(g): BF16, id(x): BF16, id(h): BF16, id(m): F16, id(i): F16})
    # the two statistics of different kinds
    y, sm, si = s(6, 16), s(6, 1), s(6, 1)
    _refused(nnc, lf, [x, sc, b], [y, sm, si], {id(x): BF16, id(y): BF16, id(sm): BF16})
    # a 16-bit h with fp32 g (and x)
    h = s(6, 16)
    _refused(nnc, rb, [g, None, x, sc, None, i], [h, s(1, 16)], {id(h): BF16})
    h = s(6, 16)
    _refused(nnc, lb, [g, None, None, x, sc, None, None, m, i], [h, s(1, 16), s(1, 16)], {id(x): F16, id(h): F16})
    # group norm: bf16 x with an fp16 y; fp16 statistics under bf16 activations
    xg = r(2, 10, 3, 3)
    gf = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, 1, 5, 1e-5, 1, (2, 3))
    y = s(2, 10, 3, 3)
    _refused(nnc, gf, [xg, r(1, 10, 1, 1), r(1, 10, 1, 1)], [y, s(2, 5, 1, 1), s(2, 5, 1, 1)], {id(xg): BF16, id(y): F16})
    y, sm, si = s(2, 10, 3, 3), s(2, 5, 1, 1), s(2, 5, 1, 1)
    _refused(nnc, gf, [xg, r(1, 10, 1, 1), r(1, 10, 1, 1)], [y, sm, si], {id(xg): BF16, id(y): BF16, id(sm): F16, id(si): F16})


# ---- against CPU_REF ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("K", KINDS)
def test_norm16_against_cpu_ref(gpu, ref, K):
    """All-K tensors (what a half-precision cnnp model hands these commands) against CPU_REF run in fp32 on the widened inputs.

    Forward: CPU_REF computes y from its own fp32 statistics, the GPU from the statistics rounded to K and then rounds y.  Each of
    the three roundings (inv_std, mean, y) is at most half a K ulp, u16 = 2^-8 (bf16) or 2^-11 (fp16) of the value: y is off by at most
    u16/2 (|xhat| + |mean| inv_std) + u16/2 |y| and |mean| inv_std, |xhat| <= max|y| for these data, so 1.5 u16 max|y| plus fp32 noise.
    The statistics and the backward outputs are one rounding each (the backward reads the same widened statistics on both sides).
    Bound: 2 u16 max|ref|."""
    nnc = gpu
    u16 = 2.0 ** -8 if K == BF16 else 2.0 ** -11
    kinds = lambda arrs: {id(a): K for a in arrs if a is not None}

    def same(got, want, what):
        for a, w in zip(got, want):
            if a is not None:
                assert np.abs(R.f64(a) - R.f64(w)).max() <= 2 * u16 * np.abs(R.f64(w)).max(), (what, K)
    # layer norm
    x, sc, b = _r(seeded((6, 10, 64), 71, -1, 1), K), _r(seeded((1, 1, 64), 72, 0.5, 1.5), K), _r(seeded((1, 1, 64), 73, -1, 1), K)
    fwd, bwd = lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, 1e-5, 1, (2,)), lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 1, (2,))
    mk = lambda: [np.zeros((6, 10, 64), np.float32), np.zeros((6, 10, 1), np.float32), np.zeros((6, 10, 1), np.float32)]
    st_r, want = ref_exec(ref, fwd, None, 0, [x, sc, b], mk())
    o = mk()
    st, got, _ = run(nnc, fwd, [x, sc, b], o, kinds([x, sc, b] + o))
    assert st_r == 0 and st == 0
    same(got, want, "ln forward")
    sm, si = got[1], got[2]
    g = _r(seeded((6, 10, 64), 74, -1, 1), K)
    mkb = lambda: [np.zeros((6, 10, 64), np.float32), np.zeros((1, 1, 64), np.float32), np.zeros((1, 1, 64), np.float32)]
    bins = [g, None, None, x, sc, None, None, sm, si]
    st_r, want = ref_exec(ref, bwd, None, 0, bins, mkb())
    o = mkb()
    st, got, _ = run(nnc, bwd, bins, o, kinds(bins + o))
    assert st_r == 0 and st == 0
    same(got, want, "ln backward")
    # rms norm
    fwd, bwd = rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, 1e-5, (2,)), rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, 1e-5, (2,))
    mk = lambda: [np.zeros((6, 10, 64), np.float32), np.zeros((6, 10, 1), np.float32)]
    st_r, want = ref_exec(ref, fwd, None, 0, [x, sc], mk())
    o = mk()
    st, got, _ = run(nnc, fwd, [x, sc], o, kinds([x, sc] + o))
    assert st_r == 0 and st == 0
    same(got, want, "rms forward")
    bins = [g, None, x, sc, None, got[1]]
    mkb = lambda: [np.zeros((6, 10, 64), np.float32), np.zeros((1, 1, 64), np.float32)]
    st_r, want = ref_exec(ref, bwd, None, 0, bins, mkb())
    o = mkb()
    st, got, _ = run(nnc, bwd, bins, o, kinds(bins + o))
    assert st_r == 0 and st == 0
    same(got, want, "rms backward")
    # group norm, NHWC, 4 groups over (H, W)
    shape, rshape, pshape = (2, 5, 6, 16), (2, 1, 1, 4), (1, 1, 1, 16)
    x, sc, b, g = _r(seeded(shape, 75, -1, 1), K), _r(seeded(pshape, 76, 0.5, 1.5), K), _r(seeded(pshape, 77, -1, 1), K), _r(seeded(shape, 78, -1, 1), K)
    fwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, 3, 4, 1e-5, 1, (1, 2))
    bwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_BACKWARD, 3, 4, 1e-5, 1, (1, 2))
    mk = lambda: [np.zeros(shape, np.float32), np.zeros(rshape, np.float32), np.zeros(rshape, np.float32)]
    st_r, want = ref_exec(ref, fwd, None, 0, [x, sc, b], mk())
    o = mk()
    st, got, _ = run(nnc, fwd, [x, sc, b], o, kinds([x, sc, b] + o))
    assert st_r == 0 and st == 0
    same(got, want, "gn forward")
    bins = [g, None, None, x, sc, None, None, got[1], got[2]]
    mkb = lambda: [np.zeros(shape, np.float32), np.zeros(pshape, np.float32), np.zeros(pshape, np.float32)]
    st_r, want = ref_exec(ref, bwd, None, 0, bins, mkb())
    o = mkb()
    st, got, _ = run(nnc, bwd, bins, o, kinds(bins + o))
    assert st_r == 0 and st == 0
    same(got, want, "gn backward")


@pytest.mark.gpu
def test_zz_report_measured_ratios16(gpu):
    """prints the largest ratio per command and output (16-bit outputs: the ratio defined in the module docstring)"""
    per_cmd = {}
    for (cmd, what), r in sorted(RATIOS.items()):
        print("ratio16 %-4s %-20s %.3f" % (cmd, what, r))
        per_cmd[cmd] = max(per_cmd.get(cmd, 0.0), r)
    print("largest ratio per command:", ", ".join("%s %.3f" % kv for kv in sorted(per_cmd.items())))
    assert all(r <= R.BOUND_C for r in per_cmd.values())
