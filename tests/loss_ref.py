"""Oracles for the loss commands (BINARY_CROSSENTROPY, SIGMOID_BINARY_CROSSENTROPY, MSE, SMOOTH_L1) over [batch, count] rows, on the
operands as CPU_REF sees them (lib/nnc/cmd/loss/*_cpu_ref.c, lib/nnc/cmd/sigmoid_loss/*_cpu_ref.c):

  forward   float64 sums of the per-element terms, with what CPU_REF rounds to fp32 before its double arithmetic rounded the same way
            (1 - a, b - 1, pos_weight - 1, the mean scale (float)(1 / count), 0.5 / beta and 0.5 beta).  Each returns (y, S): y the loss
            per row and S the sum of the magnitudes of everything added into it, scaled like y, which the error bound is stated in.
  backward  CPU_REF's fp32 operations in CPU_REF's order (numpy float32 rounds each one; there is no FMA), and the clamped division in
            double, so the result is CPU_REF's bit for bit.

`plan` restates the forward launch plan of ccv_b200/csrc/sm100_loss.cu (loss_plan)."""
import numpy as np

F32, F64 = np.float32, np.float64
BCE, SBCE, MSE, SL1 = "bce", "sbce", "mse", "sl1"
MEAN, SUM = 0, 1
U = 2.0 ** -24  # unit roundoff of fp32
# the per-term error of a term's fp32 evaluation, in units of U times the term's magnitude: the accurate logf / log1pf are within 1
# ulp and expf within 2 ulps (CUDA C++ Programming Guide, "Mathematical Functions", single precision), plus the roundings of the
# products and sums around them
TERM_ULPS = {BCE: 6.0, SBCE: 8.0, MSE: 4.0, SL1: 4.0}


def rows(x):
    """a 1-d array is one row"""
    x = np.asarray(x)
    return x.reshape(1, -1) if x.ndim == 1 else x


def bce_forward(a, b, pos_weight=1.0):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    t1 = (b - F32(1)).astype(F64) * np.log((F32(1) - a).astype(F64))
    t2 = b.astype(F64) * np.log(a.astype(F64))
    pw = float(F32(pos_weight))
    if pw == 1:
        return (t1 - t2).sum(1), (np.abs(t1) + np.abs(t2)).sum(1)
    return t1.sum(1) - pw * t2.sum(1), np.abs(t1).sum(1) + pw * np.abs(t2).sum(1)


def softplus_neg(a):
    """log(1 + e^-a) in float64 without overflow"""
    return np.logaddexp(0.0, -np.asarray(a, F64))


def sbce_forward(a, b, pos_weight=1.0):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    pwm1 = F32(F32(pos_weight) - F32(1))
    u = (F32(1) - b).astype(F64) * a.astype(F64)
    v = (F32(1) + b * pwm1).astype(F64) * softplus_neg(a)
    return (u + v).sum(1), (np.abs(u) + np.abs(v)).sum(1)


def sigmoid(a):
    a = np.asarray(a, F64)
    e = np.exp(-np.abs(a))
    return np.where(a >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def mse_scale(count, reduce_op, backward=False):
    """CPU_REF's (float)(1.0 / (float)count) (forward) / (float)(2.0 / (float)count) (backward) for the mean, 1 / 2 for the sum"""
    if reduce_op == MEAN:
        return float(F32((2.0 if backward else 1.0) / float(F32(count))))
    return 2.0 if backward else 1.0


def mse_forward(a, b, reduce_op=MEAN):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    t = (b.astype(F64) - a.astype(F64)) ** 2
    s = mse_scale(a.shape[1], reduce_op)
    return t.sum(1) * s, t.sum(1) * s


def sl1_consts(beta):
    beta = float(F32(beta))
    return beta, float(F32(0.5 * beta)), float(F32(0.5 / beta)), float(F32(1.0 / beta))


def sl1_forward(a, b, beta=1.0, huber=False):
    """the row switch of CPU_REF; huber=True is the per-element Huber loss instead (a defect the bound must reject)"""
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    beta, beta_2, beta_inv_2, _ = sl1_consts(beta)
    t = b.astype(F64) - a.astype(F64)
    if huber:
        e = np.where(np.abs(t) < beta, t * t * beta_inv_2, np.abs(t) - beta_2)
        return e.sum(1), np.abs(e).sum(1)
    s, q = np.abs(t).sum(1), (t * t).sum(1)
    quad = s < beta
    return np.where(quad, q * beta_inv_2, s - beta_2), np.where(quad, q * beta_inv_2, s + beta_2)


def sl1_margin(a, b, beta=1.0):
    """|sum |b - a| - beta| per row: how far each row is from switching branch"""
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    return np.abs(np.abs(b.astype(F64) - a.astype(F64)).sum(1) - float(F32(beta)))


def forward(op, a, b, param):
    return {BCE: bce_forward, SBCE: sbce_forward, MSE: mse_forward, SL1: sl1_forward}[op](a, b, param)


def bound(op, count, S):
    """|y - y_hat| <= C (U sqrt(K) S + eps_f S) for a row of K = count terms whose magnitudes add up to S; C = BOUND_C.  sqrt(K) U S is the
    size a rounding error of a sum of K terms reaches when the roundings are independent (the fixed tree and unit order of the kernel
    do not line them up); eps_f S is the error of the terms themselves; the finish (mean scale, pos_weight product, smooth-L1 branch)
    adds a few roundings of at most U S each, which C covers."""
    return BOUND_C * (U * np.sqrt(count) + TERM_ULPS[op] * U) * np.asarray(S, F64)


# the largest max |y - y_hat| / (bound / C) measured on an H100 80GB HBM3 over the fp32 cases of tests/test_parity_loss.py was 0.64
# (MSE on [65536, 4]); C = 2 keeps a margin of about 3
BOUND_C = 2.0


# ---- backward: CPU_REF's fp32 arithmetic ------------------------------------------------------------------------------------
def _g(g, batch):
    return None if g is None else np.asarray(g, F32).reshape(batch, 1)


def bce_backward(g, a, b, pos_weight=1.0):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    g = _g(g, a.shape[0])
    pw = F32(pos_weight)
    with np.errstate(all="ignore"):
        num = a - b if pw == 1 else (a * b * (pw - F32(1)) + a) - pw * b
        if g is not None:
            num = g * num
        den = (F32(1) - a) * a
        h = np.where(den.astype(F64) > 1e-12, num / den, (num.astype(F64) / 1e-12).astype(F32))
    return h.astype(F32)


def sbce_backward(g, b, d, pos_weight=1.0):
    d, b = rows(np.asarray(d, F32)), rows(np.asarray(b, F32))
    g = _g(g, d.shape[0])
    pw = F32(pos_weight)
    v = d - b if pw == 1 else (d - F32(1)) * b * pw + d * (F32(1) - b)
    return v if g is None else g * v


def mse_backward(g, a, b, reduce_op=MEAN):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    g = _g(g, a.shape[0])
    s = F32(mse_scale(a.shape[1], reduce_op, True))
    gs = s if g is None else s * g
    return gs * (a - b), gs * (b - a)


def sl1_backward(g, a, b, c, beta=1.0):
    a, b = rows(np.asarray(a, F32)), rows(np.asarray(b, F32))
    g = _g(g, a.shape[0])
    _, beta_2, _, inv_beta = sl1_consts(beta)
    c = np.asarray(c, F32).reshape(-1, 1)
    t = a - b
    quad = c < F32(beta_2)
    gq = F32(inv_beta) if g is None else F32(inv_beta) * g
    gl = F32(1) if g is None else g
    return np.where(quad, gq * t, np.where(t > 0, gl, -gl)).astype(F32)


# ---- the forward plan of sm100_loss.cu --------------------------------------------------------------------------------------
THREADS, CHUNK_UNITS = 256, 2048


def plan(op, pos_weight, batch, count, elem_size, with_c=True):
    """(units per row, threads per row segment, chunks per row, workspace bytes, launches)"""
    v = 16 // elem_size
    units = -(-count // v)
    np_ = 2 if (op == BCE and F32(pos_weight) != 1) or op == SL1 else 1
    if units <= 32:
        group = 1
        while group < units:
            group *= 2
    else:
        group = 32 if units <= 256 else THREADS
    chunk = min(units, CHUNK_UNITS)
    chunks = -(-units // chunk)
    split = with_c and chunks > 1
    return units, group, chunks, batch * chunks * np_ * 4 if split else 0, 2 if split else 1
