"""Float64 oracles, error bounds and the restated launch plan of the element-wise, broadcast and reduction commands: SIGMOID, TANH,
LEAKY_RELU, EWEXP, EWLOG, EWSQRT, CLAMP, EWDIV, GELU (erf and tanh forms), SWISH, REDUCE_SUM / MEAN / MAX / MIN / NORM2, MASKED_FILL,
EWSUM, ADD, MUL and SCALAR_MUL (forward / backward), for tests/test_parity_ew_paths.py.  NumPy only.

Every oracle evaluates the formula the kernel and CPU_REF evaluate, in float64, on the operands as the kernel sees them (fp32 values,
or the 16-bit values widened).  Each returns (y_hat, e): the value and a per-element bound; selections return e = 0 and must match
bit for bit.

Reference quirks restated (paths relative to lib/nnc/cmd of the reference):
  * a missing gradient reads as ones (CCV_NNC_CMD_ATTR_NULL_IS_ONES; ew/ccv_nnc_ew_cpu_ref.c:1043-1044 for EWEXP,
    reduce/ccv_nnc_reduce_max_cpu_ref.c:71-124, blas/ccv_nnc_add_cpu_ref.c, blas/ccv_nnc_mul_cpu_ref.c);
  * SIGMOID / TANH backward dereference g before testing it (sigmoid/ccv_nnc_sigmoid_cpu_ref.c:36-44, tanh/ccv_nnc_tanh_cpu_ref.c:36),
    so their backward without g has no CPU_REF oracle; the kernels read it as ones, and so does the oracle here.  GELU / SWISH backward
    need g in CPU_REF (gelu/ccv_nnc_gelu_cpu_ref.c:46, swish/ccv_nnc_swish_cpu_ref.c) and the kernels refuse a call without it;
  * REDUCE_MEAN forward scales by count(b) / count(a) (reduce/ccv_nnc_reduce_mean_cpu_ref.c:36); its backward scales by
    count(g) / count(h) with g (:100) and by 1 / (the product of h's extents along the command's axes) without g (:76-79);
  * REDUCE_MAX / MIN start from -FLT_MAX / FLT_MAX (reduce/ccv_nnc_reduce_max_cpu_ref.c:36, ..._min_cpu_ref.c:36) and keep an element
    only when it compares greater (smaller): an all -inf or all NaN slice gives -FLT_MAX (FLT_MAX for MIN, over +inf / NaN); NaN
    elements never win.  In bf16 / fp16 -FLT_MAX rounds to -inf, so that is what those kinds store;
  * REDUCE_MAX / MIN backward send g to EVERY element equal to the stored result (ties included: ..._max_cpu_ref.c:114,175);
  * LEAKY_RELU and CLAMP backward test the saved output b, not a (leaky_relu/ccv_nnc_leaky_relu_cpu_ref.c:40-60,
    ew/ccv_nnc_ew_cpu_ref.c:1424-1500);
  * MASKED_FILL with an int32 mask compares it against (int)(p + 0.5) (util/ccv_nnc_util_cpu_ref.c:1467);
  * EWSUM adds left to right, c = ((a0 + a1) + a2) + ...; when c is the storage of an operand z >= 1 that operand comes first
    (ew/ccv_nnc_ew_cpu_ref.c:29-45);
  * GELU's backward `pdf` is exp(-x^2 / 2) sqrt(2 / pi), twice the normal density (gelu/ccv_nnc_gelu_cpu_ref.c:83-88).

Bounds.  u = 2^-24, BOUND_C = 8 (norm_ref).  Per element BOUND_C u (the magnitudes of the terms the formula adds); a transcendental
adds its ulps (expf / tanhf / erff / logf are within 2 ulp) and its conditioning at its fp32-rounded argument, |f'(t)| u |t|, where t
is itself a rounded product.  Where CPU_REF's formula cancels (1 - y of the SIGMOID / TANH backward, 1 + erf(t) of GELU at large
negative x) the bound follows the terms of that formula, not the exact function.  Results below the normal range keep only their
absolute accuracy: TINY = 2^-126 of slack.  Reductions: sum_bound(K, S) for SUM / MEAN, plus one rounding for the MEAN scale and for
the NORM2 root.  16-bit outputs: rne16(y_hat - e) <= y <= rne16(y_hat + e) (norm_ref.within)."""
import math

import numpy as np

from tests.contract_ref import rne16, trunc16  # noqa: F401
from tests.norm_ref import BF16, BOUND_C, F16, F32, U, f64, ratio, sum_bound, within  # noqa: F401

TINY = 2.0 ** -126
FLT_MAX = float(np.finfo(np.float32).max)
SQRT_2_PI = 0.797884560802865355
GELU_K = 0.044715
_erf = np.frompyfunc(math.erf, 1, 1)


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def erf(x):
    return np.asarray(_erf(f64(x)), np.float64)


def store(y, kind):
    """the value a store of the float64 y (already an fp32 value where the kernel formed it in fp32) leaves in a tensor of `kind`"""
    return f32(y) if kind == F32 else rne16(f32(y), kind)


def _q(g, like):
    return np.ones_like(f64(like)) if g is None else f64(g)


# ---- unary family (ew_op in sm100_ew_more.cu, act_fwd / act_bwd in sm100_ext_ops.cu) ------------------------------------------------
def sigmoid(x):
    x = f64(x)
    with np.errstate(over="ignore"):
        y = 1.0 / (1.0 + np.exp(-x))
    return y, BOUND_C * U * 2 * np.abs(y) + TINY


def tanh(x):
    y = np.tanh(f64(x))
    return y, BOUND_C * U * np.abs(y) + TINY


def exp(x):
    with np.errstate(over="ignore"):
        y = np.exp(f64(x))
    return y, BOUND_C * U * np.abs(y) + TINY


def log(x):
    with np.errstate(divide="ignore", invalid="ignore"):
        y = np.log(f64(x))
    return y, BOUND_C * U * np.abs(y) + TINY


def sqrt(x):
    with np.errstate(invalid="ignore"):
        y = np.sqrt(f64(x))
    return y, BOUND_C * U * np.abs(y)


def leaky_relu(x, slope):
    """a selection: x, or the fp32 product x * slope"""
    x = f64(x)
    return np.where(x > 0, x, f32(x * float(np.float32(slope)))), 0.0


def clamp(x, lo, hi):
    """a selection; a NaN bound is an open side"""
    y = f64(x)
    if not math.isnan(hi):
        y = np.minimum(y, float(np.float32(hi)))
    if not math.isnan(lo):
        y = np.maximum(y, float(np.float32(lo)))
    return y, 0.0


def sigmoid_bwd(g, b):
    """h = g b (1 - b), from the saved output b"""
    gq, b = _q(g, b), f64(b)
    return gq * b * (1 - b), BOUND_C * U * np.abs(gq * b) * (1 + np.abs(b)) + TINY


def tanh_bwd(g, b):
    """h = g (1 - b^2)"""
    gq, b = _q(g, b), f64(b)
    return gq * (1 - b * b), BOUND_C * U * np.abs(gq) * (1 + b * b) + TINY


def leaky_relu_bwd(g, b, slope):
    gq, b = _q(g, b), f64(b)
    return np.where(b >= 0, gq, f32(gq * float(np.float32(slope)))), 0.0


def exp_bwd(g, b):
    gq, b = _q(g, b), f64(b)
    h = gq * b
    return h, BOUND_C * U * np.abs(h) + TINY


def log_bwd(g, a):
    """h = g / a, from the forward input a"""
    gq, a = _q(g, a), f64(a)
    with np.errstate(divide="ignore", invalid="ignore"):
        h = gq / a
    return h, BOUND_C * U * np.abs(h) + TINY


def sqrt_bwd(g, b, half=0.5):
    """h = 0.5 g / b; half: the factor (a defect the bounds must reject leaves it out)"""
    gq, b = _q(g, b), f64(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        h = half * gq / b
    return h, BOUND_C * U * np.abs(h) + TINY


def clamp_bwd(g, b, lo, hi):
    gq, b = _q(g, b), f64(b)
    cut = np.zeros(b.shape, bool)
    if not math.isnan(hi):
        cut |= b >= float(np.float32(hi))
    if not math.isnan(lo):
        cut |= b <= float(np.float32(lo))
    return np.where(cut, 0.0, gq), 0.0


def ewdiv(a, b):
    """c = a / b (a None: 1 / b)"""
    b = f64(b)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = _q(a, b) / b
    return c, BOUND_C * U * np.abs(c) + TINY


def ewdiv_bwd(g, b, c, which, sign=-1.0, use_c=True):
    """ha = g / b; hb = -g c / b.  sign / use_c: defects the bounds must reject"""
    gq, b, c = _q(g, b), f64(b), f64(c)
    if which == "a":
        h = gq / b
    else:
        h = sign * gq * (c if use_c else 1.0) / b
    return h, BOUND_C * U * np.abs(h) + TINY


def gelu(x, tanh_form=False):
    x = f64(x)
    if tanh_form:
        inner = SQRT_2_PI * (x + GELU_K * x ** 3)
        t = np.tanh(inner)
        y = 0.5 * x * (1 + t)
        dinner = (1 - t * t) * SQRT_2_PI * (np.abs(x) + GELU_K * np.abs(x) ** 3)
        return y, BOUND_C * U * (np.abs(y) + 0.5 * np.abs(x) * (1 + np.abs(t) + dinner)) + TINY
    t = x * 0.70710678118654752440
    ef = erf(t)
    y = 0.5 * x * (1 + ef)
    cond = 2 / math.sqrt(math.pi) * np.exp(-t * t) * np.abs(t)
    return y, BOUND_C * U * (np.abs(y) + 0.5 * np.abs(x) * (1 + np.abs(ef) + cond)) + TINY


def gelu_bwd(g, x, tanh_form=False):
    gq, x = _q(g, x), f64(x)
    ag = np.abs(gq)
    if tanh_form:
        x2 = x * x
        inner = SQRT_2_PI * (x + GELU_K * x2 * x)
        t = np.tanh(inner)
        dd = SQRT_2_PI * (1 + 3 * GELU_K * x2)
        h = gq * (0.5 * (1 + t) + 0.5 * x * (1 - t * t) * dd)
        dt = (1 - t * t) * SQRT_2_PI * (np.abs(x) + GELU_K * np.abs(x) ** 3) + np.abs(t)
        e = ag * (0.5 * (1 + np.abs(t)) + 0.5 * np.abs(x) * (1 + t * t) * dd) + ag * (0.5 + np.abs(x * t) * dd) * dt
        return h, BOUND_C * U * e + TINY
    t = x * 0.70710678118654752440
    ef = erf(t)
    cdf = 0.5 * (1 + ef)
    pdf = np.exp(-0.5 * x * x) * SQRT_2_PI
    h = gq * (cdf + x * pdf)
    cond = 2 / math.sqrt(math.pi) * np.exp(-t * t) * np.abs(t)
    e = ag * (np.abs(cdf) + np.abs(x * pdf) * (2 + 0.5 * x * x)) + 0.5 * ag * (1 + np.abs(ef) + cond)
    return h, BOUND_C * U * e + TINY


def swish(x):
    x = f64(x)
    with np.errstate(over="ignore"):
        y = x / (1 + np.exp(-x))
    return y, BOUND_C * U * 2 * np.abs(y) + TINY


def swish_bwd(g, x):
    gq, x = _q(g, x), f64(x)
    with np.errstate(over="ignore"):
        y = 1 / (1 + np.exp(-x))
    h = gq * (x * (y - y * y) + y)
    e = np.abs(gq) * (np.abs(x) * (y + y * y) + y + (np.abs(x) * (1 + 2 * y) + 1) * y)
    return h, BOUND_C * U * e + TINY


# name -> (forward(x, *args), backward(g, a, b, *args), the saved operand the backward reads: "a" or "b")
UNARY = {
    "SIGMOID": (sigmoid, lambda g, a, b: sigmoid_bwd(g, b), "b"),
    "TANH": (tanh, lambda g, a, b: tanh_bwd(g, b), "b"),
    "EWEXP": (exp, lambda g, a, b: exp_bwd(g, b), "b"),
    "EWLOG": (log, lambda g, a, b: log_bwd(g, a), "a"),
    "EWSQRT": (sqrt, lambda g, a, b: sqrt_bwd(g, b), "b"),
    "LEAKY_RELU": (leaky_relu, lambda g, a, b, s: leaky_relu_bwd(g, b, s), "b"),
    "CLAMP": (clamp, lambda g, a, b, lo, hi: clamp_bwd(g, b, lo, hi), "b"),
}
SELECTIONS = ("LEAKY_RELU", "CLAMP")


# ---- reductions over a right-aligned 4-d view ------------------------------------------------------------------------------------
def reduced_axes(ashape, bshape):
    """the axes of a that b reduces (b's unit extents where a's are not)"""
    return tuple(i for i in range(len(ashape)) if bshape[i] == 1 and ashape[i] != 1)


def reduce_fwd(mode, a, bshape, identity=None):
    """(b, e) with b of bshape.  identity: the MAX / MIN starting value (the reference's -FLT_MAX / FLT_MAX; -inf / inf is the old
    kernel, a defect the fixture must reject)"""
    a = f64(a)
    ax = reduced_axes(a.shape, bshape)
    K = int(np.prod([a.shape[i] for i in ax], dtype=np.int64))
    if mode in ("MAX", "MIN"):
        init = (-FLT_MAX if mode == "MAX" else FLT_MAX) if identity is None else identity
        f = np.fmax if mode == "MAX" else np.fmin
        return f.reduce(a, axis=ax, keepdims=True, initial=init).reshape(bshape), 0.0
    if mode == "NORM2":
        s = (a * a).sum(axis=ax, keepdims=True).reshape(bshape)
        y = np.sqrt(s)
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(y > 0, 0.5 * sum_bound(K, s) / np.where(y > 0, y, 1), 0.0)
        return y, e + BOUND_C * U * y + TINY
    s = a.sum(axis=ax, keepdims=True).reshape(bshape)
    S = np.abs(a).sum(axis=ax, keepdims=True).reshape(bshape)
    if mode == "SUM":
        return s, sum_bound(K, S)
    return s / K, sum_bound(K, S) / K + BOUND_C * U * np.abs(s / K)


def mean_bwd_scale(hshape, gshape, axes):
    """count(g) / count(h) with g; 1 / prod(h's extents along the command's axes) without (gshape None)"""
    if gshape is not None:
        return float(np.prod(gshape, dtype=np.int64)) / float(np.prod(hshape, dtype=np.int64))
    return 1.0 / float(np.prod([hshape[i] for i in axes if 0 <= i < len(hshape)], dtype=np.int64))


def reduce_bwd(mode, g, a, b, hshape, axes=()):
    """(h, e); g / b broadcast onto h (g None: ones)"""
    gq = np.broadcast_to(np.ones(1) if g is None else f64(g), hshape)
    if mode == "SUM":
        return np.array(gq), 0.0
    if mode == "MEAN":
        h = gq * mean_bwd_scale(hshape, None if g is None else np.shape(g), axes)
        return h, BOUND_C * U * np.abs(h)
    a, bb = f64(a), np.broadcast_to(f64(b), hshape)
    if mode == "NORM2":
        h = gq * a / bb
        return h, BOUND_C * U * np.abs(h) + TINY
    return np.where(a == bb, gq, 0.0), 0.0


# ---- MASKED_FILL ------------------------------------------------------------------------------------------------------------------
def masked_fill(a, mask, p, q, cshape):
    """c = mask == p ? q : a (a, mask broadcast onto c); an int32 mask compares against (int)(p + 0.5)"""
    mask = np.broadcast_to(mask, cshape)
    pv = int(np.float32(p) + np.float32(0.5)) if mask.dtype == np.int32 else float(np.float32(p))
    return np.where(mask == pv, float(np.float32(q)), np.broadcast_to(f64(a), cshape)), 0.0


# ---- EWSUM ------------------------------------------------------------------------------------------------------------------------
def ewsum_order(k, alias=None):
    """the order the operands are added in: an output aliasing operand z >= 1 starts from it"""
    if not alias:
        return list(range(k))
    return [alias] + [i for i in range(k) if i != alias]


def ewsum(xs, alias=None, chunk_overwrites=False):
    """(the fp32 sum in CPU_REF's order, as float64, its bound).  chunk_overwrites: every chunk of 8 after the first writes its own sum
    instead of adding onto the output (a defect the bounds must reject)"""
    order = ewsum_order(len(xs), alias)
    acc = np.asarray(xs[order[0]], np.float32).copy()
    for j, i in enumerate(order[1:], 1):
        if chunk_overwrites and j % 8 == 0:
            acc = np.asarray(xs[i], np.float32).copy()
        else:
            acc = (acc + np.asarray(xs[i], np.float32)).astype(np.float32)
    S = sum(np.abs(f64(x)) for x in xs)
    return f64(acc), sum_bound(len(xs), S)


# ---- ADD / MUL / SCALAR_MUL (fp32 kernels; 16-bit through the functional form) -------------------------------------------------------
def add(a, b, p, q, cshape):
    p, q = float(np.float32(p)), float(np.float32(q))
    ta = p * np.broadcast_to(f64(a), cshape)
    tb = 0.0 if b is None else q * np.broadcast_to(f64(b), cshape)
    return ta + tb, BOUND_C * U * (np.abs(ta) + np.abs(tb))


def mul(a, b, p, cshape):
    c = float(np.float32(p)) * np.broadcast_to(f64(a), cshape) * np.broadcast_to(f64(b), cshape)
    return c, BOUND_C * U * np.abs(c)


def sum_to(t, shape):
    """t summed over the axes along which `shape` is 1 (and t is not): (sum, S = sum |t|, K terms)"""
    ax = tuple(i for i in range(t.ndim) if shape[i] == 1 and t.shape[i] != 1)
    K = int(np.prod([t.shape[i] for i in ax], dtype=np.int64))
    return t.sum(axis=ax, keepdims=True).reshape(shape), np.abs(t).sum(axis=ax, keepdims=True).reshape(shape), K


def add_bwd(g, p, oshape, fshape, summed=True):
    """gradient of the operand of shape oshape in c = p a + q b over the full shape fshape: p g summed over the broadcast axes (g None:
    p everywhere, as the kernels and CPU_REF fill it).  summed=False: not summed (a defect)"""
    p = float(np.float32(p))
    if g is None:
        return np.full(oshape, p), 0.0
    t = p * np.broadcast_to(f64(g), fshape)
    if not summed:
        return t[tuple(slice(0, s) for s in oshape)], BOUND_C * U * np.abs(t[tuple(slice(0, s) for s in oshape)])
    s, S, K = sum_to(t, oshape)
    return s, sum_bound(K, S) + BOUND_C * U * np.abs(s)


def mul_bwd(g, other, p, oshape, fshape):
    """d(p a b)/da = p g b summed onto a's shape (other = b), likewise for b (other = a); g None: ones"""
    gq = np.ones(fshape) if g is None else np.broadcast_to(f64(g), fshape)
    t = float(np.float32(p)) * gq * np.broadcast_to(f64(other), fshape)
    s, S, K = sum_to(t, oshape)
    return s, sum_bound(K, S) + BOUND_C * U * np.abs(s)


# ---- the launch plan, restated from sm100_ew_more.cu (run_ew_t, run_reduce_t, exec_reduce_*, masked_fill), sm100_ext_ops.cu
# (run_act), sm100_ew.cu (ew_sum_f32, ew_sum_16, ew_axpby_f32, reduce_sum_bcast_f32) and sm100_backend.cu (exec_ewsum_*, exec_add_*,
# exec_mul_*, reduce_to, mul_back_plan, staged STAGE_F32) ---------------------------------------------------------------------------------
def vec_width(kind):
    return 4 if kind == F32 else 8


def ew_path(kind, aligned=True):
    """run_ew_t / run_act / relu16_t / ew_sum_16: the 16-byte vector body plus a scalar tail when every base is 16-byte aligned
    (aligned_v16), else the all-scalar form"""
    return "vector" if aligned else "scalar"


def unary_launches():
    return 1


def ewdiv_back_launches(ha, hb):
    return int(bool(ha)) + int(bool(hb))


REDUCE_WARP_MAX = 64


def reduce_path(rcount):
    """run_reduce_t: one warp per output while the reduced count is <= 64, one block per output above"""
    return "warp" if rcount <= REDUCE_WARP_MAX else "block"


def ewsum_launches(k, kind=F32):
    """fp32: one launch per chunk of 8 operands (k >= 2); k = 1 is a cudaMemcpyAsync (nothing when in place); bf16 / fp16: 1 launch
    (k <= 8); int32: 1 launch"""
    if k == 1:
        return 0
    if kind == "int32" or kind != F32:
        return 1
    return (k + 7) // 8


def ewsum_back_launches(outputs, has_g):
    """without g one fill per output; with g a cudaMemcpyAsync per output that is not g itself (no kernel)"""
    return outputs if not has_g else 0


def mul_back_launches(fused):
    """per requested output: 1 on the fused path (same shapes), 2 on the broadcast path (the product into the workspace, then
    reduce_sum_bcast_f32)"""
    return 1 if fused else 2


def staged_f32_launches(n16, n16_out, inner=1):
    """the functional form of a 16-bit call (STAGE_F32): every distinct 16-bit tensor widened (outputs too), the fp32 command, every
    16-bit output narrowed"""
    return n16 + inner + n16_out
