"""Float64 oracles, error bounds and the restated launch plan of the feeder commands of a training step: MAX_POOL and AVERAGE_POOL
(forward / backward), SOFTMAX (forward / backward), CATEGORICAL_CROSSENTROPY and SOFTMAX_CROSSENTROPY (forward / backward) and
SGD_FORWARD (one command, and the multi-tensor node the graph fuser builds from a run of them), for tests/test_parity_feeder_paths.py.
NumPy only.

Every oracle works on the operands as the kernel sees them (fp32 values, or the 16-bit values widened), in float64.

Reference quirks restated (paths relative to lib/nnc of the reference):
  * pool windows are clipped to the input, and the average divides by the CLIPPED window size in both directions
    (ccv_nnc_internal.h:209-213 SET_BORDER_OFFSET_SIZE_FOR; cmd/pool/ccv_nnc_avg_pool_cpu_ref.c:53 and :96); the output extent P comes
    from the output tensor, so an end border larger than the begin border clips the last window (pool_window);
  * max-pool backward gives the window's gradient to EVERY input equal to the window maximum (cmd/pool/ccv_nnc_max_pool_cpu_ref.c:128);
  * an fp32 class index is rounded as (int)(label + 0.5) (cmd/loss/ccv_nnc_categorical_crossentropy_cpu_ref.c:41,
    cmd/softmax_loss/ccv_nnc_softmax_crossentropy_cpu_ref.c:53); an fp32 label tensor holds indices when its "range" is 1 and a
    distribution otherwise, range = the last dimension of a tensor of more than one axis, else dim[0] when the batch is 1, else 1
    (ccv_nnc_categorical_crossentropy_cpu_ref.c:31, ccv_nnc_softmax_crossentropy_cpu_ref.c:36);
  * label smoothing: the target is trim1 at the label and trim0 elsewhere (ccv_nnc_categorical_crossentropy_cpu_ref.c:54-57);
    a distribution label is used as given, trims ignored;
  * the softmax-CE "loss" is sum_j t_j (max - a_j), without the log-sum-exp (ccv_nnc_softmax_crossentropy_cpu_ref.c:76-79, :102-103);
  * a missing g reads as ones (CCV_NNC_CMD_ATTR_NULL_IS_ONES, cmd/softmax_loss/ccv_nnc_softmax_crossentropy.c:77;
    ccv_nnc_categorical_crossentropy_cpu_ref.c:205-237);
  * SGD: nesterov requires dampening = 0 (cmd/sgd/ccv_nnc_sgd_cpu_ref.c:52-53); with nesterov n = momentum m + scale g + decay a and
    b = a - rate (scale g + momentum n) (:82-84); without, n = momentum m + (1 - dampening)(scale g + decay a), b = a - rate n (:113-114).

Bounds.  u = 2^-24 and BOUND_C = 8 as in norm_ref; a sum of K terms whose magnitudes add up to S, accumulated in fp32 in any order, is
within sum_bound(K, S) = BOUND_C u sqrt(K) S.  One term per error source:
  * max-pool forward: exact (a maximum of the inputs, np.array_equal);
  * max-pool backward: the sum of the <= K gradients of the windows whose maximum the input equals: BOUND_C u S, S = sum |g|;
  * average pool: a sum of K = |window| terms, then one division: BOUND_C u (S / m) with S = sum |x| (forward) and
    BOUND_C u sum |g_p / m_p| for the backward, which divides each window's gradient before it adds them;
  * softmax, y = exp(a - m) / s: the fp32 rounding of a - m is amplified by exp into a relative u |a - m|; expf is within 2 ulp; the
    sum s of K positive terms is within sum_bound(K, s); the reciprocal and the product are 2 more roundings.  Relative:
    u |a - m| + 2 u + BOUND_C u sqrt(K) + 2 u, taken as BOUND_C u (|a - m| + sqrt(K) + 4), plus 2^-140 absolute for the
    subnormal range of exp;
  * softmax backward, h = (g - sum g y) y: sum_bound(K, sum |g y|) |y| and BOUND_C u (|g| + |sum g y|) |y| for the two roundings,
    plus 2^-126 |g - sum g y| where y (from exp far below the maximum) is subnormal and the product is only absolutely accurate;
  * cross-entropy forward, c = -sum t log a: sum_bound(K, S) + BOUND_C u S, S = sum |t log a| (logf's ulps and the product);
    softmax-CE forward, c = sum t (m - a): sum_bound(K, S) + BOUND_C u S, S = sum |t (m - a)|;
  * the pointwise backward forms (-g t / a, g (d - t)) allow two roundings each: BOUND_C u (the magnitudes of their terms);
  * SGD: a few roundings per element, bounded by the magnitudes of the terms: BOUND_C u (|momentum m| + |scale g| + |decay a|) for n and
    BOUND_C u (|a| + |rate step|) plus rate (momentum) e_n for b.  nvcc may contract the products into FMAs, so nothing here requires
    bit equality with CPU_REF; the fused node must give the bits of the unfused commands.
16-bit outputs: rne16(y_hat - e) <= y <= rne16(y_hat + e) (contract_ref.rne16)."""
import numpy as np

from tests.contract_ref import rne16  # noqa: F401
from tests.norm_ref import BF16, BOUND_C, F16, F32, U, f64, ratio, sum_bound, within  # noqa: F401

SUBNORMAL = 2.0 ** -140
TINY = 2.0 ** -126  # a product whose result is below the normal range keeps only its absolute accuracy


# ---- pools on NHWC [N, H, W, C] -----------------------------------------------------------------------------------------------
def out_extent(H, R, stride, pad_begin, pad_end):
    return (H + pad_begin + pad_end - R) // stride + 1


def pool_window(p, R, stride, pad, H):
    """[lo, hi) of output row p's window, clipped to the input (SET_BORDER_OFFSET_SIZE_FOR)"""
    return max(p * stride - pad, 0), min(p * stride - pad + R, H)


def _windows(H, W, P, Q, geo):
    R, S, sh, sw, ph, pw = geo
    for p in range(P):
        h0, h1 = pool_window(p, R, sh, ph, H)
        for q in range(Q):
            w0, w1 = pool_window(q, S, sw, pw, W)
            yield p, q, h0, h1, w0, w1


def max_pool(a, P, Q, geo):
    a = f64(a)
    N, H, W, C = a.shape
    b = np.full((N, P, Q, C), -np.finfo(np.float32).max)
    for p, q, h0, h1, w0, w1 in _windows(H, W, P, Q, geo):
        if h1 > h0 and w1 > w0:
            b[:, p, q] = a[:, h0:h1, w0:w1].max(axis=(1, 2))
    return b


def max_pool_bwd(g, a, b, geo):
    """h and its bound; b is the forward's (exact) output, every input equal to its window's maximum receives g"""
    g, a, b = f64(g), f64(a), f64(b)
    N, H, W, C = a.shape
    P, Q = g.shape[1:3]
    h, mag = np.zeros_like(a), np.zeros_like(a)
    for p, q, h0, h1, w0, w1 in _windows(H, W, P, Q, geo):
        hit = a[:, h0:h1, w0:w1] == b[:, p:p + 1, q:q + 1]
        gv = g[:, p:p + 1, q:q + 1]
        h[:, h0:h1, w0:w1] += np.where(hit, gv, 0.0)
        mag[:, h0:h1, w0:w1] += np.where(hit, np.abs(gv), 0.0)
    return h, BOUND_C * U * mag


def avg_pool(a, P, Q, geo):
    a = f64(a)
    N, H, W, C = a.shape
    b, e = np.zeros((N, P, Q, C)), np.zeros((N, P, Q, C))
    for p, q, h0, h1, w0, w1 in _windows(H, W, P, Q, geo):
        m = (h1 - h0) * (w1 - w0)
        b[:, p, q] = a[:, h0:h1, w0:w1].sum(axis=(1, 2)) / m
        e[:, p, q] = BOUND_C * U * np.abs(a[:, h0:h1, w0:w1]).sum(axis=(1, 2)) / m
    return b, e


def avg_pool_bwd(g, H, W, geo, full_window=False):
    """h and its bound; full_window: every window divided by R S (a defect the bound must reject)"""
    g = f64(g)
    N, P, Q, C = g.shape
    h, mag = np.zeros((N, H, W, C)), np.zeros((N, H, W, C))
    for p, q, h0, h1, w0, w1 in _windows(H, W, P, Q, geo):
        m = geo[0] * geo[1] if full_window else (h1 - h0) * (w1 - w0)
        h[:, h0:h1, w0:w1] += g[:, p:p + 1, q:q + 1] / m
        mag[:, h0:h1, w0:w1] += np.abs(g[:, p:p + 1, q:q + 1]) / m
    return h, BOUND_C * U * mag


# ---- softmax / cross-entropy on rows [batch, count] (a row is everything after dim[0]) -------------------------------------------
def rows(shape):
    """(batch, count) of a tensor: dim[0] rows of everything after it; a 1-d tensor is one row"""
    return (1, int(shape[0])) if len(shape) == 1 else (int(shape[0]), int(np.prod(shape[1:])))


def softmax(a2):
    a2 = f64(a2)
    m = a2.max(axis=1, keepdims=True)
    e = np.exp(a2 - m)
    s = e.sum(axis=1, keepdims=True)
    y = e / s
    K = a2.shape[1]
    return y, y * BOUND_C * U * (np.abs(a2 - m) + np.sqrt(K) + 4) + SUBNORMAL


def softmax_bwd(g2, y2):
    g2, y2 = f64(g2), f64(y2)
    K = y2.shape[1]
    s = (g2 * y2).sum(axis=1, keepdims=True)
    h = (g2 - s) * y2
    es = sum_bound(K, np.abs(g2 * y2).sum(axis=1, keepdims=True))
    return h, (es + BOUND_C * U * (np.abs(g2) + np.abs(s))) * np.abs(y2) + np.abs(g2 - s) * TINY


def label_range(label_shape, batch):
    """the reference's "range" of an fp32 label tensor: 1 means class indices"""
    return label_shape[-1] if len(label_shape) > 1 else (label_shape[0] if batch == 1 else 1)


def targets(label, batch, count, trim0=0.0, trim1=1.0, int_label=False, truncate=False):
    """[batch, count] float64 targets t of a label tensor (int32 indices, fp32 indices, fp32 distribution) under the trims.
    truncate: fp32 indices cut instead of rounded (a defect the tests must reject)"""
    label = np.asarray(label)
    if not int_label and label_range(label.shape, batch) != 1:
        return f64(label).reshape(batch, count)
    if int_label:
        idx = label.reshape(-1).astype(np.int64)
    else:
        x = label.reshape(-1).astype(np.float32)
        idx = x.astype(np.int64) if truncate else (x + np.float32(0.5)).astype(np.int64)
    t = np.full((batch, count), float(np.float32(trim0)))
    t[np.arange(batch), idx] = float(np.float32(trim1))
    return t


def cce(a2, t):
    """c = -sum t log a; the (0, 1) fast path is the same value"""
    a2 = f64(a2)
    terms = np.where(t != 0, -t * np.log(np.where(t != 0, a2, 1.0)), 0.0)
    S = np.abs(terms).sum(axis=1)
    return terms.sum(axis=1), sum_bound(a2.shape[1], S) + BOUND_C * U * S


def cce_bwd(g, a2, t):
    """h = -g t / a (g None: ones)"""
    a2 = f64(a2)
    gp = np.ones((a2.shape[0], 1)) if g is None else f64(g).reshape(-1, 1)
    h = -gp * t / a2
    return h, BOUND_C * U * np.abs(h)


def softmax_cce(a2, t):
    """(c, its bound), (d, its bound): c = sum t (max - a)"""
    a2 = f64(a2)
    m = a2.max(axis=1, keepdims=True)
    terms = np.where(t != 0, t * (m - a2), 0.0)
    S = np.abs(terms).sum(axis=1)
    return (terms.sum(axis=1), sum_bound(a2.shape[1], S) + BOUND_C * U * S), softmax(a2)


def softmax_cce_bwd(g, d2, t):
    d2 = f64(d2)
    gp = np.ones((d2.shape[0], 1)) if g is None else f64(g).reshape(-1, 1)
    return gp * (d2 - t), BOUND_C * U * (np.abs(gp * d2) + np.abs(gp * t))


# ---- SGD --------------------------------------------------------------------------------------------------------------------------
def sgd(g, a, m, nesterov, rate, scale, decay, momentum, dampening):
    """((b, e_b), (n, e_n))"""
    g, a, m = f64(g), f64(a), f64(m)
    f = lambda v: float(np.float32(v))
    rate, scale, decay, momentum, dampening = f(rate), f(scale), f(decay), f(momentum), f(dampening)
    if nesterov:
        n = momentum * m + scale * g + decay * a
        e_n = BOUND_C * U * (np.abs(momentum * m) + np.abs(scale * g) + np.abs(decay * a))
        step = scale * g + momentum * n
        e_b = BOUND_C * U * (np.abs(a) + np.abs(rate * step) + np.abs(rate * scale * g)) + rate * momentum * e_n
    else:
        inv = f(1.0 - dampening)
        n = momentum * m + inv * (scale * g + decay * a)
        e_n = BOUND_C * U * (np.abs(momentum * m) + np.abs(inv * scale * g) + np.abs(inv * decay * a))
        step = n
        e_b = BOUND_C * U * (np.abs(a) + np.abs(rate * step)) + rate * e_n
    return (a - rate * step, e_b), (n, e_n)


# ---- the launch plan, restated from sm100_ew.cu (pool_fwd_t, pool_max_bwd_t, pool_avg_bwd_t, sgd_any, sgd_multi_any) and
# sm100_backend.cu (staged: STAGE_NCHW / STAGE_F32) ----------------------------------------------------------------------------------
def vec_width(kind):
    return 4 if kind == F32 else 8


def pool_vec_ok(C, kind, pitches, aligned=True):
    """pool_vec_ok: C and every pixel / row / image pitch a whole number of 16-byte vectors, both base pointers aligned"""
    w = vec_width(kind)
    return aligned and C % w == 0 and all(p % w == 0 for p in pitches)


def pool_fwd_path(C, kind, pitches, aligned=True):
    return "vector" if pool_vec_ok(C, kind, pitches, aligned) else "scalar"


def pool_max_bwd_path(C, kind, pitches, aligned=True):
    return "vector" if pool_vec_ok(C, kind, pitches, aligned) else "scalar"


def pool_avg_bwd_path(H, W, P, Q, geo, C, kind, pitches, aligned=True):
    """'tiles' (avgpool_bwd_tiles_kernel: windows tile the input exactly); 'shortcut' (the vector gather's non-overlapping branch:
    window = stride, no begin border, no window clipped, P R <= H); 'gather' (vector); 'scalar' (the scalar gather)"""
    R, S, sh, sw, ph, pw = geo
    vec = pool_vec_ok(C, kind, pitches, aligned)
    tiling = R == sh and S == sw and ph == 0 and pw == 0
    if tiling and H == P * R and W == Q * S and vec:
        return "tiles"
    if not vec:
        return "scalar"
    return "shortcut" if tiling and P * sh <= H and Q * sw <= W else "gather"


def pool_launches(direction, is_max, nchw=False):
    """one kernel; an NCHW call adds one layout copy per staged operand: in (a; g, a, b for the max backward; g for the average
    backward) and out (b or h)"""
    if not nchw:
        return 1
    staged_in = 1 if direction == "forward" else (3 if is_max else 1)
    return staged_in + 1 + 1


def staged_f32_launches(n16, n16_out, inner=1):
    """the functional form of a 16-bit call (STAGE_F32): every distinct 16-bit tensor widened (outputs too: the command may read them),
    the fp32 command, every 16-bit output narrowed"""
    return n16 + inner + n16_out


def softmax_threads(count):
    return 256 if count >= 1024 else 128 if count >= 256 else 64 if count >= 64 else 32


def sgd_path(count, aligned=True):
    return "vec4" if count % 4 == 0 and aligned else "scalar"


SGD_MULTI_MAX, SGD_MULTI_CHUNK = 32, 4096


def sgd_multi_plan(tensors):
    """tensors: [(count, vec_ok)] in node order -> [launch], each launch a list of tensor indices; a tensor that cannot take the vector
    kernel flushes the batch and runs alone, count-0 tensors take no block"""
    launches, cur, i = [], [], 0
    while i < len(tensors):
        count, vec = tensors[i]
        if not vec:
            if cur:
                launches.append(cur)
                cur = []
            launches.append([i])
        elif count > 0:
            cur.append(i)
            if len(cur) == SGD_MULTI_MAX:
                launches.append(cur)
                cur = []
        i += 1
    if cur:
        launches.append(cur)
    return launches
