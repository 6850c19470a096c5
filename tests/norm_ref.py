"""Float64 oracles, error bounds and the restated launch plan of the normalisation commands (BATCH_NORM, LAYER_NORM, RMSNORM,
GROUP_NORM, forward and backward) for tests/test_parity_norm_paths.py.  NumPy only.

Every oracle works on the operands as the kernel sees them (fp32 values, or the 16-bit values widened), in float64.

Reference quirks restated (paths relative to lib/nnc/cmd/norm of the reference):
  * statistics are biased (divide by n) everywhere: ccv_nnc_batch_norm_cpu_ref.c:66-110, ccv_nnc_layer_norm_cpu_ref.c:57-105;
  * batch norm, training: running_var = momentum * running_var + (1 - momentum) * (biased batch variance)
    (ccv_nnc_batch_norm_cpu_ref.c:107, before :118 turns the variance into inv_std = 1 / sqrt(var + eps));
  * batch norm, inference: y = (x - mean) * scale / (sqrt(var) + eps) + bias, the epsilon OUTSIDE the root
    (ccv_nnc_batch_norm_cpu_ref.c:277);
  * layer / rms / group norm: inv_std = 1 / sqrt(var + eps) (ccv_nnc_layer_norm_cpu_ref.c:105, ccv_nnc_rmsnorm_cpu_ref.c:90,
    ccv_nnc_group_norm_cpu_ref.c:139); rms norm has no mean;
  * group norm reads its epsilon through the LAYER-norm arm of the parameter union (ccv_nnc_group_norm_cpu_ref.c:46), which aliases
    gnorm.reduce_count: the epsilon in effect is that small integer's bits read as a float (gn_epsilon).

Bounds come in two stages, so that the conditioning of the data enters once and visibly.

Stage 1, statistics and parameter gradients (saved mean, saved inv_std, running mean / var, dscale, dbias), against the float64
two-pass value: a sum of K terms whose magnitudes add up to S, accumulated in fp32 in any order, is within
    sum_bound(K, S) = BOUND_C * u * sqrt(K) * S,   u = 2^-24
of the exact sum (each term may itself carry a few roundings: they are inside BOUND_C).  On top of that
  - the mean and the variance are rounded to fp32 once: u |mean|, u var;
  - a variance computed about a mean that is off by e_mean gains e_mean^2;
  - inv_std = 1 / sqrtf(var + eps): relative 1/2 e_var / (var + eps) from the variance, and 4 u for sqrtf, the division and the sum;
  - the running statistics add one multiply-add: BOUND_C u (|momentum * old| + |(1 - momentum) * new|).
Batch norm shifts every term by a value of the same channel before it sums, so its terms are x - mean (S = sum |x - mean|); layer,
rms and group norm sum x itself in their first pass (S = sum |x|) and (x - mean)^2 in their second.

Stage 2, element outputs (y, dx), against the float64 formula evaluated WITH THE GPU'S OWN stored statistics (and, for batch norm's
dx, its own dscale / dbias): per element BOUND_C * u * (the magnitudes of the terms actually added).  Batch norm evaluates
y = x * a + b with b = bias - mean * a and dx = a * g + p * x + q, so |x * a| + |mean * a| + |bias| is in the bound and an error that
grows as |mean| / std is accepted exactly as far as those terms explain it.  The row norms compute their two backward means inside
the kernel, so their dx bound carries sum_bound of those two sums.

16-bit outputs: rne16(y_hat - e) <= y <= rne16(y_hat + e) (contract_ref.rne16).

BOUND_C = 8, as contract_ref.C_ACC."""
import numpy as np

from tests.contract_ref import rne16

U = 2.0 ** -24
BOUND_C = 8.0
SMS = 132            # multiprocessors of an H100 SXM: the reduce grid's cap depends on it
F32, BF16, F16 = "fp32", "bf16", "fp16"


def f64(a):
    return np.asarray(a, np.float64)


def sum_bound(K, S):
    return BOUND_C * U * np.sqrt(max(K, 1)) * f64(S)


def within(y, y_hat, e, kind=F32):
    """y (stored by the kernel) against y_hat +- e, element-wise; 16-bit: the interval's ends rounded like the output"""
    y, y_hat, e = f64(y), f64(y_hat), f64(e)
    if kind == F32:
        return np.abs(y - y_hat) <= e
    return (rne16(y_hat - e, kind) <= y) & (y <= rne16(y_hat + e, kind))


def ratio(y, y_hat, e):
    """largest |y - y_hat| / (e / BOUND_C): the constant the data asked for (0 where both are exact)"""
    d, e = np.abs(f64(y) - f64(y_hat)), f64(e) / BOUND_C
    return float(np.max(np.where(d == 0, 0.0, d / np.maximum(e, 1e-300)), initial=0.0))


# ---- batch norm on x as [outer, C, inner] -------------------------------------------------------------------------------------
def bn_view(x, axis):
    """x -> [outer, C, inner] with C = x.shape[axis] (axis None: the whole tensor is one channel)"""
    x = np.asarray(x)
    if axis is None:
        return x.reshape(1, 1, -1)
    return x.reshape(int(np.prod(x.shape[:axis], dtype=np.int64)), x.shape[axis], -1)


def bn_stats(x3):
    x3 = f64(x3)
    mean = x3.mean(axis=(0, 2))
    var = ((x3 - mean[None, :, None]) ** 2).mean(axis=(0, 2))
    return mean, var


def bn_stat_bounds(x3, eps, momentum, running_mean, running_var):
    """(mean, var, inv_std, running_mean, running_var) oracle values and their stage-1 bounds"""
    x3 = f64(x3)
    K = x3.shape[0] * x3.shape[2]
    mean, var = bn_stats(x3)
    d = x3 - mean[None, :, None]
    e_mean = sum_bound(K, np.abs(d).sum(axis=(0, 2))) / K + U * np.abs(mean)
    e_var = sum_bound(K, (d * d).sum(axis=(0, 2))) / K + e_mean ** 2 + U * var
    inv_std = 1.0 / np.sqrt(var + eps)
    e_inv = inv_std * (0.5 * e_var / (var + eps) + 4 * U)
    rm, rv = f64(running_mean).ravel(), f64(running_var).ravel()
    new_rm, new_rv = momentum * rm + (1.0 - momentum) * mean, momentum * rv + (1.0 - momentum) * var
    e_rm = (1.0 - momentum) * e_mean + BOUND_C * U * (np.abs(momentum * rm) + np.abs((1.0 - momentum) * mean))
    e_rv = (1.0 - momentum) * e_var + BOUND_C * U * (np.abs(momentum * rv) + np.abs((1.0 - momentum) * var))
    return dict(mean=(mean, e_mean), var=(var, e_var), inv_std=(inv_std, e_inv), running_mean=(new_rm, e_rm), running_var=(new_rv, e_rv))


def bn_apply(x3, scale, bias, mean, inv_std, relu=False):
    """y and its stage-2 bound from the given (stored) statistics"""
    x3 = f64(x3)
    bc = lambda v: f64(v).ravel()[None, :, None]
    a = bc(scale) * bc(inv_std)
    y = x3 * a + (bc(bias) - bc(mean) * a)
    e = BOUND_C * U * (np.abs(x3 * a) + np.abs(bc(mean) * a) + np.abs(bc(bias)))
    return (np.maximum(y, 0) if relu else y), e


def bn_test_coef(scale, var, eps):
    """inference: a = scale / (sqrt(var) + eps); returned as the inv_std that makes bn_apply compute it"""
    return 1.0 / (np.sqrt(f64(var).ravel()) + eps)


def bn_mask(x3, scale, bias, mean, inv_std):
    """relu(bn(x)) > 0, decided as the kernels decide it: fp32 a = scale * inv_std, b = bias - mean * a, fmaf(x, a, b) > 0"""
    f = lambda v: np.asarray(v, np.float32).ravel()
    a = f(scale) * f(inv_std)
    b = f(bias) - f(mean) * a
    v = f64(np.asarray(x3, np.float32)) * f64(a)[None, :, None] + f64(b)[None, :, None]  # the fused multiply-add rounds once
    return v.astype(np.float32) > 0


def bn_dparam(g3, x3, mean, inv_std, mask=None):
    """(dscale, dbias) and their stage-1 bounds; mean / inv_std are inputs of the backward"""
    g3, x3 = f64(g3), f64(x3)
    if mask is not None:
        g3 = np.where(mask, g3, 0.0)
    K = x3.shape[0] * x3.shape[2]
    d = x3 - f64(mean).ravel()[None, :, None]
    r = f64(inv_std).ravel()
    dbias, dscale = g3.sum(axis=(0, 2)), (g3 * d).sum(axis=(0, 2)) * r
    e_db = sum_bound(K, np.abs(g3).sum(axis=(0, 2))) + U * np.abs(dbias)
    e_ds = sum_bound(K, np.abs(g3 * d).sum(axis=(0, 2))) * r + 2 * U * np.abs(dscale)
    return (dscale, e_ds), (dbias, e_db)


def bn_dx(g3, x3, scale, mean, inv_std, dscale, dbias, mask=None):
    """dx = a g + p x + q, p = -a inv_std dscale / n, q = -a dbias / n - p mean, from the given (stored) dscale / dbias"""
    g3, x3 = f64(g3), f64(x3)
    if mask is not None:
        g3 = np.where(mask, g3, 0.0)
    n = x3.shape[0] * x3.shape[2]
    bc = lambda v: f64(v).ravel()[None, :, None]
    a = bc(scale) * bc(inv_std)
    p = -a * bc(inv_std) * bc(dscale) / n
    q0 = -a * bc(dbias) / n
    dx = a * g3 + p * x3 + (q0 - p * bc(mean))
    e = BOUND_C * U * (np.abs(a * g3) + np.abs(p * x3) + np.abs(p * bc(mean)) + np.abs(q0))
    return dx, e


# ---- layer norm / rms norm on x as [rows, inner] -------------------------------------------------------------------------------
def row_stats(x2, eps, rms=False):
    """(mean, inv_std) with their stage-1 bounds; rms: mean = 0 exactly"""
    x2 = f64(x2)
    K = x2.shape[1]
    mean = np.zeros(x2.shape[0]) if rms else x2.mean(axis=1)
    e_mean = np.zeros(x2.shape[0]) if rms else sum_bound(K, np.abs(x2).sum(axis=1)) / K + U * np.abs(mean)
    d = x2 - mean[:, None]
    var = (d * d).mean(axis=1)
    e_var = sum_bound(K, (d * d).sum(axis=1)) / K + e_mean ** 2 + U * var
    inv_std = 1.0 / np.sqrt(var + eps)
    return (mean, e_mean), (inv_std, inv_std * (0.5 * e_var / (var + eps) + 4 * U))


def row_apply(x2, scale, bias, mean, inv_std):
    x2 = f64(x2)
    xh = (x2 - f64(mean).reshape(-1, 1)) * f64(inv_std).reshape(-1, 1)
    y = xh if scale is None else xh * f64(scale).reshape(1, -1)
    mag = np.abs(y)
    if bias is not None:
        y = y + f64(bias).reshape(1, -1)
        mag = mag + np.abs(f64(bias).reshape(1, -1))
    return y, BOUND_C * U * mag


def row_dx(g2, x2, scale, mean, inv_std, rms=False):
    """dx = r (gs - mean(gs) - xhat mean(gs xhat)), gs = g scale (rms: without the mean(gs) term); both means are fp32 row sums
    inside the kernel, so their sum_bound is part of the element's bound"""
    g2, x2 = f64(g2), f64(x2)
    K = x2.shape[1]
    r = f64(inv_std).reshape(-1, 1)
    xh = (x2 - f64(mean).reshape(-1, 1)) * r
    gs = g2 if scale is None else g2 * f64(scale).reshape(1, -1)
    s1 = np.zeros((x2.shape[0], 1)) if rms else gs.mean(axis=1, keepdims=True)
    s2 = (gs * xh).mean(axis=1, keepdims=True)
    e1 = 0.0 if rms else sum_bound(K, np.abs(gs).sum(axis=1, keepdims=True)) / K
    e2 = sum_bound(K, np.abs(gs * xh).sum(axis=1, keepdims=True)) / K
    dx = r * (gs - s1 - xh * s2)
    e = r * (BOUND_C * U * (np.abs(gs) + np.abs(s1) + np.abs(xh * s2)) + e1 + np.abs(xh) * e2)
    return dx, e


def row_dparam(g2, x2, mean, inv_std):
    """dscale[j] = sum over rows of g xhat, dbias[j] = sum over rows of g, with stage-1 bounds (K = rows)"""
    g2, x2 = f64(g2), f64(x2)
    xh = (x2 - f64(mean).reshape(-1, 1)) * f64(inv_std).reshape(-1, 1)
    R = x2.shape[0]
    return ((g2 * xh).sum(axis=0), sum_bound(R, np.abs(g2 * xh).sum(axis=0))), (g2.sum(axis=0), sum_bound(R, np.abs(g2).sum(axis=0)))


# ---- group norm: statistics slot of element i along axis d is i * rdim[d] / dim[d] (rdim divides dim) ---------------------------
def gn_epsilon(reduce_count):
    """the word the reference reads as the group norm's epsilon: gnorm.reduce_count's bits as a float (a denormal, or 0)"""
    return float(np.array([reduce_count], np.int32).view(np.float32)[0])


def gn_expand(v, shape):
    """a statistics / scale tensor broadcast to `shape`: each axis repeated dim / rdim times"""
    v = np.asarray(v)
    for d, (n, r) in enumerate(zip(shape, v.shape)):
        assert n % r == 0
        v = np.repeat(v, n // r, axis=d)
    return v


def gn_reduce(v, rshape):
    """sum of v over every slot of a tensor of dims rshape"""
    v = f64(v)
    split = []
    for n, r in zip(v.shape, rshape):
        split += [r, n // r]
    return v.reshape(split).sum(axis=tuple(range(1, 2 * v.ndim, 2)))


def gn_stats(x, rshape, eps):
    x = f64(x)
    K = x.size // int(np.prod(rshape))
    mean = gn_reduce(x, rshape) / K
    e_mean = sum_bound(K, gn_reduce(np.abs(x), rshape)) / K + U * np.abs(mean)
    d = x - gn_expand(mean, x.shape)
    m2 = gn_reduce(d * d, rshape)
    var = m2 / K
    e_var = sum_bound(K, m2) / K + e_mean ** 2 + U * var
    inv_std = 1.0 / np.sqrt(var + eps)
    return (mean, e_mean), (inv_std, inv_std * (0.5 * e_var / (var + eps) + 4 * U))


def gn_apply(x, scale, bias, mean, inv_std):
    x = f64(x)
    xh = (x - gn_expand(f64(mean), x.shape)) * gn_expand(f64(inv_std), x.shape)
    if scale is None:
        return xh, BOUND_C * U * np.abs(xh)
    s, b = gn_expand(f64(scale), x.shape), gn_expand(f64(bias), x.shape)
    return xh * s + b, BOUND_C * U * (np.abs(xh * s) + np.abs(b))


def gn_dx(g, x, scale, mean, inv_std):
    """h = gss - (sum gss + xhat sum(xhat gss)) / n over the element's slot, gss = g scale inv_std (ccv_nnc_group_norm_cpu_ref.c:412-500)"""
    g, x = f64(g), f64(x)
    rshape = np.shape(mean)
    K = x.size // int(np.prod(rshape))
    r = gn_expand(f64(inv_std), x.shape)
    xh = (x - gn_expand(f64(mean), x.shape)) * r
    gss = g * r if scale is None else g * gn_expand(f64(scale), x.shape) * r
    s1, s2 = gn_reduce(gss, rshape), gn_reduce(xh * gss, rshape)
    e1, e2 = sum_bound(K, gn_reduce(np.abs(gss), rshape)), sum_bound(K, gn_reduce(np.abs(xh * gss), rshape))
    ex = lambda v: gn_expand(v, x.shape)
    h = gss - (ex(s1) + xh * ex(s2)) / K
    e = BOUND_C * U * (np.abs(gss) + np.abs(ex(s1)) / K + np.abs(xh * ex(s2)) / K) + (ex(e1) + np.abs(xh) * ex(e2)) / K
    return h, e


def gn_dparam(g, x, mean, inv_std, sshape):
    g, x = f64(g), f64(x)
    xh = (x - gn_expand(f64(mean), x.shape)) * gn_expand(f64(inv_std), x.shape)
    K = x.size // int(np.prod(sshape))
    return ((gn_reduce(g * xh, sshape), sum_bound(K, gn_reduce(np.abs(g * xh), sshape))),
            (gn_reduce(g, sshape), sum_bound(K, gn_reduce(np.abs(g), sshape))))


# ---- the launch plan, restated from sm100_bn.cu (run_reduce, run_apply, bn_fwd_train_t, bn_bwd_t) and sm100_norm.cu ---------------
def _w(kind):
    return 4 if kind == F32 else 8  # elements of one 16-byte access


def bn_reduce_path(C, inner, kind):
    """'vector': per-block partial rows (16-byte accesses, NHWC, C a multiple of the vector); 'generic': one block per channel"""
    return "vector" if inner == 1 and C % _w(kind) == 0 else "generic"


def bn_reduce_rows(outer, C, kind, sms=SMS):
    """partial rows (gridDim.y) of the vector reduce: reduce_config"""
    cw = C // _w(kind)
    cpb = min(cw, 256)
    rpi = 256 // cpb
    gx = (cw + cpb - 1) // cpb
    return max(1, min((outer + rpi * 32 - 1) // (rpi * 32), (sms * 4 + gx - 1) // gx))


def bn_apply_path(C, inner, kind):
    """'fixed': channel-stationary threads; 'vec': 4 elements per access, coefficients reloaded; 'generic': scalar, any layout"""
    w = _w(kind)
    if inner == 1 and C % w == 0 and (256 % (C // w) == 0 or (C // w) % 256 == 0):
        return "fixed"
    return "vec" if inner == 1 and C % 4 == 0 else "generic"


def bn_plan(form, outer, C, inner, kind, mask=False, colsum=False, ext=False, dx=True):
    """form 'train' | 'test' | 'backward' -> dict(reduce, finalize, apply, colsum, launches)"""
    red, app = bn_reduce_path(C, inner, kind), bn_apply_path(C, inner, kind)
    if form == "test":
        return dict(reduce=None, finalize="test_coef", apply=app, colsum=None, launches=2)
    if form == "train":
        if ext:
            return dict(reduce=None, finalize="ext", apply=app, colsum=None, launches=2)
        return dict(reduce=red, finalize="ext" if red == "vector" else "ws", apply=app, colsum=None, launches=3)
    n = 2 + (1 if mask or red == "generic" else 0)  # [mask / a coefficients], reduce, finalize
    cs = None
    if dx:
        n += 1
        if colsum:
            cv = C // 4
            if app == "fixed" or (app == "vec" and (256 % cv == 0 or cv % 256 == 0)):
                cs, n = "apply", n + 1          # the apply pass leaves partial rows, one launch adds them
            elif C % 4 == 0 and inner == 1:
                cs, n = "two_stage", n + 2      # a separate vector column sum over dx and its fixed-order combine
            else:
                cs, n = "scalar", n + 1
    return dict(reduce=red, finalize="partials" if red == "vector" else "ws", apply=app if dx else None, colsum=cs, launches=n)


def row_threads(inner):
    return 512 if inner >= 2048 else 256 if inner >= 512 else 128 if inner >= 128 else 64 if inner >= 64 else 32


def row_dparam_blocks(rows):
    return min(rows, 296)


def row_plan(form, dx=True, dparam=False):
    """layer / rms norm: forward 1; backward 1 for dx and 2 for the parameter gradients (partial rows, fixed-order combine)"""
    return 1 if form == "forward" else (1 if dx else 0) + (2 if dparam else 0)


def gn_plan(form, dx=True, dparam=False):
    """group norm: forward statistics + apply; backward statistics + apply for h, one launch for dscale / dbias"""
    return 2 if form == "forward" else (2 if dx else 0) + (1 if dparam else 0)
