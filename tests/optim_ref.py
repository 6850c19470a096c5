"""LAMB and RMSPROP restated in numpy, in CPU_REF's order (lib/nnc/cmd/lamb/ccv_nnc_lamb_cpu_ref.c, rmsprop/ccv_nnc_rmsprop_cpu_ref.c):
every product and sum of the elementwise step is one float32 operation, in the association of the source line; LAMB's norms are
sequential float64 sums of float32 squares.  16-bit operands are widened to float32 first; the caller rounds the outputs once.

tests/golden/cpuref_optim.npz pins these to CPU_REF itself (tests/test_optim_cpu.py).  `defect` selects one plausible kernel defect,
for showing that the fixture tells it apart."""
import ctypes as C
import ctypes.util

import numpy as np

f32 = np.float32
_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype, _libm.powf.argtypes = C.c_float, [C.c_float, C.c_float]

OPTIM_MULTI_MAX, OPTIM_CHUNK = 32, 4096
LAMB_DEFECTS = ("fma", "f32_norm", "new_weight_norm", "adam_decay", "beta2_grad_sq", "shared_trust")


def powf(x, y):
    """the C library's powf, which CPU_REF calls for the bias corrections"""
    return f32(_libm.powf(float(x), float(y)))


def inv_bias_correction(beta, step):
    """(float)(1. / (1 - powf(beta, step))): the difference in float, the quotient in double"""
    return f32(1.0 / float(f32(1) - powf(beta, step)))


def _seq_sum(x):
    """sequential float64 sum, element order (np.add.accumulate does not pair)"""
    x = np.asarray(x, np.float64).ravel()
    return float(np.add.accumulate(x)[-1]) if x.size else 0.0


def _w(x):
    return np.asarray(x, np.float32).ravel()


def lamb_update(g, a, m, v, step, beta1, beta2, decay, epsilon, scale=1.0, defect=None):
    """-> (update, n, u), float32"""
    g, a, m, v = _w(g), _w(a), _w(m), _w(v)
    beta1, beta2, decay, epsilon = f32(beta1), f32(beta2), f32(decay), f32(epsilon)
    ibc1, ibc2 = inv_bias_correction(beta1, step), inv_bias_correction(beta2, step)
    with np.errstate(all="ignore"):
        grad = f32(scale) * g
        if defect == "adam_decay":
            grad = grad + decay * a
        n = beta1 * m + (f32(1) - beta1) * grad
        if defect == "beta2_grad_sq":
            u = beta2 * v + (f32(1) - beta2) * (grad * grad)
        else:
            u = beta2 * v + ((f32(1) - beta2) * grad) * grad
        q = (n * ibc1) / (np.sqrt(u * ibc2) + epsilon)
        if defect == "adam_decay":
            update = q
        elif defect == "fma":
            update = (a.astype(np.float64) * np.float64(decay) + q.astype(np.float64)).astype(np.float32)
        else:
            update = q + a * decay
    return update, n, u


def lamb_norms(a, update, defect=None):
    """(sum a^2, sum update^2) as CPU_REF keeps them: float32 squares added in float64, in element order"""
    a, update = _w(a), _w(update)
    with np.errstate(all="ignore"):
        if defect == "f32_norm":
            return float(np.add.accumulate(a * a, dtype=np.float32)[-1]), float(np.add.accumulate(update * update, dtype=np.float32)[-1])
        return _seq_sum(a * a), _seq_sum(update * update)


def trust_ratio(w_sq, u_sq):
    """float64 norms, their quotient rounded to float32; 1 unless both are > 0 (a NaN gives 1).  Also returns the float64 quotient."""
    w, u = np.sqrt(w_sq), np.sqrt(u_sq)
    if w > 0 and u > 0:
        return f32(w / u), w / u
    return f32(1), None


def lamb(g, a, m, v, step, rate, beta1, beta2, decay, epsilon, scale=1.0, defect=None):
    """one LAMB command -> (b, n, u, trust as float64 or None when it is 1)"""
    update, n, u = lamb_update(g, a, m, v, step, beta1, beta2, decay, epsilon, scale, defect)
    a = _w(a)
    w_sq, u_sq = lamb_norms(a, update, defect)
    if defect == "new_weight_norm":
        t0, _ = trust_ratio(w_sq, u_sq)
        with np.errstate(all="ignore"):
            w_sq = _seq_sum(np.square(a - (f32(rate) * t0) * update))
    trust, t64 = trust_ratio(w_sq, u_sq)
    with np.errstate(all="ignore"):
        b = a - (f32(rate) * trust) * update
    return b, n, u, t64


def lamb_multi(tensors, step, rate, beta1, beta2, decay, epsilon, scale=1.0, defect=None):
    """a fused run: tensors [(g, a, m, v)] -> [(b, n, u)]; each tensor has its own trust ratio (defect "shared_trust": one over all)"""
    if defect != "shared_trust":
        return [lamb(g, a, m, v, step, rate, beta1, beta2, decay, epsilon, scale, defect)[:3] for g, a, m, v in tensors]
    parts = [lamb_update(g, a, m, v, step, beta1, beta2, decay, epsilon, scale) for g, a, m, v in tensors]
    w_sq, u_sq = lamb_norms(np.concatenate([_w(t[1]) for t in tensors]), np.concatenate([p[0] for p in parts]))
    trust, _ = trust_ratio(w_sq, u_sq)
    with np.errstate(all="ignore"):
        return [(_w(t[1]) - (f32(rate) * trust) * p[0], p[1], p[2]) for t, p in zip(tensors, parts)]


def rmsprop(g, a, m, v, rate, decay, alpha, momentum, epsilon, scale=1.0):
    """one RMSPROP command -> (b, n, u)"""
    g, a, m, v = _w(g), _w(a), _w(m), _w(v)
    alpha = f32(alpha)
    with np.errstate(all="ignore"):
        grad = f32(scale) * g
        grad = grad + f32(decay) * a
        u = alpha * v + ((f32(1) - alpha) * grad) * grad
        n = f32(momentum) * m + grad / (np.sqrt(u) + f32(epsilon))
        b = a - f32(rate) * n
    return b, n, u


def midpoint_margin(t64):
    """relative distance of a float64 trust ratio from the nearest float32 rounding midpoint: when it is larger than the error of any
    order of the float64 sums, every order rounds to the same float32"""
    f = f32(t64)
    up, down = np.nextafter(f, f32(np.inf)), np.nextafter(f, f32(-np.inf))
    mids = [(float(f) + float(up)) / 2, (float(f) + float(down)) / 2]
    return min(abs(t64 - x) for x in mids) / abs(t64)


def optim_multi_plan(counts):
    """the launch tables of sm100_optim.cu for T commands of these element counts: the tensors in order, OPTIM_MULTI_MAX to a table
    (whatever their alignment: a CTA picks the vector or the scalar path per tensor).  RMSPROP launches once per table, LAMB three
    times (norms, trust, apply).  ResNet-50's 161 parameters in two decay groups (53 and 108 tensors) are 2 + 4 tables: 18 LAMB
    launches, 6 RMSPROP launches."""
    return [list(range(k, min(k + OPTIM_MULTI_MAX, len(counts)))) for k in range(0, len(counts), OPTIM_MULTI_MAX)]
