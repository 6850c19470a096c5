"""ADAM and ADAMW restated in numpy, in CPU_REF's order (lib/nnc/cmd/adam/ccv_nnc_adam_cpu_ref.c, ccv_nnc_adamw_cpu_ref.c): every
product, sum and quotient of the element-wise step is one float32 operation, in the association of the source line:

    grad = scale g                      (ADAM also: grad = grad + decay a, the L2 term)
    n = beta1 m + (1 - beta1) grad
    u = beta2 v + ((1 - beta2) grad) grad
    v_hat = u inv_bias_correction2      (amsgrad: um = ccv_max(vm, v_hat) = vm > v_hat ? vm : v_hat, a NaN v_hat wins)
    ADAM:  b = a - (n rate_inv_bias_correction1) / (sqrt(v_hat) + epsilon)
    ADAMW: b = (a - (rate decay) a) - (n rate_inv_bias_correction1) / (sqrt(v_hat) + epsilon)

rate_inv_bias_correction1 = rate / (1 - powf(beta1, step)) in float; inv_bias_correction2 = 1. / (1 - powf(beta2, step)), the
difference in float and the quotient in double, rounded once.  16-bit operands take the functional form (STAGE_F32): widened, this
arithmetic, each output rounded once to nearest even (the caller rounds).

tests/golden/cpuref_adam.npz pins this to CPU_REF itself (tests/test_adam_random_cpu.py).  `defect` selects one plausible kernel
defect, for showing that the fixture tells it apart."""
import numpy as np

from tests.optim_ref import powf

f32 = np.float32
ADAM_DEFECTS = ("fma", "decay_swapped", "fmaxf", "step_minus_1", "no_scale", "grad_sq")


def _w(x):
    return np.asarray(x, np.float32).ravel()


def _fma(x, y, z):
    """x y + z rounded once to float32 (the float64 product is exact; the float64 sum may round first, which a defect model may do)"""
    return (np.float64(x) * np.asarray(y, np.float64) + np.asarray(z, np.float64)).astype(f32)


def adam(g, a, m, v, step, rate, beta1, beta2, decay, epsilon, amsgrad=0, scale=1.0, vm=None, adamw=False, defect=None):
    """one ADAM (adamw=False) or ADAMW command -> (b, n, u, um); um is None unless amsgrad and vm is given"""
    g, a, m, v = _w(g), _w(a), _w(m), _w(v)
    rate, beta1, beta2, decay, epsilon = f32(rate), f32(beta1), f32(beta2), f32(decay), f32(epsilon)
    bc_step = step - 1 if defect == "step_minus_1" else step
    with np.errstate(all="ignore"):
        rib1 = f32(rate / (f32(1) - powf(beta1, bc_step)))
        ibc2 = f32(np.float64(1) / np.float64(f32(1) - powf(beta2, bc_step)))  # the difference in float, the quotient in double
        l2 = not adamw if defect != "decay_swapped" else adamw
        grad = g if defect == "no_scale" else f32(scale) * g
        if l2:
            grad = _fma(decay, a, grad) if defect == "fma" else grad + decay * a
        if defect == "fma":
            n = _fma(beta1, m, (f32(1) - beta1) * grad)
            u = _fma(beta2, v, ((f32(1) - beta2) * grad) * grad)
        else:
            n = beta1 * m + (f32(1) - beta1) * grad
            u = beta2 * v + (((f32(1) - beta2) * (grad * grad)) if defect == "grad_sq" else ((f32(1) - beta2) * grad) * grad)
        v_hat = u * ibc2
        um = None
        if amsgrad and vm is not None:
            vm = _w(vm)
            um = np.fmax(vm, v_hat) if defect == "fmaxf" else np.where(vm > v_hat, vm, v_hat)
            v_hat = um
        q = (n * rib1) / (np.sqrt(v_hat) + epsilon)
        if l2:
            b = a - q
        else:
            rd = rate * decay
            b = (_fma(-rd, a, a) if defect == "fma" else a - rd * a) - q
    return b.astype(f32), n.astype(f32), u.astype(f32), None if um is None else um.astype(f32)


def same(x, y):
    """bit for bit, every NaN alike (the device's NaN has another payload than numpy's)"""
    x, y = np.ascontiguousarray(x, np.float32).ravel(), np.ascontiguousarray(y, np.float32).ravel()
    if x.shape != y.shape:
        return False
    nx, ny = np.isnan(x), np.isnan(y)
    return np.array_equal(nx, ny) and np.array_equal(x[~nx].view(np.uint32), y[~ny].view(np.uint32))
