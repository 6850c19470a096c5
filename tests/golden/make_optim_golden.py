"""Writes tests/golden/cpuref_optim.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on LAMB and RMSPROP,
so that tests/test_optim_cpu.py pins the oracles of tests/optim_ref.py to CPU_REF without the reference present.  CPU_REF runs these
commands in fp32 only.

Cases: in place and out of place, decay 0 and non-zero, steps 1 and 1000, scale != 1, an all-zero a (LAMB's trust ratio is 1), a NaN
gradient (trust 1, NaN in that element), a rate of 1 (the update's last bits reach b), and a run of three LAMB tensors of different scales, each its own command.

  python tests/golden/make_optim_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402

# (name, count, step, rate, beta1, beta2, decay, epsilon, scale, in_place, a_zero, nan_at)
LAMB_CASES = [("base", 1000, 1, 0.002, 0.9, 0.98, 0.0, 1e-9, 1.0, False, False, None),
              ("decay_step1000", 1537, 1000, 0.01, 0.9, 0.999, 0.01, 1e-6, 0.5, True, False, None),
              ("zero_a", 777, 3, 0.01, 0.9, 0.999, 0.01, 1e-6, 1.0, False, True, None),
              ("nan_g", 513, 2, 0.01, 0.9, 0.999, 0.0, 1e-6, 1.0, True, False, 17),
              # a rate near 1 keeps the last bits of the update visible in b
              ("large_rate", 2048, 10, 1.0, 0.9, 0.999, 0.3, 1e-6, 2.0, False, False, None)]
# (name, count, rate, decay, alpha, momentum, epsilon, scale, in_place, nan_at)
RMSPROP_CASES = [("base", 1000, 0.001, 0.0, 0.9, 0.9, 1e-8, 1.0, False, None),
                 ("decay_scale", 1537, 0.01, 0.01, 0.99, 0.5, 1e-6, 0.5, True, None),
                 ("nan_g", 513, 0.01, 0.0, 0.9, 0.0, 1e-6, 1.0, False, 17)]
# a run of LAMB tensors with one command's parameters; their norms differ, so one shared trust ratio would give other bits
RUN_COUNTS, RUN_SCALES = (300, 1000, 77), (1.0, 0.01, 30.0)
RUN_HP = dict(step=5, rate=0.01, beta1=0.9, beta2=0.999, decay=0.01, epsilon=1e-6)


def state(count, seed):
    """g, a, m and a non-negative v"""
    return (seeded((count,), seed, -1, 1), seeded((count,), seed + 1, -1, 1), seeded((count,), seed + 2, -0.1, 0.1),
            seeded((count,), seed + 3, 0, 0.01))


def run(cmd, g, a, m, v, in_place):
    """CPU_REF on (g, a, m, v) -> (b, n, u); in place: b = a, n = m, u = v"""
    a, m, v = a.copy(), m.copy(), v.copy()
    outs = [a, m, v] if in_place else [np.zeros_like(a), np.zeros_like(m), np.zeros_like(v)]
    st, res = ref_exec(ref, cmd, None, 0, [g, a, m, v], outs)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {}
    for k, (name, count, step, rate, beta1, beta2, decay, eps, scale, in_place, a_zero, nan_at) in enumerate(LAMB_CASES):
        g, a, m, v = state(count, 200 + 10 * k)
        if a_zero:
            a[:] = 0
        if nan_at is not None:
            g[nan_at] = np.nan
        for key, x in zip("gamv", (g, a, m, v)):
            out["lamb_%s_%s" % (key, name)] = x
        b, n, u = run(nnc.CMD_LAMB_FORWARD(step, rate, beta1, beta2, decay, eps, scale=scale), g, a, m, v, in_place)
        out["lamb_b_" + name], out["lamb_n_" + name], out["lamb_u_" + name] = b, n, u
    for k, (name, count, rate, decay, alpha, momentum, eps, scale, in_place, nan_at) in enumerate(RMSPROP_CASES):
        g, a, m, v = state(count, 300 + 10 * k)
        if nan_at is not None:
            g[nan_at] = np.nan
        for key, x in zip("gamv", (g, a, m, v)):
            out["rmsprop_%s_%s" % (key, name)] = x
        b, n, u = run(nnc.CMD_RMSPROP_FORWARD(rate, decay, alpha, momentum, eps, scale=scale), g, a, m, v, in_place)
        out["rmsprop_b_" + name], out["rmsprop_n_" + name], out["rmsprop_u_" + name] = b, n, u
    for i, (count, s) in enumerate(zip(RUN_COUNTS, RUN_SCALES)):
        g, a, m, v = state(count, 400 + 10 * i)
        a *= np.float32(s)
        for key, x in zip("gamv", (g, a, m, v)):
            out["run_%s_%d" % (key, i)] = x
        b, n, u = run(nnc.CMD_LAMB_FORWARD(**RUN_HP), g, a, m, v, False)
        out["run_b_%d" % i], out["run_n_%d" % i], out["run_u_%d" % i] = b, n, u
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_optim.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
