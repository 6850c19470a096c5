"""Writes tests/golden/cpuref_adam.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on ADAM and ADAMW, so
that tests/test_adam_random_cpu.py pins the oracle of tests/adam_ref.py to CPU_REF without the reference present, and the GPU tests
compare the kernel with CPU_REF's own bits.  CPU_REF runs these commands in fp32 only.

Cases: ADAM and ADAMW, each with amsgrad 0 and 1; steps 1, 3 and 1000; decay 0 and non-zero; scale != 1; a rate of 1 (the last bits of
the update reach b); in place and out of place.  Every case holds NaN, +Inf, -Inf and zero gradients and zero weights at fixed
elements, and with amsgrad a vm that lies above v_hat for some elements and below it for others.

  python tests/golden/make_adam_golden.py"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402

# (name, adamw, amsgrad, count, step, rate, beta1, beta2, decay, epsilon, scale, in_place)
CASES = [("adam_base", 0, 0, 1000, 1, 0.002, 0.9, 0.999, 0.0, 1e-8, 1.0, False),
         ("adam_decay_step3", 0, 0, 1537, 3, 0.01, 0.9, 0.98, 0.01, 1e-6, 0.5, True),
         ("adam_ams_rate1", 0, 1, 1023, 1000, 1.0, 0.9, 0.999, 0.05, 1e-6, 2.0, False),
         ("adam_ams_step3", 0, 1, 777, 3, 0.002, 0.8, 0.99, 0.0, 1e-8, 1.0, True),
         ("adamw_base", 1, 0, 1000, 1, 0.002, 0.9, 0.999, 0.0, 1e-8, 1.0, False),
         ("adamw_rate1", 1, 0, 2048, 1000, 1.0, 0.9, 0.999, 0.1, 1e-6, 2.0, True),
         ("adamw_ams_step1", 1, 1, 1537, 1, 0.01, 0.9, 0.98, 0.05, 1e-6, 0.5, False),
         ("adamw_ams_rate1", 1, 1, 999, 1000, 1.0, 0.9, 0.999, 0.3, 1e-8, 1.0, True)]
NAN_AT, POS_INF_AT, NEG_INF_AT, ZERO_G, ZERO_A = 5, 6, 7, (8, 9, 10, 11), (12, 13, 14, 15)


def cmd_of(case):
    name, adamw, amsgrad, count, step, rate, beta1, beta2, decay, eps, scale, in_place = case
    make = nnc.CMD_ADAMW_FORWARD if adamw else nnc.CMD_ADAM_FORWARD
    return make(step, rate, beta1, beta2, decay, eps, amsgrad, scale=scale)


def state(count, seed, amsgrad):
    """g, a, m, v (>= 0) and, with amsgrad, vm (>= 0) with the special elements in place"""
    g, a = seeded((count,), seed, -1, 1), seeded((count,), seed + 1, -1, 1)
    m, v = seeded((count,), seed + 2, -0.1, 0.1), seeded((count,), seed + 3, 0, 0.01)
    g[NAN_AT], g[POS_INF_AT], g[NEG_INF_AT] = np.nan, np.inf, -np.inf
    g[list(ZERO_G)] = 0
    a[list(ZERO_A)] = 0
    vm = seeded((count,), seed + 4, 0, 0.04) if amsgrad else None
    return g, a, m, v, vm


def main():
    from oracle import ref
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {}
    for k, case in enumerate(CASES):
        name, amsgrad, count, in_place = case[0], case[2], case[3], case[-1]
        g, a, m, v, vm = state(count, 500 + 10 * k, amsgrad)
        for key, x in zip(("g", "a", "m", "v", "vm"), (g, a, m, v, vm)):
            if x is not None:
                out["%s_%s" % (key, name)] = x
        ins = [g, a.copy(), m.copy(), v.copy()] + ([vm.copy()] if amsgrad else [])
        outs = ins[1:] if in_place else [np.zeros_like(x) for x in ins[1:]]
        st, res = ref_exec(ref, cmd_of(case), None, 0, ins, outs)
        assert st == 0, name
        for key, x in zip(("b", "n", "u", "um"), res):
            out["%s_%s" % (key, name)] = x
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_adam.npz")
    # np.savez_compressed stamps each member with the current time; fixed stamps make the file a function of its contents
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(out[name]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
