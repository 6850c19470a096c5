"""Writes tests/golden/cpuref_addons.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on PAD, MIN / MAX,
ARGMAX / ARGMIN and REDUCE_ISNAN, so that tests/test_parity_model_addons.py pins its oracles (tests/addons_ref.py) to CPU_REF without
the reference present.  CPU_REF runs these commands in fp32 only.

The inputs hold NaN at index 0 and mid-row, ties, +0 against -0, Inf, all-equal rows, and both pad types (zero-width sides too).

  python tests/golden/make_addons_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import abi, nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402

# (name, a's shape, begin, end): 3-d and 4-d, zero-width sides, the NHWC spatial pad
PADS = [("p3", (3, 4, 5), (1, 0, 2), (0, 2, 1)), ("p4", (2, 3, 4, 5), (0, 1, 1, 0), (0, 1, 1, 0)), ("p1", (7,), (3,), (2,))]
ISNAN_OUTS = [(1, 1, 1), (4, 1, 1), (1, 5, 6), (4, 5, 6), (4, 1, 6)]
ARG_CASES = [("r2", (7, 9), 0), ("r2", (7, 9), 1), ("r3", (3, 5, 4), 1), ("r3", (3, 5, 4), 2), ("r3", (3, 5, 4), 0)]


def inputs():
    out = {}
    for name, shape, _, _ in PADS:
        a = seeded(shape, 11, -1, 1)
        a.reshape(-1)[::7] = np.nan
        a.reshape(-1)[3::11] = -0.0
        out["pad_a_" + name] = a
    a, b = seeded((6, 10), 21, -1, 1), seeded((6, 10), 22, -1, 1)
    a[0, :3], b[1, :3] = np.nan, np.nan                  # NaN in either operand
    a[2, :4] = b[2, :4] = 0.5                            # ties
    a[3, :2], b[3, :2] = 0.0, -0.0                       # +0 against -0 ...
    a[3, 2:4], b[3, 2:4] = -0.0, 0.0                     # ... and the reverse
    a[4, :2], b[4, :2] = np.inf, -np.inf
    out["cmp_a"], out["cmp_b"], out["cmp_g"] = a, b, seeded((6, 10), 23, -2, 2)
    r = seeded((7, 9), 31, -1, 1)
    r[0, 0] = np.nan                                     # NaN at index 0 stays the answer
    r[1, 4] = np.nan                                     # NaN mid-row is skipped
    r[2, :] = 0.25                                       # all equal: index 0
    r[3, 2] = r[3, 6] = 2.0                              # a tie: the first index
    r[3, 1] = r[3, 7] = -2.0
    r[4, 0], r[4, 5] = -0.0, 0.0                         # ±0 with every other value negative
    r[4, [1, 2, 3, 4, 6, 7, 8]] = -1.0
    r[5, :] = np.nan                                     # all NaN: index 0
    r[6, :3] = np.nan
    out["arg_r2"] = r
    r3 = seeded((3, 5, 4), 32, -1, 1)
    r3[0, 0, :] = np.nan
    r3[1, 2, 1] = np.nan
    r3[2, :, 3] = 0.5
    out["arg_r3"] = r3
    x = seeded((4, 5, 6), 41, -1, 1)
    x[1, 2, 3] = np.nan
    x[3, 0, 0] = np.nan
    x[2, 4, 5] = np.inf                                  # Inf is not NaN
    x[0, 1, 1] = -np.inf
    out["isnan_a"] = x
    return out


def run(cmd, ins, outs):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = inputs()
    for name, shape, begin, end in PADS:
        a = out["pad_a_" + name]
        bshape = tuple(shape[k] + begin[k] + end[k] for k in range(len(shape)))
        g = seeded(bshape, 12, -1, 1)
        out["pad_g_" + name] = g
        for t in (abi.CCV_NNC_PAD_ZERO, abi.CCV_NNC_PAD_REPLICATE):
            (out["pad_b_%s_%d" % (name, t)],) = run(nnc.CMD_PAD_FORWARD(t, begin, end), [a], [np.zeros(bshape, np.float32)])
            (out["pad_h_%s_%d" % (name, t)],) = run(nnc.CMD_PAD_BACKWARD(t, begin, end), [g], [np.zeros(shape, np.float32)])
    z = lambda: np.zeros((6, 10), np.float32)
    for op, (fwd, bwd) in (("min", (nnc.CMD_MIN_FORWARD, nnc.CMD_MIN_BACKWARD)), ("max", (nnc.CMD_MAX_FORWARD, nnc.CMD_MAX_BACKWARD))):
        (out["cmp_c_" + op],) = run(fwd(), [out["cmp_a"], out["cmp_b"]], [z()])
        out["cmp_ha_%s_g1" % op], out["cmp_hb_%s_g1" % op] = run(bwd(), [out["cmp_g"], out["cmp_a"], out["cmp_b"]], [z(), z()])
        out["cmp_ha_%s_g0" % op], out["cmp_hb_%s_g0" % op] = run(bwd(), [None, out["cmp_a"], out["cmp_b"]], [z(), z()])
    for name, shape, axis in ARG_CASES:
        bshape = tuple(1 if k == axis else shape[k] for k in range(len(shape)))
        for op, make in (("max", nnc.CMD_ARGMAX_FORWARD), ("min", nnc.CMD_ARGMIN_FORWARD)):
            (out["arg_%s_%s_%d_i32" % (op, name, axis)],) = run(make(axis), [out["arg_" + name]], [np.full(bshape, -1, np.int32)])
            (out["arg_%s_%s_%d_f32" % (op, name, axis)],) = run(make(axis), [out["arg_" + name]], [np.full(bshape, -1, np.float32)])
    for bshape in ISNAN_OUTS:
        (out["isnan_b_" + "x".join(map(str, bshape))],) = run(nnc.CMD_REDUCE_ISNAN_FORWARD(), [out["isnan_a"]], [np.full(bshape, 5, np.int32)])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_addons.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
