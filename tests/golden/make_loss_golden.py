"""Writes tests/golden/cpuref_loss.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on the loss commands
BINARY_CROSSENTROPY, SIGMOID_BINARY_CROSSENTROPY, MSE and SMOOTH_L1, forward and backward, on the reference's 10 x 100 shape, so that
tests/test_parity_loss.py pins its oracles (tests/loss_ref.py) to CPU_REF without the reference present.

Every form: pos_weight 1 and 2.5, MSE mean and sum, both smooth-L1 branches (alternate rows), the backward with and without g, the
sigmoid BCE forward with c and without it, and BCE's backward on inputs that reach the 1e-12 clamp (a = 0 and a = 1).

  python tests/golden/make_loss_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests import loss_ref as L  # noqa: E402
from tests.test_parity_loss import FORMS, commands, operands  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402


def run(cmd, ins, outs):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    z = lambda *s: np.zeros(s, np.float32)
    out = {"g": seeded((10,), 2, 0.5, 2)}
    for op in (L.BCE, L.SBCE, L.MSE, L.SL1):
        out["a_" + op], out["b_" + op] = operands(op, (10, 100), 1)
    a = seeded((10, 100), 5, 0.02, 0.98)
    a[:, ::7], a[:, 3::7] = 1.0, 0.0
    out["a_clamp"], out["b_clamp"] = a, (seeded((10, 100), 6) > 0.5).astype(np.float32)
    for name, op, param in FORMS:
        fwd, bwd = commands(nnc, op, param)
        a, b = out["a_" + op], out["b_" + op]
        if op == L.SBCE:
            c, d = run(fwd, [a, b], [z(10), z(10, 100)])
            (d2,) = run(fwd, [a, b], [None, z(10, 100)])[1:]
            assert np.array_equal(d, d2)
            out["c_" + name], out["d_" + name] = c, d
        else:
            (out["c_" + name],) = run(fwd, [a, b], [z(10)])
        for with_g in (1, 0):
            g, tag = (out["g"] if with_g else None), "%s_g%d" % (name, with_g)
            if op == L.BCE:
                (out["h_" + tag],) = run(bwd, [g, a, b], [z(10, 100)])
                (out["hclamp_" + tag],) = run(bwd, [g, out["a_clamp"], out["b_clamp"]], [z(10, 100)])
            elif op == L.SBCE:
                (out["h_" + tag],) = run(bwd, [g, None, None, b, None, out["d_" + name]], [z(10, 100)])
            elif op == L.MSE:
                out["ha_" + tag], out["hb_" + tag] = run(bwd, [g, a, b], [z(10, 100), z(10, 100)])
            else:
                (out["h_" + tag],) = run(bwd, [g, a, b, out["c_" + name]], [z(10, 100)])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_loss.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
