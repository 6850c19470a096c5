"""Writes tests/golden/cpuref_feeders.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on small seeded cases of
MAX_POOL / AVERAGE_POOL (clipped begin and end windows, stride larger than the window, ties; one call per image, since CPU_REF pools walk
image 0 only), SOFTMAX, CATEGORICAL_CROSSENTROPY and SOFTMAX_CROSSENTROPY (int32 / fp32 indices with 2.6 -> 3, distributions, the 1-d
batch-1 range rule, label smoothing, with and without g) and SGD_FORWARD (nesterov, dampening, decay), so that
tests/test_parity_feeder_paths.py pins its oracles (tests/feeder_ref.py) to CPU_REF without the reference present.

  python tests/golden/make_feeder_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests import feeder_ref as R  # noqa: E402
from tests.test_parity_feeder_paths import GOLDEN_LABELS, GOLDEN_POOLS, GOLDEN_SGD, GOLDEN_TRIMS, SGD_HP, golden_labels, pool_data, pool_hint  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402


def run(cmd, ins, outs, hint=None):
    st, res = ref_exec(ref, cmd, hint, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {}
    for name, kind, shape, geo, end in GOLDEN_POOLS:
        N, H, W, C = shape
        P, Q = R.out_extent(H, geo[0], geo[2], geo[4], end[0]), R.out_extent(W, geo[1], geo[3], geo[5], end[1])
        hint = pool_hint(geo, end)
        a, g = pool_data(shape, 1, kind == "max"), seeded((N, P, Q, C), 2, -1, 1)
        fwd = (nnc.CMD_MAX_POOL_FORWARD if kind == "max" else nnc.CMD_AVERAGE_POOL_FORWARD)(geo[0], geo[1])
        bwd = (nnc.CMD_MAX_POOL_BACKWARD if kind == "max" else nnc.CMD_AVERAGE_POOL_BACKWARD)(geo[0], geo[1])
        b, h = np.zeros((N, P, Q, C), np.float32), np.zeros(shape, np.float32)
        for n in range(N):
            b[n] = run(fwd, [np.ascontiguousarray(a[n])], [np.zeros((P, Q, C), np.float32)], hint)[0]
            ins = [np.ascontiguousarray(g[n])] + ([np.ascontiguousarray(a[n]), np.ascontiguousarray(b[n])] if kind == "max" else [])
            h[n] = run(bwd, ins, [np.zeros((H, W, C), np.float32)], hint)[0]
        out.update({name + "_a": a, name + "_g": g, name + "_b": b, name + "_h": h})
    batch, count = 5, 37
    a = seeded((batch, count), 3, -4, 4)
    g = seeded((batch,), 4, 0.5, 1.5)
    gs = seeded((batch, count), 5, -1, 1)
    (y,) = run(nnc.CMD_SOFTMAX_FORWARD(), [a], [np.zeros_like(a)])
    (hs,) = run(nnc.CMD_SOFTMAX_BACKWARD(), [gs, None, y], [np.zeros_like(a)])
    out.update(loss_a=a, loss_g=g, softmax_y=y, softmax_g=gs, softmax_h=hs)
    a1 = np.ascontiguousarray(a.reshape(-1)[:count * 1])
    out["range1d_y"] = run(nnc.CMD_SOFTMAX_FORWARD(), [a1.reshape(1, count)], [np.zeros((1, count), np.float32)])[0].reshape(-1)
    for which in GOLDEN_LABELS:
        for trims in GOLDEN_TRIMS:
            if which == "dist" and trims != (0.0, 1.0):
                continue
            b1 = 1 if which == "range1d" else batch
            shape = (count,) if which == "range1d" else (batch, count)
            x = a1 if which == "range1d" else a
            p = out["range1d_y"] if which == "range1d" else y
            lab, _ = golden_labels(which, b1, count, 6)
            key = "%s_%g_%g_" % (which, trims[0], trims[1])
            cf, cb = nnc.CMD_CATEGORICAL_CROSSENTROPY_FORWARD(*trims), nnc.CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(*trims)
            sf, sb = nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD(*trims), nnc.CMD_SOFTMAX_CROSSENTROPY_BACKWARD(*trims)
            z1, zs = (lambda: np.zeros((b1,), np.float32)), (lambda: np.zeros(shape, np.float32))
            out[key + "label"] = lab
            out[key + "cce_c"] = run(cf, [p.reshape(shape), lab], [z1()])[0]
            out[key + "cce_h"] = run(cb, [g[:b1], p.reshape(shape), lab], [zs()])[0]
            out[key + "cce_h1"] = run(cb, [None, p.reshape(shape), lab], [zs()])[0]
            c, d = run(sf, [x.reshape(shape), lab], [z1(), zs()])
            out[key + "scce_c"], out[key + "scce_d"] = c, d
            out[key + "scce_h"] = run(sb, [g[:b1], None, None, lab, None, d], [zs()])[0]
            out[key + "scce_h1"] = run(sb, [None, None, None, lab, None, d], [zs()])[0]
    sg, sa, sm = seeded((3, 5, 7), 7, -1, 1), seeded((3, 5, 7), 8, -1, 1), seeded((3, 5, 7), 9, -1, 1)
    out.update(sgd_g=sg, sgd_a=sa, sgd_m=sm)
    for name, nesterov, dampening, decay in GOLDEN_SGD:
        cmd = nnc.CMD_SGD_FORWARD(nesterov, decay=decay, dampening=dampening, **SGD_HP)
        b, n = run(cmd, [sg, sa, sm], [np.zeros_like(sa), np.zeros_like(sa)])
        out["sgd_%s_b" % name], out["sgd_%s_n" % name] = b, n
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_feeders.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
