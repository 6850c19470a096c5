"""Writes tests/golden/cpuref_ew.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on small seeded cases of
SIGMOID, TANH, LEAKY_RELU, EWEXP (also without g), EWLOG, EWSQRT, CLAMP, GELU (erf and tanh), SWISH, EWDIV (with and without a and g),
REDUCE_SUM / MEAN / MAX / MIN / NORM2 over several axis sets (all -inf / +inf and all-NaN slices, ties, backward with a broadcast g and
without g), MASKED_FILL (int32 and fp32 masks broadcast on each axis), EWSUM (left to right, the output aliasing an operand, 9 operands),
ADD / MUL (broadcast, backward with and without g) and SCALAR_MUL, so that tests/test_parity_ew_paths.py pins its oracles
(tests/ew_ref.py) to CPU_REF without the reference present.

  python tests/golden/make_ew_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.test_parity_ew_paths import (ACTS, ADD_PQ, GOLDEN_BCAST, GOLDEN_N, GOLDEN_REDUCE_AXES, MF_Q, MUL_P, UNARY_ARGS, act_cmds, bshape_of,  # noqa: E402
                                        bwd_cmd, fwd_cmd, mf_p, reduce_golden_data, unary_data)
from tests.util import ref_exec, seeded  # noqa: E402


def run(cmd, ins, outs):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def z(shape):
    return np.zeros(shape, np.float32)


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {}
    n = GOLDEN_N
    for i, name in enumerate(sorted(UNARY_ARGS)):
        a, g = unary_data(name, n, 200 + i), seeded((n,), 300 + i, -1, 1)
        (b,) = run(fwd_cmd(name), [a], [z(n)])
        (h,) = run(bwd_cmd(name), [g, a, b], [z(n)])
        out.update({name + "_a": a, name + "_g": g, name + "_b": b, name + "_h": h})
        if name == "EWEXP":
            out["EWEXP_h_nog"] = run(bwd_cmd(name), [None, a, b], [z(n)])[0]
    for i, name in enumerate(sorted(ACTS)):
        a, g = unary_data(name, n, 400 + i), seeded((n,), 500 + i, -1, 1)
        fwd, bwd = act_cmds(name)
        (b,) = run(fwd, [a], [z(n)])
        out.update({name + "_a": a, name + "_g": g, name + "_b": b, name + "_h": run(bwd, [g, a, b], [z(n)])[0]})
    a, g = seeded((n,), 600, -2, 2), seeded((n,), 601, -1, 1)
    b = seeded((n,), 602, 0.5, 2) * np.sign(seeded((n,), 603, -1, 1))
    (c,) = run(nnc.CMD_EWDIV_FORWARD(), [a, b], [z(n)])
    out.update(div_a=a, div_b=b, div_g=g, div_c=c, div_c1=run(nnc.CMD_EWDIV_FORWARD(), [None, b], [z(n)])[0])
    for gg, sfx in ((g, ""), (None, "_nog")):
        ha, hb = run(nnc.CMD_EWDIV_BACKWARD(), [gg, a, b, c], [z(n), z(n)])
        out["div_ha" + sfx], out["div_hb" + sfx] = ha, hb
    for i, mode in enumerate(("SUM", "MEAN", "MAX", "MIN", "NORM2")):
        a = reduce_golden_data(mode, 700 + i)
        out["red_%s_a" % mode] = a
        for axes in GOLDEN_REDUCE_AXES:
            key = "red_%s_%s_" % (mode, "".join(map(str, axes)))
            bs = bshape_of(a.shape, axes)
            fwd = getattr(nnc, "CMD_REDUCE_%s_FORWARD" % mode)(*axes)
            bwd = getattr(nnc, "CMD_REDUCE_%s_BACKWARD" % mode)(*axes)
            (b,) = run(fwd, [a], [z(bs)])
            g = seeded(bs, 800 + i, -1, 1)
            out[key + "b"], out[key + "g"] = b, g
            out[key + "h"] = run(bwd, [g, a, b], [z(a.shape)])[0]
            out[key + "h_nog"] = run(bwd, [None, a, b], [z(a.shape)])[0]
        if mode == "MEAN":
            # without g the scale comes from the command's axes (here 0), not from the b passed beside it (axes 1 and 3 reduced)
            b = run(nnc.CMD_REDUCE_MEAN_FORWARD(1, 3), [a], [z(bshape_of(a.shape, (1, 3)))])[0]
            out["red_MEAN_cmd0_b"] = b
            out["red_MEAN_cmd0_h_nog"] = run(nnc.CMD_REDUCE_MEAN_BACKWARD(0), [None, a, b], [z(a.shape)])[0]
    a, g = seeded((2, 3, 4), 900, -1, 1), seeded((2, 3, 4), 901, -1, 1)
    out.update(mf_a=a, mf_g=g)
    r = np.random.RandomState(902)
    for mtype in ("int32", "fp32"):
        for ax in (0, 1, 2):
            key = "mf_%s_%d_" % (mtype, ax)
            ms = tuple(1 if i == ax else d for i, d in enumerate(a.shape))
            m = r.randint(0, 3, size=ms)
            m = m.astype(np.int32) if mtype == "int32" else m.astype(np.float32)
            p = mf_p(mtype)
            out[key + "mask"] = m
            out[key + "c"] = run(nnc.CMD_MASKED_FILL_FORWARD(p, MF_Q), [a, m], [z(a.shape)])[0]
            out[key + "h"] = run(nnc.CMD_MASKED_FILL_BACKWARD(p, MF_Q), [g, a, m], [z(a.shape)])[0]
    xs = [(seeded((n,), 1000 + i, -1, 1) * 10.0 ** (i % 3)).astype(np.float32) for i in range(9)]
    for i, x in enumerate(xs):
        out["sum_x%d" % i] = x
    for k, alias in ((3, None), (3, 1), (9, None), (9, 8)):
        ins = [x.copy() for x in xs[:k]]
        o = ins[alias] if alias else z(n)
        out["sum_%d_%s" % (k, alias)] = run(nnc.CMD_EWSUM_FORWARD(), ins, [o])[0].copy()
    for name, ashape, bshape in GOLDEN_BCAST:
        cs = tuple(max(x, y) for x, y in zip(ashape, bshape))
        a, b, g = seeded(ashape, 1100, -1, 1), seeded(bshape, 1101, -1, 1), seeded(cs, 1102, -1, 1)
        out.update({name + "_a": a, name + "_b": b, name + "_g": g})
        if name == "add":
            out[name + "_c"] = run(nnc.CMD_ADD_FORWARD(*ADD_PQ), [a, b], [z(cs)])[0]
            for gg, sfx in ((g, ""), (None, "_nog")):
                h0, h1 = run(nnc.CMD_ADD_BACKWARD(*ADD_PQ), [gg, a, b], [z(ashape), z(bshape)])
                out[name + "_h0" + sfx], out[name + "_h1" + sfx] = h0, h1
            continue
        out[name + "_c"] = run(nnc.CMD_MUL_FORWARD(MUL_P), [a, b], [z(cs)])[0]
        for gg, sfx in ((g, ""), (None, "_nog")):
            h0, h1 = run(nnc.CMD_MUL_BACKWARD(MUL_P), [gg, a, b], [z(ashape), z(bshape)])
            out[name + "_h0" + sfx], out[name + "_h1" + sfx] = h0, h1
        out[name + "_smul"] = run(nnc.CMD_SCALAR_MUL_FORWARD(MUL_P), [a], [z(ashape)])[0]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_ew.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
