"""Regenerates tests/golden/*.npz from the reference's own known-answer tests and from the compiled reference
(oracle/_ref/libccv_ref.so).  Run in the build container (needs /root/reference built through `make -C oracle`):

    python tests/golden/make_golden.py
    python tests/golden/make_golden.py registry <reference>/lib/nnc/cmd/ccv_nnc_cmd.inc
    python tests/golden/make_golden.py sdpa          # cpuref_sdpa.npz only

Two kinds of fixtures:
  literal_*   inputs + expected outputs typed from the reference's unit tests (test/unit/nnc/gemm.tests.c etc.); these
              pin the oracle itself.
  cpuref_*    seeded inputs + the outputs CCV_NNC_BACKEND_CPU_REF produced for them here; these travel to the GPU box
              so parity can be checked even without the compiled reference.
  reference_cmd_registry.json   the registry tables of the reference's generated ccv_nnc_cmd.inc: command and backend ids, both
              perfect hashes, and every (command, backend, command slot, backend slot) registration call.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.util import seeded  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def literal_gemm():
    """test/unit/nnc/gemm.tests.c:13-200 (forward cases, hand-computed expectations)."""
    a = np.array([[1, 2], [3, 4], [5, 6], [7, 8]], np.float32)
    b = np.array([[7, 8, 9], [10, 11, 12]], np.float32)
    c = a.astype(np.float64) @ b.astype(np.float64)
    bias = np.array([22, 23, 24], np.float32)
    return dict(a=a, b=b, c=c.astype(np.float32), bt=np.ascontiguousarray(b.T), at=np.ascontiguousarray(a.T)[None], bias=bias,
                c_bias=(c + bias).astype(np.float32))


def cpuref_cases():
    cases = {}
    # GEMM forward NT with bias (dense layer form) and backward
    a, w, bias = seeded((12, 20), 1, -1, 1), seeded((8, 20), 2, -1, 1), seeded((8,), 3)
    b = np.zeros((12, 8), np.float32)
    assert ref.run(nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), None, 0, [a, w, bias], [b]) == 0
    g = seeded((12, 8), 4, -1, 1)
    h, dw, db = np.zeros_like(a), np.zeros_like(w), np.zeros_like(bias)
    assert ref.run(nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1)), None, 0, [g, a, w], [h, dw, db]) == 0
    cases["gemm"] = dict(a=a, w=w, bias=bias, b=b, g=g, h=h, dw=dw, db=db)
    # convolution 3x3 stride 2 pad 1 with bias, forward + backward (NHWC)
    x, wt, cb = seeded((2, 9, 11, 8), 5), seeded((12, 3, 3, 8), 6) / 72, seeded((12,), 7)
    y = np.zeros((2, 5, 6, 12), np.float32)
    hint = nnc.hint((2, 2), (1, 1))
    assert ref.run(nnc.CMD_CONVOLUTION_FORWARD(1, 12, 3, 3, 8), hint, 0, [x, wt, cb], [y]) == 0
    gy = seeded(y.shape, 8)
    gx, gw, gb = np.zeros_like(x), np.zeros_like(wt), np.zeros_like(cb)
    assert ref.run(nnc.CMD_CONVOLUTION_BACKWARD(1, 12, 3, 3, 8), hint, 0, [gy, x, wt], [gx, gw, gb]) == 0
    cases["conv"] = dict(x=x, w=wt, bias=cb, y=y, gy=gy, gx=gx, gw=gw, gb=gb)
    # batch norm training forward
    bx = seeded((4, 5, 6, 16), 9, -1, 1)
    scale, bb = seeded((1, 1, 1, 16), 10), seeded((1, 1, 1, 16), 11)
    mean, var = seeded((1, 1, 1, 16), 12), seeded((1, 1, 1, 16), 13)
    mean0, var0 = mean.copy(), var.copy()
    by, sm, sis = np.zeros_like(bx), np.zeros_like(mean), np.zeros_like(mean)
    assert ref.run(nnc.CMD_BATCH_NORM_FORWARD(1e-4, 0, 0.9), None, 0, [bx, scale, bb, mean, var], [by, mean, var, sm, sis]) == 0
    cases["bnorm"] = dict(x=bx, scale=scale, bias=bb, mean0=mean0, var0=var0, y=by, mean=mean, var=var, saved_mean=sm, saved_inv_std=sis)
    # float -> half conversion bit patterns (truncating, lib/ccv_util.c:1434-1440)
    f = np.concatenate([seeded((4096,), 14, -70000, 70000), seeded((4096,), 15, -1e-4, 1e-4), np.array([0.0, -0.0, 65504.0, 65520.0, 1e-8, 6.1e-5, 5.9e-8, np.inf, -np.inf], np.float32)]).astype(np.float32)
    cases["f2h"] = dict(f=f, h=ref.float_to_half(f))
    return cases


def cpuref_sdpa():
    """SCALED_DOT_PRODUCT_ATTENTION forward and backward of CPU_REF on the seeded calls of tests/attention_ref.PINS (GQA, causal with
    Sq < Sk and Sq > Sk, Dv != D, 3-d tensors, every mask shape): inputs and outputs, keys prefixed "<case>_"."""
    from ccv_b200 import abi
    from tests import attention_ref as ar
    out = {}
    for i in range(len(ar.PINS)):
        d = ar.pin_inputs(i)
        q, k, v, do, mask = d["q"], d["k"], d["v"], d["do"], d["mask"]
        fwd = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD)
        fwd.info.scaled_dot_product_attention.scale, fwd.info.scaled_dot_product_attention.is_causal = d["scale"], d["causal"]
        o = np.zeros(q.shape[:-1] + v.shape[-1:], np.float32)
        assert ref.run(fwd, None, 0, [q, k, v] + ([mask] if mask is not None else []), [o]) == 0
        rec = dict(q=q, k=k, v=v, o=o)
        if mask is not None:
            rec["mask"] = mask
        if d["backward"]:
            bwd = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD)
            bwd.info.scaled_dot_product_attention.scale, bwd.info.scaled_dot_product_attention.is_causal = d["scale"], d["causal"]
            dq, dk, dv = np.zeros_like(q), np.zeros_like(k), np.zeros_like(v)
            assert ref.run(bwd, None, 0, [do, None, None, q, k, v], [dq, dk, dv]) == 0
            rec.update(do=do, dq=dq, dk=dk, dv=dv)
        out.update(("%d_%s" % (i, name), a) for name, a in rec.items())
    return out


def reference_registry(inc):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_backend_ph as g
    cmds, backends, top, cases, btop, bcases = g.parse_inc(inc)
    return {"source": "lib/nnc/cmd/ccv_nnc_cmd.inc of the reference", "commands": cmds, "backends": backends,
            "cmd_ph": {"top": list(top), "cases": {str(i): list(p) for i, p in sorted(cases.items())}},
            "backend_ph": {"top": list(btop), "cases": {str(i): list(p) for i, p in sorted(bcases.items())}},
            "calls": g.registration_calls(open(inc).read())}


if __name__ == "__main__" and sys.argv[1:2] == ["registry"]:
    import json
    json.dump(reference_registry(sys.argv[2]), open(os.path.join(OUT, "reference_cmd_registry.json"), "w"), indent=0)
elif __name__ == "__main__" and sys.argv[1:2] == ["sdpa"]:
    np.savez(os.path.join(OUT, "cpuref_sdpa.npz"), **cpuref_sdpa())
elif __name__ == "__main__":
    np.savez(os.path.join(OUT, "literal_gemm.npz"), **literal_gemm())
    for name, d in cpuref_cases().items():
        np.savez(os.path.join(OUT, "cpuref_%s.npz" % name), **d)
    np.savez(os.path.join(OUT, "cpuref_sdpa.npz"), **cpuref_sdpa())
    print("wrote", sorted(os.listdir(OUT)))
