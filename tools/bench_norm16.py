"""Timing of the 16-bit LAYER_NORM, RMSNORM and GROUP_NORM (ccv_b200/csrc/sm100_norm.cu) against what a caller had to do before the
norms took 16-bit tensors: DATATYPE_CONVERSION of each 16-bit activation to fp32, the fp32 command, DATATYPE_CONVERSION of the result back.
  rows   LAYER_NORM and RMSNORM forward and backward (with dscale / dbias) at [8192, 4096], bf16 and fp16;
         GROUP_NORM forward and backward, NHWC [2, 64, 64, 320] and [2, 32, 32, 640], 32 groups over (H, W), fp16
  native every tensor of the call in the 16-bit type (what a half-precision model hands these commands)
  conv   16-bit activations converted around the fp32 command, whose parameters, statistics and parameter gradients are fp32
Bytes are the minimum the native call must move, from the shapes: forward reads x and writes y, backward reads g and x and writes h
(2 B per element each; parameters and statistics are left out, they are under 0.1 % here).  bound = bytes / 3.35 TB/s (NVIDIA's
H100 SXM data-sheet HBM3 bandwidth); x bound is the measured time over it.  Everything is timed with CUDA events (3 warm-up runs, then
the best of 3 windows of `--reps` runs); consecutive runs cycle through enough copies of the operands that at least 200 MB is touched
between two uses of one copy.  The card's name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_norm16.py [--reps R] [--json FILE]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_resnet_convs import HBM_GBS, card, time_ms  # noqa: E402
from ccv_b200 import abi, nnc  # noqa: E402
from tests.test_parity_norm_paths import gn_shapes, gnorm_cmd, lnorm_cmd, rms_cmd  # noqa: E402

NHWC = abi.CCV_TENSOR_FORMAT_NHWC
KIND = {"bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
CASES = [("layer_norm", (8192, 4096), "bf16"), ("layer_norm", (8192, 4096), "fp16"), ("rmsnorm", (8192, 4096), "bf16"), ("rmsnorm", (8192, 4096), "fp16"),
         ("group_norm", (2, 64, 64, 320), "fp16"), ("group_norm", (2, 32, 32, 640), "fp16")]


def commands(op, shape):
    """(forward, backward, statistics shape, parameter shape, has a mean, has a bias)"""
    if op == "group_norm":
        rshape, pshape = gn_shapes(shape, 3, 32, (1, 2))
        return gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, 3, 32, 1e-5, 1, (1, 2)), gnorm_cmd(abi.CCV_NNC_GROUP_NORM_BACKWARD, 3, 32, 1e-5, 1, (1, 2)), rshape, pshape, True, True
    rshape, pshape = (shape[0], 1), (1, shape[1])
    if op == "rmsnorm":
        return rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, 1e-5, (1,)), rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, 1e-5, (1,)), rshape, pshape, False, False
    return lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, 1e-5, 1, (1,)), lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 1, (1,)), rshape, pshape, True, True


class Set(object):
    """one copy of every operand: the 16-bit call's (kind dt) and the fp32 call's"""

    def __init__(self, shape, rshape, pshape, dt, rng):
        n = int(np.prod(shape))
        self.owned = []

        def t(s, d, data=None):
            x = nnc.gpu_tensor(list(s), NHWC, d)
            if data is not None:
                x.upload(data.astype(np.float32) if d == abi.CCV_32F else data.astype(np.float16) if d == abi.CCV_16F else
                         (data.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16))
            self.owned.append(x)
            return x
        xs, gs = rng.standard_normal(n).reshape(shape), rng.standard_normal(n).reshape(shape)
        sc, b = 1 + 0.1 * rng.standard_normal(int(np.prod(pshape))).reshape(pshape), 0.1 * rng.standard_normal(int(np.prod(pshape))).reshape(pshape)
        self.n = {k: t(s, dt, v) for k, s, v in (("x", shape, xs), ("g", shape, gs), ("y", shape, None), ("h", shape, None), ("scale", pshape, sc),
                                                 ("bias", pshape, b), ("sm", rshape, None), ("sis", rshape, None), ("ds", pshape, None), ("db", pshape, None))}
        self.f = {k: t(s, abi.CCV_32F, v) for k, s, v in (("x", shape, None), ("g", shape, None), ("y", shape, None), ("h", shape, None), ("scale", pshape, sc),
                                                          ("bias", pshape, b), ("sm", rshape, None), ("sis", rshape, None), ("ds", pshape, None), ("db", pshape, None))}

    def free(self):
        for x in self.owned:
            x.free()


def forward_io(t, mean, bias):
    ins = [t["x"], t["scale"]] + ([t["bias"]] if bias else [])
    outs = [t["y"]] + ([t["sm"]] if mean else []) + [t["sis"]]
    return ins, outs


def backward_io(t, mean, bias):
    if not mean:  # rms norm: g, -, x, scale, -, saved_inv_std -> h, dscale
        return [t["g"], None, t["x"], t["scale"], None, t["sis"]], [t["h"], t["ds"]]
    return [t["g"], None, None, t["x"], t["scale"], None, None, t["sm"], t["sis"]], [t["h"], t["ds"], t["db"]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_norm16.py: no CUDA device")
    stream = nnc.Stream(0)
    rng = np.random.default_rng(0)
    conv = nnc.CMD_DATATYPE_CONVERSION_FORWARD()
    info = card()
    rows = []
    for op, shape, kind in CASES:
        fwd, bwd, rshape, pshape, mean, bias = commands(op, shape)
        n = int(np.prod(shape))
        sets = [Set(shape, rshape, pshape, KIND[kind], rng) for _ in range(max(1, -(-(200 << 20) // (2 * 2 * n))))]
        ex = lambda cmd, i, o: nnc.cmd_exec(cmd, None, 0, i, o, stream)
        for s in sets:  # statistics for the backward, in both forms
            assert ex(conv, [s.n["x"]], [s.f["x"]]) == 0 and ex(conv, [s.n["g"]], [s.f["g"]]) == 0
            assert ex(fwd, *forward_io(s.n, mean, bias)) == 0 and ex(fwd, *forward_io(s.f, mean, bias)) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        for direction in ("forward", "backward"):
            moved = 2 * n * (2 if direction == "forward" else 3)
            turn = [0]

            def native(direction=direction):
                s = sets[turn[0] % len(sets)]
                turn[0] += 1
                return ex(fwd, *forward_io(s.n, mean, bias)) if direction == "forward" else ex(bwd, *backward_io(s.n, mean, bias))

            def converted(direction=direction):
                s = sets[turn[0] % len(sets)]
                turn[0] += 1
                if direction == "forward":
                    return ex(conv, [s.n["x"]], [s.f["x"]]) or ex(fwd, *forward_io(s.f, mean, bias)) or ex(conv, [s.f["y"]], [s.n["y"]])
                return (ex(conv, [s.n["g"]], [s.f["g"]]) or ex(conv, [s.n["x"]], [s.f["x"]]) or ex(bwd, *backward_io(s.f, mean, bias)) or
                        ex(conv, [s.f["h"]], [s.n["h"]]))
            row = dict(op=op, shape="x".join(map(str, shape)), kind=kind, direction=direction, bytes=moved, bound_ms=moved / (HBM_GBS * 1e6))
            for name, fn in (("native", native), ("conv", converted)):
                l0 = nnc.launch_count()
                assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
                stream.wait()
                row[name + "_launches"] = nnc.launch_count() - l0
                row[name + "_ms"] = time_ms(fn, stream, args.reps)
            rows.append(row)
            stream.wait()
        for s in sets:
            s.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-11s %-14s %-5s %-9s %8s %9s %10s %6s %8s %6s %8s %7s" % ("command", "shape", "kind", "direction", "MB", "bound ms", "native ms", "x bnd", "conv ms", "x bnd",
                                                                     "speedup", "launch"))
    for r in rows:
        print("%-11s %-14s %-5s %-9s %8.1f %9.4f %10.4f %6.2f %8.4f %6.2f %8.2f %3d/%-3d" % (
            r["op"], r["shape"], r["kind"], r["direction"], r["bytes"] * 1e-6, r["bound_ms"], r["native_ms"], r["native_ms"] / r["bound_ms"], r["conv_ms"],
            r["conv_ms"] / r["bound_ms"], r["conv_ms"] / r["native_ms"], r["native_launches"], r["conv_launches"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
