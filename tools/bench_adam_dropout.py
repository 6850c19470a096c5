"""Timing of ADAMW (ccv_b200/csrc/sm100_ext_ops.cu) and DROPOUT (sm100_ew_more.cu), both streaming element-wise passes:
  ADAMW    25.6 M fp32 parameters, in place (b = a, n = m, u = v), without and with amsgrad: reads g, a, m, v [, vm], writes b, n, u [, um]
           (28 B per element, 36 B with amsgrad)
  DROPOUT  64 M fp32 / bf16 elements, forward (reads a, writes b and one mask byte: 9 / 5 B per element) and backward (reads g and the
           mask, writes h: 9 / 5 B per element)
bound = bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.  Timed with CUDA events (3 warm-up
runs, then the best of 3 windows of `--reps` runs); consecutive runs cycle through enough copies of the operands that at least 200 MB
is touched between two uses of one copy.  The card's name, power limit and maximum SM clock are read in the same run.

--lib PATH times another build of the backend library (for example the parent commit's), so that two builds can be compared in one
session by running this script once per build, alternating.

usage: python tools/bench_adam_dropout.py [--reps R] [--json FILE] [--lib PATH]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ccv_b200 import nnc  # noqa: E402
from tests.util import pack16  # noqa: E402

ES = {nnc.CCV_32F: 4, nnc.CCV_16BF: 2}
NAME = {nnc.CCV_32F: "fp32", nnc.CCV_16BF: "bf16"}


def _filled(n, dt, rs, lo, hi):
    t = nnc.gpu_tensor([n], datatype=dt)
    v = (rs.rand(n).astype(np.float32) * (hi - lo) + lo).astype(np.float32)
    t.upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    return t


def _copies(moved):
    return max(1, -(-(200 << 20) // moved))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--lib", default="", help="time this build of libccv_nnc_sm100.so instead of the tree's")
    args = ap.parse_args()
    if args.lib:
        nnc.LIB_PATH = os.path.abspath(args.lib)
    from bench_resnet_convs import HBM_GBS, card, time_ms
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_adam_dropout.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows = []

    def record(label, dt, fn, moved):
        ms = time_ms(fn, stream, args.reps)
        bound = moved / (HBM_GBS * 1e6)
        rows.append(dict(row=label, dtype=NAME[dt], ms=ms, bytes=moved, bound_ms=bound, frac=bound / ms))
        stream.wait()

    n = 25_600_000
    for amsgrad in (0, 1):
        k = 4 + amsgrad
        moved = (2 * k - 1) * 4 * n
        copies = [[_filled(n, nnc.CCV_32F, rs, -1, 1), _filled(n, nnc.CCV_32F, rs, -1, 1), _filled(n, nnc.CCV_32F, rs, -0.1, 0.1)] +
                  [_filled(n, nnc.CCV_32F, rs, 0, 0.01) for _ in range(1 + amsgrad)] for _ in range(_copies(moved))]
        cmd = nnc.CMD_ADAMW_FORWARD(10, 0.001, 0.9, 0.999, 0.01, 1e-8, amsgrad)
        turn = [0]

        def fn(copies=copies, turn=turn, cmd=cmd):
            q = copies[turn[0] % len(copies)]
            turn[0] += 1
            return nnc.cmd_exec(cmd, None, 0, q, q[1:], stream)
        record("adamw 25.6M%s" % (" amsgrad" if amsgrad else ""), nnc.CCV_32F, fn, moved)
        for q in copies:
            for t in q:
                t.free()
    n = 64 << 20
    for dt in (nnc.CCV_32F, nnc.CCV_16BF):
        moved = (2 * ES[dt] + 1) * n
        copies = [(_filled(n, dt, rs, -1, 1), nnc.gpu_tensor([n], datatype=dt), nnc.gpu_tensor([n], datatype=nnc.CCV_8U)) for _ in range(_copies(moved))]
        fwd, bwd = nnc.CMD_DROPOUT_FORWARD(0.15), nnc.CMD_DROPOUT_BACKWARD(0.15)
        for label, cmd in (("dropout forward 64M", fwd), ("dropout backward 64M", bwd)):
            turn = [0]

            def fn(copies=copies, turn=turn, cmd=cmd, forward=cmd is fwd):
                a, b, mask = copies[turn[0] % len(copies)]
                turn[0] += 1
                if forward:
                    return nnc.cmd_exec(cmd, None, 0, [a], [b, mask], stream)
                return nnc.cmd_exec(cmd, None, 0, [a, None, None, None, mask], [b], stream)
            record(label, dt, fn, moved)
        for q in copies:
            for t in q:
                t.free()
    print("library: %s" % nnc.LIB_PATH)
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-28s %-5s %9s %8s %9s %6s" % ("row", "dtype", "ms", "GB/s", "bound ms", "frac"))
    for r in rows:
        print("%-28s %-5s %9.4f %8.0f %9.4f %6.2f" % (r["row"], r["dtype"], r["ms"], r["bytes"] / r["ms"] * 1e-6, r["bound_ms"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, library=nnc.LIB_PATH, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
