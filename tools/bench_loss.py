"""Per-command timing of the loss commands (ccv_b200/csrc/sm100_loss.cu), forward and backward, in bf16, fp16 and fp32:
  MSE mean      [8, 2^21]        few long rows: the forward splits each row into chunks (two launches)
  sigmoid BCE   [4096, 1000]     multi-label head; the forward writes d = sigmoid(a) too
  BCE           [4096, 1000]
  smooth L1     [2^20, 4]        box regression: packed short rows
Each command runs through ccv_nnc_cmd_exec and is timed with CUDA events (3 warm-up launches, then the best of 3 windows of `--reps`
launches).  Consecutive launches cycle through enough copies of the operands that what they touch between two uses of one copy is at least
200 MB, four times the 50 MB L2, so the times are HBM times and not L2 hits.  Bytes are what a command reads and writes once (a, b, c / g per row, d for sigmoid BCE, h, and the fp32 partials of split
rows written and read back); bound = bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.
The card's name, power limit and maximum SM clock are read in the same run.  With --trace DIR, every command below 0.7 of its bound
is run once more under torch.profiler and its kernel table written to DIR/traces.txt.

usage: python tools/bench_loss.py [--reps R] [--json FILE] [--trace DIR] [--types bf16,fp16,fp32]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_conv_grouped import _trace  # noqa: E402
from bench_resnet_convs import HBM_GBS, card, time_ms  # noqa: E402
from ccv_b200 import nnc  # noqa: E402
from tests import loss_ref as L  # noqa: E402
from tests.util import pack16  # noqa: E402

TYPES = {"bf16": nnc.CCV_16BF, "fp16": nnc.CCV_16F, "fp32": nnc.CCV_32F}
WORKLOADS = [("mse", L.MSE, (8, 2 ** 21)), ("sbce", L.SBCE, (4096, 1000)), ("bce", L.BCE, (4096, 1000)), ("sl1", L.SL1, (2 ** 20, 4))]


def _filled(shape, dt, rs, lo, hi):
    t = nnc.gpu_tensor(list(shape), datatype=dt)
    v = (lo + (hi - lo) * rs.rand(*shape)).astype(np.float32)
    t.upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--trace", default="", help="torch.profiler traces of the commands below 0.7 of their bound go to this directory")
    ap.add_argument("--types", default="bf16,fp16,fp32")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_loss.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows, slow = [], []
    for dtype in args.types.split(","):
        dt = TYPES[dtype]
        es = 4 if dt == nnc.CCV_32F else 2
        for name, op, (batch, count) in WORKLOADS:
            lo, hi = (0.05, 0.95) if op == L.BCE else (-1.0, 1.0)
            x = batch * count * es
            copies = max(1, -(-(200 << 20) // (3 * x)))
            owned, f_ios, b_ios = [], [], []
            for _ in range(copies):
                a, b = _filled((batch, count), dt, rs, lo, hi), _filled((batch, count), dt, rs, 0.0, 1.0)
                g, c = _filled((batch,), dt, rs, 0.5, 1.5), nnc.gpu_tensor([batch], datatype=dt)
                h, d = nnc.gpu_tensor([batch, count], datatype=dt), nnc.gpu_tensor([batch, count], datatype=dt)
                owned += [a, b, g, c, h, d]
                if op == L.BCE:
                    fwd, bwd = nnc.CMD_BINARY_CROSSENTROPY_FORWARD(2.0), nnc.CMD_BINARY_CROSSENTROPY_BACKWARD(2.0)
                    f_io, b_io = ([a, b], [c]), ([g, a, b], [h])
                elif op == L.SBCE:
                    fwd, bwd = nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_FORWARD(2.0), nnc.CMD_SIGMOID_BINARY_CROSSENTROPY_BACKWARD(2.0)
                    f_io, b_io = ([a, b], [c, d]), ([g, None, None, b, None, d], [h])
                elif op == L.MSE:
                    fwd, bwd = nnc.CMD_MSE_FORWARD(nnc.CCV_NNC_MSE_REDUCE_MEAN), nnc.CMD_MSE_BACKWARD(nnc.CCV_NNC_MSE_REDUCE_MEAN)
                    f_io, b_io = ([a, b], [c]), ([g, a, b], [h])
                else:
                    fwd, bwd = nnc.CMD_SMOOTH_L1_FORWARD(1.0), nnc.CMD_SMOOTH_L1_BACKWARD(1.0)
                    f_io, b_io = ([a, b], [c]), ([g, a, b, c], [h])
                f_ios.append(f_io), b_ios.append(b_io)
            ws = L.plan(op, 2.0, batch, count, es)[3]
            moved = {"fwd": 2 * x + batch * es + (x if op == L.SBCE else 0) + 2 * ws,
                     "bwd": 3 * x + (2 if op == L.SL1 else 1) * batch * es}
            for key, cmd, ios in (("fwd", fwd, f_ios), ("bwd", bwd, b_ios)):
                turn = [0]

                def fn(cmd=cmd, ios=ios, turn=turn):
                    ins, outs = ios[turn[0] % len(ios)]
                    turn[0] += 1
                    return nnc.cmd_exec(cmd, None, 0, ins, outs, stream)
                assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
                ms = time_ms(fn, stream, args.reps)
                bound = moved[key] / (HBM_GBS * 1e6)
                rows.append(dict(dtype=dtype, loss=name, cmd=key, shape=[batch, count], ms=ms, bytes=moved[key], bound_ms=bound, frac=bound / ms))
                if args.trace and bound / ms < 0.7:
                    slow.append((dtype, name, key, fn))
            if slow:
                _trace(args.trace, slow, stream)
                slow = []
            stream.wait()
            for t in owned:
                t.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-5s %-5s %-4s %-13s %9s %8s %9s %6s" % ("type", "loss", "cmd", "shape", "ms", "GB/s", "bound ms", "frac"))
    for r in rows:
        print("%-5s %-5s %-4s %-13s %9.4f %8.0f %9.4f %6.2f" % (r["dtype"], r["loss"], r["cmd"], "x".join(map(str, r["shape"])), r["ms"], r["bytes"] / r["ms"] * 1e-6,
                                                               r["bound_ms"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
