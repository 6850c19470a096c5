"""Per-command timing of PAD, MIN / MAX, ARGMAX and REDUCE_ISNAN (ccv_b200/csrc/sm100_ew_more.cu):
  REDUCE_ISNAN  [25.6 M] to [1]          ResNet-50's flat gradient buffer (the fp16 / bf16 loss-scaling overflow check), fp32 and 16-bit
  PAD           [64, 56, 56, 256]         zero and replicate, spatial border 1 (NHWC), forward and backward
  MIN / MAX     [64, 56, 56, 256]         forward and backward (with g)
  ARGMAX        [256, 1000] fp32, [8192, 32000] bf16, [1, 128256] bf16 along the last axis; [64, 1000, 128] fp32 along axis 1
Each command runs through ccv_nnc_cmd_exec and is timed with CUDA events (3 warm-up launches, then the best of 3 windows of `--reps`
launches).  Consecutive launches cycle through enough copies of the operands that what they touch between two uses of one copy is at
least 200 MB, four times the 50 MB L2, so the times are HBM times.  Bytes are what the algorithm reads and writes once; bound = bytes /
3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.  [256, 1000] and [1, 128256] are latency-sized.
The card's name, power limit and maximum SM clock are read in the same run.  With --trace DIR, every command below 0.7 of its bound is
run once more under torch.profiler and its kernel table written to DIR/traces.txt.

usage: python tools/bench_model_addons.py [--reps R] [--json FILE] [--trace DIR]"""
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
from tests.util import pack16  # noqa: E402

ES = {nnc.CCV_32F: 4, nnc.CCV_16BF: 2, nnc.CCV_16F: 2}
NAME = {nnc.CCV_32F: "fp32", nnc.CCV_16BF: "bf16", nnc.CCV_16F: "fp16"}


def _filled(shape, dt, rs):
    t = nnc.gpu_tensor(list(shape), datatype=dt)
    if dt == nnc.CCV_32S:
        return t
    v = rs.rand(*shape).astype(np.float32) * 2 - 1
    t.upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    return t


def workloads():
    """(label, dtype, cmd, input shapes + dtypes, output shapes + dtypes, algorithmic bytes)"""
    act = (64, 56, 56, 256)
    padded = (64, 58, 58, 256)
    n_act, n_pad = int(np.prod(act)), int(np.prod(padded))
    out = []
    for dt in (nnc.CCV_32F, nnc.CCV_16BF):
        es = ES[dt]
        out.append(("isnan [25.6M]->[1]", dt, nnc.CMD_REDUCE_ISNAN_FORWARD(), [((25_600_000,), dt)], [((1,), nnc.CCV_32S)], 25_600_000 * es + 4))
        for t, tn in ((nnc.CCV_NNC_PAD_ZERO, "zero"), (nnc.CCV_NNC_PAD_REPLICATE, "replicate")):
            out.append(("pad %s fwd %s" % (tn, "x".join(map(str, act))), dt, nnc.CMD_PAD_FORWARD(t, (0, 1, 1, 0), (0, 1, 1, 0)), [(act, dt)], [(padded, dt)], (n_act + n_pad) * es))
        out.append(("pad bwd %s" % "x".join(map(str, act)), dt, nnc.CMD_PAD_BACKWARD(nnc.CCV_NNC_PAD_ZERO, (0, 1, 1, 0), (0, 1, 1, 0)), [(padded, dt)], [(act, dt)], 2 * n_act * es))
        for op, f, b in (("min", nnc.CMD_MIN_FORWARD, nnc.CMD_MIN_BACKWARD), ("max", nnc.CMD_MAX_FORWARD, nnc.CMD_MAX_BACKWARD)):
            out.append(("%s fwd %s" % (op, "x".join(map(str, act))), dt, f(), [(act, dt), (act, dt)], [(act, dt)], 3 * n_act * es))
            out.append(("%s bwd %s" % (op, "x".join(map(str, act))), dt, b(), [(act, dt)] * 3, [(act, dt)] * 2, 5 * n_act * es))
    for shape, dt, axis in (((256, 1000), nnc.CCV_32F, 1), ((8192, 32000), nnc.CCV_16BF, 1), ((1, 128256), nnc.CCV_16BF, 1), ((64, 1000, 128), nnc.CCV_32F, 1)):
        bshape = tuple(1 if k == axis else shape[k] for k in range(len(shape)))
        out.append(("argmax %s axis %d" % ("x".join(map(str, shape)), axis), dt, nnc.CMD_ARGMAX_FORWARD(axis), [(shape, dt)], [(bshape, nnc.CCV_32S)],
                    int(np.prod(shape)) * ES[dt] + int(np.prod(bshape)) * 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--trace", default="", help="torch.profiler traces of the commands below 0.7 of their bound go to this directory")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_model_addons.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows, slow = [], []
    for label, dt, cmd, ins, outs, moved in workloads():
        copies = max(1, -(-(200 << 20) // moved))
        owned, ios = [], []
        for _ in range(copies):
            ti = [_filled(s, d, rs) for s, d in ins]
            to = [_filled(s, d, rs) for s, d in outs]
            owned += ti + to
            ios.append((ti, to))
        turn = [0]

        def fn(cmd=cmd, ios=ios, turn=turn):
            i, o = ios[turn[0] % len(ios)]
            turn[0] += 1
            return nnc.cmd_exec(cmd, None, 0, i, o, stream)
        assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
        ms = time_ms(fn, stream, args.reps)
        bound = moved / (HBM_GBS * 1e6)
        rows.append(dict(cmd=label, dtype=NAME[dt], ms=ms, bytes=moved, bound_ms=bound, frac=bound / ms))
        if args.trace and bound / ms < 0.7:
            _trace(args.trace, [(NAME[dt], label, "", fn)], stream)
        stream.wait()
        for t in owned:
            t.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-34s %-5s %9s %8s %9s %6s" % ("command", "type", "ms", "GB/s", "bound ms", "frac"))
    for r in rows:
        print("%-34s %-5s %9.4f %8.0f %9.4f %6.2f" % (r["cmd"], r["dtype"], r["ms"], r["bytes"] / r["ms"] * 1e-6, r["bound_ms"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
