"""Per-command timing of CMUL (ccv_b200/csrc/sm100_ew_more.cu) on the rotary position embedding of a Llama-7B-like layer: q [4, 4096, 32, 128]
and, with grouped-query attention, k [4, 4096, 8, 128], each multiplied by the [1, 4096, 1, 128] cos / sin table, in bf16, fp16 and fp32.

Per tensor and type, commands run through ccv_nnc_cmd_exec, each timed with CUDA events (3 warm-up launches, then the best of 3 windows of
`--reps` launches):
  fwd        CMUL_FORWARD into a contiguous output
  fwd-inpl   CMUL_FORWARD in place on the q slice of a packed [4, 4096, (32 + 2 * 8) * 128] QKV projection (q only)
  bwd-da     CMUL_BACKWARD (g, -, table) -> dq / dk
  bwd-da-db  CMUL_BACKWARD (g, x, table) -> (dx, dtable): the table's gradient is summed over batch and heads
Bytes are what a command reads and writes once; bound = bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound /
measured time.  The card's name, power limit and maximum SM clock are read in the same run.  With --trace DIR, every command below 0.7 of its
bound is run once more under torch.profiler and its kernel table written to DIR/traces.txt.

usage: python tools/bench_cmul.py [--reps R] [--json FILE] [--trace DIR] [--types bf16,fp16,fp32]"""
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

B, S, HQ, HK, D = 4, 4096, 32, 8, 128
TYPES = {"bf16": nnc.CCV_16BF, "fp16": nnc.CCV_16F, "fp32": nnc.CCV_32F}


def _filled(shape, dt, rs):
    t = nnc.gpu_tensor(list(shape), datatype=dt)
    v = (rs.rand(*shape).astype(np.float32) * 2 - 1)
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
        raise SystemExit("bench_cmul.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    fwd, bwd = nnc.CMD_CMUL_FORWARD(), nnc.CMD_CMUL_BACKWARD()
    rows, slow = [], []
    for dtype in args.types.split(","):
        dt = TYPES[dtype]
        table = _filled((1, S, 1, D), dt, rs)
        for name, heads in (("q", HQ), ("k", HK)):
            shape = (B, S, heads, D)
            x, g = _filled(shape, dt, rs), _filled(shape, dt, rs)
            c, dx, dtab = nnc.gpu_tensor(list(shape), datatype=dt), nnc.gpu_tensor(list(shape), datatype=dt), nnc.gpu_tensor([1, S, 1, D], datatype=dt)
            owned = [x, g, c, dx, dtab]
            fns = [("fwd", lambda: nnc.cmd_exec(fwd, None, 0, [x, table], [c], stream)),
                   ("bwd-da", lambda: nnc.cmd_exec(bwd, None, 0, [g, None, table], [dx], stream)),
                   ("bwd-da-db", lambda: nnc.cmd_exec(bwd, None, 0, [g, x, table], [dx, dtab], stream))]
            if name == "q":
                width = (HQ + 2 * HK) * D
                packed = _filled((B, S, width), dt, rs)
                qv = nnc.tensor_view_new(packed, list(shape), [0] * 12, [S * width, width, D, 1] + [0] * 8)
                owned += [qv, packed]
                fns.insert(1, ("fwd-inpl", lambda: nnc.cmd_exec(fwd, None, 0, [qv, table], [qv], stream)))
            xb, tb = x.nbytes, table.nbytes
            moved = {"fwd": 2 * xb + tb, "fwd-inpl": 2 * xb + tb, "bwd-da": 2 * xb + tb, "bwd-da-db": 3 * xb + 2 * tb}
            for key, fn in fns:
                ms = time_ms(fn, stream, args.reps)
                bound = moved[key] / (HBM_GBS * 1e6)
                rows.append(dict(dtype=dtype, tensor=name, cmd=key, shape=list(shape), ms=ms, bytes=moved[key], bound_ms=bound, frac=bound / ms))
                if args.trace and bound / ms < 0.7:
                    slow.append((dtype, name, key, fn))
            if slow:
                _trace(args.trace, slow, stream)
                slow = []
            stream.wait()
            for t in owned:
                t.free()
        table.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-5s %-3s %-10s %-18s %9s %8s %9s %6s" % ("type", "x", "cmd", "shape", "ms", "GB/s", "bound ms", "frac"))
    for r in rows:
        print("%-5s %-3s %-10s %-18s %9.3f %8.0f %9.3f %6.2f" % (r["dtype"], r["tensor"], r["cmd"], "x".join(map(str, r["shape"])), r["ms"], r["bytes"] / r["ms"] * 1e-6,
                                                               r["bound_ms"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
