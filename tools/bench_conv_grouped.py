"""Per-command timing of the bf16 / fp16 grouped convolutions the tensor cores do not take (ccv_b200/csrc/sm100_conv_grouped.cu): every
depthwise layer of EfficientNet-B0 (the reference's bin/nnc/imagenet.c:229-235, 224 x 224 input, N = 128) and the two narrow stages of
ResNeXt-50 32x4d (C / groups = 4 at 56 x 56 and 8 at 28 x 28, N = 64).  The same shapes in fp32 run on the FFMA kernels (one GEMM launch
per group), until now the only way to run them.

Per shape and type three commands run through ccv_nnc_cmd_exec, each timed with CUDA events (3 warm-up launches, then the best of 3
windows of `--reps` launches):
  fwd    CONVOLUTION_FORWARD, no bias (EfficientNet's depthwise layers have none)
  dgrad  CONVOLUTION_BACKWARD with only h out
  wgrad  CONVOLUTION_BACKWARD with only dw out
Flops = 2 * N * P * Q * K * R * S * C / groups (FMAs on the CUDA cores; the pixels of a window in the padding are counted).  Bytes are what a
command reads and writes once.  Bound = max(flops / 67 TFLOP/s, bytes / 3.35 TB/s), NVIDIA's H100 SXM data-sheet fp32 (CUDA-core) rate
and HBM3 bandwidth; `by` says which term is larger and `frac` = bound / measured time.  The card's name and power limit are read in the
same run.  With --trace DIR, every command below 0.3 of its bound is run once more under torch.profiler and its kernel table written to
DIR/traces.txt.

usage: python tools/bench_conv_grouped.py [--reps R] [--json FILE] [--trace DIR] [--types fp16,bf16,fp32]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_resnet_convs import HBM_GBS, card, time_ms  # noqa: E402
from ccv_b200 import nnc  # noqa: E402
from tests.util import to_bf16  # noqa: E402

FP32_TFLOPS = 67.0

# (name, N, H, C, K, groups, k, stride); padding (k - 1) / 2 as imagenet.c:175 and ResNeXt
SHAPES = [
    ("effnet b1 dw3 s1 c32", 128, 112, 32, 32, 32, 3, 1),
    ("effnet b2 dw3 s2 c96", 128, 112, 96, 96, 96, 3, 2),
    ("effnet b2r dw3 s1 c144", 128, 56, 144, 144, 144, 3, 1),
    ("effnet b3 dw5 s2 c144", 128, 56, 144, 144, 144, 5, 2),
    ("effnet b3r dw5 s1 c240", 128, 28, 240, 240, 240, 5, 1),
    ("effnet b4 dw3 s2 c240", 128, 28, 240, 240, 240, 3, 2),
    ("effnet b4r dw3 s1 c480", 128, 14, 480, 480, 480, 3, 1),
    ("effnet b5 dw5 s1 c480", 128, 14, 480, 480, 480, 5, 1),
    ("effnet b5r dw5 s1 c672", 128, 14, 672, 672, 672, 5, 1),
    ("effnet b6 dw5 s2 c672", 128, 14, 672, 672, 672, 5, 2),
    ("effnet b6r dw5 s1 c1152", 128, 7, 1152, 1152, 1152, 5, 1),
    ("effnet b7 dw3 s1 c1152", 128, 7, 1152, 1152, 1152, 3, 1),
    ("resnext s1 g32 cg4", 64, 56, 128, 128, 32, 3, 1),
    ("resnext s2 g32 cg8", 64, 28, 256, 256, 32, 3, 1),
]
TYPES = {"fp16": nnc.CCV_16F, "bf16": nnc.CCV_16BF, "fp32": nnc.CCV_32F}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--trace", default="", help="torch.profiler traces of the commands below 0.3 of their bound go to this directory")
    ap.add_argument("--types", default="fp16,bf16,fp32")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_conv_grouped.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows, slow = [], []
    for dtype in args.types.split(","):
        dt = TYPES[dtype]
        for name, n, h, c, k, groups, r, st in SHAPES:
            pad = (r - 1) // 2
            p = (h + 2 * pad - r) // st + 1
            cg = c // groups
            shapes = dict(x=[n, h, h, c], w=[k, r, r, cg], y=[n, p, p, k])
            t = dict((key, nnc.gpu_tensor(s, datatype=dt)) for key, s in shapes.items())
            t.update(h=nnc.gpu_tensor(shapes["x"], datatype=dt), dw=nnc.gpu_tensor(shapes["w"], datatype=dt))
            for key, scale in (("x", 1.0), ("y", 1.0), ("w", 1.0 / np.sqrt(r * r * cg))):
                v = ((rs.rand(*shapes[key]) - 0.5) * scale).astype(np.float32)
                t[key].upload(v.astype(np.float16) if dtype == "fp16" else to_bf16(v) if dtype == "bf16" else v)
            hint = nnc.hint((st, st), (pad, pad))
            fwd = nnc.CMD_CONVOLUTION_FORWARD(groups, k, r, r, cg)
            back = nnc.CMD_CONVOLUTION_BACKWARD(groups, k, r, r, cg)
            fns = [("fwd", lambda: nnc.cmd_exec(fwd, hint, 0, [t["x"], t["w"]], [t["y"]], stream)),
                   ("dgrad", lambda: nnc.cmd_exec(back, hint, 0, [t["y"], t["x"], t["w"]], [t["h"]], stream)),
                   ("wgrad", lambda: nnc.cmd_exec(back, hint, 0, [t["y"], t["x"], None], [None, t["dw"]], stream))]
            flops = 2.0 * n * p * p * k * r * r * cg
            nb = dict((key, tt.nbytes) for key, tt in t.items())
            for key, fn in fns:
                by = nb["x"] + nb["w"] + nb["y"]
                ms = time_ms(fn, stream, args.reps)
                bt, bb = flops / (FP32_TFLOPS * 1e9), by / (HBM_GBS * 1e6)
                row = dict(dtype=dtype, shape=name, cmd=key, N=n, ms=ms, flops=flops, bytes=by, bound_ms=max(bt, bb), bound_by="fma" if bt >= bb else "hbm",
                           frac=max(bt, bb) / ms)
                rows.append(row)
                if args.trace and row["frac"] < 0.3:
                    slow.append((dtype, name, key, fn))
            if slow and args.trace:
                _trace(args.trace, slow, stream)
                slow = []
            stream.wait()
            for tt in t.values():
                tt.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-5s %-24s %-6s %3s %9s %8s %8s %9s %4s %6s" % ("type", "shape", "cmd", "N", "ms", "TFLOP/s", "GB/s", "bound ms", "by", "frac"))
    for r in rows:
        print("%-5s %-24s %-6s %3d %9.3f %8.2f %8.0f %9.3f %4s %6.2f" % (r["dtype"], r["shape"], r["cmd"], r["N"], r["ms"], r["flops"] / r["ms"] * 1e-9,
                                                                         r["bytes"] / r["ms"] * 1e-6, r["bound_ms"], r["bound_by"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


def _trace(out_dir, slow, stream):
    """three launches of each command under torch.profiler; the kernel table of each goes to out_dir/traces.txt"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "traces.txt"), "a") as f:
        for dtype, name, key, fn in slow:
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    fn()
                stream.wait()
                torch.cuda.synchronize()
            f.write("traced %s %s %s\n%s\n" % (dtype, name, key, prof.key_averages().table(sort_by="cuda_time_total", row_limit=6, max_name_column_width=60)))


if __name__ == "__main__":
    main()
