"""Timing of COMPRESSION_LSSC forward (compress) and backward (decompress) (ccv_b200/csrc/sm100_compress.cu), fp16:
  int-test shapes   the reference's test/int/nnc/compression.tests.c shapes, NCHW: 128x512x7x7, 128x512x14x14, 128x64x113x114,
                    128x256x28x28 (the band form)
  ResNet-50         the fp16 activations ResNet-50's convolutions save for their backward, N = 256, NHWC (the 8-channel vector form)
Bytes are what one command must move, from the shapes: forward reads the original (2 B per element) and writes the compressed tensor
(4 halves per 4x4 block, about 0.5 B per element); backward the reverse.  bound = bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3
bandwidth), frac = bound / measured time.  Everything is timed with CUDA events (3 warm-up runs, then the best of 3 windows of `--reps`
runs); consecutive runs cycle through enough copies of the operands that at least 200 MB is touched between two uses of one copy.  The
card's name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_lssc.py [--reps R] [--json FILE]"""
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

INT_SHAPES = [(128, 512, 7, 7), (128, 512, 14, 14), (128, 64, 113, 114), (128, 256, 28, 28)]
RESNET50 = [(256, 112, 112, 64), (256, 56, 56, 64), (256, 56, 56, 256), (256, 28, 28, 128), (256, 28, 28, 512), (256, 14, 14, 256),
            (256, 14, 14, 1024), (256, 7, 7, 512), (256, 7, 7, 2048)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_lssc.py: no CUDA device")
    stream = nnc.Stream(0)
    rng = np.random.default_rng(0)
    info = card()
    rows = []
    cases = [(s, abi.CCV_TENSOR_FORMAT_NCHW, "NCHW") for s in INT_SHAPES] + [(s, abi.CCV_TENSOR_FORMAT_NHWC, "NHWC") for s in RESNET50]
    for shape, fmt, fname in cases:
        cshape = nnc.lssc_compressed_dims(shape, fmt)
        n, nc = int(np.prod(shape)), int(np.prod(cshape))
        moved = 2 * (n + nc)
        copies = []
        for _ in range(max(1, -(-(200 << 20) // moved))):
            x = nnc.gpu_tensor(list(shape), fmt, abi.CCV_16F).upload(rng.standard_normal(n, dtype=np.float32).astype(np.float16))
            copies.append((x, nnc.gpu_tensor(cshape, fmt, abi.CCV_16F), nnc.gpu_tensor(list(shape), fmt, abi.CCV_16F)))
        for direction in ("forward", "backward"):
            cmd = nnc.CMD_COMPRESSION_LSSC_FORWARD() if direction == "forward" else nnc.CMD_COMPRESSION_LSSC_BACKWARD()
            turn = [0]

            def fn(cmd=cmd, turn=turn, direction=direction):
                x, y, z = copies[turn[0] % len(copies)]
                turn[0] += 1
                return nnc.cmd_exec(cmd, None, 0, [x], [y], stream) if direction == "forward" else nnc.cmd_exec(cmd, None, 0, [y], [z], stream)
            if direction == "forward":  # every copy's compressed tensor holds real data before the backward is timed
                for _ in copies:
                    assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
            l0 = nnc.launch_count()
            assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
            stream.wait()
            launches = nnc.launch_count() - l0
            ms = time_ms(fn, stream, args.reps)
            bound = moved / (HBM_GBS * 1e6)
            rows.append(dict(shape="x".join(map(str, shape)), format=fname, direction=direction, ms=ms, bytes=moved, gbs=moved / ms * 1e-6,
                             bound_ms=bound, frac=bound / ms, launches=launches))
            stream.wait()
        for t in copies:
            for x in t:
                x.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-18s %-5s %-9s %9s %10s %8s %9s %6s %8s" % ("shape", "fmt", "direction", "ms", "MB", "GB/s", "bound ms", "frac", "launches"))
    for r in rows:
        print("%-18s %-5s %-9s %9.4f %10.1f %8.0f %9.4f %6.2f %8d" % (r["shape"], r["format"], r["direction"], r["ms"], r["bytes"] * 1e-6, r["gbs"], r["bound_ms"], r["frac"], r["launches"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
