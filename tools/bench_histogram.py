"""Timing of HISTOGRAM_FORWARD with statistics (ccv_b200/csrc/sm100_histogram.cu): each type (EVEN 100 bins, LOG with the reference's
defaults, BINS with 100 bounds) in fp32 and bf16 on ResNet-50's flat parameter buffer (25 557 032 values) and on a 256x56x56x256 bf16
activation, plus the one-bin case (every value equal).  Bytes are one read of a (the counts and statistics are a few KB); bound =
bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.  Timed with CUDA events (3 warm-up
runs, then the best of 3 windows of `--reps` runs).  The card's name, power limit and maximum SM clock are read in the same run.

usage: python tools/bench_histogram.py [--reps R] [--json FILE]"""
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
from tests.util import pack16  # noqa: E402

RESNET50_PARAMS = 25557032
ACTIVATION = 256 * 56 * 56 * 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_histogram.py: no CUDA device")
    stream = nnc.Stream(0)
    rng = np.random.default_rng(0)
    info = card()
    bounds_host = np.sort(rng.uniform(-0.2, 0.2, 100)).astype(np.float32)
    bounds = nnc.gpu_tensor([100]).upload(bounds_host)
    cmds = {"even": nnc.CMD_HISTOGRAM_EVEN(100, -0.2, 0.2), "log": nnc.CMD_HISTOGRAM_LOG(), "bins": nnc.CMD_HISTOGRAM_BINS()}
    cases = [("resnet50 params", RESNET50_PARAMS, abi.CCV_32F, "fp32"), ("resnet50 params", RESNET50_PARAMS, abi.CCV_16BF, "bf16"),
             ("256x56x56x256", ACTIVATION, abi.CCV_16BF, "bf16")]
    rows = []
    for name, n, kind, kname in cases:
        for dist in ("normal", "one bin"):
            x = rng.standard_normal(n, dtype=np.float32) * np.float32(0.05) if dist == "normal" else np.full(n, 0.05, np.float32)
            a = nnc.gpu_tensor([n], abi.CCV_TENSOR_FORMAT_NHWC, kind).upload(x if kind == abi.CCV_32F else pack16(x, kind))
            for typ, cmd in cmds.items():
                if dist == "one bin" and typ != "even":
                    continue
                nb = nnc.histogram_bin_count(cmd, 100)
                b = nnc.gpu_tensor([nb], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_32S)
                s = nnc.gpu_tensor([4])
                ins = [a, bounds] if typ == "bins" else [a]

                def fn(cmd=cmd, ins=ins, b=b, s=s):
                    return nnc.cmd_exec(cmd, None, 0, ins, [b, s], stream)
                l0 = nnc.launch_count()
                assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
                stream.wait()
                launches = nnc.launch_count() - l0
                ms = time_ms(fn, stream, args.reps)
                moved = n * abi.DTYPE_SIZE[kind]
                bound = moved / (HBM_GBS * 1e6)
                rows.append(dict(tensor=name, dtype=kname, data=dist, type=typ, ms=ms, us=ms * 1e3, bytes=moved, gbs=moved / ms * 1e-6,
                                 bound_ms=bound, frac=bound / ms, launches=launches))
                b.free(), s.free()
            a.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-16s %-5s %-8s %-5s %9s %9s %8s %6s %8s" % ("tensor", "dtype", "data", "type", "us", "MB", "GB/s", "frac", "launches"))
    for r in rows:
        print("%-16s %-5s %-8s %-5s %9.1f %9.1f %8.0f %6.2f %8d" % (r["tensor"], r["dtype"], r["data"], r["type"], r["us"], r["bytes"] * 1e-6, r["gbs"], r["frac"], r["launches"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    bounds.free()
    stream.free()


if __name__ == "__main__":
    main()
