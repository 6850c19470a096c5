"""Per-command timing of CONVOLUTION_TRANSPOSE on CCV_NNC_BACKEND_GPU_SM100 for the up-sampling layers of common generators and decoders,
each against its own bound, in TF32 (fp32 tensors) and bf16.

For every shape three commands run through ccv_nnc_cmd_exec, timed with CUDA events (3 warm-up launches, then 3 rounds of a window of
`--reps` launches per command; the best window counts, `spread` is the largest window over the best one):
  tfwd     CONVOLUTION_TRANSPOSE_FORWARD with bias
  mdgrad   CONVOLUTION_BACKWARD with only h out on the mirrored convolution (the same data-gradient kernels without the bias); its windows
           alternate with tfwd's in every round, so that the two are compared under the same conditions
  tback    CONVOLUTION_TRANSPOSE_BACKWARD with da, dw and dbias out
Flops = 2 * N * Hi * Wi * Cin * R * S * Cout / groups per product (tback does two).  Bytes are what a command reads and writes once.  The bound
is max(flops / tensor peak, bytes / HBM peak) with NVIDIA's H100 SXM data-sheet figures (dense TF32 494.5 TFLOP/s, dense BF16 989 TFLOP/s,
HBM3 3.35 TB/s); `frac` = bound / measured time.  The card's name, power limit and SM clocks are printed with the numbers.

usage: python tools/bench_conv_transpose.py [--reps R] [--json FILE]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import ClockSampler  # noqa: E402
from bench_resnet_convs import HBM_GBS, TF32_TFLOPS, card, time_ms  # noqa: E402
from ccv_b200 import nnc  # noqa: E402
from tests.util import to_bf16  # noqa: E402

BF16_TFLOPS = 989.0

# (name, N, Hi, Cin, Cout, k, stride, pad begin, pad end, output_padding)
SHAPES = [
    ("a unet 2x2 s2", 32, 32, 512, 256, 2, 2, 0, 0, 0),
    ("b dcgan 4x4 s2 p1", 64, 32, 256, 128, 4, 2, 1, 1, 0),
    ("c 3x3 s2 p1 op1", 32, 64, 128, 64, 3, 2, 1, 1, 1),
    ("d rgb 7x7 s2 (fallback)", 64, 112, 96, 3, 7, 2, 3, 2, 0),
]


def timed_round(fns, stream, reps, best, worst):
    """one window of `reps` launches per command, in order"""
    for key, fn in fns:
        e0, e1 = nnc.Event(), nnc.Event()
        stream.wait()
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        ms = e0.elapsed_ms(e1) / reps
        best[key] = min(best.get(key, ms), ms)
        worst[key] = max(worst.get(key, ms), ms)
        e0.free(), e1.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_conv_transpose.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for dtype in ("tf32", "bf16"):
        dt = nnc.CCV_32F if dtype == "tf32" else nnc.CCV_16BF
        peak = TF32_TFLOPS if dtype == "tf32" else BF16_TFLOPS
        for name, n, hi, cin, cout, k, st, p0, p1, op in SHAPES:
            ho = (hi - 1) * st + k - p0 - p1 + op
            shapes = dict(a=[n, hi, hi, cin], w=[cin, k, k, cout], y=[n, ho, ho, cout], bias=[cout], g=[n, ho, ho, cout], da=[n, hi, hi, cin], dw=[cin, k, k, cout], db=[cout])
            t = dict((key, nnc.gpu_tensor(s, datatype=dt)) for key, s in shapes.items())
            for key, scale in (("a", 1.0), ("g", 1.0), ("w", 1.0 / np.sqrt(k * k * cin)), ("bias", 1.0)):
                v = ((rs.rand(*shapes[key]).astype(np.float32) - 0.5) * scale)
                t[key].upload(v if dtype == "tf32" else to_bf16(v))
            hint = nnc.hint((st, st), (p0, p0), border_end=(p1, p1))
            tf = nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(1, cout, op, k, k, cin, algorithm=0)
            tb = nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD(1, cout, op, k, k, cin, algorithm=0)
            mb = nnc.CMD_CONVOLUTION_BACKWARD(1, cin, k, k, cout, algorithm=0)
            fns = [("tfwd", lambda: nnc.cmd_exec(tf, hint, 0, [t["a"], t["w"], t["bias"]], [t["y"]], stream)),
                   ("mdgrad", lambda: nnc.cmd_exec(mb, hint, 0, [t["a"], t["g"], t["w"]], [t["y"]], stream)),
                   ("tback", lambda: nnc.cmd_exec(tb, hint, 0, [t["g"], t["a"], t["w"]], [t["da"], t["dw"], t["db"]], stream))]
            for _, fn in fns:
                time_ms(fn, stream, 1)  # warm-up (and a status check) of every command before any window
            best, worst = {}, {}
            for _ in range(3):
                timed_round(fns, stream, args.reps, best, worst)
            flops = 2.0 * n * hi * hi * cin * k * k * cout
            nb = dict((key, tt.nbytes) for key, tt in t.items())
            for key, fl, by in (("tfwd", flops, nb["a"] + nb["w"] + nb["bias"] + nb["y"]), ("mdgrad", flops, nb["a"] + nb["w"] + nb["y"]),
                                ("tback", 2 * flops, nb["g"] + nb["a"] + nb["w"] + nb["da"] + nb["dw"] + nb["db"])):
                bt, bb = fl / (peak * 1e9), by / (HBM_GBS * 1e6)
                ms = best[key]
                rows.append(dict(dtype=dtype, shape=name, cmd=key, N=n, ms=ms, spread=worst[key] / ms, flops=fl, bytes=by, bound_ms=max(bt, bb),
                                 bound_by="tensor" if bt >= bb else "hbm", frac=max(bt, bb) / ms))
            stream.wait()
            for tt in t.values():
                tt.free()
    sampler.stop_flag = True
    sampler.join()
    clocks = sampler.summary()
    print("card: %s, power limit %s W, SM clock median %s MHz (max %s), clock event reasons %s"
          % (info.get("name"), info.get("power_limit_w"), clocks["sm_mhz"], clocks["sm_max_mhz"], clocks["reasons"]))
    print("%-5s %-25s %-7s %3s %9s %7s %8s %8s %9s %7s %6s" % ("type", "shape", "cmd", "N", "ms", "spread", "TFLOP/s", "GB/s", "bound ms", "by", "frac"))
    for r in rows:
        print("%-5s %-25s %-7s %3d %9.3f %7.3f %8.1f %8.0f %9.3f %7s %6.2f" % (r["dtype"], r["shape"], r["cmd"], r["N"], r["ms"], r["spread"], r["flops"] / r["ms"] * 1e-9,
                                                                          r["bytes"] / r["ms"] * 1e-6, r["bound_ms"], r["bound_by"], r["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, clocks=clocks, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
