"""Per-command timing of every distinct ResNet-50 v1d convolution of bench.py's headline step (N=256, 224x224, fp32 NHWC) on
CCV_NNC_BACKEND_GPU_SM100, each against its own bound.

For every shape three commands run through ccv_nnc_cmd_exec, each timed with CUDA events (best of 3 windows of `--reps` launches
after 3 warm-up launches):
  fwd    CONVOLUTION_FORWARD                      (the plain command; in the step a forward followed by a batch norm also emits its
                                                   statistics, which walks the M tiles differently)
  dgrad  CONVOLUTION_BACKWARD with only h out      (skipped for the stem's first convolution: the step has no image gradient)
  wgrad  CONVOLUTION_BACKWARD with only dw out
Flops are bench.py's node_cost figure, 2 * N * P * Q * K * R * S * C.  Bytes are what the command reads and writes once: fwd x + w + y,
dgrad g + w + h, wgrad g + x + dw.  The bound is max(flops / tensor peak, bytes / HBM peak) with NVIDIA's H100 SXM data-sheet peaks
(dense TF32 494.5 TFLOP/s, a third of it for 3xTF32; HBM3 3.35 TB/s); `frac` = bound / measured time.  The summary weighs each shape by
how often the step runs it.  The card's name, power limit and SM clocks are printed with the numbers.

usage: python tools/bench_resnet_convs.py [--3xtf32] [--reps R] [--only fwd,dgrad,wgrad] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402
from ccv_b200 import nnc  # noqa: E402

TF32_TFLOPS = 989.0 / 2.0  # H100 SXM data sheet: dense TF32 is half the dense BF16 rate
HBM_GBS = 3350.0


def resnet50_convs(n=256, image=224):
    """(name, H, cin, cout, k, stride, need_dx) of every convolution of ccv_b200.resnet50.Net, in step order"""
    convs, h = [], image
    for i, (cin, cout, st) in enumerate(((3, 32, 2), (32, 32, 1), (32, 64, 1))):
        convs.append(("stem.conv%d" % i, h, cin, cout, 3, st, i > 0))
        h = (h + 2 - 3) // st + 1
    h = (h + 2 - 3) // 2 + 1  # max pool 3x3 / 2
    c = 64
    for li, (f, stride, blocks) in enumerate(((64, 1, 3), (128, 2, 4), (256, 2, 6), (512, 2, 3))):
        for bi in range(blocks):
            s = stride if bi == 0 else 1
            name = "layer%d.block%d" % (li + 1, bi)
            if bi == 0:
                convs.append((name + ".conv0", h // s, c, f * 4, 1, 1, True))  # projection behind a 2x2 / 2 average pool
            convs.append((name + ".conv1", h, c, f, 1, 1, True))
            convs.append((name + ".conv2", h, f, f, 3, s, True))
            h2 = (h + 2 - 3) // s + 1
            convs.append((name + ".conv3", h2, f, f * 4, 1, 1, True))
            h, c = h2, f * 4
    return convs


def distinct_shapes(convs):
    """[(shape, count, first name)] with shape = (H, cin, cout, k, stride, need_dx)"""
    seen = {}
    for name, *shape in convs:
        key = tuple(shape)
        if key not in seen:
            seen[key] = [0, name]
        seen[key][0] += 1
    return [(k, v[0], v[1]) for k, v in seen.items()]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], timeout=10).decode().strip().split(",")
        return dict(name=out[0].strip(), power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except Exception as e:  # noqa: BLE001 -- the timing is still worth printing
        return dict(unavailable=repr(e)[:200])


def time_ms(fn, stream, reps):
    for _ in range(3):
        assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
    best = None
    for _ in range(3):
        e0, e1 = nnc.Event(), nnc.Event()
        stream.wait()
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        ms = e0.elapsed_ms(e1) / reps
        best = ms if best is None else min(best, ms)
        e0.free(), e1.free()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--3xtf32", dest="x3", action="store_true", help="algorithm 1 (3xTF32) instead of 0 (TF32)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--only", default="fwd,dgrad,wgrad", help="comma-separated commands to time (the summary covers only these)")
    ap.add_argument("--json", default="", help="also write the rows and the summary to this file")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_resnet_convs.py: no CUDA device")
    algo = 1 if args.x3 else 0
    peak = TF32_TFLOPS / (3.0 if args.x3 else 1.0)
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    n = args.batch
    info = card()
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for (h, cin, cout, k, st, need_dx), count, name in distinct_shapes(resnet50_convs(n)):
        pad = k // 2
        p = (h + 2 * pad - k) // st + 1
        x, w, y, g, dx, dw = (nnc.gpu_tensor(s) for s in ([n, h, h, cin], [cout, k, k, cin], [n, p, p, cout], [n, p, p, cout], [n, h, h, cin], [cout, k, k, cin]))
        for t in (x, g):
            t.upload(rs.rand(*t.dims).astype(np.float32) - 0.5)
        w.upload((rs.rand(cout, k, k, cin).astype(np.float32) - 0.5) / np.sqrt(k * k * cin))
        hint = nnc.hint((st, st), (pad, pad))
        fwd, bwd = nnc.CMD_CONVOLUTION_FORWARD(1, cout, k, k, cin, algorithm=algo), nnc.CMD_CONVOLUTION_BACKWARD(1, cout, k, k, cin, algorithm=algo)
        flops = 2.0 * n * p * p * cout * cin * k * k
        cmds = [("fwd", lambda: nnc.cmd_exec(fwd, hint, 0, [x, w], [y], stream), x.nbytes + w.nbytes + y.nbytes)]
        if need_dx:
            cmds.append(("dgrad", lambda: nnc.cmd_exec(bwd, hint, 0, [g, x, w], [dx], stream), g.nbytes + w.nbytes + dx.nbytes))
        cmds.append(("wgrad", lambda: nnc.cmd_exec(bwd, hint, 0, [g, x, w], [None, dw], stream), g.nbytes + x.nbytes + dw.nbytes))
        for kind, fn, nbytes in cmds:
            if kind not in args.only.split(","):
                continue
            ms = time_ms(fn, stream, args.reps)
            bound = max(flops / (peak * 1e9), nbytes / (HBM_GBS * 1e6))
            rows.append(dict(kind=kind, name=name, count=count, shape="%dx%d %d->%d /%d @%d" % (k, k, cin, cout, st, h), ms=ms, flops=flops, bytes=nbytes, bound_ms=bound,
                             bound_by="tensor" if flops / (peak * 1e9) >= nbytes / (HBM_GBS * 1e6) else "hbm", frac=bound / ms))
        stream.wait()
        for t in (x, w, y, g, dx, dw):
            t.free()
    sampler.stop_flag = True
    sampler.join()
    clocks = sampler.summary()
    print("card: %s, power limit %s W, SM clock median %s MHz (max %s), clock event reasons %s; algorithm %d (%s), N=%d"
          % (info.get("name"), info.get("power_limit_w"), clocks["sm_mhz"], clocks["sm_max_mhz"], clocks["reasons"], algo, "3xTF32" if algo else "TF32", n))
    print("%-6s %-24s %-22s %3s %9s %8s %8s %9s %7s %6s" % ("cmd", "first layer", "shape", "x", "ms", "TFLOP/s", "GB/s", "bound ms", "by", "frac"))
    for r in rows:
        print("%-6s %-24s %-22s %3d %9.3f %8.1f %8.0f %9.3f %7s %6.2f" % (r["kind"], r["name"], r["shape"], r["count"], r["ms"], r["flops"] / r["ms"] * 1e-9, r["bytes"] / r["ms"] * 1e-6,
                                                                        r["bound_ms"], r["bound_by"], r["frac"]))
    summary = {}
    for r in rows:
        s = summary.setdefault(r["kind"], dict(commands=0, ms=0.0, bound_ms=0.0))
        s["commands"] += r["count"]
        s["ms"] += r["count"] * r["ms"]
        s["bound_ms"] += r["count"] * r["bound_ms"]
    total = dict(commands=sum(s["commands"] for s in summary.values()), ms=sum(s["ms"] for s in summary.values()), bound_ms=sum(s["bound_ms"] for s in summary.values()))
    print("per step (each shape weighted by its count):")
    for kind, s in list(summary.items()) + [("all", total)]:
        s["frac"] = s["bound_ms"] / s["ms"]
        print("  %-6s %3d commands  %8.2f ms  bound %7.2f ms  frac %.2f" % (kind, s["commands"], s["ms"], s["bound_ms"], s["frac"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, clocks=clocks, algorithm=algo, batch=n, rows=rows, summary=summary, total=total), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
