"""Timing of the LAMB and RMSPROP optimizers (ccv_b200/csrc/sm100_optim.cu):
  single commands   1 M and 25.6 M elements: fp32 state with an fp32 gradient, fp32 state with a bf16 gradient, bf16 state and gradient
  ResNet-50         the 161 parameter tensors of ResNet-50 (25 557 032 elements, fp32), weights with decay and the rest without,
                    in place, as per-command graph nodes and as the fused graph (ccv_nnc_sm100_graph_fuse: one multi-tensor node per
                    decay group); time and launches per step
Bytes per element are what the algorithm reads and writes once per step, with G and S the gradient's and the state's element sizes:
  LAMB     2 (G + 3 S) + 3 S   pass 1 reads g, a, m, v; pass 3 reads them again and writes b, n, u (44 B with fp32 everything)
  RMSPROP  G + 3 S + 3 S       one streaming pass (28 B with fp32 everything)
bound = bytes / 3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.  Everything is timed with CUDA
events (3 warm-up runs, then the best of 3 windows of `--reps` runs); consecutive runs cycle through enough copies of the operands that
at least 200 MB is touched between two uses of one copy.  The card's name, power limit and maximum SM clock are read in the same run.
With --trace DIR, every row below 0.7 of its bound is run once more under torch.profiler and its kernel table written to DIR/traces.txt.

usage: python tools/bench_optimizers.py [--reps R] [--json FILE] [--trace DIR]"""
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
from tests.test_parity_feeder_paths import _resnet50_param_counts  # noqa: E402
from tests.util import pack16  # noqa: E402

ES = {nnc.CCV_32F: 4, nnc.CCV_16BF: 2}
NAME = {nnc.CCV_32F: "fp32", nnc.CCV_16BF: "bf16"}


def cmd_of(which, decay=0.01):
    if which == "lamb":
        return nnc.CMD_LAMB_FORWARD(10, 0.01, 0.9, 0.999, decay, 1e-6)
    return nnc.CMD_RMSPROP_FORWARD(0.001, decay, 0.9, 0.9, 1e-8)


def bytes_per_elem(which, gdt, sdt):
    g, s = ES[gdt], ES[sdt]
    return 2 * (g + 3 * s) + 3 * s if which == "lamb" else g + 6 * s


def _filled(n, dt, rs, lo, hi):
    t = nnc.gpu_tensor([n], datatype=dt)
    v = (rs.rand(n).astype(np.float32) * (hi - lo) + lo).astype(np.float32)
    t.upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    return t


def _quad(n, gdt, sdt, rs):
    """g, a, m, v (v >= 0)"""
    return [_filled(n, gdt, rs, -1, 1), _filled(n, sdt, rs, -1, 1), _filled(n, sdt, rs, -0.1, 0.1), _filled(n, sdt, rs, 0, 0.01)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--trace", default="", help="torch.profiler traces of the rows below 0.7 of their bound go to this directory")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_optimizers.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows = []

    def record(label, gdt, sdt, fn, moved, launches, nodes=1):
        assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
        ms = time_ms(fn, stream, args.reps)
        bound = moved / (HBM_GBS * 1e6)
        rows.append(dict(row=label, grad=NAME[gdt], state=NAME[sdt], ms=ms, bytes=moved, bound_ms=bound, frac=bound / ms, launches=launches, nodes=nodes))
        if args.trace and bound / ms < 0.7:
            _trace(args.trace, [(NAME[sdt], label, NAME[gdt], fn)], stream)
        stream.wait()

    # single commands, in place (b = a, n = m, u = v) as models call them
    for which in ("lamb", "rmsprop"):
        for n in (1 << 20, 25_600_000):
            for gdt, sdt in ((nnc.CCV_32F, nnc.CCV_32F), (nnc.CCV_16BF, nnc.CCV_32F), (nnc.CCV_16BF, nnc.CCV_16BF)):
                moved = bytes_per_elem(which, gdt, sdt) * n
                copies = [_quad(n, gdt, sdt, rs) for _ in range(max(1, -(-(200 << 20) // moved)))]
                turn, cmd = [0], cmd_of(which)

                def fn(copies=copies, turn=turn, cmd=cmd):
                    g, a, m, v = copies[turn[0] % len(copies)]
                    turn[0] += 1
                    return nnc.cmd_exec(cmd, None, 0, [g, a, m, v], [a, m, v], stream)
                l0 = nnc.launch_count()
                fn()
                stream.wait()
                record("%s %s" % (which, "1M" if n == 1 << 20 else "25.6M"), gdt, sdt, fn, moved, nnc.launch_count() - l0)
                for q in copies:
                    for t in q:
                        t.free()
    # ResNet-50's parameter set, one step per graph run (1.1 GB touched per LAMB step: one copy is enough)
    counts = _resnet50_param_counts()
    for which in ("lamb", "rmsprop"):
        quads = [_quad(c, nnc.CCV_32F, nnc.CCV_32F, rs) for c in counts]
        for fuse in (False, True):
            gr = nnc.Graph()
            for c, (g, a, m, v) in zip(counts, quads):
                gr.exec_new(cmd_of(which, 0.01 if c > 4096 else 0.0), None, 0, [g, a, m, v], [a, m, v])
            if fuse:
                gr.fuse()
            l0 = nnc.launch_count()
            assert gr.run(stream) == 0
            stream.wait()
            launches = nnc.launch_count() - l0
            record("%s resnet50 161 tensors %s" % (which, "fused" if fuse else "per command"), nnc.CCV_32F, nnc.CCV_32F, lambda gr=gr: gr.run(stream),
                   bytes_per_elem(which, nnc.CCV_32F, nnc.CCV_32F) * sum(counts), launches, len(gr))
            gr.free()
        for q in quads:
            for t in q:
                t.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-40s %-5s %-5s %9s %8s %9s %6s %8s %5s" % ("row", "grad", "state", "ms", "GB/s", "bound ms", "frac", "launches", "nodes"))
    for r in rows:
        print("%-40s %-5s %-5s %9.4f %8.0f %9.4f %6.2f %8d %5d" % (r["row"], r["grad"], r["state"], r["ms"], r["bytes"] / r["ms"] * 1e-6, r["bound_ms"], r["frac"], r["launches"], r["nodes"]))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
