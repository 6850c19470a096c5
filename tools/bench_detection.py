"""Per-command timing of ROI_ALIGN and NMS (ccv_b200/csrc/sm100_detect.cu):
  ROI_ALIGN  a [1, 200, 272, 256] map (a detector's stride-4 level at 800 x 1088), 1000 ROIs at 7x7 and 100 ROIs at 14x14, forward and
             backward, bf16 and fp32.  The ROIs overlap (x, y in [0, 0.8), sides in [0.05, 0.4)), the hard case of the gather.
  NMS        m = 1000, 6000, 12000 rows, batches 1 and 8, forward (IoU 0.5; about half the rows survive).
Each command runs through ccv_nnc_cmd_exec and is timed with CUDA events (3 warm-up launches, then the best of 3 windows of `--reps`
launches).  Consecutive launches cycle through enough copies of the operands that what they touch between two uses of one copy is at
least 200 MB, four times the 50 MB L2.  Bytes are what the algorithm must read and write once (ROI_ALIGN: the map or its gradient, the
pooled tensor and the ROIs; NMS: the rows in, the rows and indices out, and the IoU mask written and read once); bound = bytes /
3.35 TB/s (NVIDIA's H100 SXM data-sheet HBM3 bandwidth), frac = bound / measured time.  NMS rows also give the IoU compare count
m (m - 1) / 2 per item.  The card's name, power limit and maximum SM clock are read in the same run.  With --trace DIR, every command
below 0.7 of its bound is run once more under torch.profiler and its kernel table written to DIR/traces.txt.

usage: python tools/bench_detection.py [--reps R] [--json FILE] [--trace DIR]"""
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

ES = {nnc.CCV_32F: 4, nnc.CCV_16BF: 2}
NAME = {nnc.CCV_32F: "fp32", nnc.CCV_16BF: "bf16"}


def _rois(k, rs):
    xy = rs.uniform(0.0, 0.8, (k, 2))
    wh = rs.uniform(0.05, 0.4, (k, 2))
    return np.concatenate([xy, wh], 1).astype(np.float32)


def _boxes(n, m, rs):
    a = np.empty((n, m, 5), np.float32)
    a[..., 0] = rs.rand(n, m)
    a[..., 1:3] = rs.uniform(0, 1000, (n, m, 2))
    a[..., 3:5] = rs.uniform(20, 120, (n, m, 2))
    return a


def workloads(rs):
    """(label, dtype, cmd, [input arrays or (shape, dtype)], [output (shape, dtype)], algorithmic bytes, compares)"""
    out = []
    fmap = (1, 200, 272, 256)
    for dt in (nnc.CCV_16BF, nnc.CCV_32F):
        es = ES[dt]
        for k, pool in ((1000, 7), (100, 14)):
            rois = _rois(k, rs)
            pooled = (k, pool, pool, 256)
            moved = (int(np.prod(fmap)) + int(np.prod(pooled))) * es + rois.nbytes
            out.append(("roi_align fwd %d rois %dx%d" % (k, pool, pool), dt, nnc.CMD_ROI_ALIGN_FORWARD(pool, pool), [(fmap, dt), rois], [(pooled, dt)], moved, 0))
            out.append(("roi_align bwd %d rois %dx%d" % (k, pool, pool), dt, nnc.CMD_ROI_ALIGN_BACKWARD(pool, pool), [(pooled, dt), None, rois], [(fmap, dt)], moved, 0))
    for m in (1000, 6000, 12000):
        for n in (1, 8):
            a = _boxes(n, m, rs)
            words = (m + 63) // 64
            moved = n * (m * 5 * 4 * 2 + m * 4 + 2 * m * words * 8 // 2)
            out.append(("nms fwd m %d batch %d" % (m, n), nnc.CCV_32F, nnc.CMD_NMS_FORWARD(0.5), [a], [((n, m, 5), nnc.CCV_32F), ((n, m), nnc.CCV_32S)], moved, n * m * (m - 1) // 2))
    return out


def _tensor(x, rs):
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        t = nnc.gpu_tensor(list(x.shape), datatype=nnc.CCV_32F)
        t.upload(x)
        return t
    shape, dt = x
    t = nnc.gpu_tensor(list(shape), datatype=dt)
    if dt != nnc.CCV_32S:
        v = rs.rand(*shape).astype(np.float32) * 2 - 1
        t.upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--trace", default="", help="torch.profiler traces of the commands below 0.7 of their bound go to this directory")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_detection.py: no CUDA device")
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    info = card()
    rows = []
    for label, dt, cmd, ins, outs, moved, compares in workloads(rs):
        copies = max(1, -(-(200 << 20) // moved))
        owned, ios = [], []
        for _ in range(copies):
            ti = [_tensor(x, rs) for x in ins]
            to = [_tensor(x, rs) for x in outs]
            owned += [t for t in ti + to if t is not None]
            ios.append((ti, to))
        turn = [0]

        def fn(cmd=cmd, ios=ios, turn=turn):
            i, o = ios[turn[0] % len(ios)]
            turn[0] += 1
            return nnc.cmd_exec(cmd, None, 0, i, o, stream)
        assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
        ms = time_ms(fn, stream, args.reps)
        bound = moved / (HBM_GBS * 1e6)
        rows.append(dict(cmd=label, dtype=NAME[dt], ms=ms, bytes=moved, bound_ms=bound, frac=bound / ms, compares=compares))
        if args.trace and bound / ms < 0.7:
            _trace(args.trace, [(NAME[dt], label, "", fn)], stream)
        stream.wait()
        for t in owned:
            t.free()
    print("card: %s, power limit %s W, SM clock max %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("sm_max_mhz")))
    print("%-34s %-5s %9s %9s %6s %12s" % ("command", "type", "ms", "bound ms", "frac", "G compares/s"))
    for r in rows:
        print("%-34s %-5s %9.4f %9.4f %6.3f %12s" % (r["cmd"], r["dtype"], r["ms"], r["bound_ms"], r["frac"], "%.1f" % (r["compares"] / r["ms"] * 1e-6) if r["compares"] else "-"))
    if args.json:
        d = os.path.dirname(os.path.abspath(args.json))
        os.makedirs(d, exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.json, "w"), indent=1)
    stream.free()


if __name__ == "__main__":
    main()
