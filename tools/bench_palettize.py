"""Timing of GEMM_FORWARD with a palettized (CCV_QX) weight on CCV_NNC_BACKEND_GPU_SM100: the dense-layer form c[M, N] = a[M, K] w[N, K]^T
with fp16 activations and a weight palettized with fp16 palettes, for few and many rows.

For every (K, N, q, nib) one weight is made (random index bytes, finite fp16 palettes), and for every M four things are timed with CUDA
events on one stream context (3 warm-up calls, then the best of 5 windows of `--reps` calls):
  fused     the GEMM_FORWARD command on the palettized weight when M <= M_MAX (the fused kernel; "-" above it)
  unfused   the unfused path's launches: the decoder into a dense fp16 weight, then GEMM_FORWARD on it (what the command runs above M_MAX)
  dense     GEMM_FORWARD on the already decoded fp16 weight
  decode    the decoder alone (ccv_nnc_sm100_depalettize)
Bytes are what each must move at least once: fused = packed weight + a + c; unfused = packed weight + 2 x decoded weight (written, then
read) + a + c; dense = decoded weight + a + c.  `bound` is bytes / 3.35 TB/s (NVIDIA's H100 SXM HBM3 figure).  The card's name, power
limit and SM clock are printed with the numbers.

usage: python tools/bench_palettize.py [--reps R] [--json FILE] [--quick]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_resnet_convs import HBM_GBS, card  # noqa: E402
from ccv_b200 import abi, nnc  # noqa: E402
from tests import palette_ref as pr  # noqa: E402
from tests.test_parity_palettize import M_MAX  # noqa: E402

SHAPES_KN = [(4096, 4096), (4096, 11008), (1280, 5120)]
QS = [4, 6, 8]
NIBS = [128, 512]


def packed_weight(N, K, q, nib, seed):
    """Random index bytes with finite fp16 palettes in every block (N * K is a multiple of nib for every shape here)."""
    r = np.random.RandomState(seed)
    count = N * K
    assert count % nib == 0
    blocks, pal = count // nib, (1 << q) * 2
    data = r.randint(0, 256, pr.data_size(count, q, nib, 2), dtype=np.uint8)
    view = data.reshape(blocks, pal + nib * q // 8)
    view[:, :pal] = r.uniform(-0.05, 0.05, (blocks, 1 << q)).astype(np.float16).view(np.uint8).reshape(blocks, pal)
    return data


def best_ms(fn, stream, reps):
    for _ in range(3):
        assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
    best = None
    for _ in range(5):
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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--quick", action="store_true", help="one (K, N), q = 4, nib = 128 only")
    args = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_palettize: no CUDA device")
    info = card()
    print("card:", json.dumps(info), " M_MAX =", M_MAX)
    ms_list = sorted(set([1, 4, 16, M_MAX, 2 * M_MAX, 256, 4096]))
    st = nnc.Stream()
    rows = []
    hdr = "%-5s %-6s %-6s %-2s %-4s | %9s %9s %9s %9s | %8s %8s | %s" % ("M", "K", "N", "q", "nib", "fused us", "unfus us", "dense us", "decode", "bound f", "bound u", "fused/unfused")
    print(hdr)
    for K, N in (SHAPES_KN[:1] if args.quick else SHAPES_KN):
        for q in (QS[:1] if args.quick else QS):
            for nib in (NIBS[:1] if args.quick else NIBS):
                data = packed_weight(N, K, q, nib, K + N + q + nib)
                wq = nnc.gpu_palettized_tensor([N, K], abi.CCV_16F, q, nib)
                wq.upload(data)
                wd = nnc.gpu_tensor([N, K], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_16F)
                assert nnc.depalettize(wq, wd, st) == 0
                dec_ms = best_ms(lambda: nnc.depalettize(wq, wd, st), st, args.reps)
                for M in ms_list:
                    a = nnc.gpu_tensor([M, K], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_16F)
                    a.upload(np.random.RandomState(M).uniform(-1, 1, (M, K)).astype(np.float16))
                    c = nnc.gpu_tensor([M, N], abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_16F)
                    cmd = nnc.CMD_GEMM_FORWARD((0, 0), (0, 1))
                    fused = best_ms(lambda: nnc.cmd_exec(cmd, None, 0, [a, wq], [c], st), st, args.reps) if M <= M_MAX else None
                    dense = best_ms(lambda: nnc.cmd_exec(cmd, None, 0, [a, wd], [c], st), st, args.reps)
                    unfused = best_ms(lambda: nnc.depalettize(wq, wd, st) or nnc.cmd_exec(cmd, None, 0, [a, wd], [c], st), st, args.reps)
                    act = (M * K + M * N) * 2
                    b_fused, b_unfused, b_dense = wq.nbytes + act, wq.nbytes + 2 * N * K * 2 + act, N * K * 2 + act
                    row = dict(M=M, K=K, N=N, q=q, nib=nib, fused_us=None if fused is None else fused * 1e3, unfused_us=unfused * 1e3, dense_us=dense * 1e3,
                               decode_us=dec_ms * 1e3, bytes_fused=b_fused, bytes_unfused=b_unfused, bytes_dense=b_dense,
                               bound_fused_us=b_fused / (HBM_GBS * 1e3), bound_unfused_us=b_unfused / (HBM_GBS * 1e3))
                    rows.append(row)
                    print("%-5d %-6d %-6d %-2d %-4d | %9s %9.2f %9.2f %9.2f | %8.2f %8.2f | %s" % (
                        M, K, N, q, nib, "-" if fused is None else "%.2f" % (fused * 1e3), unfused * 1e3, dense * 1e3, dec_ms * 1e3,
                        row["bound_fused_us"], row["bound_unfused_us"], "-" if fused is None else "%.2fx" % (unfused / fused)))
                    a.free(), c.free()
                wq.free(), wd.free()
    st.free()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, m_max=M_MAX, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
