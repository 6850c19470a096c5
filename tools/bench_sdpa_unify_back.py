"""SCALED_DOT_PRODUCT_ATTENTION_BACKWARD through the unify-head projection (inputs[7] = w, [8] = bias, [11] = c; outputs dq, dk, dv, dw,
dbias) against the two commands it equals: GEMM_BACKWARD(transpose_b) on (g, c_flat, w) -> (dc, dw, dbias), then the backward without
weights on dc.  Both run in one process on one stream, alternated round by round, on the forward's own c and log-sum-exp; the first call of
each checks that dq and dw come out bit-identical.  Prints one JSON line per (dtype, D, causal): the median ms per call of each side over
the rounds (CUDA events over --steps calls after --warmup calls) and their ratio.  The first line names the card and its power limit.

    python tools/bench_sdpa_unify_back.py [--steps N] [--warmup W] [--rounds R] [--quick]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ccv_b200 import abi, nnc  # noqa: E402
from tools.bench_sdpa_wide import cmd, to_bf16  # noqa: E402

SHAPES = [  # (dtype, B, S, H, D): 16-bit at a training-sized sequence, fp32 (the composed per-head path) at a shorter one
    ("bf16", 4, 2048, 16, 64), ("bf16", 4, 2048, 16, 128), ("fp16", 4, 2048, 16, 64), ("fp16", 4, 2048, 16, 128),
    ("fp32", 4, 512, 16, 64), ("fp32", 4, 512, 16, 128),
]
DT = {"bf16": abi.CCV_16BF, "fp16": abi.CCV_16F, "fp32": abi.CCV_32F}


def grid(a, dtype):
    if dtype == "bf16":
        return to_bf16(a)
    if dtype == "fp16":
        return a.astype(np.float16)
    return a.astype(np.float32)


def run_shape(dtype, B, S, H, D, causal, a, rng):
    n, dt = H * D, DT[dtype]
    T = lambda dims, t=dt: nnc.gpu_tensor(list(dims), datatype=t)
    q, k, v, c, dq, dk, dv, dc = (T([B, S, H, D]) for _ in range(8))
    g, y, w, dw = T([B, S, n]), T([B, S, n]), T([n, n]), T([n, n])
    bias, db, lse = T([n], abi.CCV_32F), T([n], abi.CCV_32F), T([B, H, S], abi.CCV_32F)
    g2, c2, dc2 = (nnc.gpu_tensor([B * S, n], datatype=dt, ptr=t.data_ptr) for t in (g, c, dc))
    tensors = [q, k, v, c, dq, dk, dv, dc, g, y, w, dw, bias, db, lse, g2, c2, dc2]
    stream = nnc.Stream(0)
    try:
        for t in (q, k, v, g):
            t.upload(grid(rng.random_sample(t.dims).astype(np.float32) * 2 - 1, dtype))
        w.upload(grid((rng.random_sample((n, n)).astype(np.float32) * 2 - 1) / np.sqrt(n), dtype))
        bias.upload(rng.random_sample((n,)).astype(np.float32))
        fwd = cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, D, causal, 0)
        assert nnc.cmd_exec(fwd, None, 0, [q, k, v, None, w, bias], [y, None if dtype == "fp32" else lse, c], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        saved = None if dtype == "fp32" else lse
        bwd = cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, D, causal, 0)
        gemm = nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
        fused = lambda: nnc.cmd_exec(bwd, None, 0, [g, None, None, q, k, v, None, w, bias, y, saved, c], [dq, dk, dv, None, dw, db], stream)

        def sequence():
            rc = nnc.cmd_exec(gemm, None, 0, [g2, c2, w], [dc2, dw, db], stream)
            return rc or nnc.cmd_exec(bwd, None, 0, [dc, None, None, q, k, v, None, None, None, c, saved], [dq, dk, dv], stream)

        results = []
        for run in (fused, sequence):
            assert run() == 0, nnc.lib().ccv_nnc_sm100_last_error()
            stream.wait()
            results.append([t.download().tobytes() for t in (dq, dw)])
        assert results[0] == results[1], "the fused backward differs from the two-command sequence"
        for _ in range(a.warmup):
            fused(), sequence()
        times = {"fused": [], "sequence": []}
        e0, e1 = nnc.Event(), nnc.Event()
        try:
            for _ in range(a.rounds):
                for name, run in (("fused", fused), ("sequence", sequence)):
                    stream.wait()
                    e0.record(stream)
                    for _ in range(a.steps):
                        run()
                    e1.record(stream)
                    stream.wait()
                    times[name].append(e0.elapsed_ms(e1) / a.steps)
        finally:
            e0.free(), e1.free()
        f, s = float(np.median(times["fused"])), float(np.median(times["sequence"]))
        return dict(op="sdpa_unify_back", dtype=dtype, B=B, S=S, H=H, D=D, causal=causal, fused_ms=round(f, 4), sequence_ms=round(s, 4), ratio=round(f / s, 4),
                    fused_ms_rounds=[round(x, 4) for x in times["fused"]], sequence_ms_rounds=[round(x, 4) for x in times["sequence"]])
    finally:
        for t in tensors:
            t.free()
        stream.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="one 16-bit and one fp32 shape")
    a = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_sdpa_unify_back: no CUDA device")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}), flush=True)
    rng = np.random.RandomState(0)
    for shape in ([SHAPES[1], SHAPES[4]] if a.quick else SHAPES):
        for causal in (0, 1):
            print(json.dumps(run_shape(*shape, causal, a, rng)), flush=True)


if __name__ == "__main__":
    main()
