"""Wide-head SCALED_DOT_PRODUCT_ATTENTION (bf16, 128 < D <= 256) under algorithm 0 (the fp32 functional form) and algorithm 1 (the wide
flash kernels of sm100_fmha_wide.cu), forward and backward, through the C ABI.  Prints one JSON line per (shape, causal, direction,
algorithm): ms per call (CUDA events over the timed calls, after warm-up calls), TFLOP/s of the algorithmic count (forward 4 B H Sq Sk D,
backward 10 B H Sq Sk D, halved when causal) and the device memory the call's stream workspace took (cudaMemGetInfo before and after the
first call on a fresh stream).  The backward passes the forward's O and log-sum-exp, as a training graph does.  The first line names the
card, its power limit and its SM clocks.

    python tools/bench_sdpa_wide.py [--steps N] [--warmup W] [--quick]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ccv_b200 import abi, nnc  # noqa: E402

SHAPES = [  # (B, H, S, D)
    (4, 16, 4096, 160), (4, 16, 4096, 256),
    (2, 8, 1024, 160),   # Stable Diffusion 1.x's widest attention
]


def to_bf16(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


_cudart = None


def free_bytes():
    """free device memory (cudaMemGetInfo)"""
    global _cudart
    if _cudart is None:
        for name in ("libcudart.so", "libcudart.so.12", os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "lib64", "libcudart.so")):
            try:
                _cudart = ctypes.CDLL(name)
                break
            except OSError:
                continue
    if _cudart is None:
        import torch
        return torch.cuda.mem_get_info()[0]
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    assert _cudart.cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total)) == 0
    return free.value


def cmd(cmd_id, D, causal, algorithm):
    c = nnc._simple(cmd_id, algorithm=algorithm)
    c.info.scaled_dot_product_attention.scale = float(1.0 / np.sqrt(D))
    c.info.scaled_dot_product_attention.is_causal = causal
    return c


def timed(run, steps, warmup):
    """(ms per call, workspace bytes): the first call on a fresh stream measures the workspace it grows"""
    stream = nnc.Stream(0)
    try:
        stream.wait()
        f0 = free_bytes()
        assert run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        ws = max(0, f0 - free_bytes())
        for _ in range(warmup):
            run(stream)
        e0, e1 = nnc.Event(), nnc.Event()
        stream.wait()
        e0.record(stream)
        for _ in range(steps):
            run(stream)
        e1.record(stream)
        return e0.elapsed_ms(e1) / steps, ws
    finally:
        stream.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true", help="the small shape only")
    a = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_sdpa_wide: no CUDA device")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}), flush=True)
    rng = np.random.RandomState(0)
    for B, H, S, D in (SHAPES[2:] if a.quick else SHAPES):
        ts = [nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF) for _ in range(8)]  # q k v do o dq dk dv
        for t in ts[:4]:
            t.upload(to_bf16(rng.random_sample((B, S, H, D)).astype(np.float32) * 2 - 1))
        lse = nnc.gpu_tensor([B, H, S])
        q, k, v, do, o, dq, dk, dv = ts
        try:
            for causal in (0, 1):
                flops = 4.0 * B * H * S * S * D * (0.5 if causal else 1.0)
                for algo in (0, 1):
                    fwd = cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, D, causal, algo)
                    bwd = cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, D, causal, algo)
                    outs = [o] + ([lse] if algo == 1 else [])  # algorithm 0 keeps no log-sum-exp at these head dimensions
                    steps = max(1, a.steps // 4) if algo == 0 else a.steps
                    ms, ws = timed(lambda s: nnc.cmd_exec(fwd, None, 0, [q, k, v], outs, s), steps, a.warmup)
                    print(json.dumps({"op": "sdpa_fwd_bf16", "algorithm": algo, "B": B, "H": H, "S": S, "D": D, "causal": causal, "ms": round(ms, 4),
                                      "tflops": round(flops / ms * 1e-9, 2), "workspace_mb": round(ws / 2 ** 20, 1)}), flush=True)
                    saved = [None, None, None, o, lse] if algo == 1 else []
                    ms, ws = timed(lambda s: nnc.cmd_exec(bwd, None, 0, [do, None, None, q, k, v] + saved, [dq, dk, dv], s), steps, a.warmup)
                    print(json.dumps({"op": "sdpa_bwd_bf16", "algorithm": algo, "B": B, "H": H, "S": S, "D": D, "causal": causal, "ms": round(ms, 4),
                                      "tflops": round(2.5 * flops / ms * 1e-9, 2), "workspace_mb": round(ws / 2 ** 20, 1)}), flush=True)
        finally:
            for t in ts + [lse]:
                t.free()


if __name__ == "__main__":
    main()
