"""Masked SCALED_DOT_PRODUCT_ATTENTION forwards (bf16, an fp32 [S, S] additive mask) under algorithm 0 (the fp32 functional form) and
algorithm 2 (CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK: the flash kernels with the mask staged through shared memory), and the same call without
the mask under algorithm 1, which gives the mask's overhead on the flash kernels.  Prints one JSON line per (shape, causal, variant): ms per
call (CUDA events over the timed calls, after warm-up calls), TFLOP/s of the algorithmic count (4 B H Sq Sk D, halved when causal) and
the device memory the call's stream workspace took.  The first line names the card, its power limit and its SM clocks.

    python tools/bench_sdpa_mask.py [--steps N] [--warmup W] [--quick]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ccv_b200 import abi, nnc  # noqa: E402
from tools.bench_sdpa_wide import cmd, timed, to_bf16  # noqa: E402

SHAPES = [  # (B, H, S, D)
    (4, 16, 4096, 128), (4, 16, 4096, 160), (4, 16, 4096, 256),
    (2, 8, 1024, 160),   # Stable Diffusion 1.x's widest attention
]
VARIANTS = [  # (name, algorithm, with the mask)
    ("masked", 0, True), ("masked", abi.CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK, True), ("unmasked", abi.CCV_NNC_SM100_SDPA_ALGO_FLASH, False),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true", help="the small shape only")
    a = ap.parse_args()
    nnc.init()
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) <= 0:
        raise SystemExit("bench_sdpa_mask: no CUDA device")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"card": card}), flush=True)
    rng = np.random.RandomState(0)
    for B, H, S, D in (SHAPES[3:] if a.quick else SHAPES):
        q, k, v, o = (nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF) for _ in range(4))
        for t in (q, k, v):
            t.upload(to_bf16(rng.random_sample((B, S, H, D)).astype(np.float32) * 2 - 1))
        mask = nnc.gpu_tensor([S, S]).upload(-rng.random_sample((S, S)).astype(np.float32))
        try:
            for causal in (0, 1):
                flops = 4.0 * B * H * S * S * D * (0.5 if causal else 1.0)
                for name, algo, masked in VARIANTS:
                    fwd = cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, D, causal, algo)
                    ins = [q, k, v] + ([mask] if masked else [])
                    steps = max(1, a.steps // 4) if algo == 0 else a.steps
                    ms, ws = timed(lambda s: nnc.cmd_exec(fwd, None, 0, ins, [o], s), steps, a.warmup)
                    print(json.dumps({"op": "sdpa_fwd_bf16", "variant": name, "algorithm": algo, "B": B, "H": H, "S": S, "D": D, "causal": causal,
                                      "ms": round(ms, 4), "tflops": round(flops / ms * 1e-9, 2), "workspace_mb": round(ws / 2 ** 20, 1)}), flush=True)
        finally:
            for t in (q, k, v, o, mask):
                t.free()


if __name__ == "__main__":
    main()
