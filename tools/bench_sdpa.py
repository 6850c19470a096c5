"""BASELINE configs[4]: SDPA forward bf16, B=32 H=16 S=2048 D=128, non-causal and causal, scale 1/sqrt(128), through the
C ABI (ccv_nnc_cmd_exec on CCV_NNC_BACKEND_GPU_SM100).  Prints one JSON line per variant: ms, TFLOP/s (algorithmic
4*B*H*S*S*D, halved for causal), GB/s over Q+K+V+O+LSE, fractions of the measured peaks.  Inputs are the reference's i / count
ramps (test/int/nnc/cublas.tests.c:2786-2794) rounded to bf16; 20 timed launches after 5 warm-ups, CUDA events."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ccv_b200 import abi, nnc  # noqa: E402


def to_bf16(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


def main():
    B, H, S, D = (int(x) for x in (sys.argv[1:5] if len(sys.argv) >= 5 else (32, 16, 2048, 128)))
    nnc.init()
    stream = nnc.Stream(0)
    peaks = {"hbm": 3350.0, "bf16": 989.0}  # NVIDIA's H100 SXM data sheet (700 W)
    n = B * S * H * D
    ramp = (np.arange(n, dtype=np.float64) / n).astype(np.float32).reshape(B, S, H, D)
    tensors = [nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF) for _ in range(4)]
    for t in tensors[:3]:
        t.upload(to_bf16(ramp))
    lse = nnc.gpu_tensor([B, H, S])
    for causal in (0, 1):
        cmd = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD)
        cmd.info.scaled_dot_product_attention.scale = 1.0 / np.sqrt(D)
        cmd.info.scaled_dot_product_attention.is_causal = causal
        for _ in range(5):
            assert nnc.cmd_exec(cmd, None, 0, tensors[:3], [tensors[3], lse], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        e0, e1 = nnc.Event(), nnc.Event()
        stream.wait()
        e0.record(stream)
        reps = 20
        for _ in range(reps):
            nnc.cmd_exec(cmd, None, 0, tensors[:3], [tensors[3], lse], stream)
        e1.record(stream)
        ms = e0.elapsed_ms(e1) / reps
        flops = 4.0 * B * H * S * S * D * (0.5 if causal else 1.0)
        byts = 4.0 * n * 2 + B * H * S * 4
        print(json.dumps({"op": "sdpa_fwd_bf16", "B": B, "H": H, "S": S, "D": D, "causal": causal, "ms": ms, "tflops": flops / ms * 1e-9, "frac_of_bf16_peak": flops / ms * 1e-9 / peaks["bf16"],
                          "gbs": byts / ms * 1e-6, "frac_of_hbm_peak": byts / ms * 1e-6 / peaks["hbm"]}))


if __name__ == "__main__":
    main()
