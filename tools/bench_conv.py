"""BASELINE.json configs[1] -- CCV_NNC_CONVOLUTION_FORWARD + BACKWARD, N=64 C=64 H=W=56 K=64 3x3 stride 1 pad 1, NHWC, no bias --
through ccv_nnc_cmd_exec on CCV_NNC_BACKEND_GPU_SM100, for every math mode: fp32 one-pass TF32 (algorithm 0), 3xTF32 (1),
CUDA-core FFMA (2), bf16 and fp16 tensors.  One JSON line per mode: device milliseconds (CUDA events, 20 launches after 5
warm-ups; the 51 MB operands exceed nothing but are re-read from L2 / HBM as a real step would) and algorithmic TFLOP/s
(fwd 14.80 GFLOP, bwd 29.60 GFLOP, SURVEY.md 8d).
usage: bench_conv.py [mode ...] [reps]   modes: tf32 3xtf32 ffma bf16 f16 (default: all)"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ccv_b200 import abi, nnc  # noqa: E402

N, H, C, K = 64, 56, 64, 64
MODES = {"tf32": (abi.CCV_32F, 0), "3xtf32": (abi.CCV_32F, 1), "ffma": (abi.CCV_32F, 2), "bf16": (abi.CCV_16BF, -1), "f16": (abi.CCV_16F, -1)}


def main():
    argv = sys.argv[1:]
    reps = int(argv.pop()) if argv and argv[-1].isdigit() else 20
    modes = argv or list(MODES)
    nnc.init()
    stream = nnc.Stream(0)
    pk = 989.0  # dense BF16, NVIDIA's H100 SXM data sheet (700 W)
    rs = np.random.RandomState(0)
    hint = nnc.hint((1, 1), (1, 1))
    for mode in modes:
        dt, algo = MODES[mode]
        x, w, y, g, dx, dw = (nnc.gpu_tensor(s, datatype=dt) for s in ([N, H, H, C], [K, 3, 3, C], [N, H, H, K], [N, H, H, K], [N, H, H, C], [K, 3, 3, C]))
        for t in (x, w, g):
            a = (rs.rand(*t.dims).astype(np.float32) - 0.5)
            if dt == abi.CCV_32F:
                t.upload(a)
            elif dt == abi.CCV_16F:
                t.upload(a.astype(np.float16))
            else:
                u = a.view(np.uint32).astype(np.uint64)
                t.upload((((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16))
        fwd, bwd = nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C, algorithm=algo), nnc.CMD_CONVOLUTION_BACKWARD(1, K, 3, 3, C, algorithm=algo)
        out = {"op": "conv_cfg2", "mode": mode}
        for name, fn, flops in (("fwd", lambda: nnc.cmd_exec(fwd, hint, 0, [x, w], [y], stream), 2.0 * N * H * H * K * C * 9), ("bwd", lambda: nnc.cmd_exec(bwd, hint, 0, [g, x, w], [dx, dw], stream), 4.0 * N * H * H * K * C * 9)):
            for _ in range(min(5, reps)):
                assert fn() == 0, nnc.lib().ccv_nnc_sm100_last_error()
            e0, e1 = nnc.Event(), nnc.Event()
            stream.wait()
            e0.record(stream)
            for _ in range(reps):
                fn()
            e1.record(stream)
            ms = e0.elapsed_ms(e1) / reps
            peak = pk if dt != abi.CCV_32F else pk / 2 / (3 if algo == 1 else 1)
            out[name] = {"ms": ms, "tflops": flops / ms * 1e-9, "frac_of_tensor_peak": None if algo == 2 else flops / ms * 1e-9 / peak}
        print(json.dumps(out))
        for t in (x, w, y, g, dx, dw):
            t.free()


if __name__ == "__main__":
    main()
