"""Parity of the tensor-core contractions (GEMM, convolution; forward and backward) against the reference's own
CCV_NNC_BACKEND_CPU_REF on the same seeded inputs, through the C ABI.

Tolerance: BASELINE.json north_star -- <= 1e-3 relative for fp32, applied to max|diff| / max|ref| (tests/util.rel_err).
Algorithms: CCV_NNC_SM100_ALGO_TF32 (one wgmma tf32 pass, TMA rounds the operands to TF32: the convolution default,
as the reference's cuDNN path runs CUDNN_TENSOR_OP_MATH) is held to 1e-3; CCV_NNC_SM100_ALGO_3XTF32 (error-compensated, three
MMAs on hi / lo splits: the GEMM default, as the reference's cuBLAS path computes in CUBLAS_COMPUTE_32F) to 2e-5;
CCV_NNC_SM100_ALGO_FFMA (CUDA-core fp32) to 1e-5.  The full-size BASELINE configs (GEMM 1024^3, convolution N=64 C=64 56x56
K=64 3x3 forward + backward) are compared with CPU_REF itself at the end of this file, with the element-wise relative error
(absolute floor 1e-2 of max|ref|) reported next to the max-normalised one."""
import os

import numpy as np
import pytest

from ccv_b200 import abi
from tests.util import NCHW, NHWC, assert_close, counted, gpu_exec, ref_exec, seeded, to_bf16

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = {abi.CCV_NNC_SM100_ALGO_TF32: 1e-3, abi.CCV_NNC_SM100_ALGO_3XTF32: 2e-5, abi.CCV_NNC_SM100_ALGO_FFMA: 1e-5}
ALGOS = [abi.CCV_NNC_SM100_ALGO_TF32, abi.CCV_NNC_SM100_ALGO_3XTF32, abi.CCV_NNC_SM100_ALGO_FFMA]

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("algo", ALGOS)
def test_gemm_literal_cases_of_the_reference(gpu, algo):
    """test/unit/nnc/gemm.tests.c:13-200: small integers, so even TF32 is exact."""
    g = np.load(os.path.join(GOLDEN, "literal_gemm.npz"))
    nnc = gpu
    c = np.zeros((4, 3), np.float32)
    st, (out,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD(algorithm=algo), None, 0, [g["a"], g["b"]], [c])
    assert st == 0 and np.array_equal(out, g["c"])
    st, (out,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1), algorithm=algo), None, 0, [g["a"], g["bt"]], [c])
    assert st == 0 and np.array_equal(out, g["c"])
    c3 = np.zeros((1, 4, 3), np.float32)
    st, (out,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD((1, 2), (0, 1), algorithm=algo), None, 0, [g["at"], g["bt"]], [c3])
    assert st == 0 and np.array_equal(out[0], g["c"])
    st, (out,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD(algorithm=algo), None, 0, [g["a"], g["b"], g["bias"]], [c])
    assert st == 0 and np.array_equal(out, g["c_bias"])
    # 1-d a (a row vector): gemm.tests.c:42-62
    a1 = np.array([1, 2], np.float32)
    c1 = np.zeros((3,), np.float32)
    st, (out,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD(algorithm=algo), None, 0, [a1, g["b"]], [c1])
    assert st == 0 and np.array_equal(out, g["c"][0])


@pytest.mark.parametrize("algo", ALGOS)
def test_gemm_against_committed_cpu_ref_outputs(gpu, algo):
    g = np.load(os.path.join(GOLDEN, "cpuref_gemm.npz"))
    nnc = gpu
    st, (b,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1), algorithm=algo), None, 0, [g["a"], g["w"], g["bias"]], [np.zeros_like(g["b"])])
    assert st == 0
    assert_close(b, g["b"], TOL[algo], "gemm forward")
    st, (h, dw, db) = gpu_exec(nnc, nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1), algorithm=algo), None, 0, [g["g"], g["a"], g["w"]], [np.zeros_like(g["h"]), np.zeros_like(g["dw"]), np.zeros_like(g["db"])])
    assert st == 0
    assert_close(h, g["h"], TOL[algo], "gemm h")
    assert_close(dw, g["dw"], TOL[algo], "gemm dw")
    assert_close(db, g["db"], 1e-5, "gemm dbias")


SHAPES = [
    # (M, N, K, transpose_a, transpose_b, bias)
    (128, 128, 64, 0, 0, 0), (256, 192, 160, 0, 1, 1), (200, 136, 100, 1, 0, 1), (96, 72, 48, 1, 1, 0),
    (64, 1000, 2048, 0, 1, 1),  # the ResNet-50 classifier (a=[N,2048], w=[1000,2048] NT + bias)
    (33, 17, 21, 0, 1, 1),      # K not a multiple of 4: falls to the CUDA-core path
    (1, 64, 128, 0, 1, 0),
]


@pytest.mark.ref
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("M,N,K,ta,tb,with_bias", SHAPES)
def test_gemm_forward_backward_vs_cpu_ref(gpu, ref, algo, M, N, K, ta, tb, with_bias):
    """protocol of test/int/nnc/cublas.tests.c:1155-1750: seeded inputs, GPU backend vs CPU_REF."""
    nnc = gpu
    a = seeded((K, M) if ta else (M, K), 11, -1, 1)
    w = seeded((N, K) if tb else (K, N), 12, -1, 1)
    bias = seeded((N,), 13) if with_bias else None
    T = (0, 1)
    cmd = lambda c, **kw: c((0, 1) if ta else (0, 0), (0, 1) if tb else (0, 0), **kw)
    ins = [a, w] + ([bias] if with_bias else [])
    st_r, (b_ref,) = ref_exec(ref, cmd(nnc.CMD_GEMM_FORWARD), None, 0, ins, [np.zeros((M, N), np.float32)])
    st_g, (b_gpu,) = gpu_exec(nnc, cmd(nnc.CMD_GEMM_FORWARD, algorithm=algo), None, 0, ins, [np.zeros((M, N), np.float32)])
    assert st_r == 0 and st_g == 0
    assert_close(b_gpu, b_ref, TOL[algo], "forward")
    g = seeded((M, N), 14, -1, 1)
    outs = lambda: [np.zeros_like(a), np.zeros_like(w), np.zeros((N,), np.float32)]
    st_r, (h_r, dw_r, db_r) = ref_exec(ref, cmd(nnc.CMD_GEMM_BACKWARD), None, 0, [g, a, w], outs())
    st_g, (h_g, dw_g, db_g) = gpu_exec(nnc, cmd(nnc.CMD_GEMM_BACKWARD, algorithm=algo), None, 0, [g, a, w], outs())
    assert st_r == 0 and st_g == 0
    assert_close(h_g, h_r, TOL[algo], "h")
    assert_close(dw_g, dw_r, TOL[algo], "dw")
    assert_close(db_g, db_r, 1e-5, "dbias")


@pytest.mark.ref
def test_gemm_backward_accumulates_with_flag(gpu, ref):
    """CCV_NNC_ACCUMULATE_OUTPUT (blas/ccv_nnc_gemm_cpu_ref.c:332,362,407)."""
    nnc = gpu
    a, w, g = seeded((64, 96), 1, -1, 1), seeded((32, 96), 2, -1, 1), seeded((64, 32), 3, -1, 1)
    init = lambda: [seeded((64, 96), 4), seeded((32, 96), 5), seeded((32,), 6)]
    cmd_r = nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
    _, outs_r = ref_exec(ref, cmd_r, None, abi.CCV_NNC_ACCUMULATE_OUTPUT, [g, a, w], init())
    st, outs_g = gpu_exec(nnc, cmd_r, None, abi.CCV_NNC_ACCUMULATE_OUTPUT, [g, a, w], init())
    assert st == 0
    for x, y, n in zip(outs_g, outs_r, ("h", "dw", "dbias")):
        assert_close(x, y, 1e-3, n)


@pytest.mark.ref
def test_gemm_batched_and_views(gpu, ref):
    """batched a [B,M,K] x shared w, and a strided view of a larger tensor as operand (ccv_nnc_easy.h:421-444)."""
    nnc = gpu
    a, w = seeded((3, 40, 64), 1, -1, 1), seeded((48, 64), 2, -1, 1)
    cmd = nnc.CMD_GEMM_FORWARD((0, 0), (0, 1))
    _, (b_r,) = ref_exec(ref, cmd, None, 0, [a, w], [np.zeros((3, 40, 48), np.float32)])
    st, (b_g,) = gpu_exec(nnc, cmd, None, 0, [a, w], [np.zeros((3, 40, 48), np.float32)])
    assert st == 0
    assert_close(b_g, b_r, 1e-3, "batched")
    # view: rows 4..36, cols 8..40 of a [64, 64] tensor
    big = seeded((64, 64), 3, -1, 1)
    w2 = seeded((16, 32), 4, -1, 1)
    sub = np.ascontiguousarray(big[4:36, 8:40])
    _, (want,) = ref_exec(ref, cmd, None, 0, [sub, w2], [np.zeros((32, 16), np.float32)])
    t = nnc.gpu_tensor([64, 64]); t.upload(big)
    v = nnc.tensor_view_new(t, [32, 32], [4, 8] + [0] * 10, [64, 1] + [0] * 10)
    tw = nnc.gpu_tensor([16, 32]); tw.upload(w2)
    tb = nnc.gpu_tensor([32, 16])
    assert nnc.cmd_exec(cmd, None, 0, [v, tw], [tb]) == 0
    assert_close(tb.download(), want, 1e-3, "view")
    for x in (v, t, tw, tb):
        x.free()


CONVS = [
    # (N, H, W, C, K, R, S, stride, pad, dilation, bias)
    (2, 12, 12, 32, 64, 3, 3, 1, 1, 1, 1), (2, 13, 9, 64, 96, 3, 3, 2, 1, 1, 1), (3, 14, 14, 64, 256, 1, 1, 1, 0, 1, 1),
    (2, 15, 15, 32, 64, 3, 3, 1, 2, 2, 0), (1, 11, 11, 32, 32, 5, 5, 1, 2, 1, 1), (2, 16, 16, 3, 32, 3, 3, 2, 1, 1, 0),
    (2, 14, 14, 128, 128, 1, 1, 2, 0, 1, 0), (1, 20, 20, 16, 24, 7, 7, 2, 3, 1, 1),
]


@pytest.mark.ref
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("N,H,W,C,K,R,S,st,pad,dil,with_bias", CONVS)
def test_convolution_forward_backward_vs_cpu_ref(gpu, ref, algo, N, H, W, C, K, R, S, st, pad, dil, with_bias):
    """protocol of test/int/nnc/cudnn.tests.c:24-85,204-357: a in (0,1], w in (0,1]/(C k^2), bias; NHWC."""
    nnc = gpu
    P = (H + 2 * pad - ((R - 1) * dil + 1)) // st + 1
    Q = (W + 2 * pad - ((S - 1) * dil + 1)) // st + 1
    a = seeded((N, H, W, C), 21)
    w = seeded((K, R, S, C), 22) / (C * R * S)
    bias = (np.arange(K, dtype=np.float32) / K) if with_bias else None
    hint = nnc.hint((st, st), (pad, pad))
    ins = [a, w] + ([bias] if with_bias else [])
    fwd = lambda **kw: nnc.CMD_CONVOLUTION_FORWARD(1, K, R, S, C, (dil, dil), **kw)
    bwd = lambda **kw: nnc.CMD_CONVOLUTION_BACKWARD(1, K, R, S, C, (dil, dil), **kw)
    st_r, (b_r,) = ref_exec(ref, fwd(), hint, 0, ins, [np.zeros((N, P, Q, K), np.float32)])
    st_g, (b_g,) = gpu_exec(nnc, fwd(algorithm=algo), hint, 0, ins, [np.zeros((N, P, Q, K), np.float32)])
    assert st_r == 0 and st_g == 0
    assert_close(b_g, b_r, TOL[algo], "forward")
    g = seeded((N, P, Q, K), 23)
    outs = lambda: [np.zeros_like(a), np.zeros_like(w), np.zeros((K,), np.float32)]
    st_r, (h_r, dw_r, db_r) = ref_exec(ref, bwd(), hint, 0, [g, a, w], outs())
    st_g, (h_g, dw_g, db_g) = gpu_exec(nnc, bwd(algorithm=algo), hint, 0, [g, a, w], outs())
    assert st_r == 0 and st_g == 0
    assert_close(h_g, h_r, TOL[algo], "dgrad")
    assert_close(dw_g, dw_r, TOL[algo], "wgrad")
    assert_close(db_g, db_r, 1e-5, "dbias")


@pytest.mark.parametrize("algo", ALGOS)
def test_convolution_against_committed_cpu_ref_outputs(gpu, algo):
    g = np.load(os.path.join(GOLDEN, "cpuref_conv.npz"))
    nnc = gpu
    hint = nnc.hint((2, 2), (1, 1))
    st, (y,) = gpu_exec(nnc, nnc.CMD_CONVOLUTION_FORWARD(1, 12, 3, 3, 8, algorithm=algo), hint, 0, [g["x"], g["w"], g["bias"]], [np.zeros_like(g["y"])])
    assert st == 0
    assert_close(y, g["y"], TOL[algo], "conv forward")
    st, (gx, gw, gb) = gpu_exec(nnc, nnc.CMD_CONVOLUTION_BACKWARD(1, 12, 3, 3, 8, algorithm=algo), hint, 0, [g["gy"], g["x"], g["w"]], [np.zeros_like(g["gx"]), np.zeros_like(g["gw"]), np.zeros_like(g["gb"])])
    assert st == 0
    assert_close(gx, g["gx"], TOL[algo], "dgrad")
    assert_close(gw, g["gw"], TOL[algo], "wgrad")
    assert_close(gb, g["gb"], 1e-5, "dbias")


@pytest.mark.ref
def test_grouped_convolution_vs_cpu_ref(gpu, ref):
    nnc = gpu
    N, H, W, C, K, groups = 2, 10, 10, 16, 24, 4
    a, w, bias = seeded((N, H, W, C), 1), seeded((K, 3, 3, C // groups), 2) / 36, seeded((K,), 3)
    hint = nnc.hint((1, 1), (1, 1))
    cmd = nnc.CMD_CONVOLUTION_FORWARD(groups, K, 3, 3, C)
    _, (b_r,) = ref_exec(ref, cmd, hint, 0, [a, w, bias], [np.zeros((N, H, W, K), np.float32)])
    st, (b_g,) = gpu_exec(nnc, cmd, hint, 0, [a, w, bias], [np.zeros((N, H, W, K), np.float32)])
    assert st == 0
    assert_close(b_g, b_r, 1e-5, "grouped forward")


def test_full_size_properties_config2(gpu):
    """BASELINE.json configs[1] (N=64 C=64 56x56 K=64 3x3) at full size, through size-independent properties:
    linearity in the input, and the all-ones closed form of test/unit/nnc/forward.tests.c:14-43 (interior = R*S*C)."""
    nnc = gpu
    N, H, W, C, K = 64, 56, 56, 64, 64
    hint = nnc.hint((1, 1), (1, 1))
    cmd = nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C)
    ones_a, ones_w = np.ones((N, H, W, C), np.float32), np.ones((K, 3, 3, C), np.float32)
    st, (b,) = gpu_exec(nnc, cmd, hint, 0, [ones_a, ones_w], [np.zeros((N, H, W, K), np.float32)])
    assert st == 0
    assert np.all(b[:, 1:-1, 1:-1, :] == 9 * C) and np.all(b[:, 0, 0, :] == 4 * C) and np.all(b[:, 0, 1:-1, :] == 6 * C)
    a1, a2, w = seeded((N, H, W, C), 1, -1, 1), seeded((N, H, W, C), 2, -1, 1), seeded((K, 3, 3, C), 3, -1, 1) / 24
    t = [nnc.gpu_tensor(list(x.shape)) for x in (a1, a2, w)]
    for tt, x in zip(t, (a1, a2, w)):
        tt.upload(x)
    o1, o2, o3, s = (nnc.gpu_tensor([N, H, W, K]) for _ in range(4))
    assert nnc.cmd_exec(cmd, hint, 0, [t[0], t[2]], [o1]) == 0
    assert nnc.cmd_exec(cmd, hint, 0, [t[1], t[2]], [o2]) == 0
    assert nnc.cmd_exec(nnc.CMD_EWSUM_FORWARD(), None, 0, [t[0], t[1]], [s]) == 0
    assert nnc.cmd_exec(cmd, hint, 0, [s, t[2]], [o3]) == 0
    lhs, rhs = o3.download(), o1.download() + o2.download()
    assert_close(lhs, rhs, 1e-3, "conv(a1 + a2) == conv(a1) + conv(a2)")
    for x in t + [o1, o2, o3, s]:
        x.free()


def test_autotune_picks_a_working_algorithm(gpu):
    """registry->autotune (lib/nnc/ccv_nnc.h:323) of the contraction commands: device-timed choice between the one-pass TF32, the
    3xTF32 and the CUDA-core FFMA algorithm.  A large GEMM must come out as TF32 (algorithm 0: the fastest); a grouped convolution
    runs on the CUDA cores whichever algorithm is named, so any answer is acceptable there; the tuned command must then execute."""
    nnc = gpu
    stream = nnc.Stream(0)
    a, w, b = nnc.gpu_tensor([1024, 1024]), nnc.gpu_tensor([1024, 1024]), nnc.gpu_tensor([1024, 1024])
    a.upload(seeded((1024, 1024), 1)), w.upload(seeded((1024, 1024), 2))
    cmd = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1))
    tuned = nnc.cmd_autotune(cmd, None, 0, [a, w], [b], stream)
    assert tuned.algorithm == abi.CCV_NNC_SM100_ALGO_TF32
    assert nnc.cmd_exec(tuned, None, 0, [a, w], [b], stream) == 0
    x, f, y = nnc.gpu_tensor([2, 16, 16, 32]), nnc.gpu_tensor([64, 3, 3, 16]), nnc.gpu_tensor([2, 16, 16, 64])
    x.upload(seeded((2, 16, 16, 32), 3)), f.upload(seeded((64, 3, 3, 16), 4))
    conv = nnc.CMD_CONVOLUTION_FORWARD(2, 64, 3, 3, 32)
    hint = nnc.hint((1, 1), (1, 1))
    tuned = nnc.cmd_autotune(conv, hint, 0, [x, f], [y], stream)
    assert tuned.algorithm in (abi.CCV_NNC_SM100_ALGO_TF32, abi.CCV_NNC_SM100_ALGO_3XTF32, abi.CCV_NNC_SM100_ALGO_FFMA)
    assert nnc.cmd_exec(tuned, hint, 0, [x, f], [y], stream) == 0
    stream.wait()
    for t in (a, w, b, x, f, y, stream):
        t.free()


@pytest.mark.ref
@pytest.mark.parametrize("N,C,H,K,R,st,groups", [(2, 32, 12, 64, 3, 1, 1), (3, 16, 9, 24, 3, 2, 1), (2, 16, 10, 24, 3, 1, 4)])
def test_convolution_forward_nchw(gpu, ref, N, C, H, K, R, st, groups):
    """NCHW activations [N, C, H, W] and filters [K, C / g, kh, kw] (convolution/ccv_nnc_conv_cpu_ref.c:66-120; protocol of the NCHW
    cases of test/int/nnc/cudnn.tests.c): staged through NHWC on the device, compared with CPU_REF's own NCHW path."""
    nnc = gpu
    pad = R // 2
    P = (H + 2 * pad - R) // st + 1
    x, w, bias = seeded((N, C, H, H), 1, -1, 1), seeded((K, C // groups, R, R), 2, -1, 1) / (R * R * C) ** 0.5, seeded((K,), 3, -1, 1)
    cmd = nnc.CMD_CONVOLUTION_FORWARD(groups, K, R, R, C)
    hint = nnc.hint((st, st), (pad, pad))
    fmts = dict(in_fmts=[NCHW, NCHW, NHWC], out_fmts=[NCHW])
    st_r, (y_r,) = ref_exec(ref, cmd, hint, 0, [x, w, bias], [np.zeros((N, K, P, P), np.float32)], **fmts)
    st_g, (y_g,), n = counted(nnc, gpu_exec, cmd, hint, 0, [x, w, bias], [np.zeros((N, K, P, P), np.float32)], **fmts)
    assert st_r == 0 and st_g == 0
    assert_close(y_g, y_r, 1e-3, "NCHW convolution")
    # the same launches as the NHWC command, plus one relayout per NCHW operand in (x, w) and one per NCHW output out (y)
    t = lambda a: np.ascontiguousarray(a.transpose(0, 2, 3, 1))
    st_d, (y_d,), n_d = counted(nnc, gpu_exec, cmd, hint, 0, [t(x), t(w), bias], [np.zeros((N, P, P, K), np.float32)])
    assert st_d == 0 and n == n_d + 3, (n, n_d)
    assert np.array_equal(y_g, np.ascontiguousarray(y_d.transpose(0, 3, 1, 2)))


@pytest.mark.ref
@pytest.mark.parametrize("C,K,st,which", [(32, 64, 1, "filters"), (3, 24, 2, "filters"), (16, 32, 1, "activations")])
def test_convolution_forward_mixed_formats(gpu, ref, C, K, st, which):
    """NHWC activations against NCHW filters -- what the reference's own GPU tests run (test/int/nnc/cudnn.tests.c:24-85:
    `gwo` is GPU_TENSOR_NCHW while `ga` / `gc` are NHWC) -- and the converse; CPU_REF has no mixed path, so the check is the
    all-NHWC CPU_REF result on the transposed arrays."""
    nnc = gpu
    N, H, R = 2, 12, 3
    pad = R // 2
    P = (H + 2 * pad - R) // st + 1
    x, w, bias = seeded((N, H, H, C), 1, -1, 1), seeded((K, R, R, C), 2, -1, 1) / (R * R * C) ** 0.5, seeded((K,), 3, -1, 1)
    cmd = nnc.CMD_CONVOLUTION_FORWARD(1, K, R, R, C)
    hint = nnc.hint((st, st), (pad, pad))
    st_r, (y_r,) = ref_exec(ref, cmd, hint, 0, [x, w, bias], [np.zeros((N, P, P, K), np.float32)])
    if which == "filters":
        ins, fm = [x, np.ascontiguousarray(w.transpose(0, 3, 1, 2)), bias], dict(in_fmts=[NHWC, NCHW, NHWC], out_fmts=[NHWC])
        st_g, (y_g,) = gpu_exec(nnc, cmd, hint, 0, ins, [np.zeros((N, P, P, K), np.float32)], **fm)
    else:
        ins, fm = [np.ascontiguousarray(x.transpose(0, 3, 1, 2)), w, bias], dict(in_fmts=[NCHW, NHWC, NHWC], out_fmts=[NCHW])
        st_g, (y_g,) = gpu_exec(nnc, cmd, hint, 0, ins, [np.zeros((N, K, P, P), np.float32)], **fm)
        y_g = y_g.transpose(0, 2, 3, 1)
    assert st_r == 0 and st_g == 0
    assert_close(y_g, y_r, 1e-3, "mixed-format convolution")


@pytest.mark.ref
@pytest.mark.parametrize("C,K,st,layout", [(32, 64, 1, "nchw"), (3, 16, 2, "nchw"), (16, 32, 1, "filters"), (16, 32, 2, "nchw16")])
def test_convolution_backward_nchw_and_mixed(gpu, ref, C, K, st, layout):
    """CONVOLUTION_BACKWARD with NCHW tensors (all of them, or only the filter / its gradient as in test/int/nnc/cudnn.tests.c:
    348-497), also accumulating and in half precision: staged through NHWC; checked against CPU_REF's NHWC backward on the transposed arrays
    (CPU_REF's own backward is NHWC-only, convolution/ccv_nnc_conv_cpu_ref.c:358)."""
    nnc = gpu
    N, H, R = 2, 10, 3
    pad = R // 2
    P = (H + 2 * pad - R) // st + 1
    g, x, w = seeded((N, P, P, K), 1, -1, 1), seeded((N, H, H, C), 2, -1, 1), seeded((K, R, R, C), 3, -1, 1) / (R * R * C) ** 0.5
    half = layout == "nchw16"
    if half:
        from tests.util import round16
        g, x, w = round16(g, abi.CCV_16F), round16(x, abi.CCV_16F), round16(w, abi.CCV_16F)
    cmd = nnc.CMD_CONVOLUTION_BACKWARD(1, K, R, R, C)
    hint = nnc.hint((st, st), (pad, pad))
    st_r, (h_r, dw_r, db_r) = ref_exec(ref, cmd, hint, 0, [g, x, w], [np.zeros_like(x), np.zeros_like(w), np.zeros((K,), np.float32)])
    t = lambda a: np.ascontiguousarray(a.transpose(0, 3, 1, 2))
    if layout == "filters":
        ins, outs = [g, x, t(w)], [np.zeros_like(x), np.ones_like(t(w)), np.zeros((K,), np.float32)]
        fm = dict(in_fmts=[NHWC, NHWC, NCHW], out_fmts=[NHWC, NCHW, NHWC])
        st_g, (h_g, dw_g, db_g), n = counted(nnc, gpu_exec, cmd, hint, abi.CCV_NNC_ACCUMULATE_OUTPUT, ins, outs, **fm)
        dw_g = dw_g.transpose(0, 2, 3, 1) - 1.0  # accumulated onto ones
        # relayouts: w in, dw in (it accumulates) and out
        st_d, _, n_d = counted(nnc, gpu_exec, cmd, hint, abi.CCV_NNC_ACCUMULATE_OUTPUT, [g, x, w], [np.zeros_like(x), np.ones_like(w), np.zeros((K,), np.float32)])
        staging = 3
    else:
        ins, outs = [t(g), t(x), t(w)], [np.zeros_like(t(x)), np.zeros_like(t(w)), np.zeros((K,), np.float32)]
        fm = dict(in_fmts=[NCHW, NCHW, NCHW], out_fmts=[NCHW, NCHW, NHWC])
        dense = [g, x, w], [np.zeros_like(x), np.zeros_like(w), np.zeros((K,), np.float32)]
        if half:
            from tests.util import gpu_exec16
            st_g, (h_g, dw_g, db_g), n = counted(nnc, gpu_exec16, cmd, hint, 0, ins, outs, abi.CCV_16F, keep32=(id(outs[2]),), **fm)
            st_d, _, n_d = counted(nnc, gpu_exec16, cmd, hint, 0, *dense, abi.CCV_16F, keep32=(id(dense[1][2]),))
        else:
            st_g, (h_g, dw_g, db_g), n = counted(nnc, gpu_exec, cmd, hint, 0, ins, outs, **fm)
            st_d, _, n_d = counted(nnc, gpu_exec, cmd, hint, 0, *dense)
        h_g, dw_g = h_g.transpose(0, 2, 3, 1), dw_g.transpose(0, 2, 3, 1)
        staging = 5  # relayouts: g, x, w in; h, dw out
    assert st_r == 0 and st_g == 0 and st_d == 0
    assert n == n_d + staging, (n, n_d)
    tol = 1e-2 if half else 1e-3
    assert_close(h_g, h_r, tol, "dgrad " + layout)
    assert_close(dw_g, dw_r, tol, "wgrad " + layout)
    assert_close(db_g, db_r, tol, "dbias " + layout)


@pytest.mark.parametrize("case", ["fp16 dw", "fp16 w", "fp16 dbias", "fp16 h", "h channels", "bf16 g, fp16 dw"])
def test_convolution_backward_refuses_mixed_operands_before_any_launch(gpu, case):
    """The backend is chosen on the union of the operands' types, so CONVOLUTION_BACKWARD receives calls whose operands differ in type.
    It checks every operand (types, the dbias type, h's geometry) before its first launch: such a call returns INVALID, launches
    nothing and leaves h, dw and dbias as they were, also when dw and dbias would have been computable."""
    nnc = gpu
    N, H, C, K, R = 2, 8, 16, 32, 3
    F32, F16, BF16 = abi.CCV_32F, abi.CCV_16F, abi.CCV_16BF
    types = dict(g=F32, a=F32, w=F32, h=F32, dw=F32, dbias=F32)
    h_c = C
    if case == "h channels":
        h_c = C + 8
    elif case == "bf16 g, fp16 dw":
        types.update(g=BF16, a=BF16, w=BF16, h=BF16, dw=F16)
    else:
        types[case.split()[1]] = F16
    shapes = dict(g=(N, H, H, K), a=(N, H, H, C), w=(K, R, R, C), h=(N, H, H, h_c), dw=(K, R, R, C), dbias=(K,))
    tensors, before = {}, {}
    for i, name in enumerate(("g", "a", "w", "h", "dw", "dbias")):
        v = seeded(shapes[name], 10 + i, -1, 1)
        v = to_bf16(v) if types[name] == BF16 else v.astype(np.float16) if types[name] == F16 else v
        tensors[name] = nnc.gpu_tensor(list(shapes[name]), NHWC, types[name])
        tensors[name].upload(v)
        before[name] = tensors[name].download().tobytes()
    l0 = nnc.launch_count()
    status = nnc.cmd_exec(nnc.CMD_CONVOLUTION_BACKWARD(1, K, R, R, C), nnc.hint((1, 1), (1, 1)), 0, [tensors[n] for n in ("g", "a", "w")], [tensors[n] for n in ("h", "dw", "dbias")])
    launches = nnc.launch_count() - l0
    after = {name: t.download().tobytes() for name, t in tensors.items()}
    for t in tensors.values():
        t.free()
    assert status == abi.CCV_NNC_EXEC_INVALID, (case, status)
    assert launches == 0, (case, launches)
    for name in ("h", "dw", "dbias"):
        assert after[name] == before[name], (case, name + " changed")


# ------------------------------------------------------------------------------------------------ BASELINE configs at full size
def _report(name, got, want, tol):
    from tests.util import elem_rel_err, rel_err
    n, e = rel_err(got, want), elem_rel_err(got, want)
    print("%s: max-normalised error %.3e, element-wise relative error (floor 1e-2 max|ref|) %.3e" % (name, n, e))
    assert np.isfinite(got).all(), name
    assert n <= tol, "%s: normalised max error %.3e > %.1e" % (name, n, tol)
    assert e <= 100 * tol, "%s: element-wise relative error %.3e > %.1e" % (name, e, 100 * tol)


@pytest.mark.ref
@pytest.mark.parametrize("tb", [0, 1])
def test_baseline_config1_gemm_1024_cubed_vs_cpu_ref(gpu, ref, tb):
    """BASELINE.json configs[0]: CCV_NNC_GEMM_FORWARD fp32 1024 x 1024 x 1024 (NN and NT), the whole result against
    CCV_NNC_BACKEND_CPU_REF (sequential-k float accumulation, blas/ccv_nnc_gemm_cpu_ref.c:28-33).  The DEFAULT algorithm of
    an fp32 GEMM is the error-compensated 3xTF32 kernel (the reference computes fp32 GEMMs in CUBLAS_COMPUTE_32F), held to the
    fp32 bound of the north star with two orders of magnitude to spare; with CCV_NNC_GEMM_32TF the one-pass TF32 kernel runs."""
    nnc = gpu
    a, w = seeded((1024, 1024), 31, -1, 1), seeded((1024, 1024), 32, -1, 1)
    cmd = lambda **kw: nnc.CMD_GEMM_FORWARD((0, 0), (0, 1) if tb else (0, 0), **kw)
    _, (want,) = ref_exec(ref, cmd(), None, 0, [a, w], [np.zeros((1024, 1024), np.float32)])
    st, (got,) = gpu_exec(nnc, cmd(), None, 0, [a, w], [np.zeros((1024, 1024), np.float32)])
    assert st == 0
    _report("GEMM 1024^3 %s default (3xTF32)" % ("NT" if tb else "NN"), got, want, 1e-5)
    tf = cmd()
    tf.info.blas.flags = abi.CCV_NNC_GEMM_32TF
    st, (got,) = gpu_exec(nnc, tf, None, 0, [a, w], [np.zeros((1024, 1024), np.float32)])
    assert st == 0
    _report("GEMM 1024^3 %s CCV_NNC_GEMM_32TF" % ("NT" if tb else "NN"), got, want, 1e-3)


@pytest.mark.ref
@pytest.mark.parametrize("algo", [abi.CCV_NNC_SM100_ALGO_TF32, abi.CCV_NNC_SM100_ALGO_3XTF32])
def test_baseline_config2_convolution_full_size_vs_cpu_ref(gpu, ref, algo):
    """BASELINE.json configs[1]: CCV_NNC_CONVOLUTION_FORWARD + BACKWARD fp32 N=64 C=64 H=W=56 K=64 3x3, every element of
    y, dx, dw against CPU_REF (zero-mean data: nothing hides behind a large common offset)."""
    nnc = gpu
    N, H, C, K = 64, 56, 64, 64
    a, w, g = seeded((N, H, H, C), 41, -1, 1), seeded((K, 3, 3, C), 42, -1, 1) / 24, seeded((N, H, H, K), 43, -1, 1)
    hint = nnc.hint((1, 1), (1, 1))
    fwd, bwd = (lambda **kw: nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C, **kw)), (lambda **kw: nnc.CMD_CONVOLUTION_BACKWARD(1, K, 3, 3, C, **kw))
    _, (y_r,) = ref_exec(ref, fwd(), hint, 0, [a, w], [np.zeros((N, H, H, K), np.float32)])
    _, (h_r, dw_r) = ref_exec(ref, bwd(), hint, 0, [g, a, w], [np.zeros_like(a), np.zeros_like(w)])
    st, (y_g,) = gpu_exec(nnc, fwd(algorithm=algo), hint, 0, [a, w], [np.zeros((N, H, H, K), np.float32)])
    assert st == 0
    st, (h_g, dw_g) = gpu_exec(nnc, bwd(algorithm=algo), hint, 0, [g, a, w], [np.zeros_like(a), np.zeros_like(w)])
    assert st == 0
    tol = TOL[algo]
    _report("conv cfg2 algo %d forward" % algo, y_g, y_r, tol)
    _report("conv cfg2 algo %d dgrad" % algo, h_g, h_r, tol)
    # the filter gradient sums 200 704 products per element: CPU_REF's own sequential fp32 accumulation is only good to
    # ~1e-5 of the largest element there, so the compensated kernel is held to 1e-4 on this output
    _report("conv cfg2 algo %d wgrad" % algo, dw_g, dw_r, max(tol, 1e-4))
