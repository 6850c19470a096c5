"""Convolution launches whose CTAs walk several M tiles (more output tiles than one wave of one CTA per SM), with a ragged last
tile: the data gradient (1x1, 3x3, and 3x3 stride 2 through its residue classes) and a projection-style forward without batch
norm, against CPU_REF at the contraction tests' tolerances.  Plus one exactness check: the fp32 data gradient reads a K-major
copy of the filters, which must give the same TF32 products in the same order as the GEMM that reads them in place."""
import functools

import numpy as np
import pytest

from ccv_b200 import abi
from tests.util import assert_close, gpu_exec, ref_exec, seeded

TOL = {abi.CCV_NNC_SM100_ALGO_TF32: 1e-3, abi.CCV_NNC_SM100_ALGO_3XTF32: 2e-5}
ALGOS = sorted(TOL)

pytestmark = pytest.mark.gpu

# (N, H, C, K, R, stride): every case has more than 132 output tiles of 128 rows, and a last tile that is not full
DGRAD = [
    (17, 56, 64, 256, 1, 1),  # layer1 conv1 / conv3 shape: 53312 pixels
    (8, 75, 40, 48, 3, 1),    # 3x3: C and K not multiples of the 64 / 32 tile edges
    (8, 149, 32, 64, 3, 2),   # 3x3 stride 2: residue classes of 75 x 75, 75 x 74, 74 x 75 and 74 x 74 pixels per image
]


def _operands(N, H, C, K, R, st):
    pad = R // 2
    P = (H + 2 * pad - R) // st + 1
    g = seeded((N, P, P, K), 51, -1, 1)
    x = seeded((N, H, H, C), 52, -1, 1)
    w = seeded((K, R, R, C), 53, -1, 1) / (R * R * C) ** 0.5
    return g, x, w


@functools.lru_cache(maxsize=None)
def _dgrad_ref(nnc, ref, case):
    """CPU_REF's data gradient (the same for every algorithm of the GPU side; CPU_REF always computes dw as well)"""
    N, H, C, K, R, st = case
    g, x, w = _operands(*case)
    st_r, (h, _) = ref_exec(ref, nnc.CMD_CONVOLUTION_BACKWARD(1, K, R, R, C), nnc.hint((st, st), (R // 2, R // 2)), 0, [g, x, w], [np.zeros_like(x), np.zeros_like(w)])
    assert st_r == 0
    return h


@pytest.mark.ref
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("case", DGRAD)
def test_dgrad_walking_ctas_vs_cpu_ref(gpu, ref, algo, case):
    nnc = gpu
    N, H, C, K, R, st = case
    g, x, w = _operands(*case)
    st_g, (h,) = gpu_exec(nnc, nnc.CMD_CONVOLUTION_BACKWARD(1, K, R, R, C, algorithm=algo), nnc.hint((st, st), (R // 2, R // 2)), 0, [g, x, w], [np.zeros_like(x)])
    assert st_g == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert_close(h, _dgrad_ref(nnc, ref, case), TOL[algo], "dgrad %s" % (case,))


@functools.lru_cache(maxsize=None)
def _projection_ref(nnc, ref):
    x, w = seeded((17, 56, 56, 64), 61, -1, 1), seeded((256, 1, 1, 64), 62, -1, 1) / 8
    _, (y,) = ref_exec(ref, nnc.CMD_CONVOLUTION_FORWARD(1, 256, 1, 1, 64), nnc.hint((1, 1), (0, 0)), 0, [x, w], [np.zeros((17, 56, 56, 256), np.float32)])
    return x, w, y


@pytest.mark.ref
@pytest.mark.parametrize("algo", ALGOS)
def test_projection_forward_walking_ctas_vs_cpu_ref(gpu, ref, algo):
    """a 1x1 64 -> 256 forward without batch norm (the projection of ResNet-50's layer1): 417 x 2 output tiles"""
    nnc = gpu
    x, w, want = _projection_ref(nnc, ref)
    st_g, (y,) = gpu_exec(nnc, nnc.CMD_CONVOLUTION_FORWARD(1, 256, 1, 1, 64, algorithm=algo), nnc.hint((1, 1), (0, 0)), 0, [x, w], [np.zeros_like(want)])
    assert st_g == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert_close(y, want, TOL[algo], "projection forward")


def test_pointwise_dgrad_equals_gemm_bit_for_bit(gpu):
    """h[NHW, C] = g[NHW, K] x W[K, C]: the 1x1 data gradient and GEMM_FORWARD on the same operands, both one-pass TF32"""
    nnc = gpu
    g, x, w = _operands(*DGRAD[0])
    N, H, C, K = DGRAD[0][:4]
    tf32 = abi.CCV_NNC_SM100_ALGO_TF32
    st, (h,) = gpu_exec(nnc, nnc.CMD_CONVOLUTION_BACKWARD(1, K, 1, 1, C, algorithm=tf32), nnc.hint((1, 1), (0, 0)), 0, [g, x, w], [np.zeros_like(x)])
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    st, (c,) = gpu_exec(nnc, nnc.CMD_GEMM_FORWARD(algorithm=tf32), None, 0, [g.reshape(-1, K), w.reshape(K, C)], [np.zeros((N * H * H, C), np.float32)])
    assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
    assert np.array_equal(h.reshape(-1, C).view(np.uint32), c.view(np.uint32))
