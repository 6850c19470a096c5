"""SCALED_DOT_PRODUCT_ATTENTION forward / backward vs the reference's CPU_REF.  Shape trials follow
test/int/nnc/cublas.tests.c:2752-2953 (GQA Hq/Hk = 8/2, head dims 40/64/128, causal, inputs i / count ramps, tolerance
3e-3 absolute there; relative 2e-3 of max|ref| here) plus an additive mask case from test/unit/nnc/attention.tests.c."""
import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests.util import assert_close, gpu_exec, ref_exec, seeded

pytestmark = [pytest.mark.gpu, pytest.mark.ref]


def _cmd(cmd_id, scale, causal):
    c = _nnc._simple(cmd_id)
    s = c.info.scaled_dot_product_attention
    s.scale, s.is_causal = scale, causal
    return c


TRIALS = [
    # B, Sq, Sk, Hq, Hk, D, causal
    (2, 32, 32, 4, 4, 64, 0), (2, 32, 48, 8, 2, 64, 0), (1, 40, 40, 8, 8, 40, 1), (2, 24, 36, 4, 2, 128, 1), (1, 128, 128, 2, 2, 128, 0),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,D,causal", TRIALS)
def test_sdpa_forward_backward_vs_cpu_ref(gpu, ref, B, Sq, Sk, Hq, Hk, D, causal):
    nnc = gpu
    scale = 1.0 / np.sqrt(D)
    q, k, v = seeded((B, Sq, Hq, D), 1, -1, 1), seeded((B, Sk, Hk, D), 2, -1, 1), seeded((B, Sk, Hk, D), 3, -1, 1)
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, causal)
    mk = lambda: [np.zeros((B, Sq, Hq, D), np.float32), None]
    st_r, (o_r, _) = ref_exec(ref, fwd, None, 0, [q, k, v], mk())
    st_g, (o_g, _) = gpu_exec(nnc, fwd, None, 0, [q, k, v], mk())
    assert st_r == 0 and st_g == 0
    assert_close(o_g, o_r, 2e-3, "attention output")
    g = seeded((B, Sq, Hq, D), 4, -1, 1)
    bwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, scale, causal)
    ins = [g, None, None, q, k, v]
    mk = lambda: [np.zeros_like(q), np.zeros_like(k), np.zeros_like(v)]
    st_r, (dq_r, dk_r, dv_r) = ref_exec(ref, bwd, None, 0, ins, mk())
    st_g, (dq_g, dk_g, dv_g) = gpu_exec(nnc, bwd, None, 0, ins, mk())
    assert st_r == 0 and st_g == 0
    assert_close(dq_g, dq_r, 3e-3, "dq"), assert_close(dk_g, dk_r, 3e-3, "dk"), assert_close(dv_g, dv_r, 3e-3, "dv")


def test_sdpa_with_additive_mask(gpu, ref):
    nnc = gpu
    B, S, H, D = 2, 24, 4, 32
    q, k, v = seeded((B, S, H, D), 1, -1, 1), seeded((B, S, H, D), 2, -1, 1), seeded((B, S, H, D), 3, -1, 1)
    mask = np.where(np.random.RandomState(5).rand(1, 1, S, S) < 0.3, -1e9, 0.0).astype(np.float32)
    mask[..., np.arange(S), np.arange(S)] = 0  # never mask a whole row
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, 1.0 / np.sqrt(D), 0)
    st_r, (o_r, _) = ref_exec(ref, fwd, None, 0, [q, k, v, mask], [np.zeros_like(q), None])
    st_g, (o_g, _) = gpu_exec(nnc, fwd, None, 0, [q, k, v, mask], [np.zeros_like(q), None])
    assert st_r == 0 and st_g == 0
    assert_close(o_g, o_r, 2e-3, "masked attention")


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,D,causal,with_bias", [(2, 24, 36, 4, 2, 32, 0, 1), (1, 40, 40, 8, 8, 16, 1, 0), (2, 32, 32, 2, 2, 64, 0, 1)])
def test_sdpa_unify_head_projection_vs_cpu_ref(gpu, ref, B, Sq, Sk, Hq, Hk, D, causal, with_bias):
    """The fused "unify head" output (…attention_cpu_ref.c:26-27,184-255; test/unit/nnc/attention.tests.c): inputs (q, k, v, mask, w,
    bias) -> outputs (d = concat_heads(attention) w^T + bias, lse, c = per-head attention).  fp32 against CPU_REF: c to the attention
    bound, d to the GEMM command's 3xTF32 bound."""
    nnc = gpu
    scale = 1.0 / np.sqrt(D)
    q, k, v = seeded((B, Sq, Hq, D), 1, -1, 1), seeded((B, Sk, Hk, D), 2, -1, 1), seeded((B, Sk, Hk, D), 3, -1, 1)
    w = seeded((Hq * D, Hq * D), 4, -0.5, 0.5)
    bias = seeded((Hq * D,), 5, -1, 1) if with_bias else None
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, causal)
    ins = [q, k, v, None, w, bias]
    mk = lambda: [np.zeros((B, Sq, Hq * D), np.float32), None, np.zeros((B, Sq, Hq, D), np.float32)]
    st_r, (d_r, _, c_r) = ref_exec(ref, fwd, None, 0, ins, mk())
    st_g, (d_g, _, c_g) = gpu_exec(nnc, fwd, None, 0, ins, mk())
    assert st_r == 0 and st_g == 0
    assert_close(c_g, c_r, 2e-3, "per-head attention")
    assert_close(d_g, d_r, 2e-3, "unified output")
    # a bias without a weight matrix is refused, as the reference asserts (:27-28)
    if with_bias:
        st, _ = gpu_exec(nnc, fwd, None, 0, [q, k, v, None, None, bias], [np.zeros((B, Sq, Hq, D), np.float32), None])
        assert st == abi.CCV_NNC_EXEC_INVALID


def test_sdpa_unify_head_projection_bf16(gpu, ref):
    """The same on bf16 tensors, D = 128 (flash kernel + kind::f16 projection), fp32 bias: CPU_REF on the rounded operands, 1e-2."""
    nnc = gpu
    B, S, H, D = 2, 128, 2, 128
    scale = 1.0 / np.sqrt(D)
    arrs = [seeded((B, S, H, D), 1, -1, 1), seeded((B, S, H, D), 2, -1, 1), seeded((B, S, H, D), 3, -1, 1), seeded((H * D, H * D), 4, -0.1, 0.1)]
    bits = [_to_bf16(a) for a in arrs]
    q, k, v, w = (_from_bf16(b) for b in bits)
    bias = seeded((H * D,), 5, -1, 1)
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, 0)
    st_r, (d_r, _, c_r) = ref_exec(ref, fwd, None, 0, [q, k, v, None, w, bias], [np.zeros((B, S, H * D), np.float32), None, np.zeros((B, S, H, D), np.float32)])
    assert st_r == 0
    stream = nnc.Stream(0)
    tq, tk, tv, tw = (nnc.gpu_tensor(list(b.shape), datatype=abi.CCV_16BF).upload(b) for b in bits)
    tb = nnc.gpu_tensor([H * D]).upload(bias)
    td, tc = nnc.gpu_tensor([B, S, H * D], datatype=abi.CCV_16BF), nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF)
    assert nnc.cmd_exec(fwd, None, 0, [tq, tk, tv, None, tw, tb], [td, None, tc], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    assert_close(_from_bf16(tc.download()), c_r, 1e-2, "bf16 per-head attention")
    assert_close(_from_bf16(td.download()), d_r, 1e-2, "bf16 unified output")
    for t in (tq, tk, tv, tw, tb, td, tc, stream):
        t.free()


# ---- 16-bit flash attention (ccv_b200/csrc/sm100_fmha.cu) --------------------------------------------------------------
def _to_bf16(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)  # round to nearest even


def _from_bf16(u):
    return (u.astype(np.uint32) << 16).view(np.float32)


def _attention_f64(q, k, v, scale, causal):
    """Plain float64 restatement of ..._cpu_ref.c:88-183 on [B, S, H, D] arrays (GQA by head ratio, causal aligned to the
    bottom-right corner :147); returns (O, LSE [B, H, Sq])."""
    B, Sq, H, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    o = np.zeros((B, Sq, H, v.shape[3]))
    lse = np.zeros((B, H, Sq))
    for b in range(B):
        for h in range(H):
            hk = h // (H // Hk)
            s = scale * (q[b, :, h].astype(np.float64) @ k[b, :, hk].astype(np.float64).T)
            if causal:
                i, j = np.arange(Sq)[:, None], np.arange(Sk)[None, :]
                s = np.where(j <= i + Sk - Sq, s, -np.inf)
            m = s.max(axis=1, keepdims=True)
            e = np.exp(s - m)
            den = e.sum(axis=1, keepdims=True)
            o[b, :, h] = (e / den) @ v[b, :, hk].astype(np.float64)
            lse[b, h] = (m + np.log(den))[:, 0]
    return o, lse


FMHA_TRIALS = [
    # B, Sq, Sk, Hq, Hk, causal
    (2, 256, 256, 4, 4, 0), (2, 256, 256, 4, 4, 1), (1, 128, 384, 8, 2, 1), (1, 200, 333, 2, 2, 0), (1, 333, 333, 2, 1, 1), (1, 1024, 1024, 2, 2, 1),
]


@pytest.mark.parametrize("dtype", ["bf16", "f16"])
@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,causal", FMHA_TRIALS)
def test_flash_attention_16bit_forward(gpu, ref, B, Sq, Sk, Hq, Hk, causal, dtype):
    """bf16 / fp16 SDPA forward, D = 128 (BASELINE configs[4] shape family).  There is no 16-bit CPU_REF kernel (SURVEY 8c:
    "parity defined as fp32-oracle-on-rounded-inputs"): the inputs are rounded to the 16-bit type, CPU_REF runs on those
    values in fp32, and the GPU result is held to 1e-2 of max|ref| (BASELINE tolerance for bf16); LSE to 1e-3."""
    nnc = gpu
    D = 128
    scale = 1.0 / np.sqrt(D)
    q, k, v = seeded((B, Sq, Hq, D), 1, -1, 1), seeded((B, Sk, Hk, D), 2, -1, 1), seeded((B, Sk, Hk, D), 3, -1, 1)
    if dtype == "bf16":
        bits = [_to_bf16(x) for x in (q, k, v)]
        q, k, v = (_from_bf16(x) for x in bits)
        ccv_dt = abi.CCV_16BF
    else:
        bits = [x.astype(np.float16).view(np.uint16) for x in (q, k, v)]
        q, k, v = (x.view(np.float16).astype(np.float32) for x in bits)
        ccv_dt = abi.CCV_16F
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, causal)
    o64, lse64 = _attention_f64(q, k, v, scale, causal)
    if Sq * Sk <= 256 * 256:  # CPU_REF itself on the rounded values (small cases; it agrees with the float64 restatement)
        st_r, (o_r, _) = ref_exec(ref, fwd, None, 0, [q, k, v], [np.zeros((B, Sq, Hq, D), np.float32), None])
        assert st_r == 0
        assert_close(o_r, o64, 1e-4, "CPU_REF vs float64 restatement")
    stream = nnc.Stream(0)
    tq, tk, tv = (nnc.gpu_tensor(list(x.shape), datatype=ccv_dt) for x in (q, k, v))
    to = nnc.gpu_tensor([B, Sq, Hq, D], datatype=ccv_dt)
    tl = nnc.gpu_tensor([B, Hq, Sq])
    for t, x in zip((tq, tk, tv), bits):
        t.upload(x.view(np.float16) if ccv_dt == abi.CCV_16F else x)
    assert nnc.cmd_exec(fwd, None, 0, [tq, tk, tv], [to, tl], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    got = to.download()
    got = _from_bf16(got) if ccv_dt == abi.CCV_16BF else got.astype(np.float32)
    assert_close(got, o64, 1e-2, "flash attention output")
    assert_close(tl.download(), lse64, 1e-3, "log-sum-exp")
    for t in (tq, tk, tv, to, tl, stream):
        t.free()


BWD16 = [
    # B, Sq, Sk, Hq, Hk, causal, dtype, saved (pass the forward's o / lse as inputs[9], [10]), D
    (1, 128, 128, 2, 2, 0, "bf16", 0, 128), (2, 64, 96, 4, 2, 1, "bf16", 0, 128), (1, 256, 256, 2, 2, 1, "bf16", 1, 128), (2, 200, 328, 4, 1, 0, "bf16", 1, 128),
    (1, 328, 200, 2, 2, 1, "bf16", 0, 128), (1, 96, 160, 8, 2, 1, "f16", 1, 128), (1, 1024, 1024, 2, 1, 0, "bf16", 1, 128), (1, 40, 24, 2, 2, 1, "f16", 0, 128),
    # head dimensions below 128 (the reference trials 40 and 64, test/int/nnc/cublas.tests.c:2752-2833): same kernels, zero-filled features
    (2, 160, 224, 4, 2, 1, "bf16", 1, 64), (1, 136, 136, 2, 2, 0, "bf16", 0, 40), (1, 192, 128, 4, 4, 1, "f16", 1, 96),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,causal,dtype,saved,D", BWD16)
def test_attention_16bit_backward_fused(gpu, ref, B, Sq, Sk, Hq, Hk, causal, dtype, saved, D):
    """bf16 / fp16 SDPA backward, D <= 128: the fused deterministic wgmma kernels (sm100_fmha_bwd.cu) against CPU_REF's fp32 backward
    (…attention_cpu_ref.c:259-479) on the rounded operands; 1e-2 of max|ref| (P and dS are rounded to 16 bits on the way, like the
    reference's flash-attention backward).  Covers GQA (dk / dv summed over the query heads), causal with Sq != Sk (bottom-right
    aligned, Sq > Sk leaves fully masked rows), ragged tiles, with and without the forward's saved output / log-sum-exp, and that two
    runs are bit-identical."""
    nnc = gpu
    scale = 1.0 / np.sqrt(D)
    arrs = [seeded((B, Sq, Hq, D), 4, -1, 1), None, None, seeded((B, Sq, Hq, D), 1, -1, 1), seeded((B, Sk, Hk, D), 2, -1, 1), seeded((B, Sk, Hk, D), 3, -1, 1)]
    if dtype == "bf16":
        ccv_dt = abi.CCV_16BF
        bits = [None if a is None else _to_bf16(a) for a in arrs]
        vals = [None if b is None else _from_bf16(b) for b in bits]
        back = _from_bf16
    else:
        ccv_dt = abi.CCV_16F
        bits = [None if a is None else a.astype(np.float16) for a in arrs]
        vals = [None if b is None else b.astype(np.float32) for b in bits]
        back = lambda x: x.astype(np.float32)
    bwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD, scale, causal)
    bwd.info.scaled_dot_product_attention.deterministic = 1
    st_r, (dq_r, dk_r, dv_r) = ref_exec(ref, bwd, None, 0, vals, [np.zeros_like(vals[3]), np.zeros_like(vals[4]), np.zeros_like(vals[5])])
    assert st_r == 0
    stream = nnc.Stream(0)
    ins = [None if b is None else nnc.gpu_tensor(list(b.shape), datatype=ccv_dt).upload(b) for b in bits]
    extra = []
    if saved:
        to = nnc.gpu_tensor([B, Sq, Hq, D], datatype=ccv_dt)
        tl = nnc.gpu_tensor([B, Hq, Sq])
        fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, causal)
        assert nnc.cmd_exec(fwd, None, 0, [ins[3], ins[4], ins[5]], [to, tl], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        ins = ins + [None, None, None, to, tl]
        extra = [to, tl]
    outs = [nnc.gpu_tensor(list(vals[i].shape), datatype=ccv_dt) for i in (3, 4, 5)]
    launches = nnc.lib().ccv_nnc_sm100_launch_count()
    assert nnc.cmd_exec(bwd, None, 0, ins, outs, stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    assert nnc.lib().ccv_nnc_sm100_launch_count() - launches == (3 if saved else 4), "the fused path is prep + dK/dV + dQ (+ the forward when o / lse are not passed)"
    first = [t.download().copy() for t in outs]
    for t, want, name in zip(outs, (dq_r, dk_r, dv_r), ("dq", "dk", "dv")):
        assert_close(back(t.download()), want, 1e-2, "%s %s" % (dtype, name))
    for t in outs:
        t.upload(np.zeros(t.dims, np.uint16 if ccv_dt == abi.CCV_16BF else np.float16))
    assert nnc.cmd_exec(bwd, None, 0, ins, outs, stream) == 0
    stream.wait()
    for t, a in zip(outs, first):
        assert np.array_equal(t.download().view(np.uint16), a.view(np.uint16)), "the backward must be run-to-run identical"
    for t in [x for x in ins if x is not None] + outs + [stream]:
        t.free()


@pytest.mark.parametrize("D,masked,causal", [(40, 0, 0), (64, 0, 1), (96, 0, 0), (160, 0, 0), (224, 0, 1), (128, 1, 0)])
def test_attention_16bit_forward_other_head_dims_and_masks(gpu, ref, D, masked, causal):
    """Head dimensions the reference trials (40, 64, 160, 224: test/int/nnc/cublas.tests.c:2752-2833) and additive masks on bf16
    tensors.  D <= 128 without a mask runs on the wgmma flash kernel (one launch: the tiles stay 128 features wide, the TMA unit
    zero-fills the rest); D > 128 and masks take the functional form (widen -> fp32 path -> narrow) instead of returning NO_KERNEL.
    Against CPU_REF on the bf16-rounded operands, 1e-2 of max|ref|."""
    nnc = gpu
    B, S, H = 2, 48, 4
    scale = 1.0 / np.sqrt(D)
    bits = [_to_bf16(seeded((B, S, H, D), i + 1, -1, 1)) for i in range(3)]
    q, k, v = (_from_bf16(b) for b in bits)
    fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, scale, causal)
    mask = None
    if masked:
        mask = np.where(np.random.RandomState(5).rand(1, 1, S, S) < 0.3, -1e9, 0.0).astype(np.float32)
        mask[..., np.arange(S), np.arange(S)] = 0
    ins_r = [q, k, v] + ([mask] if masked else [])
    st_r, (o_r, _) = ref_exec(ref, fwd, None, 0, ins_r, [np.zeros((B, S, H, D), np.float32), None])
    assert st_r == 0
    stream = nnc.Stream(0)
    tq, tk, tv = (nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF).upload(b) for b in bits)
    to = nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF)
    tm = nnc.gpu_tensor(list(mask.shape)).upload(mask) if masked else None
    launches = nnc.lib().ccv_nnc_sm100_launch_count()
    assert nnc.cmd_exec(fwd, None, 0, [tq, tk, tv] + ([tm] if masked else []), [to], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    if D <= 128 and not masked:
        assert nnc.lib().ccv_nnc_sm100_launch_count() - launches == 1, "the flash kernel covers this head dimension"
    assert_close(_from_bf16(to.download()), o_r, 1e-2, "bf16 attention D=%d" % D)
    for t in (tq, tk, tv, to, stream) + ((tm,) if masked else ()):
        t.free()


def test_baseline_config5_slices_vs_compiled_reference(gpu, ref):
    """BASELINE.json configs[4] at FULL size on the GPU (bf16, B=32 H=16 S=2048 D=128, non-causal and causal, the reference's
    i / count ramps of test/int/nnc/cublas.tests.c:2786-2794) with four (b, h) slices of the result checked against the compiled
    reference itself (CPU_REF run per slice on the bf16-rounded values: O(S^2) scratch per slice is what makes the whole tensor
    unaffordable on the CPU), 1e-2 of max|ref|."""
    nnc = gpu
    B, H, S, D = 32, 16, 2048, 128
    n = B * S * H * D
    bits = _to_bf16((np.arange(n, dtype=np.float64) / n).astype(np.float32)).reshape(B, S, H, D)
    vals = _from_bf16(bits)
    stream = nnc.Stream(0)
    tq, tk, tv, to = (nnc.gpu_tensor([B, S, H, D], datatype=abi.CCV_16BF) for _ in range(4))
    for t in (tq, tk, tv):
        t.upload(bits)
    tl = nnc.gpu_tensor([B, H, S])
    for causal in (0, 1):
        fwd = _cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD, 1.0 / np.sqrt(D), causal)
        assert nnc.cmd_exec(fwd, None, 0, [tq, tk, tv], [to, tl], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        got = _from_bf16(to.download())
        for b, h in ((0, 0), (7, 3), (19, 15), (31, 8)):
            sl = np.ascontiguousarray(vals[b:b + 1, :, h:h + 1, :])
            st_r, (o_r, _) = ref_exec(ref, fwd, None, 0, [sl, sl, sl], [np.zeros((1, S, 1, D), np.float32), None])
            assert st_r == 0
            assert_close(got[b:b + 1, :, h:h + 1, :], o_r, 1e-2, "configs[4] slice (b=%d, h=%d) causal=%d" % (b, h, causal))
    for t in (tq, tk, tv, to, tl, stream):
        t.free()
