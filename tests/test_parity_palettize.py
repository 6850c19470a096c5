"""Palettized (CCV_QX) weights: the format, the GPU decoder, the commands that accept them and the fused few-row GEMM.

tests/palette_ref.py restates the format in NumPy.  The CPU tests pin it to the reference's own encoder and decoder, through the
fixture tests/golden/cpuref_palettize.npz (made by tests/golden/make_palettize_golden.py) and, where it is built, through
oracle/_ref/libccv_ref.so.  The GPU tests hold the backend to that format:
  - ccv_nnc_depalettize equals the reference's decoder bit for bit, also for a q = 8 weight with more than 2^32 index bits;
  - every command that accepts a palettized operand gives, on the unfused path, the bits of the same command on the decoded tensor;
  - the fused few-row GEMM (fp16 activations, [N, K] weights with fp16 palettes, M <= M_MAX rows) is held to contract_ref's 16-bit
    bound on the decoded operands, runs as one launch, and gives the same bits twice;
  - every refused call returns CCV_NNC_EXEC_INVALID and leaves its outputs untouched."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi
from tests import contract_ref as cr
from tests import palette_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "cpuref_palettize.npz")
NHWC, NCHW = abi.CCV_TENSOR_FORMAT_NHWC, abi.CCV_TENSOR_FORMAT_NCHW
CCV_DT = {np.dtype(np.float16): abi.CCV_16F, np.dtype(np.float32): abi.CCV_32F, np.dtype(np.float64): abi.CCV_64F}
INVALID = -1  # CCV_NNC_EXEC_INVALID


def m_max():
    """PALETTIZED_GEMM_M_MAX of ccv_b200/csrc/sm100_contract.h."""
    src = open(os.path.join(ROOT, "ccv_b200", "csrc", "sm100_contract.h")).read()
    return int(re.search(r"PALETTIZED_GEMM_M_MAX = (\d+);", src).group(1))


M_MAX = m_max()


def fused_plan(M, N, K, a_dt, w_palette, out_dt, transpose_w, w_batched=False, a_palettized=False):
    """Restates gemm_fused_qx_plan (ccv_b200/csrc/sm100_backend.cu): True when GEMM_FORWARD runs the fused few-row kernel."""
    return (not a_palettized and not w_batched and transpose_w and a_dt == np.float16 and out_dt == np.float16 and w_palette == np.float16 and 1 <= M <= M_MAX)


def planned_launches(fused, palettized_operands, dense_launches):
    """Fused: the one kernel.  Unfused: one decoder launch per palettized operand, then the dense command's launches."""
    return 1 if fused else palettized_operands + dense_launches


def fixture_cases():
    z = np.load(FIXTURE)
    for k in sorted(z.files):
        if k.endswith("_enc"):
            q, dt, count, nib = re.match(r"q(\d)_(\w+?)_n(\d+)_b(\d+)_enc", k).groups()
            yield int(q), np.dtype(dt).type, int(count), int(nib), z[k], z[k[:-4] + "_dec"]


# ================================================================================================ CPU: the format
def test_palette_ref_reproduces_the_reference_encoder_and_decoder():
    n = 0
    for q, dt, count, nib, enc, dec in fixture_cases():
        idx, pal = pr.unpack(enc, q, nib, count, dt)
        assert np.array_equal(pr.pack(idx, pal, q, nib), enc), (q, dt, count, nib)
        assert np.array_equal(pr.decode(enc, q, nib, count, dt).view(np.uint8), dec.view(np.uint8)), (q, dt, count, nib)
        # the tensor's bytes (up to ceil(count * q / 8) index bytes) decode the same as the encoder's
        size = pr.data_size(count, q, nib, np.dtype(dt).itemsize)
        assert np.array_equal(pr.decode(enc[:size], q, nib, count, dt).view(np.uint8), dec.view(np.uint8))
        n += 1
    assert n == 5 * 3 * 4
    qs = set((q, count % 8 != 0, count % nib != 0, nib > count) for q, _, count, nib, _, _ in fixture_cases())
    assert {q for q, _, _, _ in qs} == {4, 5, 6, 7, 8} and any(p for _, p, _, _ in qs) and any(p for _, _, p, _ in qs) and any(p for _, _, _, p in qs)


@pytest.mark.ref
def test_palette_ref_against_the_compiled_reference():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref/libccv_ref.so not built")
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libccv_ref.so"))
    lib.ccv_nnc_palettize.restype = C.c_size_t
    lib.ccv_nnc_palettize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.ccv_nnc_depalettize.restype = None
    lib.ccv_nnc_depalettize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    for q in range(4, 9):
        for dt in pr.PALETTE_TYPES:
            for count, nib in ((777, 96), (41, 1024), (2048, 256)):
                x = np.random.RandomState(q * 7 + count).uniform(-3, 3, count).astype(dt)
                size = pr.encoded_size(count, q, nib, np.dtype(dt).itemsize)
                enc = np.zeros(size + 64, np.uint8)
                assert lib.ccv_nnc_palettize(x.ctypes.data, CCV_DT[np.dtype(dt)], 1, count, q, nib, enc.ctypes.data, enc.size) == size
                dec = np.zeros(count, dt)
                lib.ccv_nnc_depalettize(enc.ctypes.data, CCV_DT[np.dtype(dt)], 1, size, q, nib, dec.ctypes.data, count)
                idx, pal = pr.unpack(enc[:size], q, nib, count, dt)
                assert np.array_equal(pr.pack(idx, pal, q, nib), enc[:size])
                assert np.array_equal(pr.decode(enc[:size], q, nib, count, dt).view(np.uint8), dec.view(np.uint8))


def test_host_data_size_is_the_reference_formula():
    from ccv_b200 import nnc
    for q in range(4, 9):
        for dt in pr.PALETTE_TYPES:
            for dims, nib in (([1000], 128), ([37, 41], 64), ([3, 5, 7, 11], 2048), ([4096, 4096], 128), ([1 << 29], 4096)):
                count = int(np.prod(dims))
                p = nnc.palettize_param(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, NHWC, CCV_DT[np.dtype(dt)], dims), q, nib)
                assert (p.datatype & 0xFF000) == abi.CCV_QX and (p.datatype >> 8) & 0xF == q and (p.datatype & 0xFF) << 12 == CCV_DT[np.dtype(dt)] and p.reserved == nib
                want = pr.data_size(count, q, nib, np.dtype(dt).itemsize)
                assert nnc.lib().ccv_nnc_tensor_data_size_without_padding(p) == want
                assert nnc.tensor_data_size(p) == (want + 63) // 64 * 64


QX_COMMANDS = {"GEMM_FORWARD", "GEMM_BACKWARD", "CONVOLUTION_FORWARD", "CONVOLUTION_BACKWARD", "CONVOLUTION_TRANSPOSE_FORWARD",
               "CONVOLUTION_TRANSPOSE_BACKWARD", "SCALED_DOT_PRODUCT_ATTENTION_FORWARD", "DATA_TRANSFER_FORWARD", "DATA_TRANSFER_BACKWARD"}


def test_registry_reports_qx_for_exactly_the_weight_commands():
    from ccv_b200 import nnc
    nnc.init()
    l = nnc.lib()
    l.ccv_nnc_cmd_find_backend.restype = C.c_uint32
    l.ccv_nnc_cmd_find_backend.argtypes = [abi.Cmd, C.c_int, C.c_int, C.c_int]
    ids = dict((n[len("CCV_NNC_"):], getattr(abi, n)) for n in dir(abi) if n.startswith("CCV_NNC_") and (n.endswith("_FORWARD") or n.endswith("_BACKWARD")))
    with_qx = set()
    for name, cid in ids.items():
        if not l.ccv_nnc_cmd_ok(cid, abi.CCV_NNC_BACKEND_GPU_SM100):
            continue
        cmd = abi.Cmd()
        cmd.cmd, cmd.backend, cmd.algorithm = cid, 0, -1
        if l.ccv_nnc_cmd_find_backend(cmd, abi.CCV_TENSOR_GPU_MEMORY, NHWC, abi.CCV_QX) == abi.CCV_NNC_BACKEND_GPU_SM100:
            with_qx.add(name)
    assert with_qx == QX_COMMANDS


def test_selection_restatement():
    assert M_MAX >= 1
    f16 = np.float16
    assert fused_plan(1, 4096, 4096, f16, f16, f16, True) and fused_plan(M_MAX, 5, 3, f16, f16, f16, True)
    assert [M for M, q, nib, K, N, bias in FUSED_CASES if fused_plan(M, N, K, f16, f16, f16, True)]
    assert not fused_plan(M_MAX + 1, 4096, 4096, f16, f16, f16, True)
    assert not fused_plan(1, 64, 64, f16, f16, f16, False)            # [K, N] weights
    assert not fused_plan(1, 64, 64, np.float32, np.float32, np.float32, True)
    assert not fused_plan(1, 64, 64, f16, f16, f16, True, w_batched=True)
    assert not fused_plan(1, 64, 64, f16, f16, f16, True, a_palettized=True)
    assert planned_launches(True, 1, 5) == 1 and planned_launches(False, 2, 1) == 3


def _fused_oracle(a, wdense, bias):
    """(ref, s) in float64 on the fp16 operands the kernel decodes; K_eff = K."""
    return cr.gemm(a.astype(np.float64), wdense.astype(np.float64), False, True, None if bias is None else bias.astype(np.float64))


def _fused_like(a, w, bias):
    """A correct fused result: fp32-accurate sum, rounded once to fp16."""
    y, _ = _fused_oracle(a, w, bias)
    return y.astype(np.float16)


@pytest.mark.parametrize("q,nib,K,N", [(4, 128, 256, 33), (5, 48, 200, 17), (8, 100, 97, 9), (6, 4, 130, 12)])
def test_fused_bound_rejects_decoder_defects(q, nib, K, N):
    """Each modelled decoder defect, applied to the weight bytes, puts elements outside the bound the GPU test applies."""
    M = 3
    data, w = pr.random_palettized(N * K, q, nib, np.float16, seed=q * 31 + nib)
    w = w.reshape(N, K)
    a = cr.operand((M, K), 5, cr.FP16).astype(np.float16)
    ref, s = _fused_oracle(a, w, None)
    assert cr.admits(_fused_like(a, w, None).astype(np.float64), ref, s, K, cr.FP16, cr.FP16).all()
    idx, pal = pr.unpack(data, q, nib, N * K, np.float16)
    blocks = pal.shape[0]
    bad = {}
    shifted = np.roll(idx, 1)  # every index read one position off
    bad["index one position off"] = pal[np.arange(N * K) // nib, shifted]
    neighbour = np.minimum(np.arange(N * K) // nib + 1, blocks - 1)  # the next block's palette (the last block keeps its own)
    bad["neighbouring palette"] = pal[neighbour, idx]
    rev = np.zeros_like(idx)
    for b in range(q):
        rev |= ((idx >> b) & 1) << (q - 1 - b)
    bad["bit order reversed"] = pal[np.arange(N * K) // nib, rev]
    if q == 4:
        swapped = idx.reshape(-1, 2)[:, ::-1].reshape(-1) if (N * K) % 2 == 0 else idx
        bad["nibbles swapped"] = pal[np.arange(N * K) // nib, swapped]
    dropped = pal[np.arange(N * K) // nib, idx].copy()
    tail = (N * K) % nib or nib
    dropped[-tail:] = 0
    bad["last block dropped"] = dropped
    for what, wd in bad.items():
        y = _fused_like(a, wd.reshape(N, K).astype(np.float16), None)
        assert not cr.admits(y.astype(np.float64), ref, s, K, cr.FP16, cr.FP16).all(), what


# ================================================================================================ GPU helpers
def _qx_tensor(nnc, data, dims, palette_dt, q, nib, fmt=NHWC):
    t = nnc.gpu_palettized_tensor(list(dims), CCV_DT[np.dtype(palette_dt)], q, nib, fmt)
    t.upload(data[:t.nbytes])
    return t


def _dense(nnc, arr, fmt=NHWC):
    t = nnc.gpu_tensor(list(arr.shape), fmt, CCV_DT[arr.dtype])
    t.upload(arr)
    return t


def _run(nnc, cmd, hint, flags, ins, outs):
    """cmd_exec on tensors; returns (status, downloaded outputs, launches)."""
    l0 = nnc.launch_count()
    st = nnc.cmd_exec(cmd, hint, flags, ins, outs)
    nnc.lib().ccv_nnc_stream_context_wait(None)
    return st, [None if t is None else t.download() for t in outs], nnc.launch_count() - l0


def _free(*ts):
    for t in ts:
        if t is not None:
            t.free()


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(np.uint8)


# ================================================================================================ GPU: the decoder
@pytest.mark.gpu
def test_depalettize_equals_the_reference_decoder(gpu):
    nnc = gpu
    l = nnc.lib()
    guard = 64
    for q, dt, count, nib, enc, dec in fixture_cases():
        src = _qx_tensor(nnc, enc, [count], dt, q, nib)
        it = np.dtype(dt).itemsize
        dst = nnc.gpu_tensor([count + 2 * guard], NHWC, CCV_DT[np.dtype(dt)])
        sentinel = np.full(count + 2 * guard, np.nan, dt)
        dst.upload(sentinel)
        l.ccv_nnc_depalettize(src.data_ptr, CCV_DT[np.dtype(dt)], abi.CCV_TENSOR_GPU_MEMORY, src.nbytes, q, nib, dst.data_ptr + guard * it, count)
        l.ccv_nnc_stream_context_wait(None)
        got = dst.download()
        assert np.array_equal(_bits(got[guard:guard + count]), _bits(dec)), (q, dt, count, nib)
        assert np.array_equal(_bits(got[:guard]), _bits(sentinel[:guard])) and np.array_equal(_bits(got[guard + count:]), _bits(sentinel[:guard]))
        _free(src, dst)


@pytest.mark.gpu
def test_depalettize_refusals_leave_the_output_untouched(gpu):
    nnc = gpu
    l = nnc.lib()
    data, _ = pr.random_palettized(256, 8, 64, np.float16, 1)
    src = _qx_tensor(nnc, data, [256], np.float16, 8, 64)
    dst = nnc.gpu_tensor([256], NHWC, abi.CCV_16F)
    sentinel = np.full(256, 7.0, np.float16)
    dst.upload(sentinel)
    for q, nib, dtype in ((3, 64, abi.CCV_16F), (9, 64, abi.CCV_16F), (5, 12, abi.CCV_16F), (7, 4, abi.CCV_16F), (8, 0, abi.CCV_16F), (8, 64, abi.CCV_16BF)):
        l.ccv_nnc_depalettize(src.data_ptr, dtype, abi.CCV_TENSOR_GPU_MEMORY, src.nbytes, q, nib, dst.data_ptr, 256)
        l.ccv_nnc_stream_context_wait(None)
        assert np.array_equal(_bits(dst.download()), _bits(sentinel)), (q, nib, dtype)
    _free(src, dst)


@pytest.mark.gpu
def test_depalettize_more_than_2_to_32_index_bits(gpu):
    """q = 8, 2^29 + 1000 fp16 elements: bit offsets past 2^32; the first, a middle and the last blocks are checked."""
    nnc = gpu
    l = nnc.lib()
    q, nib = 8, 4096
    count = (1 << 29) + 1000
    blocks = pr.num_blocks(count, nib)
    r = np.random.RandomState(29)
    idx = np.resize(r.randint(0, 256, 1048583).astype(np.uint8), count)  # period prime to the block size
    pal = (np.arange(blocks, dtype=np.float32)[:, None] % 509 / 256 + np.arange(256, dtype=np.float32)[None, :] / 1024).astype(np.float16)
    full = count // nib
    body = np.concatenate([pal[:full].view(np.uint8).reshape(full, 512), idx[:full * nib].reshape(full, nib)], axis=1).reshape(-1)
    data = np.concatenate([body, pal[full].view(np.uint8), idx[full * nib:]])
    del body
    assert data.size == pr.data_size(count, q, nib, 2)
    src = _qx_tensor(nnc, data, [count], np.float16, q, nib)
    del data
    dst = nnc.gpu_tensor([count + 64], NHWC, abi.CCV_16F)
    l.ccv_nnc_sm100_memcpy_h2d(dst.data_ptr + count * 2, np.full(64, np.nan, np.float16).ctypes.data, 128, None)
    l.ccv_nnc_depalettize(src.data_ptr, abi.CCV_16F, abi.CCV_TENSOR_GPU_MEMORY, src.nbytes, q, nib, dst.data_ptr, count)
    l.ccv_nnc_stream_context_wait(None)
    for lo in (0, (1 << 28) + 12345, (1 << 29) - 3 * nib - 17, count - 1500):
        n = min(10000, count + 64 - lo)
        got = np.empty(n, np.float16)
        assert l.ccv_nnc_sm100_memcpy_d2h(got.ctypes.data, dst.data_ptr + lo * 2, n * 2, None) == 0
        e = np.arange(lo, lo + n)
        inside = e < count
        want = pal[e[inside] // nib, idx[e[inside]]]
        assert np.array_equal(_bits(got[inside]), _bits(want)), lo
        assert np.isnan(got[~inside].astype(np.float32)).all()
    _free(src, dst)


@pytest.mark.gpu
def test_data_transfer_round_trips_palettized_bytes(gpu):
    nnc = gpu
    for q, dt, count, nib in ((4, np.float16, 1000, 128), (7, np.float32, 517, 64), (8, np.float64, 203, 20)):
        data, _ = pr.random_palettized(count, q, nib, dt, q)
        h = nnc.cpu_palettized_tensor([count], CCV_DT[np.dtype(dt)], q, nib)
        h.upload(data)
        g1 = nnc.gpu_palettized_tensor([count], CCV_DT[np.dtype(dt)], q, nib)
        g2 = nnc.gpu_palettized_tensor([count], CCV_DT[np.dtype(dt)], q, nib)
        h2 = nnc.cpu_palettized_tensor([count], CCV_DT[np.dtype(dt)], q, nib)
        for a, b in ((h, g1), (g1, g2), (g2, h2)):
            assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [a], [b]) == 0
        assert np.array_equal(h2.download(), data) and np.array_equal(g2.download(), data)
        # the two sides must carry the same datatype word and block size
        other = nnc.gpu_palettized_tensor([count], CCV_DT[np.dtype(dt)], q, nib * 2)
        before = other.download()
        assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [g1], [other]) == INVALID
        assert np.array_equal(other.download(), before)
        _free(h, g1, g2, h2, other)


# ================================================================================================ GPU: unfused identity
ALGOS = {"tf32": abi.CCV_NNC_SM100_ALGO_TF32, "3xtf32": abi.CCV_NNC_SM100_ALGO_3XTF32, "ffma": abi.CCV_NNC_SM100_ALGO_FFMA, "fp16": -1}


def _identity(nnc, make_cmd, hint, flags, ins, outs, qx_at, what, launches=None):
    """Run `make_cmd()` once with inputs qx_at[i] = (bytes, dims, palette type, q, nib, fmt) palettized and once on the decoded dense
    tensors (ins[i] holds them); the outputs must match bit for bit."""
    dense_in = [None if a is None else (_dense(nnc, a[0], a[1]) if isinstance(a, tuple) else _dense(nnc, a)) for a in ins]
    qx_in = list(dense_in)
    for i, spec in qx_at.items():
        qx_in[i] = _qx_tensor(nnc, *spec)
    res = []
    for tensors in (dense_in, qx_in):
        out_t = [None if o is None else _dense(nnc, o[0], o[1]) for o in outs]
        st, got, n = _run(nnc, make_cmd(), hint, flags, tensors, out_t)
        assert st == 0, (what, st, nnc.lib().ccv_nnc_sm100_last_error())
        res.append((got, n))
        _free(*out_t)
    for a, b in zip(res[0][0], res[1][0]):
        if a is not None:
            assert np.array_equal(_bits(a), _bits(b)), what
    assert res[1][1] == res[0][1] + len(qx_at), (what, res)
    _free(*set(dense_in + qx_in))


def _qx_of(shape, dt, q, nib, seed, fmt=NHWC, scale=1.0):
    """(palettized bytes spec for _qx_tensor, decoded dense array)"""
    count = int(np.prod(shape))
    data, dense = pr.random_palettized(count, q, nib, dt, seed, scale)
    return (data, list(shape), dt, q, nib, fmt), dense.reshape(shape)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", list(ALGOS))
def test_gemm_forward_unfused_identity(gpu, algo):
    nnc = gpu
    dt = np.float16 if algo == "fp16" else np.float32
    M, K, N = 40, 96, 72
    for ta in (0, 1):
        for tb in (0, 1):
            a_shape = (K, M) if ta else (M, K)
            w_shape = (N, K) if tb else (K, N)
            a_spec, a = _qx_of(a_shape, dt, 5, 64, 1)
            w_spec, w = _qx_of(w_shape, dt, 4, 128, 2)
            bias = (np.arange(N) / 16).astype(dt)
            out = [(np.zeros((M, N), dt), NHWC)]
            mk = lambda: nnc.CMD_GEMM_FORWARD((0, 1) if ta else (0, 0), (0, 1) if tb else (0, 0), algorithm=ALGOS[algo])
            _identity(nnc, mk, None, 0, [a, w, bias], out, {1: w_spec}, "w %s %d%d" % (algo, ta, tb))
            _identity(nnc, mk, None, 0, [a, w, bias], out, {0: a_spec}, "a %s %d%d" % (algo, ta, tb))
            _identity(nnc, mk, None, 0, [a, w, None], out, {0: a_spec, 1: w_spec}, "a+w %s %d%d" % (algo, ta, tb))
    # batched activations [2, M, K] against one palettized [N, K] weight
    a = cr.operand((2, M, K), 3, cr.FP16 if dt == np.float16 else cr.FP32).astype(dt)
    w_spec, w = _qx_of((N, K), dt, 6, 96, 4)
    _identity(nnc, lambda: nnc.CMD_GEMM_FORWARD((0, 0), (0, 1), algorithm=ALGOS[algo]), None, 0, [a, w, None], [(np.zeros((2, M, N), dt), NHWC)], {1: w_spec}, "batched " + algo)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", list(ALGOS))
def test_gemm_backward_unfused_identity(gpu, algo):
    nnc = gpu
    dt = np.float16 if algo == "fp16" else np.float32
    M, K, N = 48, 80, 64
    g = cr.operand((M, N), 7, cr.FP16 if dt == np.float16 else cr.FP32).astype(dt)
    a_spec, a = _qx_of((M, K), dt, 7, 64, 8)
    w_spec, w = _qx_of((N, K), dt, 8, 40, 9)
    mk = lambda: nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1), algorithm=ALGOS[algo])
    outs = [(np.zeros((M, K), dt), NHWC), (np.zeros((N, K), dt), NHWC), (np.zeros((N,), dt), NHWC)]
    _identity(nnc, mk, None, 0, [g, a, w], outs, {1: a_spec, 2: w_spec}, "h+dw " + algo)
    _identity(nnc, mk, None, 0, [g, a, w], [outs[0], None, None], {2: w_spec}, "h " + algo)
    _identity(nnc, mk, None, 0, [g, a, None], [None, outs[1], None], {1: a_spec}, "dw " + algo)


def _conv_cases(dt):
    # (N, H, W, C, K, R, groups, stride, fmt)
    yield 2, 9, 11, 16, 24, 3, 1, 1, NHWC
    yield 2, 8, 8, 32, 32, 3, 2, 2, NHWC
    yield 1, 10, 9, 16, 16, 3, 1, 1, NCHW
    yield 1, 7, 7, 16, 32, 1, 1, 1, NCHW


@pytest.mark.gpu
@pytest.mark.parametrize("algo", list(ALGOS))
def test_convolution_unfused_identity(gpu, algo):
    nnc = gpu
    dt = np.float16 if algo == "fp16" else np.float32
    mode = cr.FP16 if dt == np.float16 else cr.FP32
    for i, (N, H, W, C, K, R, groups, stride, fmt) in enumerate(_conv_cases(dt)):
        P, Q = (H + 2 * (R // 2) - R) // stride + 1, (W + 2 * (R // 2) - R) // stride + 1
        shp = (lambda n, h, w, c: (n, c, h, w) if fmt == NCHW else (n, h, w, c))
        wshape = (K, C // groups, R, R) if fmt == NCHW else (K, R, R, C // groups)
        x = cr.operand(shp(N, H, W, C), 10 + i, mode).astype(dt)
        w_spec, w = _qx_of(wshape, dt, 4 + i, 64, 20 + i, fmt, scale=0.25)
        bias = (np.arange(K) / 32).astype(dt)
        hint = abi.hint((stride, stride), (R // 2, R // 2))
        mk = lambda: nnc.CMD_CONVOLUTION_FORWARD(groups, K, R, R, C // groups, algorithm=ALGOS[algo])
        _identity(nnc, mk, hint, 0, [(x, fmt), (w, fmt), bias], [(np.zeros(shp(N, P, Q, K), dt), fmt)], {1: w_spec}, "conv fwd %s %d" % (algo, i))
        g = cr.operand(shp(N, P, Q, K), 30 + i, mode).astype(dt)
        mkb = lambda: nnc.CMD_CONVOLUTION_BACKWARD(groups, K, R, R, C // groups, algorithm=ALGOS[algo])
        _identity(nnc, mkb, hint, 0, [(g, fmt), (x, fmt), (w, fmt)], [(np.zeros(shp(N, H, W, C), dt), fmt), (np.zeros(wshape, dt), fmt), (np.zeros(K, dt), fmt)],
                  {2: w_spec}, "conv bwd %s %d" % (algo, i))
        # the transposed convolution reads its filters as [Cin, R, S, Cout / groups]: the small side x has K channels
        tw_spec, tw = _qx_of((K, R, R, C // groups) if fmt == NHWC else (K, C // groups, R, R), dt, 8 - i, 32, 40 + i, fmt, scale=0.25)
        a = cr.operand(shp(N, P, Q, K), 50 + i, mode).astype(dt)
        mkt = lambda: nnc.CMD_CONVOLUTION_TRANSPOSE_FORWARD(groups, C, 0, R, R, K, algorithm=ALGOS[algo])
        _identity(nnc, mkt, hint, 0, [(a, fmt), (tw, fmt), (np.arange(C) / 8).astype(dt)], [(np.zeros(shp(N, H, W, C), dt), fmt)], {1: tw_spec}, "convT fwd %s %d" % (algo, i))
        gy = cr.operand(shp(N, H, W, C), 60 + i, mode).astype(dt)
        mktb = lambda: nnc.CMD_CONVOLUTION_TRANSPOSE_BACKWARD(groups, C, 0, R, R, K, algorithm=ALGOS[algo])
        _identity(nnc, mktb, hint, 0, [(gy, fmt), (a, fmt), (tw, fmt)], [(np.zeros(shp(N, P, Q, K), dt), fmt), None, None], {2: tw_spec}, "convT bwd %s %d" % (algo, i))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [np.float16, np.float32])
def test_sdpa_unify_head_unfused_identity(gpu, dt):
    nnc = gpu
    B, S, H, D = 2, 64, 2, 64
    mode = cr.FP16 if dt == np.float16 else cr.FP32
    q, k, v = (cr.operand((B, S, H, D), 70 + i, mode, -1, 1).astype(dt) for i in range(3))
    w_spec, w = _qx_of((H * D, H * D), dt, 6, 128, 73, scale=0.1)
    bias = (np.arange(H * D) / 64).astype(dt)
    def mk():
        c = nnc._simple(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD)
        c.info.scaled_dot_product_attention.scale = 1.0 / np.sqrt(D)
        return c
    outs = [(np.zeros((B, S, H * D), dt), NHWC), None, (np.zeros((B, S, H, D), dt), NHWC)]
    _identity(nnc, mk, None, 0, [q, k, v, None, w, bias], outs, {4: w_spec}, "sdpa %s" % np.dtype(dt).name)


# ================================================================================================ GPU: the fused kernel
# M = 1, 2, 7, 16 and M_MAX; those above M_MAX take the unfused path and are held to the same bound
FUSED_CASES = [(M, q, nib, K, N, bias) for M, q, nib, K, N, bias in [
    (1, 4, 128, 1024, 257, None), (2, 5, 128, 640, 96, "f16"), (7, 6, 96, 1000, 65, "f32"), (16, 7, 64, 1024, 64, None),
    (M_MAX, 8, 4096, 1536, 33, "f16"), (M_MAX, 8, 100, 1030, 31, "f32"), (M_MAX, 4, 2, 997, 19, None), (M_MAX, 6, 12, 999, 40, "f16"),
    (M_MAX, 5, 24, 333, 7, None), (M_MAX, 4, 128, 96, 128, None), (M_MAX, 4, 6, 4100, 9, "f32"), (M_MAX, 7, 8, 1000, 3, "f16")]]


@pytest.mark.gpu
@pytest.mark.parametrize("M,q,nib,K,N,bias", FUSED_CASES)
def test_fused_gemm_bound_and_launches(gpu, M, q, nib, K, N, bias):
    """nib divides K (1024 / 128), does not (1000 / 96, 997 / 2), exceeds K (4096); odd N; K not a multiple of 8; palettes at odd
    addresses (q = 4, nib = 6: 3 index bytes per block)."""
    nnc = gpu
    fused = fused_plan(M, N, K, np.float16, np.float16, np.float16, True)
    w_spec, w = _qx_of((N, K), np.float16, q, nib, M * 100 + q, scale=0.5)
    a = cr.operand((M, K), M + q, cr.FP16).astype(np.float16)
    b = None if bias is None else (np.arange(N) / 64 - 0.5).astype(np.float16 if bias == "f16" else np.float32)
    ref, s = _fused_oracle(a, w, b)
    guard = 5
    wt = _qx_tensor(nnc, *w_spec)
    at = _dense(nnc, a)
    bt = None if b is None else _dense(nnc, b)
    buf = nnc.gpu_tensor([M * N + 2 * guard], NHWC, abi.CCV_16F)
    outs = []
    for rep in range(2):
        buf.upload(np.full(M * N + 2 * guard, np.nan, np.float16))
        ct = nnc.tensor_new(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, NHWC, abi.CCV_16F, [M, N]), buf.data_ptr + guard * 2)
        st, _, n = _run(nnc, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), None, 0, [at, wt, bt], [ct])
        assert st == 0, nnc.lib().ccv_nnc_sm100_last_error()
        assert (n == planned_launches(True, 1, None)) if fused else (n >= planned_launches(False, 1, 1)), (fused, n)
        got = buf.download()
        assert np.isnan(got[:guard].astype(np.float32)).all() and np.isnan(got[-guard:].astype(np.float32)).all()
        outs.append(got[guard:-guard].reshape(M, N))
        ct.free()
    assert np.array_equal(_bits(outs[0]), _bits(outs[1]))
    cr.check(outs[0].astype(np.float64), ref, s, K, cr.FP16, cr.FP16, "fused M=%d q=%d nib=%d K=%d N=%d" % (M, q, nib, K, N))
    _free(wt, at, bt, buf)


@pytest.mark.gpu
def test_fused_gemm_threshold_goes_unfused_above_m_max(gpu):
    nnc = gpu
    K, N = 256, 64
    w_spec, w = _qx_of((N, K), np.float16, 4, 128, 5)
    for M in (M_MAX, M_MAX + 1):
        a = cr.operand((M, K), M, cr.FP16).astype(np.float16)
        wt, at, ct = _qx_tensor(nnc, *w_spec), _dense(nnc, a), nnc.gpu_tensor([M, N], NHWC, abi.CCV_16F)
        st, (got,), n = _run(nnc, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), None, 0, [at, wt], [ct])
        assert st == 0
        ref, s = _fused_oracle(a, w, None)
        cr.check(got.astype(np.float64), ref, s, K, cr.FP16, cr.FP16, "M=%d" % M)
        if M <= M_MAX:
            assert n == 1
        else:
            assert n >= 2  # the decoder, then the dense GEMM
        _free(wt, at, ct)


# ================================================================================================ GPU: refusals
@pytest.mark.gpu
def test_refusals_leave_outputs_untouched(gpu):
    nnc = gpu
    M, K, N = 8, 64, 32
    a = cr.operand((M, K), 1, cr.FP16).astype(np.float16)
    a32 = a.astype(np.float32)
    w_spec, w = _qx_of((N, K), np.float16, 4, 64, 2)
    w32_spec, w32 = _qx_of((N, K), np.float32, 4, 64, 2)
    w64_spec, _ = _qx_of((N, K), np.float64, 4, 64, 2)
    cases = []
    # palette type differs from the activations
    cases.append(("palette fp32 / fp16 activations", nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), [a, w32_spec], np.float16, {1}))
    cases.append(("palette fp16 / fp32 activations", nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), [a32, w_spec], np.float32, {1}))
    cases.append(("fp64 palette", nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), [a32, w64_spec], np.float32, {1}))
    # bad parameters, written into a valid tensor's header: qbits outside 4..8, a block whose index bytes are not whole
    for q, nib in ((3, 64), (9, 64), (4, 3), (5, 12), (7, 4)):
        cases.append(("q %d nib %d" % (q, nib), nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), [a, w_spec + (q, nib)], np.float16, {1}))
    # a palettized bias is not a weight
    b_spec, _ = _qx_of((N,), np.float16, 4, 16, 3)
    cases.append(("palettized bias", nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), [a, w, b_spec], np.float16, {2}))
    for what, cmd, ins, dt, qx in cases:
        ts = []
        for i, x in enumerate(ins):
            if i in qx:
                t = _qx_tensor(nnc, *x[:6])
                if len(x) > 6:
                    info = C.cast(t.ptr, C.POINTER(abi.Tensor)).contents.info
                    info.datatype = (info.datatype & ~0xF00) | ((x[6] & 0xF) << 8)
                    info.reserved = x[7]
                ts.append(t)
            else:
                ts.append(_dense(nnc, x.astype(dt)))
        ct = nnc.gpu_tensor([M, N], NHWC, CCV_DT[np.dtype(dt)])
        before = np.full((M, N), 3.0, dt)
        ct.upload(before)
        st, (got,), n = _run(nnc, cmd, None, 0, ts, [ct])
        assert st == INVALID, (what, st)
        assert n == 0 and np.array_equal(_bits(got), _bits(before)), what
        _free(ct, *ts)
    # a palettized output, and a palettized operand where the command takes none
    ct = nnc.gpu_palettized_tensor([M, N], abi.CCV_16F, 4, 64)
    wt, at = _qx_tensor(nnc, *w_spec), _dense(nnc, a)
    before = ct.download()
    st, _, n = _run(nnc, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), None, 0, [at, wt], [ct])
    assert st == INVALID and n == 0 and np.array_equal(ct.download(), before)
    g = _dense(nnc, cr.operand((M, N), 4, cr.FP16).astype(np.float16))
    h = nnc.gpu_tensor([M, K], NHWC, abi.CCV_16F)
    h.upload(np.full((M, K), 3.0, np.float16))
    a_qx = _qx_tensor(nnc, *_qx_of((M, K), np.float16, 4, 64, 6)[0])
    st, (hh,), n = _run(nnc, nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1)), None, 0, [g, a_qx, wt], [h])  # a palettized a without dw
    assert st == INVALID and n == 0 and (hh == 3.0).all()
    relu_out = nnc.gpu_tensor([N, K], NHWC, abi.CCV_16F)
    assert nnc.cmd_exec(nnc.CMD_RELU_FORWARD(), None, 0, [wt], [relu_out]) != 0
    _free(ct, wt, at, g, h, a_qx, relu_out)
