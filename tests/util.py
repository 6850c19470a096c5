"""Shared helpers for the parity tests: run one command on the SM100 backend (through the C ABI) and on the oracle
(the reference's own CCV_NNC_BACKEND_CPU_REF) from the same numpy inputs."""
import numpy as np

from ccv_b200 import abi

NHWC = abi.CCV_TENSOR_FORMAT_NHWC
NCHW = abi.CCV_TENSOR_FORMAT_NCHW
NP_TO_CCV = {np.dtype(np.float32): abi.CCV_32F, np.dtype(np.int32): abi.CCV_32S, np.dtype(np.float64): abi.CCV_64F, np.dtype(np.float16): abi.CCV_16F, np.dtype(np.uint16): abi.CCV_16F, np.dtype(np.uint8): abi.CCV_8U}


def seeded(shape, seed, lo=0.0, hi=1.0, dtype=np.float32):
    """U(lo, hi] inputs, seeded (the reference's GPU-vs-CPU protocol, test/int/nnc/cudnn.tests.c:38-46, uses dSFMT seed 0)."""
    r = np.random.RandomState(seed)
    return (lo + (hi - lo) * (1.0 - r.random_sample(shape))).astype(dtype)


def gpu_exec(nnc, cmd, hint, flags, in_arrays, out_arrays, fmt=NHWC, in_fmts=None, out_fmts=None, stream=None):
    """Upload, ccv_nnc_cmd_exec on CCV_NNC_BACKEND_GPU_SM100, download. The same array object appearing in both lists
    (or twice) is the same GPU tensor (in-place ops). Returns (status, [output arrays])."""
    cache = {}

    def tensor_for(a, f):
        if a is None:
            return None
        if id(a) not in cache:
            t = nnc.gpu_tensor(list(a.shape), f, NP_TO_CCV[a.dtype])
            t.upload(a.view(np.float16) if a.dtype == np.uint16 else a)
            cache[id(a)] = t
        return cache[id(a)]

    ins = [tensor_for(a, in_fmts[i] if in_fmts else fmt) for i, a in enumerate(in_arrays)]
    outs = [tensor_for(a, out_fmts[i] if out_fmts else fmt) for i, a in enumerate(out_arrays)]
    status = nnc.cmd_exec(cmd, hint, flags, ins, outs, stream)
    if stream is not None:
        stream.wait()
    results = [None if t is None else t.download() for t in outs]
    for t in cache.values():
        t.free()
    return status, results


def counted(nnc, run, *args, **kwargs):
    """run(nnc, *args, **kwargs) -> (status, outputs, kernels the backend launched meanwhile, ccv_nnc_sm100_launch_count())."""
    l0 = nnc.launch_count()
    status, outs = run(nnc, *args, **kwargs)
    return status, outs, nnc.launch_count() - l0


def ref_exec(ref, cmd, hint, flags, in_arrays, out_arrays, fmt=NHWC, in_fmts=None, out_fmts=None):
    """Same command on the reference's CPU_REF. out_arrays are modified in place and returned."""
    cache = {}

    def tensor_for(a, f):
        if a is None:
            return None
        if id(a) not in cache:
            cache[id(a)] = ref.RefTensor(a, f)
        return cache[id(a)]

    ins = [tensor_for(a, in_fmts[i] if in_fmts else fmt) for i, a in enumerate(in_arrays)]
    outs = [tensor_for(a, out_fmts[i] if out_fmts else fmt) for i, a in enumerate(out_arrays)]
    status = ref.cmd_exec(cmd, hint, flags, ins, outs)
    for t in cache.values():
        t.free()
    return status, out_arrays


def rel_err(got, want):
    """max |got - want| / max(|want|): the normalised error the fp32 tolerance of BASELINE.json (<= 1e-3) is applied to."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    denom = max(np.abs(want).max(), 1e-30)
    return float(np.abs(got - want).max() / denom)


def elem_rel_err(got, want, floor=1e-2):
    """Element-wise relative error max |got - want| / max(|want|, floor * max|want|): small outputs count with their own
    magnitude down to an absolute floor of `floor` x the largest reference value (below that, fp32 summation-order noise of
    the reference itself dominates)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    scale = max(np.abs(want).max(), 1e-30)
    return float((np.abs(got - want) / np.maximum(np.abs(want), floor * scale)).max())


def assert_close(got, want, tol, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.isfinite(got).all(), what + ": non-finite output"
    e = rel_err(got, want)
    assert e <= tol, "%s: normalised max error %.3e > %.1e" % (what, e, tol)


# ---- 16-bit tensors: bf16 travels as uint16 (numpy has no bfloat16), fp16 as numpy float16 ------------------------------
def to_bf16(a):
    """fp32 -> bf16 bits (uint16), round to nearest even."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return r.reshape(np.shape(a))


def from_bf16(u):
    return (np.ascontiguousarray(u, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).reshape(np.shape(u))


def round16(a, kind):
    """The fp32 values a 16-bit tensor of this kind (abi.CCV_16BF / abi.CCV_16F) actually holds."""
    return from_bf16(to_bf16(a)) if kind == abi.CCV_16BF else np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def pack16(a, kind):
    return to_bf16(a) if kind == abi.CCV_16BF else np.asarray(a, np.float32).astype(np.float16)


def unpack16(u, kind):
    return from_bf16(u) if kind == abi.CCV_16BF else np.asarray(u, np.float16).astype(np.float32)


def gpu_exec16(nnc, cmd, hint, flags, in_arrays, out_arrays, kind, keep32=(), stream=None, in_fmts=None, out_fmts=None):
    """gpu_exec with fp32 numpy arrays travelling as 16-bit tensors of `kind`.  `keep32`: ids (id(array)) of operands that stay
    fp32 (batch-norm parameters / statistics, fp32 master weights of SGD).  Integer arrays travel unchanged.  The same array
    object in both lists is the same GPU tensor.  Returns (status, [fp32 output arrays])."""
    cache = {}

    def tensor_for(a, f=NHWC):
        if a is None:
            return None
        if id(a) not in cache:
            if a.dtype != np.float32 or id(a) in keep32:
                t = nnc.gpu_tensor(list(a.shape), f, NP_TO_CCV[a.dtype])
                t.upload(a)
            else:
                t = nnc.gpu_tensor(list(a.shape), f, kind)
                t.upload(pack16(a, kind))
            cache[id(a)] = t
        return cache[id(a)]

    ins = [tensor_for(a, in_fmts[i] if in_fmts else NHWC) for i, a in enumerate(in_arrays)]
    outs = [tensor_for(a, out_fmts[i] if out_fmts else NHWC) for i, a in enumerate(out_arrays)]
    status = nnc.cmd_exec(cmd, hint, flags, ins, outs, stream)
    if stream is not None:
        stream.wait()
    results = []
    for t in outs:
        if t is None:
            results.append(None)
        elif (t.params.datatype & 0xFF000) in (abi.CCV_16BF, abi.CCV_16F):
            results.append(unpack16(t.download(), t.params.datatype & 0xFF000))
        else:
            results.append(t.download())
    for t in cache.values():
        t.free()
    return status, results
