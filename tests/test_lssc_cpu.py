"""COMPRESSION_LSSC without a device: the restatement of tests/lssc_ref.py against CPU_REF's fixture (tests/golden/cpuref_lssc.npz) and
against plausible kernel defects, the compressed-shape helper, the command ids and the registration list."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi, nnc
from tests import lssc_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_lssc.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_lssc.npz missing")
    return np.load(GOLDEN)


def _cases(z, prefix):
    return sorted(k[len(prefix) + 1:-2] for k in z.files if k.startswith(prefix + "_") and k.endswith("_x" if prefix == "f" else "_y"))


def _disagreements(z, defect=None):
    bad = []
    for name in _cases(z, "f"):
        if not np.array_equal(R.forward(z["f_%s_x" % name], R.NCHW, defect), z["f_%s_y" % name]):
            bad.append("forward " + name)
    for name in _cases(z, "b"):
        want = z["b_%s_x" % name]
        if not np.array_equal(R.backward(z["b_%s_y" % name], want.shape, R.NCHW, defect), want):
            bad.append("backward " + name)
    return bad


def test_restatement_matches_cpu_ref_fixture_bit_for_bit():
    z = _golden()
    assert len(_cases(z, "f")) == 2 * 49 + 3 and len(_cases(z, "b")) == 2 * 49 + 5
    assert _disagreements(z) == []


def test_fixture_reaches_every_special_block():
    """NaN in cell 0 and elsewhere, +-Inf (whose code products are NaN), +-0 ties, subnormal ranges below 1e-6, and middle levels whose
    truncation and round-to-nearest differ"""
    z = _golden()
    h = z["f_special_x"].reshape(-1, 16)
    a = h.view(np.float16).astype(np.float32)
    assert np.isnan(a[:, 0]).any() and (np.isnan(a[:, 1:]).any(1) & ~np.isnan(a[:, 0])).any()
    assert np.isinf(a).any(1).sum() >= 3 and (np.abs(a) == 65504).any()
    q = z["f_special_y"].reshape(-1, 4)
    assert ((q[:, 0] == 0) & (q[:, 1] == 0)).any() and ((q[:, 0] == 0x8000) & (q[:, 1] == 0x8000)).any()  # the earlier zero stays
    finite = ~np.isnan(a).any(1) & ~np.isinf(a).any(1)
    rng = a.max(1) - a.min(1)
    assert ((rng > 0) & (rng < 1e-6) & finite).any()
    assert np.isnan(q[:, :2].view(np.float16)).any()  # NaN min / max kept as the cell's bits
    lv = z["b_levels_y"].reshape(-1, 4)
    lo, hi = lv[:, 0].view(np.float16).astype(np.float32), lv[:, 1].view(np.float16).astype(np.float32)
    v1 = hi / np.float32(3) + (lo * np.float32(2)) / np.float32(3)
    assert (R.f32_to_f16_trunc(v1) != v1.astype(np.float16).view(np.uint16)).sum() > 100


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_fixture_rejects_plausible_kernel_defects(defect):
    """fmaxf / fminf scans, zero padding, ascale kept in double, round-to-nearest middle levels, codes packed high to low"""
    assert _disagreements(_golden(), defect), defect


def test_float_ascale_is_the_same_as_the_double_one():
    """A float 1e-6 and a float quotient 3.f / max(range, 1e-6f) give ascale the same bits as CPU_REF's double ones for every float
    range: float(1e-6) = 9.99999997e-7, and no fp16 difference lies between it and 1e-6 (2^-20 < 1e-6 < 17 * 2^-24); 3 / 9.99999997e-7
    rounds to 3e6 in float as 3 / 1e-6 does; and a double quotient rounded to float is the correctly rounded float quotient (53 >= 2 *
    24 + 2).  So that defect cannot be seen in any output and is not in R.DEFECTS; this checks the claim on every fp16 range up to 2^10
    and a sample above."""
    h = np.arange(0, 0x7c00, dtype=np.uint16).view(np.float16).astype(np.float32)
    r = np.random.RandomState(3)
    rng = np.concatenate([h, (h[r.randint(0, h.size, 1 << 20)] - h[r.randint(0, h.size, 1 << 20)]).astype(np.float32)])
    rng = np.abs(rng)
    f = np.float32(3) / np.maximum(rng, np.float32(1e-6))
    d = (3.0 / np.where(rng.astype(np.float64) > 1e-6, rng.astype(np.float64), 1e-6)).astype(np.float32)
    assert np.array_equal(f, d)


@pytest.mark.parametrize("shape", [(2, 3, 7, 13), (3, 5, 14), (1, 2, 113, 114)])
def test_nhwc_restatement_is_the_nchw_transpose(shape):
    """compressed[n, by, 4 bx + k, c] is half k of plane (n, c)'s block (by, bx)"""
    x = R.f16_bits(np.random.RandomState(5).randn(*shape))
    perm = (0, 2, 3, 1) if len(shape) == 4 else (1, 2, 0)
    inv = np.argsort(perm)
    y = R.forward(x, R.NCHW)
    y_nhwc = R.forward(np.ascontiguousarray(x.transpose(perm)), R.NHWC)
    assert np.array_equal(y_nhwc.transpose(inv), y)
    assert y_nhwc.shape == R.compressed_shape(x.transpose(perm).shape, R.NHWC)
    back = R.backward(y_nhwc, x.transpose(perm).shape, R.NHWC)
    assert np.array_equal(back.transpose(inv), R.backward(y, x.shape, R.NCHW))


def test_compressed_dims_helper():
    N, C_ = abi.CCV_TENSOR_FORMAT_NCHW, abi.CCV_TENSOR_FORMAT_NHWC
    assert nnc.lssc_compressed_dims([128, 64, 113, 114], N) == [128, 64, 29, 116]
    assert nnc.lssc_compressed_dims([64, 7, 5], N) == [64, 2, 8]
    assert nnc.lssc_compressed_dims([256, 56, 56, 64], C_) == [256, 14, 56, 64]
    assert nnc.lssc_compressed_dims([13, 1, 3], C_) == [4, 4, 3]
    for fmt, f in ((N, R.NCHW), (C_, R.NHWC)):
        for s in ((2, 3, 5, 7), (3, 14, 1)):
            assert tuple(nnc.lssc_compressed_dims(s, fmt)) == R.compressed_shape(s, f)
    with pytest.raises(ValueError):
        nnc.lssc_compressed_dims([4, 4], N)
    with pytest.raises(ValueError):
        nnc.lssc_compressed_dims([1, 4, 4, 4], abi.CCV_TENSOR_FORMAT_CHWN)


# ---- ABI and registration ----------------------------------------------------------------------------------------------------------
def test_command_ids():
    assert abi.CCV_NNC_COMPRESSION_LSSC_FORWARD == 0x17ea8f72 and abi.CCV_NNC_COMPRESSION_LSSC_BACKWARD == 0x17ea8f73
    assert nnc.CMD_COMPRESSION_LSSC_FORWARD().cmd == 0x17ea8f72 and nnc.CMD_COMPRESSION_LSSC_BACKWARD().cmd == 0x17ea8f73


def test_fourth_registration_list_makes_128_commands():
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    x = lambda a, b: re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index(a):header.index(b)])
    lists = [x("#define CCV_NNC_SM100_COMMANDS(X)", "#define CCV_SM100_DECLARE_REGISTER")]
    for family in ("DETECTION", "OPTIMIZER", "COMPRESSION"):
        lists.append(x("#define CCV_NNC_SM100_%s_COMMANDS(X)" % family, "CCV_NNC_SM100_%s_COMMANDS(CCV_SM100_DECLARE_REGISTER)" % family))
    assert [len(l) for l in lists] == [118, 4, 4, 2]
    assert len(set(sum(lists, []))) == 128
    assert lists[3] == ["CCV_NNC_COMPRESSION_LSSC_FORWARD", "CCV_NNC_COMPRESSION_LSSC_BACKWARD"]
    host = open(os.path.join(ROOT, "ccv_b200", "csrc", "nnc_host.cu")).read()
    assert "CCV_NNC_SM100_COMPRESSION_COMMANDS(CCV_SM100_CALL_REGISTER)" in host
    inc = open(os.path.join(ROOT, "integration", "ccv_nnc_cmd_sm100_init.inc")).read()
    for c in lists[3]:
        assert inc.count("_register_command_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % c) == 2, c
    mk = open(os.path.join(ROOT, "integration", "Makefile")).read()
    assert re.search(r"INT_TESTS :=[^\n]*(\\\n[^\n]*)*\blamb rmsprop compression\b", mk)


class _Registry(C.Structure):
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


def test_both_commands_register_fp16_nchw_nhwc_on_gpu_memory():
    lib = nnc.lib()
    nnc.init()
    for d in ("FORWARD", "BACKWARD"):
        r = _Registry()
        getattr(lib, "_register_command_CCV_NNC_COMPRESSION_LSSC_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % d)(C.byref(r))
        assert r.exec and r.algorithms == 1 and r.tensor_memory == abi.CCV_TENSOR_GPU_MEMORY, d
        assert r.tensor_datatypes == abi.CCV_16F and r.tensor_formats == abi.CCV_TENSOR_FORMAT_NCHW | abi.CCV_TENSOR_FORMAT_NHWC
        assert lib.ccv_nnc_cmd_ok(getattr(abi, "CCV_NNC_COMPRESSION_LSSC_" + d), abi.CCV_NNC_BACKEND_GPU_SM100) == 1
