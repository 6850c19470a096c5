"""HISTOGRAM and EWPROD without a device: the restatement of tests/histogram_ref.py against CPU_REF's fixture
(tests/golden/cpuref_histogram.npz) and against plausible kernel defects, the command helpers, and the fifth registration list."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi, nnc
from tests import histogram_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_histogram.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_histogram.npz missing")
    return np.load(GOLDEN)


def _hist_cases(z):
    return sorted(k[2:-2] for k in z.files if k.startswith("h_") and k.endswith("_x"))


def host_logf_moves(x, p):
    """elements of a LOG case whose bin differs between the host's logf and the correctly rounded one"""
    if int(p[0]) != R.LOG:
        return np.zeros(len(x), bool)
    a = R.bin_index(x, R.LOG, 0, p[2], p[3], p[4], logf=R.cr_logf)
    b = R.bin_index(x, R.LOG, 0, p[2], p[3], p[4], logf=R.host_logf)
    return a != b


def _restate(z, name, defect=None, logf=R.cr_logf):
    x, p, b = z["h_%s_x" % name], z["h_%s_p" % name], z["h_%s_b" % name]
    bounds = z["h_%s_bounds" % name] if int(p[0]) == R.BINS else None
    return R.histogram(x, int(p[0]), int(p[1]), p[2], p[3], p[4], bounds, nb=len(b), logf=logf, defect=defect)


def _disagreements(z, defect=None):
    bad = []
    for name in _hist_cases(z):
        b, s = _restate(z, name, defect, logf=R.host_logf)
        if not np.array_equal(b, z["h_%s_b" % name]):
            bad.append("counts " + name)
        if not np.array_equal(s.view(np.uint32), z["h_%s_s" % name].view(np.uint32)):
            bad.append("stats " + name)
    for name in sorted(k[:-2] for k in z.files if k.startswith("e_f") and k.endswith("_c")):
        ops = list(z[name + "_in"])
        tail = name.rsplit("_", 1)[1]
        got = R.ewprod(ops, None if tail == "none" else int(tail), defect)
        if not np.array_equal(got.view(np.uint32), z[name + "_c"].view(np.uint32)):
            bad.append(name)
    return bad


def test_restatement_matches_cpu_ref_fixture_bit_for_bit():
    """with the host's logf the restatement is CPU_REF exactly; with the correctly rounded logf (the backend's definition) only the LOG
    elements the host's logf moves may land elsewhere, each in an adjacent bin"""
    z = _golden()
    assert _disagreements(z) == []
    for name in _hist_cases(z):
        p = z["h_%s_p" % name]
        b, s = _restate(z, name)
        moved = host_logf_moves(z["h_%s_x" % name], p)
        assert np.abs(b.astype(np.int64) - z["h_%s_b" % name]).sum() <= 2 * moved.sum(), name
        assert np.array_equal(s.view(np.uint32), z["h_%s_s" % name].view(np.uint32)), name
    for g in (0, 1):
        k = "e_b%d" % g
        h = R.ewprod_back(z[k + "_g"] if g else None, list(z[k + "_a"]), z[k + "_b"])
        assert np.array_equal(np.stack(h).view(np.uint32), z[k + "_h"].view(np.uint32)), k


def test_fixture_reaches_the_edge_cases():
    z = _golden()
    s = {n: z["h_%s_s" % n] for n in _hist_cases(z)}
    assert np.isnan(s["nan_last"][0]) and np.isnan(s["nan_only"][1]) and not np.isnan(s["nan_first"][0])
    # +-0 ties after a NaN ([5, NaN, -0, 0, 0, -0]): the later element's sign, -0, for both scans
    assert s["zero_ties_after_nan"][0] == 0 and np.signbit(s["zero_ties_after_nan"][:2]).all()
    assert np.isinf(s["big_squares"][3])
    for n in ("even_edges", "log_edges", "bins_at_bounds", "even_extreme"):
        assert z["h_%s_b" % n].sum() == len(z["h_%s_x" % n]), n
    assert z["h_log_long_b_b"][-5:].tolist() == [0] * 5
    assert any(k.startswith("h_view6_") for k in z.files)


@pytest.mark.parametrize("defect", ["fminf", "pairwise", "le_search", "fused_even", "plain_order"])
def test_fixture_rejects_plausible_kernel_defects(defect):
    z = _golden()
    assert _disagreements(z, defect), defect


def test_sum_bound_covers_the_fixture():
    """the double sums the fixture stores are within count 2^-53 sum|x| of the exact sums (so a kernel's fixed-order sum is too)"""
    z = _golden()
    from fractions import Fraction
    for name in _hist_cases(z):
        x = z["h_%s_x" % name]
        if not np.isfinite(x).all():
            continue
        exact = sum(Fraction(float(v)) for v in x)
        bs, _ = R.sums(x)
        eb, _ = R.sum_bound(x)
        assert abs(float(Fraction(float(bs)) - exact)) <= eb + abs(float(bs)) * 2.0 ** -24, name


def test_command_helpers():
    assert abi.CCV_NNC_HISTOGRAM_FORWARD == 0xc5473e44 and abi.CCV_NNC_EWPROD_FORWARD == 0xee07e8fe
    c = nnc.CMD_HISTOGRAM_EVEN(10, -1.0, 2.0)
    assert (c.cmd, c.info.histogram.type, c.info.histogram.bins, c.info.histogram.min, c.info.histogram.max) == (0xc5473e44, 0, 10, -1.0, 2.0)
    assert nnc.histogram_bin_count(c) == 13
    d = nnc.CMD_HISTOGRAM_LOG()
    assert d.info.histogram.type == abi.CCV_NNC_HISTOGRAM_LOGARITHMIC and np.float32(d.info.histogram.rate) == np.float32(1.1)
    assert nnc.histogram_bin_count(d) == R.bin_count(R.LOG, 0, 1e-12, 1e20, 1.1)
    assert nnc.histogram_bin_count(nnc.CMD_HISTOGRAM_BINS(), 9) == 11
    assert nnc.CMD_EWPROD_BACKWARD().cmd == 0xee07e8ff
    # the histogram arm sits at the start of the union, as in the reference's ccv_nnc_cmd_param_t
    assert abi.CmdParam.u.offset + abi._CmdUnion.histogram.offset == abi.CmdParam.size.size and C.sizeof(abi._Histogram) == 20


def test_fifth_registration_list_makes_132_commands():
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    x = lambda a, b: re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index(a):header.index(b)])
    lists = [x("#define CCV_NNC_SM100_COMMANDS(X)", "#define CCV_SM100_DECLARE_REGISTER")]
    for family in ("DETECTION", "OPTIMIZER", "COMPRESSION", "STATISTICS"):
        lists.append(x("#define CCV_NNC_SM100_%s_COMMANDS(X)" % family, "CCV_NNC_SM100_%s_COMMANDS(CCV_SM100_DECLARE_REGISTER)" % family))
    assert [len(l) for l in lists] == [118, 4, 4, 2, 4]
    assert len(set(sum(lists, []))) == 132
    host = open(os.path.join(ROOT, "ccv_b200", "csrc", "nnc_host.cu")).read()
    assert "CCV_NNC_SM100_STATISTICS_COMMANDS(CCV_SM100_CALL_REGISTER)" in host
    inc = open(os.path.join(ROOT, "integration", "ccv_nnc_cmd_sm100_init.inc")).read()
    for c in lists[4]:
        assert inc.count("_register_command_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % c) == 2, c


class _Registry(C.Structure):
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


def test_four_commands_register_on_gpu_memory():
    lib = nnc.lib()
    nnc.init()
    for name, types in (("HISTOGRAM", abi.CCV_32F | abi.CCV_16F | abi.CCV_16BF | abi.CCV_32S), ("EWPROD", abi.CCV_32F | abi.CCV_16F | abi.CCV_16BF)):
        for d in ("FORWARD", "BACKWARD"):
            r = _Registry()
            getattr(lib, "_register_command_CCV_NNC_%s_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % (name, d))(C.byref(r))
            assert r.exec and r.algorithms == 1 and r.tensor_memory == abi.CCV_TENSOR_GPU_MEMORY and r.tensor_datatypes == types, (name, d)
            assert lib.ccv_nnc_cmd_ok(getattr(abi, "CCV_NNC_%s_%s" % (name, d)), abi.CCV_NNC_BACKEND_GPU_SM100) == 1
