"""LAMB and RMSPROP without a device: the oracles of tests/optim_ref.py against CPU_REF's fixture (tests/golden/cpuref_optim.npz) and
against plausible kernel defects, the union arms and registration lists, and how ccv_nnc_sm100_graph_fuse groups runs of these
commands (host logic only: nothing is executed, tensors are host tensors)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi, nnc
from tests import optim_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_optim.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTIMIZERS = ("LAMB", "RMSPROP")


def same(x, y):
    x, y = np.ascontiguousarray(x, np.float32).ravel(), np.ascontiguousarray(y, np.float32).ravel()
    return x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_optim.npz missing")
    return np.load(GOLDEN)


def _lamb_case(z, case, defect=None):
    name, count, step, rate, beta1, beta2, decay, eps, scale, in_place, a_zero, nan_at = case
    ins = [z["lamb_%s_%s" % (k, name)] for k in "gamv"]
    return R.lamb(*ins, step, rate, beta1, beta2, decay, eps, scale, defect=defect), [z["lamb_%s_%s" % (k, name)] for k in "bnu"]


def _run(z):
    from tests.golden.make_optim_golden import RUN_COUNTS
    return [tuple(z["run_%s_%d" % (k, i)] for k in "gamv") for i in range(len(RUN_COUNTS))], \
        [tuple(z["run_%s_%d" % (k, i)] for k in "bnu") for i in range(len(RUN_COUNTS))]


# ---- the oracles against CPU_REF --------------------------------------------------------------------------------------------------
def test_lamb_oracle_matches_cpu_ref_fixture():
    from tests.golden.make_optim_golden import LAMB_CASES, RUN_HP
    z = _golden()
    for case in LAMB_CASES:
        (b, n, u, t64), want = _lamb_case(z, case)
        assert same(b, want[0]) and same(n, want[1]) and same(u, want[2]), case[0]
    # an all-zero a and a NaN gradient give trust 1; the NaN stays in its element only
    (_, _, _, t_zero), _ = _lamb_case(z, LAMB_CASES[2])
    (b_nan, _, _, t_nan), _ = _lamb_case(z, LAMB_CASES[3])
    assert t_zero is None and t_nan is None
    assert np.isnan(b_nan).sum() == 1 and np.isnan(b_nan[LAMB_CASES[3][-1]])
    ins, want = _run(z)
    for got, w in zip(R.lamb_multi(ins, **RUN_HP), want):
        assert all(same(x, y) for x, y in zip(got, w))


def test_rmsprop_oracle_matches_cpu_ref_fixture():
    from tests.golden.make_optim_golden import RMSPROP_CASES
    z = _golden()
    for name, count, rate, decay, alpha, momentum, eps, scale, in_place, nan_at in RMSPROP_CASES:
        got = R.rmsprop(*[z["rmsprop_%s_%s" % (k, name)] for k in "gamv"], rate, decay, alpha, momentum, eps, scale)
        for x, k in zip(got, "bnu"):
            assert same(x, z["rmsprop_%s_%s" % (k, name)]), (name, k)


@pytest.mark.parametrize("defect", R.LAMB_DEFECTS)
def test_lamb_fixture_rejects_plausible_kernel_defects(defect):
    """an FMA-contracted update, fp32 norm sums, the norm of the new weights, ADAM's L2 decay, (1 - beta2) (grad grad) and one trust
    ratio shared by a fused run each give other bits than CPU_REF somewhere in the fixture"""
    from tests.golden.make_optim_golden import LAMB_CASES, RUN_HP
    z = _golden()
    differs = False
    for case in LAMB_CASES:
        (b, n, u, _), want = _lamb_case(z, case, defect)
        differs |= not (same(b, want[0]) and same(n, want[1]) and same(u, want[2]))
    ins, want = _run(z)
    for got, w in zip(R.lamb_multi(ins, **RUN_HP, defect=defect), want):
        differs |= not all(same(x, y) for x, y in zip(got, w))
    assert differs, defect


def test_midpoint_margin_holds_for_the_fixture():
    """the float64 trust ratios of the fixture sit far from a float32 rounding midpoint, so any order of the float64 sums rounds alike"""
    from tests.golden.make_optim_golden import LAMB_CASES
    z = _golden()
    for case in LAMB_CASES[:2]:
        (_, _, _, t64), _ = _lamb_case(z, case)
        assert R.midpoint_margin(t64) > 2.0 ** -40, case[0]


def test_launch_plan():
    assert R.optim_multi_plan([4] * 70) == [list(range(32)), list(range(32, 64)), list(range(64, 70))]
    assert R.optim_multi_plan([4, 1, 5, 3]) == [[0, 1, 2, 3]]
    from tests.test_parity_feeder_paths import _resnet50_param_counts
    groups = [[c for c in _resnet50_param_counts() if (c > 4096) == w] for w in (True, False)]
    assert [len(g) for g in groups] == [53, 108] and [len(R.optim_multi_plan(g)) for g in groups] == [2, 4]


# ---- ABI and registration ----------------------------------------------------------------------------------------------------------
def test_arms_sit_at_the_reference_offsets():
    """lib/nnc/ccv_nnc.h:189-205: lamb = (step, rate, scale, beta1, beta2, decay, epsilon), rmsprop = (rate, scale, decay, alpha, momentum,
    epsilon), both from byte 48; the block stays 120 bytes"""
    base = abi.CmdParam.u.offset
    for i, f in enumerate(("step", "rate", "scale", "beta1", "beta2", "decay", "epsilon")):
        assert base + abi._CmdUnion.lamb.offset + getattr(abi._Lamb, f).offset == 48 + 4 * i, f
    for i, f in enumerate(("rate", "scale", "decay", "alpha", "momentum", "epsilon")):
        assert base + abi._CmdUnion.rmsprop.offset + getattr(abi._Rmsprop, f).offset == 48 + 4 * i, f
    assert C.sizeof(abi.CmdParam) == 120
    c = nnc.CMD_LAMB_FORWARD(7, 0.5, 0.25, 0.125, 0.0625, 1e-3)
    assert c.cmd == abi.CCV_NNC_LAMB_FORWARD == 0x450edb1a and c.info.lamb.step == 7 and c.info.lamb.scale == 1.0
    assert (c.info.lamb.rate, c.info.lamb.beta1, c.info.lamb.beta2, c.info.lamb.decay) == (0.5, 0.25, 0.125, 0.0625)
    r = nnc.CMD_RMSPROP_FORWARD(0.5, 0.25, 0.125, 0.0625, 1e-3, scale=2.0)
    assert r.cmd == abi.CCV_NNC_RMSPROP_FORWARD == 0x9c886b1c
    assert (r.info.rmsprop.rate, r.info.rmsprop.decay, r.info.rmsprop.alpha, r.info.rmsprop.momentum, r.info.rmsprop.scale) == (0.5, 0.25, 0.125, 0.0625, 2.0)
    assert nnc.CMD_LAMB_BACKWARD(1, 0.1, 0.9, 0.99, 0, 1e-6).cmd == 0x450edb1b and nnc.CMD_RMSPROP_BACKWARD(0.1, 0, 0.9, 0, 1e-6).cmd == 0x9c886b1d


def test_three_registration_lists_hold_126_distinct_commands():
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    x = lambda a, b: re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index(a):header.index(b)])
    first = x("#define CCV_NNC_SM100_COMMANDS(X)", "#define CCV_SM100_DECLARE_REGISTER")
    second = x("#define CCV_NNC_SM100_DETECTION_COMMANDS(X)", "CCV_NNC_SM100_DETECTION_COMMANDS(CCV_SM100_DECLARE_REGISTER)")
    third = x("#define CCV_NNC_SM100_OPTIMIZER_COMMANDS(X)", "CCV_NNC_SM100_OPTIMIZER_COMMANDS(CCV_SM100_DECLARE_REGISTER)")
    assert (len(first), len(second), len(third)) == (118, 4, 4)
    assert len(set(first + second + third)) == 126
    assert sorted(third) == sorted("CCV_NNC_%s_%s" % (n, d) for n in OPTIMIZERS for d in ("FORWARD", "BACKWARD"))
    inc = open(os.path.join(ROOT, "integration", "ccv_nnc_cmd_sm100_init.inc")).read()
    for c in third:
        assert inc.count("_register_command_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % c) == 2, c
    mk = open(os.path.join(ROOT, "integration", "Makefile")).read()
    assert re.search(r"INT_TESTS :=[^\n]*(\\\n[^\n]*)*\blamb rmsprop\b", mk)


class _Registry(C.Structure):
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


def test_every_new_symbol_is_exported_and_fills_its_record():
    lib = nnc.lib()
    for name in OPTIMIZERS:
        for d in ("FORWARD", "BACKWARD"):
            r = _Registry()
            getattr(lib, "_register_command_CCV_NNC_%s_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % (name, d))(C.byref(r))
            assert r.exec and r.tensor_memory == abi.CCV_TENSOR_GPU_MEMORY and r.algorithms == 1, (name, d)
            assert r.tensor_datatypes == abi.CCV_32F | abi.CCV_16F | abi.CCV_16BF
            assert lib.ccv_nnc_cmd_ok(getattr(abi, "CCV_NNC_%s_%s" % (name, d)), abi.CCV_NNC_BACKEND_GPU_SM100) == 1


# ---- graph fusion (host logic) -----------------------------------------------------------------------------------------------------
def _t(n, dt=abi.CCV_32F):
    return nnc.cpu_tensor([n], abi.CCV_TENSOR_FORMAT_NHWC, dt)


def _quad(n=64, state=abi.CCV_32F, grad=abi.CCV_32F):
    return _t(n, grad), _t(n, state), _t(n, state), _t(n, state)


def _kinds(g):
    return [k for _, k, _, _ in g.nodes()]


def test_fuse_groups_interleaved_lamb_nodes_by_parameters():
    nnc.init()
    params = [_quad() for _ in range(6)]
    g = nnc.Graph()
    for i, (gr, a, m, v) in enumerate(params):
        g.exec_new(nnc.CMD_LAMB_FORWARD(3, 0.01, 0.9, 0.999, 0.01 if i % 2 == 0 else 0.0, 1e-6), None, 0, [gr, a, m, v], [a, m, v])
    assert g.fuse() == 4
    nodes = g.nodes()
    assert _kinds(g) == [9, 9]
    for (cmd, _, ins, outs), group in zip(nodes, (params[0::2], params[1::2])):
        assert cmd == abi.CCV_NNC_LAMB_FORWARD
        assert ins == [t.ptr for q in group for t in q]
        assert outs == [t.ptr for q in group for t in q[1:]]
    g.free()


def test_fuse_breaks_a_lamb_run_at_a_dependent_node():
    """the third node reads the first one's b: the run ends before it, and it starts the next one"""
    nnc.init()
    (g1, a1, m1, v1), (g2, a2, m2, v2), (g3, _, m3, v3), (g4, a4, m4, v4) = (_quad() for _ in range(4))
    b1 = _t(64)
    cmd = nnc.CMD_LAMB_FORWARD(1, 0.01, 0.9, 0.999, 0.0, 1e-6)
    g = nnc.Graph()
    g.exec_new(cmd, None, 0, [g1, a1, m1, v1], [b1, m1, v1])
    g.exec_new(cmd, None, 0, [g2, a2, m2, v2], [a2, m2, v2])
    g.exec_new(cmd, None, 0, [g3, b1, m3, v3], [b1, m3, v3])
    g.exec_new(cmd, None, 0, [g4, a4, m4, v4], [a4, m4, v4])
    assert g.fuse() == 2
    assert _kinds(g) == [9, 9]
    assert [len(ins) for _, _, ins, _ in g.nodes()] == [8, 8]
    g.free()


def test_fuse_keeps_state_types_and_gradient_types_apart():
    nnc.init()
    cmd = nnc.CMD_LAMB_FORWARD(1, 0.01, 0.9, 0.999, 0.0, 1e-6)
    quads = [_quad(), _quad(state=abi.CCV_16BF), _quad(), _quad(state=abi.CCV_16BF), _quad(grad=abi.CCV_16F)]
    g = nnc.Graph()
    for gr, a, m, v in quads:
        g.exec_new(cmd, None, 0, [gr, a, m, v], [a, m, v])
    assert g.fuse() == 2
    assert _kinds(g) == [9, 9, 0]
    assert [len(ins) // 4 for _, _, ins, _ in g.nodes()] == [2, 2, 1]
    assert g.nodes()[1][2][1] == quads[1][1].ptr
    g.free()


def test_fuse_rmsprop_runs_and_leaves_sgd_runs_as_they_were():
    """an SGD run next to an RMSPROP run and a LAMB run: each fuses on its own, the SGD one exactly as before (kind 5)"""
    nnc.init()
    g = nnc.Graph()
    sgd = [(_t(64), _t(64), _t(64)) for _ in range(3)]
    for gr, a, m in sgd:
        g.exec_new(nnc.CMD_SGD_FORWARD(1, 0.1, 1.0 / 256, 1e-4, 0.9, 0.0), None, 0, [gr, a, m], [a, m])
    rms = [_quad() for _ in range(3)]
    for gr, a, m, v in rms:
        g.exec_new(nnc.CMD_RMSPROP_FORWARD(0.01, 0.0, 0.9, 0.9, 1e-8), None, 0, [gr, a, m, v], [a, m, v])
    lamb = [_quad() for _ in range(2)]
    for gr, a, m, v in lamb:
        g.exec_new(nnc.CMD_LAMB_FORWARD(1, 0.01, 0.9, 0.999, 0.0, 1e-6), None, 0, [gr, a, m, v], [a, m, v])
    assert g.fuse() == 2 + 2 + 1
    nodes = g.nodes()
    assert _kinds(g) == [5, 10, 9]
    assert [c for c, _, _, _ in nodes] == [abi.CCV_NNC_SGD_FORWARD, abi.CCV_NNC_RMSPROP_FORWARD, abi.CCV_NNC_LAMB_FORWARD]
    assert nodes[0][2] == [t.ptr for q in sgd for t in q] and nodes[1][2] == [t.ptr for q in rms for t in q]
    g.free()
