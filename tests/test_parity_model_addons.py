"""PAD, MIN / MAX, ARGMAX / ARGMIN and REDUCE_ISNAN (forward / backward) on CCV_NNC_BACKEND_GPU_SM100 against the oracles of
tests/addons_ref.py, which are pinned to the reference's CPU_REF by tests/golden/cpuref_addons.npz.

None of these commands does arithmetic, so every result is compared exactly, on raw bits: fp32 equals CPU_REF bit for bit and 16-bit
equals CPU_REF on the widened values, NaN payloads and signed zeros of PAD and MIN / MAX included."""
import os
import re

import numpy as np
import pytest

from ccv_b200 import abi
from tests import addons_ref as R
from tests.util import NHWC, seeded, to_bf16

KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cpuref_addons.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(x, kname):
    """raw element bits of fp32 values x stored as `kname` (16-bit: round to nearest even)"""
    x = np.asarray(x, np.float32)
    if kname == "fp32":
        return x.copy()
    if kname == "bf16":
        return to_bf16(x)
    return x.astype(np.float16).view(np.uint16)


def same(x, y):
    """bitwise equality"""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    if x.dtype == np.float32:
        x, y = x.view(np.uint32), np.ascontiguousarray(y, np.float32).view(np.uint32)
    return x.shape == y.shape and np.array_equal(x, y)


def plant(x, kname, seed):
    """x's bits with NaNs that carry payloads (and a sign), +0 and -0 planted at seeded positions"""
    x = x.copy()
    flat = x.reshape(-1)
    r = np.random.RandomState(seed)
    n = max(1, flat.size // 50)
    pos = r.choice(flat.size, min(flat.size, 4 * n), replace=False)
    if kname == "fp32":
        u = flat.view(np.uint32)
        u[pos[:n]] = 0x7fa00001       # a signalling NaN with a payload
        u[pos[n:2 * n]] = 0xffc00123  # a negative quiet NaN
        u[pos[2 * n:3 * n]] = 0x80000000
        u[pos[3 * n:]] = 0
    else:
        nan1, nan2 = (0x7f81, 0xffc3) if kname == "bf16" else (0x7d01, 0xfe03)
        flat[pos[:n]], flat[pos[n:2 * n]], flat[pos[2 * n:3 * n]], flat[pos[3 * n:]] = nan1, nan2, 0x8000, 0
    return x


def widen(x, kname):
    return R.widen(x, kname)


# ---- CPU: the oracles against CPU_REF's fixture, and against defects ----------------------------------------------------------
def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/cpuref_addons.npz missing")
    return np.load(GOLDEN)


def test_pad_oracle_matches_cpu_ref_fixture():
    from tests.golden.make_addons_golden import PADS
    z = _golden()
    for name, shape, begin, end in PADS:
        for t in (R.ZERO, R.REPLICATE):
            assert same(R.pad_forward(z["pad_a_" + name], begin, end, t), z["pad_b_%s_%d" % (name, t)]), (name, t)
            assert same(R.pad_backward(z["pad_g_" + name], begin, shape), z["pad_h_%s_%d" % (name, t)]), (name, t)


def test_cmp_oracle_matches_cpu_ref_fixture():
    z = _golden()
    a, b, g = z["cmp_a"], z["cmp_b"], z["cmp_g"]
    for op in ("min", "max"):
        assert same(R.cmp_forward(a, b, "fp32", op == "min"), z["cmp_c_" + op])
        for with_g in (1, 0):
            ha, hb = R.cmp_backward(g if with_g else None, a, b, "fp32", op == "min")
            assert same(ha, z["cmp_ha_%s_g%d" % (op, with_g)]) and same(hb, z["cmp_hb_%s_g%d" % (op, with_g)]), (op, with_g)


def test_arg_and_isnan_oracles_match_cpu_ref_fixture():
    from tests.golden.make_addons_golden import ARG_CASES, ISNAN_OUTS
    z = _golden()
    for name, shape, axis in ARG_CASES:
        for op in ("max", "min"):
            want = R.argext(z["arg_" + name], axis, op == "min")
            assert np.array_equal(z["arg_%s_%s_%d_i32" % (op, name, axis)], want), (op, name, axis)
            assert np.array_equal(z["arg_%s_%s_%d_f32" % (op, name, axis)], want.astype(np.float32)), (op, name, axis)
    for bshape in ISNAN_OUTS:
        assert np.array_equal(R.reduce_isnan(z["isnan_a"], bshape), z["isnan_b_" + "x".join(map(str, bshape))]), bshape


def test_oracles_reject_plausible_kernel_defects():
    """fmaxf / fminf instead of the > / < select (NaN and ±0 rows), np.argmax's NaN rule (the first NaN wins), and a replicate
    backward that accumulates the border into the edge all disagree with CPU_REF's fixture"""
    from tests.golden.make_addons_golden import PADS
    z = _golden()
    a, b = z["cmp_a"], z["cmp_b"]
    assert not same(np.fmax(a, b), z["cmp_c_max"]) and not same(np.fmin(a, b), z["cmp_c_min"])
    assert not same(np.fmax(a[3:4], b[3:4]), z["cmp_c_max"][3:4])  # ±0 alone: fmax may return either zero; CPU_REF returns b's
    assert not np.array_equal(np.argmax(z["arg_r2"], axis=1)[:, None], z["arg_max_r2_1_i32"])
    assert not np.array_equal(np.nanargmax(np.where(np.isnan(z["arg_r2"]), -np.inf, z["arg_r2"]), axis=1)[:, None], z["arg_max_r2_1_i32"])
    for name, shape, begin, end in PADS:
        g = z["pad_g_" + name].astype(np.float64)
        acc = np.zeros(shape)
        for idx in np.ndindex(*g.shape):
            src = tuple(min(shape[k] - 1, max(0, idx[k] - begin[k])) for k in range(len(shape)))
            acc[src] += g[idx]
        assert not same(acc.astype(np.float32), z["pad_h_%s_%d" % (name, R.REPLICATE)]), name


def test_pad_arm_sits_at_the_reference_offsets():
    """type at byte 48 of ccv_nnc_cmd_param_t (after size.dim[12]), end[] at 52, and the parameter block stays 120 bytes"""
    import ctypes as C
    assert abi.CmdParam.u.offset + abi._CmdUnion.pad.offset + abi._Pad.type.offset == 48
    assert abi.CmdParam.u.offset + abi._CmdUnion.pad.offset + abi._Pad.end.offset == 52
    assert C.sizeof(abi.CmdParam) == 120
    from ccv_b200 import nnc
    c = nnc.CMD_PAD_FORWARD(abi.CCV_NNC_PAD_REPLICATE, (0, 1, 2, 0), (0, 3, 4, 0))
    assert list(c.info.size.dim[:5]) == [0, 1, 2, 0, 0] and c.info.pad.type == 1 and list(c.info.pad.end[:5]) == [0, 3, 4, 0, 0]


@pytest.mark.ref
def test_constructors_run_cpu_ref_to_the_fixture(ref):
    """the CMD_* constructors of ccv_b200.nnc, run on the compiled reference's CPU_REF, give the fixture's results"""
    from ccv_b200 import nnc
    from tests.golden.make_addons_golden import ARG_CASES, ISNAN_OUTS, PADS
    from tests.util import ref_exec
    z = _golden()

    def run(cmd, ins, outs):
        st, res = ref_exec(ref, cmd, None, 0, ins, outs)
        assert st == 0, hex(cmd.cmd)
        return res
    for name, shape, begin, end in PADS:
        bshape = tuple(shape[k] + begin[k] + end[k] for k in range(len(shape)))
        for t in (R.ZERO, R.REPLICATE):
            assert same(run(nnc.CMD_PAD_FORWARD(t, begin, end), [z["pad_a_" + name]], [np.zeros(bshape, np.float32)])[0], z["pad_b_%s_%d" % (name, t)])
            assert same(run(nnc.CMD_PAD_BACKWARD(t, begin, end), [z["pad_g_" + name]], [np.zeros(shape, np.float32)])[0], z["pad_h_%s_%d" % (name, t)])
    for op, (fwd, bwd) in (("min", (nnc.CMD_MIN_FORWARD, nnc.CMD_MIN_BACKWARD)), ("max", (nnc.CMD_MAX_FORWARD, nnc.CMD_MAX_BACKWARD))):
        assert same(run(fwd(), [z["cmp_a"], z["cmp_b"]], [np.zeros((6, 10), np.float32)])[0], z["cmp_c_" + op])
        ha, hb = run(bwd(), [None, z["cmp_a"], z["cmp_b"]], [np.zeros((6, 10), np.float32), np.zeros((6, 10), np.float32)])
        assert same(ha, z["cmp_ha_%s_g0" % op]) and same(hb, z["cmp_hb_%s_g0" % op])
    for name, shape, axis in ARG_CASES:
        bshape = tuple(1 if k == axis else shape[k] for k in range(len(shape)))
        (got,) = run(nnc.CMD_ARGMAX_FORWARD(axis), [z["arg_" + name]], [np.zeros(bshape, np.int32)])
        assert np.array_equal(got, z["arg_max_%s_%d_i32" % (name, axis)])
    for bshape in ISNAN_OUTS:
        (got,) = run(nnc.CMD_REDUCE_ISNAN_FORWARD(), [z["isnan_a"]], [np.zeros(bshape, np.int32)])
        assert np.array_equal(got, z["isnan_b_" + "x".join(map(str, bshape))])


def test_registry_count_from_the_header():
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    block = header[header.index("#define CCV_NNC_SM100_COMMANDS(X)"):header.index("#define CCV_SM100_DECLARE_REGISTER")]
    cmds = re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", block)
    assert len(cmds) == len(set(cmds)) == 118
    for name in ("PAD", "MIN", "MAX", "ARGMAX", "ARGMIN", "REDUCE_ISNAN"):
        assert "CCV_NNC_%s_FORWARD" % name in cmds and "CCV_NNC_%s_BACKWARD" % name in cmds


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
class _Dev(object):
    """GPU tensors holding raw bits; everything made here is freed by free()"""

    def __init__(self, nnc):
        self.nnc, self.owned = nnc, []

    def up(self, x, kname=None, shape=None):
        """x: float32 (fp32), uint16 bits (kname says which 16-bit type) or int32"""
        kind = abi.CCV_32S if x.dtype == np.int32 else KINDS[kname or "fp32"]
        t = self.nnc.gpu_tensor(list(shape or x.shape), NHWC, kind)
        t.upload(x.view(np.float16) if kind == abi.CCV_16F else x)
        self.owned.append(t)
        return t

    def view(self, base, dims, ofs, stride):
        v = self.nnc.tensor_view_new(base, list(dims), list(ofs) + [0] * (12 - len(ofs)), list(stride) + [0] * (12 - len(stride)))
        self.owned.append(v)
        return v

    @staticmethod
    def down(t):
        x = t.download()
        return x.view(np.uint16) if x.dtype == np.float16 else x

    def run(self, cmd, ins, outs, flags=0):
        l0 = self.nnc.launch_count()
        st = self.nnc.cmd_exec(cmd, None, flags, ins, outs)
        return st, self.nnc.launch_count() - l0

    def free(self):
        for t in reversed(self.owned):
            t.free()
        self.owned = []


@pytest.fixture
def dev(gpu):
    d = _Dev(gpu)
    yield d
    d.free()


def _exec(dev, cmd, ins, outs, kname, launches=None):
    """upload ins (arrays) and outs (arrays: initial contents), run, download outs"""
    ti = [None if x is None else dev.up(x, kname) for x in ins]
    to = [None if x is None else dev.up(x, kname) for x in outs]
    st, n = dev.run(cmd, ti, to)
    assert st == 0, dev.nnc.lib().ccv_nnc_sm100_last_error()
    if launches is not None:
        assert n == launches, (n, launches)
    return [None if t is None else dev.down(t) for t in to]


def _sentinel_like(shape, kname):
    return bits(np.full(shape, 7.0, np.float32), kname)


PAD_CASES = [((13,), (2,), (5,)), ((13,), (0,), (0,)), ((6, 7), (1, 0), (2, 3)), ((5, 6, 7), (0, 2, 1), (3, 0, 2)), ((2, 5, 6, 7), (1, 2, 0, 3), (0, 1, 2, 1)),
             ((8, 56, 56, 256), (0, 1, 1, 0), (0, 1, 1, 0)), ((4, 9, 9, 3), (0, 0, 0, 0), (0, 0, 0, 5)), ((3, 4, 4, 16), (0, 2, 0, 0), (0, 0, 3, 0))]


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
@pytest.mark.parametrize("pad_type", [R.ZERO, R.REPLICATE])
@pytest.mark.parametrize("case", range(len(PAD_CASES)))
def test_pad(dev, kname, pad_type, case):
    """forward on packed tensors (vector path where the inner axis is not padded), on an offset copy of a (element path: the same
    bits), and the backward on packed tensors and on views"""
    nnc = dev.nnc
    shape, begin, end = PAD_CASES[case]
    bshape = tuple(shape[k] + begin[k] + end[k] for k in range(len(shape)))
    a = plant(bits(seeded(shape, case, -2, 2), kname), kname, case)
    want = R.pad_forward(a, begin, end, pad_type)
    fwd, bwd = nnc.CMD_PAD_FORWARD(pad_type, begin, end), nnc.CMD_PAD_BACKWARD(pad_type, begin, end)
    (got,) = _exec(dev, fwd, [a], [_sentinel_like(bshape, kname)], kname, launches=1)
    assert same(got, want)
    # a and b one element into larger buffers: not 16-byte aligned, so the element path
    m = int(np.prod(bshape))
    abase = dev.up(np.concatenate([a.reshape(-1)[:1], a.reshape(-1)]), kname)
    bbase = dev.up(_sentinel_like((m + 1,), kname), kname)
    sz = 4 if kname == "fp32" else 2
    at = nnc.tensor_new(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, NHWC, KINDS[kname], list(shape)), abase.data_ptr + sz)
    bt = nnc.tensor_new(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, NHWC, KINDS[kname], list(bshape)), bbase.data_ptr + sz)
    dev.owned.extend([at, bt])
    st, launches = dev.run(fwd, [at], [bt])
    assert st == 0 and launches == 1
    assert same(dev.down(bbase)[1:].reshape(bshape), want)
    # backward: h = g[begin : begin + dim]
    g = plant(bits(seeded(bshape, case + 50, -2, 2), kname), kname, case + 50)
    (h,) = _exec(dev, bwd, [g], [_sentinel_like(shape, kname)], kname, launches=1)
    assert same(h, R.pad_backward(g, begin, shape))
    if len(shape) >= 2 and shape[0] * shape[1] < 10 ** 6:
        # g and h as views: g inside a wider buffer, h as a pitched slice whose surroundings must stay untouched
        gw = np.concatenate([g, _sentinel_like(bshape[:-1] + (3,), kname)], axis=-1)
        hw = _sentinel_like(shape[:-1] + (shape[-1] + 2,), kname)
        gbase, hbase = dev.up(np.ascontiguousarray(gw), kname), dev.up(hw, kname)
        gs = [int(np.prod(gw.shape[k + 1:])) for k in range(len(shape))]
        hs = [int(np.prod(hw.shape[k + 1:])) for k in range(len(shape))]
        gv = dev.view(gbase, bshape, [0] * len(shape), gs)
        hv = dev.view(hbase, shape, [0] * (len(shape) - 1) + [1], hs)
        st, launches = dev.run(bwd, [gv], [hv])
        assert st == 0 and launches == 1
        got = dev.down(hbase)
        want_h = hw.copy()
        want_h[..., 1:1 + shape[-1]] = R.pad_backward(g, begin, shape)
        assert same(got, want_h)


CMP_SHAPES = [(7,), (64, 33), (3, 5, 7, 9), (8, 56, 56, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
@pytest.mark.parametrize("op", ["min", "max"])
@pytest.mark.parametrize("shape", CMP_SHAPES)
def test_min_max(dev, kname, op, shape):
    nnc = dev.nnc
    is_min = op == "min"
    fwd, bwd = (nnc.CMD_MIN_FORWARD(), nnc.CMD_MIN_BACKWARD()) if is_min else (nnc.CMD_MAX_FORWARD(), nnc.CMD_MAX_BACKWARD())
    a = plant(bits(seeded(shape, 1, -1, 1), kname), kname, 2)
    b = plant(bits(seeded(shape, 3, -1, 1), kname), kname, 4)
    flat_a, flat_b = a.reshape(-1), b.reshape(-1)
    flat_b[::5] = flat_a[::5]                      # ties (NaN against the same NaN too)
    g = plant(bits(seeded(shape, 5, -2, 2), kname), kname, 6)
    (c,) = _exec(dev, fwd, [a, b], [_sentinel_like(shape, kname)], kname, launches=1)
    assert same(c, R.cmp_forward(a, b, kname, is_min))
    for gg in (g, None):
        ha, hb = _exec(dev, bwd, [gg, a, b], [_sentinel_like(shape, kname)] * 2, kname, launches=1)
        wa, wb = R.cmp_backward(gg, a, b, kname, is_min)
        assert same(ha, wa) and same(hb, wb)
    # pitched views: every operand a slice of a wider buffer along its last axis
    if len(shape) >= 2:
        pitch = shape[-1] + 3

        def wide(x):
            w = _sentinel_like(shape[:-1] + (pitch,), kname)
            if x is not None:
                w[..., 2:2 + shape[-1]] = x
            base = dev.up(w, kname)
            st = [int(np.prod(w.shape[k + 1:])) for k in range(len(shape))]
            return base, w, dev.view(base, shape, [0] * (len(shape) - 1) + [2], st)
        (_, _, av), (_, _, bv), (_, _, gv) = wide(a), wide(b), wide(g)
        cbase, cw, cv = wide(None)
        assert dev.run(fwd, [av, bv], [cv]) == (0, 1)
        want = cw.copy()
        want[..., 2:2 + shape[-1]] = R.cmp_forward(a, b, kname, is_min)
        assert same(dev.down(cbase), want)
        for gg, ggv in ((g, gv), (None, None)):
            habase, haw, hav = wide(None)
            hbbase, hbw, hbv = wide(None)
            assert dev.run(bwd, [ggv, av, bv], [hav, hbv]) == (0, 1)
            wa, wb = R.cmp_backward(gg, a, b, kname, is_min)
            want_a, want_b = haw.copy(), hbw.copy()
            want_a[..., 2:2 + shape[-1]], want_b[..., 2:2 + shape[-1]] = wa, wb
            assert same(dev.down(habase), want_a) and same(dev.down(hbbase), want_b), gg is None


ARG_SHAPES = [(5, 1), (7, 1000), (3, 4097), (2, 128256), (4, 6, 33), (3, 5, 7, 9), (2, 300, 40), (64, 32000)]


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
@pytest.mark.parametrize("shape", ARG_SHAPES)
def test_argmax_argmin(dev, kname, shape):
    """every axis; NaN at index 0 and mid-row, all-equal rows, ties; int32 and fp32 outputs"""
    nnc = dev.nnc
    x = bits(np.round(seeded(shape, 7, -4, 4) * 8) / 8, kname)   # coarse values: many ties
    w = widen(x, kname)
    for axis in range(len(shape)):
        xa = np.moveaxis(x.copy(), axis, -1)
        rows = xa.reshape(-1, shape[axis])
        nan = bits(np.float32(np.nan), kname).reshape(-1)[0] if kname != "fp32" else np.float32(np.nan)
        if rows.shape[0] >= 1:
            rows[0, 0] = nan
        if rows.shape[0] >= 2 and shape[axis] > 2:
            rows[1, shape[axis] // 2] = nan
        if rows.shape[0] >= 3:
            rows[2, :] = rows[2, -1]
        xx = np.ascontiguousarray(np.moveaxis(rows.reshape(xa.shape), -1, axis))
        bshape = tuple(1 if k == axis else shape[k] for k in range(len(shape)))
        for op in ("max", "min"):
            cmd = nnc.CMD_ARGMAX_FORWARD(axis) if op == "max" else nnc.CMD_ARGMIN_FORWARD(axis)
            want = R.argext(widen(xx, kname), axis, op == "min")
            for out in (np.full(bshape, -1, np.int32), np.full(bshape, -1, np.float32)):
                ta, tb = dev.up(xx, kname), dev.nnc.gpu_tensor(list(bshape), NHWC, abi.CCV_32S if out.dtype == np.int32 else abi.CCV_32F).upload(out)
                dev.owned.append(tb)
                assert dev.run(cmd, [ta], [tb]) == (0, 1)
                got = dev.down(tb)
                assert np.array_equal(got, want.astype(out.dtype)), (axis, op, out.dtype)
    del w


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
def test_reduce_isnan_full_buffer(dev, kname):
    """REDUCE_ISNAN of a 25.6 M-element buffer to [1]: 0, one NaN at the first / last / a middle element, many NaNs; Inf never counts"""
    nnc = dev.nnc
    n = 25_600_000
    x = bits(seeded((n,), 9, -1, 1), kname)
    x[::1000] = bits(np.float32(np.inf), kname).reshape(-1)[0] if kname != "fp32" else np.inf
    nan = bits(np.float32(np.nan), kname).reshape(-1)[0] if kname != "fp32" else np.float32(np.nan)
    t = dev.up(x, kname)
    b = dev.up(np.full((1,), 5, np.int32))
    cmd = nnc.CMD_REDUCE_ISNAN_FORWARD()
    assert dev.run(cmd, [t], [b]) == (0, 2) and dev.down(b)[0] == 0
    for pos in (0, n - 1, n // 2 + 3, "many"):
        y = x.copy()
        if pos == "many":
            y[7::997] = nan
        else:
            y[pos] = nan
        t.upload(y.view(np.float16) if kname == "fp16" else y)
        b.upload(np.full((1,), 5, np.int32))
        assert dev.run(cmd, [t], [b]) == (0, 2) and dev.down(b)[0] == 1, pos
    t2 = dev.up(x[:n - 1], kname)  # not a whole number of vectors per row: the element path
    assert dev.run(cmd, [t2], [b]) == (0, 2) and dev.down(b)[0] == 0


ISNAN_CASES = [((4, 5, 6), (1, 1, 1)), ((4, 5, 6), (4, 1, 1)), ((4, 5, 6), (1, 5, 6)), ((4, 5, 6), (4, 5, 6)), ((4, 5, 6), (4, 1, 6)),
               ((3, 7, 9, 16), (3, 1, 1, 16)), ((3, 7, 9, 16), (1, 7, 1, 1)), ((64, 1000), (64, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("kname", list(KINDS))
@pytest.mark.parametrize("case", range(len(ISNAN_CASES)))
def test_reduce_isnan_axes_and_views(dev, kname, case):
    nnc = dev.nnc
    shape, bshape = ISNAN_CASES[case]
    x = bits(seeded(shape, case, -1, 1), kname)
    flat = x.reshape(-1)
    nan = bits(np.float32(np.nan), kname).reshape(-1)[0] if kname != "fp32" else np.float32(np.nan)
    inf = bits(np.float32(np.inf), kname).reshape(-1)[0] if kname != "fp32" else np.float32(np.inf)
    flat[::37], flat[5::41] = nan, inf
    want = R.reduce_isnan(widen(x, kname), bshape)
    (got,) = _exec(dev, nnc.CMD_REDUCE_ISNAN_FORWARD(), [x], [np.full(bshape, 5, np.int32)], kname, launches=2)
    assert np.array_equal(got, want)
    # a as a pitched view, b as a view into a wider int32 buffer
    pitch = shape[-1] + 4
    aw = np.concatenate([x, np.tile(nan, shape[:-1] + (4,)).astype(x.dtype)], axis=-1)
    abase = dev.up(np.ascontiguousarray(aw), kname)
    av = dev.view(abase, shape, [0] * len(shape), [int(np.prod(aw.shape[k + 1:])) for k in range(len(shape))])
    bw = np.full(bshape[:-1] + (bshape[-1] + 2,), 5, np.int32)
    bbase = dev.up(bw)
    bv = dev.view(bbase, bshape, [0] * (len(bshape) - 1) + [1], [int(np.prod(bw.shape[k + 1:])) for k in range(len(bshape))])
    assert dev.run(nnc.CMD_REDUCE_ISNAN_FORWARD(), [av], [bv]) == (0, 2)
    want_w = bw.copy()
    want_w[..., 1:1 + bshape[-1]] = want
    assert np.array_equal(dev.down(bbase), want_w)
    del pitch


@pytest.mark.gpu
def test_backward_of_argmax_argmin_isnan_is_invalid(dev):
    nnc = dev.nnc
    a, b = dev.up(seeded((4, 8), 1)), dev.up(np.full((4, 1), 5, np.int32))
    for cmd in (abi.CCV_NNC_ARGMAX_BACKWARD, abi.CCV_NNC_ARGMIN_BACKWARD, abi.CCV_NNC_REDUCE_ISNAN_BACKWARD):
        c = nnc._reduce(cmd, (1,))
        assert dev.run(c, [b, a], [a]) == (INVALID, 0)


@pytest.mark.gpu
def test_refusals(dev):
    """INVALID with no kernel launched and every output untouched"""
    nnc = dev.nnc
    S = 7.0

    def refused(cmd, ins, outs):
        st, n = dev.run(cmd, ins, outs)
        assert st == INVALID and n == 0, (hex(cmd.cmd), st, n)
        for t in outs:
            if t is not None:
                x = dev.down(t)
                assert (x == (5 if x.dtype == np.int32 else S)).all() or (x.dtype == np.uint16 and (x == bits(np.float32(S), "bf16")[()]).all())
    f = lambda *s: dev.up(seeded(s, 1))
    sent = lambda *s: dev.up(np.full(s, S, np.float32))
    h16 = lambda *s: dev.up(bits(np.full(s, S, np.float32), "bf16"), "bf16")
    i32 = lambda *s: dev.up(np.full(s, 5, np.int32))
    pz, pr = nnc.CMD_PAD_FORWARD(R.ZERO, (1, 1), (1, 1)), nnc.CMD_PAD_BACKWARD(R.REPLICATE, (1, 1), (1, 1))
    refused(pz, [f(4, 4)], [sent(6, 7)])                                     # mismatched shape
    refused(pz, [f(4, 4)], [h16(6, 6)])                                      # mixed types
    refused(nnc.CMD_PAD_FORWARD(R.ZERO, (-1, 1), (1, 1)), [f(4, 4)], [sent(4, 6)])  # negative begin
    refused(nnc.CMD_PAD_FORWARD(R.ZERO, (0,) * 5, (1,) * 5), [f(2, 2, 2, 2, 2)], [sent(3, 3, 3, 3, 3)])  # 5 axes
    bad_type = nnc.CMD_PAD_FORWARD(R.ZERO, (1, 1), (1, 1))
    bad_type.info.pad.type = 2
    refused(bad_type, [f(4, 4)], [sent(6, 6)])
    refused(pr, [f(6, 6)], [sent(4, 5)])
    refused(pr, [None], [sent(4, 4)])
    mx, mxb = nnc.CMD_MAX_FORWARD(), nnc.CMD_MAX_BACKWARD()
    refused(mx, [f(4, 8), f(4, 9)], [sent(4, 8)])                            # no broadcasting
    refused(mx, [f(4, 8), f(1, 8)], [sent(4, 8)])
    refused(mx, [f(4, 8), f(4, 8)], [h16(4, 8)])
    refused(mx, [f(4, 8), None], [sent(4, 8)])
    refused(mxb, [f(4, 8), f(4, 8), None], [sent(4, 8), sent(4, 8)])         # b missing
    refused(mxb, [f(4, 8), f(4, 8), f(4, 8)], [sent(4, 8), None])            # hb missing
    refused(mxb, [f(4, 9), f(4, 8), f(4, 8)], [sent(4, 8), sent(4, 8)])
    am = nnc.CMD_ARGMAX_FORWARD(1)
    refused(am, [f(4, 8)], [i32(4, 2)])                                      # count mismatch
    refused(am, [f(4, 8)], [i32(2, 2)])                                      # the right count, the wrong shape
    refused(am, [f(4, 8)], [i32(1, 4)])
    refused(am, [f(4, 8)], [i32(4)])                                         # the reduced axis dropped
    refused(nnc.CMD_ARGMAX_FORWARD(2), [f(4, 8)], [i32(4, 1)])               # axis out of range
    two = nnc._reduce(abi.CCV_NNC_ARGMAX_FORWARD, (0, 1))
    refused(two, [f(4, 8)], [i32(1, 1)])                                     # reduce.count != 1
    refused(am, [f(4, 8)], [h16(4, 1)])                                      # a 16-bit index
    base = f(4, 16)
    refused(am, [dev.view(base, [4, 8], [0, 0], [16, 1])], [i32(4, 1)])      # a view
    isn = nnc.CMD_REDUCE_ISNAN_FORWARD()
    refused(isn, [f(4, 8)], [sent(1, 1)])                                    # fp32 flag
    refused(isn, [f(4, 8)], [i32(3, 1)])                                     # not broadcast onto a
    refused(isn, [f(2, 2, 2, 2, 2)], [i32(1, 1, 1, 1, 1)])
    q = nnc.gpu_palettized_tensor([4, 8], abi.CCV_32F, 4, 8)
    q.upload(np.zeros(q.nbytes, np.uint8))
    dev.owned.append(q)
    refused(mx, [q, f(4, 8)], [sent(4, 8)])
    refused(isn, [q], [i32(1, 1)])
    refused(am, [q], [i32(4, 1)])
    refused(pz, [q], [sent(6, 10)])


@pytest.mark.gpu
def test_accumulate_output_overwrites_and_results_repeat(dev):
    nnc = dev.nnc
    a, b = bits(seeded((8, 56, 56, 64), 3, -1, 1), "bf16"), plant(bits(seeded((8, 56, 56, 64), 4, -1, 1), "bf16"), "bf16", 1)
    ta, tb, tc = dev.up(a, "bf16"), dev.up(b, "bf16"), dev.up(_sentinel_like(a.shape, "bf16"), "bf16")
    first = None
    for flags in (0, abi.CCV_NNC_ACCUMULATE_OUTPUT, 0):
        st, n = dev.run(nnc.CMD_MAX_FORWARD(), [ta, tb], [tc], flags)
        assert (st, n) == (0, 1)
        got = dev.down(tc)
        first = got if first is None else first
        assert same(got, first)
    assert same(first, R.cmp_forward(a, b, "bf16", False))
    x = bits(seeded((64, 32000), 5, -1, 1), "bf16")
    tx, ti = dev.up(x, "bf16"), dev.up(np.zeros((64, 1), np.int32))
    outs = []
    for _ in range(3):
        assert dev.run(nnc.CMD_ARGMAX_FORWARD(1), [tx], [ti], abi.CCV_NNC_ACCUMULATE_OUTPUT) == (0, 1)
        outs.append(dev.down(ti))
    assert all(np.array_equal(o, outs[0]) for o in outs)


@pytest.mark.gpu
@pytest.mark.parametrize("kname", ["bf16", "fp16"])
def test_training_step_overflow_check(gpu, kname):
    """ccv_cnnp_model_parameter_gradients_isnan (lib/nnc/ccv_cnnp_model_addons.c:180-199) on the 16-bit ResNet-50 driver: REDUCE_ISNAN
    over the flat 16-bit gradient buffer, then the int32 EWSUM into an accumulator: 0 after a clean backward, 1 with one NaN gradient"""
    from ccv_b200 import resnet50
    from tests.test_resnet_parity import BATCH, CLASSES, IMAGE, _inputs
    from tests.util import pack16
    nnc, kind = gpu, KINDS[kname]
    stream = nnc.Stream(0)
    x, lab = _inputs()
    net = resnet50.Net(BATCH, image=IMAGE, classes=CLASSES, seed=7, dtype=kind)
    flag, acc = nnc.gpu_tensor([1], NHWC, abi.CCV_32S), nnc.gpu_tensor([1], NHWC, abi.CCV_32S)
    try:
        net.input.upload(pack16(x, kind)), net.labels.upload(lab)
        for cmd, hint, flags, ins, outs in net.fwd + net.bwd:
            assert nnc.cmd_exec(cmd, hint, flags, ins, outs, stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()

        def check():
            acc.upload(np.zeros(1, np.int32))
            assert nnc.cmd_exec(nnc.CMD_REDUCE_ISNAN_FORWARD(), None, 0, [net.g_flat], [flag], stream) == 0
            assert nnc.cmd_exec(nnc.CMD_EWSUM_FORWARD(), None, 0, [acc, flag], [acc], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
            stream.wait()
            return int(acc.download()[0])
        assert check() == 0
        g = net.g_flat.download()
        g16 = g.view(np.uint16).copy()
        assert np.isfinite(R.widen(g16, kname)).all() and (g16 != 0).any()
        g16[g16.size // 3] = 0x7fc0 if kname == "bf16" else 0x7e00
        net.g_flat.upload(g16.view(np.float16) if kname == "fp16" else g16)
        assert check() == 1
    finally:
        for t in (flag, acc, net, stream):
            t.free()


@pytest.mark.gpu
def test_reference_addon_programs_pass_on_the_dropin_build(gpu, tmp_path):
    """int.compare and int.pad (every case) and the argmin / argmax / isnan cases of int.reduce, through
    integration/run_reference_tests.py: they pass and none is skipped"""
    import json
    import subprocess
    import sys
    build = os.path.join(ROOT, "integration", "_build")
    progs = ("int.compare", "int.pad", "int.reduce")
    if not os.path.exists(os.path.join(build, "libccv_dropin.so")) or not all(os.path.exists(os.path.join(build, p + ".tests")) for p in progs):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    out = str(tmp_path / "report.json")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_reference_tests.py"), "--only", ",".join(progs), "--budget-s", "300",
                        "--case-timeout", "60", "--out", out], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=400)
    assert p.returncode == 0, p.stdout.decode()[-2000:]
    rep = json.load(open(out))["programs"]
    cmp_, pad, red = rep["int.compare.tests"], rep["int.pad.tests"], rep["int.reduce.tests"]
    for prog, count in ((cmp_, 4), (pad, 12)):
        assert len(prog["passed"]) == count and not prog["skipped"] and not prog["failed"] and not prog["crashed"], prog
    mine = ("argmin with float", "argmax with float", "reduce isnan float", "reduce isnan in half precision")
    assert all(n in red["passed"] for n in mine), red
    assert not any(n in red["skipped"] or n in red["failed"] for n in mine), red


# ---- a chain through ccv_nnc_cmd_exec against CPU_REF --------------------------------------------------------------------------
# fp32: the convolution's bound of the fp32 parity tests (1e-3 of max|ref|; PAD, MAX and the routing of the MAX gradient are exact);
# bf16: the 16-bit rule of tests/test_parity_16bit.py (1e-2 of max|ref|: CPU_REF in fp32 on the rounded inputs, every GPU output rounded
# to bf16 once).  The second MAX operand sits at least 5 % of max|y| away from the convolution's output, so that neither bound can flip
# which side a MAX gradient goes to.
CHAIN_BOUND = {"fp32": 1e-3, "bf16": 1e-2}


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_pad_conv_max_argmax_chain(gpu, ref, kname):
    """replicate PAD (1 pixel) -> 3x3 CONVOLUTION without border -> MAX with a second tensor -> ARGMAX over channels, then MAX_BACKWARD ->
    CONVOLUTION_BACKWARD -> PAD_BACKWARD, on the GPU and on CPU_REF; argmax indices are compared where CPU_REF's top-two margin exceeds
    twice the bound"""
    from tests.util import ref_exec, round16, pack16, unpack16
    nnc, kind = gpu, KINDS[kname]
    N, H, W, C, K = 2, 16, 16, 16, 32
    r16 = (lambda v: v) if kname == "fp32" else (lambda v: round16(v, kind))
    z = lambda *s: np.zeros(s, np.float32)
    x = r16(seeded((N, H, W, C), 61, -1, 1))
    w = r16((seeded((K, 3, 3, C), 62, -1, 1) / np.sqrt(9 * C)).astype(np.float32))
    bias = r16(seeded((K,), 63, -0.1, 0.1))
    g = r16(seeded((N, H, W, K), 64, -1, 1))
    pad_f = nnc.CMD_PAD_FORWARD(abi.CCV_NNC_PAD_REPLICATE, (0, 1, 1, 0), (0, 1, 1, 0))
    pad_b = nnc.CMD_PAD_BACKWARD(abi.CCV_NNC_PAD_REPLICATE, (0, 1, 1, 0), (0, 1, 1, 0))
    conv_f, conv_b = nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, C), nnc.CMD_CONVOLUTION_BACKWARD(1, K, 3, 3, C)
    hint = nnc.hint((1, 1), (0, 0))
    mx_f, mx_b, am = nnc.CMD_MAX_FORWARD(), nnc.CMD_MAX_BACKWARD(), nnc.CMD_ARGMAX_FORWARD(3)

    def cpu(cmd, ins, outs, h=None):
        st, res = ref_exec(ref, cmd, h, 0, ins, outs)
        assert st == 0, hex(cmd.cmd)
        return res
    (xp,) = cpu(pad_f, [x], [z(N, H + 2, W + 2, C)])
    (y,) = cpu(conv_f, [xp, w, bias], [z(N, H, W, K)], hint)
    scale = np.abs(y).max()
    sign = np.where(seeded(y.shape, 65) > 0.5, 1.0, -1.0)
    m = r16((y + sign * scale * (0.05 + 0.2 * seeded(y.shape, 66))).astype(np.float32))
    (zz,) = cpu(mx_f, [y, m], [z(N, H, W, K)])
    (idx,) = cpu(am, [zz], [np.zeros((N, H, W, 1), np.int32)])
    gy, gm = cpu(mx_b, [g, y, m], [z(N, H, W, K), z(N, H, W, K)])
    dxp, dw, db = cpu(conv_b, [gy, xp, w], [z(N, H + 2, W + 2, C), z(K, 3, 3, C), z(K)], hint)
    (dx,) = cpu(pad_b, [dxp], [z(N, H, W, C)])
    want = dict(xp=xp, y=y, z=zz, gy=gy, gm=gm, dxp=dxp, dw=dw, db=db, dx=dx)

    owned, stream = [], nnc.Stream(0)

    def new(shape, dt=kind):
        t = nnc.gpu_tensor(list(shape), NHWC, dt)
        owned.append(t)
        return t

    def up(arr):
        return new(arr.shape).upload(arr if kname == "fp32" else pack16(arr, kind))

    def run(cmd, ins, outs, h=None):
        assert nnc.cmd_exec(cmd, h, 0, ins, outs, stream) == 0, (hex(cmd.cmd), nnc.lib().ccv_nnc_sm100_last_error())
        return outs

    def down(t):
        stream.wait()
        d = t.download()
        return d if (t.params.datatype & 0xFF000) in (abi.CCV_32F, abi.CCV_32S) else unpack16(d, kind)
    try:
        xg, wg, bg, gg, mg = up(x), up(w), up(bias), up(g), up(m)
        (xpg,) = run(pad_f, [xg], [new((N, H + 2, W + 2, C))])
        (yg,) = run(conv_f, [xpg, wg, bg], [new((N, H, W, K))], hint)
        (zg,) = run(mx_f, [yg, mg], [new((N, H, W, K))])
        (ig,) = run(am, [zg], [new((N, H, W, 1), abi.CCV_32S)])
        gyg, gmg = run(mx_b, [gg, yg, mg], [new((N, H, W, K)), new((N, H, W, K))])
        dxpg, dwg, dbg = run(conv_b, [gyg, xpg, wg], [new((N, H + 2, W + 2, C)), new((K, 3, 3, C)), new((K,))], hint)
        (dxg,) = run(pad_b, [dxpg], [new((N, H, W, C))])
        got = dict(xp=down(xpg), y=down(yg), z=down(zg), gy=down(gyg), gm=down(gmg), dxp=down(dxpg), dw=down(dwg), db=down(dbg), dx=down(dxg))
        idx_g = down(ig)
    finally:
        stream.wait()
        for t in reversed(owned):
            t.free()
        stream.free()
    tol = CHAIN_BOUND[kname]
    errs = dict((k, float(np.abs(got[k].astype(np.float64) - want[k]).max() / max(np.abs(want[k]).max(), 1e-30))) for k in want)
    print("pad / conv / max / argmax chain %s: max error / max|ref| %s" % (kname, ", ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    for k, e in errs.items():
        assert np.isfinite(got[k]).all() and e <= tol, (kname, k, errs)
    # PAD and the routing of g are exact: the padded input and the MAX gradients hold the same bits as CPU_REF (16-bit: as its rounded inputs)
    assert np.array_equal(got["xp"], want["xp"]) and np.array_equal(got["gy"], want["gy"]) and np.array_equal(got["gm"], want["gm"])
    top2 = np.sort(zz, axis=3)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 2 * tol * np.abs(zz).max()
    assert clear.mean() > 0.5, clear.mean()
    assert np.array_equal(idx_g[..., 0][clear], idx[..., 0][clear])
