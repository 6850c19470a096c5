"""ADAM / ADAMW, RANDOM_UNIFORM / RANDOM_NORMAL and DROPOUT on CCV_NNC_BACKEND_GPU_SM100, bit for bit against the restatements of
tests/adam_ref.py (pinned to CPU_REF by tests/golden/cpuref_adam.npz) and tests/random_ref.py (Philox 4x32-10 and the host's seeds).

Every output lives between NaN guards that must stay NaN; every call is made twice (the generator re-seeded in between) and must give
the same bits; the launches are the restated plan (one kernel, or for 16-bit optimizer state the functional form: widen every distinct
16-bit tensor, the fp32 kernel, narrow every 16-bit output, aliased tensors sharing one shadow).  The normal is held to a per-element
bound, since the device's logf / cosf / sinf are not correctly rounded; everything else is exact."""
import ctypes as C

import numpy as np
import pytest

from ccv_b200 import abi
from tests import adam_ref as A
from tests import contract_ref as cr
from tests import random_ref as R
from tests.feeder_ref import staged_f32_launches
from tests.golden.make_adam_golden import NAN_AT, NEG_INF_AT, POS_INF_AT, ZERO_A, ZERO_G
from tests.test_parity_feeder_paths import BF16, DT, F16, F32, GUARD, INVALID, SENTINEL, Dev, _refused, run, run_twice
from tests.util import NHWC, ref_exec, round16, seeded

KINDS = (F32, BF16, F16)
f32 = np.float32


def one_pass():
    """threads in one grid-stride pass of a 256-thread launch, the grid capped at 8 blocks per SM"""
    return 8 * cr.device_sms() * 256


def r16(x, kind):
    return np.asarray(x, f32) if kind == F32 else round16(x, DT[kind])


def seeder(nnc):
    lib = nnc.lib()
    lib.ccv_nnc_stream_context_set_seed.argtypes = [C.c_void_p, C.c_uint32]
    lib.ccv_nnc_stream_context_set_seed.restype = None
    return lambda stream, seed: lib.ccv_nnc_stream_context_set_seed(stream, seed)


# ---- ADAM / ADAMW -------------------------------------------------------------------------------------------------------------------
HP = dict(step=3, rate=0.01, beta1=0.9, beta2=0.999, decay=0.05, epsilon=1e-8, scale=0.5)
COUNTS = [1, 3, 255, 256, 257, 10007, "pass+1"]


def adam_cmd(nnc, adamw, amsgrad, hp=HP):
    hp = dict(hp)
    scale = hp.pop("scale")
    return (nnc.CMD_ADAMW_FORWARD if adamw else nnc.CMD_ADAM_FORWARD)(amsgrad=amsgrad, scale=scale, **hp)


def adam_state(count, seed, gkind=F32, skind=F32):
    """g (of gkind), a, m, v >= 0, vm >= 0 (of skind); NaN, +-Inf and zero gradients and zero weights where the count reaches them"""
    g, a = seeded((count,), seed, -1, 1), seeded((count,), seed + 1, -1, 1)
    m, v, vm = seeded((count,), seed + 2, -0.1, 0.1), seeded((count,), seed + 3, 0, 0.01), seeded((count,), seed + 4, 0, 0.04)
    for i, x in ((NAN_AT, np.nan), (POS_INF_AT, np.inf), (NEG_INF_AT, -np.inf)) + tuple((i, 0.0) for i in ZERO_G):
        if i < count:
            g[i] = x
    for i in ZERO_A:
        if i < count:
            a[i] = 0
    return r16(g, gkind), r16(a, skind), r16(m, skind), r16(v, skind), r16(vm, skind)


def adam_want(adamw, amsgrad, g, a, m, v, vm, hp=HP, skind=F32, with_vm=True):
    b, n, u, um = A.adam(g, a, m, v, amsgrad=amsgrad, vm=vm if with_vm else None, adamw=bool(adamw), **hp)
    return [r16(x, skind) for x in (b, n, u)] + ([] if um is None else [r16(um, skind)])


def assert_same(got, want, what):
    for i, (x, y) in enumerate(zip(got, want)):
        if not A.same(x, y):
            x, y = np.asarray(x).ravel(), np.asarray(y).ravel()
            nan = np.isnan(x) & np.isnan(y)
            bad = np.flatnonzero(~nan & ((x != y) | (np.signbit(x) != np.signbit(y))))
            raise AssertionError("%s output %d: %d elements differ, first %s: got %r want %r" % (what, i, bad.size, bad[:4].tolist(), x[bad[:4]].tolist(), y[bad[:4]].tolist()))


@pytest.mark.gpu
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("amsgrad", [0, 1])
@pytest.mark.parametrize("adamw", [0, 1])
def test_adam_paths(gpu, adamw, amsgrad, count):
    """fp32 state with fp32, bf16 and fp16 gradients: one launch, CPU_REF's bits out of place and the same bits in place (b = a, n = m,
    u = v, um = vm); count "pass+1" is one element past a single grid-stride pass"""
    nnc = gpu
    count = one_pass() + 1 if count == "pass+1" else count
    cmd = adam_cmd(nnc, adamw, amsgrad)
    for gkind in KINDS:
        g, a, m, v, vm = adam_state(count, 11 + count % 7, gkind)
        ins = [g, a, m, v] + ([vm] if amsgrad else [])
        want = adam_want(adamw, amsgrad, g, a, m, v, vm)
        kg = lambda i, o: {id(i[0]): gkind}
        st, got, launches = run_twice(nnc, cmd, lambda: (ins, [np.zeros(count, f32) for _ in ins[1:]]), kg)
        assert st == 0 and launches == 1, (st, launches)
        assert_same(got, want, "out of place, g %s" % gkind)
        inplace = [x.copy() for x in ins[1:]]
        st, got_i, _ = run(nnc, cmd, [g] + inplace, inplace, {id(g): gkind})
        assert st == 0
        assert_same(got_i, got, "in place, g %s" % gkind)


@pytest.mark.gpu
@pytest.mark.parametrize("adamw", [0, 1])
def test_adam_partial_aliases_and_odd_offset(gpu, adamw):
    """b = a alone, n = m and u = v alone, um = vm alone each give the out-of-place bits; so does every operand at an odd element offset"""
    nnc = gpu
    count = 10007
    cmd = adam_cmd(nnc, adamw, 1)
    g, a, m, v, vm = adam_state(count, 41)
    want = adam_want(adamw, 1, g, a, m, v, vm)
    for alias in ({0}, {1, 2}, {3}):
        ins = [g, a.copy(), m.copy(), v.copy(), vm.copy()]
        outs = [ins[1 + k] if k in alias else np.zeros(count, f32) for k in range(4)]
        st, got, launches = run(nnc, cmd, ins, outs)
        assert st == 0 and launches == 1
        assert_same(got, want, "aliases %s" % sorted(alias))
    st, got, _ = run(nnc, cmd, [g, a, m, v, vm], [np.zeros(count, f32) for _ in range(4)], offset=1)
    assert st == 0
    assert_same(got, want, "odd offset")


@pytest.mark.gpu
@pytest.mark.parametrize("adamw", [0, 1])
def test_adam_amsgrad_needs_both_vm_and_um(gpu, adamw):
    """amsgrad without vm / um, or with vm but no um, is the plain update; vm / um under amsgrad 0 are ignored and um is not written"""
    nnc = gpu
    count = 4099
    g, a, m, v, vm = adam_state(count, 61)
    plain = adam_want(adamw, 0, g, a, m, v, vm)
    z = lambda: np.zeros(count, f32)
    for amsgrad, ins, outs in ((1, [g, a, m, v], [z(), z(), z()]), (1, [g, a, m, v, vm], [z(), z(), z()]),
                               (0, [g, a, m, v, vm], [z(), z(), z(), np.full(count, SENTINEL, f32)])):
        st, got, launches = run(nnc, adam_cmd(nnc, adamw, amsgrad), ins, outs)
        assert st == 0 and launches == 1
        assert_same(got[:3], plain[:3], "amsgrad %d, %d inputs, %d outputs" % (amsgrad, len(ins), len(outs)))
        if len(got) == 4:
            assert (got[3] == SENTINEL).all()


@pytest.mark.gpu
@pytest.mark.parametrize("skind", [BF16, F16])
@pytest.mark.parametrize("amsgrad", [0, 1])
@pytest.mark.parametrize("adamw", [0, 1])
def test_adam_16bit_state(gpu, adamw, amsgrad, skind):
    """bf16 / fp16 parameters and moments take the functional form: each output is the fp32 update of the widened operands, rounded
    once; in place the shadows are shared (one widen per tensor), out of place every distinct tensor is widened"""
    nnc = gpu
    count = 3001
    cmd = adam_cmd(nnc, adamw, amsgrad)
    for gkind in (F32, skind):
        g, a, m, v, vm = adam_state(count, 71, gkind, skind)
        state = [a, m, v] + ([vm] if amsgrad else [])
        want = adam_want(adamw, amsgrad, g, a, m, v, vm, skind=skind)
        g16 = int(gkind != F32)
        outs = [np.zeros(count, f32) for _ in state]
        kinds = lambda i, o: dict([(id(i[0]), gkind)] + [(id(x), skind) for x in i[1:] + o])
        st, got, launches = run_twice(nnc, cmd, lambda: ([g] + state, outs), kinds)
        assert st == 0 and launches == staged_f32_launches(g16 + 2 * len(state), len(state)), launches
        assert_same(got, want, "%s state, g %s, out of place" % (skind, gkind))
        inplace = [x.copy() for x in state]
        st, got_i, launches = run(nnc, cmd, [g] + inplace, inplace, kinds([g] + inplace, []))
        assert st == 0 and launches == staged_f32_launches(g16 + len(state), len(state)), launches
        assert_same(got_i, want, "%s state, g %s, in place" % (skind, gkind))


@pytest.mark.gpu
def test_adam_fixture_cases(gpu):
    """the committed CPU_REF fixture, case by case (in place where CPU_REF ran in place): the kernel gives CPU_REF's bits"""
    import os
    from tests.golden.make_adam_golden import CASES, cmd_of
    path = os.path.join(os.path.dirname(__file__), "golden", "cpuref_adam.npz")
    z = np.load(path)
    nnc = gpu
    for case in CASES:
        name, amsgrad, in_place = case[0], case[2], case[-1]
        ins = [z["%s_%s" % (k, name)] for k in ("g", "a", "m", "v")] + ([z["vm_" + name]] if amsgrad else [])
        ins = [ins[0]] + [x.copy() for x in ins[1:]]
        outs = ins[1:] if in_place else [np.zeros_like(x) for x in ins[1:]]
        st, got, launches = run(nnc, cmd_of(case), ins, outs)
        assert st == 0 and launches == 1
        assert_same(got, [z["%s_%s" % (k, name)] for k in ("b", "n", "u", "um")[:3 + amsgrad]], name)


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("adamw", [0, 1])
def test_adam_against_cpu_ref(gpu, ref, adamw):
    """a fresh case against the compiled reference: step 1000, rate 1, amsgrad, a bf16 gradient widened for CPU_REF"""
    nnc = gpu
    hp = dict(step=1000, rate=1.0, beta1=0.9, beta2=0.999, decay=0.1, epsilon=1e-6, scale=2.0)
    cmd = adam_cmd(nnc, adamw, 1, hp)
    for gkind in (F32, BF16):
        g, a, m, v, vm = adam_state(20011, 81, gkind)
        st_r, want = ref_exec(ref, cmd, None, 0, [g, a, m, v, vm], [np.zeros_like(a) for _ in range(4)])
        st, got, _ = run(nnc, cmd, [g, a, m, v, vm], [np.zeros_like(a) for _ in range(4)], {id(g): gkind})
        assert st_r == 0 and st == 0
        assert_same(got, want, "against CPU_REF, g %s" % gkind)
        assert_same(want, adam_want(adamw, 1, g, a, m, v, vm, hp), "oracle against CPU_REF")


@pytest.mark.gpu
def test_adam_refusals(gpu):
    """views, step 0, a count that differs, a 16-bit vm under fp32 state and the backward commands: INVALID, nothing launched, outputs
    untouched"""
    nnc = gpu
    r = lambda n, s=3: seeded((n,), s, 0.1, 0.9)
    s = lambda n: np.full(n, SENTINEL, f32)
    for adamw in (0, 1):
        _refused(nnc, adam_cmd(nnc, adamw, 0, dict(HP, step=0)), [r(8), r(8), r(8), r(8)], [s(8), s(8), s(8)])
        _refused(nnc, adam_cmd(nnc, adamw, 0), [r(8), r(8), r(7), r(8)], [s(8), s(8), s(8)])
        _refused(nnc, adam_cmd(nnc, adamw, 0), [r(8), r(8), r(8), r(8)], [s(8), s(9), s(8)])
        vm = r(8)
        _refused(nnc, adam_cmd(nnc, adamw, 1), [r(8), r(8), r(8), r(8), vm], [s(8), s(8), s(8), s(8)], {id(vm): BF16})
        back = adam_cmd(nnc, adamw, 0)
        back.cmd = abi.CCV_NNC_ADAMW_BACKWARD if adamw else abi.CCV_NNC_ADAM_BACKWARD
        _refused(nnc, back, [r(8), r(8), r(8), r(8)], [s(8), s(8), s(8)])
        # a parameter that is a view with a wider row pitch
        wide = nnc.gpu_tensor([4, 12]).upload(seeded((4, 12), 5, 0.1, 0.9))
        v = nnc.tensor_view_new(wide, [4, 10], [0] * 12, [12, 1] + [0] * 10)
        ts = [nnc.gpu_tensor([4, 10]).upload(seeded((4, 10), 6 + i, 0.1, 0.9)) for i in range(3)]
        outs = [nnc.gpu_tensor([4, 10]).upload(s(40).reshape(4, 10)) for _ in range(3)]
        try:
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(adam_cmd(nnc, adamw, 0), None, 0, [ts[0], v, ts[1], ts[2]], outs) == INVALID and nnc.launch_count() == l0
            assert all((o.download() == SENTINEL).all() for o in outs)
        finally:
            for t in [v, wide] + ts + outs:
                t.free()


# ---- RANDOM_UNIFORM / RANDOM_NORMAL ----------------------------------------------------------------------------------------------------
RANDOM_COUNTS = [1, 2, 3, 5, 1023, "4pass+5"]
UNIFORM_BOUNDS = [(-2.0, 3.0), (0.0, 1.0), (-5.0, -1.0), (1.0, 7.0)]
NORMAL_PARAMS = [(1.0, 0.0), (2.0, 1.0), (0.02, -3.0)]
SEED = 0x5EED0


def _fill(nnc, set_seed, cmd, n, kind, seed):
    """the command on a fresh guarded tensor, the thread's generator seeded first, made twice -> (values, launches)"""
    def make():
        set_seed(None, seed)
        return [], [np.zeros(n, f32)]
    st, (y,), launches = run_twice(nnc, cmd, make, lambda i, o: {id(o[0]): kind})
    assert st == 0 and launches == 1, (st, launches)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", RANDOM_COUNTS)
def test_random_uniform(gpu, n, kind):
    """fp32 is the restated stream bit for bit; bf16 / fp16 hold that value rounded once.  A second call draws the next seed.  Count
    "4pass+5" makes the quad loop stride."""
    nnc = gpu
    set_seed = seeder(nnc)
    n = 4 * one_pass() + 5 if n == "4pass+5" else n
    for lo, hi in UNIFORM_BOUNDS:
        cmd = nnc.CMD_RANDOM_UNIFORM_FORWARD(lo, hi)
        t = R.Seeds(SEED)
        y = _fill(nnc, set_seed, cmd, n, kind, SEED)
        assert_same([y], [r16(R.uniform(t.next(), n, lo, hi), kind)], "uniform [%g, %g] %s" % (lo, hi, kind))
        st, (y2,), _ = run(nnc, cmd, [], [np.zeros(n, f32)], {})  # fp32, the generator as the two calls above left it
        assert st == 0
        assert_same([y2], [R.uniform(t.next(), n, lo, hi)], "the next call draws the next seed")
        assert lo <= y.min() and y.max() <= hi


def _within_normal(y, want, e, kind):
    """fp32: |y - want| <= e; 16-bit: y lies between the roundings of want - e and want + e"""
    if kind == F32:
        return np.abs(y.astype(np.float64) - want) <= e
    return (r16((want - e).astype(f32), kind) <= y) & (y <= r16((want + e).astype(f32), kind))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", RANDOM_COUNTS)
def test_random_normal(gpu, n, kind):
    """Box-Muller on the restated stream, each element within its derived bound of the exact value on the device's float32 inputs"""
    nnc = gpu
    set_seed = seeder(nnc)
    n = 4 * one_pass() + 5 if n == "4pass+5" else n
    for std, mean in NORMAL_PARAMS:
        t = R.Seeds(SEED + 1)
        y = _fill(nnc, set_seed, nnc.CMD_RANDOM_NORMAL_FORWARD(std, mean), n, kind, SEED + 1)
        want, e = R.normal(t.next(), n, std, mean)
        ok = _within_normal(y, want, e, kind)
        assert ok.all(), ("normal", std, mean, kind, int((~ok).sum()), np.flatnonzero(~ok)[:4].tolist())


@pytest.mark.gpu
def test_random_seeds_from_a_stream_context(gpu):
    """a Stream's own generator, seeded on its own: its calls draw consecutive seeds from it and leave the thread's alone; an unseeded
    Stream seeds itself from the thread's generator"""
    nnc = gpu
    set_seed = seeder(nnc)
    n, cmd = 1029, nnc.CMD_RANDOM_UNIFORM_FORWARD(-1.0, 1.0)
    streams = [nnc.Stream(0), nnc.Stream(0)]
    ts = [nnc.gpu_tensor([n]) for _ in range(5)]
    try:
        set_seed(None, 5)
        set_seed(streams[0].ptr, 6)
        thread, own = R.Seeds(5), R.Seeds(6)
        for t in ts[:2]:
            assert nnc.cmd_exec(cmd, None, 0, [], [t], streams[0]) == 0
        assert nnc.cmd_exec(cmd, None, 0, [], [ts[2]]) == 0
        assert nnc.cmd_exec(cmd, None, 0, [], [ts[3]], streams[1]) == 0
        assert nnc.cmd_exec(cmd, None, 0, [], [ts[4]]) == 0
        for s in streams:
            s.wait()
        want = [own.next(), own.next(), thread.next()]
        fresh = R.Seeds.from_thread(thread)
        want += [fresh.next(), thread.next()]
        for t, seed in zip(ts, want):
            assert_same([t.download()], [R.uniform(seed, n, -1.0, 1.0)], "seed %#x" % seed)
    finally:
        for t in ts:
            t.free()
        for s in streams:
            s.free()


@pytest.mark.gpu
def test_random_refusals(gpu):
    """an int32 tensor and a view: INVALID, nothing launched, the tensor untouched and no seed drawn"""
    nnc = gpu
    set_seed = seeder(nnc)
    cmd = nnc.CMD_RANDOM_UNIFORM_FORWARD(0.0, 1.0)
    set_seed(None, 9)
    wide = nnc.gpu_tensor([4, 12]).upload(np.full((4, 12), SENTINEL, f32))
    v = nnc.tensor_view_new(wide, [4, 10], [0] * 12, [12, 1] + [0] * 10)
    it = nnc.gpu_tensor([16], NHWC, abi.CCV_32S).upload(np.full(16, 7, np.int32))
    try:
        for t in (v, it):
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(cmd, None, 0, [], [t]) == INVALID and nnc.launch_count() == l0
        assert (wide.download() == SENTINEL).all() and (it.download() == 7).all()
    finally:
        for t in (v, wide, it):
            t.free()
    st, (y,), _ = run(nnc, cmd, [], [np.zeros(64, f32)])
    assert st == 0
    assert_same([y], [R.uniform(R.Seeds(9).next(), 64, 0.0, 1.0)], "the first seed after the refusals")


# ---- DROPOUT ----------------------------------------------------------------------------------------------------------------------------
DROP_P = [0.0, 0.15, 0.2, 0.5, 0.9, 1.0]
FILL = 0xA5


def drop_shapes(p):
    """ragged shapes; with p 0.15 and 0.9 also one whose quads (and elements) stride past one grid pass"""
    shapes = [(1,), (3, 37, 41), (2, 1, 5)]
    if p in (0.15, 0.9):
        cols = 4 * one_pass() // 255 + 2
        shapes.append((255, cols | 1))
    return shapes


def mask_shape(shape, kind, entirety):
    """the reference's reserved mask (dropout/ccv_nnc_dropout.c:21-44): the input's type in 128-byte lines; for `entirety` the int32
    decision, one element of an fp32 tensor (the backend refuses a mask of fewer than four bytes, such as one 16-bit element)"""
    inc = 4 if kind == F32 else 2
    return [4 // inc] if entirety else [128 // inc, (shape[0] + 127) // 128 * int(np.prod(shape[1:]))]


def mask_tensor(nnc, dev, dims, kind, raw=None, dt=None):
    """a mask tensor of these dims between GUARD bytes, every byte FILL (or `raw`) -> (tensor, the guarded byte buffer)"""
    dt = DT[kind] if dt is None else dt
    size = int(np.prod(dims)) * abi.DTYPE_SIZE[dt]
    host = np.full(size + 2 * GUARD, FILL, np.uint8)
    if raw is not None:
        host[GUARD:GUARD + raw.size] = raw
    big = nnc.gpu_tensor([host.size], NHWC, abi.CCV_8U).upload(host)
    t = nnc.gpu_tensor(list(dims), NHWC, dt, ptr=big.data_ptr + GUARD)
    dev.owned += [t, big]
    return t, big


def dropout_fwd(nnc, cmd, a, kind, mdims):
    """-> (status, b, mask bytes with their guards, launches); b lives between NaN guards"""
    dev = Dev(nnc)
    try:
        ta, tb = dev.put(a, kind), dev.put(np.zeros_like(a), kind, guard=True)
        tm, big = mask_tensor(nnc, dev, mdims, kind)
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(cmd, None, 0, [ta], [tb, tm])
        launches = nnc.launch_count() - l0
        b = dev.get(tb, kind)
        dev.check()
        return st, b, big.download(), launches
    finally:
        dev.free()


def dropout_bwd(nnc, cmd, g, kind, mdims, raw, mdt=None):
    dev = Dev(nnc)
    try:
        tg, th = dev.put(g, kind), dev.put(np.zeros_like(g), kind, guard=True)
        tm, _ = mask_tensor(nnc, dev, mdims, kind, raw, mdt)
        l0 = nnc.launch_count()
        st = nnc.cmd_exec(cmd, None, 0, [tg, None, None, None, tm], [th])
        launches = nnc.launch_count() - l0
        h = dev.get(th, kind)
        dev.check()
        return st, h, launches
    finally:
        dev.free()


@pytest.mark.gpu
@pytest.mark.parametrize("p", DROP_P)
@pytest.mark.parametrize("entirety", [0, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_dropout_forward_backward(gpu, kind, entirety, p):
    """the forward's mask is the restated stream (u <= p, one byte per element, or the int32 decision in mask[0]) and b the kept elements
    times 1 / (1 - p) rounded once from double, bit for bit; the mask bytes past n keep their contents; the backward on that mask is the
    same arithmetic on g"""
    nnc = gpu
    set_seed = seeder(nnc)
    fwd, bwd = nnc.CMD_DROPOUT_FORWARD(p, entirety), nnc.CMD_DROPOUT_BACKWARD(p, entirety)
    for shape in drop_shapes(p):
        n = int(np.prod(shape))
        a, g = r16(seeded(shape, 1, -2, 2), kind), r16(seeded(shape, 2, -2, 2), kind)
        mdims = mask_shape(shape, kind, entirety)
        first = None
        for _ in range(2):
            set_seed(None, SEED + 2)
            got = dropout_fwd(nnc, fwd, a, kind, mdims)
            assert got[0] == 0 and got[3] == 1, (got[0], got[3])
            if first is not None:
                assert A.same(got[1], first[1]) and np.array_equal(got[2], first[2]), "two runs differ"
            first = got
        _, b, raw, _ = first
        mask = raw[GUARD:raw.size - GUARD]
        want_mask = R.dropout_mask(R.Seeds(SEED + 2).next(), n, p, entirety)
        assert np.array_equal(mask[:want_mask.size], want_mask), (shape, int((mask[:want_mask.size] != want_mask).sum()))
        assert (mask[want_mask.size:] == FILL).all() and (raw[:GUARD] == FILL).all() and (raw[raw.size - GUARD:] == FILL).all()
        assert_same([b], [r16(R.dropout_apply(a, want_mask, p, entirety), kind).reshape(shape)], "forward %s p %g %s" % (shape, p, kind))
        st, h, launches = dropout_bwd(nnc, bwd, g, kind, mdims, mask)
        assert st == 0 and launches == 1
        assert_same([h], [r16(R.dropout_apply(g, want_mask, p, entirety), kind).reshape(shape)], "backward %s p %g %s" % (shape, p, kind))


@pytest.mark.gpu
@pytest.mark.ref
@pytest.mark.parametrize("entirety", [0, 1])
def test_dropout_backward_on_cpu_ref_mask(gpu, ref, entirety):
    """the backward on CPU_REF's own mask (drawn from its generator) is CPU_REF's backward, bit for bit"""
    nnc = gpu
    shape, p = (3, 37, 41), 0.15
    a, g = seeded(shape, 1, -2, 2), seeded(shape, 2, -2, 2)
    mdims = mask_shape(shape, F32, entirety)
    st, (_, mask) = ref_exec(ref, nnc.CMD_DROPOUT_FORWARD(p, entirety), None, 0, [a], [np.zeros_like(a), np.zeros(mdims, f32)])
    assert st == 0
    bwd = nnc.CMD_DROPOUT_BACKWARD(p, entirety)
    st, (h_r,) = ref_exec(ref, bwd, None, 0, [g, None, None, None, mask], [np.zeros_like(g)])
    assert st == 0
    raw = mask.view(np.uint8).reshape(-1)
    for kind in KINDS:
        gk = r16(g, kind)
        st, h, _ = dropout_bwd(nnc, bwd, gk, kind, mdims, raw, abi.CCV_32F)
        assert st == 0
        assert_same([h], [r16(R.dropout_apply(gk, raw, p, entirety), kind).reshape(shape)], "backward on CPU_REF's mask, %s" % kind)
        if kind == F32:
            assert_same([h], [h_r], "against CPU_REF's backward")


@pytest.mark.gpu
def test_dropout_refusals(gpu):
    """a mask smaller than n (or than the int32 of `entirety`) and views: INVALID, nothing launched, b / h and the mask untouched"""
    nnc = gpu
    n = 100
    a = seeded((n,), 3, 0.1, 0.9)
    for entirety, small in ((0, n - 1), (1, 3)):
        fwd, bwd = nnc.CMD_DROPOUT_FORWARD(0.5, entirety), nnc.CMD_DROPOUT_BACKWARD(0.5, entirety)
        dev = Dev(nnc)
        try:
            ta, tb = dev.put(a), dev.put(np.full(n, SENTINEL, f32), guard=True)
            tm, big = mask_tensor(nnc, dev, [small], F32, dt=abi.CCV_8U)
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(fwd, None, 0, [ta], [tb, tm]) == INVALID
            assert nnc.cmd_exec(bwd, None, 0, [ta, None, None, None, tm], [tb]) == INVALID and nnc.launch_count() == l0
            assert (dev.get(tb) == SENTINEL).all() and (big.download() == FILL).all()
            dev.check()
        finally:
            dev.free()
    wide = nnc.gpu_tensor([4, 12]).upload(seeded((4, 12), 5, 0.1, 0.9))
    v = nnc.tensor_view_new(wide, [4, 10], [0] * 12, [12, 1] + [0] * 10)
    b = nnc.gpu_tensor([4, 10]).upload(np.full((4, 10), SENTINEL, f32))
    t = nnc.gpu_tensor([4, 10]).upload(seeded((4, 10), 6, 0.1, 0.9))
    m = nnc.gpu_tensor([64], NHWC, abi.CCV_8U).upload(np.full(64, FILL, np.uint8))
    try:
        l0 = nnc.launch_count()
        assert nnc.cmd_exec(nnc.CMD_DROPOUT_FORWARD(0.5), None, 0, [v], [b, m]) == INVALID
        assert nnc.cmd_exec(nnc.CMD_DROPOUT_FORWARD(0.5), None, 0, [t], [v, m]) == INVALID
        assert nnc.cmd_exec(nnc.CMD_DROPOUT_BACKWARD(0.5), None, 0, [v, None, None, None, m], [b]) == INVALID
        assert nnc.launch_count() == l0 and (b.download() == SENTINEL).all() and (m.download() == FILL).all()
    finally:
        for x in (v, wide, b, t, m):
            x.free()
