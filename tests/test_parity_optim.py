"""LAMB and RMSPROP on CCV_NNC_BACKEND_GPU_SM100 against the reference's CPU_REF (the `ref` fixture), bit for bit.

The kernels round every product and sum on their own in CPU_REF's association, so RMSPROP's b, n, u and LAMB's n, u equal CPU_REF's bits.
LAMB's b also depends on the trust ratio, a quotient of float64 norms whose sums run in another order on the GPU; it equals CPU_REF's
bits whenever the float64 quotient is far from a float32 rounding midpoint, and every case here asserts that margin (2^-40, relative).
16-bit operands: CPU_REF on the widened values, each output rounded once."""
import numpy as np
import pytest

from ccv_b200 import abi
from tests import optim_ref as R
from tests.test_parity_feeder_paths import _resnet50_param_counts
from tests.util import NHWC, from_bf16, pack16, ref_exec, round16, seeded

pytestmark = pytest.mark.gpu

KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID
LAMB_HP = dict(step=3, rate=0.01, beta1=0.9, beta2=0.999, decay=0.01, epsilon=1e-6, scale=0.5)
RMSPROP_HP = dict(rate=0.001, decay=0.01, alpha=0.9, momentum=0.9, epsilon=1e-6, scale=0.5)
LAMB_LAUNCHES, RMSPROP_LAUNCHES = 3, 1
COUNTS = [1, 3, 4095, 4096, 4097, 10007, (1 << 20) + 3]
# the aliasing forms of the reference's own tests: out of place, in place, (b, m, v) and (a, n, u)
ALIASES = ("out", "in_place", "b_mv", "a_nu")


def _cmd(nnc, which, **over):
    if which == "lamb":
        hp = dict(LAMB_HP, **over)
        return nnc.CMD_LAMB_FORWARD(hp["step"], hp["rate"], hp["beta1"], hp["beta2"], hp["decay"], hp["epsilon"], scale=hp["scale"])
    hp = dict(RMSPROP_HP, **over)
    return nnc.CMD_RMSPROP_FORWARD(hp["rate"], hp["decay"], hp["alpha"], hp["momentum"], hp["epsilon"], scale=hp["scale"])


def _inputs(count, seed, gk="fp32", sk="fp32"):
    """g, a, m, v (v >= 0) holding values of their kinds, as float32"""
    x = [seeded((count,), seed, -1, 1), seeded((count,), seed + 1, -1, 1), seeded((count,), seed + 2, -0.1, 0.1), seeded((count,), seed + 3, 0, 0.01)]
    return [x[0] if gk == "fp32" else round16(x[0], KINDS[gk])] + [y if sk == "fp32" else round16(y, KINDS[sk]) for y in x[1:]]


def _bits(x, kind="fp32"):
    """float32 values -> the bits a tensor of `kind` holds (one rounding for 16-bit kinds)"""
    x = np.ascontiguousarray(x, np.float32).ravel()
    return x.view(np.uint32) if kind == "fp32" else np.asarray(pack16(x, KINDS[kind])).view(np.uint16)


def _widen(bits, kind):
    if kind == "fp32":
        return bits.view(np.float32)
    return from_bf16(bits) if kind == "bf16" else bits.view(np.float16).astype(np.float32)


def _same(got, want, kind="fp32"):
    """bitwise, except that any NaN matches any NaN (CPU_REF's x86 NaN and the GPU's canonical NaN differ in sign and payload)"""
    w = _bits(want, kind)
    g = np.ascontiguousarray(got).ravel()
    g = g.view(np.uint32) if g.dtype == np.float32 else g.view(np.uint16)
    if g.shape != w.shape:
        return False
    nan = np.isnan(_widen(w, kind))
    return np.array_equal(np.isnan(_widen(g, kind)), nan) and np.array_equal(g[~nan], w[~nan])


def _cpu_ref(ref, which, ins, **over):
    """CPU_REF on float32 (widened) inputs -> (b, n, u) float32"""
    c = len(ins[1])
    from ccv_b200 import nnc
    st, outs = ref_exec(ref, _cmd(nnc, which, **over), None, 0, [np.ascontiguousarray(x, np.float32) for x in ins], [np.zeros(c, np.float32) for _ in range(3)])
    assert st == 0
    return outs


def _assert_margin(ins, **over):
    hp = dict(LAMB_HP, **over)
    _, _, _, t64 = R.lamb(*ins, hp["step"], hp["rate"], hp["beta1"], hp["beta2"], hp["decay"], hp["epsilon"], hp["scale"])
    assert t64 is None or R.midpoint_margin(t64) > 2.0 ** -40, t64


class _Dev(object):
    """GPU tensors, each a slice at element offset `off` of a larger buffer; all freed by free()"""

    def __init__(self, nnc):
        self.nnc, self.owned = nnc, []

    def up(self, x, kind="fp32", off=0):
        dt = KINDS[kind]
        big = self.nnc.gpu_tensor([x.size + off + 1], NHWC, dt)
        host = np.concatenate([np.zeros(off, np.float32), np.asarray(x, np.float32).ravel(), np.zeros(1, np.float32)])
        big.upload(host if kind == "fp32" else pack16(host, dt))
        t = self.nnc.gpu_tensor([x.size], NHWC, dt, ptr=big.data_ptr + off * (4 if kind == "fp32" else 2))
        self.owned += [t, big]
        return t

    @staticmethod
    def down(t):
        x = t.download()
        return x.view(np.uint16) if x.dtype == np.float16 else x

    def run(self, cmd, ins, outs):
        l0 = self.nnc.launch_count()
        st = self.nnc.cmd_exec(cmd, None, 0, ins, outs)
        return st, self.nnc.launch_count() - l0

    def free(self):
        for t in reversed(self.owned):
            t.free()
        self.owned = []


def _gpu(nnc, which, ins, gk="fp32", sk="fp32", off=0, alias="out", cmd=None):
    """one command on GPU copies of ins -> (status, launches, b, n, u as raw arrays)"""
    d = _Dev(nnc)
    try:
        tg = d.up(ins[0], gk, off)
        ta, tm, tv = (d.up(x, sk, off) for x in ins[1:])
        fresh = lambda: d.up(np.zeros(len(ins[1]), np.float32), sk, off)
        outs = {"out": lambda: [fresh(), fresh(), fresh()], "in_place": lambda: [ta, tm, tv], "b_mv": lambda: [fresh(), tm, tv], "a_nu": lambda: [ta, fresh(), fresh()]}[alias]()
        st, launches = d.run(cmd or _cmd(nnc, which), [tg, ta, tm, tv], outs)
        return (st, launches) + tuple(d.down(t) for t in outs)
    finally:
        d.free()


# ---- fp32 -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("which", ["lamb", "rmsprop"])
def test_fp32_matches_cpu_ref(gpu, ref, which, count, offset):
    """aligned (4-element vectors when the count allows) and misaligned-by-one slices; every aliasing form; two runs, same bits"""
    ins = _inputs(count, 11 + count % 97)
    want = _cpu_ref(ref, which, ins)
    if which == "lamb":
        _assert_margin(ins)
    first = None
    for alias in ALIASES:
        st, launches, b, n, u = _gpu(gpu, which, ins, off=offset, alias=alias)
        assert st == 0 and launches == (LAMB_LAUNCHES if which == "lamb" else RMSPROP_LAUNCHES), (st, launches)
        assert _same(b, want[0]) and _same(n, want[1]) and _same(u, want[2]), (which, alias)
        first = first or (b, n, u)
    again = _gpu(gpu, which, ins, off=offset)[2:]
    assert all(np.array_equal(x, y) for x, y in zip(first, again))


@pytest.mark.parametrize("gk", ["bf16", "fp16"])
@pytest.mark.parametrize("which", ["lamb", "rmsprop"])
def test_16bit_gradient_with_fp32_state(gpu, ref, which, gk):
    for count, off in ((10007, 0), (4096, 0), (4097, 1)):
        ins = _inputs(count, 23, gk=gk)
        want = _cpu_ref(ref, which, ins)
        if which == "lamb":
            _assert_margin(ins)
        st, _, b, n, u = _gpu(gpu, which, ins, gk=gk, off=off)
        assert st == 0 and _same(b, want[0]) and _same(n, want[1]) and _same(u, want[2]), (count, off)


@pytest.mark.parametrize("gk", ["fp32", "same"])
@pytest.mark.parametrize("sk", ["bf16", "fp16"])
@pytest.mark.parametrize("which", ["lamb", "rmsprop"])
def test_16bit_state(gpu, ref, which, sk, gk):
    """CPU_REF on the widened inputs; b, n, u each rounded once.  LAMB's norms are over the widened a and the unrounded update."""
    gk = sk if gk == "same" else gk
    for count, off, alias in ((10007, 0, "out"), (4096, 0, "in_place"), (4097, 1, "b_mv")):
        ins = _inputs(count, 31, gk=gk, sk=sk)
        want = _cpu_ref(ref, which, ins)
        if which == "lamb":
            _assert_margin(ins)
        st, _, b, n, u = _gpu(gpu, which, ins, gk=gk, sk=sk, off=off, alias=alias)
        assert st == 0 and _same(b, want[0], sk) and _same(n, want[1], sk) and _same(u, want[2], sk), (count, off, alias)


def test_edge_cases(gpu, ref):
    """zero weights (trust 1), a zero update with decay 0 (trust 1), NaN and +-Inf gradients (trust 1 for LAMB: a NaN norm)"""
    count = 4099
    g, a, m, v = _inputs(count, 41)
    cases = {"zero_a": ([g, np.zeros(count, np.float32), m, v], {}),
             "zero_update": ([np.zeros(count, np.float32), a, np.zeros(count, np.float32), v], dict(decay=0.0)),
             "nan_inf_g": ([np.where(np.arange(count) % 1000 == 7, np.float32(np.nan), np.where(np.arange(count) % 1000 == 8, np.float32(np.inf), np.where(np.arange(count) % 1000 == 9, np.float32(-np.inf), g))).astype(np.float32), a, m, v], {})}
    for name, (ins, over) in cases.items():
        for which in ("lamb", "rmsprop"):
            want = _cpu_ref(ref, which, ins, **over)
            st, _, b, n, u = _gpu(gpu, which, ins, cmd=_cmd(gpu, which, **over))
            assert st == 0 and _same(b, want[0]) and _same(n, want[1]) and _same(u, want[2]), (name, which)
        if name != "nan_inf_g":
            hp = dict(LAMB_HP, **over)
            assert R.lamb(*ins, hp["step"], hp["rate"], hp["beta1"], hp["beta2"], hp["decay"], hp["epsilon"], hp["scale"])[3] is None, name


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing_and_leave_outputs_untouched(gpu):
    nnc, count = gpu, 4096
    d = _Dev(nnc)
    try:
        g, a, m, v = (d.up(x) for x in _inputs(count, 51))
        outs = [d.up(np.full(count, 7, np.float32)) for _ in range(3)]
        g16 = d.up(np.zeros(count, np.float32), "bf16")
        short = d.up(np.zeros(count - 1, np.float32))
        ints = nnc.gpu_tensor([count], NHWC, abi.CCV_32S)
        qx = nnc.gpu_palettized_tensor([count], abi.CCV_32F, 4, 128)
        base = d.up(np.zeros(2 * count, np.float32))
        strided = nnc.tensor_view_new(base, [count // 64, 64], [0] * 12, [128, 1] + [0] * 10)
        d.owned += [ints, qx, strided]
        bad = {"step 0 (lamb)": (("lamb",), [g, a, m, v], outs, dict(step=0)),
               "3 inputs": (("lamb", "rmsprop"), [g, a, m], outs, {}),
               "2 outputs": (("lamb", "rmsprop"), [g, a, m, v], outs[:2], {}),
               "NULL operand": (("lamb", "rmsprop"), [g, a, None, v], outs, {}),
               "NULL output": (("lamb", "rmsprop"), [g, a, m, v], [outs[0], None, outs[2]], {}),
               "counts differ": (("lamb", "rmsprop"), [g, a, short, v], outs, {}),
               "mixed state types": (("lamb", "rmsprop"), [g, a, g16, v], outs, {}),
               "integer operand": (("lamb", "rmsprop"), [ints, a, m, v], outs, {}),
               "palettized operand": (("lamb", "rmsprop"), [g, qx, m, v], outs, {}),
               "non-contiguous view": (("lamb", "rmsprop"), [g, a, m, strided], outs, {})}
        for name, (whiches, ins, os_, over) in bad.items():
            for which in whiches:
                st, launches = d.run(_cmd(nnc, which, **over), ins, os_)
                assert (st, launches) == (INVALID, 0), (name, which, st, launches)
        for t in outs:
            assert np.all(t.download() == 7)
        for which in ("lamb", "rmsprop"):
            bwd = nnc.CMD_LAMB_BACKWARD(1, 0.1, 0.9, 0.99, 0, 1e-6) if which == "lamb" else nnc.CMD_RMSPROP_BACKWARD(0.1, 0, 0.9, 0, 1e-6)
            assert d.run(bwd, [g, a, m, v], outs) == (INVALID, 0)
    finally:
        d.free()


# ---- fused graph runs -------------------------------------------------------------------------------------------------------------
def _fused(nnc, which, counts, gk="fp32", sk="fp32", odd=(), decays=None):
    """T commands in one graph, fused and not -> (data, [(b, n, u) per tensor], launches, nodes) for each of fused / unfused"""
    data = [_inputs(c, 100 + 3 * i, gk, sk) for i, c in enumerate(counts)]
    stream = nnc.Stream(0)
    d = _Dev(nnc)
    try:
        res = []
        for fuse in (True, False):
            ts = [[d.up(x, gk if j == 0 else sk, 1 if i in odd else 0) for j, x in enumerate(q)] for i, q in enumerate(data)]
            gr = nnc.Graph()
            try:
                for i, (tg, ta, tm, tv) in enumerate(ts):
                    over = {} if decays is None else dict(decay=decays[i])
                    gr.exec_new(_cmd(nnc, which, **over), None, 0, [tg, ta, tm, tv], [ta, tm, tv])
                if fuse:
                    gr.fuse()
                nodes = [k for _, k, _, _ in gr.nodes()]
                l0 = nnc.launch_count()
                assert gr.run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
                stream.wait()
                launches = nnc.launch_count() - l0
            finally:
                gr.free()
            res.append(([tuple(d.down(t) for t in q[1:]) for q in ts], launches, nodes))
            d.free()
        return data, res
    finally:
        d.free()
        stream.free()


FUSED = [([4] * 1, ()), ([4096] * 31, ()), ([4100] * 33, ()), ([8188, 8196, 4] * 11, ()), ([4, 4096, 4100, 8188, 8196, 1, 4] * 10, ()),
         ([4096, 4100, 4099, 8192, 8192], (2, 3)), ([4100] * 70, ())]


@pytest.mark.parametrize("counts,odd", FUSED, ids=lambda v: "T%d" % len(v) if isinstance(v, list) else str(v))
@pytest.mark.parametrize("which", ["lamb", "rmsprop"])
def test_fused_is_the_unfused_commands(gpu, which, counts, odd):
    """runs longer than one launch's table, mixed counts, an odd count and misaligned tensors in the middle: the fused node gives the
    bits of the single commands (each LAMB tensor its own trust ratio), in the restated plan's launches"""
    data, ((bf, lf, kf), (bu, lu, ku)) = _fused(gpu, which, counts, odd=odd)
    per = LAMB_LAUNCHES if which == "lamb" else RMSPROP_LAUNCHES
    assert kf == ([9 if which == "lamb" else 10] if len(counts) > 1 else [0])
    assert lf == per * len(R.optim_multi_plan(counts)) and lu == per * len(counts), (lf, lu)
    for i in range(len(counts)):
        assert all(np.array_equal(x, y) for x, y in zip(bf[i], bu[i])), "tensor %d: the fused node differs from the command" % i


@pytest.mark.parametrize("gk", ["fp32", "bf16"])
@pytest.mark.parametrize("which", ["lamb", "rmsprop"])
def test_fused_resnet50_parameters(gpu, ref, which, gk):
    """ResNet-50's 161 parameters, weights with decay and the rest without, interleaved as the model lists them: two nodes (one per
    decay group), the restated plan's launches, every tensor the bits of its own command (and CPU_REF's for a sample of them)"""
    counts = _resnet50_param_counts()
    assert len(counts) == 161 and sum(counts) == 25557032
    decays = [0.01 if c > 4096 else 0.0 for c in counts]
    data, ((bf, lf, kf), (bu, lu, _)) = _fused(gpu, which, counts, gk=gk, decays=decays)
    kind = 9 if which == "lamb" else 10
    assert kf == [kind, kind]
    groups = [[c for c, dk in zip(counts, decays) if dk == x] for x in (0.01, 0.0)]
    per = LAMB_LAUNCHES if which == "lamb" else RMSPROP_LAUNCHES
    assert lf == per * sum(len(R.optim_multi_plan(g)) for g in groups) and lu == per * 161
    for i in range(len(counts)):
        assert all(np.array_equal(x, y) for x, y in zip(bf[i], bu[i])), i
    for i in (0, 1, 3, 150, 159, 160):
        if which == "lamb":
            _assert_margin(data[i], decay=decays[i])
        want = _cpu_ref(ref, which, data[i], decay=decays[i])
        assert all(_same(x, w) for x, w in zip(bf[i], want)), i


# ---- the reference's own programs on the drop-in build ---------------------------------------------------------------------------
def test_reference_lamb_and_rmsprop_programs_pass_on_the_dropin_build(gpu, tmp_path):
    from tests.test_dropin import _built, _run
    if not _built(["int.lamb", "int.rmsprop"]):
        pytest.skip("integration/_build is not built (make -C integration; needs the reference sources)")
    rep = _run(["int.lamb", "int.rmsprop"], 300, tmp_path)
    for prog in ("int.lamb.tests", "int.rmsprop.tests"):
        r = rep["programs"][prog]
        assert not r["failed"] and not r["crashed"] and r["tally"]["PASS"] == 3, (prog, r)
