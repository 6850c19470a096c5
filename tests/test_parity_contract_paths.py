"""Every launch path of the tensor-core contraction kernel against a float64 oracle at rounding-level bounds
(tests/contract_ref.py holds the oracle, the bounds and the restated launch planner).

Each case names the path it was written for: one tile per CTA, CTAs walking M tiles, or split-K with the ordered combine.  The
test fails when the planner, run with the device's SM count, puts the case elsewhere, or when ccv_nnc_sm100_launch_count()
disagrees with the planned launches.  Every output lives inside a sentinel-filled buffer (GEMM outputs are views with a pitch
wider than N), is poisoned with NaN before a call that does not accumulate, must leave every guard element untouched, and must
come out bit-identical from a second run.  The cases are written for an H100 SXM (132 SMs).

The CPU tests pin the oracle to the committed CPU_REF fixtures and show, on every case shape, that the bounds reject the oracle
with each defect a kernel could plausibly have.  TF32 operands truncated instead of rounded is rejected on every fp32 case of the
matrix, not only those with K_eff <= 1024 (K_eff runs up to 4000 for the split GEMMs and 3136 for the weight gradients): the
operands have a positive mean, so the truncation bias grows with K_eff as fast as the scale does."""
import functools
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from ccv_b200 import abi
from tests import contract_ref as cr
from tests.contract_ref import BF16, FP16, FP32, TF32, X3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NHWC = abi.CCV_TENSOR_FORMAT_NHWC
ALGO = {TF32: abi.CCV_NNC_SM100_ALGO_TF32, X3: abi.CCV_NNC_SM100_ALGO_3XTF32, FP32: abi.CCV_NNC_SM100_ALGO_FFMA, BF16: -1, FP16: -1}
MODES = [TF32, X3, FP32, BF16, FP16]
SENTINEL = {FP32: 0x7FBADBAD, BF16: 0x7FBB, FP16: 0x7DBB}  # NaN patterns: an element the kernel never writes fails the bound


def _out_kind(mode):
    return mode if mode in (BF16, FP16) else FP32


def _dt(mode):
    return {BF16: abi.CCV_16BF, FP16: abi.CCV_16F}.get(mode, abi.CCV_32F)


def _kind(mode):
    return {BF16: 1, FP16: 2}.get(mode, 0)


# ------------------------------------------------------------------------------------------------ the case matrix
class Case(object):
    def __init__(self, op, path, modes=MODES, bias=0, acc=False, bn=None, view=None, **kw):
        self.op, self.path, self.modes, self.bias, self.acc, self.bn, self.view = op, path, modes, bias, acc, bn, view
        self.kw = kw
        if op == "gemm":
            self.M, self.N, self.K, self.ta, self.tb = kw["M"], kw["N"], kw["K"], kw["ta"], kw["tb"]
            self.g = None
        else:
            self.g = cr.Geom(**dict((k, v) for k, v in kw.items() if k != "cview"))

    @property
    def family(self):
        if self.op == "gemm":
            return "gemm " + "NT"[self.ta] + "NT"[self.tb]
        if self.op == "dgrad":
            return "dgrad %s"
        if self.op == "wgrad":
            return "wgrad 1x1" if cr.pointwise(self.g) else "wgrad taps"
        return self.op

    def fam(self, mode):
        f = self.family
        return f % ("fp32" if _kind(mode) == 0 else "16-bit") if "%" in f else f

    def __repr__(self):
        if self.op == "gemm":
            s = "gemm%s %dx%dx%d" % ("NT"[self.ta] + "NT"[self.tb], self.M, self.N, self.K)
        else:
            g = self.g
            s = "%s N%d %dx%d C%d K%d %dx%d s%s p%s/%s d%s" % (self.op, g.N, g.H, g.W, g.C, g.K, g.R, g.S, g.st[0] if g.st[0] == g.st[1] else g.st, g.pad, g.pad_end, g.dil[0])
            if self.kw.get("cview"):
                s += " cview"
        return s + (" bias%d" % self.bias if self.bias else "") + (" acc" if self.acc else "") + (" BN%s" % self.bn if self.bn else "") + " ->" + self.path


def _gemm(path, M, N, K, **kw):
    return [Case("gemm", path, M=M, N=N, K=K, ta=ta, tb=tb, **kw) for ta in (0, 1) for tb in (0, 1)]


CASES = (
    # GEMM: all four transposes on every path; ragged M, N and K (K ragged for the 16-bit 64-deep steps)
    _gemm("tile", 296, 200, 96, bias=1, view=(8, 0))
    + _gemm("walk", 20000, 96, 264, view=(3, 1))
    + _gemm("walk", 20000, 200, 96, bias=2, view=(4, 0))
    + _gemm("split", 296, 200, 4000, bias=1, view=(5, 1))
    + [Case("gemm", "walk", M=20000, N=200, K=96, ta=0, tb=1, bn="64", view=(8, 0)),      # wide output on the 64-column kernel
       Case("gemm", "tile", M=1000, N=40, K=136, ta=1, tb=0, bn="128", view=(8, 1)),      # narrow output on the 128-column kernel
       Case("gemm", "tile", M=296, N=200, K=96, ta=0, tb=1, acc=True, view=(4, 0)),
       Case("gemm", "tile", M=296, N=200, K=96, ta=1, tb=0, acc=True, view=(3, 1)),
       Case("gemm", "split", M=296, N=200, K=4000, ta=0, tb=0, acc=True, view=(4, 0)),
       Case("gemm", "split", M=296, N=200, K=4000, ta=1, tb=0, acc=True, view=(5, 1)),
       Case("gemm", "walk", M=20000, N=96, K=264, ta=0, tb=1, acc=True, view=(8, 0))]
    # forward (IM2COL / K2D)
    + [Case("fwd", "tile", bias=1, N=2, H=14, W=14, C=40, K=48, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("fwd", "tile", N=4, H=29, W=29, C=48, K=72, R=3, S=3, stride=(2, 2), pad=(0, 0), pad_end=(1, 1)),
       Case("fwd", "tile", bias=2, N=2, H=15, W=15, C=72, K=64, R=3, S=3, stride=(1, 1), pad=(2, 2), dil=(2, 2)),
       Case("fwd", "tile", N=2, H=32, W=32, C=16, K=64, R=7, S=7, stride=(2, 2), pad=(3, 3)),
       Case("fwd", "tile", N=2, H=12, W=12, C=40, K=64, R=3, S=3, stride=(1, 1), pad=(1, 0), pad_end=(0, 1), cview=(8, 64)),
       Case("fwd", "tile", N=2, H=14, W=14, C=64, K=128, R=1, S=1, stride=(2, 2), pad=(0, 0)),
       Case("fwd", "walk", bias=1, N=8, H=56, W=56, C=64, K=64, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("fwd", "walk", N=32, H=63, W=63, C=40, K=72, R=3, S=3, stride=(2, 2), pad=(1, 1), pad_end=(0, 0)),
       Case("fwd", "walk", N=8, H=55, W=55, C=40, K=64, R=3, S=3, stride=(1, 1), pad=(1, 1), cview=(24, 72), bn="128")]
    # data gradient (fp32: filter copy + IM2COL / K2D; 16-bit: IM2COL / MN2D), by residue class of the stride
    + [Case("dgrad", "tile", N=2, H=13, W=13, C=40, K=48, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("dgrad", "tile", N=2, H=15, W=15, C=48, K=40, R=3, S=3, stride=(2, 2), pad=(0, 1), pad_end=(1, 0)),
       Case("dgrad", "tile", N=2, H=17, W=17, C=40, K=72, R=3, S=3, stride=(3, 3), pad=(1, 1)),
       Case("dgrad", "tile", N=2, H=15, W=15, C=64, K=128, R=1, S=1, stride=(2, 2), pad=(0, 0)),  # 3 of 4 classes have no tap
       Case("dgrad", "tile", N=2, H=15, W=15, C=64, K=72, R=3, S=3, stride=(1, 1), pad=(2, 2), dil=(2, 2)),
       Case("dgrad", "walk", N=8, H=56, W=56, C=64, K=64, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("dgrad", "walk", N=8, H=121, W=121, C=40, K=48, R=3, S=3, stride=(2, 2), pad=(1, 1))]
    # weight gradient, taps on grid z (MN2D / IM2COL) and 1x1 (MN2D / MN2D)
    + [Case("wgrad", "tile", N=2, H=7, W=7, C=1024, K=1024, R=3, S=3, stride=(1, 1), pad=(1, 1)),      # 576 tiles
       Case("wgrad", "tile", acc=True, N=2, H=7, W=7, C=512, K=512, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("wgrad", "split", N=4, H=28, W=28, C=64, K=128, R=3, S=3, stride=(1, 1), pad=(1, 1)),
       Case("wgrad", "split", acc=True, N=16, H=29, W=29, C=40, K=48, R=3, S=3, stride=(2, 2), pad=(0, 0), pad_end=(1, 1)),
       Case("wgrad", "tile", acc=True, N=2, H=7, W=7, C=256, K=512, R=1, S=1),
       Case("wgrad", "split", N=4, H=28, W=28, C=64, K=256, R=1, S=1),
       Case("wgrad", "split", acc=True, N=4, H=28, W=28, C=64, K=256, R=1, S=1, bn="128")]
)
PARAMS = [pytest.param(c, m, id="%s-%s" % (c, m)) for c in CASES for m in c.modes]

# statistics epilogue: convolution -> training batch norm, fused by the graph (N, H, C, K, R, channel offset)
STATS = [(8, 55, 64, 256, 3, 0.0),     # ragged last tile, two column blocks
         (8, 55, 64, 128, 3, 100.0),   # channel means ~100 standard deviations from zero
         (8, 55, 64, 256, 1, -60.0)]   # 1x1: the GEMM form of the forward
STATS_MODES = [TF32, BF16, FP16]

COVERAGE = {}
RAN = set()
REQUIRED = [("gemm " + t, p) for t in ("NN", "NT", "TN", "TT") for p in ("tile", "walk", "split")] + [
    ("fwd", "tile"), ("fwd", "walk"), ("dgrad fp32", "tile"), ("dgrad fp32", "walk"), ("dgrad 16-bit", "tile"), ("dgrad 16-bit", "walk"),
    ("wgrad taps", "tile"), ("wgrad taps", "split"), ("wgrad 1x1", "tile"), ("wgrad 1x1", "split"), ("stats", "walk")]
CALIBRATION = {}


# ------------------------------------------------------------------------------------------------ operands and oracle
def _seen_key(mode):
    return {TF32: "tf32", X3: "raw", FP32: "raw"}.get(mode, mode)


def _op_mode(mode):
    return mode if mode in (BF16, FP16) else FP32


@functools.lru_cache(maxsize=None)
def operands(case, mode):
    """host operands of `case` as the kernel receives them (fp32 arrays; 16-bit cases hold values on the 16-bit grid)"""
    om = _op_mode(mode)
    seed = zlib.crc32(repr(case).encode()) % 100000
    d = {}
    if case.op == "gemm":
        d["a"] = cr.operand((case.K, case.M) if case.ta else (case.M, case.K), seed + 1, om)
        d["b"] = cr.operand((case.N, case.K) if case.tb else (case.K, case.N), seed + 2, om)
        out_shape = (case.M, case.N)
    else:
        g = case.g
        if case.op in ("fwd", "wgrad"):
            cv = case.kw.get("cview")
            xs = (g.N, g.H, g.W, cv[1] if cv else g.C)
            d["xbig"] = cr.operand(xs, seed + 1, om)
            d["x"] = d["xbig"][..., cv[0]:cv[0] + g.C] if cv else d["xbig"]
        if case.op in ("fwd", "dgrad"):
            d["w"] = cr.operand((g.K, g.R, g.S, g.C), seed + 2, om)
        if case.op in ("dgrad", "wgrad"):
            d["gy"] = cr.operand((g.N, g.P, g.Q, g.K), seed + 3, om)
        out_shape = {"fwd": (g.N, g.P, g.Q, g.K), "dgrad": (g.N, g.H, g.W, g.C), "wgrad": (g.K, g.R, g.S, g.C)}[case.op]
    n = out_shape[-1]
    if case.bias:
        d["bias"] = cr.operand((n,), seed + 4, om if case.bias == 2 else FP32, 0.0, 2.0)
    if case.acc:
        d["old"] = cr.operand(out_shape, seed + 5, _out_kind(mode), -2.0, 2.0)
    d["out_shape"] = out_shape
    return d


def _f64(a):
    return None if a is None else np.asarray(a, np.float64)


@functools.lru_cache(maxsize=None)
def oracle(case, seen_key):
    """(y, s, K_eff) in float64 for the operands as the MMAs of this mode see them"""
    mode = {"tf32": TF32, "raw": FP32}.get(seen_key, seen_key)
    d = operands(case, mode)
    S = lambda a: cr.seen(a, mode)
    bias, old = _f64(d.get("bias")), _f64(d.get("old"))
    if case.op == "gemm":
        y, s = cr.gemm(S(d["a"]), S(d["b"]), case.ta, case.tb, bias, old)
        return y, s, float(case.K)
    g = case.g
    if case.op == "fwd":
        y, s = cr.with_scale(functools.partial(cr.conv_fwd, g), S(d["x"]), S(d["w"]), bias=bias)
        return y, s, float(g.R * g.S * g.C)
    if case.op == "dgrad":
        y, s = cr.with_scale(functools.partial(cr.conv_dgrad, g), S(d["gy"]), S(d["w"]))
        return y, s, g.keff_dgrad()
    y, s = cr.with_scale(functools.partial(cr.conv_wgrad, g), S(d["gy"]), S(d["x"]), old=old)
    return y, s, float(g.N * g.P * g.Q)


# ------------------------------------------------------------------------------------------------ CPU: the oracle pinned, the bounds able to fail
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_oracle_reproduces_committed_cpu_ref_gemm():
    f = np.load(os.path.join(GOLDEN, "cpuref_gemm.npz"))
    a, w, bias, g = (f[k].astype(np.float64) for k in ("a", "w", "bias", "g"))
    y, s = cr.gemm(a, w, 0, 1, bias)
    cr.check(f["b"], y, s, a.shape[1], FP32, FP32, "gemm forward")
    h, s = cr.gemm(g, w, 0, 0)
    cr.check(f["h"], h, s, g.shape[1], FP32, FP32, "gemm h")
    dw, s = cr.gemm(g, a, 1, 0)
    cr.check(f["dw"], dw, s, g.shape[0], FP32, FP32, "gemm dw")
    db, s = cr.gemm(np.ones((1, g.shape[0])), g, 0, 0)
    cr.check(f["db"], db[0], s[0], g.shape[0], FP32, FP32, "gemm dbias")


def test_oracle_reproduces_committed_cpu_ref_convolution():
    f = np.load(os.path.join(GOLDEN, "cpuref_conv.npz"))
    x, w, bias, gy = (f[k].astype(np.float64) for k in ("x", "w", "bias", "gy"))
    g = cr.Geom(2, 9, 11, 8, 12, 3, 3, stride=(2, 2), pad=(1, 1), P=5, Q=6)
    y, s = cr.with_scale(functools.partial(cr.conv_fwd, g), x, w, bias=bias)
    cr.check(f["y"], y, s, 72, FP32, FP32, "conv forward")
    h, s = cr.with_scale(functools.partial(cr.conv_dgrad, g), gy, w)
    cr.check(f["gx"], h, s, g.keff_dgrad(), FP32, FP32, "conv dgrad")
    dw, s = cr.with_scale(functools.partial(cr.conv_wgrad, g), gy, x)
    cr.check(f["gw"], dw, s, 60, FP32, FP32, "conv wgrad")
    db, s = cr.gemm(np.ones((1, 60)), gy.reshape(60, 12), 0, 0)
    cr.check(f["gb"], db[0], s[0], 60, FP32, FP32, "conv dbias")


@pytest.mark.ref
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_matches_compiled_reference(ref, seed):
    """GEMM and the three convolution products of CPU_REF on two seeded shapes each"""
    from ccv_b200 import nnc
    from tests.util import ref_exec
    r = np.random.RandomState(seed)
    M, N, K = (int(v) for v in r.randint(8, 70, 3))
    a, w, bias = cr.operand((M, K), seed, FP32), cr.operand((N, K), seed + 1, FP32), cr.operand((N,), seed + 2, FP32)
    _, (b,) = ref_exec(ref, nnc.CMD_GEMM_FORWARD((0, 0), (0, 1)), None, 0, [a, w, bias], [np.zeros((M, N), np.float32)])
    y, s = cr.gemm(_f64(a), _f64(w), 0, 1, _f64(bias))
    cr.check(b, y, s, K, FP32, FP32, "CPU_REF gemm")
    g = cr.Geom(2, 9 + seed, 8 + 2 * seed, 4 * seed, 6, 3, 3, stride=(seed, seed), pad=(1, 1))
    x, wt, gy = cr.operand((2, g.H, g.W, g.C), seed + 3, FP32), cr.operand((6, 3, 3, g.C), seed + 4, FP32), cr.operand((2, g.P, g.Q, 6), seed + 5, FP32)
    hint = nnc.hint(g.st, g.pad)
    _, (yr,) = ref_exec(ref, nnc.CMD_CONVOLUTION_FORWARD(1, 6, 3, 3, g.C), hint, 0, [x, wt], [np.zeros((2, g.P, g.Q, 6), np.float32)])
    _, (hr, dwr) = ref_exec(ref, nnc.CMD_CONVOLUTION_BACKWARD(1, 6, 3, 3, g.C), hint, 0, [gy, x, wt], [np.zeros_like(x), np.zeros_like(wt)])
    y, s = cr.with_scale(functools.partial(cr.conv_fwd, g), _f64(x), _f64(wt))
    cr.check(yr, y, s, 9 * g.C, FP32, FP32, "CPU_REF conv forward")
    h, s = cr.with_scale(functools.partial(cr.conv_dgrad, g), _f64(gy), _f64(wt))
    cr.check(hr, h, s, g.keff_dgrad(), FP32, FP32, "CPU_REF conv dgrad")
    dw, s = cr.with_scale(functools.partial(cr.conv_wgrad, g), _f64(gy), _f64(x))
    cr.check(dwr, dw, s, 2 * g.P * g.Q, FP32, FP32, "CPU_REF conv wgrad")


def _contribution(case, mode, part):
    """float64 contribution of one reduction chunk ("chunk"), one tap ("tap") or the first half of the reduction ("half")"""
    d = operands(case, mode)
    S = lambda a: cr.seen(a, mode)
    ck = 32 if _kind(mode) == 0 else 64
    if case.op == "gemm":
        A, B = S(d["a"]), S(d["b"])
        A, B = (A.T if case.ta else A), (B.T if case.tb else B)
        k = ck if part == "chunk" else case.K // 2
        return A[:, :k] @ B[:k]
    g = case.g
    mid = [(g.R // 2, g.S // 2)]
    if case.op == "fwd":
        x, w = S(d["x"]), S(d["w"])
        if part == "chunk":
            return cr.conv_fwd(g, x[..., :ck], w[..., :ck], taps=mid)
        return cr.conv_fwd(g, x, w, taps=mid) if part == "tap" else cr.conv_fwd(g, x[..., :g.C // 2], w[..., :g.C // 2])
    if case.op == "dgrad":
        gy, w = S(d["gy"]), S(d["w"])
        if part == "chunk":
            return cr.conv_dgrad(g, gy[..., :ck], w[:ck], taps=mid)
        return cr.conv_dgrad(g, gy, w, taps=mid) if part == "tap" else cr.conv_dgrad(g, gy[..., :g.K // 2], w[:g.K // 2])
    gy, x = S(d["gy"]), S(d["x"])
    if part == "tap":
        full = cr.conv_wgrad(g, gy, x)
        out = np.zeros_like(full)
        out[:, mid[0][0], mid[0][1]] = full[:, mid[0][0], mid[0][1]]
        return out
    return cr.conv_wgrad(g, gy, x, rows=slice(0, ck if part == "chunk" else g.N * g.P * g.Q // 2))


DEFECT_MODES = [TF32, BF16, FP16]


@pytest.mark.parametrize("case,mode", [pytest.param(c, m, id="%s-%s" % (c, m)) for c in CASES for m in DEFECT_MODES if m in c.modes])
def test_bounds_reject_defective_results(case, mode):
    """The oracle itself passes; with each defect of the kernel's arithmetic it does not."""
    out = _out_kind(mode)
    y, s, keff = oracle(case, _seen_key(mode))
    fin = (lambda v: cr.rne16(v, out)) if out != FP32 else (lambda v: np.asarray(v, np.float32).astype(np.float64))
    cr.check(fin(y), y, s, keff, mode, out, "correct result")

    def rejects(bad, what):
        assert not cr.admits(bad, y, s, keff, mode, out).all(), "%s: the %s bound admits %s" % (case, mode, what)

    d = operands(case, mode)
    rejects(fin(y - _contribution(case, mode, "chunk")), "one dropped reduction chunk")
    if case.op != "gemm":
        rejects(fin(y - _contribution(case, mode, "tap")), "one dropped tap")
    if out != FP32:
        rejects(cr.trunc16(y, out), "truncation instead of round-to-nearest-even")
        half = _contribution(case, mode, "half") + (_f64(d["old"]) if case.acc else 0.0)
        rejects(cr.rne16(cr.rne16(half, out) + cr.rne16(y - half, out), out), "a result rounded twice")
    if case.bias:
        rejects(fin(y + _f64(d["bias"])), "the bias added once more (once per split)")
    if case.acc:
        rejects(fin(y - _f64(d["old"])), "accumulation that ignores the old output")
    if mode == TF32:
        tr = lambda a: cr.seen(a, TF32, trunc=True)
        if case.op == "gemm":
            yt, _ = cr.gemm(tr(d["a"]), tr(d["b"]), case.ta, case.tb, _f64(d.get("bias")), _f64(d.get("old")))
        elif case.op == "fwd":
            yt = cr.conv_fwd(case.g, tr(d["x"]), tr(d["w"]), _f64(d.get("bias")))
        elif case.op == "dgrad":
            yt = cr.conv_dgrad(case.g, tr(d["gy"]), tr(d["w"]))
        else:
            yt = cr.conv_wgrad(case.g, tr(d["gy"]), tr(d["x"]), old=_f64(d.get("old")))
        rejects(fin(yt), "TF32 operands truncated instead of rounded")


def _rt(c, **kw):
    return Case("gemm", "tile", modes=[TF32], M=c[0], N=c[1], K=c[2], ta=c[3], tb=c[4], **kw)


def test_planner_restatement_on_hand_worked_shapes(monkeypatch):
    """launch_umma / pick_splits / fit_splits worked by hand for 132 and 114 SMs"""
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    p = cr.plan("gemm", 0, 132, M=4096, N=4096, K=64)
    assert p["launches"][0]["tiles"] == (32, 32, 1) and p["path"] == "walk" and p["launches"][0]["grid_x"] == 4
    assert cr.plan("gemm", 0, 114, M=4096, N=4096, K=64)["path"] == "tile"  # 1024 tiles: 3 CTAs per column would cost 11 rounds, not 9
    p = cr.plan("gemm", 0, 132, M=300, N=200, K=4096)  # 6 tiles: 2 * 132 / 6 = 44 splits, capped at 128 / 8 = 16
    assert p["launches"][0]["splits"] == 16 and p["kernels"] == 2 and p["path"] == "split"
    assert cr.plan("gemm", 1, 132, M=300, N=200, K=4096)["launches"][0]["splits"] == 8
    assert cr.plan("gemm", 1, 132, M=300, N=200, K=4096, bias16=True)["launches"][0]["splits"] == 1
    p = cr.plan("gemm", 0, 132, M=20000, N=200, K=96)  # 157 x 2 tiles: 66 CTAs per column, 3 tiles each
    assert p["launches"][0]["grid_x"] == 66 and p["path"] == "walk"
    g = cr.Geom(2, 7, 7, 1024, 1024, 3, 3, pad=(1, 1))
    p = cr.plan("wgrad", 0, 132, g=g)  # 8 x 8 x 9 = 576 >= 4 * 132 tiles: no split, and weight gradients never walk
    assert p["launches"][0]["tiles"] == (8, 8, 9) and p["path"] == "tile" and p["kernels"] == 1
    g = cr.Geom(2, 15, 15, 64, 128, 1, 1, stride=(2, 2))
    p = cr.plan("dgrad", 0, 132, g=g)  # one residue class of four has the tap (2 x 8 x 8 pixels): filter copy + one launch
    assert len(p["launches"]) == 1 and p["kernels"] == 2 and p["launches"][0]["tiles"] == (1, 1, 1)
    g = cr.Geom(2, 17, 17, 40, 72, 3, 3, stride=(3, 3), pad=(1, 1))
    assert [l["k_iters"] for l in cr.plan("dgrad", 1, 132, g=g)["launches"]] == [2] * 9  # one tap per class and axis
    assert cr.plan("fwd", 0, 132, g=cr.Geom(8, 55, 55, 64, 256, 3, 3, pad=(1, 1)), stats=True)["launches"][0]["grid_x"] == 66
    monkeypatch.setenv("CCV_NNC_SM100_BN", "64")
    assert cr.plan("gemm", 0, 132, M=20000, N=200, K=96)["launches"][0]["tiles"] == (157, 4, 1)


def test_the_matrix_stays_on_its_paths_at_132_sms(monkeypatch):
    for c in CASES:
        with monkeypatch.context() as m:
            m.delenv("CCV_NNC_SM100_BN", raising=False)
            if c.bn:
                m.setenv("CCV_NNC_SM100_BN", c.bn)
            for mode in c.modes:
                if mode != FP32:
                    assert _plan(c, mode, 132)["path"] == c.path, (c, mode)
                    assert c.op == "gemm" or cr.tensor_core_ok(c.op, c.g, _kind(mode), bool(c.kw.get("cview"))), (c, mode)


# ------------------------------------------------------------------------------------------------ GPU
def _plan(case, mode, sms):
    kind = _kind(mode)
    if case.op == "gemm":
        return cr.plan("gemm", kind, sms, M=case.M, N=case.N, K=case.K, bias16=case.bias == 2 and kind != 0)
    return cr.plan(case.op, kind, sms, g=case.g, bias16=case.bias == 2 and kind != 0)


def _bits(a, mode):
    if _kind(mode):
        return cr.to_bits16(np.asarray(a, np.float64), mode)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _upload_bits(t, bits, mode):
    t.upload(bits.view(np.float16) if mode == FP16 else bits if mode == BF16 else bits.view(np.float32))


def _download_bits(t, mode):
    d = t.download()
    return d.view(np.uint16) if _kind(mode) else d.view(np.uint32)


def _values(bits, mode):
    return cr.from_bits16(bits, mode) if _kind(mode) else bits.view(np.float32).astype(np.float64)


class Guarded(object):
    """An output inside a sentinel-filled buffer: a [rows, cols] view of pitch cols + extra at column c0 (view=(extra, c0)), or a
    dense tensor at an offset into a larger allocation."""

    def __init__(self, nnc, shape, mode, old=None, view=None):
        self.mode, self.shape = mode, tuple(shape)
        dt, sent = _dt(mode), SENTINEL[_out_kind(mode)]
        bits_t = np.uint16 if _kind(mode) else np.uint32
        if view:
            rows, cols = shape
            extra, c0 = view
            self.host = np.full((rows + 6, cols + extra), sent, bits_t)
            self.mask = np.zeros(self.host.shape, bool)
            self.mask[3:3 + rows, c0:c0 + cols] = True
            self.base = nnc.gpu_tensor(list(self.host.shape), NHWC, dt)
            self.t = nnc.tensor_view_new(self.base, list(shape), [3, c0] + [0] * 10, [cols + extra, 1] + [0] * 10)
        else:
            n, guard = int(np.prod(shape)), 64
            self.host = np.full((n + 2 * guard,), sent, bits_t)
            self.mask = np.zeros(self.host.shape, bool)
            self.mask[guard:guard + n] = True
            self.base = nnc.gpu_tensor([n + 2 * guard], NHWC, dt)
            self.t = nnc.gpu_tensor(list(shape), NHWC, dt, ptr=self.base.data_ptr + guard * self.host.itemsize)
        if old is not None:
            self.host[self.mask] = _bits(old, _out_kind(mode)).reshape(-1)

    def arm(self):
        _upload_bits(self.base, self.host, _out_kind(self.mode))

    def result(self):
        got = _download_bits(self.base, _out_kind(self.mode))
        changed = (got != self.host) & ~self.mask
        assert not changed.any(), "%d guard elements overwritten, first at %s" % (changed.sum(), np.argwhere(changed)[0])
        return got[self.mask].reshape(self.shape)

    def free(self):
        self.t.free(), self.base.free()


def _input(nnc, a, mode, keep32=False):
    m = FP32 if keep32 else _op_mode(mode)
    t = nnc.gpu_tensor(list(a.shape), NHWC, _dt(m))
    _upload_bits(t, _bits(a, m), m)
    return t


def _command(nnc, case, mode, d, tensors):
    """(cmd, hint, flags, inputs, outputs-before-the-guarded-one, index of the guarded output)"""
    algo = ALGO[mode]
    T = lambda a, keep32=False: tensors.append(_input(nnc, a, mode, keep32)) or tensors[-1]
    flags = abi.CCV_NNC_ACCUMULATE_OUTPUT if case.acc else 0
    if case.op == "gemm":
        tr = lambda t: (0, 1) if t else (0, 0)
        if not case.acc:
            ins = [T(d["a"]), T(d["b"])] + ([T(d["bias"], keep32=case.bias == 1)] if case.bias else [])
            return nnc.CMD_GEMM_FORWARD(tr(case.ta), tr(case.tb), algorithm=algo), None, flags, ins, []
        if not case.ta:  # h[M, N] (+)= g[M, K] w^T with g = a, w = b ([N, K], or [K, N] read through transpose_b)
            return nnc.CMD_GEMM_BACKWARD((0, 0), tr(not case.tb), algorithm=algo), None, flags, [T(d["a"]), None, T(d["b"])], []
        assert not case.tb  # dw[M, N] (+)= a^T g with a = a ([K, M]) and g = b ([K, N])
        return nnc.CMD_GEMM_BACKWARD(algorithm=algo), None, flags, [T(d["b"]), T(d["a"])], [None]
    g = case.g
    hint = nnc.hint(g.st, g.pad, border_end=g.pad_end)
    kw = dict(algorithm=algo) if algo >= 0 else {}
    if case.op == "fwd":
        cv = case.kw.get("cview")
        x = T(d["xbig"])
        if cv:
            Cb = cv[1]
            x = nnc.tensor_view_new(x, [g.N, g.H, g.W, g.C], [0, 0, 0, cv[0]] + [0] * 8, [g.H * g.W * Cb, g.W * Cb, Cb, 1] + [0] * 8)
            tensors.append(x)
        ins = [x, T(d["w"])] + ([T(d["bias"], keep32=case.bias == 1)] if case.bias else [])
        return nnc.CMD_CONVOLUTION_FORWARD(1, g.K, g.R, g.S, g.C, g.dil, **kw), hint, flags, ins, []
    cmd = nnc.CMD_CONVOLUTION_BACKWARD(1, g.K, g.R, g.S, g.C, g.dil, **kw)
    if case.op == "dgrad":
        return cmd, hint, flags, [T(d["gy"]), T(np.zeros((g.N, g.H, g.W, g.C), np.float32)), T(d["w"])], []
    return cmd, hint, flags, [T(d["gy"]), T(d["x"])], [None]


@pytest.fixture(scope="module")
def sms(gpu):
    n = cr.device_sms()
    yield n
    _print_coverage(n)


def _print_coverage(n):
    fams = sorted(set(f for f, _ in COVERAGE) | set(f for f, _ in REQUIRED))
    paths = ["tile", "walk", "split", "ffma"]
    print("\ncontraction paths covered on %d SMs (cases per cell; * = required)" % n)
    print("%-14s" % "family" + "".join("%8s" % p for p in paths))
    for f in fams:
        print("%-14s" % f + "".join("%7d%s" % (COVERAGE.get((f, p), 0), "*" if (f, p) in REQUIRED else " ") for p in paths))
    if CALIBRATION:
        k = max(CALIBRATION, key=CALIBRATION.get)
        print("largest bound ratio |y - y^| / (2^-24 sqrt(K_eff) s): %.3f (%s); C_ACC = %g" % (CALIBRATION[k], k, cr.C_ACC))


def _record(key, ratio):
    CALIBRATION[key] = ratio


@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", PARAMS)
def test_contraction_path(gpu, sms, monkeypatch, case, mode):
    nnc = gpu
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    if case.bn:
        monkeypatch.setenv("CCV_NNC_SM100_BN", case.bn)
    d = operands(case, mode)
    p = None if mode == FP32 else _plan(case, mode, sms)
    if p is not None:
        assert p["path"] == case.path, "%s: the planner puts this case on the %s path on %d SMs" % (case, p["path"], sms)
    tensors = []
    out = Guarded(nnc, d["out_shape"], mode, d.get("old"), case.view)
    try:
        cmd, hint, flags, ins, lead = _command(nnc, case, mode, d, tensors)
        outs = lead + [out.t]
        results = []
        for _ in range(2):
            out.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, hint, flags, ins, outs)
            assert st == 0, "%s: status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
            if p is not None:
                assert nnc.launch_count() - l0 == p["kernels"], "%s: %d launches, planned %d" % (case, nnc.launch_count() - l0, p["kernels"])
            results.append(out.result())
        assert np.array_equal(results[0], results[1]), "%s: two runs differ" % case
    finally:
        for t in reversed(tensors):
            t.free()
        out.free()
    y, s, keff = oracle(case, _seen_key(mode))
    ratio = cr.check(_values(results[0], _out_kind(mode)), y, s, keff, mode, _out_kind(mode), "%s %s" % (case, mode))
    _record("%s %s" % (case, mode), ratio)
    cell = (case.fam(mode), case.path if p else "ffma")
    COVERAGE[cell] = COVERAGE.get(cell, 0) + 1
    RAN.add((repr(case), mode))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", STATS_MODES)
@pytest.mark.parametrize("N,H,C,K,R,offset", STATS)
def test_statistics_epilogue(gpu, sms, monkeypatch, mode, N, H, C, K, R, offset):
    """Convolution -> training batch norm, fused by the graph: the saved mean and inv_std must be the float64 statistics of the y
    the same kernel stored (after its 16-bit rounding) up to summation error, and y itself must meet its bound."""
    nnc = gpu
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    pad = R // 2
    g = cr.Geom(N, H, H, C, K, R, R, pad=(pad, pad))
    case = Case("fwd", "walk", modes=[mode], bias=1, N=N, H=H, W=H, C=C, K=K, R=R, S=R, pad=(pad, pad))
    d = operands(case, mode)
    bias = (d["bias"] + np.float32(offset)).astype(np.float32)
    p = cr.plan("fwd", _kind(mode), sms, g=g, stats=True)
    l = p["launches"][0]
    assert p["path"] == "walk", (case, p)
    eps = 1e-4
    stream = nnc.Stream(0)
    f32 = lambda a: _input(nnc, a, FP32, keep32=True)
    tx, tw, tb = _input(nnc, d["x"], mode), _input(nnc, d["w"], mode), f32(bias)
    tscale, tbias = f32(np.ones((1, 1, 1, K), np.float32)), f32(np.zeros((1, 1, 1, K), np.float32))
    tmean, tvar = f32(np.zeros((1, 1, 1, K), np.float32)), f32(np.ones((1, 1, 1, K), np.float32))
    ty, tz = (nnc.gpu_tensor([N, g.P, g.Q, K], NHWC, _dt(mode)) for _ in range(2))
    tsm, tsis = (nnc.gpu_tensor([1, 1, 1, K]) for _ in range(2))
    graph = nnc.Graph()
    graph.exec_new(nnc.CMD_CONVOLUTION_FORWARD(1, K, R, R, C, algorithm=ALGO[mode]), nnc.hint((1, 1), (pad, pad)), 0, [tx, tw, tb], [ty])
    graph.exec_new(nnc.CMD_BATCH_NORM_FORWARD(eps, 0, 0.9), None, 0, [ty, tscale, tbias, tmean, tvar], [tz, tmean, tvar, tsm, tsis])
    graph.fuse()
    try:
        assert [k for _, k, _, _ in graph.nodes()] == [6, 7]
        assert graph.run(stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        stream.wait()
        rows = abi.Tensor.from_address(graph.nodes()[0][3][1]).sig
        assert rows == 4 * l["grid_x"], "statistics rows %d, planned %d CTAs per column" % (rows, l["grid_x"])
        yb = _download_bits(ty, mode)
        sm, sis = tsm.download().reshape(-1).astype(np.float64), tsis.download().reshape(-1).astype(np.float64)
    finally:
        for t in (tx, tw, tb, tscale, tbias, tmean, tvar, ty, tz, tsm, tsis, graph, stream):
            t.free()
    y = _values(yb, _out_kind(mode)).reshape(-1, K)
    ref, s, keff = oracle(case, _seen_key(mode))
    ref, s = ref + (bias - d["bias"]).astype(np.float64), s + np.abs(bias - d["bias"]).astype(np.float64)
    _record("stats %s %s" % (case, mode), cr.check(y.reshape(ref.shape), ref, s, keff, mode, _out_kind(mode), "stats conv output"))
    mean, var = y.mean(0), y.var(0)
    std = np.sqrt(var)
    tol = 1e-6 * (np.abs(mean) + std)
    assert (np.abs(sm - mean) <= tol).all(), "saved mean off by %.3g of (|mean| + std)" % (np.abs(sm - mean) / (np.abs(mean) + std)).max()
    want = 1.0 / np.sqrt(var + eps)
    # inv_std error from a variance error dv: |d inv_std| = dv / (2 (var + eps)^1.5), dv ~ 2 std * tol
    assert (np.abs(sis - want) <= 2 * std * tol / (var + eps) ** 1.5).all(), "saved inv_std off by %.3g relative" % (np.abs(sis - want) / want).max()
    COVERAGE[("stats", "walk")] = COVERAGE.get(("stats", "walk"), 0) + 1
    RAN.add(("stats " + repr(case), mode))


def _tf32_rounding_probe():
    """The TF32 GEMM case with K_eff <= 1024 (a 1000 x 40 x 136 product): 0 when the bound holds, 3 when it does not."""
    from ccv_b200 import nnc
    nnc.init()
    case = Case("gemm", "tile", modes=[TF32], M=1000, N=40, K=136, ta=1, tb=0)
    d = operands(case, TF32)
    tensors = []
    out = Guarded(nnc, d["out_shape"], TF32)
    cmd, hint, flags, ins, lead = _command(nnc, case, TF32, d, tensors)
    out.arm()
    assert nnc.cmd_exec(cmd, hint, flags, ins, lead + [out.t]) == 0
    y = _values(out.result(), FP32)
    for t in tensors:
        t.free()
    out.free()
    ref, s, keff = oracle(case, "tf32")
    return 0 if cr.admits(y, ref, s, keff, TF32, FP32).all() else 3


@pytest.mark.gpu
def test_tma_rounds_fp32_operands_to_nearest_tf32(gpu):
    """With CU_TENSOR_MAP_DATA_TYPE_FLOAT32 operand maps (CCV_NNC_SM100_TMA_DTYPE=7, read once per process, hence the subprocess)
    the tensor core truncates each operand's low 13 bits, which the round-to-nearest oracle must reject; with the default TFLOAT32
    maps the same product meets the bound."""
    assert _tf32_rounding_probe() == 0
    env = dict(os.environ, CCV_NNC_SM100_TMA_DTYPE="7")
    code = "import sys; from tests.test_parity_contract_paths import _tf32_rounding_probe as p; sys.exit(p())"
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 3, "exit %d (3 = bound violated); stderr: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.gpu
def test_every_required_path_was_covered(gpu, sms):
    """Runs last: every (family, path) cell of the matrix was exercised by at least one case on this device."""
    if len(RAN) < len(PARAMS) + len(STATS) * len(STATS_MODES):
        pytest.skip("only part of the matrix ran")
    missing = [c for c in REQUIRED if not COVERAGE.get(c)]
    assert not missing, missing
