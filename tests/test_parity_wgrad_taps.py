"""The convolution weight gradient with its filter taps laid along the output tile's columns, against the float64 oracle of
tests/contract_ref.py at rounding-level bounds, and bit for bit against the per-tap grid it replaces.

conv_wgrad_any (ccv_b200/csrc/sm100_contract.cu) can run a non-pointwise weight gradient as one GEMM
dW[K, R*S*C] = grad^T [K, NPQ] x im2col(x) [NPQ, R*S*C]: output column n = tap * C + c, and each 32-channel (fp32) or 64-channel
(16-bit) B box of a tile loads the tap its columns belong to.  It does so when C is a multiple of the box and the column tiles need
fewer rounds of CTAs over the SMs than the per-tap grid (one launch, the filter tap on gridDim.z); otherwise it runs the per-tap
grid.  Both take the split-K factor the per-tap grid is planned with (tests/contract_ref.plan), so every dW element is the same sum
over the same pixel ranges, combined in the same order: the bits do not depend on the layout.  local_plan() restates the choice.

GPU: every case meets the bound in TF32, 3xTF32, bf16 and fp16, inside a NaN-filled guard buffer, with the same bits from a second
run, the planned launch count, and on 132 SMs the bits of the build before the column layout (SHA-256 digests in
tests/golden/wgrad_taps_digests.json; `python -m tests.test_parity_wgrad_taps --write-digests FILE` writes them from the build at
hand).

CPU: the plan on hand-worked shapes and on every weight-gradient case of tests/test_parity_contract_paths.py, and bounds that reject
a result whose box was loaded at its neighbouring tap."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from tests import contract_ref as cr
from tests.contract_ref import BF16, FP16, FP32, TF32, X3
from tests.test_parity_contract_paths import CASES as PATH_CASES
from tests.test_parity_contract_paths import Case, Guarded, _command, _kind, _out_kind, _seen_key, _values, operands, oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_taps_digests.json")
MODES = [TF32, X3, BF16, FP16]
DEFECT_MODES = [TF32, BF16, FP16]


def W(path, N, H, C, K, R, acc=False, **kw):
    return Case("wgrad", path, modes=MODES, acc=acc, N=N, H=H, W=kw.pop("W", H), C=C, K=K, R=R, S=kw.pop("S", R), **kw)


# path = the fp32 plan at 132 SMs ("split" or "tile"); which layout each kind takes is asserted in test_cases_take_their_layouts
CASES = [
    W("split", 8, 44, 32, 32, 3, pad=(1, 1)),                                   # the stem's 32 -> 32: 288 columns, a ragged third tile
    W("split", 8, 44, 32, 64, 3, acc=True, pad=(1, 1)),                         # 32 -> 64, accumulating
    W("tile", 1, 16, 32, 2048, 3, acc=True, pad=(1, 1)),                        # unsplit (8 k-iterations): 16 x 3 column tiles
    W("split", 8, 88, 32, 32, 3, stride=(2, 2), pad=(1, 1)),                    # stride 2
    W("split", 8, 44, 32, 32, 3, pad=(2, 2), dil=(2, 2)),                       # dilation 2
    W("split", 8, 44, 32, 64, 3, pad=(1, 0), pad_end=(0, 1)),                   # asymmetric padding
    W("split", 8, 26, 32, 32, 5, pad=(2, 2)),                                   # 5 x 5: 800 columns
    W("split", 10, 32, 32, 64, 7, stride=(2, 2), pad=(3, 3)),                   # 7 x 7 / 2: 1568 columns
    W("split", 8, 48, 64, 64, 3, acc=True, pad=(1, 1)),                         # 64 -> 64: columns in 16-bit, the per-tap grid in fp32
    W("split", 4, 28, 64, 64, 3, pad=(1, 1)),                                   # 64 -> 64 with few splits: the per-tap grid
    W("split", 4, 28, 128, 128, 3, acc=True, pad=(1, 1)),                       # 128 -> 128: the per-tap grid
    W("split", 8, 28, 40, 16, 3, pad=(1, 1)),                                   # C = 40: two taps would share a box, the per-tap grid
    W("tile", 2, 9, 40, 48, 3, acc=True, W=11, stride=(2, 2), pad=(1, 1)),      # C = 40, unsplit, accumulating
]
PARAMS = [pytest.param(c, m, id="%s-%s" % (c, m)) for c in CASES for m in c.modes]


# ------------------------------------------------------------------------------------------------ the plan
def local_plan(g, kind, sms):
    """conv_wgrad_any's launch: {"tap_cols", "bn", "tiles": (m, n, taps), "splits", "kernels", "path"}"""
    grid = cr.plan("wgrad", kind, sms, g=g)  # the per-tap grid (or the pointwise GEMM) and its split factor
    s = grid["launches"][0]["splits"]
    bk = 32 if kind == 0 else 64
    tm, rsc = -(-g.K // cr.BLOCK_M), g.R * g.S * g.C
    col_bn = cr.pick_bn(rsc)
    rounds = lambda ctas: -(-ctas // sms)
    grid_ctas = tm * -(-g.C // cr.pick_bn(g.C)) * g.R * g.S * s
    tap_cols = not cr.pointwise(g) and g.C % bk == 0 and rounds(tm * -(-rsc // col_bn) * s) < rounds(grid_ctas)
    if not tap_cols:
        l = grid["launches"][0]
        return dict(tap_cols=False, bn=l["bn"], tiles=l["tiles"], splits=s, kernels=grid["kernels"], path=grid["path"])
    return dict(tap_cols=True, bn=col_bn, tiles=(tm, -(-rsc // col_bn), 1), splits=s, kernels=1 + (s > 1), path="split" if s > 1 else "tile")


def test_plan_on_hand_worked_shapes(monkeypatch):
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    stem = cr.Geom(256, 112, 112, 32, 32, 3, 3, pad=(1, 1))  # 3.2 M pixels: 100 352 fp32 k-iterations
    p = local_plan(stem, 0, 132)  # per-tap grid: 9 tiles x 29 splits = 261 CTAs, two rounds; columns: 3 x 29 = 87, one round
    assert p["tap_cols"] and p["tiles"] == (1, 3, 1) and p["splits"] == 29 and p["kernels"] == 2
    assert not local_plan(stem, 1, 132)["tap_cols"]  # 16-bit: 32 channels are half a 64-channel box
    layer1 = cr.Geom(256, 56, 56, 64, 64, 3, 3, pad=(1, 1))  # 9 x 29 = 261 CTAs against 5 x 29 = 145: two rounds either way
    assert not local_plan(layer1, 0, 132)["tap_cols"] and not local_plan(layer1, 2, 132)["tap_cols"]
    p = local_plan(cr.Geom(8, 48, 48, 64, 64, 3, 3, pad=(1, 1)), 1, 132)  # 16-bit, 18 splits: 162 CTAs against 90
    assert p["tap_cols"] and p["tiles"] == (1, 5, 1) and p["splits"] == 18
    p = local_plan(cr.Geom(2, 7, 7, 1024, 1024, 3, 3, pad=(1, 1)), 0, 132)  # C fills whole tiles: as many CTAs either way
    assert not p["tap_cols"] and p["tiles"] == (8, 8, 9) and p["splits"] == 1 and p["path"] == "tile"
    p = local_plan(cr.Geom(16, 29, 29, 40, 48, 3, 3, stride=(2, 2), pad_end=(1, 1)), 0, 132)
    assert not p["tap_cols"] and p["tiles"] == (1, 1, 9)


def test_contract_path_cases_keep_their_path_and_launches(monkeypatch):
    """every weight-gradient case of the contraction path matrix keeps contract_ref.plan's path and launch count"""
    for c in PATH_CASES:
        if c.op != "wgrad":
            continue
        with monkeypatch.context() as m:
            m.delenv("CCV_NNC_SM100_BN", raising=False)
            if c.bn:
                m.setenv("CCV_NNC_SM100_BN", c.bn)
            for mode in c.modes:
                if mode == FP32:
                    continue
                old, new = cr.plan("wgrad", _kind(mode), 132, g=c.g), local_plan(c.g, _kind(mode), 132)
                assert new["path"] == old["path"] == c.path and new["kernels"] == old["kernels"], (c, mode, old, new)


def test_cases_take_their_layouts_at_132_sms(monkeypatch):
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    for c in CASES:
        assert local_plan(c.g, 0, 132)["path"] == c.path, c
        assert cr.tensor_core_ok("wgrad", c.g, 0) and cr.tensor_core_ok("wgrad", c.g, 1), c
    fp32 = [local_plan(c.g, 0, 132)["tap_cols"] for c in CASES]
    half = [local_plan(c.g, 1, 132)["tap_cols"] for c in CASES]
    assert fp32 == [True] * 8 + [False] * 5 and half == [False] * 8 + [True] + [False] * 4, (fp32, half)
    plans = [local_plan(c.g, 0, 132) for c in CASES[:8]]
    assert any(p["splits"] == 1 for p in plans) and any(p["splits"] > 1 for p in plans)


# ------------------------------------------------------------------------------------------------ CPU: the bound sees a box at the wrong tap
@pytest.mark.parametrize("case,mode", [pytest.param(c, m, id="%s-%s" % (c, m)) for c in CASES for m in DEFECT_MODES])
def test_bounds_reject_a_box_at_its_neighbouring_tap(case, mode):
    out = _out_kind(mode)
    y, s, keff = oracle(case, _seen_key(mode))
    fin = (lambda v: cr.rne16(v, out)) if out != FP32 else (lambda v: np.asarray(v, np.float32).astype(np.float64))
    cr.check(fin(y), y, s, keff, mode, out, "correct result")
    g, bk = case.g, 32 if _kind(mode) == 0 else 64
    taps = g.R * g.S
    old = operands(case, mode).get("old")
    base = y - (0.0 if old is None else np.asarray(old, np.float64))  # the product alone, per tap
    for t in (0, taps // 2, taps - 2):
        bad = y.reshape(g.K, taps, g.C).copy()
        prod = base.reshape(g.K, taps, g.C)
        w = min(bk, g.C)
        bad[:, t, :w] += prod[:, t + 1, :w] - prod[:, t, :w]  # the first box of tap t loaded at tap t + 1
        assert not cr.admits(fin(bad.reshape(y.shape)), y, s, keff, mode, out).all(), "%s %s: a box loaded at the next tap passes (tap %d)" % (case, mode, t)


# ------------------------------------------------------------------------------------------------ GPU
def _run(nnc, case, mode):
    """(output bits, launches per call) of two guarded runs, checked to agree"""
    d = operands(case, mode)
    tensors = []
    out = Guarded(nnc, d["out_shape"], mode, d.get("old"))
    try:
        cmd, hint, flags, ins, lead = _command(nnc, case, mode, d, tensors)
        results, launches = [], []
        for _ in range(2):
            out.arm()
            l0 = nnc.launch_count()
            st = nnc.cmd_exec(cmd, hint, flags, ins, lead + [out.t])
            assert st == 0, "%s: status %d, %s" % (case, st, nnc.lib().ccv_nnc_sm100_last_error())
            launches.append(nnc.launch_count() - l0)
            results.append(out.result())
        assert np.array_equal(results[0], results[1]), "%s %s: two runs differ" % (case, mode)
        assert launches[0] == launches[1]
    finally:
        for t in reversed(tensors):
            t.free()
        out.free()
    return results[0], launches[0]


def _digest(bits):
    return hashlib.sha256(np.ascontiguousarray(bits).tobytes()).hexdigest()


@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", PARAMS)
def test_wgrad_taps(gpu, monkeypatch, case, mode):
    nnc = gpu
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    sms = cr.device_sms()
    p = local_plan(case.g, _kind(mode), sms)
    bits, launches = _run(nnc, case, mode)
    assert launches == p["kernels"], "%s %s: %d launches, planned %d" % (case, mode, launches, p["kernels"])
    assert launches == cr.plan("wgrad", _kind(mode), sms, g=case.g)["kernels"]
    y, s, keff = oracle(case, _seen_key(mode))
    cr.check(_values(bits, _out_kind(mode)), y, s, keff, mode, _out_kind(mode), "%s %s" % (case, mode))
    golden = json.load(open(GOLDEN))
    if sms == golden["sms"]:  # the split factor, and so the bits, depend on the SM count
        want = golden["digests"].get("%s-%s" % (case, mode))
        assert want is not None and _digest(bits) == want, "%s %s: the bits differ from the per-tap grid's" % (case, mode)


def _write_digests(path):
    from ccv_b200 import nnc
    nnc.init()
    digests = dict(("%s-%s" % (case, mode), _digest(_run(nnc, case, mode)[0])) for case in CASES for mode in case.modes)
    with open(path, "w") as f:
        json.dump(dict(sms=cr.device_sms(), digests=digests), f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--write-digests":
        _write_digests(sys.argv[2])
    else:
        raise SystemExit("usage: python -m tests.test_parity_wgrad_taps --write-digests FILE")
