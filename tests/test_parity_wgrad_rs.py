"""The TF32 convolution weight gradient with A = grad^T read from the staged tile into wgmma registers and output tiles 64, 128 or
256 columns wide, against the float64 oracle of tests/contract_ref.py at rounding-level bounds, and bit for bit against the build
whose TF32 weight gradient transposed both operands in shared memory and never ran tiles wider than 128.

conv_wgrad_any (ccv_b200/csrc/sm100_contract.cu) keeps the split-K factor the per-tap grid is planned with (tests/contract_ref.plan)
and picks the TF32 tile width and layout (the per-tap grid, or the filter taps along the columns) by the fewest rounds of CTAs
over the SMs, then the narrower tile, then the fewer CTAs; rs_plan() restates the rule.  Every dW element stays the same sum over
the same pixel ranges, combined in the same order, whatever the width, the layout and the operand path.

GPU: every case meets the bound inside a NaN-filled guard buffer, gives the same bits from a second run, advances the launch count
as planned, and on 132 SMs gives the bits of the earlier build (SHA-256 digests in tests/golden/wgrad_rs_digests.json;
`python -m tests.test_parity_wgrad_rs --write-digests FILE` writes them from the build at hand)."""
import json
import os
import sys

import pytest

from tests import contract_ref as cr
from tests.contract_ref import TF32
from tests.test_parity_contract_paths import Case, _kind, _out_kind, _seen_key, _values, oracle
from tests.test_parity_wgrad_taps import _digest, _run

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_rs_digests.json")


def rs_plan(g, sms):
    """the TF32 launch of conv_wgrad_any: {"bn", "layout" (1x1 | grid | columns), "ctas", "rounds", "splits", "kernels", "path"}"""
    grid = cr.plan("wgrad", 0, sms, g=g)
    s = grid["launches"][0]["splits"]
    tm, rsc, pw = -(-g.K // cr.BLOCK_M), g.R * g.S * g.C, cr.pointwise(g)
    rounds = lambda ctas: -(-ctas // sms)
    best = None
    for w in (64, 128, 256):
        for cols in (False, True):
            if cols and (pw or g.C % 32):
                continue
            ctas = tm * (-(-rsc // w) if cols or pw else -(-g.C // w) * g.R * g.S) * s
            if best is None or rounds(ctas) < best["rounds"] or (rounds(ctas) == best["rounds"] and w == best["bn"] and ctas < best["ctas"]):
                best = dict(bn=w, layout="1x1" if pw else ("columns" if cols else "grid"), ctas=ctas, rounds=rounds(ctas))
    return dict(best, splits=s, kernels=grid["kernels"], path=grid["path"])


def T(layout, bn, N, H, C, K, R, acc=False, **kw):
    c = Case("wgrad", "split", modes=[TF32], acc=acc, N=N, H=H, W=kw.pop("W", H), C=C, K=K, R=R, S=kw.pop("S", R), **kw)
    c.path = cr.plan("wgrad", 0, 132, g=c.g)["path"]
    c.want = (layout, bn)
    return c


# (layout, width) each case takes at 132 SMs; N*P*Q % 32 != 0 where marked
CASES = [
    T("1x1", 64, 8, 28, 64, 128, 1),                                         # C = 64: every width is one column tile
    T("1x1", 64, 1, 8, 256, 1024, 1, acc=True),                              # unsplit, accumulating
    T("1x1", 128, 4, 26, 320, 2048, 1),                                      # N*P*Q % 32 = 16; 2.5 column tiles
    T("1x1", 256, 2, 64, 256, 1024, 1, acc=True),                            # 512 -> 256 -> 128 CTAs: one round at 256
    T("grid", 64, 4, 28, 40, 16, 3, pad=(1, 1)),                             # C = 40: two taps would share a box
    T("grid", 64, 8, 28, 40, 200, 3, acc=True, pad=(1, 1)),                  # C = 40, ragged K = 200
    T("grid", 128, 19, 28, 128, 128, 3, pad=(1, 1)),                         # N*P*Q % 32 = 16
    T("grid", 256, 20, 14, 256, 256, 3, acc=True, pad=(1, 1)),               # ResNet-50's 3 x 3 256 -> 256, 7 splits
    T("grid", 256, 2, 7, 1024, 1024, 3, pad=(1, 1)),                         # unsplit, N*P*Q = 98
    T("columns", 64, 2, 15, 32, 48, 3, acc=True, stride=(2, 2), pad=(1, 1)), # unsplit, K = 48
    T("columns", 128, 8, 44, 32, 32, 3, pad=(1, 1)),                         # the stem's 32 -> 32
    T("columns", 256, 8, 56, 64, 64, 3, acc=True, pad=(1, 1)),               # layer1's 3 x 3 64 -> 64: 576 columns, a ragged third tile
    T("columns", 256, 8, 56, 64, 200, 3, pad=(1, 1)),                        # ragged K = 200
    T("columns", 256, 8, 112, 64, 64, 3, stride=(2, 2), pad=(1, 1)),         # stride 2
    T("columns", 256, 8, 56, 64, 64, 3, pad=(2, 2), dil=(2, 2)),             # dilation 2
    T("columns", 256, 8, 56, 64, 48, 3, pad=(1, 0), pad_end=(0, 1)),         # asymmetric padding, N*P*Q % 32 = 8
]


# ------------------------------------------------------------------------------------------------ the plan
def test_plan_on_hand_worked_resnet50_shapes():
    layer1 = cr.Geom(256, 56, 56, 64, 64, 3, 3, pad=(1, 1))  # per-tap grid 9 x 29 = 261 CTAs (two rounds); columns at 256: 3 x 29
    p = rs_plan(layer1, 132)
    assert (p["layout"], p["bn"], p["ctas"], p["splits"], p["rounds"]) == ("columns", 256, 87, 29, 1), p
    for k in (32, 64):  # the stem's 32 -> 32 and 32 -> 64: 87 CTAs at 128 and 58 at 256 are both one round, so the narrower
        p = rs_plan(cr.Geom(256, 112, 112, 32, k, 3, 3, pad=(1, 1)), 132)
        assert (p["layout"], p["bn"], p["ctas"]) == ("columns", 128, 87), p
    for k, h in ((256, 56), (64, 56)):  # the C = 64 1 x 1 layers: one column tile at every width
        p = rs_plan(cr.Geom(256, h, h, 64, k, 1, 1), 132)
        assert (p["layout"], p["bn"]) == ("1x1", 64), p
    p = rs_plan(cr.Geom(256, 14, 14, 256, 256, 3, 3, pad=(1, 1)), 132)  # 252 CTAs in two rounds at 128
    assert p["bn"] == 256 and p["ctas"] == 126 and p["rounds"] == 1 and p["splits"] == 7, p
    p = rs_plan(cr.Geom(256, 7, 7, 512, 512, 3, 3, pad=(1, 1)), 132)  # 5 rounds at 128
    assert p["bn"] == 256 and p["rounds"] == 3, p


def test_cases_take_their_width_and_layout_at_132_sms():
    for c in CASES:
        p = rs_plan(c.g, 132)
        assert (p["layout"], p["bn"]) == c.want, (c, p)
        assert cr.tensor_core_ok("wgrad", c.g, 0), c
    assert any(rs_plan(c.g, 132)["splits"] == 1 for c in CASES) and any(rs_plan(c.g, 132)["splits"] > 1 for c in CASES)
    assert any(c.acc for c in CASES) and any((c.g.N * c.g.P * c.g.Q) % 32 for c in CASES)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", [pytest.param(c, id=repr(c)) for c in CASES])
def test_wgrad_rs(gpu, monkeypatch, case):
    nnc, mode = gpu, TF32
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    sms = cr.device_sms()
    bits, launches = _run(nnc, case, mode)
    assert launches == rs_plan(case.g, sms)["kernels"], "%s: %d launches" % (case, launches)
    y, s, keff = oracle(case, _seen_key(mode))
    cr.check(_values(bits, _out_kind(mode)), y, s, keff, mode, _out_kind(mode), repr(case))
    golden = json.load(open(GOLDEN))
    if sms == golden["sms"]:  # the split factor, and so the bits, depend on the SM count
        want = golden["digests"].get(repr(case))
        assert want is not None and _digest(bits) == want, "%s: the bits differ from the shared-memory A path's" % case


def _write_digests(path):
    from ccv_b200 import nnc
    nnc.init()
    digests = dict((repr(c), _digest(_run(nnc, c, TF32)[0])) for c in CASES)
    with open(path, "w") as f:
        json.dump(dict(sms=cr.device_sms(), digests=digests), f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--write-digests":
        _write_digests(sys.argv[2])
    else:
        raise SystemExit("usage: python -m tests.test_parity_wgrad_rs --write-digests FILE")
