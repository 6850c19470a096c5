"""The TF32 weight gradient of narrow layers with swapped operands, against the float64 oracle of tests/contract_ref.py at
rounding-level bounds, and bit for bit against the build whose TF32 weight gradient put the output channels along the MMA rows.

conv_wgrad_any (ccv_b200/csrc/sm100_contract.cu) computes dW^T[R*S*C, K] = im2col(x)^T [R*S*C, NPQ] x grad [NPQ, K] when the
convolution is not pointwise, C is a multiple of 32 and K <= 64: the filter taps run along the MMA rows, K along one 32- or
64-column tile, and the epilogue stores the tile transposed into dW.  It keeps the split-K factor of the per-tap grid
(tests/contract_ref.plan), so every dW element is the same sum over the same pixel ranges, combined in the same order; the tile
height is 128 rows unless 256 needs fewer rounds of CTAs over the SMs.  swap_plan() restates the choice.

GPU: every case meets the bound inside a NaN-filled guard buffer, gives the same bits from a second run, advances the launch count
as planned, and on 132 SMs gives the bits of the earlier build (SHA-256 digests in tests/golden/wgrad_swap_digests.json;
`python -m tests.test_parity_wgrad_swap --write-digests FILE` writes them from the build at hand)."""
import json
import os
import sys

import pytest

from tests import contract_ref as cr
from tests.contract_ref import TF32
from tests.test_parity_contract_paths import Case, _out_kind, _seen_key, _values, oracle
from tests.test_parity_wgrad_rs import CASES as RS_CASES
from tests.test_parity_wgrad_taps import CASES as TAPS_CASES
from tests.test_parity_wgrad_taps import _digest, _run

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgrad_swap_digests.json")


def swap_plan(g, sms):
    """the TF32 launch of conv_wgrad_any when it swaps the operands, else None: {"bm", "bn", "ctas", "splits", "kernels", "path"}"""
    if cr.pointwise(g) or g.C % 32 or g.K > 64:
        return None
    grid = cr.plan("wgrad", 0, sms, g=g)
    s, rsc = grid["launches"][0]["splits"], g.R * g.S * g.C
    rounds = lambda ctas: -(-ctas // sms)
    bm = 256 if rounds(-(-rsc // 256) * s) < rounds(-(-rsc // 128) * s) else 128
    return dict(bm=bm, bn=32 if g.K <= 32 else 64, ctas=-(-rsc // bm) * s, splits=s, kernels=grid["kernels"], path=grid["path"])


def X(bm, bn, N, H, C, K, R, acc=False, **kw):
    c = Case("wgrad", "split", modes=[TF32], acc=acc, N=N, H=H, W=kw.pop("W", H), C=C, K=K, R=R, S=kw.pop("S", R), **kw)
    c.path = cr.plan("wgrad", 0, 132, g=c.g)["path"]
    c.want = (bm, bn)
    return c


# ResNet-50's narrow 3 x 3 layers at a short batch, and the shapes around them: (tile height, width) at 132 SMs
CASES = [
    X(128, 32, 8, 112, 32, 32, 3, pad=(1, 1)),                     # the stem's 32 -> 32
    X(128, 32, 8, 112, 32, 32, 3, acc=True, pad=(1, 1)),           # accumulating
    X(128, 64, 8, 112, 32, 64, 3, pad=(1, 1)),                     # the stem's 32 -> 64
    X(256, 64, 16, 56, 64, 64, 3, pad=(1, 1)),                     # layer1's 64 -> 64: 576 rows, a half-empty third 128-row tile
    X(256, 64, 16, 56, 64, 64, 3, acc=True, pad=(1, 1)),           # accumulating
    X(256, 32, 8, 56, 64, 32, 3, pad=(1, 1)),                      # 256-row tiles 32 wide
    X(128, 64, 8, 56, 64, 48, 3, stride=(2, 2), pad=(1, 1)),       # ragged K = 48, stride 2
    X(128, 32, 1, 8, 32, 16, 3, acc=True, pad=(1, 1)),             # unsplit (2 k-iterations), accumulating, K = 16
    X(128, 64, 2, 13, 64, 64, 3, pad=(1, 1)),                      # unsplit, N*P*Q % 32 = 18
]


# ------------------------------------------------------------------------------------------------ the plan
def test_plan_on_resnet50_narrow_layers():
    stem = cr.Geom(256, 112, 112, 32, 32, 3, 3, pad=(1, 1))  # 288 rows: 3 x 29 = 87 CTAs at 128 rows and 58 at 256, one round each
    assert swap_plan(stem, 132) == dict(bm=128, bn=32, ctas=87, splits=29, kernels=2, path="split")
    stem2 = cr.Geom(256, 112, 112, 32, 64, 3, 3, pad=(1, 1))
    assert swap_plan(stem2, 132) == dict(bm=128, bn=64, ctas=87, splits=29, kernels=2, path="split")
    layer1 = cr.Geom(256, 56, 56, 64, 64, 3, 3, pad=(1, 1))  # 576 rows: 5 x 29 = 145 CTAs (two rounds) at 128, 3 x 29 = 87 at 256
    assert swap_plan(layer1, 132) == dict(bm=256, bn=64, ctas=87, splits=29, kernels=2, path="split")
    # every other ResNet-50 convolution keeps its layout: K >= 128, pointwise, or the 3-channel stem (explicit im2col)
    for g in (cr.Geom(256, 56, 56, 64, 64, 1, 1), cr.Geom(256, 56, 56, 256, 64, 1, 1), cr.Geom(256, 28, 28, 128, 128, 3, 3, pad=(1, 1)),
              cr.Geom(256, 14, 14, 256, 256, 3, 3, pad=(1, 1)), cr.Geom(256, 7, 7, 512, 512, 3, 3, pad=(1, 1))):
        assert swap_plan(g, 132) is None, g


def test_existing_wgrad_cases_that_take_the_swap_at_132_sms():
    taps = [swap_plan(c.g, 132) for c in TAPS_CASES]
    assert [p and (p["bm"], p["bn"]) for p in taps] == [(128, 32), (128, 64), None, (128, 32), (128, 32), (128, 64), (128, 32), (128, 64), (256, 64), (128, 64), None, None, None]
    rs = [swap_plan(c.g, 132) for c in RS_CASES]
    assert [p and (p["bm"], p["bn"]) for p in rs] == [None] * 9 + [(128, 64), (128, 32), (256, 64), None, (256, 64), (256, 64), (256, 64)]
    for c in TAPS_CASES + RS_CASES:  # the launch count stays the per-tap grid's
        p = swap_plan(c.g, 132)
        if p:
            assert p["kernels"] == cr.plan("wgrad", 0, 132, g=c.g)["kernels"] == 1 + (p["splits"] > 1), c


def test_cases_take_their_tile_at_132_sms():
    for c in CASES:
        p = swap_plan(c.g, 132)
        assert p is not None and (p["bm"], p["bn"]) == c.want, (c, p)
        assert cr.tensor_core_ok("wgrad", c.g, 0), c
    plans = [swap_plan(c.g, 132) for c in CASES]
    assert any(p["splits"] == 1 for p in plans) and any(p["splits"] > 1 for p in plans)
    assert any(c.acc and p["splits"] == 1 for c, p in zip(CASES, plans)) and any(c.acc and p["splits"] > 1 for c, p in zip(CASES, plans))
    assert any((c.g.N * c.g.P * c.g.Q) % 32 for c in CASES)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", [pytest.param(c, id=repr(c)) for c in CASES])
def test_wgrad_swap(gpu, monkeypatch, case):
    nnc, mode = gpu, TF32
    monkeypatch.delenv("CCV_NNC_SM100_BN", raising=False)
    sms = cr.device_sms()
    bits, launches = _run(nnc, case, mode)
    assert launches == swap_plan(case.g, sms)["kernels"], "%s: %d launches" % (case, launches)
    y, s, keff = oracle(case, _seen_key(mode))
    cr.check(_values(bits, _out_kind(mode)), y, s, keff, mode, _out_kind(mode), repr(case))
    golden = json.load(open(GOLDEN))
    if sms == golden["sms"]:  # the split factor, and so the bits, depend on the SM count
        want = golden["digests"].get(repr(case))
        assert want is not None and _digest(bits) == want, "%s: the bits differ from the unswapped layout's" % case


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
        raise SystemExit("usage: python -m tests.test_parity_wgrad_swap --write-digests FILE")
