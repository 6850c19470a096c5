"""Writes tests/golden/cpuref_lssc.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on COMPRESSION_LSSC
forward and backward, so that tests/test_lssc_cpu.py pins the restatement of tests/lssc_ref.py to CPU_REF without the reference
present.  CPU_REF registers NCHW only; the NHWC form is defined as the NCHW transpose and needs no fixture of its own.

Forward cases (fp16 bits in, fp16 bits out):
  - every H and W in {1, 3, 4, 5, 7, 13, 14}, as [2, 3, H, W] and as [3, H, W], plus one [1, 2, 113, 114];
  - "special": one 4x4 block per row of the SPECIAL table below (all-equal, subnormal ranges below 1e-6, +-0 ties, NaN in cell 0 and
    elsewhere, +-Inf, +-65504), in a [K, 4, 4] tensor, and the same cells cut off at 3 x 3 ([K, 3, 3]) so that padding sees them too.
Backward cases (compressed bits in, fp16 bits out):
  - the forward outputs above, decoded;
  - "levels": random (min, max) pairs and random codes, many of which have a middle level whose truncation and round-to-nearest
    differ;
  - "nan_levels": (min, max) pairs with NaN (quiet, signalling, negative), +-Inf and finite members, every code 0-3, so that the bits
    of NaN middle levels are pinned.

  python tests/golden/make_lssc_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import abi, nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.util import ref_exec  # noqa: E402

SIZES = (1, 3, 4, 5, 7, 13, 14)
QNAN, SNAN, NQNAN, INF, NINF, MAX16, PZ, NZ = 0x7e00, 0x7d01, 0xfe37, 0x7c00, 0xfc00, 0x7bff, 0x0000, 0x8000


def _bits(v):
    return np.asarray(v, np.float16).view(np.uint16)


def special_blocks():
    """(K, 16) fp16 bits: one block per row"""
    r = np.random.RandomState(7)
    rows = []
    rows.append(np.full(16, _bits(1.5)))                                       # all equal: range 0
    rows.append(np.full(16, _bits(-0.25)))
    rows.append(np.arange(16, dtype=np.uint16) % 5 + 1)                        # subnormals 1..5 ulps: range 4 * 2^-24 < 1e-6
    rows.append(np.array([3, 3, 7, 7, 1, 19, 2, 16, 8, 4, 1, 1, 19, 0, 0, 5], np.uint16))      # range 19 * 2^-24 > 1e-6
    rows.append(np.array([0x8003, 3, 0x8001, 0, 2, 0x8000, 1, 0x8002] * 2, np.uint16))        # signed subnormals
    rows.append(np.array([PZ, NZ] * 8, np.uint16))                             # +0 first: both min and max keep +0
    rows.append(np.array([NZ, PZ] * 8, np.uint16))                             # -0 first
    rows.append(np.array([NZ, PZ, _bits(1.0), NZ] + [PZ] * 12, np.uint16))     # a max above the tie
    rows.append(np.array([QNAN] + list(_bits(r.randn(15))), np.uint16))        # NaN in cell 0
    rows.append(np.array([SNAN] + list(_bits(r.randn(15))), np.uint16))        # signalling NaN in cell 0
    rows.append(np.array([NQNAN] + [_bits(2.0)] * 15, np.uint16))
    b = _bits(r.randn(16))
    b[[3, 9, 15]] = (QNAN, SNAN, NQNAN)                                        # NaN elsewhere
    rows.append(b)
    b = _bits(r.randn(16))
    b[5] = INF                                                                 # +Inf
    rows.append(b)
    b = _bits(r.randn(16))
    b[0] = NINF                                                                # -Inf in cell 0
    rows.append(b)
    rows.append(np.array([INF, NINF] * 8, np.uint16))                          # both
    rows.append(np.array([_bits(1.0), INF, NINF, QNAN] * 4, np.uint16))
    rows.append(np.array([MAX16, MAX16 | 0x8000] * 8, np.uint16))             # +-65504
    b = _bits(r.uniform(-65504, 65504, 16))
    b[[2, 11]] = (MAX16, MAX16 | 0x8000)
    rows.append(b)
    for _ in range(24):                                                        # random blocks of several scales
        rows.append(_bits(r.randn(16) * 10.0 ** r.randint(-6, 5)))
    return np.stack(rows).astype(np.uint16)


def level_pairs(rng, n):
    """(n, 4) compressed blocks with random (min, max) and random codes"""
    lo = rng.randn(n) * 10.0 ** rng.randint(-5, 4, n)
    hi = lo + np.abs(rng.randn(n)) * 10.0 ** rng.randint(-5, 4, n)
    q = np.stack([_bits(lo), _bits(hi), rng.randint(0, 65536, n), rng.randint(0, 65536, n)], -1)
    return q.astype(np.uint16)


def nan_level_pairs():
    members = (QNAN, SNAN, NQNAN, INF, NINF, _bits(1.5), _bits(-3.0), MAX16)
    q = [(lo, hi, 0b11100100 * 0x101, 0b00011011 * 0x101) for lo in members for hi in members]  # every code, twice
    return np.array(q, np.uint16)


def run(cmd, x, out_shape):
    y = np.zeros(out_shape, np.float16)
    st, (y,) = ref_exec(ref, cmd, None, 0, [x.view(np.float16)], [y], fmt=abi.CCV_TENSOR_FORMAT_NCHW)
    assert st == 0, hex(cmd.cmd)
    return np.ascontiguousarray(y).view(np.uint16)


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    r = np.random.RandomState(1)
    NCHW = abi.CCV_TENSOR_FORMAT_NCHW
    cases = {}
    for H in SIZES:
        for W in SIZES:
            cases["n4_%dx%d" % (H, W)] = _bits(r.randn(2, 3, H, W) * 4)
            cases["n3_%dx%d" % (H, W)] = _bits(r.randn(3, H, W))
    cases["n4_113x114"] = _bits(r.randn(1, 2, 113, 114))
    sp = special_blocks()
    cases["special"] = sp.reshape(-1, 4, 4)
    cases["special_cut"] = sp.reshape(-1, 4, 4)[:, :3, :3].copy()
    out = {}
    for name, x in cases.items():
        x = np.ascontiguousarray(x, np.uint16)
        y = run(nnc.CMD_COMPRESSION_LSSC_FORWARD(), x, nnc.lssc_compressed_dims(x.shape, NCHW))
        out["f_%s_x" % name], out["f_%s_y" % name] = x, y
        out["b_%s_y" % name], out["b_%s_x" % name] = y, run(nnc.CMD_COMPRESSION_LSSC_BACKWARD(), y, x.shape)
    for name, q in (("levels", level_pairs(np.random.RandomState(2), 4096)), ("nan_levels", nan_level_pairs())):
        y = q.reshape(-1, 1, 4)  # [C, 1, 4] compressed <-> [C, 4, 4] original
        out["b_%s_y" % name], out["b_%s_x" % name] = y, run(nnc.CMD_COMPRESSION_LSSC_BACKWARD(), y, (y.shape[0], 4, 4))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_lssc.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
