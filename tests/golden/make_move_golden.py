"""Writes tests/golden/cpuref_move.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on DATATYPE_CONVERSION
f32 -> f16 and f64 -> f16 over the special values (zeros, subnormal boundaries, the top of the half range, infinities, NaNs with high
and low payloads) plus random bit patterns, f16 -> f32 over every code, UPSAMPLE forward and backward for every (type, align_corners,
format) at the geometries of tests/test_parity_move_paths.UP_CASES, and INDEX_SELECT (copy, fp32-index lerp, backward with repeated
indices), so that tests/test_parity_move_paths.py pins its oracles (tests/move_ref.py) to CPU_REF without the reference present.

  python tests/golden/make_move_golden.py"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests import move_ref as R  # noqa: E402
from tests.test_parity_move_paths import LERP_IDX, UP_CASES, up_data, up_shape, upsample_cmd  # noqa: E402
from tests.util import NCHW, NHWC, ref_exec, seeded  # noqa: E402


def run(cmd, ins, outs, fmt=NHWC):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs, fmt=fmt)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {}
    conv = nnc.CMD_DATATYPE_CONVERSION_FORWARD()
    r = np.random.RandomState(1)
    x = np.concatenate([R.f16_specials(), r.randint(0, 2 ** 32, size=4096, dtype=np.uint64).astype(np.uint32).view(np.float32)])
    out["f2h_x"] = x
    out["f2h_h"] = run(conv, [x], [np.zeros(x.shape, np.float16)])[0].view(np.uint16)
    d = np.concatenate([R.f16_specials().astype(np.float64), [65519.99999999, 65520.000001, 2.0 ** -25 * (1 + 2.0 ** -30), 1 + 2.0 ** -24 + 2.0 ** -40, 1e300, -1e300, 1e-300],
                        r.uniform(-70000, 70000, 1024), r.standard_normal(1024) * 1e-5])
    out["d2h_x"] = d
    out["d2h_h"] = run(conv, [d], [np.zeros(d.shape, np.float16)])[0].view(np.uint16)
    codes = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)
    out["h2f_f"] = run(conv, [codes], [np.zeros(codes.shape, np.float32)])[0]
    for k, (H, W, OH, OW) in enumerate(UP_CASES):
        for bilinear in (0, 1):
            for align in (0, 1):
                for nchw in (0, 1):
                    key = "up_%d_%d_%d_%d_%d_%d_%d_" % (H, W, OH, OW, bilinear, align, nchw)
                    fmt = NCHW if nchw else NHWC
                    ishape, oshape = up_shape(2, 3, H, W, nchw), up_shape(2, 3, OH, OW, nchw)
                    a, g = up_data(ishape, 60 + k), up_data(oshape, 70 + k)
                    out[key + "a"], out[key + "g"] = a, g
                    out[key + "b"] = run(upsample_cmd(0, bilinear, align, H, W, OH, OW), [a], [np.zeros(oshape, np.float32)], fmt)[0]
                    out[key + "h"] = run(upsample_cmd(1, bilinear, align, H, W, OH, OW), [g], [np.zeros(ishape, np.float32)], fmt)[0]
    a = seeded((7, 5), 2, -2, 2)
    idx = np.array([3, 0, 6, 3, 3, 5, 1, 6], np.int32)
    g = seeded((len(idx), 5), 3, -1, 1) * np.float32(100) ** seeded((len(idx), 1), 4, -1, 1)
    out["is_a"], out["is_idx"], out["is_g"] = a, idx, g.astype(np.float32)
    out["is_lerp"] = run(nnc.CMD_INDEX_SELECT_FORWARD(), [a, LERP_IDX], [np.zeros((len(LERP_IDX), 5), np.float32)])[0]
    out["is_b"] = run(nnc.CMD_INDEX_SELECT_FORWARD(), [a, idx], [np.zeros((len(idx), 5), np.float32)])[0]
    out["is_h"] = run(nnc.CMD_INDEX_SELECT_BACKWARD(), [out["is_g"], None, idx], [np.zeros((7, 5), np.float32)])[0]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_move.npz")
    # np.savez_compressed stamps each member with the current time; fixed stamps make the file a function of its contents
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(out[name]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
