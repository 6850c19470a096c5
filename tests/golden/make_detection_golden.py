"""Writes tests/golden/cpuref_detection.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on ROI_ALIGN and
NMS, forward and backward, so that tests/test_parity_detection.py pins its oracles (tests/detection_ref.py) to CPU_REF without the
reference present.  CPU_REF runs these commands in fp32 NHWC only.

ROI_ALIGN: ROIs inside, partly outside (above / left: CPU_REF's row shift), wholly outside, below one pixel, larger than the map and of
negative size; pools 1x1, 7x7 and 14x14; the three batch forms (one map and k ROIs, k maps and one ROI, k of each).
NMS: chained suppression (a box suppressed by a kept one cannot suppress), thresholds 0.5, 0 and 1, a batch of 2, and no tied scores
(CPU_REF's quicksort is unstable on ties).

  python tests/golden/make_detection_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402

BOXES = np.array([[0.10, 0.15, 0.50, 0.40],    # inside
                  [-0.20, -0.30, 0.80, 0.90],  # partly above and left of the map
                  [0.70, 0.60, 0.60, 0.70],    # partly below and right
                  [1.50, 1.20, 0.30, 0.30],    # wholly outside
                  [0.40, 0.45, 0.01, 0.02],    # below one pixel
                  [-0.10, 0.05, 1.40, 1.30],   # larger than the map
                  [0.30, 0.30, -0.20, 0.30]], np.float32)  # negative width: empty
# (name, a's shape, ROI rows (None: one [4] ROI, row 1), pool)
ROI_CASES = [("one_map_k_rois", (12, 16, 5), list(range(7)), (7, 7)),
             ("k_maps_one_roi", (3, 12, 16, 5), None, (1, 1)),
             ("k_maps_k_rois", (3, 12, 16, 5), [0, 2, 5], (14, 14)),
             ("pool_7_single", (12, 16, 5), [1], (7, 7))]
NMS_THRESHOLDS = (0.5, 0.0, 1.0)


def nms_boxes():
    """rows (score, x, y, w, h): 0 > 1 overlap at IoU 0.6, 1 > 2 at 0.6 and 0, 2 apart (2 survives because 1 is suppressed), a duplicate
    of 3 at lower score, a zero-area box, disjoint boxes; the second item is a permuted, shifted copy"""
    a = np.array([[0.90, 0.0, 0.0, 10.0, 10.0],
                  [0.80, 2.5, 0.0, 10.0, 10.0],
                  [0.70, 5.0, 0.0, 10.0, 10.0],
                  [0.65, 40.0, 40.0, 8.0, 8.0],
                  [0.55, 40.0, 40.0, 8.0, 8.0],
                  [0.50, 20.0, 20.0, 0.0, 0.0],
                  [0.45, 60.0, 0.0, 4.0, 4.0],
                  [0.40, 61.0, 1.0, 4.0, 4.0],
                  [0.35, 0.0, 60.0, 6.0, 3.0],
                  [0.30, 100.0, 100.0, 1.0, 1.0]], np.float32)
    r = np.random.RandomState(5)
    b = a[r.permutation(len(a))].copy()
    b[:, 1:3] += 3.0
    b[:, 0] -= 0.01
    return np.stack([a[r.permutation(len(a))], b])


def run(cmd, ins, outs):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    out = {"boxes": BOXES}
    for k, (name, shape, rows, (ph, pw)) in enumerate(ROI_CASES):
        a = seeded(shape, 70 + k, -1, 1)
        b = BOXES[1] if rows is None else BOXES[rows]
        n = max(shape[0] if len(shape) == 4 else 1, 1 if b.ndim == 1 else len(b))
        cshape = (ph, pw, shape[-1]) if len(shape) == 3 and b.ndim == 1 else (n, ph, pw, shape[-1])
        g = seeded(cshape, 80 + k, -1, 1)
        out["roi_a_" + name], out["roi_b_" + name], out["roi_g_" + name] = a, b, g
        (out["roi_c_" + name],) = run(nnc.CMD_ROI_ALIGN_FORWARD(ph, pw), [a, b], [np.zeros(cshape, np.float32)])
        (out["roi_h_" + name],) = run(nnc.CMD_ROI_ALIGN_BACKWARD(ph, pw), [g, None, b], [np.zeros(shape, np.float32)])
    a = nms_boxes()
    out["nms_a"] = a
    for t in NMS_THRESHOLDS:
        b, c = run(nnc.CMD_NMS_FORWARD(t), [a], [np.zeros_like(a), np.zeros(a.shape[:2], np.int32)])
        out["nms_b_%g" % t], out["nms_c_%g" % t] = b, c
        g = seeded(a.shape, 90, -1, 1)
        out["nms_g_%g" % t] = g
        (out["nms_h_%g" % t],) = run(nnc.CMD_NMS_BACKWARD(t), [g, None, None, None, c], [np.full(a.shape, 7, np.float32)])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_detection.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
