"""Writes tests/golden/cpuref_norm.npz: the reference's CPU_REF (oracle/_ref, built from the reference's sources) on small seeded cases of
BATCH_NORM (training, inference, backward; NHWC and NCHW), LAYER_NORM (with and without affine), RMSNORM and GROUP_NORM (NCHW and NHWC group
axes, without affine, without reduced axes), forward and backward, so that tests/test_parity_norm_paths.py pins its oracles
(tests/norm_ref.py) to CPU_REF without the reference present.

  python tests/golden/make_norm_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from ccv_b200 import abi, nnc  # noqa: E402
from oracle import ref  # noqa: E402
from tests.test_parity_norm_paths import EPS, GOLDEN_BN, GOLDEN_GN, MOMENTUM, gn_shapes, gnorm_cmd, lnorm_cmd, rms_cmd  # noqa: E402
from tests.util import ref_exec, seeded  # noqa: E402


def run(cmd, ins, outs, fmt=abi.CCV_TENSOR_FORMAT_NHWC):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs, fmt=fmt)
    assert st == 0, hex(cmd.cmd)
    return res


def main():
    assert ref.available(), "build oracle/_ref first (make -C oracle)"
    ref.ref()
    z = lambda s: np.zeros(s, np.float32)
    out = {}
    for name, shape, axis, fmt in GOLDEN_BN:
        ps = tuple(d if i == axis else 1 for i, d in enumerate(shape))
        axes = tuple(i for i in range(4) if i != axis)
        x, g = seeded(shape, 1, -1, 1) + np.float32(0.5), seeded(shape, 2, -1, 1)
        scale, bias, rm, rv = seeded(ps, 3, 0.5, 1.5), seeded(ps, 4, -1, 1), seeded(ps, 5, -1, 1), seeded(ps, 6, 0.5, 1.5)
        m, v = rm.copy(), rv.copy()
        y, m, v, sm, sis = run(nnc.CMD_BATCH_NORM_FORWARD(EPS, 0, MOMENTUM, axes=axes), [x, scale, bias, m, v], [z(shape), m, v, z(ps), z(ps)], fmt)
        (yt,) = run(nnc.CMD_BATCH_NORM_FORWARD(EPS, 1, MOMENTUM, axes=axes), [x, scale, bias, rm, rv], [z(shape)], fmt)
        h, ds, db = run(nnc.CMD_BATCH_NORM_BACKWARD(EPS, 0, MOMENTUM, axes=axes), [g] + [None] * 4 + [x, scale] + [None] * 6 + [sm, sis], [z(shape), z(ps), z(ps)], fmt)
        for k, a in dict(x=x, g=g, scale=scale, bias=bias, rm=rm, rv=rv, y=y, running_mean=m, running_var=v, mean=sm, inv_std=sis, ytest=yt, h=h, dscale=ds, dbias=db).items():
            out["%s_%s" % (name, k)] = a
    shape, axes = (5, 3, 40), (1, 2)
    rs, ps = (5, 1, 1), (1, 3, 40)
    x, g, scale, bias = seeded(shape, 11, -1, 1) + np.float32(0.5), seeded(shape, 12, -1, 1), seeded(ps, 13, 0.5, 1.5), seeded(ps, 14, -1, 1)
    for name, affine in (("ln", 1), ("ln_noaffine", 0)):
        y, sm, sis = run(lnorm_cmd(abi.CCV_NNC_LAYER_NORM_FORWARD, 1e-5, affine, axes), [x, scale, bias] if affine else [x], [z(shape), z(rs), z(rs)])
        d = dict(x=x, g=g, y=y, mean=sm, inv_std=sis)
        if affine:
            h, ds, db = run(lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 1, axes), [g, None, None, x, scale, None, None, sm, sis], [z(shape), z(ps), z(ps)])
            d.update(scale=scale, bias=bias, h=h, dscale=ds, dbias=db)
        else:
            (h,) = run(lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 0, axes), [g, None, None, x, None, sm, sis], [z(shape)])
            d.update(h=h)
        for k, a in d.items():
            out["%s_%s" % (name, k)] = a
    y, sis = run(rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD, 1e-5, axes), [x, scale], [z(shape), z(rs)])
    h, ds = run(rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, 1e-5, axes), [g, None, x, scale, None, sis], [z(shape), z(ps)])
    for k, a in dict(x=x, g=g, scale=scale, y=y, inv_std=sis, h=h, dscale=ds).items():
        out["rms_" + k] = a
    for name, shape, group_axis, groups, reduce_axes, affine in GOLDEN_GN:
        rs, ps = gn_shapes(shape, group_axis, groups, reduce_axes)
        x, g, scale, bias = seeded(shape, 21, -1, 1), seeded(shape, 22, -1, 1), seeded(ps, 23, 0.5, 1.5), seeded(ps, 24, -1, 1)
        fwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_FORWARD, group_axis, groups, 1e-5, affine, reduce_axes)
        bwd = gnorm_cmd(abi.CCV_NNC_GROUP_NORM_BACKWARD, group_axis, groups, 1e-5, affine, reduce_axes)
        y, sm, sis = run(fwd, [x, scale, bias] if affine else [x], [z(shape), z(rs), z(rs)])
        d = dict(x=x, g=g, y=y, mean=sm, inv_std=sis)
        if affine:
            h, ds, db = run(bwd, [g, None, None, x, scale, None, None, sm, sis], [z(shape), z(ps), z(ps)])
            d.update(scale=scale, bias=bias, h=h, dscale=ds, dbias=db)
        else:
            (h,) = run(bwd, [g, None, None, x, None, sm, sis], [z(shape)])
            d.update(h=h)
        for k, a in d.items():
            out["%s_%s" % (name, k)] = a
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpuref_norm.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
