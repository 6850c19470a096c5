"""Timing of the normalisation commands whose reductions a change can slow down (ccv_b200/csrc/sm100_bn.cu, sm100_norm.cu):
  BATCH_NORM forward (training) and backward on ResNet-50 activation shapes, batch 64, fp32 and bf16;
  LAYER_NORM and RMSNORM backward with dscale / dbias on a transformer-sized [8192, 4096].
Each command runs through ccv_nnc_cmd_exec and is timed with CUDA events (3 warm-up launches, then the best of 3 windows of `--reps`
launches).  The card's name, power limit and maximum SM clock are read in the same run and printed beside the numbers.

--lib FILE loads that build of libccv_nnc_sm100.so instead of the package's.  --compare OLD NEW runs the whole table in child
processes that alternate between the two builds (`--rounds` each) and prints, per row, the best time of each and their ratio, so a
change to a kernel is measured against its predecessor in one call on one card.

usage: python tools/bench_norm.py [--reps R] [--lib FILE] [--compare OLD NEW [--rounds N]] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

BN_SHAPES = [(64, 112, 112, 64), (64, 56, 56, 64), (64, 56, 56, 256), (64, 28, 28, 512), (64, 14, 14, 1024), (64, 7, 7, 2048)]
ROW_SHAPE = (8192, 4096)


def rows():
    from bench_resnet_convs import time_ms
    from ccv_b200 import abi, nnc
    from tests.test_parity_norm_paths import lnorm_cmd, rms_cmd
    from tests.util import pack16
    nnc.init()
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    out = []

    def filled(shape, dt=nnc.CCV_32F, lo=-1.0, hi=1.0):
        v = (lo + (hi - lo) * rs.rand(*shape)).astype(np.float32)
        return nnc.gpu_tensor(list(shape), datatype=dt).upload(v if dt == nnc.CCV_32F else pack16(v, dt))
    for kname, dt in (("fp32", nnc.CCV_32F), ("bf16", nnc.CCV_16BF)):
        for shape in BN_SHAPES:
            C = shape[-1]
            ps = (1, 1, 1, C)
            x, g, y, h = filled(shape, dt), filled(shape, dt), filled(shape, dt), filled(shape, dt)
            scale, bias, rm, rv, sm, sis, ds, db = filled(ps, lo=0.5, hi=1.5), filled(ps), filled(ps), filled(ps, lo=0.5, hi=1.5), filled(ps), filled(ps), filled(ps), filled(ps)
            fwd, bwd = nnc.CMD_BATCH_NORM_FORWARD(1e-4, 0, 0.9), nnc.CMD_BATCH_NORM_BACKWARD(1e-4, 0, 0.9)
            t_f = time_ms(lambda: nnc.cmd_exec(fwd, None, 0, [x, scale, bias, rm, rv], [y, rm, rv, sm, sis], stream), stream, ARGS.reps)
            t_b = time_ms(lambda: nnc.cmd_exec(bwd, None, 0, [g] + [None] * 4 + [x, scale] + [None] * 6 + [sm, sis], [h, ds, db], stream), stream, ARGS.reps)
            out.append(("bn_fwd %s %s" % (kname, "x".join(map(str, shape))), t_f))
            out.append(("bn_bwd %s %s" % (kname, "x".join(map(str, shape))), t_b))
            for t in (x, g, y, h, scale, bias, rm, rv, sm, sis, ds, db):
                t.free()
    R, I = ROW_SHAPE
    x, g, h = filled(ROW_SHAPE), filled(ROW_SHAPE), filled(ROW_SHAPE)
    scale, ds, db, sm, sis = filled((1, I), lo=0.5, hi=1.5), filled((1, I)), filled((1, I)), filled((R, 1), lo=-0.1, hi=0.1), filled((R, 1), lo=1.5, hi=2.0)
    lb, rb = lnorm_cmd(abi.CCV_NNC_LAYER_NORM_BACKWARD, 1e-5, 1, (1,)), rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD, 1e-5, (1,))
    out.append(("lnorm_bwd fp32 %dx%d" % ROW_SHAPE, time_ms(lambda: nnc.cmd_exec(lb, None, 0, [g, None, None, x, scale, None, None, sm, sis], [h, ds, db], stream), stream, ARGS.reps)))
    out.append(("rmsnorm_bwd fp32 %dx%d" % ROW_SHAPE, time_ms(lambda: nnc.cmd_exec(rb, None, 0, [g, None, x, scale, None, sis], [h, ds], stream), stream, ARGS.reps)))
    stream.wait()
    return out


def main():
    global ARGS
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--lib", default="")
    ap.add_argument("--compare", nargs=2, metavar=("OLD", "NEW"))
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default="")
    ARGS = ap.parse_args()
    from bench_resnet_convs import card
    if ARGS.compare:
        best = [{}, {}]
        order = []
        for _ in range(ARGS.rounds):
            for which, lib in enumerate(ARGS.compare):
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--reps", str(ARGS.reps), "--lib", lib, "--json", "-"], stdout=subprocess.PIPE, check=True)
                for name, ms in json.loads(p.stdout.decode().strip().splitlines()[-1])["rows"]:
                    if name not in order:
                        order.append(name)
                    best[which][name] = min(best[which].get(name, ms), ms)
        c = card()
        print("card:", c)
        print("%-36s %10s %10s %7s" % ("command", "old ms", "new ms", "new/old"))
        for name in order:
            print("%-36s %10.4f %10.4f %7.3f" % (name, best[0][name], best[1][name], best[1][name] / best[0][name]))
        if ARGS.json and ARGS.json != "-":
            json.dump(dict(card=c, old=best[0], new=best[1]), open(ARGS.json, "w"), indent=1)
        return
    if ARGS.lib:
        from ccv_b200 import nnc
        nnc.LIB_PATH = os.path.abspath(ARGS.lib)
    r = rows()
    c = card()
    if ARGS.json == "-":
        print(json.dumps(dict(card=c, rows=r)))
        return
    print("card:", c)
    for name, ms in r:
        print("%-36s %10.4f ms" % (name, ms))
    if ARGS.json:
        json.dump(dict(card=c, rows=r), open(ARGS.json, "w"), indent=1)


if __name__ == "__main__":
    main()
