"""Timing of the feeder kernels whose pointer qualifiers or loops a change can alter (ccv_b200/csrc/sm100_ew.cu): SOFTMAX forward and
backward, CATEGORICAL_CROSSENTROPY forward and backward and SOFTMAX_CROSSENTROPY forward (out of place and in place) on ResNet-50's
head ([batch, 1000], batch 256 and 4096), and SGD_FORWARD in place on one tensor of ResNet-50's size (25 557 032 parameters) and on its
classifier weight (2 048 000).
Each command runs through ccv_nnc_cmd_exec and is timed with CUDA events (3 warm-up launches, then the best of 3 windows of `--reps`
launches).  The card's name, power limit and maximum SM clock are read in the same run and printed beside the numbers.

--lib FILE loads that build of libccv_nnc_sm100.so instead of the package's.  --compare OLD NEW runs the whole table in child
processes that alternate between the two builds (`--rounds` each) and prints, per row, the best time of each and their ratio, so a
change to a kernel is measured against its predecessor in one call on one card.

usage: python tools/bench_feeders.py [--reps R] [--lib FILE] [--compare OLD NEW [--rounds N]] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HEADS = [(256, 1000), (4096, 1000)]
SGD_COUNTS = [25557032, 2048000]


def rows():
    from bench_resnet_convs import time_ms
    from ccv_b200 import nnc
    nnc.init()
    stream = nnc.Stream(0)
    rs = np.random.RandomState(0)
    out = []

    def filled(shape, lo=-1.0, hi=1.0):
        return nnc.gpu_tensor(list(shape)).upload((lo + (hi - lo) * rs.rand(*shape)).astype(np.float32))
    for B, K in HEADS:
        a, y, g, h, d = filled((B, K), -4, 4), filled((B, K), 0.001, 0.002), filled((B, K)), filled((B, K)), filled((B, K))
        c, gl = filled((B,)), filled((B,), 0.5, 1.5)
        lab = nnc.gpu_tensor([B], datatype=nnc.CCV_32S).upload(rs.randint(0, K, size=B).astype(np.int32))
        tag = "%dx%d" % (B, K)
        sf, cf, cb, sc = nnc.CMD_SOFTMAX_FORWARD(), nnc.CMD_CATEGORICAL_CROSSENTROPY_FORWARD(), nnc.CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(), nnc.CMD_SOFTMAX_CROSSENTROPY_FORWARD()
        out.append(("softmax_fwd " + tag, time_ms(lambda: nnc.cmd_exec(sf, None, 0, [a], [d], stream), stream, ARGS.reps)))
        out.append(("softmax_bwd " + tag, time_ms(lambda: nnc.cmd_exec(nnc.CMD_SOFTMAX_BACKWARD(), None, 0, [g, None, y], [h], stream), stream, ARGS.reps)))
        out.append(("cce_fwd " + tag, time_ms(lambda: nnc.cmd_exec(cf, None, 0, [y, lab], [c], stream), stream, ARGS.reps)))
        out.append(("cce_bwd " + tag, time_ms(lambda: nnc.cmd_exec(cb, None, 0, [None, y, lab], [h], stream), stream, ARGS.reps)))
        out.append(("softmax_cce_fwd " + tag, time_ms(lambda: nnc.cmd_exec(sc, None, 0, [a, lab], [c, d], stream), stream, ARGS.reps)))
        # in place: the logits are overwritten by the probabilities on every launch, which keeps them in [0, 1]
        out.append(("softmax_cce_fwd in place " + tag, time_ms(lambda: nnc.cmd_exec(sc, None, 0, [h, lab], [c, h], stream), stream, ARGS.reps)))
        for t in (a, y, g, h, d, c, gl, lab):
            t.free()
    for n in SGD_COUNTS:
        g, w, m = filled((n,)), filled((n,)), filled((n,))
        cmd = nnc.CMD_SGD_FORWARD(1, 0.1, 1.0 / 256, 0.0001, 0.9, 0.0)
        out.append(("sgd in place %d" % n, time_ms(lambda: nnc.cmd_exec(cmd, None, 0, [g, w, m], [w, m], stream), stream, ARGS.reps)))
        for t in (g, w, m):
            t.free()
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
