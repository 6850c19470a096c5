"""CCV_NNC_COMM_ALLREDUCE_FORWARD on CCV_NNC_BACKEND_GPU_SM100 (ccv_b200/csrc/sm100_comm.cu), the protocol of
test/int/nnc/nccl.tests.c:13-44: every participant contributes a tensor, every participant ends with the element-wise
sum.  Integer-valued fp32 inputs make the sum exact, so the check is bit-for-bit.  With one visible GPU the command is
checked in its single-participant forms; with two or more, two ranks (one process per GPU) run the real exchange and a
2-way data-parallel step of a small model is compared with the single-device step on the concatenated batch
(test/int/nnc/parallel.tests.c:192-371)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_allreduce_single_participant_is_a_copy(gpu):
    nnc = gpu
    stream = nnc.Stream(0)
    a, b = nnc.gpu_tensor([1000]), nnc.gpu_tensor([1000])
    x = np.arange(1000, dtype=np.float32)
    a.upload(x), b.upload(np.zeros(1000, np.float32))
    cmd = nnc.CMD_COMM_ALLREDUCE_FORWARD()
    assert nnc.cmd_exec(cmd, None, 0, [a], [b], stream) == 0
    stream.wait()
    assert np.array_equal(b.download(), x)
    assert nnc.cmd_exec(cmd, None, 0, [a], [a], stream) == 0  # in place
    stream.wait()
    assert np.array_equal(a.download(), x)
    for t in (a, b, stream):
        t.free()


def test_allreduce_world_of_one_through_nccl(gpu):
    nnc = gpu
    nnc.comm_init_rank(nnc.comm_unique_id(), 1, 0)
    stream = nnc.Stream(0)
    a, b = nnc.gpu_tensor([4, 250]), nnc.gpu_tensor([4, 250])
    x = np.random.RandomState(0).randint(-100, 100, size=(4, 250)).astype(np.float32)
    a.upload(x)
    l0 = nnc.launch_count()
    assert nnc.cmd_exec(nnc.CMD_COMM_ALLREDUCE_FORWARD(), None, 0, [a, b], [a, b], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    stream.wait()
    assert nnc.launch_count() == l0 + 1  # both tensors in one NCCL group
    assert np.array_equal(a.download(), x)
    nnc.lib().ccv_nnc_sm100_comm_destroy()
    for t in (a, b, stream):
        t.free()


WORKER = r"""
import os, sys
import numpy as np
sys.path.insert(0, %(root)r)
import torch
import torch.distributed as dist
from ccv_b200 import dp, nnc, resnet50

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("gloo")  # side channel only: carries the 128-byte communicator id
nnc.init()
stream = nnc.Stream(rank)


class TinyNet(resnet50.Net):
    def _build_body(self, x, xs):
        x, xs = self._conv(x, xs, 3, 8, 3, 2, 1, True, "c0", need_dx=False)
        x = self._relu(x, xs, "r0")
        x, xs = self._conv(x, xs, 8, 8, 3, 1, 1, True, "c1")
        x = self._relu(x, xs, "r1")
        return x, xs


def run(batch, global_batch, x, y, allreduce):
    net = TinyNet(batch, image=8, classes=5, global_batch=global_batch, device=rank, seed=3, learn_rate=0.1, algorithm=2)
    net.input.upload(x), net.labels.upload(y)
    for node in net.fwd + net.bwd:
        assert nnc.cmd_exec(*node, stream=stream) == 0
    if allreduce:
        allreduce(net)
    for node in net.opt:
        assert nnc.cmd_exec(*node, stream=stream) == 0
    stream.wait()
    return net


rs = np.random.RandomState(5)
x, y = rs.rand(8, 8, 8, 3).astype(np.float32), rs.randint(0, 5, size=(8,)).astype(np.int32)
exchange = {}


def allreduce(net):
    if "op" not in exchange:
        exchange["op"] = dp.CommandAllreduce(net, dist, stream, rank, world)
    exchange["op"].net = net
    exchange["op"]()

# 1. plain allreduce of integer-valued tensors: exact sum on every rank
t = nnc.gpu_tensor([3, 1000], device=rank)
t.upload(np.full((3, 1000), rank + 1, np.float32) * np.arange(1000, dtype=np.float32))
holder = type("N", (), {"g_flat": t})()
allreduce(holder)
stream.wait()
want = np.arange(1000, dtype=np.float32) * sum(range(1, world + 1))
assert np.array_equal(t.download(), np.broadcast_to(want, (3, 1000))), "allreduce sum wrong on rank %%d" %% rank

# 2. 2-way data parallel step == single-device step on the concatenated batch
sharded = run(8 // world, 8, dp.shard(x, rank, world), dp.shard(y, rank, world), allreduce)
single = run(8, 8, x, y, None)
w_dp, w_1 = sharded.w_flat.download(), single.w_flat.download()
err = np.abs(w_dp - w_1).max() / np.abs(w_1).max()
assert err < 1e-5, "rank %%d: data-parallel weights differ from single-device weights by %%g" %% (rank, err)

# 3. the same step with the exchange woven into the backward GRAPH: one COMM_ALLREDUCE node per gradient bucket on the graph's
#    side stream (ccv_b200/resnet50.py: backward_with_exchange), eagerly and as a captured CUDA graph with the NCCL kernels inside
def step_single(net):
    for node in net.fwd + net.bwd + net.opt:
        assert nnc.cmd_exec(*node, stream=stream) == 0
    stream.wait()

net_g = TinyNet(8 // world, image=8, classes=5, global_batch=8, device=rank, seed=3, learn_rate=0.1, algorithm=2)
net_g.input.upload(dp.shard(x, rank, world)), net_g.labels.upload(dp.shard(y, rank, world))
g = nnc.Graph()
for node in net_g.fwd:
    g.exec_new(*node)
nodes, side = net_g.backward_with_exchange(2)
assert len(side) == 2
for j, node in enumerate(nodes):
    idx = g.exec_new(*node)
    if j in side:
        g.set_side_stream(idx)
for node in net_g.opt:
    g.exec_new(*node)
g.fuse()
assert g.run(stream) == 0
stream.wait()
err = np.abs(net_g.w_flat.download() - w_1).max() / np.abs(w_1).max()
assert err < 1e-5, "rank %%d: graph with side-stream exchange differs from the single-device step by %%g" %% (rank, err)
cid = g.capture(stream)          # capture = one more eager step, then the recording
assert g.replay(cid, stream) == 0
stream.wait()
step_single(single), step_single(single)
w_3 = single.w_flat.download()
err3 = np.abs(net_g.w_flat.download() - w_3).max() / np.abs(w_3).max()
assert err3 < 1e-4, "rank %%d: captured graph with the exchange inside differs after 3 steps by %%g" %% (rank, err3)
print("rank %%d ok %%g %%g %%g" %% (rank, err, 0.0, err3))
dist.barrier()
dist.destroy_process_group()
"""


def test_two_rank_allreduce_and_data_parallel_step(gpu, tmp_path):
    nnc = gpu
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) < 2:
        pytest.skip("needs two GPUs (run with gpurun --gpus 2)")
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT})
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            out, _ = p.communicate(timeout=300)
        except subprocess.TimeoutExpired:
            p.kill()
            out, _ = p.communicate()
        outs.append(out)
    for rank, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (rank, out[-3000:])
        assert "rank %d ok" % rank in out


def test_one_process_two_devices_convolution_and_allreduce(gpu, ref):
    """The reference's own shape (comm/gpu/ccv_nnc_comm_gpu_nccl.cu:12-58, test/int/nnc/nccl.tests.c:13-44): ONE process drives
    several devices.  A tensor-core convolution (dynamic shared memory attribute, stream workspace, tensor maps) runs on device 1
    through a stream context of device 1 while device 0 is current, and is checked against CPU_REF; then one
    COMM_ALLREDUCE command sums a tensor per device, its per-device streams found through neighbour discovery."""
    from tests.util import assert_close, ref_exec, seeded
    nnc = gpu
    if nnc.lib().ccv_nnc_device_count(nnc.CCV_STREAM_CONTEXT_GPU) < 2:
        pytest.skip("needs two GPUs (run with gpurun --gpus 2)")
    s0, s1 = nnc.Stream(0), nnc.Stream(1)
    s0.set_neighbors({0: s0, 1: s1})
    N, H, Cc, K = 4, 28, 64, 128
    a, w, bias = seeded((N, H, H, Cc), 1, -1, 1), seeded((K, 3, 3, Cc), 2, -1, 1) / 24, seeded((K,), 3)
    hint = nnc.hint((1, 1), (1, 1))
    cmd = nnc.CMD_CONVOLUTION_FORWARD(1, K, 3, 3, Cc)
    want = np.zeros((N, H, H, K), np.float32)
    assert ref_exec(ref, cmd, hint, 0, [a, w, bias], [want])[0] == 0
    outs = []
    for dev, st in ((0, s0), (1, s1)):
        ta, tw, tb = (nnc.gpu_tensor(list(v.shape), device=dev).upload(v) for v in (a, w, bias))
        ty = nnc.gpu_tensor([N, H, H, K], device=dev)
        assert nnc.cmd_exec(cmd, hint, 0, [ta, tw, tb], [ty], st) == 0, nnc.lib().ccv_nnc_sm100_last_error()
        st.wait()
        assert_close(ty.download(), want, 1e-3, "convolution on device %d" % dev)
        outs.append(ty)
        for t in (ta, tw, tb):
            t.free()
    # integer-valued payloads: the sum is exact
    x0, x1 = np.arange(4096, dtype=np.float32), np.arange(4096, dtype=np.float32)[::-1] * 3
    t0, t1 = nnc.gpu_tensor([4096], device=0).upload(x0), nnc.gpu_tensor([4096], device=1).upload(x1)
    assert nnc.cmd_exec(nnc.CMD_COMM_ALLREDUCE_FORWARD(), None, 0, [t0, t1], [t0, t1], s0) == 0, nnc.lib().ccv_nnc_sm100_last_error()
    s0.wait(), s1.wait()
    assert np.array_equal(t0.download(), x0 + x1) and np.array_equal(t1.download(), x0 + x1)
    # a stream context that cannot name the other device's stream is refused (nothing would order the reduction there)
    lonely = nnc.Stream(0)
    assert nnc.cmd_exec(nnc.CMD_COMM_ALLREDUCE_FORWARD(), None, 0, [t0, t1], [t0, t1], lonely) != 0
    nnc.lib().ccv_nnc_sm100_comm_destroy()
    for t in outs + [t0, t1, lonely, s0, s1]:
        t.free()


def test_stream_signals_order_two_stream_contexts(gpu):
    """ccv_nnc_stream_context_emit_signal / wait_signal (lib/nnc/ccv_nnc.h:1041-1053): work on stream B that waits for a signal emitted
    on stream A sees everything A enqueued before the emit (the mechanism bench.py's end-to-end leg uses to prefetch the next
    batch on a copy stream)."""
    nnc = gpu
    a_stream, b_stream = nnc.Stream(0), nnc.Stream(0)
    sig = nnc.Signal(0)
    n = 1 << 24
    src, dst = nnc.gpu_tensor([n]), nnc.gpu_tensor([n])
    dst.upload(np.zeros(n, np.float32))
    for value in (3.0, 7.0):
        assert nnc.cmd_exec(nnc.CMD_SET_FORWARD(value), None, 0, [], [src], a_stream) == 0   # a long enough fill on A
        sig.emit(a_stream)
        sig.wait(b_stream)
        assert nnc.cmd_exec(nnc.CMD_DATA_TRANSFER_FORWARD(), None, 0, [src], [dst], b_stream) == 0
        b_stream.wait()
        assert np.all(dst.download() == value)
        a_stream.wait()
    for t in (src, dst, sig, a_stream, b_stream):
        t.free()
