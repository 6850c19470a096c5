"""Graph rewrites (h) and (i) of ccv_nnc_sm100_graph_fuse (ccv_b200/csrc/nnc_host.cu), on CPU: BATCH_NORM_FORWARD ; EWSUM ;
RELU_FORWARD at the end of a residual block becomes one node y = relu(bn(x) + s), and AVERAGE_POOL_BACKWARD ; EWSUM ; RELU_BACKWARD
at the shortcut of a strided block one node out = y > 0 ? r + pool_backward(g) : 0.  The pass only inspects node descriptions and
tensor identities, so nothing is executed here and the tensors are host tensors."""
from ccv_b200 import abi, nnc, resnet50


class HostFactory(object):
    """resnet50.Net's allocator on host memory: the node list is built exactly as on the device."""

    def alloc(self, shape, datatype=abi.CCV_32F):
        return nnc.cpu_tensor(list(shape), datatype=datatype)

    def alias(self, base, elem_offset, shape, datatype=abi.CCV_32F):
        params = abi.tensor_param(abi.CCV_TENSOR_CPU_MEMORY, abi.CCV_TENSOR_FORMAT_NHWC, datatype, list(shape))
        return nnc.tensor_new(params, base.data_ptr + elem_offset * abi.DTYPE_SIZE[datatype])


def _t(*dims):
    return nnc.cpu_tensor(list(dims))


def _junction(g, x, z, short, out):
    scale, bias, mean, var, sm, sis = (_t(1, 1, 1, x.dims[-1]) for _ in range(6))
    g.exec_new(nnc.CMD_BATCH_NORM_FORWARD(1e-4, 0, 0.9), None, 0, [x, scale, bias, mean, var], [z, mean, var, sm, sis])
    g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [z, short], [out])
    g.exec_new(nnc.CMD_RELU_FORWARD(), None, 0, [out], [out])
    return [x, scale, bias, mean, var], [out, mean, var, sm, sis]


def test_every_resnet50_junction_fuses():
    nnc.init()
    net = resnet50.Net(2, image=32, classes=10, factory=HostFactory())
    g = nnc.Graph()
    for cmd, hint, flags, ins, outs in net.fwd + net.bwd:
        g.exec_new(cmd, hint, flags, ins, outs)
    n_before = len(g)
    removed = g.fuse()
    nodes = g.nodes()
    assert removed == n_before - len(nodes)
    ends = [L for L in net.layers if L["kind"] == "block_end"]
    assert len(ends) == 16
    fused = [(kind, ins, outs) for cmd, kind, ins, outs in nodes if cmd == abi.CCV_NNC_BATCH_NORM_FORWARD and len(outs) == 6]
    assert len(fused) == 16
    for (kind, ins, outs), L in zip(fused, ends):
        # the output is the block's y, the residual addend (6th output, read only) the shortcut; the inputs are the batch norm's own
        # (rule (f), which would append the statistics tensor, links device tensors only)
        assert kind == 7 and len(ins) == 5 and outs[5] == L["short"].ptr and outs[0] == L["y"].ptr
    # no forward EWSUM is left: every residual sum of the forward pass went into a batch norm
    fwd_sums = [k for cmd, k, ins, outs in nodes if cmd == abi.CCV_NNC_EWSUM_FORWARD and k == 3]
    assert fwd_sums == []
    # (i): the three strided blocks' shortcut pools take their block's gradient sum and ReLU mask; the other 12 sums behind a ReLU
    # and the one behind the max pool stay EWSUM nodes
    strided = [L for L in net.layers if L["kind"] == "avgpool" and L["name"].endswith(".avgdown")]
    assert len(strided) == 3
    pools = [(ins, outs) for cmd, kind, ins, outs in nodes if cmd == abi.CCV_NNC_AVERAGE_POOL_BACKWARD and kind == 0 and len(ins) == 3]
    assert len(pools) == 3
    by_x = {L["x"].ptr: L for L in net.layers if L["kind"] == "block_end"}
    for ins, outs in pools:
        # the mask is the block input (the previous block's y), the output the block input's gradient, the addend the main branch's
        assert ins[2] in by_x and outs[0] == ins[1]
    assert sum(1 for cmd, k, _, _ in nodes if cmd == abi.CCV_NNC_EWSUM_FORWARD and k == 4) == 12
    g.free()


def test_junction_fuses_on_its_own():
    nnc.init()
    N, H, C = 2, 4, 16
    x, z, short, out = (_t(N, H, H, C) for _ in range(4))
    g = nnc.Graph()
    ins, outs = _junction(g, x, z, short, out)
    assert g.fuse() == 2
    (cmd, kind, fins, fouts), = g.nodes()
    assert cmd == abi.CCV_NNC_BATCH_NORM_FORWARD and kind == 7
    assert fins == [t.ptr for t in ins]
    assert fouts == [t.ptr for t in outs] + [short.ptr]
    g.free()


def test_junction_with_the_sum_reversed_fuses():
    nnc.init()
    N, H, C = 2, 4, 16
    x, z, short, out = (_t(N, H, H, C) for _ in range(4))
    g = nnc.Graph()
    scale, bias, mean, var, sm, sis = (_t(1, 1, 1, C) for _ in range(6))
    g.exec_new(nnc.CMD_BATCH_NORM_FORWARD(1e-4, 0, 0.9), None, 0, [x, scale, bias, mean, var], [z, mean, var, sm, sis])
    g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [short, z], [out])
    g.exec_new(nnc.CMD_RELU_FORWARD(), None, 0, [out], [out])
    assert g.fuse() == 2
    (_, _, fins, fouts), = g.nodes()
    assert len(fins) == 5 and fouts[5] == short.ptr and fouts[0] == out.ptr
    g.free()


def test_junction_whose_batch_norm_output_is_read_later_is_left_alone():
    nnc.init()
    N, H, C = 2, 4, 16
    x, z, short, out, other = (_t(N, H, H, C) for _ in range(5))
    for reader in ("same tensor", "view"):
        g = nnc.Graph()
        _junction(g, x, z, short, out)
        # a later node reads the batch norm's output, directly or through a view of part of its memory
        r = z if reader == "same tensor" else nnc.tensor_view_new(z, [1, H, H, C], [1, 0, 0, 0], [H * H * C, H * C, C, 1])
        g.exec_new(nnc.CMD_RELU_FORWARD(), None, 0, [r], [other])
        g.fuse()
        kinds = [k for _, k, _, _ in g.nodes()]
        cmds = [c for c, _, _, _ in g.nodes()]
        # the sum and its ReLU still fuse with each other (rule (c)), the batch norm stays a node of its own
        assert cmds[:2] == [abi.CCV_NNC_BATCH_NORM_FORWARD, abi.CCV_NNC_EWSUM_FORWARD] and kinds[:2] == [0, 3], (reader, kinds)
        assert len(g.nodes()[0][3]) == 5
        g.free()


def test_junction_with_a_view_as_batch_norm_output_is_left_alone():
    nnc.init()
    N, H, C = 2, 4, 16
    x, zbase, short, out = _t(N, H, H, C), _t(N + 1, H, H, C), _t(N, H, H, C), _t(N, H, H, C)
    z = nnc.tensor_view_new(zbase, [N, H, H, C], [1, 0, 0, 0], [H * H * C, H * C, C, 1])
    g = nnc.Graph()
    _junction(g, x, z, short, out)
    g.fuse()
    assert [k for _, k, _, _ in g.nodes()] == [0, 3]
    assert len(g.nodes()[0][3]) == 5
    g.free()


def test_batch_norm_in_test_mode_is_left_alone():
    nnc.init()
    N, H, C = 2, 4, 16
    x, z, short, out = (_t(N, H, H, C) for _ in range(4))
    scale, bias, mean, var = (_t(1, 1, 1, C) for _ in range(4))
    g = nnc.Graph()
    g.exec_new(nnc.CMD_BATCH_NORM_FORWARD(1e-4, 1, 0.9), None, 0, [x, scale, bias, mean, var], [z])
    g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [z, short], [out])
    g.exec_new(nnc.CMD_RELU_FORWARD(), None, 0, [out], [out])
    g.fuse()
    assert [k for _, k, _, _ in g.nodes()] == [0, 3]
    g.free()


def _pool_junction(g, gp, gs, gmain, y):
    g.exec_new(nnc.CMD_AVERAGE_POOL_BACKWARD(2, 2), nnc.hint((2, 2), (0, 0)), 0, [gp], [gs])
    g.exec_new(nnc.CMD_EWSUM_FORWARD(), None, 0, [gmain, gs], [gmain])
    g.exec_new(nnc.CMD_RELU_BACKWARD(), None, 0, [gmain, None, y], [gmain])


def test_pool_junction_fuses_on_its_own():
    nnc.init()
    N, H, C = 2, 8, 16
    gp, gs, gmain, y = _t(N, H // 2, H // 2, C), _t(N, H, H, C), _t(N, H, H, C), _t(N, H, H, C)
    g = nnc.Graph()
    _pool_junction(g, gp, gs, gmain, y)
    assert g.fuse() == 2
    (cmd, kind, ins, outs), = g.nodes()
    assert cmd == abi.CCV_NNC_AVERAGE_POOL_BACKWARD and kind == 0
    assert ins == [gp.ptr, gmain.ptr, y.ptr] and outs == [gmain.ptr]
    g.free()


def test_pool_junction_whose_pool_gradient_is_read_later_is_left_alone():
    nnc.init()
    N, H, C = 2, 8, 16
    gp, gs, gmain, y, other = _t(N, H // 2, H // 2, C), _t(N, H, H, C), _t(N, H, H, C), _t(N, H, H, C), _t(N, H, H, C)
    g = nnc.Graph()
    _pool_junction(g, gp, gs, gmain, y)
    g.exec_new(nnc.CMD_RELU_BACKWARD(), None, 0, [gs, None, y], [other])
    g.fuse()
    # the pool stays; the sum and its ReLU backward still fuse with each other (rule (d))
    assert [(c, k) for c, k, _, _ in g.nodes()][:2] == [(abi.CCV_NNC_AVERAGE_POOL_BACKWARD, 0), (abi.CCV_NNC_EWSUM_FORWARD, 4)]
    assert len(g.nodes()[0][2]) == 1
    g.free()
