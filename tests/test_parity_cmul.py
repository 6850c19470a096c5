"""CMUL forward / backward (complex multiplication of (real, imaginary) pairs along the last axis: rotary position embeddings) on
CCV_NNC_BACKEND_GPU_SM100 against the reference's CPU_REF (blas/ccv_nnc_cmul_cpu_ref.c).

Both sides round every product and sum on its own, in CPU_REF's order, so every comparison is exact (np.array_equal): fp32 against
CPU_REF directly, bf16 / fp16 against CPU_REF on the widened 16-bit inputs, rounded to nearest even.  Inputs are seeded U(-1, 1)."""
import numpy as np
import pytest

from ccv_b200 import abi, nnc as _nnc
from tests.util import NHWC, counted, gpu_exec, gpu_exec16, pack16, ref_exec, rel_err, round16, seeded, unpack16

pytestmark = [pytest.mark.gpu, pytest.mark.ref]
KINDS = {"fp32": abi.CCV_32F, "bf16": abi.CCV_16BF, "fp16": abi.CCV_16F}
INVALID = abi.CCV_NNC_EXEC_INVALID


def _inputs(shapes, kind, seed=1):
    """seeded U(-1, 1) arrays holding values a tensor of `kind` can hold exactly"""
    arrs = [seeded(s, seed + i, -1, 1) for i, s in enumerate(shapes)]
    return arrs if kind == abi.CCV_32F else [round16(a, kind) for a in arrs]


def _oracle(ref, cmd, ins, outs, kind):
    st, res = ref_exec(ref, cmd, None, 0, ins, outs)
    assert st == 0
    return [None if r is None else (r if kind == abi.CCV_32F else round16(r, kind)) for r in res]


def _gpu(nnc, cmd, ins, outs, kind):
    if kind == abi.CCV_32F:
        return gpu_exec(nnc, cmd, None, 0, ins, outs)
    return gpu_exec16(nnc, cmd, None, 0, ins, outs, kind)


def _z(shape):
    return np.zeros(shape, np.float32)


FORWARD_SHAPES = [
    ((20, 10), (20, 10)),                # cublas.tests.c "cmul in float"
    ((1, 5, 8, 128), (1, 5, 1, 128)),    # cublas.tests.c "cmul with broadcast"
    ((2, 64, 8, 64), (1, 64, 1, 64)),    # RoPE: [B, S, H, D] x [1, S, 1, D]
    ((4, 1, 6), (1, 3, 6)),              # both operands broadcast
    ((7, 12), (1, 12)),                  # 2-d
    ((3, 5, 16), (3, 1, 16)),            # 3-d
    ((4, 3, 18), (1, 3, 18)),            # last axis not a whole number of 16-byte vectors: one pair per thread
    ((2, 3, 130), (2, 1, 130)),
]


@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("sa,sb", FORWARD_SHAPES)
def test_cmul_forward(gpu, ref, sa, sb, kname):
    nnc, kind = gpu, KINDS[kname]
    a, b = _inputs((sa, sb), kind)
    sc = np.broadcast_shapes(sa, sb)
    (c_r,) = _oracle(ref, nnc.CMD_CMUL_FORWARD(), [a, b], [_z(sc)], kind)
    st, (c_g,) = _gpu(nnc, nnc.CMD_CMUL_FORWARD(), [a, b], [_z(sc)], kind)
    assert st == 0
    assert np.array_equal(c_g, c_r), (sa, sb, kname, np.abs(c_g - c_r).max())


# ---- strided views: q and k as slices of a packed [B, S, 16 * D] projection -------------------------------------------------
B, S, D, HQ, HK = 2, 32, 64, 8, 4
WIDTH = (HQ + 2 * HK) * D


class _Packed(object):
    """One packed [B, S, WIDTH] tensor of `kind` on the GPU and its CPU_REF twin (the values rounded to `kind`)."""

    def __init__(self, nnc, ref, host, kind):
        self.nnc, self.ref, self.kind, self.host = nnc, ref, kind, np.array(host, np.float32)  # a copy: CPU_REF writes into it
        self.t = nnc.gpu_tensor([B, S, WIDTH], NHWC, kind)
        self.t.upload(self.host if kind == abi.CCV_32F else pack16(self.host, kind))
        self.r = ref.RefTensor(self.host)
        self.gviews, self.rviews = [], []

    def view(self, heads, head0):
        """the [B, S, heads, D] slice starting at head `head0`"""
        dims, stride, ofs = [B, S, heads, D], [S * WIDTH, WIDTH, D, 1] + [0] * 8, [0, 0, 0, head0 * D] + [0] * 8
        g, r = self.nnc.tensor_view_new(self.t, dims, ofs, stride), self.r.view(dims, ofs, stride)
        self.gviews.append(g), self.rviews.append(r)
        return g, r

    def download(self):
        d = self.t.download()
        return d if self.kind == abi.CCV_32F else unpack16(d, self.kind)

    def free(self):
        for v in self.gviews + self.rviews + [self.t, self.r]:
            v.free()


def _table(kind, s=S, d=D):
    """the [1, s, 1, d] cos / sin table of theta = 10000 as complex pairs"""
    inv = 10000.0 ** (-np.arange(0, d, 2) / d)
    ang = np.arange(s)[:, None] * inv[None, :]
    t = np.stack([np.cos(ang), np.sin(ang)], -1).reshape(1, s, 1, d).astype(np.float32)
    return t if kind == abi.CCV_32F else round16(t, kind)


def _dense(nnc, ref, host, kind):
    t = nnc.gpu_tensor(list(host.shape), NHWC, kind)
    t.upload(host if kind == abi.CCV_32F else pack16(host, kind))
    return t, ref.RefTensor(host)


def _down(t, kind):
    d = t.download()
    return d if kind == abi.CCV_32F else unpack16(d, kind)


@pytest.mark.parametrize("kname", sorted(KINDS))
def test_cmul_views_and_in_place(gpu, ref, kname):
    nnc, kind = gpu, KINDS[kname]
    fwd = nnc.CMD_CMUL_FORWARD()
    (qkv,) = _inputs([(B, S, WIDTH)], kind, 11)
    table = _table(kind)
    tg, tr = _dense(nnc, ref, table, kind)
    stream = nnc.Stream(0)
    try:
        # 1. q and k slices into contiguous outputs
        p = _Packed(nnc, ref, qkv, kind)
        for heads, head0 in ((HQ, 0), (HK, HQ)):
            vg, vr = p.view(heads, head0)
            out = _z((B, S, heads, D))
            og, orr = _dense(nnc, ref, out.copy(), kind)
            assert ref.cmd_exec(fwd, None, 0, [vr, tr], [orr]) == 0
            assert nnc.cmd_exec(fwd, None, 0, [vg, tg], [og], stream) == 0, nnc.lib().ccv_nnc_sm100_last_error()
            stream.wait()
            want = orr.array if kind == abi.CCV_32F else round16(orr.array, kind)
            assert np.array_equal(_down(og, kind), want), (kname, heads)
            og.free(), orr.free()
        p.free()
        # 2. the k slice into the k slot of another packed tensor: everything outside the slot keeps its sentinel
        src = _Packed(nnc, ref, qkv, kind)
        dst = _Packed(nnc, ref, np.full((B, S, WIDTH), 7.0, np.float32), kind)
        kg, kr = src.view(HK, HQ)
        dg, dr = dst.view(HK, HQ)
        assert ref.cmd_exec(fwd, None, 0, [kr, tr], [dr]) == 0
        assert nnc.cmd_exec(fwd, None, 0, [kg, tg], [dg], stream) == 0
        stream.wait()
        got, want = dst.download(), dst.host if kind == abi.CCV_32F else round16(dst.host, kind)
        assert np.array_equal(got, want), kname
        slot = np.zeros(WIDTH, bool)
        slot[HQ * D:(HQ + HK) * D] = True
        assert (got[..., ~slot] == 7.0).all()
        src.free(), dst.free()
        # 3. in place on the q slice (c aliases a): the k and v columns are untouched
        p = _Packed(nnc, ref, qkv, kind)
        vg, vr = p.view(HQ, 0)
        assert ref.cmd_exec(fwd, None, 0, [vr, tr], [vr]) == 0
        assert nnc.cmd_exec(fwd, None, 0, [vg, tg], [vg], stream) == 0
        stream.wait()
        got, want = p.download(), p.host if kind == abi.CCV_32F else round16(p.host, kind)
        assert np.array_equal(got, want), kname
        assert np.array_equal(got[..., HQ * D:], qkv[..., HQ * D:])
        assert not np.array_equal(got[..., :HQ * D], qkv[..., :HQ * D])
        p.free()
    finally:
        tg.free(), tr.free(), stream.free()


# ---- backward ---------------------------------------------------------------------------------------------------------------
BACKWARD_SHAPES = [
    ((4, 6, 32), (4, 6, 32)),            # no broadcasting: every gradient on the full-shape kernel
    ((2, 16, 4, 64), (1, 16, 1, 64)),    # RoPE: da full shape, db (the table's gradient) reduced over B and H
    ((4, 1, 6), (1, 3, 6)),              # both gradients reduced
    ((3, 5, 18), (1, 5, 18)),            # scalar pairs in the full-shape kernel
]


@pytest.mark.parametrize("kname", sorted(KINDS))
@pytest.mark.parametrize("sa,sb", BACKWARD_SHAPES)
def test_cmul_backward(gpu, ref, sa, sb, kname):
    """Each form the reference accepts (both gradients; da from (g, b); db from (g, a)), with g and without it.  Without g CPU_REF
    returns conj(other) when nothing is broadcast but sums the other operand unconjugated when something is (:334-420); both pinned."""
    nnc, kind = gpu, KINDS[kname]
    sc = np.broadcast_shapes(sa, sb)
    g, a, b = _inputs((sc, sa, sb), kind, 5)
    bwd = nnc.CMD_CMUL_BACKWARD()
    for with_g in (1, 0):
        gg = g if with_g else None
        for form, ins, outs in (("da+db", [gg, a, b], lambda: [_z(sa), _z(sb)]), ("da", [gg, None, b], lambda: [_z(sa)]),
                                ("db", [gg, a, None], lambda: [None, _z(sb)])):
            want = _oracle(ref, bwd, ins, outs(), kind)
            st, got = _gpu(nnc, bwd, ins, outs(), kind)
            assert st == 0, (form, with_g)
            for w, x, name in zip(want, got, ("da", "db")):
                if w is not None:
                    assert np.array_equal(x, w), (sa, sb, kname, form, with_g, name, np.abs(x - w).max())
    # the quirk the comparisons above pin: without g, da is conj(b) when nothing is broadcast and b itself (summed) when it is
    (da0,) = _oracle(ref, bwd, [None, None, b], [_z(sa)], kind)
    if sa == sb:
        assert np.array_equal(da0[..., 0::2], b[..., 0::2]) and np.array_equal(da0[..., 1::2], -b[..., 1::2])
    elif sa == sc:
        assert np.array_equal(da0, np.broadcast_to(b, sa))


def test_cmul_backward_ignores_accumulate(gpu, ref):
    """CPU_REF zeroes the gradients and ignores CCV_NNC_ACCUMULATE_OUTPUT; so does this backend."""
    nnc = gpu
    sa, sb = (2, 16, 4, 64), (1, 16, 1, 64)
    g, a, b = _inputs((sa, sa, sb), abi.CCV_32F, 9)
    bwd = nnc.CMD_CMUL_BACKWARD()
    st_r, want = ref_exec(ref, bwd, None, abi.CCV_NNC_ACCUMULATE_OUTPUT, [g, a, b], [np.ones(sa, np.float32), np.ones(sb, np.float32)])
    st_g, got = gpu_exec(nnc, bwd, None, abi.CCV_NNC_ACCUMULATE_OUTPUT, [g, a, b], [np.ones(sa, np.float32), np.ones(sb, np.float32)])
    assert st_r == 0 and st_g == 0
    for w, x in zip(want, got):
        assert np.array_equal(x, w)


# ---- refusals ---------------------------------------------------------------------------------------------------------------
SENTINEL = 7.0


def _refused(nnc, cmd, ins, outs):
    """INVALID, no launch, and every output still holds the sentinel"""
    st, res, launches = counted(nnc, gpu_exec, cmd, None, 0, ins, outs)
    assert st == INVALID and launches == 0, (st, launches)
    for r in res:
        assert r is None or (r == SENTINEL).all()


def _s(shape, dtype=np.float32):
    return np.full(shape, SENTINEL, dtype)


def test_cmul_refusals(gpu):
    nnc = gpu
    fwd, bwd = nnc.CMD_CMUL_FORWARD(), nnc.CMD_CMUL_BACKWARD()
    r = lambda *s: seeded(s, 3, -1, 1)
    # more than 4 axes
    _refused(nnc, fwd, [r(1, 2, 2, 2, 4), r(1, 2, 2, 2, 4)], [_s((1, 2, 2, 2, 4))])
    # odd last axis; last axes that differ; shapes that do not broadcast; an output that is not the broadcast shape
    _refused(nnc, fwd, [r(4, 5), r(4, 5)], [_s((4, 5))])
    _refused(nnc, fwd, [r(4, 6), r(4, 8)], [_s((4, 6))])
    _refused(nnc, fwd, [r(4, 6), r(3, 6)], [_s((4, 6))])
    _refused(nnc, fwd, [r(4, 6), r(1, 6)], [_s((2, 6))])
    # mixed types
    _refused(nnc, fwd, [r(4, 6), r(4, 6).astype(np.float16)], [_s((4, 6))])
    _refused(nnc, bwd, [r(4, 6), r(4, 6), r(4, 6)], [_s((4, 6), np.float16), None])
    # a missing operand the requested gradient needs: da needs b, db needs a
    _refused(nnc, bwd, [r(4, 6), r(4, 6), None], [_s((4, 6)), None])
    _refused(nnc, bwd, [r(4, 6), None, r(4, 6)], [None, _s((4, 6))])
    # g that the operands do not broadcast onto
    _refused(nnc, bwd, [r(2, 6), r(4, 6), r(4, 6)], [_s((4, 6)), _s((4, 6))])
    # a palettized operand; a view whose last axis is not contiguous
    a, out = nnc.gpu_tensor([4, 64]).upload(r(4, 64)), nnc.gpu_tensor([4, 64]).upload(_s((4, 64)))
    q = nnc.gpu_palettized_tensor([4, 64], abi.CCV_32F, 4, 64)
    q.upload(np.zeros(q.nbytes, np.uint8))
    base = nnc.gpu_tensor([4, 128]).upload(r(4, 128))
    v = nnc.tensor_view_new(base, [4, 64], [0] * 12, [128, 2] + [0] * 10)
    try:
        for ins in ([a, q], [q, a], [v, a]):
            l0 = nnc.launch_count()
            assert nnc.cmd_exec(fwd, None, 0, ins, [out]) == INVALID and nnc.launch_count() == l0
            assert (out.download() == SENTINEL).all()
    finally:
        for t in (v, base, q, out, a):
            t.free()


# ---- a rotary decoder block through ccv_nnc_cmd_exec ------------------------------------------------------------------------
BB, SS, CC, BHQ, BHK, BD = 2, 128, 256, 4, 2, 64
QKV = (BHQ + 2 * BHK) * BD
ROWS = BB * SS


def _rms_cmd(cmd_id):
    c = _nnc._simple(cmd_id)
    c.info.rmsnorm.axis[0], c.info.rmsnorm.count, c.info.rmsnorm.epsilon = 1, 1, 1e-5
    return c


def _sdpa_cmd(cmd_id):
    c = _nnc._simple(cmd_id)
    c.info.scaled_dot_product_attention.scale, c.info.scaled_dot_product_attention.is_causal = 1.0 / np.sqrt(BD), 1
    return c


def _block_params(kind):
    """x, dy and the weights (RMSNORM scales, packed QKV, output, SwiGLU gate / up / down), values a `kind` tensor holds exactly"""
    shapes = dict(x=(ROWS, CC), g1=(1, CC), wqkv=(QKV, CC), wo=(CC, BHQ * BD), g2=(1, CC), w1=(2 * CC, CC), w3=(2 * CC, CC), w2=(CC, 2 * CC), dy=(ROWS, CC))
    p = {}
    for i, (k, s) in enumerate(sorted(shapes.items())):
        lo, hi = (0.5, 1.5) if k in ("g1", "g2") else (-1, 1)
        v = seeded(s, 40 + i, lo, hi)
        if k.startswith("w"):
            v = (v / np.sqrt(s[1])).astype(np.float32)
        p[k] = v if kind == abi.CCV_32F else round16(v, kind)
    p["table"] = _table(kind, SS, BD)
    return p


def _block_cpu_ref(nnc, ref, p):
    """the block on CPU_REF in fp32; returns {name: array} of y, dx and every weight gradient"""
    def run(cmd, ins, outs):
        st, res = ref_exec(ref, cmd, None, 0, ins, outs)
        assert st == 0, cmd.cmd
        return res
    gemm, gemm_b = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1)), nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
    add, fwd, bwd = nnc.CMD_ADD_FORWARD(1.0, 1.0), nnc.CMD_CMUL_FORWARD(), nnc.CMD_CMUL_BACKWARD()
    h1, r1 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD), [p["x"], p["g1"]], [_z((ROWS, CC)), _z((ROWS, 1))])
    (qkv,) = run(gemm, [h1, p["wqkv"]], [_z((ROWS, QKV))])
    q4 = qkv.reshape(BB, SS, QKV)
    q = np.ascontiguousarray(q4[..., :BHQ * BD]).reshape(BB, SS, BHQ, BD)
    k = np.ascontiguousarray(q4[..., BHQ * BD:(BHQ + BHK) * BD]).reshape(BB, SS, BHK, BD)
    v = np.ascontiguousarray(q4[..., (BHQ + BHK) * BD:]).reshape(BB, SS, BHK, BD)
    (qr,) = run(fwd, [q, p["table"]], [_z(q.shape)])
    (kr,) = run(fwd, [k, p["table"]], [_z(k.shape)])
    o, _ = run(_sdpa_cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD), [qr, kr, v], [_z(qr.shape), None])
    o2 = o.reshape(ROWS, BHQ * BD)
    (a,) = run(gemm, [o2, p["wo"]], [_z((ROWS, CC))])
    (x1,) = run(add, [p["x"], a], [_z((ROWS, CC))])
    h2, r2 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD), [x1, p["g2"]], [_z((ROWS, CC)), _z((ROWS, 1))])
    (u,) = run(gemm, [h2, p["w1"]], [_z((ROWS, 2 * CC))])
    (v3,) = run(gemm, [h2, p["w3"]], [_z((ROWS, 2 * CC))])
    (su,) = run(nnc.CMD_SWISH_FORWARD(), [u], [_z(u.shape)])
    (m,) = run(nnc.CMD_MUL_FORWARD(1.0), [su, v3], [_z(u.shape)])
    (dn,) = run(gemm, [m, p["w2"]], [_z((ROWS, CC))])
    (y,) = run(add, [x1, dn], [_z((ROWS, CC))])
    dy = p["dy"]
    dm, dw2 = run(gemm_b, [dy, m, p["w2"]], [_z(m.shape), _z(p["w2"].shape)])
    dsu, dv3 = run(nnc.CMD_MUL_BACKWARD(1.0), [dm, su, v3], [_z(u.shape), _z(u.shape)])
    (du,) = run(nnc.CMD_SWISH_BACKWARD(), [dsu, u, su], [_z(u.shape)])
    dh2a, dw1 = run(gemm_b, [du, h2, p["w1"]], [_z(h2.shape), _z(p["w1"].shape)])
    dh2b, dw3 = run(gemm_b, [dv3, h2, p["w3"]], [_z(h2.shape), _z(p["w3"].shape)])
    (dh2,) = run(add, [dh2a, dh2b], [_z(h2.shape)])
    dx1n, dg2 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD), [dh2, None, x1, p["g2"], None, r2], [_z(x1.shape), _z(p["g2"].shape)])
    (dx1,) = run(add, [dy, dx1n], [_z(x1.shape)])
    do2, dwo = run(gemm_b, [dx1, o2, p["wo"]], [_z(o2.shape), _z(p["wo"].shape)])
    dqr, dkr, dv = run(_sdpa_cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD), [do2.reshape(o.shape), None, None, qr, kr, v], [_z(qr.shape), _z(kr.shape), _z(v.shape)])
    (dq,) = run(bwd, [dqr, None, p["table"]], [_z(q.shape)])
    (dk,) = run(bwd, [dkr, None, p["table"]], [_z(k.shape)])
    dqkv = np.concatenate([dq.reshape(BB, SS, -1), dk.reshape(BB, SS, -1), dv.reshape(BB, SS, -1)], -1).reshape(ROWS, QKV)
    dh1, dwqkv = run(gemm_b, [dqkv, h1, p["wqkv"]], [_z(h1.shape), _z(p["wqkv"].shape)])
    dxn, dg1 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD), [dh1, None, p["x"], p["g1"], None, r1], [_z(h1.shape), _z(p["g1"].shape)])
    (dx,) = run(add, [dx1, dxn], [_z(h1.shape)])
    return dict(y=y, dx=dx, dg1=dg1, dwqkv=dwqkv, dwo=dwo, dg2=dg2, dw1=dw1, dw3=dw3, dw2=dw2)


class _GpuBlock(object):
    """the same block on CCV_NNC_BACKEND_GPU_SM100: GEMMs, CMUL, SDPA, SWISH and MUL on `kind` tensors; the residual stream and RMSNORM
    in fp32 (DATATYPE_CONVERSION between them when `kind` is 16-bit).  q, k and v are views of the packed QKV output; dq, dk and dv are
    written into the matching views of one packed gradient."""

    def __init__(self, nnc, kind):
        self.nnc, self.kind, self.stream, self.owned = nnc, kind, nnc.Stream(0), []

    def new(self, shape, dt=None, ptr=None):
        t = self.nnc.gpu_tensor(list(shape), NHWC, self.kind if dt is None else dt, ptr=ptr)
        self.owned.append(t)
        return t

    def up(self, arr, dt):
        t = self.new(arr.shape, dt)
        t.upload(arr if dt == abi.CCV_32F else pack16(arr, dt))
        return t

    def heads(self, packed, heads, head0):
        t = self.nnc.tensor_view_new(packed, [BB, SS, heads, BD], [0, 0, 0, head0 * BD] + [0] * 8, [SS * QKV, QKV, BD, 1] + [0] * 8)
        self.owned.append(t)
        return t

    def run(self, cmd, ins, outs):
        assert self.nnc.cmd_exec(cmd, None, 0, ins, outs, self.stream) == 0, (hex(cmd.cmd), self.nnc.lib().ccv_nnc_sm100_last_error())
        return outs

    def to(self, t, dt):
        if (t.params.datatype & 0xFF000) == dt:
            return t
        return self.run(self.nnc.CMD_DATATYPE_CONVERSION_FORWARD(), [t], [self.new(t.dims, dt)])[0]

    def down(self, t):
        self.stream.wait()
        d = t.download()
        return d if (t.params.datatype & 0xFF000) == abi.CCV_32F else unpack16(d, t.params.datatype & 0xFF000)

    def free(self):
        self.stream.wait()
        for t in reversed(self.owned):
            t.free()
        self.stream.free()

    def __call__(self, p):
        nnc, K, F = self.nnc, self.kind, abi.CCV_32F
        run, new, to = self.run, self.new, self.to
        gemm, gemm_b = nnc.CMD_GEMM_FORWARD(transpose_b=(0, 1)), nnc.CMD_GEMM_BACKWARD((0, 0), (0, 1))
        add, fwd, bwd = nnc.CMD_ADD_FORWARD(1.0, 1.0), nnc.CMD_CMUL_FORWARD(), nnc.CMD_CMUL_BACKWARD()
        x, g1, g2, dy = (self.up(p[k], F) for k in ("x", "g1", "g2", "dy"))
        wqkv, wo, w1, w3, w2, table = (self.up(p[k], K) for k in ("wqkv", "wo", "w1", "w3", "w2", "table"))
        h1, r1 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD), [x, g1], [new((ROWS, CC), F), new((ROWS, 1), F)])
        h1k = to(h1, K)
        (qkv,) = run(gemm, [h1k, wqkv], [new((ROWS, QKV))])
        qkv3 = new((BB, SS, QKV), ptr=qkv.data_ptr)
        q, k, v = self.heads(qkv3, BHQ, 0), self.heads(qkv3, BHK, BHQ), self.heads(qkv3, BHK, BHQ + BHK)
        (qr,) = run(fwd, [q, table], [new((BB, SS, BHQ, BD))])
        (kr,) = run(fwd, [k, table], [new((BB, SS, BHK, BD))])
        (o,) = run(_sdpa_cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD), [qr, kr, v], [new((BB, SS, BHQ, BD)), None])[:1]
        o2 = new((ROWS, BHQ * BD), ptr=o.data_ptr)
        (a,) = run(gemm, [o2, wo], [new((ROWS, CC))])
        (x1,) = run(add, [x, to(a, F)], [new((ROWS, CC), F)])
        h2, r2 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_FORWARD), [x1, g2], [new((ROWS, CC), F), new((ROWS, 1), F)])
        h2k = to(h2, K)
        (u,) = run(gemm, [h2k, w1], [new((ROWS, 2 * CC))])
        (v3,) = run(gemm, [h2k, w3], [new((ROWS, 2 * CC))])
        (su,) = run(nnc.CMD_SWISH_FORWARD(), [u], [new(u.dims)])
        (m,) = run(nnc.CMD_MUL_FORWARD(1.0), [su, v3], [new(u.dims)])
        (dn,) = run(gemm, [m, w2], [new((ROWS, CC))])
        (y,) = run(add, [x1, to(dn, F)], [new((ROWS, CC), F)])
        dm, dw2 = run(gemm_b, [to(dy, K), m, w2], [new(m.dims), new(w2.dims)])
        dsu, dv3 = run(nnc.CMD_MUL_BACKWARD(1.0), [dm, su, v3], [new(u.dims), new(u.dims)])
        (du,) = run(nnc.CMD_SWISH_BACKWARD(), [dsu, u, su], [new(u.dims)])
        dh2a, dw1 = run(gemm_b, [du, h2k, w1], [new(h2.dims), new(w1.dims)])
        dh2b, dw3 = run(gemm_b, [dv3, h2k, w3], [new(h2.dims), new(w3.dims)])
        (dh2,) = run(add, [dh2a, dh2b], [new(h2.dims)])
        dx1n, dg2 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD), [to(dh2, F), None, x1, g2, None, r2], [new(x1.dims, F), new(g2.dims, F)])
        (dx1,) = run(add, [dy, dx1n], [new(x1.dims, F)])
        do2, dwo = run(gemm_b, [to(dx1, K), o2, wo], [new(o2.dims), new(wo.dims)])
        do = new((BB, SS, BHQ, BD), ptr=do2.data_ptr)
        dqkv = new((ROWS, QKV))
        dqkv3 = new((BB, SS, QKV), ptr=dqkv.data_ptr)
        dq, dk, dv = self.heads(dqkv3, BHQ, 0), self.heads(dqkv3, BHK, BHQ), self.heads(dqkv3, BHK, BHQ + BHK)
        dqr, dkr = new(qr.dims), new(kr.dims)
        run(_sdpa_cmd(abi.CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD), [do, None, None, qr, kr, v], [dqr, dkr, dv])
        run(bwd, [dqr, None, table], [dq])
        run(bwd, [dkr, None, table], [dk])
        dh1, dwqkv = run(gemm_b, [dqkv, h1k, wqkv], [new(h1.dims), new(wqkv.dims)])
        dxn, dg1 = run(_rms_cmd(abi.CCV_NNC_RMSNORM_BACKWARD), [to(dh1, F), None, x, g1, None, r1], [new(x.dims, F), new(g1.dims, F)])
        (dx,) = run(add, [dx1, dxn], [new(x.dims, F)])
        out = dict(y=y, dx=dx, dg1=dg1, dwqkv=dwqkv, dwo=dwo, dg2=dg2, dw1=dw1, dw3=dw3, dw2=dw2)
        return dict((name, self.down(t)) for name, t in out.items())


@pytest.mark.parametrize("kname", ["fp32", "bf16"])
def test_rotary_decoder_block(gpu, ref, kname):
    """A pre-norm rotary decoder block, x [2, 128, 256], Hq = 4, Hk = 2, D = 64: RMSNORM, packed QKV GEMM [512, 256], CMUL of the q and k
    views by a theta = 10000 table, causal GQA SDPA, output GEMM and residual ADD, RMSNORM, SwiGLU MLP (GEMMs [512, 256] x 2, SWISH, MUL,
    GEMM [256, 512]) and residual ADD; then the backward from a seeded dy to dx and every weight gradient.  Each output is compared with
    the same commands on CPU_REF in fp32, relative to max|ref|.

    fp32: <= 1e-3.  The GEMMs run 3xTF32 (fp32-grade), the attention's GEMMs one-pass TF32, whose products carry a relative error of about
    2^-11 ~ 5e-4 each; the softmax and the output projection average them down (DESIGN §5 records 6e-5 to 4e-4).
    bf16 (16-bit GEMMs, flash attention forward and backward, CMUL, SWISH, MUL; RMSNORM and the residual stream in fp32): the oracle is
    fp32 CPU_REF on the same bf16-rounded inputs and weights, so what is measured is the rounding of the intermediates.  Each command's
    output is rounded to bf16 once (relative error <= 2^-9 ~ 2e-3), and the attention rounds P to bf16 before P V.  The forward passes
    through about 8 such roundings between x and y; the longest backward path (dy -> MLP -> RMSNORM -> attention -> QKV GEMM -> dx) through
    about 14.  Independent roundings add like a random walk, sqrt(14) * 2e-3 ~ 8e-3, and products of large sums (the weight gradients,
    sums over 256 rows) can cancel, which raises an error relative to max|ref| by a small factor: 3e-2 keeps a factor of about 3 of margin."""
    nnc, kind = gpu, KINDS[kname]
    p = _block_params(kind)
    want = _block_cpu_ref(nnc, ref, p)
    blk = _GpuBlock(nnc, kind)
    try:
        got = blk(p)
    finally:
        blk.free()
    bound = 1e-3 if kind == abi.CCV_32F else 3e-2
    errs = dict((k, rel_err(got[k], want[k])) for k in want)
    print("rotary decoder block %s: max error / max|ref| %s" % (kname, ", ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    for name, e in errs.items():
        assert np.isfinite(got[name]).all() and e <= bound, (kname, name, e, errs)
