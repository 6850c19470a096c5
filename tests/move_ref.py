"""Exact oracles for the commands that only move or resample data: DATA_TRANSFER, FORMAT_TRANSFORM, TRANSPOSE, DATATYPE_CONVERSION,
INDEX_SELECT and UPSAMPLE, restated from the reference's CPU_REF (util/ccv_nnc_util_cpu_ref.c, lib/ccv_util.c:1434-1453,
index/ccv_nnc_index_select_cpu_ref.c, upsample/ccv_nnc_upsample_cpu_ref.c) in numpy with the reference's own arithmetic: double where
it computes in double, float elsewhere, in its association and summation order.  tests/golden/cpuref_move.npz pins these to CPU_REF.

Every result here is exact, so the GPU must reproduce it bit for bit."""
import numpy as np

f32 = np.float32


def view(buf, ofs, dims, strides):
    """the elements a tensor view of `buf` (flat) names: offset `ofs`, element strides `strides`"""
    buf = np.asarray(buf)
    return np.lib.stride_tricks.as_strided(buf[ofs:], shape=tuple(dims), strides=tuple(s * buf.itemsize for s in strides), writeable=False)


def transpose(a, ax0, ax1):
    """TRANSPOSE: b[..., i, ..., j, ...] = a[..., j, ..., i, ...]"""
    return np.ascontiguousarray(np.swapaxes(a, ax0, ax1))


def nhwc_to_nchw(a):
    return np.ascontiguousarray(np.moveaxis(a, -1, -3))


def nchw_to_nhwc(a):
    return np.ascontiguousarray(np.moveaxis(a, -3, -1))


# ---- datatype conversion ------------------------------------------------------------------------------------------------------------
def _half_tables():
    """lib/ccv_util.c's _ccv_base_table / _ccv_shift_table, indexed by the float's sign and exponent (9 bits)"""
    base, shift = np.zeros(512, np.uint32), np.zeros(512, np.uint32)
    for i in range(256):
        e = i - 127
        if e < -24:
            b, s = 0, 24
        elif e < -14:
            b, s = 0x0400 >> (-e - 14), -e - 1
        elif e <= 15:
            b, s = (e + 15) << 10, 13
        elif e < 128:
            b, s = 0x7C00, 24
        else:
            b, s = 0x7C00, 13
        base[i], base[i | 0x100], shift[i], shift[i | 0x100] = b, b | 0x8000, s, s
    return base, shift


_BASE, _SHIFT = _half_tables()


def f32_to_f16(x):
    """ccv_float_to_half_precision: the truncating table conversion (a NaN whose payload sits only in the low 13 bits becomes Inf)"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    k = (u >> 23) & 0x1FF
    return (_BASE[k] + ((u & 0x007FFFFF) >> _SHIFT[k])).astype(np.uint16)


def f64_to_f16(x):
    """ccv_double_to_half_precision: round to float, then the same table"""
    with np.errstate(over="ignore"):
        return f32_to_f16(np.asarray(x, np.float64).astype(np.float32))


def f16_to_f32(h):
    """exact"""
    return np.ascontiguousarray(h, np.uint16).view(np.float16).astype(np.float32)


def f32_to_bf16(x):
    """round to nearest even on the bits (tests/util.pack16); defined for non-NaN x only (a NaN must stay a NaN)"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16).reshape(np.shape(x))


def bf16_to_f32(h):
    return (np.ascontiguousarray(h, np.uint16).astype(np.uint32) << 16).view(np.float32)


def f16_specials():
    """the values where a float -> half conversion goes wrong: zeros, f32 and f16 subnormal boundaries, the top of the f16 range
    (65504 is the largest half, 65519 still truncates to it, 65520 rounds to Inf under round-to-nearest), infinities and NaNs
    with high and with low payloads"""
    v = [0.0, -0.0, 1.0, -1.0, 0.1, -2.5, 1e-45, 1e-40, 2.0 ** -126, -(2.0 ** -126), 2.0 ** -149,
         2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -24 * 1.9, 2.0 ** -14, 2.0 ** -14 * (1 - 2.0 ** -11), 2.0 ** -15, -(2.0 ** -20) * 3,
         65504.0, -65504.0, 65519.0, 65519.99, 65520.0, -65520.0, 65536.0, 1e10, -1e10, 3.4e38,
         1 + 2.0 ** -11, 1 + 2.0 ** -10 + 2.0 ** -11, 2049.0, 2051.0, 0.33333334]
    x = np.array(v, np.float32)
    bits = np.array([0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7F801FFF, 0xFF800FFF, 0x7F802000, 0x7FFFFFFF,
                     0x7FA00000, 0x00000001, 0x807FFFFF, 0x00400000, 0x33000000, 0x33000001, 0x387FE000, 0x387FFFFF, 0x477FE000,
                     0x477FEFFF, 0x477FF000, 0x477FFFFF], np.uint32).view(np.float32)
    return np.concatenate([x, bits])


# ---- index select -------------------------------------------------------------------------------------------------------------------
def index_select(a, idx, b=None):
    """32S indices: b[i] = a[idx[i]]; an index outside [0, rows) leaves b's row as it was"""
    b = np.zeros((len(idx),) + a.shape[1:], a.dtype) if b is None else b.copy()
    for i, j in enumerate(idx):
        if 0 <= j < a.shape[0]:
            b[i] = a[j]
    return b


def index_select_lerp(a, fidx):
    """32F indices (index_select_cpu_ref.c:47-63): rows j0 = (int)f and min(j0 + 1, rows - 1), b = a0 * w0 + a1 * w1, all in float"""
    a = np.asarray(a, np.float32)
    b = np.zeros((len(fidx),) + a.shape[1:], np.float32)
    for i, f in enumerate(np.asarray(fidx, np.float32)):
        j0 = int(f)
        j1 = min(j0 + 1, a.shape[0] - 1)
        w1 = f32(f - f32(j0))
        w0 = f32(f32(1) - w1)
        b[i] = (a[j0] * w0) + (a[j1] * w1)
    return b


def index_select_back(g, idx, rows):
    """h[r] = sum of g[i] over idx[i] == r, in increasing i, accumulated in float (the 16-bit forms round the float sum once)"""
    g = np.asarray(g, np.float32)
    h = np.zeros((rows,) + g.shape[1:], np.float32)
    for i, j in enumerate(idx):
        h[j] = h[j] + g[i]
    return h


# ---- upsample -----------------------------------------------------------------------------------------------------------------------
def ratio(i, o, align):
    """rheight / rwidth: float"""
    return f32(f32(i - 1) / f32(max(1, o - 1))) if align else f32(f32(i) / f32(o))


def nearest_index(i, o, align, double=True):
    """the source row / column of each output one: (int)((x + 0.5) * r) or (int)(x * r + 0.5), both in double with r and x * r in
    float (upsample_cpu_ref.c:48,62).  double=False is the float-only arithmetic, a defect the tests show the bound catches."""
    r = ratio(i, o, align)
    x = np.arange(o)
    if not double:
        s = (x.astype(np.float32) * r + f32(0.5)) if align else ((x.astype(np.float32) + f32(0.5)) * r)
    elif align:
        s = (x.astype(np.float32) * r).astype(np.float64) + 0.5
    else:
        s = (x + 0.5) * np.float64(r)
    return np.minimum(s.astype(np.int64), i - 1)


def bilinear_coeffs(i, o, align):
    """_ccv_nnc_init_bi_coeffs (upsample_cpu_ref.c:220-243): (si0, si1, sc0, sc1) per output row / column"""
    r = ratio(i, o, align)
    x = np.arange(o)
    if align:
        xs = x.astype(np.float32) * r
    else:
        xs = ((x + 0.5) * np.float64(r) - 0.5).astype(np.float32)
    si0 = xs.astype(np.int64)  # truncation toward zero: xs in (-1, 0) gives 0 and a negative sc1
    si1 = np.minimum((xs + f32(1)).astype(np.int64), i - 1)
    sc1 = (xs - si0.astype(np.float32)).astype(np.float32)
    sc0 = (f32(1) - sc1).astype(np.float32)
    return si0, si1, sc0, sc1


def _to_nchw(a, nchw):
    """(n, c, h, w) float32 view of a 3-d or 4-d NHWC / NCHW tensor"""
    a = np.asarray(a, np.float32)
    if a.ndim == 3:
        a = a[None]
    return a if nchw else np.moveaxis(a, 3, 1)


def _from_nchw(x, nchw, nd):
    x = x if nchw else np.moveaxis(x, 1, 3)
    return np.ascontiguousarray(x[0] if nd == 3 else x)


def upsample_forward(a, oh, ow, bilinear, align, nchw):
    """b of the reference's upsample forward; a 3-d / 4-d, NHWC or NCHW"""
    x = _to_nchw(a, nchw)
    H, W = x.shape[2], x.shape[3]
    if not bilinear:
        yi, xi = nearest_index(H, oh, align), nearest_index(W, ow, align)
        return _from_nchw(x[:, :, yi][:, :, :, xi], nchw, np.ndim(a))
    ys0, ys1, ysc0, ysc1 = bilinear_coeffs(H, oh, align)
    xs0, xs1, xsc0, xsc1 = bilinear_coeffs(W, ow, align)
    rows0, rows1 = x[:, :, ys0], x[:, :, ys1]
    a00, a01, a10, a11 = rows0[..., xs0], rows0[..., xs1], rows1[..., xs0], rows1[..., xs1]
    yc0, yc1 = ysc0[:, None], ysc1[:, None]
    if nchw:
        # ap1[si0] * sc0 * ysc0 + ...: ((a * xsc) * ysc)
        t = [(a00 * xsc0) * yc0, (a01 * xsc1) * yc0, (a10 * xsc0) * yc1, (a11 * xsc1) * yc1]
    else:
        # c00 = sc0 * ysc0; ap00 * c00 + ...
        t = [a00 * (xsc0 * yc0), a01 * (xsc1 * yc0), a10 * (xsc0 * yc1), a11 * (xsc1 * yc1)]
    return _from_nchw(((t[0] + t[1]) + t[2]) + t[3], nchw, np.ndim(a))


def upsample_backward(g, h, w, bilinear, align, nchw, order=None):
    """h of the reference's upsample backward: zeroed, then every output pixel's gradient added in output raster order (the four
    bilinear corners 00, 01, 10, 11 in turn), in float.  order: a permutation of the raster (a defect the tests show the bound
    catches)."""
    y = _to_nchw(g, nchw)
    OH, OW = y.shape[2], y.shape[3]
    out = np.zeros(y.shape[:2] + (h, w), np.float32)
    pix = [(yd, xd) for yd in range(OH) for xd in range(OW)]
    if order is not None:
        pix = [pix[k] for k in order]
    if not bilinear:
        yi, xi = nearest_index(h, OH, align), nearest_index(w, OW, align)
        for yd, xd in pix:
            out[:, :, yi[yd], xi[xd]] += y[:, :, yd, xd]
        return _from_nchw(out, nchw, np.ndim(g))
    ys0, ys1, ysc0, ysc1 = bilinear_coeffs(h, OH, align)
    xs0, xs1, xsc0, xsc1 = bilinear_coeffs(w, OW, align)
    for yd, xd in pix:
        v = y[:, :, yd, xd]
        for sy, cy in ((ys0[yd], ysc0[yd]), (ys1[yd], ysc1[yd])):
            for sx, cx in ((xs0[xd], xsc0[xd]), (xs1[xd], xsc1[xd])):
                # NCHW: bp1[xd] * ysc * sc (upsample_cpu_ref.c:425-428); NHWC: bp1[cd] * (sc * ysc) (:468-481)
                out[:, :, sy, sx] += (v * cy) * cx if nchw else v * f32(cx * cy)
    return _from_nchw(out, nchw, np.ndim(g))
