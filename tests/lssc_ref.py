"""COMPRESSION_LSSC restated in numpy, in CPU_REF's order (lib/nnc/cmd/compression/ccv_nnc_lssc_cpu_ref.c of the reference).

Each (n, c) plane is cut into 4x4 blocks; a block becomes 4 halves.
  forward   cells past the bottom / right edge take the block's first cell.  min / max are the scans `a > m ? a : m` / `a < m ? a : m`
            from cell 0 (ccv_max / ccv_min: a NaN cell 0 makes both NaN, a later NaN is ignored, of +0 / -0 the earlier stays), stored as
            the selected cell's own bits.  abottom = min * 7 / 6 - max / 6 (float); ascale = (float)(3.0 / max((double)(max - min), 1e-6))
            (a NaN range gives 1e-6); code = clamp((int)((a - abottom) * ascale), 0, 3), truncating, a NaN product giving 0.  Cells 0-7
            go into half 2 and 8-15 into half 3, cell c at bits 2 (c mod 8).
  backward  levels min, max / 3 + min * 2 / 3, max * 2 / 3 + min / 3, max (float), the middle two narrowed with the reference's
            truncating f32 -> f16 table; a cell inside the original tensor gets level[code].  A NaN middle level has the bits x86-64
            SSE gives it (see mid_level).

Arrays are fp16 bit patterns (uint16).  NCHW is [N, C, H, W] or [C, H, W]; NHWC is [N, H, W, C] or [H, W, C], restated as the NCHW
transpose.  `defect` switches in one plausible kernel mistake, for the tests that show the CPU_REF fixture tells it apart."""
import numpy as np

NCHW, NHWC = "NCHW", "NHWC"
DEFECTS = ("fmax_scan", "zero_pad", "double_ascale", "rn_levels", "codes_high_to_low")


def compressed_shape(shape, fmt):
    s = list(shape)
    hw = len(s) - 2 if fmt == NCHW else len(s) - 3
    s[hw], s[hw + 1] = (s[hw] + 3) // 4, (s[hw + 1] + 3) // 4 * 4
    return tuple(s)


def f16_bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float16)).view(np.uint16)


def _f32(bits):
    return np.asarray(bits, np.uint16).view(np.float16).astype(np.float32)


def f32_to_f16_trunc(f):
    """lib/ccv_util.c:1434-1440: the base / shift tables, i.e. the mantissa truncated, below 2^-24 to signed zero, >= 2^16 to inf, NaN
    keeping its top mantissa bits"""
    u = np.ascontiguousarray(f, np.float32).view(np.uint32).astype(np.int64)
    sign = (u >> 16) & 0x8000
    e = ((u >> 23) & 0xff) - 127
    m = u & 0x7fffff
    sub = np.where((e >= -24) & (e < -14), (0x400 >> np.clip(-e - 14, 0, 31)) + (m >> np.clip(-e - 1, 0, 63)), 0)
    out = np.select([e < -24, e < -14, e <= 15, e < 128], [0, sub, ((e + 15) << 10) + (m >> 13), 0x7c00], 0x7c00 + (m >> 13))
    return (sign | out).astype(np.uint16)


def _is_nan16(h):
    return (np.asarray(h, np.uint16) & 0x7fff) > 0x7c00


def mid_level(v, lo, hi):
    """The fp16 bits of a middle level v (float32) = t1 + t2 with t1 from hi and t2 from lo.  Not NaN: the truncating narrowing.  NaN,
    as x86-64 SSE makes it in CPU_REF: a NaN operand propagates quieted (fp16 NaN bits h come back as h | 0x200), hi's when both are
    NaN (the first operand of the addition); Inf - Inf with no NaN operand is the default NaN 0xffc00000, 0xfe00 as fp16."""
    nan = np.where(_is_nan16(hi), hi | 0x200, np.where(_is_nan16(lo), lo | 0x200, 0xfe00)).astype(np.uint16)
    return np.where(np.isnan(v), nan, f32_to_f16_trunc(v))


def _planes(x, fmt):
    """-> (P, H, W) planes of an NCHW / NHWC array, and the function that puts planes of another width / height back"""
    x = np.asarray(x)
    if fmt == NHWC:
        lead = x.shape[:-3]
        t = np.moveaxis(x, -1, -3)  # [.., C, H, W]
        back = lambda p: np.ascontiguousarray(np.moveaxis(p.reshape(lead + (x.shape[-1],) + p.shape[-2:]), -3, -1))
    else:
        t = x
        back = lambda p: np.ascontiguousarray(p.reshape(x.shape[:-2] + p.shape[-2:]))
    return np.ascontiguousarray(t).reshape((-1,) + t.shape[-2:]), back


def _blocks(p, pad_with_first=True):
    """(P, H, W) -> (P, Hb, Wb, 16) cells in row-major order, and the validity mask"""
    P, H, W = p.shape
    Hb, Wb = (H + 3) // 4, (W + 3) // 4
    full = np.zeros((P, 4 * Hb, 4 * Wb), p.dtype)
    full[:, :H, :W] = p
    valid = np.zeros((4 * Hb, 4 * Wb), bool)
    valid[:H, :W] = True
    cells = full.reshape(P, Hb, 4, Wb, 4).transpose(0, 1, 3, 2, 4).reshape(P, Hb, Wb, 16)
    mask = valid.reshape(Hb, 4, Wb, 4).transpose(0, 2, 1, 3).reshape(Hb, Wb, 16)
    if pad_with_first:
        cells = np.where(mask, cells, cells[..., :1])
    return cells, mask


def encode_blocks(h, defect=None):
    """h: (..., 16) fp16 bits -> (..., 4) fp16 bits (min, max, codes of cells 0-7, codes of cells 8-15)"""
    h = np.asarray(h, np.uint16)
    a = _f32(h)
    with np.errstate(invalid="ignore", over="ignore"):
        amax, amin, hmax, hmin = a[..., 0].copy(), a[..., 0].copy(), h[..., 0].copy(), h[..., 0].copy()
        for c in range(1, 16):
            if defect == "fmax_scan":  # fmaxf / fminf: a NaN running value is replaced
                gt = (a[..., c] > amax) | (np.isnan(amax) & ~np.isnan(a[..., c]))
                lt = (a[..., c] < amin) | (np.isnan(amin) & ~np.isnan(a[..., c]))
            else:
                gt, lt = a[..., c] > amax, a[..., c] < amin
            amax, hmax = np.where(gt, a[..., c], amax), np.where(gt, h[..., c], hmax)
            amin, hmin = np.where(lt, a[..., c], amin), np.where(lt, h[..., c], hmin)
        abottom = (amin * np.float32(7)) / np.float32(6) - amax / np.float32(6)
        rng = (amax - amin).astype(np.float64)
        ascale64 = 3.0 / np.where(rng > 1e-6, rng, 1e-6)
        if defect == "double_ascale":  # ascale kept in double, the product taken in double
            prod = (a - abottom[..., None]).astype(np.float64) * ascale64[..., None]
        else:
            prod = (a - abottom[..., None]) * ascale64.astype(np.float32)[..., None]
        # x86-64 truncates a NaN to INT_MIN and CUDA to 0, which clamp alike, and any finite product of magnitude below 2^31 truncates
        # alike.  A block of range > 0 gives about [0.5, 3.5]; an all-equal block gives (a - abottom) * 3e6 with abottom a rounding step
        # away from a, at most 11718.75 in magnitude over every fp16 value (either sign, so the codes of such a block are 0 or 3)
        assert defect or np.all(np.isnan(prod) | (np.abs(prod) < 2 ** 14)), "an LSSC code product beyond 2^14"
        k = np.clip(np.trunc(np.where(np.isnan(prod), 0, prod)), 0, 3).astype(np.uint32)
    shift = (2 * (7 - np.arange(8)) if defect == "codes_high_to_low" else 2 * np.arange(8)).astype(np.uint32)
    lo_codes = (k[..., :8] << shift).sum(-1).astype(np.uint16)
    hi_codes = (k[..., 8:] << shift).sum(-1).astype(np.uint16)
    return np.stack([hmin, hmax, lo_codes, hi_codes], -1).astype(np.uint16)


def decode_blocks(q, defect=None):
    """q: (..., 4) fp16 bits -> (..., 16) fp16 bits"""
    q = np.asarray(q, np.uint16)
    lo, hi = _f32(q[..., 0]), _f32(q[..., 1])
    with np.errstate(invalid="ignore", over="ignore"):
        v1 = hi / np.float32(3) + (lo * np.float32(2)) / np.float32(3)
        v2 = (hi * np.float32(2)) / np.float32(3) + lo / np.float32(3)
    if defect == "rn_levels":
        l1, l2 = v1.astype(np.float16).view(np.uint16), v2.astype(np.float16).view(np.uint16)
    else:
        l1, l2 = mid_level(v1, q[..., 0], q[..., 1]), mid_level(v2, q[..., 0], q[..., 1])
    levels = np.stack([q[..., 0], l1, l2, q[..., 1]], -1)
    shift = 2 * (7 - np.arange(8)) if defect == "codes_high_to_low" else 2 * np.arange(8)
    codes = np.concatenate([(q[..., 2:3].astype(np.int64) >> shift) & 3, (q[..., 3:4].astype(np.int64) >> shift) & 3], -1)
    return np.take_along_axis(levels, codes, -1).astype(np.uint16)


def forward(x, fmt=NCHW, defect=None):
    """fp16 bits of the original -> fp16 bits of the compressed tensor"""
    p, back = _planes(np.asarray(x, np.uint16), fmt)
    P, H, W = p.shape
    cells, _ = _blocks(p, pad_with_first=defect != "zero_pad")
    q = encode_blocks(cells, defect)  # (P, Hb, Wb, 4)
    return back(q.reshape(P, q.shape[1], -1))


def backward(y, shape, fmt=NCHW, defect=None):
    """fp16 bits of the compressed tensor -> fp16 bits of the original (shape), every cell of which is some block's cell"""
    p0, back = _planes(np.zeros(shape, np.uint16), fmt)
    P, H, W = p0.shape
    yp, _ = _planes(np.asarray(y, np.uint16), fmt)
    Hb, Wb = (H + 3) // 4, (W + 3) // 4
    cells = decode_blocks(yp.reshape(P, Hb, Wb, 4), defect)  # (P, Hb, Wb, 16)
    full = cells.reshape(P, Hb, Wb, 4, 4).transpose(0, 1, 3, 2, 4).reshape(P, 4 * Hb, 4 * Wb)
    return back(full[:, :H, :W])
