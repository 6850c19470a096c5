"""numpy oracles for ROI_ALIGN and NMS (forward / backward) in the source order of the reference's CPU_REF
(lib/nnc/cmd/roi/ccv_nnc_roi_align_cpu_ref.c, lib/nnc/cmd/nms/ccv_nnc_nms_cpu_ref.c), every fp32 operation rounded on its own.

Features are NHWC [n?, H, W, C] float32 (16-bit results: run on the widened inputs, round once).  The backend's rules where CPU_REF is
undefined are restated here too: a ROI with a non-finite value, or whose per-axis bin sample count ceil(size / pool) exceeds 4 x the map's
extent on that axis (or bin * pool exceeds 2^30), is an empty ROI (zeros); NMS sorts stably on the order-preserving 32-bit key of the score."""
import numpy as np

F32 = np.float32
FLT_MAX = np.finfo(np.float32).max
MAX_BINS_PER_PIXEL = 4
MAX_SAMPLES = 1 << 30


def _axis(v, vs, size, pool):
    """one axis of _ccv_nnc_bilinear_coeffs (roi_align_cpu_ref.c:18-99): (bin, i0[], i1[], r[], live[]) over bin * pool samples, or None
    for an empty ROI"""
    roi = F32(F32(v) * F32(size))
    rs = F32(F32(vs) * F32(size))
    with np.errstate(all="ignore"):
        bins = np.ceil(F32(rs / F32(pool)))
    if not (np.isfinite(roi) and np.isfinite(rs)) or not bins >= 1 or bins > MAX_BINS_PER_PIXEL * size or bins * pool > MAX_SAMPLES:
        return None
    b = int(bins)
    scale = F32(rs / F32(b * pool))
    k = np.arange(b * pool, dtype=np.float64)
    a = ((np.float64(roi) + (k + 0.5) * np.float64(scale)) - 0.5).astype(np.float32)  # double, as the 0.5 literals make it
    with np.errstate(invalid="ignore"):  # only muted samples can sit beyond int64
        i = np.floor(a).astype(np.int64)
    r = (a - i.astype(np.float32)).astype(np.float32)
    live = ~((i + 1 < 0) | (i > size - 1))
    return b, np.clip(i, 0, size - 1), np.clip(i + 1, 0, size - 1), r, live


def _coeffs(box, h, w, ph, pw):
    ay, ax = _axis(box[1], box[3], h, ph), _axis(box[0], box[2], w, pw)
    if ay is None or ax is None:
        return None
    cy = ay[4].reshape(ph, ay[0]).sum(1)
    cx = ax[4].reshape(pw, ax[0]).sum(1)
    return ay, ax, cy, cx


def _range(counts):
    """CPU_REF's start / end bins: the first bin with a live sample, one past the last (pool, 0 when none)"""
    nz = np.nonzero(counts > 0)[0]
    return (int(nz[0]), int(nz[-1]) + 1) if len(nz) else (len(counts), 0)


def _corner_weights(ry, rx):
    one = F32(1)
    return (F32(one - ry) * F32(one - rx), F32(one - ry) * rx, ry * F32(one - rx), ry * rx)


def _out_row(i, start_h):
    """the output row CPU_REF writes bin row i to (its row pointer starts at row 0 while i starts at start_h)"""
    return i - start_h


def roi_align_forward(a, b, ph, pw):
    """a [n?, H, W, C], b [4] or [k, 4] -> c [max(a_n, b_n), ph, pw, C] (or [ph, pw, C] when both are single).  CPU_REF writes bin row
    i to output row i - start_h (roi_align_cpu_ref.c:186-196): rows past end_h - start_h stay zero."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    a4, b2 = a.reshape((-1,) + a.shape[-3:]), b.reshape(-1, 4)
    H, W, C = a4.shape[1:]
    N = max(len(a4), len(b2))
    c = np.zeros((N, ph, pw, C), np.float32)
    for n in range(N):
        co = _coeffs(b2[n % len(b2)], H, W, ph, pw)
        if co is None:
            continue
        (bh, iy0, iy1, ry, ly), (bw, ix0, ix1, rx, lx), cy, cx = co
        sh, eh = _range(cy)
        sw, ew = _range(cx)
        an = a4[n % len(a4)]
        for i in range(sh, eh):
            for j in range(sw, ew):
                ys = [y for y in range(i * bh, (i + 1) * bh) if ly[y]]
                xs = [x for x in range(j * bw, (j + 1) * bw) if lx[x]]
                acc = np.zeros(C, np.float32)
                for y in ys:
                    for x in xs:
                        c00, c01, c10, c11 = _corner_weights(ry[y], rx[x])
                        s = an[iy0[y], ix0[x]] * c00 + an[iy0[y], ix1[x]] * c01
                        s = s + an[iy1[y], ix0[x]] * c10
                        s = s + an[iy1[y], ix1[x]] * c11
                        acc = acc + s
                inv = F32(1.0 / float(int(cy[i]) * int(cx[j])))
                c[n, _out_row(i, sh), j] = acc * inv
    return c if a.ndim == 4 or b.ndim == 2 else c[0]


def roi_align_backward(g, b, shape):
    """g [n?, ph, pw, C], b ROIs -> o of `shape` ([n?, H, W, C]): every pixel adds (g c) inv in CPU_REF's order, ROI n ascending, bins
    i, j, samples y, x, corners 00, 01, 10, 11 (roi_align_cpu_ref.c:248-303).  np.add.at adds its rows in index order."""
    g = np.asarray(g, np.float32)
    g4, b2 = g.reshape((-1,) + g.shape[-3:]), np.asarray(b, np.float32).reshape(-1, 4)
    ph, pw, C = g4.shape[1:]
    H, W = shape[-3], shape[-2]
    on = shape[0] if len(shape) == 4 else 1
    o = np.zeros((on, H * W, C), np.float32)
    for n in range(len(g4)):
        co = _coeffs(b2[n % len(b2)], H, W, ph, pw)
        if co is None:
            continue
        (bh, iy0, iy1, ry, ly), (bw, ix0, ix1, rx, lx), cy, cx = co
        idx, terms = [], []
        for i in range(ph):
            for j in range(pw):
                if not cy[i] or not cx[j]:
                    continue
                inv = F32(1.0 / float(int(cy[i]) * int(cx[j])))
                gz = g4[n, i, j]
                for y in range(i * bh, (i + 1) * bh):
                    if not ly[y]:
                        continue
                    for x in range(j * bw, (j + 1) * bw):
                        if not lx[x]:
                            continue
                        cs = _corner_weights(ry[y], rx[x])
                        for (yy, xx), cw in zip(((iy0[y], ix0[x]), (iy0[y], ix1[x]), (iy1[y], ix0[x]), (iy1[y], ix1[x])), cs):
                            idx.append(yy * W + xx)
                            terms.append((gz * cw) * inv)
        if idx:
            np.add.at(o[n % on], np.array(idx), np.stack(terms).astype(np.float32))
    return o.reshape(shape)


# ---- NMS ---------------------------------------------------------------------------------------------------------------------------
def score_key(s):
    """order-preserving 32-bit key: larger score, larger key; -0 folded onto +0; NaNs ordered by their bits"""
    u = np.ascontiguousarray(s, np.float32).view(np.uint32).copy()
    u[u == 0x80000000] = 0
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def _iou_ge(bx, by, thr):
    """CPU_REF's test (nms_cpu_ref.c:77-86) of one box bx (higher score) against rows by, float32 term by term"""
    with np.errstate(all="ignore"):
        area1 = F32(bx[3] * bx[4])
        area2 = (by[:, 3] * by[:, 4]).astype(np.float32)
        xe0, xe1 = F32(bx[1] + bx[3]), (by[:, 1] + by[:, 3]).astype(np.float32)
        ye0, ye1 = F32(bx[2] + bx[4]), (by[:, 2] + by[:, 4]).astype(np.float32)
        xd = (np.where(xe0 < xe1, xe0, xe1) - np.where(bx[1] > by[:, 1], bx[1], by[:, 1])).astype(np.float32)
        yd = (np.where(ye0 < ye1, ye0, ye1) - np.where(bx[2] > by[:, 2], bx[2], by[:, 2])).astype(np.float32)
        xdiff, ydiff = np.where(0 > xd, F32(0), xd), np.where(0 > yd, F32(0), yd)
        inter = (xdiff * ydiff).astype(np.float32)
        iou = (inter / ((area1 + area2).astype(np.float32) - inter)).astype(np.float32)
        return iou >= F32(thr)


def _order(scores):
    """the stable descending order of the scores: ties keep input order"""
    return np.argsort(-score_key(scores).astype(np.int64), kind="stable")


def nms_forward(a, thr):
    """a [m, 5] or [n, m, 5] float32 -> (b, c): per item, a stable descending sort by score, greedy suppression, kept rows first in
    score order; the tail gets c = -1, score -FLT_MAX and the sorted array's coordinates at its own positions"""
    a = np.asarray(a, np.float32)
    a3 = a.reshape((-1,) + a.shape[-2:])
    b, c = np.empty_like(a3), np.empty(a3.shape[:2], np.int32)
    for it in range(len(a3)):
        order = _order(a3[it, :, 0])
        s = a3[it, order].copy()
        m = len(s)
        gone = s[:, 0] == -FLT_MAX
        for x in range(m):
            if gone[x]:
                continue
            y = np.arange(x + 1, m)
            hit = _iou_ge(s[x], s[x + 1:], thr) & ~gone[x + 1:]
            gone[y[hit]] = True
        kept = np.nonzero(~gone)[0]
        k = len(kept)
        b[it] = s
        b[it, :k] = s[kept]
        b[it, k:, 0] = -FLT_MAX
        c[it, :k] = order[kept]
        c[it, k:] = -1
    return b.reshape(a.shape), c.reshape(a.shape[:-1])


def nms_backward(g, c):
    """g [n?, m, 5], c [n?, m] -> h: zero, then h[c[x]] = g[x] up to the first negative index"""
    g = np.asarray(g, np.float32)
    g3, c2 = g.reshape((-1,) + g.shape[-2:]), np.asarray(c).reshape(-1, g.shape[-2])
    h = np.zeros_like(g3)
    for it in range(len(g3)):
        for x, k in enumerate(c2[it]):
            if k < 0:
                break
            h[it, k] = g3[it, x]
    return h.reshape(g.shape)
