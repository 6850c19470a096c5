"""Float64 oracle, rounding-level error bounds and a restatement of the launch planner for the tensor-core contraction kernel
(umma_gemm_kernel in ccv_b200/csrc/sm100_umma_gemm.cuh, planned by ccv_b200/csrc/sm100_contract.cu).

Oracle.  Every product is computed in float64 on the operands exactly as the kernel's MMAs see them: TF32 operands rounded to
nearest at 10 mantissa bits (what the TMA unit writes with CU_TENSOR_MAP_DATA_TYPE_TFLOAT32), raw fp32 values for 3xTF32 and
FFMA, and the 16-bit values themselves for bf16 / fp16.  Test data never holds a TF32 rounding tie (low 13 mantissa bits exactly
0x1000), so the oracle does not depend on how the hardware breaks ties.

Bounds.  The same product on absolute values gives a per-element scale s = sum |a~||b~| (+ |bias| + |old output|).  With K_eff
the number of terms in the element's reduction (GEMM: K; forward: R*S*C; data gradient: the taps of the element's residue class
times K; weight gradient: N*P*Q):
  fp32 outputs      |y - y^| <= e,  e = C_ACC * 2^-24 * sqrt(K_eff) * s
  3xTF32            e += 2^-20 * s   (the dropped lo*lo term and the TF32 truncation of lo)
  16-bit outputs    rne16(y^ - e) <= y <= rne16(y^ + e): correctly rounded up to the accumulation error.
C_ACC was calibrated on an H100 80GB HBM3 (SXM, 132 SMs, 400 W power limit, SM clock at most 1980 MHz): over every case of
tests/test_parity_contract_paths.py the largest ratio |y - y^| / (2^-24 sqrt(K_eff) s) (for 16-bit outputs, the smallest e
that admits y) was 1.86 (a walking 3xTF32 forward), so C_ACC = 8 leaves a 4.3x margin."""
import os

import numpy as np

C_ACC = 8.0
BLOCK_M = 128
SCRATCH_BYTES = 96 << 20  # CONTRACT_SCRATCH_BYTES
MAX_TAPS = 64              # UMMA_MAX_TAPS
STATS_MAX_ROWS = 4 * 160   # rows of the statistics tensor the graph's conv -> batch-norm rewrite allocates, over 4 planes

FP32, TF32, X3, BF16, FP16 = "fp32", "tf32", "3xtf32", "bf16", "fp16"  # operand / math modes (fp32 = FFMA)


# ------------------------------------------------------------------------------------------------ rounding
def untie_tf32(a):
    """fp32 copy of `a` in which no value is a TF32 rounding tie (low 13 mantissa bits 0x1000 -> 0x1001)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).copy()
    u[(u & 0x1FFF) == 0x1000] += 1
    return u.view(np.float32).reshape(np.shape(a))


def tf32_round(a):
    """Round fp32 to nearest TF32 (10 mantissa bits; data carries no ties)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32).reshape(np.shape(a))


def tf32_trunc(a):
    """What the tensor core does with raw fp32 operands: drop the low 13 mantissa bits."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32).reshape(np.shape(a))


def to_bits16(x, out):
    """float64 -> 16-bit pattern (uint16), round to nearest even, directly from float64 (no double rounding)."""
    x = np.asarray(x, np.float64)
    if out == FP16:
        return x.astype(np.float16).view(np.uint16)
    m, e = np.frexp(x)
    r = np.ldexp(np.rint(m * 256.0), e - 8)  # 8 significant bits, ties to even
    return (r.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def from_bits16(u, out):
    u = np.asarray(u, np.uint16)
    if out == FP16:
        return u.view(np.float16).astype(np.float64)
    return (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def rne16(x, out):
    return from_bits16(to_bits16(x, out), out)


def trunc16(x, out):
    """Round toward zero to the 16-bit format (a defect the bounds must catch)."""
    x = np.asarray(x, np.float64)
    r = rne16(x, out)
    too_big = np.abs(r) > np.abs(x)
    key = _key16(to_bits16(x, out))
    return np.where(too_big, from_bits16(_unkey16(key - np.sign(key).astype(np.int32)), out), r)


def _key16(bits):
    """Monotone integer image of 16-bit floats: order of the keys = numeric order (both zeros -> 0)."""
    b = np.asarray(bits, np.uint16).astype(np.int32)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def _unkey16(k):
    k = np.asarray(k, np.int32)
    return np.where(k < 0, 0x8000 | (-k), k).astype(np.uint16)


def operand(shape, seed, mode, lo=-0.5, hi=1.0):
    """Seeded U(lo, hi] operand as the kernel receives it: fp32 without TF32 ties, or values already on the 16-bit grid.  A
    positive mean keeps |y| comparable to the scale, so one-ulp and one-bit operand errors stay visible in long reductions."""
    r = np.random.RandomState(seed)
    a = (lo + (hi - lo) * (1.0 - r.random_sample(shape))).astype(np.float32)
    if mode in (BF16, FP16):
        return from_bits16(to_bits16(a, mode), mode).astype(np.float32)
    return untie_tf32(a)


def seen(a, mode, trunc=False):
    """float64 values of operand `a` as the MMAs of `mode` multiply them."""
    if mode == TF32:
        return (tf32_trunc(a) if trunc else tf32_round(a)).astype(np.float64)
    return np.asarray(a, np.float64)


# ------------------------------------------------------------------------------------------------ oracle
def gemm(a, b, ta, tb, bias=None, old=None):
    """(y, s): y = op(a) op(b) (+ bias) (+ old) and the scale on absolute values; a, b, bias, old already float64."""
    A, B = (a.T if ta else a), (b.T if tb else b)
    y, s = A @ B, np.abs(A) @ np.abs(B)
    for t in (bias, old):
        if t is not None:
            y, s = y + t, s + np.abs(t)
    return y, s


class Geom(object):
    """NHWC convolution geometry; the end padding is whatever the output extent implies (conv_geom in sm100_backend.cu)."""

    def __init__(self, N, H, W, C, K, R, S, stride=(1, 1), pad=(0, 0), dil=(1, 1), P=None, Q=None, pad_end=None):
        self.N, self.H, self.W, self.C, self.K, self.R, self.S = N, H, W, C, K, R, S
        self.st, self.pad, self.dil = tuple(stride), tuple(pad), tuple(dil)
        pe = pad if pad_end is None else pad_end
        self.P = P if P is not None else (H + pad[0] + pe[0] - ((R - 1) * dil[0] + 1)) // stride[0] + 1
        self.Q = Q if Q is not None else (W + pad[1] + pe[1] - ((S - 1) * dil[1] + 1)) // stride[1] + 1
        self.pad_end = ((self.P - 1) * stride[0] + (R - 1) * dil[0] + 1 - H - pad[0], (self.Q - 1) * stride[1] + (S - 1) * dil[1] + 1 - W - pad[1])

    def taps(self):
        return [(r, s) for r in range(self.R) for s in range(self.S)]

    def _padded(self):
        return (max(self.pad[0] + self.H, (self.P - 1) * self.st[0] + (self.R - 1) * self.dil[0] + 1),
                max(self.pad[1] + self.W, (self.Q - 1) * self.st[1] + (self.S - 1) * self.dil[1] + 1))

    def _win(self, r, s):
        return (slice(r * self.dil[0], r * self.dil[0] + (self.P - 1) * self.st[0] + 1, self.st[0]),
                slice(s * self.dil[1], s * self.dil[1] + (self.Q - 1) * self.st[1] + 1, self.st[1]))

    def pad_input(self, x):
        Hp, Wp = self._padded()
        xp = np.zeros((x.shape[0], Hp, Wp, x.shape[3]), x.dtype)
        xp[:, self.pad[0]:self.pad[0] + self.H, self.pad[1]:self.pad[1] + self.W] = x
        return xp

    def keff_dgrad(self):
        """taps of each input pixel's residue class (times K): [H, W, 1]"""
        th = [sum((a + self.pad[0] - r * self.dil[0]) % self.st[0] == 0 for r in range(self.R)) for a in range(self.st[0])]
        tw = [sum((a + self.pad[1] - s * self.dil[1]) % self.st[1] == 0 for s in range(self.S)) for a in range(self.st[1])]
        h = np.array([th[i % self.st[0]] for i in range(self.H)], np.float64)
        w = np.array([tw[i % self.st[1]] for i in range(self.W)], np.float64)
        return (h[:, None] * w[None, :] * self.K)[:, :, None]


def conv_fwd(g, x, w, bias=None, taps=None):
    """y[N, P, Q, K] = sum over taps of the window of x times w[:, r, s, :]; x, w float64 ([.., C'] and [K, R, S, C'])"""
    xp = g.pad_input(x)
    y = np.zeros((x.shape[0], g.P, g.Q, w.shape[0]))
    for r, s in (taps or g.taps()):
        hs, ws = g._win(r, s)
        y += xp[:, hs, ws, :] @ w[:, r, s, :].T
    return y if bias is None else y + bias


def conv_dgrad(g, gy, w, taps=None):
    """h[N, H, W, C] = sum over taps of gy scattered back through the window; gy [N, P, Q, K'], w [K', R, S, C]"""
    Hp, Wp = g._padded()
    hp = np.zeros((gy.shape[0], Hp, Wp, w.shape[3]))
    for r, s in (taps or g.taps()):
        hs, ws = g._win(r, s)
        hp[:, hs, ws, :] += gy @ w[:, r, s, :]
    return hp[:, g.pad[0]:g.pad[0] + g.H, g.pad[1]:g.pad[1] + g.W, :]


def conv_wgrad(g, gy, x, rows=None, old=None):
    """dw[K, R, S, C] = sum over output pixels of gy (x) window of x; `rows`: only these flattened N*P*Q pixels"""
    xp = g.pad_input(x)
    gf = gy.reshape(-1, gy.shape[3])
    dw = np.zeros((gy.shape[3], g.R, g.S, x.shape[3]))
    for r, s in g.taps():
        hs, ws = g._win(r, s)
        xf = xp[:, hs, ws, :].reshape(-1, x.shape[3])
        dw[:, r, s, :] = (gf[rows].T @ xf[rows]) if rows is not None else gf.T @ xf
    return dw if old is None else dw + old


def with_scale(fn, *args, **kw):
    """(y, s) of a linear product: fn on the operands and on their absolute values (`old` / `bias` keywords are added as |.|)"""
    extra = [kw.pop(k) for k in ("old", "bias") if kw.get(k) is not None]
    kw.pop("old", None), kw.pop("bias", None)
    y, s = fn(*args, **kw), fn(*[np.abs(a) if isinstance(a, np.ndarray) else a for a in args], **kw)
    for t in extra:
        y, s = y + t, s + np.abs(t)
    return y, s


# ------------------------------------------------------------------------------------------------ bounds
def bound(s, keff, mode, c=C_ACC):
    e = c * 2.0 ** -24 * np.sqrt(keff) * s
    return e + 2.0 ** -20 * s if mode == X3 else e


def needed(y, ref, s, keff, mode, out):
    """Per element, the smallest c for which the bound admits y (the calibration ratio); inf for non-finite y."""
    y = np.asarray(y, np.float64)
    unit = 2.0 ** -24 * np.sqrt(keff) * s
    if out == FP32:
        err = np.abs(y - ref) - (2.0 ** -20 * s if mode == X3 else 0.0)
    else:
        k = _key16(to_bits16(y, out))
        below, above = from_bits16(_unkey16(k - 1), out), from_bits16(_unkey16(k + 1), out)
        r = rne16(ref, out)
        err = np.where(y > r, (y + below) / 2 - ref, np.where(y < r, ref - (y + above) / 2, 0.0))
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.maximum(err, 0.0) / np.maximum(unit, 1e-300)
    return np.where(np.isfinite(y), ratio, np.inf)


def admits(y, ref, s, keff, mode, out, c=C_ACC):
    """Boolean mask: elements of y (fp32 values, or fp32 images of 16-bit values) that the bound accepts."""
    y = np.asarray(y, np.float64)
    e = bound(s, keff, mode, c)
    if out == FP32:
        return np.abs(y - ref) <= e  # NaN -> False
    return (rne16(ref - e, out) <= y) & (y <= rne16(ref + e, out))


def check(y, ref, s, keff, mode, out, what="", c=C_ACC):
    """Assert the bound on every element; returns the largest calibration ratio."""
    ok = admits(y, ref, s, keff, mode, out, c)
    if not ok.all():
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        yv = np.asarray(y, np.float64)[i]
        raise AssertionError("%s: %d of %d elements outside the %s bound (c = %g); first at %s: got %r, oracle %r, scale %r, K_eff %r"
                             % (what, len(bad), ok.size, mode, c, i, yv, ref[i], s[i], np.broadcast_to(keff, ref.shape)[i]))
    r = needed(y, ref, s, keff, mode, out)
    return float(r.max()) if r.size else 0.0


# ------------------------------------------------------------------------------------------------ the launch planner
def pick_bn(n):
    e = os.environ.get("CCV_NNC_SM100_BN")
    try:
        bn = int(e) if e else (64 if n <= 64 else 128)
    except ValueError:
        bn = 0
    return 64 if bn == 64 else 128


def _trim(k, k_iters):
    while k > 1 and ((k_iters + k - 1) // k) * (k - 1) >= k_iters:
        k -= 1
    return max(k, 1)


def pick_splits(tiles, k_iters, min_iters, sms):
    max_s = max(1, k_iters // min_iters)
    if tiles >= 4 * sms or max_s == 1:
        return 1
    if tiles < sms:
        return _trim(min(2 * sms // max(tiles, 1), max_s), k_iters)
    limit = min(max(4, 2 * sms // max(tiles, 1)), max_s)
    cost = lambda k: -(-tiles * k // sms) / k
    best = min(cost(k) for k in range(1, limit + 1))
    if best > -(-tiles // sms) * 0.8:
        return 1
    return _trim(next(k for k in range(1, limit + 1) if cost(k) <= best * 1.05), k_iters)


def fit_splits(splits, k_iters, slice_bytes):
    return 1 if splits <= 1 else _trim(min(splits, SCRATCH_BYTES // slice_bytes), k_iters)


def grid_x(tiles_m, columns, sms, splits=1, grid_taps=1):
    """launch_umma's walk rule: CTAs per column (== tiles_m when every CTA takes one tile)"""
    ctas = tiles_m * columns
    if splits != 1 or grid_taps != 1 or ctas <= sms:
        return tiles_m
    gx = max(1, min(tiles_m, sms // columns))
    return gx if -(-gx * columns // sms) * -(-tiles_m // gx) <= -(-ctas // sms) else tiles_m


def stats_grid_x(tiles_m, tiles_n, sms):
    return min(max(sms // tiles_n, 1), STATS_MAX_ROWS // 4, tiles_m)


def _launch(M, N, bn, k_iters, sms, splits=1, grid_taps=1, stats=False):
    tm, tn = -(-M // BLOCK_M), -(-N // bn)
    gx = stats_grid_x(tm, tn, sms) if stats else grid_x(tm, tn * grid_taps * splits, sms, splits, grid_taps)
    return dict(bn=bn, tiles=(tm, tn, grid_taps), splits=splits, grid_x=gx, k_iters=k_iters)


def _gemm_plan(M, N, K, kind, sms, bias16=False, stats=False):
    bn, bk = pick_bn(N), 32 if kind == 0 else 64
    ki = -(-K // bk)
    s = 1 if bias16 else fit_splits(pick_splits(-(-M // BLOCK_M) * -(-N // bn), ki, 8, sms), ki, M * ((N + 3) & ~3) * 4)
    return [_launch(M, N, bn, ki, sms, splits=s, stats=stats and s == 1)]


def pointwise(g):
    return g.R == 1 and g.S == 1 and g.st == (1, 1) and g.pad == (0, 0) and g.pad_end == (0, 0)


def tensor_core_ok(op, g, kind, in_view=False):
    """the conditions under which the contraction kernel takes a convolution (else the callers fall back)"""
    al = 4 if kind == 0 else 8
    lower = [-p for p in g.pad]
    upper = [pe - (k - 1) * d for pe, k, d in zip(g.pad_end, (g.R, g.S), g.dil)]
    return (g.R * g.S <= MAX_TAPS and g.C % al == 0 and g.K % al == 0 and all(-128 <= v <= 127 for v in lower + upper)
            and all(1 <= s <= 8 for s in g.st) and not (op == "dgrad" and in_view) and not (pointwise(g) and in_view))


def plan(op, kind, sms, M=None, N=None, K=None, g=None, bias16=False, stats=False):
    """Launches of one contraction call: {"launches": [dict(bn, tiles=(m, n, taps), splits, grid_x)], "kernels": n, "path"}.
    op: gemm | fwd | dgrad | wgrad; kind: 0 fp32 (TF32 / 3xTF32), 1 bf16, 2 fp16.  `kernels` is what ccv_nnc_sm100_launch_count()
    advances by: contraction launches, one ordered combine per split launch, the fp32 data gradient's filter copy."""
    extra = 0
    if op == "gemm":
        ls = _gemm_plan(M, N, K, kind, sms, bias16, stats)
    elif op == "fwd":
        if pointwise(g):
            ls = _gemm_plan(g.N * g.P * g.Q, g.K, g.C, kind, sms, bias16, stats)
        else:
            ki = g.R * g.S * -(-g.C // (32 if kind == 0 else 64))
            ls = [_launch(g.N * g.P * g.Q, g.K, pick_bn(g.K), ki, sms, stats=stats)]
    elif op == "dgrad":
        extra = 1 if kind == 0 else 0
        if pointwise(g):
            ls = _gemm_plan(g.N * g.H * g.W, g.C, g.K, kind, sms)
        else:
            ls = []
            keff = g.keff_dgrad()[..., 0] / g.K
            for ah in range(min(g.st[0], g.H)):
                for aw in range(min(g.st[1], g.W)):
                    taps = int(keff[ah, aw])
                    if taps:
                        M = g.N * -(-(g.H - ah) // g.st[0]) * -(-(g.W - aw) // g.st[1])
                        ls.append(_launch(M, g.C, pick_bn(g.C), taps * -(-g.K // (32 if kind == 0 else 64)), sms))
    elif op == "wgrad":
        bn, bk = pick_bn(g.C), 32 if kind == 0 else 64
        ki = -(-(g.N * g.P * g.Q) // bk)
        tiles = -(-g.K // BLOCK_M) * -(-g.C // bn) * g.R * g.S
        s = fit_splits(pick_splits(tiles, ki, 16, sms), ki, g.K * g.R * g.S * g.C * 4)
        taps = 1 if pointwise(g) else g.R * g.S
        ls = [_launch(g.K, g.C, bn, ki, sms, splits=s, grid_taps=taps)]
    else:
        raise ValueError(op)
    kernels = extra + sum(1 + (l["splits"] > 1) for l in ls)
    if any(l["splits"] > 1 for l in ls):
        path = "split"
    elif any(l["grid_x"] < l["tiles"][0] for l in ls):
        path = "walk"
    else:
        path = "tile"
    return dict(launches=ls, kernels=kernels, path=path)


def device_sms():
    """SM count of device 0 (cudaDevAttrMultiProcessorCount through the runtime library torch ships with, or torch itself)."""
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:
        pass
    import ctypes
    for name in ("libcudart.so", "libcudart.so.12"):
        try:
            rt = ctypes.CDLL(name)
        except OSError:
            continue
        v = ctypes.c_int(0)
        if rt.cudaDeviceGetAttribute(ctypes.byref(v), 16, 0) == 0:  # cudaDevAttrMultiProcessorCount
            return v.value
    raise RuntimeError("cannot read the SM count of device 0")
