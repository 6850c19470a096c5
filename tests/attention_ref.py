"""Float64 oracle, rounding-level error bounds and a restatement of the launch planner for SCALED_DOT_PRODUCT_ATTENTION
(forward and backward: the 16-bit flash kernels of ccv_b200/csrc/sm100_fmha.cu and sm100_fmha_bwd.cu, the fp32 path of
sm100_sdpa.cu, and the 16-bit functional form of sm100_backend_ext.cu that widens, runs the fp32 path and narrows).

Oracle.  O = softmax(scale Q K^T + mask) V with GQA (query head h reads key head h / (H / Hk)), causal masks aligned to the
bottom-right corner (query i sees keys j <= i + Sk - Sq, so Sq > Sk leaves fully masked rows: O = 0, LSE = -inf, dQ = 0), an
additive mask broadcast from [Sq, Sk], [X, Sq, Sk] (X = heads) or [1|B, 1|H, Sq, Sk], Dv != D; and dQ, dK, dV with dK / dV summed
over the query heads of a group.  Everything is float64 on the operands as each path sees them:
  flash / fused   the 16-bit values themselves; delta_i = sum_d dO_id O_id is formed from the STORED 16-bit O, as the prep kernel does
  fp32 TF32       q, k, v, dO rounded to nearest TF32 (the TMA unit); raw fp32 where a GEMM declines the tensor maps and FFMA runs
  functional      the 16-bit values (exact in TF32: bf16 has 8 significant bits, fp16 11), then the fp32 path
fp32 outputs are held to |y - y^| <= e; 16-bit outputs to the window R(y^ - e) <= y <= R(y^ + e), with R = round to nearest even
for the flash kernels and for bf16 narrowing, R = round toward zero for fp16 narrowing (convert_dtype code 1 truncates, like the
reference's f32 -> f16 table).

Bounds.  e = C_ATT * (sum of the terms below), per element, from float64 sums of absolute values.  u_P is the relative half-ulp of the
format P and dS are rounded to before their MMAs (bf16 2^-8, fp16 2^-11, TF32 2^-11, 2^-24 when an FFMA GEMM reads them raw); (t, f)
is the subnormal threshold and absolute rounding floor of that format (fp16: 2^-14, 2^-25); u = 2^-24; p = exact probabilities,
p~ = exp(s - max), l = sum p~, n = ceil(Sk / 128) key blocks.
  exponent argument  eps_ij = u (sqrt(D) |scale| sum_d |q||k| + 2 |s_ij| + |max_i| + |mask_ij|) + 2^-22   (S accumulated in fp32, the
                     scale * log2 e product, the subtraction; ex2.approx / expf relative error)
  O                  u_P sqrt(sum_j p^2 v^2)                           P rounded before the PV MMA (random walk, as contract_ref)
                     + sum_{0 < p~ < t} min(p~, f) |v| / l              P below the format's normal range (need not average out)
                     + sum_j p eps (|v| + |O|)                          exponent errors, through numerator and denominator
                     + u sqrt(Sk + 2n + 2) (sum_j p |v| + |O|)          fp32 accumulation, rescales by alpha, the row sum, 1 / l
  LSE                u sqrt(Sk + 2n) + sum_j p eps + u (2 |max| + |ln l| + |lse|)
  backward           eps'_ij = eps_ij + u |lse_i| + the LSE term above (P recomputed from the stored log-sum-exp; fp32 path: its own
                     softmax, + u sqrt(Sk))
    dP, delta        e_dP = u sqrt(Dv) sum_d |dO||v| + u |dP|;  fused: e_delta = u sqrt(Dv) sum_d |dO||O16|;
                     fp32: e_delta = u sqrt(Sk) sum_j p |dP| + sum_j p (e_dP + eps' |dP|)
    dS               e_dS = eps' |dS| + p (e_dP + e_delta) + 2 u |dS|
    dV               u_P sqrt(sum_i p^2 dO^2) + sum_{0 < p < t} min(p, f) |dO| + sum_i p eps' |dO| + u sqrt(G Sq + 2) sum_i p |dO|
    dQ (dK alike)    |scale| (u_P sqrt(sum_j dS^2 k^2) + sum_{0 < |dS| < t} min(|dS|, f) |k| + sum_j e_dS |k| + u sqrt(Sk + 2) sum_j |dS||k|)
                     + 2 u |dQ|
C_ATT was calibrated on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit, SM clock at most 1980 MHz): over every case of
tests/test_parity_attention_paths.py the largest ratio (the smallest C that admits the result) per path was
  flash forward O       bf16 1.54, fp16 1.11;  LSE 0.33
  fused backward        bf16 1.72, fp16 1.28
  fp32 path             forward 1.81, backward 1.66 (TF32 and FFMA GEMMs)
  functional form       forward bf16 1.35, fp16 1.44;  backward bf16 0.65, fp16 1.00
  bench.py's shape      O 1.72, LSE 0.17, backward 1.83   (bf16, B = 32, H = 16, S = 2048, D = 128, q = k = v = dout)
so C_ATT = 8 leaves a margin of 4.4x.  A rounding defect of P shows once a row spreads its weight over about (2 C_ATT)^2 keys."""
import numpy as np

from tests.contract_ref import BF16, FP16, FP32, _key16, _unkey16, from_bits16, rne16, tf32_round, to_bits16, trunc16

C_ATT = 8.0
U32 = 2.0 ** -24
EX2 = 2.0 ** -22
U16 = {BF16: 2.0 ** -8, FP16: 2.0 ** -11}  # unit roundoff: 8 and 11 significant bits
TINY = (2.0 ** -126, 2.0 ** -126)  # fp32 / bf16 / TF32 below the normal range: ex2.approx.ftz flushes, bf16 keeps 2^-133 steps
FLOOR = {BF16: TINY, FP16: (2.0 ** -14, 2.0 ** -25)}
U_TF32 = 2.0 ** -11
FM_BLOCK = 128  # keys per block of the forward kernel; the backward streams 64-row blocks


# ------------------------------------------------------------------------------------------------ paths
class Model(object):
    """How one path computes: p_fmt, the format P and dS are rounded to before their MMAs (bf16 / fp16 / "tf32", None = read raw by
    FFMA), its u_p and (threshold, floor), and whether the backward recomputes P with the fp32 path's own softmax."""

    def __init__(self, path, p_fmt):
        self.path, self.p_fmt = path, p_fmt
        self.u_p = {None: U32, "tf32": U_TF32}.get(p_fmt) or U16[p_fmt]
        self.floor = FLOOR.get(p_fmt, TINY)
        self.fp32_softmax = path not in ("flash", "fused")


def model_for(dtype, plan):
    """The arithmetic model of a planned path: dtype is bf16 / fp16 / fp32; plan from plan_forward / plan_backward."""
    if plan["path"] in ("flash", "fused"):
        return Model(plan["path"], dtype)
    return Model(plan["path"], "tf32" if plan["gemm_p"] == "tf32" else None)


def seen_p(x, plan):
    """operands of the GEMMs that read P / dS (V, dO, K, Q) as those GEMMs see them: TF32-rounded or raw"""
    return tf32_round(x).astype(np.float64) if plan.get("gemm_p") == "tf32" else np.asarray(x, np.float64)


def seen_s(x, plan):
    """operands of the GEMMs S = Q K^T and dP = dO V^T"""
    return tf32_round(x).astype(np.float64) if plan.get("gemm_s") == "tf32" else np.asarray(x, np.float64)


def _flash_ok(D, Dv, H, Hk, aligned):
    return 8 <= D <= 128 and D % 8 == 0 and Dv == D and H % Hk == 0 and aligned


def _fp32_gemms(D, Dv, Sk, aligned4=True):
    """The fp32 gemm_any declines (and gemm_ffma runs) when an operand's tensor map cannot be encoded: fp32 rows must start on 16 bytes.
    S = Q K^T reads q / k rows of D floats; P V, P^T dO, dS K and dS^T Q read the [Sq, Sk] score matrix with pitch Sk."""
    return dict(gemm_s="tf32" if D % 4 == 0 and Dv % 4 == 0 and aligned4 else "ffma", gemm_p="tf32" if Sk % 4 == 0 and D % 4 == 0 and Dv % 4 == 0 and aligned4 else "ffma")


def plan_forward(dtype, B, H, Hk, Sq, Sk, D, Dv, mask=False, view=False, lse=False, aligned=True):
    """(path, launches) of one forward call as sdpa_forw_core / sdpa_forward_f16 / sdpa_forward_f32 choose it; launches is what
    ccv_nnc_sm100_launch_count() advances by.  path: flash | fp32 | func | refused (NO_KERNEL)."""
    if dtype == FP32:
        return dict(path="fp32", launches=3 * B * H, **_fp32_gemms(D, Dv, Sk, aligned))  # per (b, h): S GEMM, softmax, P V GEMM
    if not mask and _flash_ok(D, Dv, H, Hk, aligned):
        return dict(path="flash", launches=1)
    if lse or view:
        return dict(path="refused", launches=0)
    return dict(path="func", launches=3 + 3 * B * H + 1, **_fp32_gemms(D, Dv, Sk))  # widen q, k, v; fp32 path; narrow o


def plan_backward(dtype, B, H, Hk, Sq, Sk, D, Dv, saved=False, view=False, aligned=True):
    """fused: prep + dK/dV + dQ (+ the forward when o / lse are not passed); fp32: per (b, h) S, softmax, dV, dP, dsoftmax, dQ, dK"""
    if dtype == FP32:
        return dict(path="fp32", launches=7 * B * H, **_fp32_gemms(D, Dv, Sk, aligned))
    if _flash_ok(D, Dv, H, Hk, aligned):
        return dict(path="fused", launches=3 if saved else 4)
    if view:
        return dict(path="refused", launches=0)
    return dict(path="func", launches=4 + 7 * B * H + 3, **_fp32_gemms(D, Dv, Sk))  # widen g, q, k, v; fp32 path; narrow 3


# ------------------------------------------------------------------------------------------------ oracle
def mask4(mask, B, H):
    """additive mask as a [1|B, 1|H, Sq, Sk] float64 array (2-d: [Sq, Sk]; 3-d: [X, Sq, Sk] with X on the head axis)"""
    if mask is None:
        return None
    m = np.asarray(mask, np.float64)
    return m.reshape((1,) * (4 - m.ndim) + m.shape)


def _bhsd(x):
    return np.ascontiguousarray(np.asarray(x, np.float64).transpose(0, 2, 1, 3))


def visible(Sq, Sk, causal, extra=0):
    """[Sq, Sk] keys each query attends (causal: bottom-right aligned); `extra` lets a row see keys past its horizon (a defect)"""
    if not causal:
        return np.ones((Sq, Sk), bool)
    return np.arange(Sk)[None, :] <= np.arange(Sq)[:, None] + (Sk - Sq) + extra


def expand_kv(x, H, gqa="div"):
    """[B, Hk, S, D] -> [B, H, S, D]: query head h reads key head h / (H / Hk) ("mod": h % Hk, a defect)"""
    Hk = x.shape[1]
    idx = np.arange(H) // (H // Hk) if gqa == "div" else np.arange(H) % Hk
    return x[:, idx]


def group_sum(x, Hk):
    B, H = x.shape[:2]
    return x.reshape((B, Hk, H // Hk) + x.shape[2:]).sum(2)


class Forward(object):
    """The exact forward of one call on float64 operands [B, S, H, D] (already as the path sees them) and its bound terms.
    Attributes ([B, H, ...] layout): s (logits), vis, m, pt (p~), l, p, o, lse, unit_o, unit_lse.  `defect` applies a modelled
    kernel defect to the result (see DEFECTS)."""

    def __init__(self, q, k, v, scale, causal, mask=None, model=None, defect=None, drop=None):
        self.model = model
        q, k, v = _bhsd(q), _bhsd(k), _bhsd(v)
        B, H, Sq, D = q.shape
        Hk, Sk, Dv = k.shape[1], k.shape[2], v.shape[3]
        self.B, self.H, self.Hk, self.Sq, self.Sk, self.D, self.Dv, self.scale = B, H, Hk, Sq, Sk, D, Dv, scale
        gqa = "mod" if defect == "gqa_mod" else "div"
        self.ke, self.ve = expand_kv(k, H, gqa), expand_kv(v, H, gqa)
        self.q = q
        s = scale * np.einsum("bhid,bhjd->bhij", q, self.ke)
        sabs = abs(scale) * np.einsum("bhid,bhjd->bhij", np.abs(q), np.abs(self.ke))
        mk = mask4(mask, B, H)
        vis = np.broadcast_to(visible(Sq, Sk, causal, 1 if defect == "extra_key" else 0), s.shape).copy()
        if drop is not None:
            vis[..., drop] = False
        if mk is not None:
            s = s + mk
        s = np.where(vis, s, -np.inf)
        m = s.max(-1, keepdims=True)
        live = np.isfinite(m)
        m0 = np.where(live, m, 0.0)
        pt = np.where(vis, np.exp(s - m0), 0.0)
        l = pt.sum(-1, keepdims=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            p = np.where(live, pt / np.where(live, l, 1.0), 0.0)
            lse = np.where(live[..., 0], (m0 + np.log(np.where(live, l, 1.0)))[..., 0], -np.inf)
        self.s, self.vis, self.m, self.pt, self.l, self.p, self.lse, self.live = np.where(vis, s, 0.0), vis, m0, pt, l, p, lse, live
        self.o = p @ self.ve
        if defect == "alpha1":  # the running max moves but O and l are not rescaled
            w = np.zeros_like(pt)
            run = np.full(m.shape, -np.inf)
            for j0 in range(0, Sk, FM_BLOCK):
                blk = slice(j0, j0 + FM_BLOCK)
                run = np.maximum(run, np.where(vis[..., blk], s[..., blk], -np.inf).max(-1, keepdims=True))
                w[..., blk] = np.where(vis[..., blk], np.exp(s[..., blk] - np.where(np.isfinite(run), run, 0.0)), 0.0)
            lw = w.sum(-1, keepdims=True)
            with np.errstate(invalid="ignore", divide="ignore"):
                self.o = np.where(live, (w @ self.ve) / np.where(lw > 0, lw, 1.0), 0.0)
        elif defect in ("p_trunc", "p_twice") and model.p_fmt is not None:
            f = model.p_fmt
            if defect == "p_trunc":
                r = _tf32_trunc64 if f == "tf32" else (lambda x: trunc16(x, f))
            else:
                r = lambda x: _round_bits(x, 7)  # through bf16 first (7 stored bits), then the format: exact after that
            if model.path == "flash":  # p~ (relative to the row max) is rounded; the row sum l is not
                with np.errstate(invalid="ignore", divide="ignore"):
                    self.o = np.where(live, (r(pt) @ self.ve) / np.where(live, l, 1.0), 0.0)
            else:  # the fp32 softmax's normalised P, rounded as the P V GEMM reads it
                self.o = r(p) @ self.ve
        if defect == "lse_key":  # the row sum misses the first visible key
            first = np.argmax(vis, -1)[..., None]
            pj = np.take_along_axis(pt, first, -1)
            with np.errstate(invalid="ignore", divide="ignore"):
                self.lse = np.where(live[..., 0] & (l > pj)[..., 0], (m0 + np.log(np.maximum(l - pj, 1e-300)))[..., 0], self.lse)
        if model is None:
            return
        u, (thr, fl) = model.u_p, model.floor
        eps = U32 * (np.sqrt(D) * sabs + 2 * np.abs(self.s) + np.abs(m0) + (np.abs(np.broadcast_to(mk, s.shape)) if mk is not None else 0.0)) + EX2
        eps = np.where(vis, eps, 0.0)
        self.eps = eps
        nblk = -(-Sk // FM_BLOCK)
        va = np.abs(self.ve)
        with np.errstate(invalid="ignore", divide="ignore"):
            small = np.where((pt > 0) & (pt < thr), np.minimum(pt, fl), 0.0)
            t_floor = (small @ va) / np.where(live, l, 1.0)
        pe = p * eps
        self.unit_o = (u * np.sqrt((p ** 2) @ (self.ve ** 2)) + t_floor + pe @ va + pe.sum(-1, keepdims=True) * np.abs(self.o)
                       + U32 * np.sqrt(Sk + 2 * nblk + 2) * (p @ va + np.abs(self.o)))
        with np.errstate(invalid="ignore", divide="ignore"):
            self.unit_lse = np.where(live[..., 0], (U32 * np.sqrt(Sk + 2 * nblk) + pe.sum(-1, keepdims=True) + U32 * (2 * np.abs(m0) + np.abs(np.log(np.where(live, l, 1.0)))))[..., 0]
                                     + U32 * np.abs(np.where(live[..., 0], self.lse, 0.0)), 0.0)

    def out(self):
        """O as [B, Sq, H, Dv] and its unit, LSE as [B, H, Sq] and its unit"""
        t = lambda x: np.ascontiguousarray(x.transpose(0, 2, 1, 3))
        return t(self.o), t(self.unit_o), self.lse, self.unit_lse


def _tf32_trunc64(x):
    return np.asarray(np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000), np.uint32).view(np.float32).reshape(np.shape(x)).astype(np.float64)


def _round_bits(x, bits):
    """round to nearest even at `bits` stored mantissa bits (P packed through bf16 before the fp16 / TF32 operand: rounded twice)"""
    mnt, e = np.frexp(np.asarray(x, np.float64))
    return np.ldexp(np.rint(mnt * 2.0 ** bits), e - bits)


class Backward(object):
    """dQ, dK, dV of one call and their bound units, from a Forward `f` (with its model) and dO [B, Sq, H, Dv] as the path sees it.
    `o16`: the stored 16-bit O [B, Sq, H, Dv] the fused prep kernel forms delta from (None: the fp32 path's sum_j p dP).
    Operands of the P / dS GEMMs (V, dO, K, Q) come as `p_ops` = (v, do, k, q) when they differ from the S / dP GEMMs' (TF32 vs raw)."""

    def __init__(self, f, do, o16=None, p_ops=None, dp_v=None, defect=None):
        mdl = f.model
        u, (thr, fl) = mdl.u_p, mdl.floor
        B, H, Hk, Sq, Sk, D, Dv, scale = f.B, f.H, f.Hk, f.Sq, f.Sk, f.D, f.Dv, f.scale
        do = _bhsd(do)
        if p_ops is None:
            doP, kP, qP = do, f.ke, f.q
        else:
            doP, kP, qP = _bhsd(p_ops[1]), expand_kv(_bhsd(p_ops[2]), H), _bhsd(p_ops[3])
        p = f.p
        ve = f.ve if dp_v is None else expand_kv(_bhsd(dp_v), H)  # V as dP = dO V^T reads it
        dp = do @ np.swapaxes(ve, -1, -2)
        e_dp = U32 * np.sqrt(Dv) * (np.abs(do) @ np.swapaxes(np.abs(ve), -1, -2)) + U32 * np.abs(dp)
        lse_err = np.where(f.live[..., 0], U32 * np.abs(np.where(f.live[..., 0], f.lse, 0.0)) + f.unit_lse, 0.0)[..., None]
        eps = f.eps + np.where(f.vis, lse_err + (U32 * np.sqrt(Sk) if mdl.fp32_softmax else 0.0), 0.0)
        if o16 is not None:
            ob = _bhsd(o16)
            ref_o = p @ ve if defect == "delta_exact" else ob
            delta = (do * ref_o).sum(-1, keepdims=True)
            e_delta = U32 * np.sqrt(Dv) * (np.abs(do) * np.abs(ob)).sum(-1, keepdims=True)
        else:
            delta = (p * dp).sum(-1, keepdims=True)
            e_delta = U32 * np.sqrt(Sk) * (p * np.abs(dp)).sum(-1, keepdims=True) + (p * (e_dp + eps * np.abs(dp))).sum(-1, keepdims=True)
        ds = p * (dp - delta)
        e_ds = eps * np.abs(ds) + p * (e_dp + e_delta) + 2 * U32 * np.abs(ds)
        pT, dsT = np.swapaxes(p, -1, -2), np.swapaxes(ds, -1, -2)
        sc = 1.0 if defect == "no_scale" else scale
        heads = np.ones(H, bool)
        if defect == "group_head":
            heads[H // Hk - 1::H // Hk] = False  # the last query head of every group is left out of dK / dV
        hm = heads[None, :, None, None].astype(np.float64)
        self.dq = sc * (ds @ kP)
        self.dk = group_sum(hm * sc * (dsT @ qP), Hk)
        self.dv = group_sum(hm * (pT @ doP), Hk)
        # below the format's normal range the rounding error is at most min(|x|, floor) and need not average out (a run of values
        # under half the smallest subnormal all round to zero): these terms add up linearly
        sp = np.where((p > 0) & (p < thr), np.minimum(p, fl), 0.0)
        sd = np.where((ds != 0) & (np.abs(ds) < thr), np.minimum(np.abs(ds), fl), 0.0)
        n_g = H // Hk
        # sums over the group first, then the square roots: the random walk runs over every (head, query) of the group
        self.unit_dv = (u * np.sqrt(group_sum((pT ** 2) @ (doP ** 2), Hk)) + group_sum(np.swapaxes(sp, -1, -2) @ np.abs(doP), Hk)
                        + group_sum(np.swapaxes(p * eps, -1, -2) @ np.abs(doP), Hk) + U32 * np.sqrt(Sq * n_g + 2) * group_sum(pT @ np.abs(doP), Hk))
        a = abs(scale)
        self.unit_dq = a * (u * np.sqrt((ds ** 2) @ (kP ** 2)) + sd @ np.abs(kP) + e_ds @ np.abs(kP) + U32 * np.sqrt(Sk + 2) * (np.abs(ds) @ np.abs(kP))) + 2 * U32 * np.abs(self.dq)
        self.unit_dk = a * (u * np.sqrt(group_sum((dsT ** 2) @ (qP ** 2), Hk)) + group_sum(np.swapaxes(sd, -1, -2) @ np.abs(qP), Hk)
                            + group_sum(np.swapaxes(e_ds, -1, -2) @ np.abs(qP), Hk) + U32 * np.sqrt(Sq * n_g + 2) * group_sum(np.abs(dsT) @ np.abs(qP), Hk)) + 2 * U32 * np.abs(self.dk)

    def out(self):
        """(dq, unit), (dk, unit), (dv, unit) in the tensors' [B, S, H, D] layout"""
        t = lambda x: np.ascontiguousarray(x.transpose(0, 2, 1, 3))
        return (t(self.dq), t(self.unit_dq)), (t(self.dk), t(self.unit_dk)), (t(self.dv), t(self.unit_dv))


# ------------------------------------------------------------------------------------------------ CPU_REF pins
# fp32 calls the oracle is pinned to CCV_NNC_BACKEND_CPU_REF with (tests/golden/cpuref_sdpa.npz holds inputs and outputs):
# (B, Sq, Sk, H, Hk, D, Dv, causal, mask shape or None, 3-d tensors, backward)
PINS = [
    (2, 24, 40, 4, 2, 16, 16, 1, None, False, True),   # GQA 2, causal with Sq < Sk
    (1, 40, 24, 4, 1, 8, 8, 1, None, False, True),     # GQA 4 (Hk = 1), causal with Sq > Sk: fully masked rows
    (2, 16, 20, 2, 2, 12, 20, 0, None, False, True),   # Dv != D
    (3, 17, 19, 1, 1, 8, 8, 0, None, True, True),      # 3-d [B, S, D] tensors
    (2, 12, 20, 2, 2, 8, 8, 0, (12, 20), False, False),
    (2, 12, 20, 2, 2, 8, 8, 0, (1, 2, 12, 20), False, False),
    (2, 12, 20, 2, 2, 8, 8, 1, (2, 1, 12, 20), False, False),
    (2, 12, 20, 2, 2, 8, 8, 0, (2, 2, 12, 20), False, False),
    (2, 12, 20, 2, 2, 8, 8, 0, (2, 12, 20), False, False),  # 3-d mask: [H, Sq, Sk]
]
CPU_MODEL = Model("cpu", None)


def pin_inputs(i):
    """seeded fp32 operands of PINS[i] in the tensors' own shapes: dict(q, k, v, do, mask, scale, causal, backward, three_d)"""
    B, Sq, Sk, H, Hk, D, Dv, causal, mshape, three, bwd = PINS[i]
    r = np.random.RandomState(100 + i)
    u = lambda shape, lo, hi: (lo + (hi - lo) * r.random_sample(shape)).astype(np.float32)
    sh = (lambda S, d: (B, S, d)) if three else (lambda S, d, h: (B, S, h, d))
    q = u(sh(Sq, D) if three else sh(Sq, D, H), -1, 1)
    k = u(sh(Sk, D) if three else sh(Sk, D, Hk), -1, 1)
    v = u(sh(Sk, Dv) if three else sh(Sk, Dv, Hk), -0.5, 1)
    do = u(sh(Sq, Dv) if three else sh(Sq, Dv, H), -0.5, 1)
    mask = np.where(r.random_sample(mshape) < 0.25, -30.0, 0.0).astype(np.float32) + u(mshape, -2, 2) if mshape else None
    return dict(q=q, k=k, v=v, do=do, mask=mask, scale=float(np.float32(1.0 / np.sqrt(D))), causal=causal, backward=bwd, three_d=three)


def as4(x, three_d):
    """a 3-d [B, S, D] tensor as the [B, S, 1, D] one it stands for"""
    return None if x is None else (np.asarray(x)[:, :, None, :] if three_d else np.asarray(x))


# ------------------------------------------------------------------------------------------------ bounds
def rounding_of(path, dtype):
    """how an output of this path reaches its tensor: fp32 | (rne, fmt) | (trunc, fmt)"""
    if dtype == FP32:
        return FP32
    if path == "func" and dtype == FP16:
        return ("trunc", FP16)
    return ("rne", dtype)


def _round(x, rnd):
    return rne16(x, rnd[1]) if rnd[0] == "rne" else trunc16(x, rnd[1])


def finish(y, rnd):
    """the oracle's (or a defective) float64 result as the output tensor would hold it"""
    if rnd == FP32:
        return np.asarray(y, np.float32).astype(np.float64)
    return _round(y, rnd)


def admits(y, ref, unit, rnd, c=C_ATT):
    y = np.asarray(y, np.float64)
    e = c * unit
    if rnd == FP32:
        return np.abs(y - ref) <= e  # NaN -> False
    return (_round(ref - e, rnd) <= y) & (y <= _round(ref + e, rnd))


def needed(y, ref, unit, rnd):
    """Per element, the smallest C for which the bound admits y (the calibration ratio); inf for non-finite y."""
    y = np.asarray(y, np.float64)
    if rnd == FP32:
        err = np.abs(y - ref)
    else:
        fmt = rnd[1]
        k = _key16(to_bits16(y, fmt))
        below, above = from_bits16(_unkey16(k - 1), fmt), from_bits16(_unkey16(k + 1), fmt)
        if rnd[0] == "rne":
            lo, hi = (y + below) / 2, (y + above) / 2
        else:  # toward zero: y collects [y, above) when y >= 0, (below, y] when y < 0
            lo, hi = np.where(y > 0, y, below), np.where(y < 0, y, above)
            lo = np.where(y == 0, below, lo)
        err = np.maximum(np.maximum(lo - ref, ref - hi), 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err > 0, err / np.maximum(unit, 1e-300), 0.0)
    return np.where(np.isfinite(y), r, np.inf)


def check(y, ref, unit, rnd, what="", c=C_ATT):
    """Assert the bound on every element; returns the largest calibration ratio."""
    ok = admits(y, ref, unit, rnd, c)
    if not ok.all():
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        raise AssertionError("%s: %d of %d elements outside the bound (C = %g); first at %s: got %r, oracle %r, unit %r"
                             % (what, len(bad), ok.size, c, i, np.asarray(y, np.float64)[i], ref[i], unit[i]))
    r = needed(y, ref, unit, rnd)
    return float(r.max()) if r.size else 0.0


def check_lse(y, ref, unit, what="", c=C_ATT):
    """fp32 log-sum-exp; fully masked rows must read -inf exactly"""
    y = np.asarray(y, np.float64)
    dead = ~np.isfinite(ref)
    assert (y[dead] == -np.inf).all(), "%s: a fully masked row's log-sum-exp is not -inf" % what
    return check(y[~dead], ref[~dead], unit[~dead], FP32, what, c) if (~dead).any() else 0.0
