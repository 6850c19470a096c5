// sm100_fmha_bwd.cu -- SCALED_DOT_PRODUCT_ATTENTION backward for 16-bit tensors (bf16 / fp16), head dimension <= 128 (multiples of 8;
// the tiles are always 128 features wide, missing features are zero-filled by the TMA unit and never stored): a fused
// flash-attention backward on the Hopper wgmma tensor cores, deterministic (no atomics, every sum in one fixed order).
// Semantics: scaled_dot_product_attention/ccv_nnc_scaled_dot_product_attention_cpu_ref.c:259-479 (dq, dk, dv of
// O = softmax(scale * Q K^T [causal, bottom-right aligned]) V, GQA gradients summed over the query heads of a key head); the reference's
// GPU form is gpu/ccv_nnc_scaled_dot_product_attention_flash_attn.cu:221-451 (recomputation from O and the saved log-sum-exp,
// :410-440 its deterministic split accumulator, :444-449 the GQA sum).
//
//   P  = exp(scale * Q K^T - LSE)            recomputed per tile from the saved log-sum-exp
//   dV = P^T dO
//   dP = dO V^T,   dS = P o (dP - delta),    delta_i = sum_d dO_id O_id
//   dQ = scale * dS K,   dK = scale * dS^T Q
//
// Three launches:
//   fmha_bwd_prep_kernel    (lse * log2 e, delta) pairs per query row, padded to whole tiles (padding rows: lse = +inf -> P = 0)
//   fmha_bwd_kernel<0>      one CTA per 128 keys of one (batch, KEY head): K, V tiles resident in shared memory, Q_i / dO_i blocks of
//                           64 queries streamed for every query head of the group; dV, dK accumulate in registers over the whole loop
//   fmha_bwd_kernel<1>      one CTA per 128 queries of one (batch, query head): Q, dO resident, K_j / V_j blocks of 64 keys streamed;
//                           dQ accumulates in registers
// Both recompute S and dP (7 GEMMs instead of 5) so that no gradient is ever accumulated across CTAs: that is what makes the result
// run-to-run identical without the reference's per-split fp32 dq_accum buffers.
//
// One kernel body serves both (MODE 0 = dK/dV, 1 = dQ).  R1 / R2 = the resident 128-row tiles, T1 / T2 = the streamed 64-row blocks:
//   MODE 0: R1 = K, R2 = V, T1 = Q_i, T2 = dO_i:  X = R1 T1^T = S^T,  Y = R2 T2^T = dP^T,  acc1 += P^T T2 (dV),  acc2 += dS^T T1 (dK)
//   MODE 1: R1 = Q, R2 = dO, T1 = K_j, T2 = V_j:  X = R1 T1^T = S,    Y = R2 T2^T = dP,    acc2 += dS T1 (dQ)
// 384 threads: warps 0-7 = two consumer warpgroups of 64 resident rows (X, Y from shared memory; P, dS turned into 16-bit register
// fragments that are the A operand of the accumulating MMAs, whose B operand is T1 / T2 read MN-major), warps 8-11 = the producer warpgroup (one thread issues the TMA loads; setmaxnreg moves its registers to the consumers).
// smem: R 64 KB + T ring 4 x 32 KB = 192 KB.
#include "sm100_contract.h"
#include "sm100_fmha.cuh"
#include <string.h>

namespace sm100 {

namespace {

constexpr int FB_R = 128;                     // resident rows per CTA
constexpr int FB_T = 64;                      // streamed rows per block
constexpr int FB_D = 128;                     // head dimension
constexpr int FB_R_ATOM = FB_R * 128;         // 16 KB: 128 rows x 64 features
constexpr int FB_R_BYTES = 2 * FB_R_ATOM;     // 32 KB
constexpr int FB_T_ATOM = FB_T * 128;         // 8 KB
constexpr int FB_T_BYTES = 2 * FB_T_ATOM;     // 16 KB
constexpr int FB_THREADS = 384;

struct FmhaBwdParams {
	int H, Hk, Sq, Sk, Sq_r;
	int D; // actual head dimension (<= 128, a multiple of 8): tiles are 128 wide, missing features are zero-filled and never stored
	int causal;
	int is_bf16;
	float scale, scale_log2;
	const float4* stat;          // [B, H, Sq_r / 2] (-lse2_0, -lse2_1, -delta_0, -delta_1) per query pair, lse2 = lse * log2 e
	void* out1;                  // MODE 0: dV
	void* out2;                  // MODE 0: dK, MODE 1: dQ
	long long o1_b, o1_s, o1_h;  // element strides
	long long o2_b, o2_s, o2_h;
};

struct FmhaBwdSmem {
	static constexpr int NST = 4;                 // stages of the streamed ring
	static constexpr int R1_OFF = 0;
	static constexpr int R2_OFF = R1_OFF + FB_R_BYTES;
	static constexpr int T_OFF = R2_OFF + FB_R_BYTES; // stage s: T1 at + s * 2 * FB_T_BYTES, T2 right behind it
	static constexpr int BAR_OFF = T_OFF + NST * 2 * FB_T_BYTES;
	static constexpr int TOTAL = BAR_OFF + 256 + 1024;
	static_assert(TOTAL <= 232448, "227 KB of shared memory per CTA");
};

// (-lse * log2 e, -delta) per query row: 16 lanes per row, 8 features each
__global__ void __launch_bounds__(256) fmha_bwd_prep_kernel(const uint16_t* __restrict__ dout, const uint16_t* __restrict__ out, const float* __restrict__ lse, float* __restrict__ stat, int B, int H, int Sq, int Sq_r, int D, int is_bf16,
	long long do_b, long long do_s, long long do_h, long long o_b, long long o_s, long long o_h)
{
	const long long row = (long long)blockIdx.x * 16 + (threadIdx.x >> 4);
	const int sub = threadIdx.x & 15;
	const long long rows = (long long)B * H * Sq_r;
	if (row >= rows)
		return;
	const int q = (int)(row % Sq_r);
	const int h = (int)((row / Sq_r) % H);
	const int b = (int)(row / ((long long)Sq_r * H));
	float acc = 0.f;
	if (q < Sq && sub * 8 < D)
	{
		const uint4 a = *reinterpret_cast<const uint4*>(dout + b * do_b + (long long)q * do_s + h * do_h + sub * 8);
		const uint4 c = *reinterpret_cast<const uint4*>(out + b * o_b + (long long)q * o_s + h * o_h + sub * 8);
		const uint32_t aw[4] = { a.x, a.y, a.z, a.w }, cw[4] = { c.x, c.y, c.z, c.w };
#pragma unroll
		for (int i = 0; i < 4; i++)
		{
			acc = fmaf(widen16((uint16_t)(aw[i] & 0xffff), is_bf16), widen16((uint16_t)(cw[i] & 0xffff), is_bf16), acc);
			acc = fmaf(widen16((uint16_t)(aw[i] >> 16), is_bf16), widen16((uint16_t)(cw[i] >> 16), is_bf16), acc);
		}
	}
	// fixed-order tree over the 16 lanes of the row
#pragma unroll
	for (int m = 8; m >= 1; m >>= 1)
		acc += __shfl_xor_sync(0xffffffffu, acc, m);
	if (sub == 0)
	{
		float l2 = INFINITY; // padding rows and fully masked rows (lse = -inf): P = exp2(x - inf) = 0
		if (q < Sq)
		{
			const float l = lse[((long long)b * H + h) * Sq + q];
			if (l != -INFINITY)
				l2 = l * 1.4426950408889634f;
		}
		// query pair (2j, 2j + 1) -> (-l, -l', -d, -d'): Sq_r is even, so a pair never straddles two heads
		float* const dst = stat + (row >> 1) * 4 + (row & 1);
		dst[0] = -l2;
		dst[2] = q < Sq ? -acc : 0.f;
	}
}

template <int MODE, int BF16> // element type as a template parameter: one basic block per MMA batch
__global__ void __launch_bounds__(FB_THREADS, 1) fmha_bwd_kernel(const __grid_constant__ CUtensorMap tmR1, const __grid_constant__ CUtensorMap tmR2, const __grid_constant__ CUtensorMap tmT1, const __grid_constant__ CUtensorMap tmT2, const FmhaBwdParams p)
{
	using L = FmhaBwdSmem;
	constexpr int NST = L::NST;
	extern __shared__ uint8_t smem_raw[];
	uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
	uint64_t* bars = (uint64_t*)(smem + L::BAR_OFF);
	uint64_t* r_full = bars;
	uint64_t* t_full = bars + 1;         // [NST]
	uint64_t* t_empty = bars + 1 + NST;  // [NST] one arrival per consumer warpgroup

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int r0 = blockIdx.x * FB_R;    // first resident row (MODE 0: key, MODE 1: query)
	const int hr = blockIdx.y, b = blockIdx.z; // MODE 0: key head, MODE 1: query head
	const int group = p.H / p.Hk;
	const int shift = p.Sk - p.Sq;       // causal: query i sees keys <= i + shift
	// streamed blocks: MODE 0 = (query head of the group, 64-query block) from the first block a key of this tile can see;
	// MODE 1 = 64-key blocks up to this tile's causal horizon
	int first = 0, n_per = 0, n_total = 0;
	if (MODE == 0)
	{
		const int nq = (p.Sq + FB_T - 1) / FB_T;
		first = p.causal ? min(nq, max(0, (r0 - shift) / FB_T)) : 0;
		n_per = nq - first;
		n_total = n_per * group;
	} else {
		const int kv_end = p.causal ? min(p.Sk, max(r0 + FB_R + shift, 0)) : p.Sk;
		n_per = n_total = (kv_end + FB_T - 1) / FB_T;
	}

	if (threadIdx.x == 0)
	{
		mbar_init(r_full, 1);
		for (int s = 0; s < NST; s++)
			mbar_init(&t_full[s], 1), mbar_init(&t_empty[s], 2);
		fence_mbar_init();
	}
	__syncthreads();

	if (warp >= 8)
	{
		// the producer warpgroup hands most of its registers to the consumers (dV and dK accumulators: 128 fp32 registers per thread)
		asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
		if (warp == 8 && elect_one())
		{
			tma_prefetch_desc(&tmR1);
			tma_prefetch_desc(&tmR2);
			tma_prefetch_desc(&tmT1);
			tma_prefetch_desc(&tmT2);
			mbar_expect_tx(r_full, 2 * FB_R_BYTES);
			for (int a = 0; a < 2; a++)
			{
				tma_load_4d(smem + L::R1_OFF + a * FB_R_ATOM, &tmR1, r_full, 64 * a, hr, r0, b);
				tma_load_4d(smem + L::R2_OFF + a * FB_R_ATOM, &tmR2, r_full, 64 * a, hr, r0, b);
			}
			for (int n = 0; n < n_total; n++)
			{
				const int s = n % NST;
				const uint32_t ph = (uint32_t)(n / NST) & 1;
				const int row = MODE == 0 ? (first + n % n_per) * FB_T : n * FB_T;
				const int head = MODE == 0 ? hr * group + n / n_per : hr / group; // MODE 0: query head of the group; MODE 1: the key head
				uint8_t* const t1 = smem + L::T_OFF + s * 2 * FB_T_BYTES;
				mbar_wait(&t_empty[s], ph ^ 1);
				mbar_expect_tx(&t_full[s], 2 * FB_T_BYTES);
				for (int a = 0; a < 2; a++)
				{
					tma_load_4d(t1 + a * FB_T_ATOM, &tmT1, &t_full[s], 64 * a, head, row, b);
					tma_load_4d(t1 + FB_T_BYTES + a * FB_T_ATOM, &tmT2, &t_full[s], 64 * a, head, row, b);
				}
			}
		}
		return;
	}

	// ------------------------------------------------------------------ consumers: resident rows rr + 8 * hh of this thread
	asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
	const int wg = warp >> 2, t4 = lane & 3;
	const int rr = r0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
	constexpr int is_bf16 = BF16;
	float acc1[64], acc2[64]; // acc1: MODE 0 only
#pragma unroll
	for (int i = 0; i < 64; i++)
		acc2[i] = 0.f;
#pragma unroll
	for (int i = 0; i < 64; i++)
		acc1[i] = 0.f;
	// MODE 1: the (-lse2, -delta) of the thread's two query rows, fixed for the whole loop
	float nl[2] = { 0.f, 0.f }, nd[2] = { 0.f, 0.f };
	if (MODE == 1)
	{
#pragma unroll
		for (int hh = 0; hh < 2; hh++)
		{
			const int q = rr + 8 * hh;
			const float4 st = p.stat[(((long long)b * p.H + hr) * p.Sq_r + q) >> 1];
			nl[hh] = (q & 1) ? st.y : st.x;
			nd[hh] = (q & 1) ? st.w : st.z;
		}
	}
	const uint32_t r1_base = smem_u32(smem + L::R1_OFF) + wg * 8192, r2_base = smem_u32(smem + L::R2_OFF) + wg * 8192;
	mbar_wait(r_full, 0);
	for (int n = 0; n < n_total; n++)
	{
		const int s = n % NST;
		const uint32_t ph = (uint32_t)(n / NST) & 1;
		const int c0 = MODE == 0 ? (first + n % n_per) * FB_T : n * FB_T; // first streamed row (MODE 0: query, MODE 1: key)
		const int hq = MODE == 0 ? hr * group + n / n_per : hr;
		mbar_wait(&t_full[s], ph);
		const uint32_t t1_base = smem_u32(smem + L::T_OFF + s * 2 * FB_T_BYTES), t2_base = t1_base + FB_T_BYTES;
		float x[32], y[32];
#pragma unroll
		for (int i = 0; i < 32; i++)
			x[i] = y[i] = 0.f;
		fence_regs(x);
		fence_regs(y);
		wgmma_fence();
#pragma unroll
		for (int k = 0; k < FB_D / 16; k++)
		{
			const uint32_t roff = (uint32_t)(k >> 2) * FB_R_ATOM + (uint32_t)(k & 3) * 32, toff = (uint32_t)(k >> 2) * FB_T_ATOM + (uint32_t)(k & 3) * 32;
			if constexpr (BF16 != 0)
			{
				wgmma_bf16_ss_n64<0, 0>(x, wgmma_desc(r1_base + roff, 16, 1024), wgmma_desc(t1_base + toff, 16, 1024));
				wgmma_bf16_ss_n64<0, 0>(y, wgmma_desc(r2_base + roff, 16, 1024), wgmma_desc(t2_base + toff, 16, 1024));
			} else {
				wgmma_f16_ss_n64<0, 0>(x, wgmma_desc(r1_base + roff, 16, 1024), wgmma_desc(t1_base + toff, 16, 1024));
				wgmma_f16_ss_n64<0, 0>(y, wgmma_desc(r2_base + roff, 16, 1024), wgmma_desc(t2_base + toff, 16, 1024));
			}
		}
		wgmma_commit();
		fence_regs(x);
		fence_regs(y);
		wgmma_wait<0>();
		fence_regs(x);
		fence_regs(y);
		// accumulator i: resident row rr + 8 * ((i >> 1) & 1), streamed column c0 + 8 * (i >> 2) + 2 * t4 + (i & 1).
		// P = exp2(scale_log2 * X - lse2) (0 where the causal mask hides the pair, or the key is past Sk), dS = P (Y - delta)
#pragma unroll
		for (int jn = 0; jn < 8; jn++)
		{
			const int c = c0 + 8 * jn + 2 * t4;
			float cl[2], cd[2];
			if (MODE == 0)
			{
				const float4 st = p.stat[(((long long)b * p.H + hq) * p.Sq_r + c) >> 1];
				cl[0] = st.x, cl[1] = st.y, cd[0] = st.z, cd[1] = st.w;
			}
#pragma unroll
			for (int e = 0; e < 4; e++)
			{
				const int i = 4 * jn + e, hh = e >> 1, col = c + (e & 1);
				const int row = rr + 8 * hh;
				const float lse2 = MODE == 0 ? cl[e & 1] : nl[hh];
				const float delta = MODE == 0 ? cd[e & 1] : nd[hh];
				const int key = MODE == 0 ? row : col, query = MODE == 0 ? col : row;
				const bool visible = key < p.Sk && (!p.causal || key <= query + shift);
				const float pv = visible ? ex2_approx(fmaf(x[i], p.scale_log2, lse2)) : 0.f;
				x[i] = pv;
				y[i] = pv * (y[i] + delta);
			}
		}
		// every A fragment is packed before the MMAs start: registers an in-flight wgmma reads must not be written between them
		uint32_t fp[FB_T / 16][4], fds[FB_T / 16][4];
#pragma unroll
		for (int kk = 0; kk < FB_T / 16; kk++)
		{
			acc_to_a(y, kk, is_bf16, fds[kk]);
			if constexpr (MODE == 0)
				acc_to_a(x, kk, is_bf16, fp[kk]);
		}
		fence_regs(acc2);
		if constexpr (MODE == 0)
			fence_regs(acc1);
		wgmma_fence();
#pragma unroll
		for (int kk = 0; kk < FB_T / 16; kk++)
		{
			// T1 / T2 [64 streamed rows x 128 d] as MN-major B operands: d atoms 8 KB apart (LBO), 8-row groups 1 KB apart, 16 rows = 2 KB per MMA
			const uint64_t d1 = wgmma_desc(t1_base + kk * 2048, FB_T_ATOM, 1024), d2 = wgmma_desc(t2_base + kk * 2048, FB_T_ATOM, 1024);
			const uint32_t (&ap)[4] = fp[kk], (&ads)[4] = fds[kk];
			if constexpr (BF16 != 0)
			{
				if constexpr (MODE == 0)
					wgmma_bf16_rs_n128<1>(acc1, ap, d2);
				wgmma_bf16_rs_n128<1>(acc2, ads, d1);
			} else {
				if constexpr (MODE == 0)
					wgmma_f16_rs_n128<1>(acc1, ap, d2);
				wgmma_f16_rs_n128<1>(acc2, ads, d1);
			}
		}
		wgmma_commit();
		fence_regs(acc2);
		if constexpr (MODE == 0)
			fence_regs(acc1);
		wgmma_wait<0>();
		fence_regs(acc2);
		if constexpr (MODE == 0)
			fence_regs(acc1);
		if ((threadIdx.x & 127) == 0)
			mbar_arrive(&t_empty[s]);
	}
	// epilogue: MODE 0 writes dV (acc1) and scale * dK (acc2) for keys < Sk; MODE 1 scale * dQ for queries < Sq
#pragma unroll
	for (int hh = 0; hh < 2; hh++)
	{
		const int row = rr + 8 * hh;
		if (row >= (MODE == 0 ? p.Sk : p.Sq))
			continue;
		uint16_t* const o2 = (uint16_t*)p.out2 + b * p.o2_b + (long long)row * p.o2_s + hr * p.o2_h;
		uint16_t* const o1 = MODE == 0 ? (uint16_t*)p.out1 + b * p.o1_b + (long long)row * p.o1_s + hr * p.o1_h : 0;
#pragma unroll
		for (int jn = 0; jn < 16; jn++)
		{
			const int d = 8 * jn + 2 * t4;
			if (d >= p.D)
				continue;
			const int i = 4 * jn + 2 * hh;
			*reinterpret_cast<uint32_t*>(o2 + d) = pack2(acc2[i] * p.scale, acc2[i + 1] * p.scale, is_bf16);
			if (MODE == 0)
				*reinterpret_cast<uint32_t*>(o1 + d) = pack2(acc1[i], acc1[i + 1], is_bf16);
		}
	}
}

template <int MODE, int BF16>
int launch_bwd_t(cudaStream_t stream, const CUtensorMap& r1, const CUtensorMap& r2, const CUtensorMap& t1, const CUtensorMap& t2, const FmhaBwdParams& p, int tiles, int heads, int B)
{
	static bool configured_on[64]; // the attribute is per device
	int dev = 0;
	cudaGetDevice(&dev);
	bool& configured = configured_on[dev & 63];
	if (!configured)
	{
		const cudaError_t e = cudaFuncSetAttribute(fmha_bwd_kernel<MODE, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, FmhaBwdSmem::TOTAL);
		if (e != cudaSuccess)
		{
			set_last_error("cudaFuncSetAttribute(fmha_bwd_kernel)", e);
			return -1;
		}
		configured = true;
	}
	fmha_bwd_kernel<MODE, BF16><<<dim3(tiles, heads, B), FB_THREADS, FmhaBwdSmem::TOTAL, stream>>>(r1, r2, t1, t2, p);
	return launched("fmha_bwd_kernel launch");
}

template <int MODE>
int launch_bwd(cudaStream_t stream, const CUtensorMap& r1, const CUtensorMap& r2, const CUtensorMap& t1, const CUtensorMap& t2, const FmhaBwdParams& p, int tiles, int heads, int B)
{
	return p.is_bf16 ? launch_bwd_t<MODE, 1>(stream, r1, r2, t1, t2, p, tiles, heads, B) : launch_bwd_t<MODE, 0>(stream, r1, r2, t1, t2, p, tiles, heads, B);
}

} // namespace

size_t sdpa_backward_f16_workspace_bytes(const SdpaGeom& g, int need_forward)
{
	const size_t sq_r = (size_t)(g.Sq + FB_R - 1) / FB_R * FB_R;
	size_t bytes = (size_t)g.B * g.H * sq_r * 2 * sizeof(float) + 256;
	if (need_forward) // O (16-bit, packed [B, Sq, H, D]) and the log-sum-exp [B, H, Sq]
		bytes += (size_t)g.B * g.Sq * g.H * g.Dv * 2 + 256 + (size_t)g.B * g.H * g.Sq * sizeof(float) + 256;
	return bytes;
}

// g: q / k / v strides, o_* = the strides of dout; dg: the strides of dq / dk / dv in its q_* / k_* / v_* fields.  `out` (strides oo_*)
// and `lse` are the forward's saved outputs; when either is NULL both are recomputed into the workspace with the forward kernel.
// returns 0 on success, 1 when the shape is outside these kernels (D = Dv <= 128 and a multiple of 8, 16-byte aligned strides), < 0 on CUDA errors
bool sdpa_backward_f16_takes(const SdpaGeom& g, const SdpaGeom& dg, const int wide, const void* const* const ptrs, const int ptr_count)
{
	const bool d_ok = wide ? g.D > FB_D && g.D <= 256 : g.D >= 8 && g.D <= FB_D;
	if (!d_ok || (g.D & 7) || g.Dv != g.D || g.B <= 0 || g.H <= 0 || g.Hk <= 0 || g.H % g.Hk != 0 || g.Sq <= 0 || g.Sk <= 0)
		return false;
	for (int i = 0; i < ptr_count; i++)
		if (((uintptr_t)ptrs[i]) & 15)
			return false;
	for (const long long st : { g.q_b, g.q_s, g.q_h, g.k_b, g.k_s, g.k_h, g.v_b, g.v_s, g.v_h, dg.q_b, dg.q_s, dg.q_h, dg.k_b, dg.k_s, dg.k_h, dg.v_b, dg.v_s, dg.v_h, g.o_b, g.o_s, g.o_h })
		if (st & 7)
			return false;
	return true;
}

int sdpa_backward_f16(cudaStream_t stream, const SdpaGeom& g, const SdpaGeom& dg, int is_bf16, const void* dout, const void* q, const void* k, const void* v, const void* out, long long oo_b, long long oo_s, long long oo_h,
	const float* lse, void* dq, void* dk, void* dv, void* workspace)
{
	const void* const ptrs[7] = { dq, dk, dv, dout, q, k, v };
	if (!sdpa_backward_f16_takes(g, dg, 0, ptrs, 7) || !encode_init())
		return 1;
	CUtensorMap tmQr, tmQt, tmKr, tmKt, tmVr, tmVt, tmGr, tmGt;
	if (!make_map_bshd(&tmQr, q, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h, is_bf16, FB_R) || !make_map_bshd(&tmQt, q, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h, is_bf16, FB_T) ||
		!make_map_bshd(&tmKr, k, g.B, g.Sk, g.Hk, g.D, g.k_b, g.k_s, g.k_h, is_bf16, FB_R) || !make_map_bshd(&tmKt, k, g.B, g.Sk, g.Hk, g.D, g.k_b, g.k_s, g.k_h, is_bf16, FB_T) ||
		!make_map_bshd(&tmVr, v, g.B, g.Sk, g.Hk, g.Dv, g.v_b, g.v_s, g.v_h, is_bf16, FB_R) || !make_map_bshd(&tmVt, v, g.B, g.Sk, g.Hk, g.Dv, g.v_b, g.v_s, g.v_h, is_bf16, FB_T) ||
		!make_map_bshd(&tmGr, dout, g.B, g.Sq, g.H, g.Dv, g.o_b, g.o_s, g.o_h, is_bf16, FB_R) || !make_map_bshd(&tmGt, dout, g.B, g.Sq, g.H, g.Dv, g.o_b, g.o_s, g.o_h, is_bf16, FB_T))
		return 1;
	const int sq_r = (g.Sq + FB_R - 1) / FB_R * FB_R;
	uint8_t* ws = (uint8_t*)workspace;
	float* const stat = (float*)ws;
	ws += (((size_t)g.B * g.H * sq_r * 2 * sizeof(float)) + 255) & ~(size_t)255;
	if (!out || !lse)
	{
		void* const o_ws = ws;
		ws += (((size_t)g.B * g.Sq * g.H * g.Dv * 2) + 255) & ~(size_t)255;
		float* const lse_ws = (float*)ws;
		SdpaGeom fg = g;
		fg.o_h = g.Dv, fg.o_s = (long long)g.H * g.Dv, fg.o_b = (long long)g.Sq * g.H * g.Dv;
		const int rc = sdpa_forward_f16(stream, fg, is_bf16, q, k, v, o_ws, lse_ws);
		if (rc != 0)
			return rc;
		out = o_ws, lse = lse_ws;
		oo_b = fg.o_b, oo_s = fg.o_s, oo_h = fg.o_h;
	}
	if ((((uintptr_t)out) & 15) || (oo_b & 7) || (oo_s & 7) || (oo_h & 7))
		return 1;
	const long long rows = (long long)g.B * g.H * sq_r;
	fmha_bwd_prep_kernel<<<(unsigned)((rows + 15) / 16), 256, 0, stream>>>((const uint16_t*)dout, (const uint16_t*)out, lse, stat, g.B, g.H, g.Sq, sq_r, g.D, is_bf16, g.o_b, g.o_s, g.o_h, oo_b, oo_s, oo_h);
	count_launch();
	FmhaBwdParams p;
	memset(&p, 0, sizeof(p));
	p.H = g.H, p.Hk = g.Hk, p.Sq = g.Sq, p.Sk = g.Sk, p.Sq_r = sq_r, p.D = g.D;
	p.causal = g.is_causal, p.is_bf16 = is_bf16;
	p.scale = g.scale, p.scale_log2 = g.scale * 1.4426950408889634f;
	p.stat = (const float4*)stat;
	// dK, dV: one CTA per 128 keys of a (batch, key head)
	p.out1 = dv, p.o1_b = dg.v_b, p.o1_s = dg.v_s, p.o1_h = dg.v_h;
	p.out2 = dk, p.o2_b = dg.k_b, p.o2_s = dg.k_s, p.o2_h = dg.k_h;
	int rc = launch_bwd<0>(stream, tmKr, tmVr, tmQt, tmGt, p, (g.Sk + FB_R - 1) / FB_R, g.Hk, g.B);
	if (rc != 0)
		return rc;
	// dQ: one CTA per 128 queries of a (batch, query head)
	p.out1 = 0;
	p.out2 = dq, p.o2_b = dg.q_b, p.o2_s = dg.q_s, p.o2_h = dg.q_h;
	return launch_bwd<1>(stream, tmQr, tmGr, tmKt, tmVt, p, (g.Sq + FB_R - 1) / FB_R, g.H, g.B);
}

} // namespace sm100
