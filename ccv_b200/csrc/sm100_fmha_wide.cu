// sm100_fmha_wide.cu -- SCALED_DOT_PRODUCT_ATTENTION for 16-bit tensors (bf16 / fp16) with wide heads, 128 < D = Dv <= 256 (multiples
// of 8): a flash-attention forward and a fused, deterministic backward on the Hopper wgmma tensor cores.  They are algorithm 1
// (CCV_NNC_SM100_SDPA_ALGO_FLASH) of the command; algorithm 0 runs these head dimensions through the fp32 functional form.
// Semantics are those of sm100_fmha.cu / sm100_fmha_bwd.cu (causal masks aligned bottom-right, GQA through H / Hk, fully masked rows
// give O = 0 and LSE = -inf, the log-sum-exp as [B, H, Sq] fp32, any 16-byte aligned strides); the reference's flash backend takes
// these head dimensions with 64-key blocks (gpu/ccv_nnc_scaled_dot_product_attention_flash_attn.cu:175).
//
// Every tile is 256 features wide: four 64-feature, 128-byte-swizzled atoms (make_map_bshd's box).  The TMA unit zero-fills the
// features from D to 255 and the epilogues store only d < D, so 128 < D < 256 runs on the same tiles.
//
// Forward: one CTA = 128 query rows of one (batch, head); 384 threads.
//   warps 0-7   two consumer warpgroups of 64 query rows.  Per block of 64 keys: S_j = Q K_j^T (wgmma n64, 16 k-steps), online
//               softmax in registers, O += P_j V_j as two n128 MMAs per 16 keys (features 0-127 and 128-255).  O is 64 x 256 fp32 per
//               warpgroup = 128 registers per thread, S 32 more
//   warps 8-11  producer warpgroup: one thread issues the TMA loads (Q once, K_j / V_j through two-stage rings); setmaxnreg gives its
//               registers to the consumers (24 / 240 instead of 168 each)
//   smem: Q 64 KB + K 2 x 32 KB + V 2 x 32 KB = 192 KB.
//   MASK (1 = fp32, 2 = 16-bit; CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK): an additive mask, staged and applied as in sm100_fmha.cu.  Its tile
//   per key block (128 query rows x 64 keys) takes one more buffer of 32 KB fp32 / 16 KB 16-bit: 224 / 208 KB in all.
//
// Backward (the equations of sm100_fmha_bwd.cu): prep (lse * log2 e, delta) + one dK/dV launch + one dQ launch, no atomics.  A CTA
// holds 64 resident rows (MODE 0: keys of a key head, MODE 1: queries of a query head) and streams 64-row blocks of the other side.
// dK + dV for 64 keys x 256 features is 256 fp32 registers per thread in one warpgroup, so the feature axis is split instead of the
// rows: warpgroup w owns features [128 w, 128 w + 128) of every accumulator (dV and dK, or dQ: 64 x 128 each, 64 registers).  Both
// need the whole 64 x 64 P and dP of a block; warpgroup 0 computes X = R1 T1^T, warpgroup 1 Y = R2 T2^T (each the full 256-feature
// reduction, so the work stays even), and they swap the fp32 results through shared memory.  Both then form P and dS from the same
// values with the same instructions, so the two halves of a gradient row come from identical P / dS.
//   smem: R1 32 KB + R2 32 KB + T ring 2 x (32 + 32) KB + exchange 32 KB = 224 KB.  Registers: producer 40, consumers 232 (setmaxnreg).
#include "sm100_contract.h"
#include "sm100_fmha.cuh"
#include <string.h>

namespace sm100 {

namespace {

constexpr int FW_D = 256;                      // tile width in features
constexpr int FW_Q = 128;                      // forward: query rows per CTA
constexpr int FW_K = 64;                       // forward: keys per block; backward: resident and streamed rows
constexpr int FW_Q_ATOM = FW_Q * 128;          // 16 KB: 128 rows x 64 features
constexpr int FW_ATOM = FW_K * 128;            // 8 KB: 64 rows x 64 features
constexpr int FW_Q_BYTES = 4 * FW_Q_ATOM;      // 64 KB
constexpr int FW_TILE = 4 * FW_ATOM;           // 32 KB
constexpr int FW_THREADS = 384;
constexpr int FW_STAT_ROWS = 128;              // the statistics rows are padded as sdpa_backward_f16_workspace_bytes pads them

struct WideFwdParams {
	int H, Hk, Sq, Sk;
	int D; // actual head dimension (129..256, a multiple of 8)
	int causal;
	float scale_log2; // scale * log2(e)
	void* o;
	long long o_b, o_s, o_h; // element strides
	float* lse;              // [B, H, Sq] or NULL
	// MASK only
	float scale;
	int mask_h, mask_b; // the mask has a head / batch axis (else broadcast)
};

template <int MASK>
struct WideFwdSmem {
	static constexpr int Q_OFF = 0;
	static constexpr int K_OFF = Q_OFF + FW_Q_BYTES;
	static constexpr int V_OFF = K_OFF + 2 * FW_TILE;
	static constexpr int M_OFF = V_OFF + 2 * FW_TILE;
	static constexpr int M_BYTES = MASK == 0 ? 0 : FW_Q * FW_K * (MASK == 1 ? 4 : 2);
	static constexpr int BAR_OFF = M_OFF + M_BYTES;
	static constexpr int TOTAL = BAR_OFF + 256 + 1024;
	static_assert(TOTAL <= 232448, "227 KB of shared memory per CTA");
};

template <int BF16, int MASK>
__global__ void __launch_bounds__(FW_THREADS, 1) fmha_wide_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const WideFwdParams p, const __grid_constant__ CUtensorMap tmM)
{
	using L = WideFwdSmem<MASK>;
	extern __shared__ uint8_t smem_raw[];
	uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
	uint64_t* bars = (uint64_t*)(smem + L::BAR_OFF);
	uint64_t* q_full = bars;
	uint64_t* k_full = bars + 1;  // [2]
	uint64_t* k_empty = bars + 3; // [2] one arrival per consumer warpgroup
	uint64_t* v_full = bars + 5;  // [2]
	uint64_t* v_empty = bars + 7; // [2]
	uint64_t* m_full = bars + 9;
	uint64_t* m_empty = bars + 10; // one arrival per consumer warp

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	// causal: the last query tiles see the most keys; issue them first so the tail of the launch is made of short tiles
	const int q_tile = p.causal ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x;
	const int q0 = q_tile * FW_Q;
	const int h = blockIdx.y, b = blockIdx.z;
	const int hk = h / (p.H / p.Hk);
	const int shift = p.Sk - p.Sq; // causal: query i sees keys <= i + shift
	int kv_end = p.Sk;
	if (p.causal)
		kv_end = min(p.Sk, max(q0 + FW_Q + shift, 0));
	const int n_blk = (kv_end + FW_K - 1) / FW_K;

	if (threadIdx.x == 0)
	{
		mbar_init(q_full, 1);
		for (int s = 0; s < 2; s++)
		{
			mbar_init(&k_full[s], 1), mbar_init(&k_empty[s], 2);
			mbar_init(&v_full[s], 1), mbar_init(&v_empty[s], 2);
		}
		if constexpr (MASK != 0)
			mbar_init(m_full, 1), mbar_init(m_empty, 8);
		fence_mbar_init();
	}
	__syncthreads();

	if (warp >= 8)
	{
		setmaxnreg_dec<24>();
		if (warp == 8 && n_blk > 0 && elect_one())
		{
			tma_prefetch_desc(&tmQ);
			tma_prefetch_desc(&tmK);
			tma_prefetch_desc(&tmV);
			if constexpr (MASK != 0)
				tma_prefetch_desc(&tmM);
			mbar_expect_tx(q_full, FW_Q_BYTES);
			for (int a = 0; a < 4; a++)
				tma_load_4d(smem + L::Q_OFF + a * FW_Q_ATOM, &tmQ, q_full, 64 * a, h, q0, b);
			for (int j = 0; j < n_blk; j++)
			{
				const int s = j & 1;
				const uint32_t ph = (uint32_t)(j >> 1) & 1;
				uint8_t* const sk = smem + L::K_OFF + s * FW_TILE;
				uint8_t* const sv = smem + L::V_OFF + s * FW_TILE;
				mbar_wait(&k_empty[s], ph ^ 1);
				mbar_expect_tx(&k_full[s], FW_TILE);
				for (int a = 0; a < 4; a++)
					tma_load_4d(sk + a * FW_ATOM, &tmK, &k_full[s], 64 * a, hk, j * FW_K, b);
				if constexpr (MASK != 0)
				{
					mbar_wait(m_empty, ((uint32_t)j & 1) ^ 1);
					mbar_expect_tx(m_full, L::M_BYTES);
					for (int a = 0; a < L::M_BYTES / MASK_ATOM_BYTES; a++)
						tma_load_4d(smem + L::M_OFF + a * MASK_ATOM_BYTES, &tmM, m_full, j * FW_K + a * (MASK == 1 ? 32 : 64), q0, p.mask_h ? h : 0, p.mask_b ? b : 0);
				}
				mbar_wait(&v_empty[s], ph ^ 1);
				mbar_expect_tx(&v_full[s], FW_TILE);
				for (int a = 0; a < 4; a++)
					tma_load_4d(sv + a * FW_ATOM, &tmV, &v_full[s], 64 * a, hk, j * FW_K, b);
			}
		}
		return;
	}

	// ------------------------------------------------------------------ consumers: rows r0 and r0 + 8 of this thread
	setmaxnreg_inc<240>();
	const int wg = warp >> 2;
	const int t4 = lane & 3;
	const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
	int kv_limit[2]; // keys [0, kv_limit) are visible to the row
#pragma unroll
	for (int hh = 0; hh < 2; hh++)
		kv_limit[hh] = p.causal ? min(p.Sk, q0 + r0 + 8 * hh + shift + 1) : p.Sk;
	float o0[64], o1[64], sacc[32]; // O features 0-127 and 128-255
#pragma unroll
	for (int i = 0; i < 64; i++)
		o0[i] = o1[i] = 0.f;
	float m[2] = { -INFINITY, -INFINITY }, l[2] = { 0.f, 0.f };
	const uint32_t q_base = smem_u32(smem + L::Q_OFF) + wg * 8192;
	if (n_blk > 0)
		mbar_wait(q_full, 0);
	for (int j = 0; j < n_blk; j++)
	{
		const int s = j & 1;
		const uint32_t ph = (uint32_t)(j >> 1) & 1;
		// S_j = Q K_j^T
		mbar_wait(&k_full[s], ph);
		const uint32_t k_base = smem_u32(smem + L::K_OFF + s * FW_TILE);
#pragma unroll
		for (int i = 0; i < 32; i++)
			sacc[i] = 0.f;
		fence_regs(sacc);
		wgmma_fence();
#pragma unroll
		for (int k = 0; k < FW_D / 16; k++)
		{
			const uint64_t dq = wgmma_desc(q_base + (uint32_t)(k >> 2) * FW_Q_ATOM + (uint32_t)(k & 3) * 32, 16, 1024);
			const uint64_t dk = wgmma_desc(k_base + (uint32_t)(k >> 2) * FW_ATOM + (uint32_t)(k & 3) * 32, 16, 1024);
			if constexpr (BF16 != 0)
				wgmma_bf16_ss_n64<0, 0>(sacc, dq, dk);
			else
				wgmma_f16_ss_n64<0, 0>(sacc, dq, dk);
		}
		wgmma_commit();
		fence_regs(sacc);
		wgmma_wait<0>();
		fence_regs(sacc);
		if ((threadIdx.x & 127) == 0)
			mbar_arrive(&k_empty[s]);
		// online softmax: key of accumulator i = j * 64 + 8 * (i >> 2) + 2 * t4 + (i & 1), row r0 + 8 * ((i >> 1) & 1)
		const int kv0 = j * FW_K + 2 * t4;
		const bool edge = j * FW_K + FW_K > min(kv_limit[0], kv_limit[1]);
		if constexpr (MASK != 0)
		{
			// t = scale * s + mask in CPU_REF's order; keys past the row's horizon are overwritten with -inf below
			mbar_wait(m_full, (uint32_t)j & 1);
			add_mask<MASK, BF16>(sacc, smem + L::M_OFF, r0, t4, p.scale);
			__syncwarp();
			if (lane == 0)
				mbar_arrive(m_empty);
		}
		// the running max and the exponents in log2 units: S scaled here, or the masked t = scale * S + mask
		const float scale_log2 = MASK != 0 ? 1.4426950408889634f : p.scale_log2;
		float mx[2] = { -INFINITY, -INFINITY };
#pragma unroll
		for (int i = 0; i < 32; i++)
		{
			const int hh = (i >> 1) & 1;
			if (edge && kv0 + 8 * (i >> 2) + (i & 1) >= kv_limit[hh])
				sacc[i] = -INFINITY;
			mx[hh] = fmaxf(mx[hh], sacc[i]);
		}
		float alpha[2], m_use[2];
#pragma unroll
		for (int hh = 0; hh < 2; hh++)
		{
			mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
			mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
			const float m_new = fmaxf(m[hh], mx[hh] * scale_log2);
			m_use[hh] = m_new == -INFINITY ? 0.f : m_new; // a fully masked row keeps p = 0 without NaN
			alpha[hh] = exp2f(m[hh] - m_use[hh]);          // m = -inf -> 0
			m[hh] = m_new;
		}
		float sum[2] = { 0.f, 0.f };
#pragma unroll
		for (int i = 0; i < 32; i++)
		{
			const int hh = (i >> 1) & 1;
			const float e = ex2_approx(fmaf(sacc[i], scale_log2, -m_use[hh])); // exp2(-inf) = 0 for the masked keys
			sacc[i] = e;
			sum[hh] += e;
		}
#pragma unroll
		for (int i = 0; i < 64; i++)
		{
			const int hh = (i >> 1) & 1;
			o0[i] *= alpha[hh];
			o1[i] *= alpha[hh];
		}
		l[0] = fmaf(l[0], alpha[0], sum[0]), l[1] = fmaf(l[1], alpha[1], sum[1]);
		// O += P_j V_j
		mbar_wait(&v_full[s], ph);
		const uint32_t v_base = smem_u32(smem + L::V_OFF + s * FW_TILE);
		// every A fragment is packed before the MMAs start: registers an in-flight wgmma reads must not be written between them
		uint32_t pa[FW_K / 16][4];
#pragma unroll
		for (int kk = 0; kk < FW_K / 16; kk++)
			acc_to_a(sacc, kk, BF16, pa[kk]);
		fence_regs(o0);
		fence_regs(o1);
		wgmma_fence();
#pragma unroll
		for (int kk = 0; kk < FW_K / 16; kk++)
		{
			const uint32_t (&a)[4] = pa[kk];
			// V [64 keys x 256 d] as MN-major B operands: 64-wide d atoms 8 KB apart (LBO), 8-key groups 1 KB apart (SBO), 16 keys =
			// 2 KB per MMA; features 128-255 start two atoms in
			const uint64_t dv0 = wgmma_desc(v_base + kk * 2048, FW_ATOM, 1024), dv1 = wgmma_desc(v_base + 2 * FW_ATOM + kk * 2048, FW_ATOM, 1024);
			if constexpr (BF16 != 0)
			{
				wgmma_bf16_rs_n128<1>(o0, a, dv0);
				wgmma_bf16_rs_n128<1>(o1, a, dv1);
			} else {
				wgmma_f16_rs_n128<1>(o0, a, dv0);
				wgmma_f16_rs_n128<1>(o1, a, dv1);
			}
		}
		wgmma_commit();
		fence_regs(o0);
		fence_regs(o1);
		wgmma_wait<0>();
		fence_regs(o0);
		fence_regs(o1);
		if ((threadIdx.x & 127) == 0)
			mbar_arrive(&v_empty[s]);
	}
	// the row sum is spread over the quad's four lanes
#pragma unroll
	for (int hh = 0; hh < 2; hh++)
	{
		l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
		l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
	}
#pragma unroll
	for (int hh = 0; hh < 2; hh++)
	{
		const int qi = q0 + r0 + 8 * hh;
		if (qi >= p.Sq)
			continue;
		const float inv = l[hh] > 0.f ? 1.f / l[hh] : 0.f;
		uint16_t* const orow = (uint16_t*)p.o + b * p.o_b + (long long)qi * p.o_s + h * p.o_h;
#pragma unroll
		for (int jn = 0; jn < 16; jn++)
		{
			const int d = 8 * jn + 2 * t4;
			*reinterpret_cast<uint32_t*>(orow + d) = pack2(o0[4 * jn + 2 * hh] * inv, o0[4 * jn + 2 * hh + 1] * inv, BF16); // D > 128
			if (d + 128 < p.D) // the padded feature columns are not part of the tensor
				*reinterpret_cast<uint32_t*>(orow + d + 128) = pack2(o1[4 * jn + 2 * hh] * inv, o1[4 * jn + 2 * hh + 1] * inv, BF16);
		}
		if (p.lse && t4 == 0) // (a NaN in the mask makes l NaN: the masked kernels pass it on)
			p.lse[((long long)b * p.H + h) * p.Sq + qi] = (MASK != 0 ? l[hh] != 0.f : l[hh] > 0.f) ? (m[hh] + log2f(l[hh])) * 0.6931471805599453f : -INFINITY;
	}
}

// ------------------------------------------------------------------------------------------------ backward
struct WideBwdParams {
	int H, Hk, Sq, Sk, Sq_r;
	int D;
	int causal;
	float scale, scale_log2;
	const float4* stat;          // [B, H, Sq_r / 2] (-lse2_0, -lse2_1, -delta_0, -delta_1) per query pair, lse2 = lse * log2 e
	void* out1;                  // MODE 0: dV
	void* out2;                  // MODE 0: dK, MODE 1: dQ
	long long o1_b, o1_s, o1_h;  // element strides
	long long o2_b, o2_s, o2_h;
};

struct WideBwdSmem {
	static constexpr int NST = 2;                 // stages of the streamed ring
	static constexpr int R1_OFF = 0;
	static constexpr int R2_OFF = R1_OFF + FW_TILE;
	static constexpr int T_OFF = R2_OFF + FW_TILE; // stage s: T1 at + s * 2 * FW_TILE, T2 right behind it
	static constexpr int XCH_OFF = T_OFF + NST * 2 * FW_TILE; // [2 warpgroups][32 accumulators][128 threads] fp32
	static constexpr int BAR_OFF = XCH_OFF + 2 * 32 * 128 * 4;
	static constexpr int TOTAL = BAR_OFF + 256 + 1024;
	static_assert(TOTAL <= 232448, "227 KB of shared memory per CTA");
};

// (-lse * log2 e, -delta) per query row, as fmha_bwd_prep_kernel forms them, over up to 256 features: 16 lanes per row, 16 features each
__global__ void __launch_bounds__(256) fmha_wide_bwd_prep_kernel(const uint16_t* __restrict__ dout, const uint16_t* __restrict__ out, const float* __restrict__ lse, float* __restrict__ stat, int B, int H, int Sq, int Sq_r, int D, int is_bf16,
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
	if (q < Sq)
	{
#pragma unroll
		for (int c = 0; c < 2; c++)
		{
			const int d0 = sub * 16 + c * 8;
			if (d0 >= D)
				break;
			const uint4 a = *reinterpret_cast<const uint4*>(dout + b * do_b + (long long)q * do_s + h * do_h + d0);
			const uint4 e = *reinterpret_cast<const uint4*>(out + b * o_b + (long long)q * o_s + h * o_h + d0);
			const uint32_t aw[4] = { a.x, a.y, a.z, a.w }, ew[4] = { e.x, e.y, e.z, e.w };
#pragma unroll
			for (int i = 0; i < 4; i++)
			{
				acc = fmaf(widen16((uint16_t)(aw[i] & 0xffff), is_bf16), widen16((uint16_t)(ew[i] & 0xffff), is_bf16), acc);
				acc = fmaf(widen16((uint16_t)(aw[i] >> 16), is_bf16), widen16((uint16_t)(ew[i] >> 16), is_bf16), acc);
			}
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
		float* const dst = stat + (row >> 1) * 4 + (row & 1);
		dst[0] = -l2;
		dst[2] = q < Sq ? -acc : 0.f;
	}
}

// MODE 0 = dK/dV (R1 = K, R2 = V, T1 = Q_i, T2 = dO_i), MODE 1 = dQ (R1 = Q, R2 = dO, T1 = K_j, T2 = V_j), as in sm100_fmha_bwd.cu
template <int MODE, int BF16>
__global__ void __launch_bounds__(FW_THREADS, 1) fmha_wide_bwd_kernel(const __grid_constant__ CUtensorMap tmR1, const __grid_constant__ CUtensorMap tmR2, const __grid_constant__ CUtensorMap tmT1, const __grid_constant__ CUtensorMap tmT2, const WideBwdParams p)
{
	using L = WideBwdSmem;
	constexpr int NST = L::NST;
	extern __shared__ uint8_t smem_raw[];
	uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
	uint64_t* bars = (uint64_t*)(smem + L::BAR_OFF);
	uint64_t* r_full = bars;
	uint64_t* t_full = bars + 1;         // [NST]
	uint64_t* t_empty = bars + 1 + NST;  // [NST] one arrival per consumer warpgroup

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int r0 = blockIdx.x * FW_K;    // first resident row (MODE 0: key, MODE 1: query)
	const int hr = blockIdx.y, b = blockIdx.z; // MODE 0: key head, MODE 1: query head
	const int group = p.H / p.Hk;
	const int shift = p.Sk - p.Sq;       // causal: query i sees keys <= i + shift
	int first = 0, n_per = 0, n_total = 0;
	if (MODE == 0)
	{
		const int nq = (p.Sq + FW_K - 1) / FW_K;
		first = p.causal ? min(nq, max(0, (r0 - shift) / FW_K)) : 0;
		n_per = nq - first;
		n_total = n_per * group;
	} else {
		const int kv_end = p.causal ? min(p.Sk, max(r0 + FW_K + shift, 0)) : p.Sk;
		n_per = n_total = (kv_end + FW_K - 1) / FW_K;
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
		setmaxnreg_dec<40>(); // (the producer's index arithmetic needs more than 24)
		if (warp == 8 && elect_one())
		{
			tma_prefetch_desc(&tmR1);
			tma_prefetch_desc(&tmR2);
			tma_prefetch_desc(&tmT1);
			tma_prefetch_desc(&tmT2);
			mbar_expect_tx(r_full, 2 * FW_TILE);
			for (int a = 0; a < 4; a++)
			{
				tma_load_4d(smem + L::R1_OFF + a * FW_ATOM, &tmR1, r_full, 64 * a, hr, r0, b);
				tma_load_4d(smem + L::R2_OFF + a * FW_ATOM, &tmR2, r_full, 64 * a, hr, r0, b);
			}
			for (int n = 0; n < n_total; n++)
			{
				const int s = n % NST;
				const uint32_t ph = (uint32_t)(n / NST) & 1;
				const int row = MODE == 0 ? (first + n % n_per) * FW_K : n * FW_K;
				const int head = MODE == 0 ? hr * group + n / n_per : hr / group;
				uint8_t* const t1 = smem + L::T_OFF + s * 2 * FW_TILE;
				mbar_wait(&t_empty[s], ph ^ 1);
				mbar_expect_tx(&t_full[s], 2 * FW_TILE);
				for (int a = 0; a < 4; a++)
				{
					tma_load_4d(t1 + a * FW_ATOM, &tmT1, &t_full[s], 64 * a, head, row, b);
					tma_load_4d(t1 + FW_TILE + a * FW_ATOM, &tmT2, &t_full[s], 64 * a, head, row, b);
				}
			}
		}
		return;
	}

	// ------------------------------------------------------------------ consumers: resident rows rr + 8 * hh, features [128 wg, 128 wg + 128)
	setmaxnreg_inc<232>();
	const int wg = warp >> 2, t4 = lane & 3, tid = threadIdx.x & 127;
	const int rr = r0 + (warp & 3) * 16 + (lane >> 2);
	constexpr int is_bf16 = BF16;
	float acc1[64], acc2[64]; // acc1: MODE 0 only
#pragma unroll
	for (int i = 0; i < 64; i++)
		acc2[i] = 0.f;
#pragma unroll
	for (int i = 0; i < 64; i++)
		acc1[i] = 0.f;
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
	// warpgroup 0 forms X = R1 T1^T, warpgroup 1 Y = R2 T2^T
	const uint32_t r_base = smem_u32(smem + (wg == 0 ? L::R1_OFF : L::R2_OFF));
	float* const xch = (float*)(smem + L::XCH_OFF);
	mbar_wait(r_full, 0);
	for (int n = 0; n < n_total; n++)
	{
		const int s = n % NST;
		const uint32_t ph = (uint32_t)(n / NST) & 1;
		const int c0 = MODE == 0 ? (first + n % n_per) * FW_K : n * FW_K; // first streamed row (MODE 0: query, MODE 1: key)
		const int hq = MODE == 0 ? hr * group + n / n_per : hr;
		mbar_wait(&t_full[s], ph);
		const uint32_t t1_base = smem_u32(smem + L::T_OFF + s * 2 * FW_TILE), t2_base = t1_base + FW_TILE;
		const uint32_t t_base = wg == 0 ? t1_base : t2_base;
		float z[32];
#pragma unroll
		for (int i = 0; i < 32; i++)
			z[i] = 0.f;
		fence_regs(z);
		wgmma_fence();
#pragma unroll
		for (int k = 0; k < FW_D / 16; k++)
		{
			const uint32_t off = (uint32_t)(k >> 2) * FW_ATOM + (uint32_t)(k & 3) * 32;
			if constexpr (BF16 != 0)
				wgmma_bf16_ss_n64<0, 0>(z, wgmma_desc(r_base + off, 16, 1024), wgmma_desc(t_base + off, 16, 1024));
			else
				wgmma_f16_ss_n64<0, 0>(z, wgmma_desc(r_base + off, 16, 1024), wgmma_desc(t_base + off, 16, 1024));
		}
		wgmma_commit();
		fence_regs(z);
		wgmma_wait<0>();
		fence_regs(z);
		// swap X and Y: thread t of either warpgroup holds the same (row, column) positions.  Both read both back, so that z is dead
		// before x and y are live
#pragma unroll
		for (int i = 0; i < 32; i++)
			xch[(wg * 32 + i) * 128 + tid] = z[i];
		named_bar_sync(1, 256);
		float x[32], y[32];
#pragma unroll
		for (int i = 0; i < 32; i++)
			x[i] = xch[i * 128 + tid], y[i] = xch[(32 + i) * 128 + tid];
		named_bar_sync(1, 256); // both have read: the buffer is free for the next block
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
		uint32_t fp[FW_K / 16][4], fds[FW_K / 16][4];
#pragma unroll
		for (int kk = 0; kk < FW_K / 16; kk++)
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
		for (int kk = 0; kk < FW_K / 16; kk++)
		{
			// this warpgroup's 128 features of T1 / T2 as MN-major B operands: atoms 2 wg and 2 wg + 1, 8 KB apart (LBO)
			const uint32_t half = (uint32_t)(2 * wg * FW_ATOM + kk * 2048);
			const uint64_t d1 = wgmma_desc(t1_base + half, FW_ATOM, 1024), d2 = wgmma_desc(t2_base + half, FW_ATOM, 1024);
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
		if (tid == 0)
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
			const int d = 128 * wg + 8 * jn + 2 * t4;
			if (d >= p.D)
				continue;
			const int i = 4 * jn + 2 * hh;
			*reinterpret_cast<uint32_t*>(o2 + d) = pack2(acc2[i] * p.scale, acc2[i + 1] * p.scale, is_bf16);
			if (MODE == 0)
				*reinterpret_cast<uint32_t*>(o1 + d) = pack2(acc1[i], acc1[i + 1], is_bf16);
		}
	}
}

// the dynamic shared memory attribute is per device: `configured_on` is the caller's flag per device for this kernel
template <typename K>
int configure(K* kernel, const int bytes, const char* what, bool (&configured_on)[64])
{
	int dev = 0;
	cudaGetDevice(&dev);
	bool& configured = configured_on[dev & 63];
	if (!configured)
	{
		const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
		if (e != cudaSuccess)
		{
			set_last_error(what, e);
			return -1;
		}
		configured = true;
	}
	return 0;
}

template <int MODE, int BF16>
int launch_wide_bwd(cudaStream_t stream, const CUtensorMap& r1, const CUtensorMap& r2, const CUtensorMap& t1, const CUtensorMap& t2, const WideBwdParams& p, int tiles, int heads, int B)
{
	static bool configured_on[64];
	if (configure(fmha_wide_bwd_kernel<MODE, BF16>, WideBwdSmem::TOTAL, "cudaFuncSetAttribute(fmha_wide_bwd_kernel)", configured_on))
		return -1;
	fmha_wide_bwd_kernel<MODE, BF16><<<dim3(tiles, heads, B), FW_THREADS, WideBwdSmem::TOTAL, stream>>>(r1, r2, t1, t2, p);
	return launched("fmha_wide_bwd_kernel launch");
}

template <int MODE>
int launch_wide_bwd(cudaStream_t stream, const int is_bf16, const CUtensorMap& r1, const CUtensorMap& r2, const CUtensorMap& t1, const CUtensorMap& t2, const WideBwdParams& p, int tiles, int heads, int B)
{
	return is_bf16 ? launch_wide_bwd<MODE, 1>(stream, r1, r2, t1, t2, p, tiles, heads, B) : launch_wide_bwd<MODE, 0>(stream, r1, r2, t1, t2, p, tiles, heads, B);
}

template <int BF16, int MASK>
int launch_wide_fwd(cudaStream_t stream, const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const WideFwdParams& p, const CUtensorMap& m, const dim3 grid)
{
	static bool configured_on[64];
	if (configure(fmha_wide_fwd_kernel<BF16, MASK>, WideFwdSmem<MASK>::TOTAL, "cudaFuncSetAttribute(fmha_wide_fwd_kernel)", configured_on))
		return -1;
	fmha_wide_fwd_kernel<BF16, MASK><<<grid, FW_THREADS, WideFwdSmem<MASK>::TOTAL, stream>>>(q, k, v, p, m);
	return launched("fmha_wide_fwd_kernel launch");
}

bool wide_shape(const SdpaGeom& g)
{
	return g.D > 128 && g.D <= FW_D && (g.D & 7) == 0 && g.Dv == g.D && g.B > 0 && g.H > 0 && g.Hk > 0 && g.H % g.Hk == 0 && g.Sq > 0 && g.Sk > 0 && encode_init();
}

} // namespace

// returns 0 on success, 1 when the shape is outside this kernel (128 < D = Dv <= 256, a multiple of 8; 16-byte aligned strides; a mask's
// base and pitches 16-byte aligned), < 0 on CUDA errors
int sdpa_forward_f16_wide(cudaStream_t stream, const SdpaGeom& g, int is_bf16, const void* q, const void* k, const void* v, void* o, float* lse, const void* mask, int mask_f32)
{
	if (!wide_shape(g))
		return 1;
	if ((((uintptr_t)o) & 15) || (g.o_b & 7) || (g.o_s & 7) || (g.o_h & 7))
		return 1;
	CUtensorMap tmQ, tmK, tmV, tmM;
	memset(&tmM, 0, sizeof(tmM));
	if (mask && !make_map_mask(&tmM, mask, g.B, g.H, g.Sq, g.Sk, g.mask_b, g.mask_h, g.mask_s, mask_f32 ? 4 : 2, is_bf16))
		return 1;
	if (!make_map_bshd(&tmQ, q, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h, is_bf16, FW_Q) || !make_map_bshd(&tmK, k, g.B, g.Sk, g.Hk, g.D, g.k_b, g.k_s, g.k_h, is_bf16, FW_K) ||
		!make_map_bshd(&tmV, v, g.B, g.Sk, g.Hk, g.Dv, g.v_b, g.v_s, g.v_h, is_bf16, FW_K))
		return 1;
	WideFwdParams p;
	memset(&p, 0, sizeof(p));
	p.H = g.H, p.Hk = g.Hk, p.Sq = g.Sq, p.Sk = g.Sk, p.D = g.D;
	p.causal = g.is_causal;
	p.scale_log2 = g.scale * 1.4426950408889634f;
	p.o = o, p.o_b = g.o_b, p.o_s = g.o_s, p.o_h = g.o_h;
	p.lse = lse;
	p.scale = g.scale;
	p.mask_h = g.mask_h != 0, p.mask_b = g.mask_b != 0;
	const dim3 grid((g.Sq + FW_Q - 1) / FW_Q, g.H, g.B);
	const int kind = mask ? (mask_f32 ? 1 : 2) : 0;
	if (is_bf16)
		return kind == 0 ? launch_wide_fwd<1, 0>(stream, tmQ, tmK, tmV, p, tmM, grid) : kind == 1 ? launch_wide_fwd<1, 1>(stream, tmQ, tmK, tmV, p, tmM, grid) : launch_wide_fwd<1, 2>(stream, tmQ, tmK, tmV, p, tmM, grid);
	return kind == 0 ? launch_wide_fwd<0, 0>(stream, tmQ, tmK, tmV, p, tmM, grid) : kind == 1 ? launch_wide_fwd<0, 1>(stream, tmQ, tmK, tmV, p, tmM, grid) : launch_wide_fwd<0, 2>(stream, tmQ, tmK, tmV, p, tmM, grid);
}

// The arguments and the workspace of sdpa_backward_f16 (sdpa_backward_f16_workspace_bytes covers this path: the same statistics, and
// O / LSE when the forward runs first).  Same return convention as the forward.
int sdpa_backward_f16_wide(cudaStream_t stream, const SdpaGeom& g, const SdpaGeom& dg, int is_bf16, const void* dout, const void* q, const void* k, const void* v, const void* out, long long oo_b, long long oo_s, long long oo_h,
	const float* lse, void* dq, void* dk, void* dv, void* workspace)
{
	const void* const ptrs[7] = { dq, dk, dv, dout, q, k, v };
	if (!wide_shape(g) || !sdpa_backward_f16_takes(g, dg, 1, ptrs, 7))
		return 1;
	CUtensorMap tmQ, tmK, tmV, tmG;
	if (!make_map_bshd(&tmQ, q, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h, is_bf16, FW_K) || !make_map_bshd(&tmK, k, g.B, g.Sk, g.Hk, g.D, g.k_b, g.k_s, g.k_h, is_bf16, FW_K) ||
		!make_map_bshd(&tmV, v, g.B, g.Sk, g.Hk, g.Dv, g.v_b, g.v_s, g.v_h, is_bf16, FW_K) || !make_map_bshd(&tmG, dout, g.B, g.Sq, g.H, g.Dv, g.o_b, g.o_s, g.o_h, is_bf16, FW_K))
		return 1;
	const int sq_r = (g.Sq + FW_STAT_ROWS - 1) / FW_STAT_ROWS * FW_STAT_ROWS;
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
		const int rc = sdpa_forward_f16_wide(stream, fg, is_bf16, q, k, v, o_ws, lse_ws);
		if (rc != 0)
			return rc;
		out = o_ws, lse = lse_ws;
		oo_b = fg.o_b, oo_s = fg.o_s, oo_h = fg.o_h;
	}
	if ((((uintptr_t)out) & 15) || (oo_b & 7) || (oo_s & 7) || (oo_h & 7))
		return 1;
	const long long rows = (long long)g.B * g.H * sq_r;
	fmha_wide_bwd_prep_kernel<<<(unsigned)((rows + 15) / 16), 256, 0, stream>>>((const uint16_t*)dout, (const uint16_t*)out, lse, stat, g.B, g.H, g.Sq, sq_r, g.D, is_bf16, g.o_b, g.o_s, g.o_h, oo_b, oo_s, oo_h);
	if (launched("fmha_wide_bwd_prep_kernel launch"))
		return -1;
	WideBwdParams p;
	memset(&p, 0, sizeof(p));
	p.H = g.H, p.Hk = g.Hk, p.Sq = g.Sq, p.Sk = g.Sk, p.Sq_r = sq_r, p.D = g.D;
	p.causal = g.is_causal;
	p.scale = g.scale, p.scale_log2 = g.scale * 1.4426950408889634f;
	p.stat = (const float4*)stat;
	// dK, dV: one CTA per 64 keys of a (batch, key head)
	p.out1 = dv, p.o1_b = dg.v_b, p.o1_s = dg.v_s, p.o1_h = dg.v_h;
	p.out2 = dk, p.o2_b = dg.k_b, p.o2_s = dg.k_s, p.o2_h = dg.k_h;
	int rc = launch_wide_bwd<0>(stream, is_bf16, tmK, tmV, tmQ, tmG, p, (g.Sk + FW_K - 1) / FW_K, g.Hk, g.B);
	if (rc != 0)
		return rc;
	// dQ: one CTA per 64 queries of a (batch, query head)
	p.out1 = 0;
	p.out2 = dq, p.o2_b = dg.q_b, p.o2_s = dg.q_s, p.o2_h = dg.q_h;
	return launch_wide_bwd<1>(stream, is_bf16, tmQ, tmG, tmK, tmV, p, (g.Sq + FW_K - 1) / FW_K, g.H, g.B);
}

} // namespace sm100
