// sm100_fmha.cu -- SCALED_DOT_PRODUCT_ATTENTION forward for 16-bit tensors (bf16 / fp16), head dimension <= 128:
// one flash-attention kernel on the Hopper wgmma tensor cores.  Semantics: scaled_dot_product_attention/
// ccv_nnc_scaled_dot_product_attention_cpu_ref.c:16-183 (O = softmax(scale * Q K^T [causal, bottom-right aligned :147]) V,
// GQA through H / Hk :99,113), the same restrictions as the reference's flash-attention backend
// (gpu/ccv_nnc_scaled_dot_product_attention_flash_attn.cu:13-205: 16-bit only, no additive mask, no unify-head weights).
//
// One CTA = 128 query rows of one (batch, head); 288 threads:
//   warps 0-7  two consumer warpgroups of 64 query rows.  Per block of 128 keys: S_j = Q K_j^T (wgmma, both operands from shared
//              memory, fp32 in registers), online softmax in registers (a row lives in the four lanes of a quad), then
//              O += P_j V_j with P_j as 16-bit register fragments (wgmma A from registers) and V_j as an MN-major operand
//   warp 8     TMA producer: Q once, then K_j / V_j through two-stage rings (4-D tensor maps over the caller's [B, S, H, D]
//              strides, 128-byte swizzle, two 64-feature atoms per tile)
// smem: Q 32 KB + K 2 x 32 KB + V 2 x 32 KB = 160 KB.
//
// MASK (1 = fp32, 2 = 16-bit of the activations' type; CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK): an additive mask [B|1, H|1, Sq, Sk].  The
// producer stages the mask tile of each key block (128 query rows x 128 keys, make_map_mask) in one more buffer: 64 KB fp32 / 32 KB
// 16-bit, 224 / 192 KB in all.  The consumers form t = fmaf(s, scale, mask) (CPU_REF's order), cut the causal / Sk horizon, and run
// the online softmax on t in log2 units; the buffer is released (one arrival per warp) before P V, so the next tile loads under the
// MMAs.  These kernels run 384 threads: warps 8-11 are the producer warpgroup (see fm_threads).
#include "sm100_contract.h"
#include "sm100_fmha.cuh"
#include <string.h>

namespace sm100 {

namespace {

constexpr int FM_BLOCK = 128; // query rows per CTA = keys per block
constexpr int FM_D = 128;     // head dimension (q/k and v)
constexpr int FM_TILE_BYTES = FM_BLOCK * FM_D * 2; // 32 KB: two 128 x 64 swizzle atoms
constexpr int FM_ATOM_BYTES = FM_BLOCK * 128;      // 16 KB
constexpr int FM_THREADS = 288;
// the masked kernels: a whole producer warpgroup, so that setmaxnreg can move its registers to the consumers (40 / 232 instead of
// 168 each); 168 registers leave no room for the mask next to S, O and the softmax state
constexpr int fm_threads(const int mask) { return mask ? 384 : FM_THREADS; }

struct FmhaParams {
	int H, Hk, Sq, Sk;
	int D; // actual head dimension (<= 128, a multiple of 8): the tiles are always 128 wide, TMA zero-fills the rest
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
struct FmhaSmem {
	static constexpr int Q_OFF = 0;
	static constexpr int K_OFF = Q_OFF + FM_TILE_BYTES;
	static constexpr int V_OFF = K_OFF + 2 * FM_TILE_BYTES;
	static constexpr int M_OFF = V_OFF + 2 * FM_TILE_BYTES;
	static constexpr int M_BYTES = MASK == 0 ? 0 : FM_BLOCK * FM_BLOCK * (MASK == 1 ? 4 : 2);
	static constexpr int BAR_OFF = M_OFF + M_BYTES;
	static constexpr int TOTAL = BAR_OFF + 256 + 1024;
	static_assert(TOTAL <= 232448, "227 KB of shared memory per CTA");
};

// element type and mask kind as template parameters: one basic block per MMA batch; tmM is only read when MASK != 0
template <int BF16, int MASK>
__global__ void __launch_bounds__(fm_threads(MASK), 1) fmha_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const FmhaParams p, const __grid_constant__ CUtensorMap tmM)
{
	using L = FmhaSmem<MASK>;
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
	const int q0 = q_tile * FM_BLOCK;
	const int h = blockIdx.y, b = blockIdx.z;
	const int hk = h / (p.H / p.Hk);
	// keys this tile attends: causal is aligned to the bottom-right corner (query i sees keys <= i + Sk - Sq)
	const int shift = p.Sk - p.Sq;
	int kv_end = p.Sk;
	if (p.causal)
		kv_end = min(p.Sk, max(q0 + FM_BLOCK + shift, 0));
	const int n_blk = (kv_end + FM_BLOCK - 1) / FM_BLOCK;

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

	if (MASK != 0 ? warp >= 8 : warp == 8)
	{
		if constexpr (MASK != 0)
			setmaxnreg_dec<40>(); // (with 24 / 240 the fp32-mask kernel spilled)
		if ((MASK == 0 || warp == 8) && n_blk > 0 && elect_one())
		{
			tma_prefetch_desc(&tmQ);
			tma_prefetch_desc(&tmK);
			tma_prefetch_desc(&tmV);
			if constexpr (MASK != 0)
				tma_prefetch_desc(&tmM);
			mbar_expect_tx(q_full, FM_TILE_BYTES);
			tma_load_4d(smem + L::Q_OFF, &tmQ, q_full, 0, h, q0, b);
			tma_load_4d(smem + L::Q_OFF + FM_ATOM_BYTES, &tmQ, q_full, 64, h, q0, b);
			for (int j = 0; j < n_blk; j++)
			{
				const int s = j & 1;
				const uint32_t ph = (uint32_t)(j >> 1) & 1;
				uint8_t* const sk = smem + L::K_OFF + s * FM_TILE_BYTES;
				uint8_t* const sv = smem + L::V_OFF + s * FM_TILE_BYTES;
				mbar_wait(&k_empty[s], ph ^ 1);
				mbar_expect_tx(&k_full[s], FM_TILE_BYTES);
				tma_load_4d(sk, &tmK, &k_full[s], 0, hk, j * FM_BLOCK, b);
				tma_load_4d(sk + FM_ATOM_BYTES, &tmK, &k_full[s], 64, hk, j * FM_BLOCK, b);
				if constexpr (MASK != 0)
				{
					mbar_wait(m_empty, ((uint32_t)j & 1) ^ 1);
					mbar_expect_tx(m_full, L::M_BYTES);
					for (int a = 0; a < L::M_BYTES / MASK_ATOM_BYTES; a++)
						tma_load_4d(smem + L::M_OFF + a * MASK_ATOM_BYTES, &tmM, m_full, j * FM_BLOCK + a * (MASK == 1 ? 32 : 64), q0, p.mask_h ? h : 0, p.mask_b ? b : 0);
				}
				mbar_wait(&v_empty[s], ph ^ 1);
				mbar_expect_tx(&v_full[s], FM_TILE_BYTES);
				tma_load_4d(sv, &tmV, &v_full[s], 0, hk, j * FM_BLOCK, b);
				tma_load_4d(sv + FM_ATOM_BYTES, &tmV, &v_full[s], 64, hk, j * FM_BLOCK, b);
			}
		}
		return;
	}

	// ------------------------------------------------------------------ consumers: rows r0 and r0 + 8 of this thread
	if constexpr (MASK != 0)
		setmaxnreg_inc<232>();
	const int wg = warp >> 2;
	const int t4 = lane & 3;
	const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
	int kv_limit[2]; // keys [0, kv_limit) are visible to the row
#pragma unroll
	for (int hh = 0; hh < 2; hh++)
		kv_limit[hh] = p.causal ? min(p.Sk, q0 + r0 + 8 * hh + shift + 1) : p.Sk;
	float o[64], sacc[64];
#pragma unroll
	for (int i = 0; i < 64; i++)
		o[i] = 0.f;
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
		const uint32_t k_base = smem_u32(smem + L::K_OFF + s * FM_TILE_BYTES);
#pragma unroll
		for (int i = 0; i < 64; i++)
			sacc[i] = 0.f;
		fence_regs(sacc);
		wgmma_fence();
#pragma unroll
		for (int k = 0; k < FM_D / 16; k++)
		{
			const uint32_t off = (uint32_t)(k >> 2) * FM_ATOM_BYTES + (uint32_t)(k & 3) * 32;
			const uint64_t dq = wgmma_desc(q_base + off, 16, 1024), dk = wgmma_desc(k_base + off, 16, 1024);
			if constexpr (BF16 != 0)
				wgmma_bf16_ss_n128<0, 0>(sacc, dq, dk);
			else
				wgmma_f16_ss_n128<0, 0>(sacc, dq, dk);
		}
		wgmma_commit();
		fence_regs(sacc);
		wgmma_wait<0>();
		fence_regs(sacc);
		if ((threadIdx.x & 127) == 0)
			mbar_arrive(&k_empty[s]);
		// online softmax: key of accumulator i = j * 128 + 8 * (i >> 2) + 2 * t4 + (i & 1), row r0 + 8 * ((i >> 1) & 1)
		const int kv0 = j * FM_BLOCK + 2 * t4;
		const bool edge = j * FM_BLOCK + FM_BLOCK > min(kv_limit[0], kv_limit[1]);
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
		for (int i = 0; i < 64; i++)
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
		for (int i = 0; i < 64; i++)
		{
			const int hh = (i >> 1) & 1;
			const float e = ex2_approx(fmaf(sacc[i], scale_log2, -m_use[hh])); // exp2(-inf) = 0 for the masked keys
			sacc[i] = e;
			sum[hh] += e;
			o[i] *= alpha[hh];
		}
		l[0] = fmaf(l[0], alpha[0], sum[0]), l[1] = fmaf(l[1], alpha[1], sum[1]);
		// O += P_j V_j
		mbar_wait(&v_full[s], ph);
		const uint32_t v_base = smem_u32(smem + L::V_OFF + s * FM_TILE_BYTES);
		// every A fragment is packed before the MMAs start: registers an in-flight wgmma reads must not be written between them
		uint32_t pa[FM_BLOCK / 16][4];
#pragma unroll
		for (int kk = 0; kk < FM_BLOCK / 16; kk++)
			acc_to_a(sacc, kk, BF16, pa[kk]);
		fence_regs(o);
		wgmma_fence();
#pragma unroll
		for (int kk = 0; kk < FM_BLOCK / 16; kk++)
		{
			const uint32_t (&a)[4] = pa[kk];
			// V [128 keys x 128 d] as an MN-major B operand: two 64-wide d atoms 16 KB apart (LBO), 8-key groups 1 KB apart (SBO),
			// one MMA consumes 16 keys = 2 KB
			const uint64_t dv = wgmma_desc(v_base + kk * 2048, FM_ATOM_BYTES, 1024);
			if constexpr (BF16 != 0)
				wgmma_bf16_rs_n128<1>(o, a, dv);
			else
				wgmma_f16_rs_n128<1>(o, a, dv);
		}
		wgmma_commit();
		fence_regs(o);
		wgmma_wait<0>();
		fence_regs(o);
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
			if (d < p.D) // head dimensions below 128: the padded feature columns are not part of the tensor
				*reinterpret_cast<uint32_t*>(orow + d) = pack2(o[4 * jn + 2 * hh] * inv, o[4 * jn + 2 * hh + 1] * inv, BF16);
		}
		if (p.lse && t4 == 0) // (a NaN in the mask makes l NaN: the masked kernels pass it on)
			p.lse[((long long)b * p.H + h) * p.Sq + qi] = (MASK != 0 ? l[hh] != 0.f : l[hh] > 0.f) ? (m[hh] + log2f(l[hh])) * 0.6931471805599453f : -INFINITY;
	}
}

template <int BF16, int MASK>
int launch_fwd(cudaStream_t stream, const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const FmhaParams& p, const CUtensorMap& m, const dim3 grid)
{
	// the attribute is per device: one flag per device (a process may drive several GPUs)
	static bool configured_on[64];
	int dev = 0;
	cudaGetDevice(&dev);
	bool& configured = configured_on[dev & 63];
	if (!configured)
	{
		const cudaError_t e = cudaFuncSetAttribute(fmha_fwd_kernel<BF16, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, FmhaSmem<MASK>::TOTAL);
		if (e != cudaSuccess)
		{
			set_last_error("cudaFuncSetAttribute(fmha_fwd_kernel)", e);
			return -1;
		}
		configured = true;
	}
	fmha_fwd_kernel<BF16, MASK><<<grid, fm_threads(MASK), FmhaSmem<MASK>::TOTAL, stream>>>(q, k, v, p, m);
	return launched("fmha_fwd_kernel launch");
}

} // namespace

// returns 0 on success, 1 when the shape is outside this kernel (D = Dv <= 128 and a multiple of 8 -- head dimensions below 128 run on the
// same 128-wide tiles, the TMA unit zero-fills the missing features; 16-byte aligned strides; a mask's base and pitches 16-byte aligned),
// < 0 on CUDA errors
int sdpa_forward_f16(cudaStream_t stream, const SdpaGeom& g, int is_bf16, const void* q, const void* k, const void* v, void* o, float* lse, const void* mask, int mask_f32)
{
	if (g.D > FM_D || g.D < 8 || (g.D & 7) || g.Dv != g.D || g.B <= 0 || g.H <= 0 || g.Hk <= 0 || g.H % g.Hk != 0 || g.Sq <= 0 || g.Sk <= 0 || !encode_init())
		return 1;
	if ((((uintptr_t)o) & 15) || (g.o_b & 7) || (g.o_s & 7) || (g.o_h & 7))
		return 1;
	CUtensorMap tmQ, tmK, tmV, tmM;
	memset(&tmM, 0, sizeof(tmM));
	if (mask && !make_map_mask(&tmM, mask, g.B, g.H, g.Sq, g.Sk, g.mask_b, g.mask_h, g.mask_s, mask_f32 ? 4 : 2, is_bf16))
		return 1;
	if (!make_map_bshd(&tmQ, q, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h, is_bf16, FM_BLOCK) || !make_map_bshd(&tmK, k, g.B, g.Sk, g.Hk, g.D, g.k_b, g.k_s, g.k_h, is_bf16, FM_BLOCK) ||
		!make_map_bshd(&tmV, v, g.B, g.Sk, g.Hk, g.Dv, g.v_b, g.v_s, g.v_h, is_bf16, FM_BLOCK))
		return 1;
	FmhaParams p;
	memset(&p, 0, sizeof(p));
	p.H = g.H, p.Hk = g.Hk, p.Sq = g.Sq, p.Sk = g.Sk, p.D = g.D;
	p.causal = g.is_causal;
	p.scale_log2 = g.scale * 1.4426950408889634f;
	p.o = o, p.o_b = g.o_b, p.o_s = g.o_s, p.o_h = g.o_h;
	p.lse = lse;
	p.scale = g.scale;
	p.mask_h = g.mask_h != 0, p.mask_b = g.mask_b != 0;
	const dim3 grid((g.Sq + FM_BLOCK - 1) / FM_BLOCK, g.H, g.B);
	const int kind = mask ? (mask_f32 ? 1 : 2) : 0;
	if (is_bf16)
		return kind == 0 ? launch_fwd<1, 0>(stream, tmQ, tmK, tmV, p, tmM, grid) : kind == 1 ? launch_fwd<1, 1>(stream, tmQ, tmK, tmV, p, tmM, grid) : launch_fwd<1, 2>(stream, tmQ, tmK, tmV, p, tmM, grid);
	return kind == 0 ? launch_fwd<0, 0>(stream, tmQ, tmK, tmV, p, tmM, grid) : kind == 1 ? launch_fwd<0, 1>(stream, tmQ, tmK, tmV, p, tmM, grid) : launch_fwd<0, 2>(stream, tmQ, tmK, tmV, p, tmM, grid);
}

} // namespace sm100
