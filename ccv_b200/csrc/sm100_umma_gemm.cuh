// sm100_umma_gemm.cuh -- the one tensor-core contraction kernel of the backend (Hopper wgmma).
//
//   D[M, N] (+)= A[M, Kdim] * B[Kdim, N]        fp32 accumulators in registers
//
// GEMM fwd/bwd, convolution fprop / dgrad / wgrad (implicit GEMM, NHWC) are all this kernel with a different way of
// bringing the A and B tiles into shared memory (OperandMode).  One CTA computes one 128 x BN output tile (optional split-K
// and filter taps along gridDim.z) with 288 threads:
//
//   warps 0-7  two consumer warpgroups, 64 output rows each: wgmma.mma_async from 128-byte-swizzled K-major tiles (16-bit MN-major
//              tiles through the descriptor's transpose bit), then the epilogue straight from the accumulator registers
//              (+bias, +C, 16-bit rounding; split-K: into this split's scratch slice)
//   warp 8     TMA producer: cp.async.bulk.tensor (tile mode or im2col mode) into a ring of STAGES stages, mbarrier tx counts
//
// fp32 operands run as TF32 (kind 0; the TMA unit rounds them to TF32 on the way in) or as 3xTF32 (X3).  wgmma reads TF32 operands
// K-major only, so the fp32 kernels whose operands arrive MN-major, and the 3xTF32 kernels, pass every stage through a transform
// step first: the consumers copy the staged tiles into one of two K-major operand slots (transposing MN-major tiles, splitting
// 3xTF32 operands into hi / lo) and release the stage to the producer before the MMAs run.  The TF32 weight gradient (A =
// OP_MN2D_RS) transposes only B: its A = grad^T goes from the stage into registers, and its tiles are up to 256 columns wide.  For
// output-channel counts K <= 64 it swaps the operands (A = OP_IM2COL_RS, the filter taps along M, tiles of 128 or 256 rows, N = K).
#pragma once
#include "sm100_ptx.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace sm100 {

enum OperandMode {
	OP_K2D = 0,    // K-major 2-D tensor [rows, K]: one box {one 128-byte span of k, rows} per stage
	OP_MN2D = 1,   // MN-major 2-D tensor [K, rows]: boxes {BK mn, BK k} per stage
	OP_IM2COL = 2, // NHWC tensor through im2col-mode TMA.  As A: pixels are rows (K-major, channels = K).
	               //                                       As B: pixels are K   (MN-major, channels = N).
	OP_MN2D_RS = 3, // A only, TF32 only: an OP_MN2D tile staged 128-byte swizzled, which the consumers read straight into wgmma A
	                // fragments (see load_a_frags): it never goes through the transform step
	OP_IM2COL_RS = 4, // A only, TF32 only: the weight gradient's im2col(x)^T, rows = filter tap * C_tap + channel.  Each 32-row box of
	                  // the tile is one tap's 32-channel span of 32 pixels (the reduction), staged 128-byte swizzled like OP_MN2D_RS and
	                  // read into registers the same way; the epilogue stores the tile transposed (row m -> column m of the output)
};

constexpr int UMMA_BLOCK_M = 128;
constexpr int UMMA_BLOCK_K = 32; // fp32 elements per stage along K = one 128-byte span
constexpr int UMMA_MAX_TAPS = 64;
constexpr int GEMM_THREADS = 288;
// A from registers: a producer warpgroup, so that setmaxnreg can hand the consumers 224 registers (128 accumulators at BN = 256);
// without it the register file's split over the four schedulers caps 9 warps at 168
constexpr int GEMM_THREADS_RS = 384;

struct UmmaRowMap {
	// output row m -> element offset.  mode 0: m * ld.  mode 1: m = (n, i, j) over a (Pc x Qc) grid per image:
	// n * n_stride + i * h_stride + j * w_stride (used by strided dgrad, which writes every other pixel).
	int mode;
	int Pc, Qc;
	long long ld, n_stride, h_stride, w_stride;
};

struct UmmaGemmParams {
	int M, N;
	int k_iters;        // BK iterations over the whole reduction (all taps x chunks)
	int chunks_per_tap; // k-iteration it -> tap = it / chunks_per_tap, chunk = it % chunks_per_tap
	int splits;         // split-K factor; gridDim.z = grid_taps * splits.  Split s writes its partial tile to out + s * split_out_stride
	                    // (a scratch slice per split, plain stores); splitk_reduce_kernel then adds the slices in a fixed order, so the
	                    // result does not depend on CTA arrival order (no red.global.add anywhere in the contraction kernels)
	long long split_out_stride;
	int grid_taps;      // > 1 only for wgrad: the filter tap is a grid dimension
	long long grid_tap_out_stride; // output column offset per grid tap
	int C_tap;          // B = OP_IM2COL (wgrad): channels per filter tap.  B column n < N reads the grid tap + n / C_tap, channel n % C_tap
	// im2col geometry of the operand that uses OP_IM2COL: base pixel p -> (w, h, n) TMA coordinates
	int P, Q;
	int stride_h, stride_w;
	int base_h, base_w;
	unsigned short tap_off_h[UMMA_MAX_TAPS], tap_off_w[UMMA_MAX_TAPS];
	int tap_b_col[UMMA_MAX_TAPS]; // B's column (or row-block) origin for this tap
	int tap_b_row[UMMA_MAX_TAPS]; // K-major B: row origin for this tap (the data gradient's filter copy [tap][c][k])
	// epilogue
	float* out;
	const float* bias;
	int accumulate; // 1: D += existing output (CCV_NNC_ACCUMULATE_OUTPUT)
	UmmaRowMap rowmap;
	// optional per-column statistics of the output (batch-norm forward fused into the producing convolution; kernels without the
	// transform step only).  Four planes of stats_rows x N floats: count, shift k, sum(v - k), sum((v - k)^2).  Row blockIdx.x * 4 + quarter
	// belongs to one 32-row quarter of the tiles of one CTA column (gridDim.x CTAs walk the M tiles, blockIdx.x + i * gridDim.x), and every
	// (row, column) slot to one thread, which merges the per-warp shifted sums of each tile into it in a fixed order: no atomics, and the
	// shift (the first value seen) keeps the one-pass variance well conditioned.  The count plane must be zero on entry.
	float* stats;
	int stats_rows;
	int kind16;         // 0: fp32 operands (TF32 / 3xTF32); 1: 16-bit operands (the kernel is compiled per operand size, template K16)
	int out_kind;       // 16-bit operands: 1 = bf16, 2 = fp16 (also the output element type of OUT16 kernels)
	const void* bias16; // OUT16 kernels: bias in the output's 16-bit type (p.bias, fp32, wins when both are given)
};

// 16-bit output helpers: kind 1 = bf16, 2 = fp16, round to nearest even
__device__ __forceinline__ uint32_t pack16x2(const float a, const float b, const int kind)
{
	if (kind == 1)
	{
		const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
		return *reinterpret_cast<const uint32_t*>(&v);
	}
	const __half2 v = __floats2half2_rn(a, b);
	return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ float cvt16(const uint16_t x, const int kind)
{
	return kind == 1 ? __uint_as_float((uint32_t)x << 16) : __half2float(__ushort_as_half(x));
}

// X3 = 1 selects the error-compensated "3xTF32" form (CCV_NNC_SM100_ALGO_3XTF32): the operands arrive as raw fp32 (tensor map data type
// FLOAT32, no rounding); the transform step splits every element into hi = x with the low 13 mantissa bits cleared (exactly representable
// in TF32) and lo = x - hi (exact in fp32), and three MMAs per k-step -- lo*hi + hi*lo + hi*hi (lo*lo ~ 2^-22 is dropped) -- accumulate
// into the same fp32 registers.  The product then carries ~2^-21 relative error per term instead of TF32's 2^-11: fp32-grade results
// (the reference's fp32 GEMM is CUBLAS_COMPUTE_32F, lib/nnc/gpu/ccv_nnc_compat.cu:786-803) at a third of the tensor rate.
template <int AMODE, int BMODE, int K16, int X3>
struct GemmXform {
	static constexpr bool A_RS = AMODE == OP_MN2D_RS || AMODE == OP_IM2COL_RS; // A from registers (TF32 only)
	static constexpr bool A_T = !K16 && AMODE == OP_MN2D; // fp32 MN-major A: transposed into the K-major slot
	static constexpr bool B_T = !K16 && BMODE != OP_K2D;  // fp32 MN-major B (2-D or im2col)
	static constexpr bool ANY = A_T || B_T || X3;
};

template <int BN, int STAGES, bool XF, int X3, bool ARS = false, int BM = UMMA_BLOCK_M>
struct UmmaSmem {
	static constexpr int A_BYTES = BM * 128;
	static constexpr int B_BYTES = BN * 128;
	static constexpr int RAW_BYTES = A_BYTES + B_BYTES;            // one TMA stage
	static constexpr int SLOT_A_BYTES = ARS ? 0 : A_BYTES;          // where B starts in the operand the MMAs read (A from registers: B alone)
	static constexpr int SLOT_BYTES = (SLOT_A_BYTES + B_BYTES) * (X3 ? 2 : 1); // one K-major operand slot: [A hi][B hi] ([A lo][B lo])
	static constexpr int SLOT_OFFSET = STAGES * RAW_BYTES;
	static constexpr int STATS_OFFSET = SLOT_OFFSET + (XF ? 2 * SLOT_BYTES : 0);
	static constexpr int STATS_BYTES = XF ? 0 : 4 * BN * 4 * 4 + 2 * 4 * BN * 3 * 4; // running (n, k, s1, s2) per slot + per-warp partials
	static constexpr int BAR_OFFSET = STATS_OFFSET + STATS_BYTES;
	static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;           // barriers + slack for the 1024-byte alignment
};

// stages per kernel: as deep as 227 KB of shared memory allows with the transform slots (A from registers: 3 stages of 48 KB and
// two 32 KB B slots at BN = 256; 4 at BN = 64 / 128, which ran ResNet-50's weight gradients no slower than 6).  The swapped weight
// gradient (A = OP_IM2COL_RS, BN <= 64) does little MMA work per stage, so it keeps more stages in flight: 8 of up to 24 KB with
// 128-row tiles, 5 of up to 40 KB with 256-row tiles.
template <int BN, bool XF, int X3, bool ARS = false, int BM = UMMA_BLOCK_M, bool SWAP = false>
struct GemmStages {
	static constexpr int value = SWAP ? (BM == 256 ? 5 : 8) : ARS ? (BN == 256 ? 3 : 4) : X3 ? (BN == 128 ? 3 : 4) : (XF ? 4 : (BN == 128 ? 5 : 6));
};

// one staged fp32 operand tile (rows x 32 k) -> K-major 128-byte-swizzled slot (16-byte chunk c of row r at chunk c ^ (r & 7)).
// MN-major input (T): 32-wide MN boxes of 32 k-rows of 128 B, no swizzle; K-major input: already in the slot layout.
template <bool T, int X3>
__device__ __forceinline__ void xform_tile(const float* __restrict__ raw, float* __restrict__ hi, float* __restrict__ lo, const int rows, const int tid)
{
	for (int idx = tid; idx < rows * 8; idx += 256)
	{
		float4 x;
		int dst;
		if (T)
		{
			const int mn = idx % rows, c = idx / rows;
			const float* const src = raw + (mn >> 5) * 1024 + (c * 4) * 32 + (mn & 31);
			x = make_float4(src[0], src[32], src[64], src[96]);
			dst = mn * 32 + ((c ^ (mn & 7)) << 2);
		} else {
			x = reinterpret_cast<const float4*>(raw)[idx];
			dst = idx * 4;
		}
		if (X3)
		{
			float4 h, l;
			h.x = __uint_as_float(__float_as_uint(x.x) & 0xffffe000u), h.y = __uint_as_float(__float_as_uint(x.y) & 0xffffe000u);
			h.z = __uint_as_float(__float_as_uint(x.z) & 0xffffe000u), h.w = __uint_as_float(__float_as_uint(x.w) & 0xffffe000u);
			// x - hi is exact; an infinity keeps lo = 0 so that inf stays inf instead of turning into inf - inf
			l.x = fabsf(x.x) < __int_as_float(0x7f800000) ? x.x - h.x : 0.f, l.y = fabsf(x.y) < __int_as_float(0x7f800000) ? x.y - h.y : 0.f;
			l.z = fabsf(x.z) < __int_as_float(0x7f800000) ? x.z - h.z : 0.f, l.w = fabsf(x.w) < __int_as_float(0x7f800000) ? x.w - h.w : 0.f;
			*reinterpret_cast<float4*>(hi + dst) = h;
			*reinterpret_cast<float4*>(lo + dst) = l;
		} else
			*reinterpret_cast<float4*>(hi + dst) = x;
	}
}

// A = OP_MN2D_RS: one consumer warp's wgmma A fragments of a stage (4 MMA steps of k = 8) from the staged MN-major tile, four
// 32-row boxes of 32 k-rows of 128 B.  The stage is 128-byte swizzled: 16-byte chunk c of k-row k sits at c ^ (k & 7).  A fragment
// load takes 8 rows (lane / 4) x 4 k (lane % 4); rows are contiguous, so unswizzled those 32 words fall in 8 banks (4-way conflict)
// and swizzled with the natural rows in 16 (2-way).  So fragment row lane / 4 = i (a0 / a2; a1 / a3: h = 1) of warp w holds row
// a_row(w, lane, h) = 32 (w >> 1) + 16 (i >> 2) + 8 (w & 1) + 4 h + (i & 3) of the warpgroup's 64: chunk (4 (i >> 2) + 2 (w & 1) + h)
// ^ (k & 7), word i & 3, 32 distinct banks.  The accumulator rows follow the A rows, so the epilogue stores them by the same map.
__device__ __forceinline__ int a_row(const int warp, const int lane, const int h)
{
	const int i = lane >> 2;
	return 32 * ((warp >> 1) & 1) + 16 * (i >> 2) + 8 * (warp & 1) + 4 * h + (i & 3);
}
__device__ __forceinline__ void load_a_frags(uint32_t (&af)[4][4], const float* __restrict__ raw_wg, const int warp, const int lane)
{
	const int i = lane >> 2, j = lane & 3;
	// k = 8 step + j + 4 e: k-row offset 32 k; chunk ((4 (i >> 2) + 2 (w & 1)) ^ j) ^ h ^ 4 e
	const float* const src = raw_wg + ((warp >> 1) & 1) * 1024 + j * 32 + (i & 3);
	const int c = ((4 * (i >> 2) + 2 * (warp & 1)) ^ j) << 2;
#pragma unroll
	for (int step = 0; step < 4; step++)
#pragma unroll
		for (int e = 0; e < 2; e++)
#pragma unroll
			for (int h = 0; h < 2; h++)
				af[step][2 * e + h] = __float_as_uint(src[step * 256 + e * 128 + (c ^ (h << 2) ^ (e << 4))]);
}

// K16 = 1 / 2: bf16 / fp16 operands (p.out_kind holds the same kind), 64 elements per 128-byte row, K = 16 per MMA; K16 = 0: fp32
// operands (32 per row, K = 8 per MMA).  The element type is a template parameter so that every wgmma of a k-step sits in one basic
// block (a runtime type branch makes ptxas fence each MMA on its own).  OUT16 = 1: the output tensor (and an optional 16-bit bias) is bf16 / fp16 (p.out_kind).
// BM: output rows per tile, 128 (64 per consumer warpgroup) or, for A = OP_IM2COL_RS only, 256 (two m64 blocks per warpgroup).
template <int AMODE, int BMODE, int BN, int STAGES, int X3 = 0, int K16 = 0, int OUT16 = 0, int BM = UMMA_BLOCK_M>
__global__ void __launch_bounds__(AMODE == OP_MN2D_RS || AMODE == OP_IM2COL_RS ? GEMM_THREADS_RS : GEMM_THREADS, 1) umma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const UmmaGemmParams p)
{
	using XF = GemmXform<AMODE, BMODE, K16, X3>;
	using S = UmmaSmem<BN, STAGES, XF::ANY, X3, XF::A_RS, BM>;
	constexpr bool SWAP = AMODE == OP_IM2COL_RS;
	constexpr int MSUB = BM / UMMA_BLOCK_M; // m64 blocks per consumer warpgroup
	extern __shared__ uint8_t smem_raw[];
	uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
	uint64_t* full_bar = (uint64_t*)(smem + S::BAR_OFFSET);
	uint64_t* empty_bar = full_bar + STAGES;

	constexpr int BK = K16 ? 64 : 32;          // K elements per stage = MN elements per MN-major box: one 128-byte span
	constexpr int MN_BOX_BYTES = BK * 128;     // an MN-major box: BK k-rows of 128 bytes
	const int warp = threadIdx.x >> 5;
	const int lane = threadIdx.x & 31;
	const int tiles_m = (p.M + BM - 1) / BM; // M tiles blockIdx.x, blockIdx.x + gridDim.x, ... (launch_umma picks gridDim.x)
	const int n0 = blockIdx.y * BN;
	const int split = blockIdx.z % p.splits;
	const int gtap = blockIdx.z / p.splits;
	const int per = (p.k_iters + p.splits - 1) / p.splits;
	const int it_begin = split * per;
	const int it_end = min(p.k_iters, it_begin + per);
	const int n_it = max(it_end - it_begin, 0);

	if (threadIdx.x == 0)
	{
		for (int s = 0; s < STAGES; s++)
		{
			mbar_init(&full_bar[s], 1);
			mbar_init(&empty_bar[s], XF::ANY ? 1 : 2); // transform: one arrival after the consumers' barrier; else one per warpgroup
		}
		fence_mbar_init();
	}
	__syncthreads();

	if (XF::A_RS ? warp >= 8 : warp == 8)
	{
		// ------------------------------------------------------------------ TMA producer
		if constexpr (XF::A_RS)
		{
			setmaxnreg_dec<56>(); // 2 x 224 + 56 registers per scheduler: the whole file
			if (warp != 8)
				return;
		}
		if (elect_one())
		{
			tma_prefetch_desc(&tmA);
			tma_prefetch_desc(&tmB);
			// B = OP_IM2COL: each BK-column box of the tile loads one filter tap's channel span (C_tap is a multiple of BK when a
			// tile holds several taps; with the tap on the grid, N = C_tap and every box is at the grid tap); a box past the last
			// column asks for channels beyond C, which the TMA unit fills with zeros
			int b_ch[BN / BK], b_off_w[BN / BK], b_off_h[BN / BK];
#pragma unroll
			for (int j = 0; j < BN / BK; j++)
			{
				const int col = n0 + BK * j;
				const int t = BMODE == OP_IM2COL && col < p.N ? col / p.C_tap : 0;
				b_ch[j] = col - t * p.C_tap;
				if (BMODE == OP_IM2COL)
					b_off_w[j] = p.tap_off_w[gtap + t], b_off_h[j] = p.tap_off_h[gtap + t];
			}
			int stage = 0;
			uint32_t phase = 0;
			for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x)
			{
			const int m0 = mt * BM;
			// A = OP_IM2COL_RS: box j holds rows [m0 + 32 j, +32), one tap's channel span (C_tap is a multiple of 32); a box past the
			// last row asks for channels beyond C, which the TMA unit fills with zeros
			int a_ch[SWAP ? BM / 32 : 1], a_off_w[SWAP ? BM / 32 : 1], a_off_h[SWAP ? BM / 32 : 1];
			if constexpr (SWAP)
			{
#pragma unroll
				for (int j = 0; j < BM / 32; j++)
				{
					const int row = m0 + 32 * j;
					const int t = row < p.M ? row / p.C_tap : 0;
					a_ch[j] = row - t * p.C_tap, a_off_w[j] = p.tap_off_w[t], a_off_h[j] = p.tap_off_h[t];
				}
			}
			int a_w = 0, a_h = 0, a_n = 0;
			if (AMODE == OP_IM2COL)
			{
				const int q = m0 % p.Q;
				const int t = m0 / p.Q;
				a_w = q * p.stride_w + p.base_w;
				a_h = (t % p.P) * p.stride_h + p.base_h;
				a_n = t / p.P;
			}
			for (int it = it_begin; it < it_end; it++)
			{
				const int tap = it / p.chunks_per_tap;
				const int chunk = it - tap * p.chunks_per_tap;
				mbar_wait(&empty_bar[stage], phase ^ 1);
				uint8_t* sA = smem + stage * S::RAW_BYTES;
				uint8_t* sB = sA + S::A_BYTES;
				mbar_expect_tx(&full_bar[stage], S::RAW_BYTES);
				if (AMODE == OP_K2D)
					tma_load_2d(sA, &tmA, &full_bar[stage], chunk * BK, m0);
				else if (AMODE == OP_IM2COL_RS) {
					// pixels are the reduction: this iteration covers base pixels [it * BK, it * BK + BK)
					const int pix = it * BK;
					const int q = pix % p.Q;
					const int t = pix / p.Q;
					const int x_w = q * p.stride_w + p.base_w;
					const int x_h = (t % p.P) * p.stride_h + p.base_h;
					const int x_n = t / p.P;
#pragma unroll
					for (int j = 0; j < BM / 32; j++)
						tma_load_im2col_4d(sA + j * MN_BOX_BYTES, &tmA, &full_bar[stage], a_ch[j], x_w, x_h, x_n, (uint16_t)a_off_w[j], (uint16_t)a_off_h[j]);
				} else if (AMODE == OP_MN2D || AMODE == OP_MN2D_RS) {
#pragma unroll
					for (int j = 0; j < UMMA_BLOCK_M / BK; j++)
						tma_load_2d(sA + j * MN_BOX_BYTES, &tmA, &full_bar[stage], m0 + BK * j, it * BK);
				} else
					tma_load_im2col_4d(sA, &tmA, &full_bar[stage], chunk * BK, a_w, a_h, a_n, p.tap_off_w[tap], p.tap_off_h[tap]);
				if (BMODE == OP_K2D)
					tma_load_2d(sB, &tmB, &full_bar[stage], p.tap_b_col[tap] + chunk * BK, p.tap_b_row[tap] + n0);
				else if (BMODE == OP_MN2D) {
#pragma unroll
					for (int j = 0; j < BN / BK; j++)
						tma_load_2d(sB + j * MN_BOX_BYTES, &tmB, &full_bar[stage], p.tap_b_col[tap] + n0 + BK * j, chunk * BK);
				} else {
					// pixels are the reduction: this iteration covers base pixels [it * BK, it * BK + BK)
					const int pix = it * BK;
					const int q = pix % p.Q;
					const int t = pix / p.Q;
					const int b_w = q * p.stride_w + p.base_w;
					const int b_h = (t % p.P) * p.stride_h + p.base_h;
					const int b_n = t / p.P;
#pragma unroll
					for (int j = 0; j < BN / BK; j++)
						tma_load_im2col_4d(sB + j * MN_BOX_BYTES, &tmB, &full_bar[stage], b_ch[j], b_w, b_h, b_n, (uint16_t)b_off_w[j], (uint16_t)b_off_h[j]);
				}
				if (++stage == STAGES) { stage = 0; phase ^= 1; }
			}
			}
		}
		return;
	}

	// ------------------------------------------------------------------ consumers (warps 0..7)
	if constexpr (XF::A_RS)
		setmaxnreg_inc<224>();
	const int wg = warp >> 2; // output rows [64 * MSUB * wg, +64 * MSUB) of the tile
	float acc[MSUB * BN / 2];
	constexpr bool A_MN16 = K16 && AMODE == OP_MN2D, B_MN16 = K16 && BMODE != OP_K2D;
	constexpr uint32_t A_STEP = A_MN16 ? 2048 : 32, B_STEP = B_MN16 ? 2048 : 32; // bytes per MMA step along K
	int stage = 0;
	uint32_t phase = 0;
	int prev_stage = 0;
	int gi = 0; // k-iterations of all tiles so far: the operand slot parity
	float* const st_run = reinterpret_cast<float*>(smem + S::STATS_OFFSET); // [4 quarters][BN] x (n, k, s1, s2)
	float* const st_part = st_run + 4 * BN * 4;                                // [2 warps of a quarter][4 quarters][BN] x (k, s1, s2)
	const bool stats = !XF::ANY && p.stats != 0;
	if (stats)
		for (int i = threadIdx.x; i < 4 * BN; i += 256)
			st_run[i * 4] = 0.f;
	for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x)
	{
	const int m0 = mt * BM;
#pragma unroll
	for (int i = 0; i < MSUB * BN / 2; i++)
		acc[i] = 0.f;
	uint32_t af[MSUB][4][4]; // A from registers: this k-iteration's A fragments
	for (int it = 0; it < n_it; it++, gi++)
	{
		mbar_wait(&full_bar[stage], phase);
		uint8_t* op = smem + stage * S::RAW_BYTES;
		if (XF::ANY)
		{
			// every consumer has retired the MMAs that read slot (it & 1) two iterations ago (wgmma_wait<1> below)
			named_bar_sync(1, 256);
			op = smem + S::SLOT_OFFSET + (gi & 1) * S::SLOT_BYTES;
			const float* const raw = reinterpret_cast<const float*>(smem + stage * S::RAW_BYTES);
			float* const hi = reinterpret_cast<float*>(op);
			float* const lo = reinterpret_cast<float*>(op + S::RAW_BYTES);
			if constexpr (!XF::A_RS)
				xform_tile<XF::A_T, X3>(raw, hi, lo, UMMA_BLOCK_M, threadIdx.x);
			xform_tile<XF::B_T, X3>(raw + S::A_BYTES / 4, hi + S::SLOT_A_BYTES / 4, lo + S::SLOT_A_BYTES / 4, BN, threadIdx.x);
			if constexpr (XF::A_RS)
			{
				// B went into slot gi & 1 while the MMAs of iteration it - 1 still ran.  Those read the fragment registers until they
				// complete (overwritten in flight, ptxas would serialise every wgmma), so only now load this stage's; the stage is
				// released below
				wgmma_wait<0>();
#pragma unroll
				for (int u = 0; u < MSUB; u++)
					load_a_frags(af[u], raw + (wg * MSUB + u) * 2048, warp, lane);
			}
			fence_proxy_async(); // the tensor core reads shared memory through the async proxy
			named_bar_sync(1, 256);
			if (threadIdx.x == 0)
				mbar_arrive(&empty_bar[stage]); // the raw stage has been consumed
		}
		const uint32_t base = smem_u32(op);
		const uint64_t da0 = wgmma_desc(base + wg * 8192, 16, 1024);
		const uint64_t db0 = wgmma_desc(base + S::SLOT_A_BYTES, 8192, 1024);
		fence_regs(acc);
		wgmma_fence();
#pragma unroll
		for (int k = 0; k < 4; k++)
		{
			const uint64_t da = da0 + ((k * A_STEP) >> 4), db = db0 + ((k * B_STEP) >> 4);
			if constexpr (K16 != 0)
			{
				if constexpr (K16 == 1)
				{
					if constexpr (BN == 128)
						wgmma_bf16_ss_n128<A_MN16, B_MN16>(*reinterpret_cast<float(*)[64]>(acc), da, db);
					else
						wgmma_bf16_ss_n64<A_MN16, B_MN16>(*reinterpret_cast<float(*)[32]>(acc), da, db);
				} else {
					if constexpr (BN == 128)
						wgmma_f16_ss_n128<A_MN16, B_MN16>(*reinterpret_cast<float(*)[64]>(acc), da, db);
					else
						wgmma_f16_ss_n64<A_MN16, B_MN16>(*reinterpret_cast<float(*)[32]>(acc), da, db);
				}
			} else if constexpr (XF::A_RS) {
#pragma unroll
				for (int u = 0; u < MSUB; u++)
				{
					float* const d = acc + u * (BN / 2);
					if constexpr (BN == 256)
						wgmma_tf32_rs_n256(*reinterpret_cast<float(*)[128]>(d), af[u][k], db);
					else if constexpr (BN == 128)
						wgmma_tf32_rs_n128(*reinterpret_cast<float(*)[64]>(d), af[u][k], db);
					else if constexpr (BN == 64)
						wgmma_tf32_rs_n64(*reinterpret_cast<float(*)[32]>(d), af[u][k], db);
					else
						wgmma_tf32_rs_n32(*reinterpret_cast<float(*)[16]>(d), af[u][k], db);
				}
			} else {
				constexpr uint32_t LO = (uint32_t)(S::RAW_BYTES >> 4);
				if constexpr (BN == 128)
				{
					float (&d)[64] = *reinterpret_cast<float(*)[64]>(acc);
					if (X3)
					{
						// small terms first, then hi * hi
						wgmma_tf32_ss_n128(d, da + LO, db);
						wgmma_tf32_ss_n128(d, da, db + LO);
					}
					wgmma_tf32_ss_n128(d, da, db);
				} else {
					float (&d)[32] = *reinterpret_cast<float(*)[32]>(acc);
					if (X3)
					{
						wgmma_tf32_ss_n64(d, da + LO, db);
						wgmma_tf32_ss_n64(d, da, db + LO);
					}
					wgmma_tf32_ss_n64(d, da, db);
				}
			}
		}
		wgmma_commit();
		fence_regs(acc);
		wgmma_wait<1>(); // the MMAs of iteration it - 1 are complete
		if (!XF::ANY && it > 0 && (threadIdx.x & 127) == 0)
			mbar_arrive(&empty_bar[prev_stage]);
		prev_stage = stage;
		if (++stage == STAGES) { stage = 0; phase ^= 1; }
	}
	wgmma_wait<0>();
	fence_regs(acc);
	if (!XF::ANY && n_it > 0 && (threadIdx.x & 127) == 0)
		mbar_arrive(&empty_bar[prev_stage]); // the last stage of this tile

	// ------------------------------------------------------------------ epilogue: accumulator i -> (row, column), see sm100_ptx.cuh
	if constexpr (SWAP)
	{
		// the tile is the transpose of the output: row m (filter tap * C_tap + channel) -> output column m, column n -> output row n
		// (dW[K, R*S*C], or this split's slice of it); no bias, no 16-bit output, no statistics
		float* const out = p.out + (long long)split * p.split_out_stride;
		const bool accumulate = p.accumulate != 0;
#pragma unroll
		for (int u = 0; u < MSUB; u++)
#pragma unroll
			for (int h = 0; h < 2; h++)
			{
				const int row = m0 + (wg * MSUB + u) * 64 + a_row(warp, lane, h);
				if (row >= p.M)
					continue;
#pragma unroll
				for (int j = 0; j < BN / 8; j++)
#pragma unroll
					for (int e = 0; e < 2; e++)
					{
						const int col = n0 + 8 * j + 2 * (lane & 3) + e;
						if (col >= p.N)
							continue;
						float* const o = out + col * p.rowmap.ld + row;
						// + 0.f: the other layouts' epilogue adds a zero bias, which turns a -0 sum into +0
						const float v = acc[u * (BN / 2) + 4 * j + 2 * h + e] + 0.f;
						*o = accumulate ? *o + v : v;
					}
			}
		continue;
	}
	constexpr int OSZ = OUT16 ? 2 : 4;
	const bool add_bias = split == 0;
	const float* const bias = p.bias;
	const uint16_t* const bias16 = OUT16 && !p.bias ? reinterpret_cast<const uint16_t*>(p.bias16) : 0;
	char* orow[2];
#pragma unroll
	for (int h = 0; h < 2; h++)
	{
		const int row = m0 + wg * 64 + (XF::A_RS ? a_row(warp, lane, h) : (warp & 3) * 16 + (lane >> 2) + 8 * h);
		long long off;
		if (p.rowmap.mode == 0)
			off = (long long)row * p.rowmap.ld;
		else {
			const int pq = p.rowmap.Pc * p.rowmap.Qc;
			const int n = row / pq;
			const int rem = row - n * pq;
			const int ii = rem / p.rowmap.Qc;
			const int jj = rem - ii * p.rowmap.Qc;
			off = n * p.rowmap.n_stride + ii * p.rowmap.h_stride + jj * p.rowmap.w_stride;
		}
		orow[h] = row < p.M ? reinterpret_cast<char*>(p.out) + (off + (long long)gtap * p.grid_tap_out_stride + (long long)split * p.split_out_stride) * OSZ : 0;
	}
	const int N = p.N;
	const bool accumulate = p.accumulate != 0;
#pragma unroll
	for (int j = 0; j < BN / 8; j++)
	{
		const int col = n0 + 8 * j + 2 * (lane & 3);
		if (col >= N)
			continue;
		const bool two = col + 1 < N;
		float b0 = 0.f, b1 = 0.f;
		if (add_bias && bias)
			b0 = __ldg(bias + col), b1 = two ? __ldg(bias + col + 1) : 0.f;
		else if (add_bias && bias16)
			b0 = cvt16(__ldg(bias16 + col), p.out_kind), b1 = two ? cvt16(__ldg(bias16 + col + 1), p.out_kind) : 0.f;
#pragma unroll
		for (int h = 0; h < 2; h++)
		{
			if (!orow[h])
				continue;
			float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
			if (!OUT16)
			{
				float* const o = reinterpret_cast<float*>(orow[h]) + col;
				if (two && ((((uintptr_t)o) & 7) == 0))
				{
					if (accumulate)
					{
						const float2 e = *reinterpret_cast<const float2*>(o);
						v0 += e.x, v1 += e.y;
					}
					*reinterpret_cast<float2*>(o) = make_float2(v0, v1);
				} else {
					o[0] = accumulate ? o[0] + v0 : v0;
					if (two)
						o[1] = accumulate ? o[1] + v1 : v1;
				}
			} else {
				uint16_t* const o = reinterpret_cast<uint16_t*>(orow[h]) + col;
				if (two && ((((uintptr_t)o) & 3) == 0))
				{
					if (accumulate)
					{
						const uint32_t e = *reinterpret_cast<const uint32_t*>(o);
						v0 += cvt16((uint16_t)(e & 0xffffu), p.out_kind), v1 += cvt16((uint16_t)(e >> 16), p.out_kind);
					}
					*reinterpret_cast<uint32_t*>(o) = pack16x2(v0, v1, p.out_kind);
				} else {
					o[0] = (uint16_t)(pack16x2(accumulate ? cvt16(o[0], p.out_kind) + v0 : v0, 0.f, p.out_kind) & 0xffffu);
					if (two)
						o[1] = (uint16_t)(pack16x2(accumulate ? cvt16(o[1], p.out_kind) + v1 : v1, 0.f, p.out_kind) & 0xffffu);
				}
			}
		}
	}
	if (stats)
	{
		// per warp: shifted sums of its 16 rows (as stored: after the bias and the 16-bit rounding) per column, shift = the warp's first
		// row; lanes 0..3 leave them in st_part for the slot owners
		const int quarter = wg * 2 + ((warp & 3) >> 1), half = warp & 1;
		const int row0 = m0 + wg * 64 + (warp & 3) * 16;
		const int valid = max(0, min(16, p.M - row0));
		const bool r1_ok = (lane >> 2) + 8 < valid, r0_ok = (lane >> 2) < valid;
		float* const part = st_part + ((half * 4 + quarter) * BN) * 3;
#pragma unroll
		for (int j = 0; j < BN / 8; j++)
#pragma unroll
			for (int e = 0; e < 2; e++)
			{
				const int c = n0 + 8 * j + 2 * (lane & 3) + e;
				float v0 = acc[4 * j + e] + (bias && c < p.N ? __ldg(bias + c) : (bias16 && c < p.N ? cvt16(__ldg(bias16 + c), p.out_kind) : 0.f));
				float v1 = acc[4 * j + 2 + e] + (bias && c < p.N ? __ldg(bias + c) : (bias16 && c < p.N ? cvt16(__ldg(bias16 + c), p.out_kind) : 0.f));
				if (OUT16)
					v0 = cvt16((uint16_t)(pack16x2(v0, 0.f, p.out_kind) & 0xffffu), p.out_kind), v1 = cvt16((uint16_t)(pack16x2(v1, 0.f, p.out_kind) & 0xffffu), p.out_kind);
				const float k = __shfl_sync(0xffffffffu, v0, lane & 3);
				const float d0 = r0_ok ? v0 - k : 0.f, d1 = r1_ok ? v1 - k : 0.f;
				float s1 = d0 + d1, s2 = fmaf(d0, d0, d1 * d1);
#pragma unroll
				for (int m = 4; m <= 16; m <<= 1)
					s1 += __shfl_xor_sync(0xffffffffu, s1, m), s2 += __shfl_xor_sync(0xffffffffu, s2, m);
				if (lane < 4)
				{
					float* const q = part + (8 * j + 2 * lane + e) * 3;
					q[0] = k, q[1] = s1, q[2] = s2;
				}
			}
		named_bar_sync(1, 256);
		// slot owners: (quarter, column) -> merge the two warps' sums, shifted to the slot's own k (exact algebra: d' = d + (k_w - k))
		for (int i = threadIdx.x; i < 4 * BN; i += 256)
		{
			const int q = i / BN, c = i - q * BN;
			float* const run = st_run + i * 4;
#pragma unroll
			for (int h = 0; h < 2; h++)
			{
				const float nw = (float)max(0, min(16, p.M - (m0 + q * 32 + h * 16)));
				if (nw <= 0.f)
					continue;
				const float* const w = st_part + ((h * 4 + q) * BN + c) * 3;
				if (run[0] == 0.f)
					run[1] = w[0], run[2] = 0.f, run[3] = 0.f;
				const float dk = w[0] - run[1];
				run[3] += w[2] + 2.f * dk * w[1] + nw * dk * dk;
				run[2] += w[1] + nw * dk;
				run[0] += nw;
			}
		}
		named_bar_sync(1, 256);
	}
	}
	if (stats)
	{
		const size_t plane = (size_t)p.stats_rows * p.N;
		for (int i = threadIdx.x; i < 4 * BN; i += 256)
		{
			const int q = i / BN, c = n0 + i - q * BN;
			const float* const run = st_run + i * 4;
			if (c < p.N && run[0] > 0.f)
			{
				float* const slot = p.stats + ((size_t)blockIdx.x * 4 + q) * p.N + c;
				slot[0] = run[0], slot[plane] = run[1], slot[2 * plane] = run[2], slot[3 * plane] = run[3];
			}
		}
	}
}

} // namespace sm100
