// sm100_contract.cu -- host-side launchers for the wgmma/TMA contraction kernel (sm100_umma_gemm.cuh):
// tensor-map encoding (tile and im2col mode) and the mapping of GEMM / convolution fprop / dgrad / wgrad
// onto its operand modes.  Reference semantics being reproduced: lib/nnc/cmd/blas/ccv_nnc_gemm_cpu_ref.c:110-448,
// lib/nnc/cmd/convolution/ccv_nnc_conv_cpu_ref.c:13-345 (NHWC).
#include "sm100_contract.h"
#include "sm100_umma_gemm.cuh"
#include "sm100_elem.cuh"
#include "sm100_ew.h"
#include <atomic>
#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace sm100 {

// ------------------------------------------------------------------------------------------------ bookkeeping
static std::atomic<unsigned long long> g_launches(0);
static char g_last_error[256] = "";
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
unsigned long long launch_count() { return g_launches.load(std::memory_order_relaxed); }
void set_last_error(const char* what, cudaError_t err)
{
	snprintf(g_last_error, sizeof(g_last_error), "%s: %s", what, cudaGetErrorString(err));
	fprintf(stderr, "[ccv_nnc_sm100] %s\n", g_last_error);
}
const char* last_error() { return g_last_error; }

// ------------------------------------------------------------------------------------------------ TMA descriptors
typedef CUresult (*encode_tiled_f)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*encode_im2col_f)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_f g_encode_tiled = 0;
static encode_im2col_f g_encode_im2col = 0;
static int g_driver_version = 0;
static int g_tma_dtype = -1; // CUtensorMapDataType used for fp32 operands

static bool tma_api_init()
{
	static std::once_flag once;
	std::call_once(once, []() {
		void* fn = 0;
		cudaDriverEntryPointQueryResult qres;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
			g_encode_tiled = (encode_tiled_f)fn;
		fn = 0;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
			g_encode_im2col = (encode_im2col_f)fn;
		cudaDriverGetVersion(&g_driver_version);
		// TFLOAT32 makes the TMA unit write round-to-nearest TF32 values into shared memory, so the tensor core's
		// implicit truncation of the low 13 mantissa bits becomes a no-op (unbiased error instead of a 2^-11 bias).
		const char* e = getenv("CCV_NNC_SM100_TMA_DTYPE");
		g_tma_dtype = e ? atoi(e) : (int)CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;
	});
	return g_encode_tiled != 0 && g_encode_im2col != 0;
}

// Math mode of the launches a contraction entry point issues: 0 = one-pass TF32 (operands rounded to TF32 by the TMA unit),
// 1 = 3xTF32 (raw fp32 operands, hi / lo split in shared memory, three MMAs per k-step).  Set by the
// entry points for the duration of the call (host thread local, like the statistics request).
static thread_local int t_x3 = 0;
struct X3Scope {
	int saved;
	explicit X3Scope(int x3) : saved(t_x3) { t_x3 = x3; }
	~X3Scope() { t_x3 = saved; }
};
static inline int operand_dtype() { return t_x3 ? (int)CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : g_tma_dtype; }

// fp32 2-D row-major [rows, cols] with row pitch `ld` elements; box = {box_cols (<= 32), box_rows}.  K-major operand tiles are
// 128-byte swizzled (the wgmma layout); MN-major ones land unswizzled and the kernel transposes them (sm100_umma_gemm.cuh)
static bool make_map_2d(CUtensorMap* map, const float* ptr, long long rows, long long cols, long long ld, int box_cols, int box_rows, bool mn_major = false, int dtype = -1)
{
	if (dtype < 0)
		dtype = operand_dtype();
	if ((((uintptr_t)ptr) & 15) || ((ld * 4) & 15) || ld * 4 >= (1ll << 40))
		return false;
	cuuint64_t dims[2] = { (cuuint64_t)cols, (cuuint64_t)rows };
	cuuint64_t strides[1] = { (cuuint64_t)ld * 4 };
	cuuint32_t box[2] = { (cuuint32_t)box_cols, (cuuint32_t)box_rows };
	cuuint32_t estr[2] = { 1, 1 };
	CUresult r = g_encode_tiled(map, (CUtensorMapDataType)dtype, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, mn_major ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	return r == CUDA_SUCCESS;
}

// 16-bit (bf16 / fp16) 2-D row-major [rows, cols], row pitch `ld` elements; box = {box_cols (<= 64 = one 128-byte span), box_rows}.
// kind: 1 = bf16, 2 = fp16.  MN-major 16-bit operands use the same 128-byte swizzle (64-element atoms, wgmma's transposed layout).
static bool make_map_2d16(CUtensorMap* map, const void* ptr, int kind, long long rows, long long cols, long long ld, int box_cols, int box_rows)
{
	if ((((uintptr_t)ptr) & 15) || ((ld * 2) & 15) || ld * 2 >= (1ll << 40))
		return false;
	cuuint64_t dims[2] = { (cuuint64_t)cols, (cuuint64_t)rows };
	cuuint64_t strides[1] = { (cuuint64_t)ld * 2 };
	cuuint32_t box[2] = { (cuuint32_t)box_cols, (cuuint32_t)box_rows };
	cuuint32_t estr[2] = { 1, 1 };
	const CUresult r = g_encode_tiled(map, kind == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
		CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	return r == CUDA_SUCCESS;
}
// 16-bit NHWC tensor {C, W, H, N} in im2col mode (element strides sn, sh, sw; channel stride 1)
static bool make_map_im2col16(CUtensorMap* map, const void* ptr, int kind, int N, int H, int W, int C, long long sn, long long sh, long long sw, int lower_h, int lower_w, int upper_h, int upper_w, int trav_h, int trav_w, int channels, int pixels)
{
	if ((((uintptr_t)ptr) & 15) || ((sw * 2) & 15) || ((sh * 2) & 15) || ((sn * 2) & 15))
		return false;
	if (lower_h < -128 || lower_h > 127 || lower_w < -128 || lower_w > 127 || upper_h < -128 || upper_h > 127 || upper_w < -128 || upper_w > 127)
		return false;
	if (trav_h < 1 || trav_h > 8 || trav_w < 1 || trav_w > 8)
		return false;
	cuuint64_t dims[4] = { (cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N };
	cuuint64_t strides[3] = { (cuuint64_t)sw * 2, (cuuint64_t)sh * 2, (cuuint64_t)sn * 2 };
	int lower[2] = { lower_w, lower_h };
	int upper[2] = { upper_w, upper_h };
	cuuint32_t estr[4] = { 1, (cuuint32_t)trav_w, (cuuint32_t)trav_h, 1 };
	const CUresult r = g_encode_im2col(map, kind == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)ptr, dims, strides, lower, upper, (cuuint32_t)channels, (cuuint32_t)pixels, estr,
		CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS)
		return false;
	if (g_driver_version <= 13010 && (long long)N * sn * 2 < 131072) // same driver workaround as make_map_im2col
		reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
	return true;
}

// fp32 NHWC tensor {C, W, H, N} in im2col mode. Base pixels run over [lower, dim + upper) per spatial axis with the
// given traversal stride; each load fetches `pixels` base pixels x `channels` channels at base + tap offset.
static bool make_map_im2col(CUtensorMap* map, const float* ptr, int N, int H, int W, int C, long long sn, long long sh, long long sw, int lower_h, int lower_w, int upper_h, int upper_w, int trav_h, int trav_w, int channels, int pixels, bool mn_major = false, int dtype = -1)
{
	if (dtype < 0)
		dtype = operand_dtype();
	if ((((uintptr_t)ptr) & 15) || ((sw * 4) & 15) || ((sh * 4) & 15) || ((sn * 4) & 15))
		return false;
	if (lower_h < -128 || lower_h > 127 || lower_w < -128 || lower_w > 127 || upper_h < -128 || upper_h > 127 || upper_w < -128 || upper_w > 127)
		return false;
	if (trav_h < 1 || trav_h > 8 || trav_w < 1 || trav_w > 8)
		return false;
	cuuint64_t dims[4] = { (cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N };
	cuuint64_t strides[3] = { (cuuint64_t)sw * 4, (cuuint64_t)sh * 4, (cuuint64_t)sn * 4 };
	int lower[2] = { lower_w, lower_h };
	int upper[2] = { upper_w, upper_h };
	cuuint32_t estr[4] = { 1, (cuuint32_t)trav_w, (cuuint32_t)trav_h, 1 };
	CUresult r = g_encode_im2col(map, (CUtensorMapDataType)dtype, 4, (void*)ptr, dims, strides, lower, upper, (cuuint32_t)channels, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, mn_major ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS)
		return false;
	// Same driver workaround CUTLASS applies (cute/atom/copy_traits_sm90_im2col.hpp): for tensors under 128 KiB, drivers
	// <= 13.1 set a descriptor bit that makes im2col loads fault.
	if (g_driver_version <= 13010 && (long long)N * sn * 4 < 131072)
		reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
	return true;
}

// ------------------------------------------------------------------------------------------------ launch
static int g_num_sms = 0;
static int num_sms()
{
	if (!g_num_sms)
	{
		int dev = 0;
		cudaGetDevice(&dev);
		cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
		if (g_num_sms <= 0)
			g_num_sms = 132;
	}
	return g_num_sms;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: each launcher keeps one flag per device (a single
// process may drive several GPUs, comm/gpu/ccv_nnc_comm_gpu_nccl.cu:12-58)
constexpr int MAX_DEVICES = 64;
template <typename Kern>
static int ensure_dynamic_smem(Kern kern, int bytes, bool (&done)[MAX_DEVICES], const char* what)
{
	int dev = 0;
	cudaGetDevice(&dev);
	if (dev < 0 || dev >= MAX_DEVICES)
		dev = 0;
	if (done[dev])
		return 0;
	const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
	if (e != cudaSuccess)
	{
		set_last_error(what, e);
		return -1;
	}
	done[dev] = true;
	return 0;
}

// ------------------------------------------------------------------------------------------------ ordered split-K combine
// out[r, c] = (accumulate ? out[r, c] : 0) + part[0][r, c] + part[1][r, c] + ... in that order: the deterministic second half of
// every split-K launch (the contraction kernels write one scratch slice per split with plain stores).
// 16-bit outputs (out_kind 1 = bf16, 2 = fp16): out16 replaces out, the sum is rounded once at the end
__global__ void __launch_bounds__(256) splitk_reduce16_kernel(const float* __restrict__ part, const int splits, const long long split_stride, const int rows, const int cols, const long long ldp, uint16_t* __restrict__ out, const long long ldo, const int accumulate, const int out_kind)
{
	const long long total = (long long)rows * cols;
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		const int r = (int)(i / cols), c = (int)(i - (long long)r * cols);
		const float* src = part + (long long)r * ldp + c;
		uint16_t* const dst = out + (long long)r * ldo + c;
		float acc = accumulate ? cvt16(*dst, out_kind) : 0.f;
		for (int k = 0; k < splits; k++, src += split_stride)
			acc += *src;
		*dst = (uint16_t)(pack16x2(acc, 0.f, out_kind) & 0xffffu);
	}
}
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, const int splits, const long long split_stride, const int rows, const int cols, const long long ldp, float* __restrict__ out, const long long ldo, const int accumulate, const int vec)
{
	if (vec)
	{
		const int cv = cols >> 2;
		const long long total = (long long)rows * cv;
		for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
		{
			const int r = (int)(i / cv), c = (int)(i - (long long)r * cv) << 2;
			const float* src = part + (long long)r * ldp + c;
			float* const dst = out + (long long)r * ldo + c;
			float4 acc = accumulate ? *reinterpret_cast<const float4*>(dst) : make_float4(0.f, 0.f, 0.f, 0.f);
			int k = 0;
			for (; k + 1 < splits; k += 2, src += 2 * split_stride)
			{
				const float4 u = *reinterpret_cast<const float4*>(src), v = *reinterpret_cast<const float4*>(src + split_stride);
				acc.x += u.x, acc.y += u.y, acc.z += u.z, acc.w += u.w;
				acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
			}
			if (k < splits)
			{
				const float4 u = *reinterpret_cast<const float4*>(src);
				acc.x += u.x, acc.y += u.y, acc.z += u.z, acc.w += u.w;
			}
			*reinterpret_cast<float4*>(dst) = acc;
		}
	} else {
		const long long total = (long long)rows * cols;
		for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
		{
			const int r = (int)(i / cols), c = (int)(i - (long long)r * cols);
			const float* src = part + (long long)r * ldp + c;
			float* const dst = out + (long long)r * ldo + c;
			float acc = accumulate ? *dst : 0.f;
			for (int k = 0; k < splits; k++, src += split_stride)
				acc += *src;
			*dst = acc;
		}
	}
}
int splitk_reduce(cudaStream_t stream, const float* part, int splits, long long split_stride, int rows, int cols, long long ldp, float* out, long long ldo, int accumulate, int out_kind)
{
	if (out_kind)
	{
		long long blocks = ((long long)rows * cols + 255) / 256;
		if (blocks > (long long)num_sms() * 8)
			blocks = (long long)num_sms() * 8;
		splitk_reduce16_kernel<<<(unsigned)(blocks < 1 ? 1 : blocks), 256, 0, stream>>>(part, splits, split_stride, rows, cols, ldp, (uint16_t*)out, ldo, accumulate, out_kind);
		count_launch();
		const cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
		{
			set_last_error("splitk_reduce16_kernel", e);
			return -1;
		}
		return 0;
	}
	const int vec = cols % 4 == 0 && ldp % 4 == 0 && ldo % 4 == 0 && split_stride % 4 == 0 && ((((uintptr_t)part) | ((uintptr_t)out)) & 15) == 0;
	const long long work = (long long)rows * (vec ? cols / 4 : cols);
	long long blocks = (work + 255) / 256;
	if (blocks > (long long)num_sms() * 8)
		blocks = (long long)num_sms() * 8;
	if (blocks < 1)
		blocks = 1;
	splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, stream>>>(part, splits, split_stride, rows, cols, ldp, out, ldo, accumulate, vec);
	count_launch();
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		set_last_error("splitk_reduce_kernel", e);
		return -1;
	}
	return 0;
}
// the largest split factor <= splits whose slices fit the scratch and none of which is empty
static int fit_splits(int splits, int k_iters, size_t slice_bytes, const Scratch& scratch)
{
	if (splits <= 1 || !scratch.ptr || slice_bytes == 0)
		return 1;
	const size_t room = scratch.bytes / slice_bytes;
	long long k = splits;
	if ((size_t)k > room)
		k = (long long)room;
	while (k > 1 && (long long)((k_iters + k - 1) / k) * (k - 1) >= k_iters)
		k--;
	return (int)(k < 1 ? 1 : k);
}

// One-shot request (per host thread) for per-column output statistics from the next forward-shaped launch: set by the fused
// convolution + batch-norm command, consumed (and cleared) by launch_umma when the launch qualifies.
struct StatsRequest {
	float* part;
	int max_rows;
	int* rows_out;
};
static thread_local StatsRequest t_stats_request = { 0, 0, 0 };
void conv_stats_request(float* part, int max_rows, int* rows_out)
{
	t_stats_request.part = part, t_stats_request.max_rows = max_rows, t_stats_request.rows_out = rows_out;
	if (rows_out)
		*rows_out = 0;
}

template <int AMODE, int BMODE, int BN, int X3 = 0, int K16 = 0, int OUT16 = 0>
static int launch_umma(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const UmmaGemmParams& p)
{
	constexpr bool XF = GemmXform<AMODE, BMODE, K16, X3>::ANY;
	constexpr int STAGES = GemmStages<BN, XF, X3>::value;
	using S = UmmaSmem<BN, STAGES, XF, X3>;
	auto kern = umma_gemm_kernel<AMODE, BMODE, BN, STAGES, X3, K16, OUT16>;
	static bool configured[MAX_DEVICES];
	if (ensure_dynamic_smem(kern, S::TOTAL, configured, "cudaFuncSetAttribute(umma_gemm_kernel)"))
		return -1;
	const int tiles_m = (p.M + UMMA_BLOCK_M - 1) / UMMA_BLOCK_M, tiles_n = (p.N + BN - 1) / BN;
	dim3 grid(tiles_m, tiles_n, p.grid_taps * p.splits);
	UmmaGemmParams q = p;
	q.stats = 0, q.stats_rows = 0;
	if (t_stats_request.part)
	{
		const StatsRequest r = t_stats_request;
		t_stats_request.part = 0;
		// forward-shaped launches only (one statistics slot row per CTA column and 32-row quarter): each CTA walks every gridDim.x-th
		// M tile, so the slots fit the statistics tensor and the launch still fills the SMs once
		if (!XF && AMODE != OP_MN2D && BMODE == OP_K2D && p.splits == 1 && p.grid_taps == 1 && p.rowmap.mode == 0 && !p.accumulate && r.max_rows >= 4)
		{
			int gx = num_sms() / tiles_n;
			gx = gx < 1 ? 1 : gx;
			gx = gx < r.max_rows / 4 ? gx : r.max_rows / 4;
			gx = gx < tiles_m ? gx : tiles_m;
			const cudaError_t e = cudaMemsetAsync(r.part, 0, (size_t)gx * 4 * p.N * sizeof(float), stream); // the count plane
			if (e != cudaSuccess)
			{
				set_last_error("memset(conv stats)", e);
				return -1;
			}
			grid.x = gx;
			q.stats = r.part, q.stats_rows = gx * 4;
			*r.rows_out = gx * 4;
		}
	}
	const long long sms = num_sms(), columns = (long long)grid.y * grid.z, ctas = tiles_m * columns;
	if (!q.stats && p.splits == 1 && p.grid_taps == 1 && ctas > sms)
	{
		// more tiles than one wave of one CTA per SM: gx CTAs per column walk the M tiles, so the producer loads the next tile while the
		// consumers store this one.  Taken only when it costs no more rounds of tiles than one tile per CTA does.  Not for split-K or
		// per-tap launches (the weight gradients): their few M tiles share one large B slice per column, which side-by-side CTAs read
		// from L2 once and walking CTAs read again from HBM (walked, ResNet-50's 1x1 weight gradients ran 12-19 % slower on an H100)
		long long gx = sms / columns;
		gx = gx < 1 ? 1 : (gx > tiles_m ? tiles_m : gx);
		if ((gx * columns + sms - 1) / sms * ((tiles_m + gx - 1) / gx) <= (ctas + sms - 1) / sms)
			grid.x = (unsigned)gx;
	}
	kern<<<grid, GEMM_THREADS, S::TOTAL, stream>>>(tmA, tmB, q);
	count_launch();
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		set_last_error("umma_gemm_kernel launch", e);
		return -1;
	}
	return 0;
}

// output tile width: 64 columns for narrow outputs, else 128 (wgmma m64n128 per consumer warpgroup: 64 fp32 accumulator registers)
static int pick_bn(int N)
{
	const char* e = getenv("CCV_NNC_SM100_BN");
	int bn = e ? atoi(e) : (N <= 64 ? 64 : 128);
	return bn == 64 ? 64 : 128;
}

static void init_params(UmmaGemmParams& p)
{
	memset(&p, 0, sizeof(p));
	p.splits = 1;
	p.grid_taps = 1;
	p.stride_h = p.stride_w = 1;
	p.P = p.Q = 1;
}

static int pick_splits(long long tiles, int k_iters, int min_iters_per_split)
{
	// Split-K factor against wave quantisation.  Model: `tiles * s` work items of size 1 / s run in rounds of one per SM, so the
	// launch costs ceil(tiles * s / SMs) / s tile-times.  5 tiles -> s = 59 (295 CTAs, one wave of 2 CTAs per SM; s = 60 would
	// spill 4 CTAs into a second wave and double the time); 196 tiles (7 x 7 layers, N = 512)
	// -> s = 3 (588 items, 3.97 rounds of thirds instead of 2 rounds of which the second is 1/3 full).  When the tiles already fill
	// the machine a split is only taken if it buys more than 20 % (partial tiles cost a zero-fill, red.add traffic and the fused
	// batch-norm statistics of the epilogue), never finer than `min_iters_per_split`.
	const long long sms = num_sms();
	long long max_s = k_iters / min_iters_per_split;
	if (max_s < 1)
		max_s = 1;
	if (tiles >= 4 * sms || max_s == 1)
		return 1;
	if (tiles < sms)
	{
		// fewer tiles than SMs: one wave of two co-resident CTAs per SM (the one-tile kernels overlap each other's epilogue)
		long long k = 2 * sms / (tiles > 0 ? tiles : 1);
		if (k > max_s)
			k = max_s;
		while (k > 1 && (long long)((k_iters + k - 1) / k) * (k - 1) >= k_iters)
			k--;
		return (int)(k < 1 ? 1 : k);
	}
	long long limit = 2 * sms / (tiles > 0 ? tiles : 1);
	if (limit < 4)
		limit = 4;
	if (limit > max_s)
		limit = max_s;
	double best_cost = 1e30;
	for (long long k = 1; k <= limit; k++)
	{
		const double cost = (double)((tiles * k + sms - 1) / sms) / (double)k;
		if (cost < best_cost)
			best_cost = cost;
	}
	const double unsplit = (double)((tiles + sms - 1) / sms);
	if (tiles >= sms && best_cost > unsplit * 0.8)
		return 1;
	for (long long k = 1; k <= limit; k++)
	{
		const double cost = (double)((tiles * k + sms - 1) / sms) / (double)k;
		if (cost <= best_cost * 1.05)
		{
			// no empty splits: per = ceil(k_iters / k) must leave the last split non-empty
			while (k > 1 && (long long)((k_iters + k - 1) / k) * (k - 1) >= k_iters)
				k--;
			return (int)k;
		}
	}
	return 1;
}

// launches the kernel family for (AMODE, BMODE); when p.splits > 1 the partial tiles land in scratch slices [rows, cols] (pitch
// ldp) that are then added into `out` in split order
// ------------------------------------------------------------------------------------------------ element kinds
// Every contraction below exists for three element kinds: 0 = fp32 (kind::tf32 or 3xTF32), 1 = bf16, 2 = fp16 (kind::f16, fp32
// accumulate).  The kind only changes how many elements a 128-byte operand row holds, the tensor-map data type, the
// instruction / MN-major descriptors and the epilogue's output conversion; tiling, split-K and the launch logic are shared.
static inline int kind_bk(int kind) { return kind ? 64 : UMMA_BLOCK_K; }
static inline size_t kind_esz(int kind) { return kind ? 2 : 4; }
static inline int kind_align(int kind) { return kind ? 8 : 4; } // elements per 16 bytes: what TMA asks of every stride
// 2-D row-major [rows, cols] (pitch ld): box = one 128-byte span of columns x box_rows
static bool map_2d(CUtensorMap* map, int kind, const void* ptr, long long rows, long long cols, long long ld, int box_rows, bool mn_major)
{
	if (kind == 0)
		return make_map_2d(map, (const float*)ptr, rows, cols, ld, 32, box_rows, mn_major);
	return make_map_2d16(map, ptr, kind, rows, cols, ld, 64, box_rows);
}
static bool map_im2col(CUtensorMap* map, int kind, const void* ptr, int N, int H, int W, int C, long long sn, long long sh, long long sw, int lower_h, int lower_w, int upper_h, int upper_w, int trav_h, int trav_w, int pixels, bool mn_major)
{
	if (kind == 0)
		return make_map_im2col(map, (const float*)ptr, N, H, W, C, sn, sh, sw, lower_h, lower_w, upper_h, upper_w, trav_h, trav_w, 32, pixels, mn_major);
	return make_map_im2col16(map, ptr, kind, N, H, W, C, sn, sh, sw, lower_h, lower_w, upper_h, upper_w, trav_h, trav_w, 64, pixels);
}
static void init_params_kind(UmmaGemmParams& p, int kind)
{
	init_params(p);
	if (kind)
	{
		// 16-bit operands: 64 elements per 128-byte row, K = 16 per MMA
		p.kind16 = 1;
		p.out_kind = kind;
	}
}
// kernel per kind: fp32 as TF32 or 3xTF32 (t_x3); bf16 / fp16 (one kernel per element type) with a 16-bit output (out16) or fp32
// split-K slices.  launch_kind16 covers the 16-bit kinds only, for operand modes that fp32 operands never take.
template <int AMODE, int BMODE>
static int launch_kind16(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const UmmaGemmParams& p, int bn, int kind, bool out16)
{
	if (kind == 1)
	{
		if (out16)
			return bn == 64 ? launch_umma<AMODE, BMODE, 64, 0, 1, 1>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128, 0, 1, 1>(stream, tmA, tmB, p);
		return bn == 64 ? launch_umma<AMODE, BMODE, 64, 0, 1, 0>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128, 0, 1, 0>(stream, tmA, tmB, p);
	}
	if (out16)
		return bn == 64 ? launch_umma<AMODE, BMODE, 64, 0, 2, 1>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128, 0, 2, 1>(stream, tmA, tmB, p);
	return bn == 64 ? launch_umma<AMODE, BMODE, 64, 0, 2, 0>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128, 0, 2, 0>(stream, tmA, tmB, p);
}
template <int AMODE, int BMODE>
static int launch_kind(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, const UmmaGemmParams& p, int bn, int kind, bool out16)
{
	if (kind == 0)
	{
		if (t_x3)
			return bn == 64 ? launch_umma<AMODE, BMODE, 64, 1>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128, 1>(stream, tmA, tmB, p);
		return bn == 64 ? launch_umma<AMODE, BMODE, 64>(stream, tmA, tmB, p) : launch_umma<AMODE, BMODE, 128>(stream, tmA, tmB, p);
	}
	return launch_kind16<AMODE, BMODE>(stream, tmA, tmB, p, bn, kind, out16);
}

// Launch with the split factor already chosen in p.splits.  One split: straight into `out` (pitch ldo, element kind `kind`).
// Several: fp32 slices [rows, ldp] in the scratch, one per split, then the ordered combine into `out` (which also applies
// CCV_NNC_ACCUMULATE_OUTPUT and rounds once for 16-bit outputs).
template <int AMODE, int BMODE>
static int launch_umma_split(cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB, UmmaGemmParams& p, int bn, int kind, const Scratch& scratch, int rows, int cols, void* out, long long ldo, int accumulate)
{
	if (p.splits <= 1)
	{
		p.splits = 1, p.split_out_stride = 0, p.accumulate = accumulate;
		p.out = (float*)out;
		return launch_kind<AMODE, BMODE>(stream, tmA, tmB, p, bn, kind, kind != 0);
	}
	// slices are dense [rows, cols] tiles of pitch cols rounded up to 4 floats (for a filter gradient cols = R * S * C is already
	// a multiple of 4, so a slice has dW's own layout and tap-as-grid-dimension launches address it unchanged)
	const long long slice_ld = ((long long)cols + 3) & ~3ll;
	p.out = (float*)scratch.ptr;
	p.rowmap.mode = 0, p.rowmap.ld = slice_ld;
	p.split_out_stride = (long long)rows * slice_ld;
	p.accumulate = 0;
	p.bias16 = 0; // a 16-bit bias is only read by the 16-bit epilogue: callers do not split when they pass one
	const int rc = launch_kind<AMODE, BMODE>(stream, tmA, tmB, p, bn, kind, false);
	if (rc)
		return rc;
	return splitk_reduce(stream, (const float*)scratch.ptr, p.splits, p.split_out_stride, rows, cols, slice_ld, (float*)out, ldo, accumulate, kind);
}
static inline size_t slice_bytes(long long rows, long long cols)
{
	return (size_t)rows * (size_t)((cols + 3) & ~3ll) * sizeof(float);
}

// C[M, N] (+)= op(A) * op(B) + bias for element kind `kind` (bias: fp32 `bias`, or for 16-bit kinds `bias16` in the element type)
static int gemm_any(cudaStream_t stream, int kind, int M, int N, int K, const void* a, long long lda, int trans_a, const void* b, long long ldb, int trans_b, void* c, long long ldc, const float* bias, const void* bias16, int accumulate, const Scratch& scratch, int x3)
{
	const X3Scope math(kind == 0 ? x3 : 0);
	if (!tma_api_init() || M <= 0 || N <= 0 || K <= 0)
		return 1;
	const int bn = pick_bn(N), bk = kind_bk(kind);
	CUtensorMap tmA, tmB;
	bool ok;
	if (!trans_a)
		ok = map_2d(&tmA, kind, a, M, K, lda, UMMA_BLOCK_M, false);
	else
		ok = map_2d(&tmA, kind, a, K, M, lda, bk, true);
	if (!ok)
		return 1;
	if (trans_b) // stored [N, K]: K-major
		ok = map_2d(&tmB, kind, b, N, K, ldb, bn, false);
	else // stored [K, N]: N contiguous
		ok = map_2d(&tmB, kind, b, K, N, ldb, bk, true);
	if (!ok)
		return 1;
	UmmaGemmParams p;
	init_params_kind(p, kind);
	p.M = M, p.N = N;
	p.k_iters = (K + bk - 1) / bk;
	p.chunks_per_tap = p.k_iters;
	p.bias = bias, p.bias16 = bias ? 0 : bias16;
	p.rowmap.mode = 0, p.rowmap.ld = ldc;
	const long long tiles = (long long)((M + 127) / 128) * ((N + bn - 1) / bn);
	p.splits = p.bias16 ? 1 : fit_splits(pick_splits(tiles, p.k_iters, 8), p.k_iters, slice_bytes(M, N), scratch);
	if (!trans_a && trans_b)
		return launch_umma_split<OP_K2D, OP_K2D>(stream, tmA, tmB, p, bn, kind, scratch, M, N, c, ldc, accumulate);
	if (!trans_a && !trans_b)
		return launch_umma_split<OP_K2D, OP_MN2D>(stream, tmA, tmB, p, bn, kind, scratch, M, N, c, ldc, accumulate);
	if (trans_a && trans_b)
		return launch_umma_split<OP_MN2D, OP_K2D>(stream, tmA, tmB, p, bn, kind, scratch, M, N, c, ldc, accumulate);
	return launch_umma_split<OP_MN2D, OP_MN2D>(stream, tmA, tmB, p, bn, kind, scratch, M, N, c, ldc, accumulate);
}
int gemm_tf32(cudaStream_t stream, int M, int N, int K, const float* a, long long lda, int trans_a, const float* b, long long ldb, int trans_b, float* c, long long ldc, const float* bias, int accumulate, const Scratch& scratch, int x3)
{
	return gemm_any(stream, 0, M, N, K, a, lda, trans_a, b, ldb, trans_b, c, ldc, bias, 0, accumulate, scratch, x3);
}
int gemm_16(cudaStream_t stream, int kind, int M, int N, int K, const void* a, long long lda, int trans_a, const void* b, long long ldb, int trans_b, void* c, long long ldc, const float* bias32, const void* bias16, int accumulate, const Scratch& scratch)
{
	if (kind != 1 && kind != 2)
		return 1;
	return gemm_any(stream, kind, M, N, K, a, lda, trans_a, b, ldb, trans_b, c, ldc, bias32, bias16, accumulate, scratch, 0);
}

static bool conv_is_pointwise(const ConvGeom& g)
{
	return g.R == 1 && g.S == 1 && g.stride_h == 1 && g.stride_w == 1 && g.pad_h0 == 0 && g.pad_h1 == 0 && g.pad_w0 == 0 && g.pad_w1 == 0 &&
		g.aw == g.C && g.ah == (long long)g.W * g.C && g.an == (long long)g.H * g.W * g.C && g.bw == g.K && g.bh == (long long)g.Q * g.K && g.bn == (long long)g.P * g.Q * g.K;
}

static bool conv_out_contiguous(const ConvGeom& g)
{
	return g.bw == g.K && g.bh == (long long)g.Q * g.K && g.bn == (long long)g.P * g.Q * g.K;
}

static bool conv_in_contiguous(const ConvGeom& g)
{
	return g.aw == g.C && g.ah == (long long)g.W * g.C && g.an == (long long)g.H * g.W * g.C;
}

static bool conv_shape_consistent(const ConvGeom& g)
{
	const int eff_r = (g.R - 1) * g.dil_h + 1, eff_s = (g.S - 1) * g.dil_w + 1;
	return (g.H + g.pad_h0 + g.pad_h1 - eff_r) / g.stride_h + 1 == g.P && (g.W + g.pad_w0 + g.pad_w1 - eff_s) / g.stride_w + 1 == g.Q &&
		g.R * g.S <= UMMA_MAX_TAPS && g.C % 4 == 0 && g.K % 4 == 0;
}

static int conv_fprop_any(cudaStream_t stream, int kind, const ConvGeom& g, const void* a, const void* w, const float* bias, const void* bias16, void* b, const Scratch& scratch, int x3)
{
	const X3Scope math(kind == 0 ? x3 : 0);
	if (!tma_api_init() || !conv_shape_consistent(g) || !conv_out_contiguous(g) || g.C % kind_align(kind) || g.K % kind_align(kind))
		return 1;
	const long long M = (long long)g.N * g.P * g.Q;
	if (M > 0x7fffffffll)
		return 1;
	if (conv_is_pointwise(g)) // a plain [NHW, C] x [K, C]^T GEMM
		return gemm_any(stream, kind, (int)M, g.K, g.C, a, g.C, 0, w, g.C, 1, b, g.K, bias, bias16, 0, scratch, x3);
	const int bn = pick_bn(g.K), bk = kind_bk(kind);
	CUtensorMap tmA, tmB;
	if (!map_im2col(&tmA, kind, a, g.N, g.H, g.W, g.C, g.an, g.ah, g.aw, -g.pad_h0, -g.pad_w0, g.pad_h1 - (g.R - 1) * g.dil_h, g.pad_w1 - (g.S - 1) * g.dil_w, g.stride_h, g.stride_w, UMMA_BLOCK_M, false))
		return 1;
	const long long rsc = (long long)g.R * g.S * g.C;
	if (!map_2d(&tmB, kind, w, g.K, rsc, rsc, bn, false))
		return 1;
	UmmaGemmParams p;
	init_params_kind(p, kind);
	p.M = (int)M, p.N = g.K;
	// a tap's channels are walked in spans of bk; a last span that runs past C reads zeros from the input (TMA bounds) and the
	// next tap's filter columns from w, whose products with those zeros vanish
	p.chunks_per_tap = (g.C + bk - 1) / bk;
	p.k_iters = g.R * g.S * p.chunks_per_tap;
	p.P = g.P, p.Q = g.Q;
	p.stride_h = g.stride_h, p.stride_w = g.stride_w;
	p.base_h = -g.pad_h0, p.base_w = -g.pad_w0;
	for (int r = 0; r < g.R; r++)
		for (int s = 0; s < g.S; s++)
		{
			const int t = r * g.S + s;
			p.tap_off_h[t] = (unsigned short)(r * g.dil_h);
			p.tap_off_w[t] = (unsigned short)(s * g.dil_w);
			p.tap_b_col[t] = t * g.C;
		}
	p.out = (float*)b, p.bias = bias, p.bias16 = bias ? 0 : bias16;
	p.rowmap.mode = 0, p.rowmap.ld = g.K;
	return launch_kind<OP_IM2COL, OP_K2D>(stream, tmA, tmB, p, bn, kind, kind != 0);
}
int conv_fprop_tf32(cudaStream_t stream, const ConvGeom& g, const float* a, const float* w, const float* bias, float* b, const Scratch& scratch, int x3)
{
	return conv_fprop_any(stream, 0, g, a, w, bias, 0, b, scratch, x3);
}
int conv_fprop_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* a, const void* w, const float* bias32, const void* bias16, void* b, const Scratch& scratch)
{
	return kind == 1 || kind == 2 ? conv_fprop_any(stream, kind, g, a, w, bias32, bias16, b, scratch, 0) : 1;
}

// The data gradient reads the filters w[K, R*S*C] as its B operand with k = the output channel.  wgmma reads TF32 operands K-major
// only, so fp32 filters are first copied to wt[R*S*C, K] ([tap][c][k], the head of the workspace) and taken as a K-major B: the
// kernel runs without the transform step, and its products see the same TF32-rounded values in the same k order.  16-bit filters
// are read in place as an MN-major B (the wgmma descriptor transposes 16-bit tiles).
static size_t dgrad_filter_copy_bytes(const ConvGeom& g)
{
	return ((size_t)g.K * g.R * g.S * g.C * sizeof(float) + 511) & ~(size_t)511;
}
size_t conv_dgrad_workspace_bytes(const ConvGeom& g)
{
	return dgrad_filter_copy_bytes(g) + CONTRACT_SCRATCH_BYTES;
}

// wt: room for the fp32 filter copy (kind 0; NULL for 16-bit kinds)
static int conv_dgrad_any(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* w, float* wt, void* grad_a, const Scratch& scratch, int x3)
{
	const X3Scope math(kind == 0 ? x3 : 0);
	const long long rsc = (long long)g.R * g.S * g.C;
	if (!tma_api_init() || !conv_shape_consistent(g) || !conv_out_contiguous(g) || !conv_in_contiguous(g) || g.C % kind_align(kind) || g.K % kind_align(kind) || g.K * rsc > 0x7fffffffll)
		return 1;
	if (kind == 0)
	{
		const int dim[4] = { 1, 1, g.K, (int)rsc }, w_stride[4] = { 0, 0, (int)rsc, 1 }, wt_stride[4] = { 0, 0, 1, g.K };
		if (copy_strided(stream, w, w_stride, wt, wt_stride, dim, 4))
			return -1;
	}
	if (conv_is_pointwise(g)) // dA[NHW, C] = dB[NHW, K] x W[K, C]
	{
		if (kind == 0)
			return gemm_any(stream, kind, g.N * g.H * g.W, g.C, g.K, grad_b, g.K, 0, wt, g.K, 1, grad_a, g.C, 0, 0, 0, scratch, x3);
		return gemm_any(stream, kind, g.N * g.H * g.W, g.C, g.K, grad_b, g.K, 0, w, g.C, 0, grad_a, g.C, 0, 0, 0, scratch, x3);
	}
	const int bn = pick_bn(g.C), bk = kind_bk(kind);
	const size_t esz = kind_esz(kind);
	CUtensorMap tmB;
	if (kind == 0 ? !map_2d(&tmB, kind, wt, rsc, g.K, g.K, bn, false) : !map_2d(&tmB, kind, w, g.K, rsc, rsc, bk, true))
		return 1;
	// Decompose by output-pixel residue class (ah, aw) modulo the stride: within a class, pixel h = i * stride + ah
	// receives from filter row r iff (ah + pad - r * dil) % stride == 0, reading grad_b row i + (ah + pad - r * dil) / stride.
	bool need_zero = false;
	struct ClassPlan {
		int ntaps_h, ntaps_w;
		int e_h[UMMA_MAX_TAPS], r_h[UMMA_MAX_TAPS], e_w[UMMA_MAX_TAPS], s_w[UMMA_MAX_TAPS];
	};
	for (int ah = 0; ah < g.stride_h; ah++)
		for (int aw = 0; aw < g.stride_w; aw++)
		{
			ClassPlan cp;
			cp.ntaps_h = cp.ntaps_w = 0;
			for (int r = 0; r < g.R; r++)
			{
				const int num = ah + g.pad_h0 - r * g.dil_h;
				if (((num % g.stride_h) + g.stride_h) % g.stride_h == 0)
					cp.e_h[cp.ntaps_h] = (num >= 0 ? num / g.stride_h : -((-num) / g.stride_h)), cp.r_h[cp.ntaps_h++] = r;
			}
			for (int s = 0; s < g.S; s++)
			{
				const int num = aw + g.pad_w0 - s * g.dil_w;
				if (((num % g.stride_w) + g.stride_w) % g.stride_w == 0)
					cp.e_w[cp.ntaps_w] = (num >= 0 ? num / g.stride_w : -((-num) / g.stride_w)), cp.s_w[cp.ntaps_w++] = s;
			}
			const int Hc = (g.H - ah + g.stride_h - 1) / g.stride_h, Wc = (g.W - aw + g.stride_w - 1) / g.stride_w;
			if (Hc <= 0 || Wc <= 0)
				continue;
			if (cp.ntaps_h == 0 || cp.ntaps_w == 0)
			{
				need_zero = true;
				continue;
			}
		}
	if (need_zero)
	{
		cudaError_t e = cudaMemsetAsync(grad_a, 0, (size_t)g.N * g.H * g.W * g.C * esz, stream);
		if (e != cudaSuccess)
		{
			set_last_error("memset(dgrad)", e);
			return -1;
		}
	}
	for (int ah = 0; ah < g.stride_h; ah++)
		for (int aw = 0; aw < g.stride_w; aw++)
		{
			ClassPlan cp;
			cp.ntaps_h = cp.ntaps_w = 0;
			int lo_h = 1 << 30, lo_w = 1 << 30;
			for (int r = 0; r < g.R; r++)
			{
				const int num = ah + g.pad_h0 - r * g.dil_h;
				if (((num % g.stride_h) + g.stride_h) % g.stride_h == 0)
				{
					const int e = num >= 0 ? num / g.stride_h : -((-num) / g.stride_h);
					cp.e_h[cp.ntaps_h] = e, cp.r_h[cp.ntaps_h++] = r;
					if (e < lo_h)
						lo_h = e;
				}
			}
			for (int s = 0; s < g.S; s++)
			{
				const int num = aw + g.pad_w0 - s * g.dil_w;
				if (((num % g.stride_w) + g.stride_w) % g.stride_w == 0)
				{
					const int e = num >= 0 ? num / g.stride_w : -((-num) / g.stride_w);
					cp.e_w[cp.ntaps_w] = e, cp.s_w[cp.ntaps_w++] = s;
					if (e < lo_w)
						lo_w = e;
				}
			}
			const int Hc = (g.H - ah + g.stride_h - 1) / g.stride_h, Wc = (g.W - aw + g.stride_w - 1) / g.stride_w;
			if (Hc <= 0 || Wc <= 0 || cp.ntaps_h == 0 || cp.ntaps_w == 0)
				continue;
			CUtensorMap tmA;
			// base pixels i in [0, Hc) map to grad_b rows i + lo_h + offset: bounding box [lo_h, P + (Hc - P + lo_h))
			if (!map_im2col(&tmA, kind, grad_b, g.N, g.P, g.Q, g.K, g.bn, g.bh, g.bw, lo_h, lo_w, Hc - g.P + lo_h, Wc - g.Q + lo_w, 1, 1, UMMA_BLOCK_M, false))
				return 1;
			UmmaGemmParams p;
			init_params_kind(p, kind);
			p.M = g.N * Hc * Wc, p.N = g.C;
			p.chunks_per_tap = (g.K + bk - 1) / bk;
			p.k_iters = cp.ntaps_h * cp.ntaps_w * p.chunks_per_tap;
			p.P = Hc, p.Q = Wc;
			p.base_h = lo_h, p.base_w = lo_w;
			for (int i = 0; i < cp.ntaps_h; i++)
				for (int j = 0; j < cp.ntaps_w; j++)
				{
					const int t = i * cp.ntaps_w + j;
					p.tap_off_h[t] = (unsigned short)(cp.e_h[i] - lo_h);
					p.tap_off_w[t] = (unsigned short)(cp.e_w[j] - lo_w);
					(kind == 0 ? p.tap_b_row : p.tap_b_col)[t] = (cp.r_h[i] * g.S + cp.s_w[j]) * g.C;
				}
			p.out = (float*)((char*)grad_a + ((long long)ah * g.W + aw) * g.C * esz);
			p.rowmap.mode = 1;
			p.rowmap.Pc = Hc, p.rowmap.Qc = Wc;
			p.rowmap.n_stride = (long long)g.H * g.W * g.C;
			p.rowmap.h_stride = (long long)g.stride_h * g.W * g.C;
			p.rowmap.w_stride = (long long)g.stride_w * g.C;
			const int rc = kind == 0 ? launch_kind<OP_IM2COL, OP_K2D>(stream, tmA, tmB, p, bn, kind, false) : launch_kind16<OP_IM2COL, OP_MN2D>(stream, tmA, tmB, p, bn, kind, true);
			if (rc)
				return rc;
		}
	return 0;
}
int conv_dgrad_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* w, float* grad_a, void* workspace, int x3)
{
	const Scratch scratch = { (char*)workspace + dgrad_filter_copy_bytes(g), CONTRACT_SCRATCH_BYTES };
	return conv_dgrad_any(stream, 0, g, grad_b, w, (float*)workspace, grad_a, scratch, x3);
}
int conv_dgrad_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* w, void* grad_a, const Scratch& scratch)
{
	return kind == 1 || kind == 2 ? conv_dgrad_any(stream, kind, g, grad_b, w, 0, grad_a, scratch, 0) : 1;
}

static int conv_wgrad_any(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* a, void* grad_w, int accumulate, const Scratch& scratch, int x3)
{
	const X3Scope math(kind == 0 ? x3 : 0);
	if (!tma_api_init() || !conv_shape_consistent(g) || !conv_out_contiguous(g) || g.C % kind_align(kind) || g.K % kind_align(kind))
		return 1;
	const int bk = kind_bk(kind);
	const long long npq = (long long)g.N * g.P * g.Q;
	if (npq > 0x7fffffffll)
		return 1;
	const int bn = pick_bn(g.C);
	const long long rsc = (long long)g.R * g.S * g.C;
	CUtensorMap tmA, tmB;
	// A = grad_b^T: [K, NPQ] read from the [NPQ, K] tensor as an MN-major operand
	if (!map_2d(&tmA, kind, grad_b, npq, g.K, g.K, bk, true))
		return 1;
	UmmaGemmParams p;
	init_params_kind(p, kind);
	p.M = g.K, p.N = g.C;
	p.k_iters = (int)((npq + bk - 1) / bk);
	p.chunks_per_tap = p.k_iters;
	p.rowmap.mode = 0, p.rowmap.ld = rsc;
	const long long tiles = (long long)((g.K + 127) / 128) * ((g.C + bn - 1) / bn) * g.R * g.S;
	// split-K slices have the layout of dW itself ([K, RSC]); splitk_reduce adds them (and the old dW when accumulating)
	const size_t dw_bytes = (size_t)g.K * rsc * sizeof(float);
	p.splits = fit_splits(pick_splits(tiles, p.k_iters, 16), p.k_iters, dw_bytes, scratch);
	if (conv_is_pointwise(g))
	{
		// B = a: [NHW, C], also MN-major
		if (!map_2d(&tmB, kind, a, npq, g.C, g.C, bk, true))
			return 1;
		return launch_umma_split<OP_MN2D, OP_MN2D>(stream, tmA, tmB, p, bn, kind, scratch, g.K, (int)rsc, grad_w, rsc, accumulate);
	}
	if (!map_im2col(&tmB, kind, a, g.N, g.H, g.W, g.C, g.an, g.ah, g.aw, -g.pad_h0, -g.pad_w0, g.pad_h1 - (g.R - 1) * g.dil_h, g.pad_w1 - (g.S - 1) * g.dil_w, g.stride_h, g.stride_w, bk, true))
		return 1;
	p.grid_taps = g.R * g.S;
	p.grid_tap_out_stride = g.C;
	p.P = g.P, p.Q = g.Q;
	p.stride_h = g.stride_h, p.stride_w = g.stride_w;
	p.base_h = -g.pad_h0, p.base_w = -g.pad_w0;
	for (int r = 0; r < g.R; r++)
		for (int s = 0; s < g.S; s++)
		{
			const int t = r * g.S + s;
			p.tap_off_h[t] = (unsigned short)(r * g.dil_h);
			p.tap_off_w[t] = (unsigned short)(s * g.dil_w);
		}
	return launch_umma_split<OP_MN2D, OP_IM2COL>(stream, tmA, tmB, p, bn, kind, scratch, g.K, (int)rsc, grad_w, rsc, accumulate);
}
int conv_wgrad_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* a, float* grad_w, int accumulate, const Scratch& scratch, int x3)
{
	return conv_wgrad_any(stream, 0, g, grad_b, a, grad_w, accumulate, scratch, x3);
}
int conv_wgrad_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* a, void* grad_w, int accumulate, const Scratch& scratch)
{
	return kind == 1 || kind == 2 ? conv_wgrad_any(stream, kind, g, grad_b, a, grad_w, accumulate, scratch, 0) : 1;
}

// ------------------------------------------------------------------------------------------------ explicit im2col
// Small-channel convolutions whose pixels TMA cannot address (C * element size not a multiple of 16 bytes: the 3-channel stem):
// patches [N*P*Q, Kp] with Kp = R*S*C rounded up to one operand span (32 fp32 / 64 16-bit elements, zero padded), then the GEMM.
static inline int im2col_kp(const ConvGeom& g, int kind) { const int span = kind_bk(kind); return (g.R * g.S * g.C + span - 1) / span * span; }
static inline bool im2col_applicable(const ConvGeom& g, int kind)
{
	return g.R * g.S * g.C <= 256 && (long long)g.N * g.P * g.Q <= 0x7fffffffll && g.K % kind_align(kind) == 0 && g.bw == g.K && g.bh == (long long)g.Q * g.K && g.bn == (long long)g.P * g.Q * g.K;
}
static size_t im2col_used_bytes(const ConvGeom& g, int kind)
{
	const size_t kp = im2col_kp(g, kind);
	// patches [NPQ, Kp] + packed filters [K, Kp] + packed filter gradient [K, Kp]
	return ((((size_t)g.N * g.P * g.Q * kp + 2 * (size_t)g.K * kp) * kind_esz(kind)) + 511) & ~(size_t)511;
}
size_t conv_im2col_workspace_bytes(const ConvGeom& g, int kind)
{
	return im2col_used_bytes(g, kind) + 512 + CONTRACT_SCRATCH_BYTES;
}
static Scratch im2col_scratch(const ConvGeom& g, int kind, void* workspace)
{
	Scratch s = { (char*)workspace + im2col_used_bytes(g, kind), CONTRACT_SCRATCH_BYTES };
	return s;
}
// patches[m, (r, s, c)] = a[n, p * stride - pad + r * dil, q * stride - pad + s * dil, c] (0 outside / in the padding columns)
// One thread = 4 consecutive k of one patch row (one 16- or 8-byte store); k -> (tap row offset, tap column offset, channel)
// comes from a table in shared memory, all index math is 32-bit.
template <typename T>
__global__ void __launch_bounds__(256) im2col_kernel(const ConvGeom g, const T* __restrict__ a, T* __restrict__ out, const int kp, const unsigned rows)
{
	__shared__ int tab_h[256], tab_w[256], tab_c[256];
	const int rsc = g.R * g.S * g.C;
	for (int k = threadIdx.x; k < kp; k += blockDim.x)
	{
		const int c = k % g.C, t = k / g.C;
		tab_h[k] = k < rsc ? (t / g.S) * g.dil_h - g.pad_h0 : -(1 << 28);
		tab_w[k] = k < rsc ? (t % g.S) * g.dil_w - g.pad_w0 : -(1 << 28);
		tab_c[k] = c;
	}
	__syncthreads();
	const unsigned kq = (unsigned)kp >> 2;
	const unsigned long long total = (unsigned long long)rows * kq;
	for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x)
	{
		const unsigned m = (unsigned)(i / kq), k0 = ((unsigned)(i - (unsigned long long)m * kq)) << 2;
		const unsigned q = m % (unsigned)g.Q, u = m / (unsigned)g.Q;
		const unsigned pp = u % (unsigned)g.P, n = u / (unsigned)g.P;
		const int h0 = (int)pp * g.stride_h, w0 = (int)q * g.stride_w;
		const T* const an = a + (long long)n * g.an;
		float v[4];
#pragma unroll
		for (int j = 0; j < 4; j++)
		{
			const int h = h0 + tab_h[k0 + j], w = w0 + tab_w[k0 + j];
			v[j] = (h >= 0 && h < g.H && w >= 0 && w < g.W) ? ldf(an + h * g.ah + w * g.aw + tab_c[k0 + j]) : 0.f;
		}
		st4(out + (unsigned long long)m * kp + k0, make_float4(v[0], v[1], v[2], v[3]));
	}
}
// dir 0: packed[k, 0..kp) = w[k, 0..rsc) zero padded.  dir 1: w[k, j] (+)= packed[k, j]
template <typename T>
__global__ void pack_filters_kernel(T* __restrict__ w, T* __restrict__ packed, const int K, const int rsc, const int kp, const int dir, const int accumulate)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= K * kp)
		return;
	const int k = i / kp, j = i % kp;
	if (dir == 0)
		stf(packed + i, j < rsc ? ldf(w + (size_t)k * rsc + j) : 0.f);
	else if (j < rsc)
		stf(w + (size_t)k * rsc + j, accumulate ? ldf(w + (size_t)k * rsc + j) + ldf(packed + i) : ldf(packed + i));
}
template <typename T>
static int run_im2col(cudaStream_t stream, const ConvGeom& g, const T* a, T* patches, int kp)
{
	const size_t rows = (size_t)g.N * g.P * g.Q;
	size_t blocks = (rows * (kp / 4) + 255) / 256;
	if (blocks > (size_t)num_sms() * 32)
		blocks = (size_t)num_sms() * 32;
	im2col_kernel<T><<<(unsigned)blocks, 256, 0, stream>>>(g, a, patches, kp, (unsigned)rows);
	count_launch();
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		set_last_error("im2col_kernel", e);
		return -1;
	}
	return 0;
}
template <typename T>
static int conv_fprop_im2col_t(cudaStream_t stream, const ConvGeom& g, const T* a, const T* w, const float* bias, const void* bias16, T* b, void* workspace, int x3)
{
	constexpr int kind = ElemKind<T>::value;
	if (!tma_api_init() || !im2col_applicable(g, kind) || !workspace)
		return 1;
	const int kp = im2col_kp(g, kind), rsc = g.R * g.S * g.C;
	const size_t m = (size_t)g.N * g.P * g.Q;
	T* patches = (T*)workspace;
	T* wp = patches + m * kp;
	if (run_im2col<T>(stream, g, a, patches, kp))
		return -1;
	pack_filters_kernel<T><<<(g.K * kp + 255) / 256, 256, 0, stream>>>((T*)w, wp, g.K, rsc, kp, 0, 0);
	count_launch();
	return gemm_any(stream, kind, (int)m, g.K, kp, patches, kp, 0, wp, kp, 1, b, g.K, bias, bias16, 0, im2col_scratch(g, kind, workspace), x3);
}
template <typename T>
static int conv_wgrad_im2col_t(cudaStream_t stream, const ConvGeom& g, const T* grad_b, const T* a, T* grad_w, int accumulate, void* workspace, int x3)
{
	constexpr int kind = ElemKind<T>::value;
	if (!tma_api_init() || !im2col_applicable(g, kind) || !workspace)
		return 1;
	const int kp = im2col_kp(g, kind), rsc = g.R * g.S * g.C;
	const size_t m = (size_t)g.N * g.P * g.Q;
	T* patches = (T*)workspace;
	T* dwp = patches + m * kp + (size_t)g.K * kp;
	if (run_im2col<T>(stream, g, a, patches, kp))
		return -1;
	// dWp[K, Kp] = grad_b^T [K, NPQ] * patches [NPQ, Kp]
	const int rc = gemm_any(stream, kind, g.K, kp, (int)m, grad_b, g.K, 1, patches, kp, 0, dwp, kp, 0, 0, 0, im2col_scratch(g, kind, workspace), x3);
	if (rc)
		return rc;
	pack_filters_kernel<T><<<(g.K * kp + 255) / 256, 256, 0, stream>>>(grad_w, dwp, g.K, rsc, kp, 1, accumulate);
	count_launch();
	return 0;
}
int conv_fprop_im2col_tf32(cudaStream_t stream, const ConvGeom& g, const float* a, const float* w, const float* bias, float* b, void* workspace, int x3)
{
	return conv_fprop_im2col_t<float>(stream, g, a, w, bias, 0, b, workspace, x3);
}
int conv_wgrad_im2col_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* a, float* grad_w, int accumulate, void* workspace, int x3)
{
	return conv_wgrad_im2col_t<float>(stream, g, grad_b, a, grad_w, accumulate, workspace, x3);
}
int conv_fprop_im2col_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* a, const void* w, const float* bias32, const void* bias16, void* b, void* workspace)
{
	if (kind == 1)
		return conv_fprop_im2col_t<__nv_bfloat16>(stream, g, (const __nv_bfloat16*)a, (const __nv_bfloat16*)w, bias32, bias16, (__nv_bfloat16*)b, workspace, 0);
	return conv_fprop_im2col_t<__half>(stream, g, (const __half*)a, (const __half*)w, bias32, bias16, (__half*)b, workspace, 0);
}
int conv_wgrad_im2col_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* a, void* grad_w, int accumulate, void* workspace)
{
	if (kind == 1)
		return conv_wgrad_im2col_t<__nv_bfloat16>(stream, g, (const __nv_bfloat16*)grad_b, (const __nv_bfloat16*)a, (__nv_bfloat16*)grad_w, accumulate, workspace, 0);
	return conv_wgrad_im2col_t<__half>(stream, g, (const __half*)grad_b, (const __half*)a, (__half*)grad_w, accumulate, workspace, 0);
}

} // namespace sm100
