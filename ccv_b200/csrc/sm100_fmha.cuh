// sm100_fmha.cuh -- helpers shared by the 16-bit flash-attention kernels (sm100_fmha.cu forward, sm100_fmha_bwd.cu backward):
// 16-bit packing, the 4-D TMA tensor map over a [B, S, H, D] tensor, and the register form of P / dS as a wgmma A operand; the tensor map
// and the shared-memory reads of an additive mask (sm100_fmha.cu, sm100_fmha_wide.cu under CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK).
#pragma once
#include "sm100_ptx.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <mutex>
#include <stdlib.h>

namespace sm100 {
namespace {

__device__ __forceinline__ uint32_t pack2(const float a, const float b, const int is_bf16)
{
	if (is_bf16)
	{
		const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
		return *reinterpret_cast<const uint32_t*>(&v);
	}
	const __half2 v = __floats2half2_rn(a, b);
	return *reinterpret_cast<const uint32_t*>(&v);
}

__device__ __forceinline__ float widen16(const uint16_t u, const int is_bf16)
{
	return is_bf16 ? __uint_as_float((uint32_t)u << 16) : __half2float(__ushort_as_half(u));
}

// the m16n8k16 A fragment of 16 key columns [16 kk, 16 kk + 16) of a wgmma accumulator (see sm100_ptx.cuh), rounded to 16 bits
template <int R>
__device__ __forceinline__ void acc_to_a(const float (&x)[R], const int kk, const int is_bf16, uint32_t (&a)[4])
{
	a[0] = pack2(x[8 * kk], x[8 * kk + 1], is_bf16), a[1] = pack2(x[8 * kk + 2], x[8 * kk + 3], is_bf16);
	a[2] = pack2(x[8 * kk + 4], x[8 * kk + 5], is_bf16), a[3] = pack2(x[8 * kk + 6], x[8 * kk + 7], is_bf16);
}

typedef CUresult (*encode_tiled_f)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline encode_tiled_f& encode_fn()
{
	static encode_tiled_f fn = 0;
	return fn;
}

inline bool encode_init()
{
	static std::once_flag once;
	std::call_once(once, []() {
		void* fn = 0;
		cudaDriverEntryPointQueryResult qres;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
			encode_fn() = (encode_tiled_f)fn;
	});
	return encode_fn() != 0;
}

// 16-bit [B, S, H, D] tensor with element strides (sb, ss, sh), D contiguous: box = {64 d, 1 head, box_rows rows, 1 batch}
inline bool make_map_bshd(CUtensorMap* map, const void* ptr, int B, int S, int H, int D, long long sb, long long ss, long long sh, int is_bf16, int box_rows)
{
	if ((((uintptr_t)ptr) & 15) || ((sb * 2) & 15) || ((ss * 2) & 15) || ((sh * 2) & 15))
		return false;
	// a stride of 0 is not encodable; extents of 1 never advance, any positive multiple of 16 bytes will do
	if (H == 1 && sh <= 0)
		sh = D;
	if (B == 1 && sb <= 0)
		sb = (long long)S * ss;
	cuuint64_t dims[4] = { (cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)S, (cuuint64_t)B };
	cuuint64_t strides[3] = { (cuuint64_t)sh * 2, (cuuint64_t)ss * 2, (cuuint64_t)sb * 2 };
	cuuint32_t box[4] = { 64, 1, (cuuint32_t)box_rows, 1 };
	cuuint32_t estr[4] = { 1, 1, 1, 1 };
	return encode_fn()(map, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Additive attention mask [B | 1, H | 1, Sq, Sk] with element strides (sb, sh, ss), 0 = broadcast, keys contiguous; esz = 4 (fp32) or 2
// (the activations' 16-bit type).  box = {128 bytes of keys, 128 query rows, 1 head, 1 batch}, 128-byte swizzle; the TMA unit zero-fills
// keys past Sk and rows past Sq, so a tile never reads outside the tensor.  false when a pitch or the base is not a multiple of 16 bytes.
inline bool make_map_mask(CUtensorMap* map, const void* ptr, int B, int H, int Sq, int Sk, long long sb, long long sh, long long ss, int esz, int is_bf16)
{
	if ((((uintptr_t)ptr) & 15) || ss <= 0 || ((ss * esz) & 15) || ((sh * esz) & 15) || ((sb * esz) & 15))
		return false;
	const int Hm = sh ? H : 1, Bm = sb ? B : 1;
	if (!sh)
		sh = (long long)Sq * ss;
	if (!sb)
		sb = (long long)Hm * sh;
	cuuint64_t dims[4] = { (cuuint64_t)Sk, (cuuint64_t)Sq, (cuuint64_t)Hm, (cuuint64_t)Bm };
	cuuint64_t strides[3] = { (cuuint64_t)(ss * esz), (cuuint64_t)(sh * esz), (cuuint64_t)(sb * esz) };
	cuuint32_t box[4] = { (cuuint32_t)(128 / esz), 128, 1, 1 };
	cuuint32_t estr[4] = { 1, 1, 1, 1 };
	const CUtensorMapDataType t = esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : (is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
	return encode_fn()(map, t, 4, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

constexpr int MASK_ATOM_BYTES = 128 * 128; // one make_map_mask box: 128 rows x 128 bytes

// mask[r][8 c + 2 t4], mask[r][8 c + 2 t4 + 1] (r < 128, t4 < 4; c a constant after unrolling) from a stage of make_map_mask boxes,
// one 16 KB atom per 128 bytes of keys, 16-byte chunks XOR-swizzled by r & 7 (the stage is 1024-byte aligned).  row = stage + 128 r,
// x = r & 7.  MASK 1 = fp32, 2 = 16-bit (widened exactly).
template <int MASK, int BF16>
__device__ __forceinline__ float2 mask_pair(const uint8_t* row, const int x, const int c, const int t4)
{
	if constexpr (MASK == 1)
		return *reinterpret_cast<const float2*>(row + (c >> 2) * MASK_ATOM_BYTES + (((2 * (c & 3) + (t4 >> 1)) ^ x) << 4) + 8 * (t4 & 1));
	else {
		const uint32_t u = *reinterpret_cast<const uint32_t*>(row + (c >> 3) * MASK_ATOM_BYTES + (((c & 7) ^ x) << 4) + 4 * t4);
		return make_float2(widen16((uint16_t)(u & 0xffff), BF16), widen16((uint16_t)(u >> 16), BF16));
	}
}

// S (a wgmma accumulator of R / 4 groups of 8 keys, rows r and r + 8) -> scale * S + mask, in CPU_REF's order; the loads four groups
// at a time.
template <int MASK, int BF16, int R>
__device__ __forceinline__ void add_mask(float (&sacc)[R], const uint8_t* stage, const int r, const int t4, const float scale)
{
#pragma unroll
	for (int c0 = 0; c0 < R / 4; c0 += 4)
	{
		float2 mk[4][2];
#pragma unroll
		for (int c = 0; c < 4; c++)
#pragma unroll
			for (int hh = 0; hh < 2; hh++)
				mk[c][hh] = mask_pair<MASK, BF16>(stage + 128 * (r + 8 * hh), r & 7, c0 + c, t4);
#pragma unroll
		for (int c = 0; c < 4; c++)
#pragma unroll
			for (int hh = 0; hh < 2; hh++)
			{
				const int i = 4 * (c0 + c) + 2 * hh;
				sacc[i] = fmaf(sacc[i], scale, mk[c][hh].x);
				sacc[i + 1] = fmaf(sacc[i + 1], scale, mk[c][hh].y);
			}
	}
}

} // namespace
} // namespace sm100
