// sm100_fmha.cuh -- helpers shared by the 16-bit flash-attention kernels (sm100_fmha.cu forward, sm100_fmha_bwd.cu backward):
// 16-bit packing, the 4-D TMA tensor map over a [B, S, H, D] tensor, and the register form of P / dS as a wgmma A operand.
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

} // namespace
} // namespace sm100
