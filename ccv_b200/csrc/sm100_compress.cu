// sm100_compress.cu -- COMPRESSION_LSSC forward (compress) and backward (decompress), fp16, NCHW and NHWC.  Semantics are CPU_REF's
// (lib/nnc/cmd/compression/ccv_nnc_lssc_cpu_ref.c of the reference; DESIGN.md §2 restates them).  Each (n, c) plane is cut into 4x4
// blocks; a block becomes 4 halves: its min, its max and two halves of 2-bit codes (cells 0-7, then 8-15, cell c at bits 2 (c mod 8)).
//   forward   cells past the bottom / right edge take the block's first cell; min / max are the `a > m ? a : m` scans from cell 0, and
//             are stored as the selected cell's own bits; abottom = min * 7 / 6 - max / 6; ascale = (float)(3.0 / max((double)(max - min),
//             1e-6)); code = clamp((int)((a - abottom) * ascale), 0, 3), truncating toward zero (a NaN product clamps to 0).
//   backward  levels min, (max / 3 + min * 2 / 3), (max * 2 / 3 + min / 3), max; the two middle ones narrowed with the reference's
//             truncating f32 -> f16 (f32_to_f16_trunc); each cell inside the original tensor gets level[code].
// Every product, quotient and sum is rounded on its own (__f*_rn; nothing here may be contracted).  Outputs are overwritten whatever
// CCV_NNC_ACCUMULATE_OUTPUT says.
//
// Shapes (the reference's _ccv_nnc_lssc_tensor_auto_forw): NCHW [N, C, H, W] / [C, H, W] <-> [N, C, ceil(H/4), 4 ceil(W/4)]; NHWC
// [N, H, W, C] / [H, W, C] <-> [N, ceil(H/4), 4 ceil(W/4), C], where compressed[n, by, 4 bx + k, c] is half k of plane (n, c)'s block
// (by, bx).  Operands are contiguous.  A call carries n (original, compressed) pairs; every pair is checked before the first launch,
// and each pair is one launch.  No workspace, no atomics.
//
// Kernel forms (all give the same bits: they share lssc_encode / lssc_decode):
//   NCHW, W <= LSSC_BAND_MAX_W     a 4-row band of a plane is one contiguous span of (rows x W) halves, and its compressed row one
//                                  contiguous span of 4 ceil(W/4) halves; consecutive bands are consecutive spans of both tensors.
//                                  A CTA owns a run of bands: it stages the run's span through shared memory with 16-byte accesses
//                                  (scalar head and tail wherever the span is not 16-byte aligned), codes every block of the run from
//                                  shared memory, and writes the other side's span the same way.  Small planes (7x7) put many bands in
//                                  one CTA.
//   NHWC, C % 8 == 0, bases 16-byte aligned
//                                  one thread per (pixel block, 8 channels): 16 16-byte loads and 4 16-byte stores forward (the
//                                  reverse backward), coalesced along C.
//   otherwise (NHWC, NCHW wider than LSSC_BAND_MAX_W)
//                                  one thread per (block, channel), the same scan on scalar accesses, channel fastest.
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

using namespace sm100;

namespace {

constexpr int LSSC_THREADS = 256;
constexpr long long LSSC_SPAN = 8192;     // halves of either side staged by one CTA of the band form (16 KB)
constexpr int LSSC_BAND_MAX_W = 2048;     // LSSC_SPAN / 4: one 4-row band fits
constexpr int LSSC_CTAS_PER_SM = 8;       // the band form spreads its bands over at least this many CTAs per SM when it can

// ------------------------------------------------------------------------------------------------ one block (CPU_REF's arithmetic)
__device__ __forceinline__ float h2f(const uint16_t h) { return __half2float(__ushort_as_half(h)); }

// h: the 16 cells in row-major order (padding already replaced by cell 0) -> q: min, max, codes of cells 0-7, codes of cells 8-15
__device__ __forceinline__ void lssc_encode(const uint16_t (&h)[16], uint16_t (&q)[4])
{
	float a[16];
#pragma unroll
	for (int c = 0; c < 16; c++)
		a[c] = h2f(h[c]);
	float amax = a[0], amin = a[0];
	uint16_t hmax = h[0], hmin = h[0];
#pragma unroll
	for (int c = 1; c < 16; c++)
	{
		// ccv_max / ccv_min: the later cell replaces the running value only when strictly greater / smaller (a NaN never does, a NaN
		// cell 0 is never replaced, and of +0 / -0 the earlier one stays)
		if (a[c] > amax)
			amax = a[c], hmax = h[c];
		if (a[c] < amin)
			amin = a[c], hmin = h[c];
	}
	const float abottom = __fsub_rn(__fdiv_rn(__fmul_rn(amin, 7.f), 6.f), __fdiv_rn(amax, 6.f));
	// ccv_max(amax - amin, 1e-6) compares and divides in double; a NaN range gives 1e-6
	const double range = (double)__fsub_rn(amax, amin);
	const float ascale = __double2float_rn(__ddiv_rn(3.0, range > 1e-6 ? range : 1e-6));
	uint32_t code[2] = { 0, 0 };
#pragma unroll
	for (int c = 0; c < 16; c++)
	{
		// the product is NaN or finite below 2^14 in magnitude (about [0.5, 3.5] when the range is > 0; up to +-11718.75 for an
		// all-equal block, where abottom is a rounding step away from the cells and ascale is 3e6), so truncation toward zero gives
		// CPU_REF's int; a NaN gives 0 here and INT_MIN on x86-64, and both clamp to 0
		int k = __float2int_rz(__fmul_rn(__fsub_rn(a[c], abottom), ascale));
		k = k < 0 ? 0 : (k > 3 ? 3 : k);
		code[c >> 3] |= (uint32_t)k << ((c & 7) << 1);
	}
	q[0] = hmin, q[1] = hmax, q[2] = (uint16_t)code[0], q[3] = (uint16_t)code[1];
}

// a NaN middle level gets the bits CPU_REF's x86-64 SSE arithmetic gives it: a NaN operand propagates quieted (for a NaN that came
// from fp16 bits h, the truncated result is h | 0x200); when both terms are NaN the first operand of the final addition wins; Inf - Inf
// with no NaN operand is the default NaN 0xffc00000, 0xfe00 as fp16
__device__ __forceinline__ uint16_t mid_level(const float v, const uint16_t lo, const uint16_t hi)
{
	if (!isnan(v))
		return f32_to_f16_trunc(v);
	const bool lo_nan = (lo & 0x7fffu) > 0x7c00u, hi_nan = (hi & 0x7fffu) > 0x7c00u;
	if (hi_nan)
		return hi | 0x200u;
	if (lo_nan)
		return lo | 0x200u;
	return 0xfe00u;
}

// q: min, max, codes -> h: the 16 cells in row-major order
__device__ __forceinline__ void lssc_decode(const uint16_t (&q)[4], uint16_t (&h)[16])
{
	const float lo = h2f(q[0]), hi = h2f(q[1]);
	const uint16_t l1 = mid_level(__fadd_rn(__fdiv_rn(hi, 3.f), __fdiv_rn(__fmul_rn(lo, 2.f), 3.f)), q[0], q[1]);
	const uint16_t l2 = mid_level(__fadd_rn(__fdiv_rn(__fmul_rn(hi, 2.f), 3.f), __fdiv_rn(lo, 3.f)), q[0], q[1]);
	// the four levels as one register (level k at bits 16 k), so that the lookup by code stays out of local memory
	const uint64_t level = (uint64_t)q[0] | ((uint64_t)l1 << 16) | ((uint64_t)l2 << 32) | ((uint64_t)q[1] << 48);
#pragma unroll
	for (int c = 0; c < 16; c++)
		h[c] = (uint16_t)(level >> (((q[2 + (c >> 3)] >> ((c & 7) << 1)) & 3) << 4));
}

// ------------------------------------------------------------------------------------------------ NCHW: runs of 4-row bands
// The tensor is P planes of H x W; band g (of G = P Hb) starts at element (g / Hb) H W + (g % Hb) 4 W of the original and at g Wc of
// the compressed tensor, and ends where band g + 1 starts.
struct BandGeom {
	long long H, W, Hb, Wc, G, HW;
	int bands; // bands per CTA
};

__device__ __forceinline__ long long band_start(const BandGeom& b, const long long g)
{
	return (g / b.Hb) * b.HW + (g % b.Hb) * 4 * b.W;
}

// where band (pj planes after the run's first, row by) starts, counted from the run's first band (row by0 of its plane)
__device__ __forceinline__ long long band_offset(const BandGeom& b, const int pj, const int by, const int by0)
{
	return (long long)pj * b.HW + (long long)(by - by0) * 4 * b.W;
}

// n halves of global memory g <-> shared memory s, where s and g have the same address modulo 16: 16-byte accesses in between a scalar
// head and tail
template <bool LOAD>
__device__ __forceinline__ void copy_span(uint16_t* s, uint16_t* g, const long long n)
{
	long long head = (long long)(((16u - ((unsigned)(uintptr_t)g & 15u)) & 15u) >> 1);
	head = head < n ? head : n;
	const long long nv = (n - head) >> 3;
	for (long long i = threadIdx.x; i < head; i += blockDim.x)
		LOAD ? (void)(s[i] = g[i]) : (void)(g[i] = s[i]);
	uint4* const sv = reinterpret_cast<uint4*>(s + head);
	uint4* const gv = reinterpret_cast<uint4*>(g + head);
	for (long long i = threadIdx.x; i < nv; i += blockDim.x)
		LOAD ? (void)(sv[i] = gv[i]) : (void)(gv[i] = sv[i]);
	for (long long i = head + nv * 8 + threadIdx.x; i < n; i += blockDim.x)
		LOAD ? (void)(s[i] = g[i]) : (void)(g[i] = s[i]);
}

// the staging buffers: the original side's span (at most LSSC_SPAN halves) and the compressed side's (at most LSSC_SPAN halves), each
// offset by its global address modulo 16 so that the 16-byte part of the copy is 16-byte aligned on both sides
__device__ __forceinline__ unsigned mis(const void* p) { return ((unsigned)(uintptr_t)p & 15u) >> 1; }

__global__ void __launch_bounds__(LSSC_THREADS) lssc_forw_band_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, const BandGeom b)
{
	extern __shared__ __align__(16) uint16_t smem[];
	const long long g0 = (long long)blockIdx.x * b.bands;
	const long long g1 = g0 + b.bands < b.G ? g0 + b.bands : b.G;
	const long long xs = band_start(b, g0), xe = g1 < b.G ? band_start(b, g1) : (b.G / b.Hb) * b.HW;
	const unsigned xo = mis(x + xs), yo = mis(y + g0 * b.Wc);
	uint16_t* const sx = smem + xo;
	uint16_t* const sy = smem + LSSC_SPAN + 8 + yo;
	copy_span<true>(sx, const_cast<uint16_t*>(x) + xs, xe - xs);
	__syncthreads();
	const int wb = (int)(b.Wc >> 2), W = (int)b.W, H = (int)b.H, Hb = (int)b.Hb;
	const int by0 = (int)(g0 % b.Hb); // band j of the run is band by0 + j of the run's first plane, counting on into the next planes
	const int blocks = (int)(g1 - g0) * wb;
	for (int i = threadIdx.x; i < blocks; i += blockDim.x)
	{
		const int j = i / wb, bx = i - j * wb;
		const int t = by0 + j, pj = t / Hb, by = t - pj * Hb;
		const int rows = H - 4 * by < 4 ? H - 4 * by : 4;
		const int cols = W - 4 * bx < 4 ? W - 4 * bx : 4;
		const uint16_t* const p = sx + band_offset(b, pj, by, by0) + 4 * bx;
		uint16_t h[16];
		h[0] = p[0];
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r + k > 0)
					h[4 * r + k] = r < rows && k < cols ? p[r * W + k] : h[0];
		uint16_t q[4];
		lssc_encode(h, q);
		uint16_t* const o = sy + (long long)j * b.Wc + 4 * bx;
		o[0] = q[0], o[1] = q[1], o[2] = q[2], o[3] = q[3];
	}
	__syncthreads();
	copy_span<false>(sy, y + g0 * b.Wc, (g1 - g0) * b.Wc);
}

__global__ void __launch_bounds__(LSSC_THREADS) lssc_back_band_kernel(const uint16_t* __restrict__ y, uint16_t* __restrict__ x, const BandGeom b)
{
	extern __shared__ __align__(16) uint16_t smem[];
	const long long g0 = (long long)blockIdx.x * b.bands;
	const long long g1 = g0 + b.bands < b.G ? g0 + b.bands : b.G;
	const long long xs = band_start(b, g0), xe = g1 < b.G ? band_start(b, g1) : (b.G / b.Hb) * b.HW;
	const unsigned xo = mis(x + xs), yo = mis(y + g0 * b.Wc);
	uint16_t* const sx = smem + xo;
	uint16_t* const sy = smem + LSSC_SPAN + 8 + yo;
	copy_span<true>(sy, const_cast<uint16_t*>(y) + g0 * b.Wc, (g1 - g0) * b.Wc);
	__syncthreads();
	const int wb = (int)(b.Wc >> 2), W = (int)b.W, H = (int)b.H, Hb = (int)b.Hb;
	const int by0 = (int)(g0 % b.Hb); // band j of the run is band by0 + j of the run's first plane, counting on into the next planes
	const int blocks = (int)(g1 - g0) * wb;
	for (int i = threadIdx.x; i < blocks; i += blockDim.x)
	{
		const int j = i / wb, bx = i - j * wb;
		const int t = by0 + j, pj = t / Hb, by = t - pj * Hb;
		const int rows = H - 4 * by < 4 ? H - 4 * by : 4;
		const int cols = W - 4 * bx < 4 ? W - 4 * bx : 4;
		const uint16_t* const o = sy + (long long)j * b.Wc + 4 * bx;
		const uint16_t q[4] = { o[0], o[1], o[2], o[3] };
		uint16_t h[16];
		lssc_decode(q, h);
		uint16_t* const p = sx + band_offset(b, pj, by, by0) + 4 * bx;
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r < rows && k < cols)
					p[r * W + k] = h[4 * r + k];
	}
	__syncthreads();
	// the band run's span holds exactly the cells inside the tensor, and every one of them was written above
	copy_span<false>(sx, x + xs, xe - xs);
}

// ------------------------------------------------------------------------------------------------ per-block forms
// Element (o, y, x, c) of the original is at o os + y rs + x cs + c, of the compressed (o, by, 4 bx + k, c) at o cos + by crs + (4 bx
// + k) ccs + c.  NCHW: o = plane, C = 1; NHWC: o = n.
struct BlockGeom {
	long long os, rs, cs, cos, crs, ccs;
	int H, W, Hb, Wb, C;
	long long blocks; // outer x Hb x Wb x C (scalar form) or x C / 8 (vector form)
};

template <int V> // channels per thread: 1 (scalar) or 8 (16-byte vectors)
__device__ __forceinline__ void block_of(const BlockGeom& b, const long long i, long long& o, int& by, int& bx, int& c)
{
	const int cv = b.C / V;
	long long t = i;
	c = (int)(t % cv) * V, t /= cv;
	bx = (int)(t % b.Wb), t /= b.Wb;
	by = (int)(t % b.Hb), o = t / b.Hb;
}

__global__ void __launch_bounds__(LSSC_THREADS) lssc_forw_scalar_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, const BlockGeom b)
{
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.blocks; i += (long long)gridDim.x * blockDim.x)
	{
		long long o;
		int by, bx, c;
		block_of<1>(b, i, o, by, bx, c);
		const int rows = b.H - 4 * by < 4 ? b.H - 4 * by : 4, cols = b.W - 4 * bx < 4 ? b.W - 4 * bx : 4;
		const uint16_t* const p = x + o * b.os + (long long)(4 * by) * b.rs + (long long)(4 * bx) * b.cs + c;
		uint16_t h[16];
		h[0] = p[0];
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r + k > 0)
					h[4 * r + k] = r < rows && k < cols ? p[r * b.rs + k * b.cs] : h[0];
		uint16_t q[4];
		lssc_encode(h, q);
		uint16_t* const d = y + o * b.cos + by * b.crs + (long long)(4 * bx) * b.ccs + c;
#pragma unroll
		for (int k = 0; k < 4; k++)
			d[k * b.ccs] = q[k];
	}
}

__global__ void __launch_bounds__(LSSC_THREADS) lssc_back_scalar_kernel(const uint16_t* __restrict__ y, uint16_t* __restrict__ x, const BlockGeom b)
{
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.blocks; i += (long long)gridDim.x * blockDim.x)
	{
		long long o;
		int by, bx, c;
		block_of<1>(b, i, o, by, bx, c);
		const int rows = b.H - 4 * by < 4 ? b.H - 4 * by : 4, cols = b.W - 4 * bx < 4 ? b.W - 4 * bx : 4;
		const uint16_t* const s = y + o * b.cos + by * b.crs + (long long)(4 * bx) * b.ccs + c;
		const uint16_t q[4] = { s[0], s[b.ccs], s[2 * b.ccs], s[3 * b.ccs] };
		uint16_t h[16];
		lssc_decode(q, h);
		uint16_t* const p = x + o * b.os + (long long)(4 * by) * b.rs + (long long)(4 * bx) * b.cs + c;
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r < rows && k < cols)
					p[r * b.rs + k * b.cs] = h[4 * r + k];
	}
}

__device__ __forceinline__ uint16_t lane16(const uint4& v, const int ch)
{
	const uint32_t w = ch < 2 ? v.x : ch < 4 ? v.y : ch < 6 ? v.z : v.w;
	return (uint16_t)(w >> ((ch & 1) << 4));
}
__device__ __forceinline__ void set_lane16(uint4& v, const int ch, const uint16_t h)
{
	uint32_t& w = ch < 2 ? v.x : ch < 4 ? v.y : ch < 6 ? v.z : v.w;
	const int s = (ch & 1) << 4;
	w = (w & ~(0xffffu << s)) | ((uint32_t)h << s);
}

// NHWC, C % 8 == 0, 16-byte aligned bases: one thread per (block, 8 channels)
__global__ void __launch_bounds__(LSSC_THREADS) lssc_forw_vec_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, const BlockGeom b)
{
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.blocks; i += (long long)gridDim.x * blockDim.x)
	{
		long long o;
		int by, bx, c;
		block_of<8>(b, i, o, by, bx, c);
		const int rows = b.H - 4 * by < 4 ? b.H - 4 * by : 4, cols = b.W - 4 * bx < 4 ? b.W - 4 * bx : 4;
		const uint16_t* const p = x + o * b.os + (long long)(4 * by) * b.rs + (long long)(4 * bx) * b.cs + c;
		uint4 v[16];
		v[0] = *reinterpret_cast<const uint4*>(p);
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r + k > 0)
					v[4 * r + k] = r < rows && k < cols ? *reinterpret_cast<const uint4*>(p + r * b.rs + k * b.cs) : v[0];
		uint4 out[4] = {};
#pragma unroll
		for (int ch = 0; ch < 8; ch++)
		{
			uint16_t h[16], q[4];
#pragma unroll
			for (int e = 0; e < 16; e++)
				h[e] = lane16(v[e], ch);
			lssc_encode(h, q);
#pragma unroll
			for (int k = 0; k < 4; k++)
				set_lane16(out[k], ch, q[k]);
		}
		uint16_t* const d = y + o * b.cos + by * b.crs + (long long)(4 * bx) * b.ccs + c;
#pragma unroll
		for (int k = 0; k < 4; k++)
			*reinterpret_cast<uint4*>(d + k * b.ccs) = out[k];
	}
}

__global__ void __launch_bounds__(LSSC_THREADS) lssc_back_vec_kernel(const uint16_t* __restrict__ y, uint16_t* __restrict__ x, const BlockGeom b)
{
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.blocks; i += (long long)gridDim.x * blockDim.x)
	{
		long long o;
		int by, bx, c;
		block_of<8>(b, i, o, by, bx, c);
		const int rows = b.H - 4 * by < 4 ? b.H - 4 * by : 4, cols = b.W - 4 * bx < 4 ? b.W - 4 * bx : 4;
		const uint16_t* const s = y + o * b.cos + by * b.crs + (long long)(4 * bx) * b.ccs + c;
		uint4 in[4];
#pragma unroll
		for (int k = 0; k < 4; k++)
			in[k] = *reinterpret_cast<const uint4*>(s + k * b.ccs);
		uint4 v[16] = {};
#pragma unroll
		for (int ch = 0; ch < 8; ch++)
		{
			const uint16_t q[4] = { lane16(in[0], ch), lane16(in[1], ch), lane16(in[2], ch), lane16(in[3], ch) };
			uint16_t h[16];
			lssc_decode(q, h);
#pragma unroll
			for (int e = 0; e < 16; e++)
				set_lane16(v[e], ch, h[e]);
		}
		uint16_t* const p = x + o * b.os + (long long)(4 * by) * b.rs + (long long)(4 * bx) * b.cs + c;
#pragma unroll
		for (int r = 0; r < 4; r++)
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (r < rows && k < cols)
					*reinterpret_cast<uint4*>(p + r * b.rs + k * b.cs) = v[4 * r + k];
	}
}

// ------------------------------------------------------------------------------------------------ host side

// one (original, compressed) pair, checked: the original's geometry and layout
struct Pair {
	const ccv_nnc_tensor_t* x; // original
	const ccv_nnc_tensor_t* y; // compressed
	bool nchw;
	long long outer; // NCHW: N x C planes; NHWC: N
	int H, W, C;     // C: NHWC channels (1 for NCHW)
};

bool fp16_dense(const ccv_nnc_tensor_t* const t)
{
	// CCV_GET_DATA_TYPE keeps the CCV_QX bit, so a palettized tensor (datatype CCV_QX | ...) is not CCV_16F here
	return t && t->info.datatype == CCV_16F && CCV_IS_TENSOR_CONTIGUOUS(t) && CCV_TENSOR_GET_MEMORY(t->info.type) == CCV_TENSOR_GPU_MEMORY && t->data.u8;
}

// x original, y compressed: refused unless y has exactly the shape _ccv_nnc_lssc_tensor_auto_forw gives x
bool check_pair(const ccv_nnc_tensor_t* const x, const ccv_nnc_tensor_t* const y, Pair& p)
{
	if (!fp16_dense(x) || !fp16_dense(y))
		return false;
	const int format = x->info.format;
	if ((format != CCV_TENSOR_FORMAT_NCHW && format != CCV_TENSOR_FORMAT_NHWC) || y->info.format != format)
		return false;
	const int nd = nd_of(x);
	if ((nd != 3 && nd != 4) || nd_of(y) != nd)
		return false;
	const int* const d = x->info.dim;
	const int hw = format == CCV_TENSOR_FORMAT_NCHW ? nd - 2 : nd - 3; // ccv_nnc_tensor_hw
	for (int i = 0; i < nd; i++)
	{
		const long long want = i == hw ? ((long long)d[i] + 3) / 4 : i == hw + 1 ? ((long long)d[i] + 3) / 4 * 4 : d[i];
		if (y->info.dim[i] != want)
			return false;
	}
	p.x = x, p.y = y;
	p.nchw = format == CCV_TENSOR_FORMAT_NCHW;
	p.H = d[hw], p.W = d[hw + 1];
	p.C = p.nchw ? 1 : d[hw + 2];
	p.outer = 1;
	for (int i = 0; i < hw; i++)
		p.outer *= d[i];
	return true;
}

int run_pair(const Pair& p, const bool forward, cudaStream_t s)
{
	uint16_t* const xp = reinterpret_cast<uint16_t*>(p.x->data.u8);
	uint16_t* const yp = reinterpret_cast<uint16_t*>(p.y->data.u8);
	const long long Hb = (p.H + 3) / 4, Wb = (p.W + 3) / 4, Wc = 4 * Wb;
	if (p.outer == 0)
		return 0;
	if (p.nchw && p.W <= LSSC_BAND_MAX_W)
	{
		BandGeom b;
		b.H = p.H, b.W = p.W, b.Hb = Hb, b.Wc = Wc, b.G = p.outer * Hb, b.HW = (long long)p.H * p.W;
		// as many bands as fit (LSSC_SPAN halves of the original per CTA), but no fewer than LSSC_CTAS_PER_SM CTAs per SM when the
		// tensor has that many bands
		const long long fit = LSSC_SPAN / (4 * b.W), spread = (b.G + (long long)sm_count() * LSSC_CTAS_PER_SM - 1) / ((long long)sm_count() * LSSC_CTAS_PER_SM);
		b.bands = (int)(spread < fit ? (spread > 0 ? spread : 1) : fit);
		const long long ctas = (b.G + b.bands - 1) / b.bands;
		// the original's span is at most 4 W bands halves, the compressed one's bands Wc <= LSSC_SPAN (W >= 1); 8 halves of slack
		// each for the alignment offset
		const size_t shm = (size_t)(2 * LSSC_SPAN + 16) * sizeof(uint16_t);
		if (forward)
			lssc_forw_band_kernel<<<(unsigned)ctas, LSSC_THREADS, shm, s>>>(xp, yp, b);
		else
			lssc_back_band_kernel<<<(unsigned)ctas, LSSC_THREADS, shm, s>>>(yp, xp, b);
		return launched(forward ? "lssc_forw_band" : "lssc_back_band");
	}
	BlockGeom b;
	b.H = p.H, b.W = p.W, b.Hb = (int)Hb, b.Wb = (int)Wb, b.C = p.C;
	if (p.nchw)
	{
		b.os = (long long)p.H * p.W, b.rs = p.W, b.cs = 1;
		b.cos = Hb * Wc, b.crs = Wc, b.ccs = 1;
	} else {
		b.os = (long long)p.H * p.W * p.C, b.rs = (long long)p.W * p.C, b.cs = p.C;
		b.cos = Hb * Wc * p.C, b.crs = Wc * p.C, b.ccs = p.C;
	}
	const bool vec = !p.nchw && p.C % 8 == 0 && aligned_v16(xp) && aligned_v16(yp);
	b.blocks = p.outer * Hb * Wb * (vec ? p.C / 8 : p.C);
	const int grid = grid_for((size_t)b.blocks, LSSC_THREADS, 16);
	if (vec)
	{
		if (forward)
			lssc_forw_vec_kernel<<<grid, LSSC_THREADS, 0, s>>>(xp, yp, b);
		else
			lssc_back_vec_kernel<<<grid, LSSC_THREADS, 0, s>>>(yp, xp, b);
		return launched(forward ? "lssc_forw_vec" : "lssc_back_vec");
	}
	if (forward)
		lssc_forw_scalar_kernel<<<grid, LSSC_THREADS, 0, s>>>(xp, yp, b);
	else
		lssc_back_scalar_kernel<<<grid, LSSC_THREADS, 0, s>>>(yp, xp, b);
	return launched(forward ? "lssc_forw_scalar" : "lssc_back_scalar");
}

// forward: inputs (x_1 .. x_n) -> outputs (y_1 .. y_n), input_size == output_size; backward: inputs (y_1 .. y_m) -> outputs (x_1 ..
// x_n), n <= m (_ccv_nnc_lssc_forw_bitmask / _back_bitmask).  Every pair is checked before the first launch.
template <bool FORWARD>
int exec_lssc(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (output_size < 1 || (FORWARD ? input_size != output_size : input_size < output_size) || !inputs || !outputs)
		return CCV_NNC_EXEC_INVALID;
	Pair stack[8];
	Pair* const pairs = output_size <= 8 ? stack : new Pair[output_size];
	bool ok = true;
	for (int i = 0; i < output_size && ok; i++)
		ok = FORWARD ? check_pair(inputs[i], outputs[i], pairs[i]) : check_pair(outputs[i], inputs[i], pairs[i]);
	int rc = ok ? CCV_NNC_EXEC_SUCCESS : CCV_NNC_EXEC_INVALID;
	cudaStream_t s = (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context);
	for (int i = 0; i < output_size && rc == CCV_NNC_EXEC_SUCCESS; i++)
		if (run_pair(pairs[i], FORWARD, s))
			rc = CCV_NNC_EXEC_INVALID;
	if (pairs != stack)
		delete[] pairs;
	return rc;
}

} // namespace

REGISTER_SM100(CCV_NNC_COMPRESSION_LSSC_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_16F, 1, exec_lssc<true>); }
REGISTER_SM100(CCV_NNC_COMPRESSION_LSSC_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_16F, 1, exec_lssc<false>); }
