// sm100_palettize.cu -- palettized (CCV_QX) weights: the decoder behind ccv_nnc_depalettize on GPU memory and the unfused
// QX commands, and a fused few-row GEMM that reads the packed weight directly.
//
// Format (ccv_nnc_tensor_palettize / ccv_nnc_palettize): elements in flat order, in blocks of `nib`.  A block stores its palette
// (2^q entries of the palette type) followed by its indices, q bits each, packed most significant bit first; every 8 indices fill
// q bytes.  The block stride is 2^q * sizeof(palette) + nib * q / 8 bytes, so nib * q must be a multiple of 8.  The last block may
// be partial; its index bytes end at ceil(count * q / 8) of the whole tensor's index bytes, the unused bits are zero.
#include "sm100_contract.h"
#include <cuda_fp16.h>
#include <stdint.h>

namespace sm100 {

bool palettize_params_ok(const int qbits, const int nib)
{
	return qbits >= 4 && qbits <= 8 && nib > 0 && ((long long)nib * qbits) % 8 == 0;
}

size_t palettize_data_bytes(const size_t count, const int qbits, const int nib, const size_t palette_elem)
{
	const size_t blocks = (count + (size_t)nib - 1) / (size_t)nib;
	return ((size_t)1 << qbits) * palette_elem * blocks + (count * (size_t)qbits + 7) / 8;
}

namespace {

// index j (q bits at bit j * q, MSB first) of a block's index bytes; `avail` bytes of them exist
__device__ __forceinline__ unsigned index_at(const uint8_t* const idx, const long long j, const int q, const long long avail)
{
	const long long bit = j * q;
	const long long byte = bit >> 3;
	const int sh = (int)(bit & 7);
	unsigned w = (unsigned)__ldg(idx + byte) << 8;
	if (sh + q > 8 && byte + 1 < avail)
		w |= __ldg(idx + byte + 1);
	return (w >> (16 - sh - q)) & ((1u << q) - 1);
}

// the 8 indices packed in q bytes (one group), as a 64-bit big-endian word's top 8q bits; bytes past `avail` read as zero
__device__ __forceinline__ uint64_t group_bits(const uint8_t* const p, const int q, const long long avail)
{
	uint64_t v = 0;
	for (int b = 0; b < 8; b++)
		if (b < q)
			v |= (uint64_t)(b < avail ? __ldg(p + b) : 0) << (56 - 8 * b);
	return v;
}

// 8 consecutive elements, as 16-byte stores when dst is 16-byte aligned
__device__ __forceinline__ void store8(uint16_t* const dst, const uint16_t (&v)[8], const bool vec)
{
	if (vec)
		*(uint4*)dst = make_uint4(v[0] | ((unsigned)v[1] << 16), v[2] | ((unsigned)v[3] << 16), v[4] | ((unsigned)v[5] << 16), v[6] | ((unsigned)v[7] << 16));
	else
#pragma unroll
		for (int i = 0; i < 8; i++)
			dst[i] = v[i];
}
__device__ __forceinline__ void store8(float* const dst, const float (&v)[8], const bool vec)
{
	if (vec)
		((float4*)dst)[0] = make_float4(v[0], v[1], v[2], v[3]), ((float4*)dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
	else
#pragma unroll
		for (int i = 0; i < 8; i++)
			dst[i] = v[i];
}
__device__ __forceinline__ void store8(double* const dst, const double (&v)[8], const bool vec)
{
	if (vec)
#pragma unroll
		for (int i = 0; i < 4; i++)
			((double2*)dst)[i] = make_double2(v[2 * i], v[2 * i + 1]);
	else
#pragma unroll
		for (int i = 0; i < 8; i++)
			dst[i] = v[i];
}

// One warp per block (grid-stride): the warp copies the block's palette to its slice of shared memory, then each lane decodes
// one 8-index group (q bytes) per step and stores 8 elements, with 16-byte stores where the output is 16-byte aligned.
template <class T>
__global__ void __launch_bounds__(256) depalettize_kernel(const uint8_t* const in, const int q, const int nib, const size_t count, T* const out)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int entries = 1 << q;
	T* const pal = (T*)smem_raw + (size_t)warp * entries;
	unsigned char* const pal_b = (unsigned char*)pal;
	const size_t pal_bytes = (size_t)entries * sizeof(T), idx_bytes = (size_t)nib * q / 8, stride = pal_bytes + idx_bytes;
	const size_t blocks = (count + nib - 1) / nib;
	const long long total_idx = (long long)((count * q + 7) / 8);
	for (size_t b = (size_t)blockIdx.x * (blockDim.x >> 5) + warp; b < blocks; b += (size_t)gridDim.x * (blockDim.x >> 5))
	{
		const uint8_t* const base = in + b * stride;
		__syncwarp();
		// byte copies: a block's palette sits wherever the previous blocks' index bytes end (an odd address for q = 4, nib = 6)
		for (int i = lane; i < (int)pal_bytes; i += 32)
			pal_b[i] = __ldg(base + i);
		__syncwarp();
		const size_t first = b * (size_t)nib;
		const int n = (int)(count - first < (size_t)nib ? count - first : (size_t)nib);
		const uint8_t* const idx = base + pal_bytes;
		// index bytes of this block that exist: the whole stride for a full block, up to the tensor's last index byte otherwise
		const long long avail = total_idx - (long long)(b * idx_bytes);
		const bool vec = ((first * sizeof(T)) % 16 == 0) && (((uintptr_t)out) % 16 == 0);
		for (int g = lane; g * 8 < n; g += 32)
		{
			const uint64_t bits = group_bits(idx + (size_t)g * q, q, avail - (long long)g * q);
			T v[8];
#pragma unroll
			for (int e = 0; e < 8; e++)
				v[e] = pal[(unsigned)(bits >> (64 - q * (e + 1))) & (entries - 1)];
			T* const dst = out + first + (size_t)g * 8;
			if (g * 8 + 8 <= n)
				store8(dst, v, vec);
			else
#pragma unroll
				for (int e = 0; e < 8; e++)
					if (g * 8 + e < n)
						dst[e] = v[e];
		}
	}
}

template <class T>
int launch_depalettize(cudaStream_t stream, const uint8_t* in, int q, int nib, size_t count, T* out)
{
	const size_t blocks = (count + nib - 1) / nib;
	const int warps = 8;
	const size_t grid = (blocks + warps - 1) / warps;
	const unsigned g = (unsigned)(grid < (size_t)132 * 64 ? grid : (size_t)132 * 64);
	const size_t smem = (size_t)warps * ((size_t)1 << q) * sizeof(T);
	depalettize_kernel<T><<<g, warps * 32, smem, stream>>>(in, q, nib, count, out);
	return launched("depalettize_kernel launch");
}

// palette entry i of a block whose palette starts at `pal` (2-byte aligned when `aligned`; else read as two bytes)
__device__ __forceinline__ float palette_f16(const uint8_t* const pal, const unsigned i, const bool aligned)
{
	if (aligned)
		return __half2float(__ldg((const __half*)pal + i));
	const unsigned short u = (unsigned short)(__ldg(pal + 2 * i) | ((unsigned)__ldg(pal + 2 * i + 1) << 8));
	return __half2float(__ushort_as_half(u));
}

// Fused few-row GEMM: c[m, n] = sum_k a[m, k] * w[n, k] (+ bias[n]) with w [N, K] palettized (fp16 palettes), a and c fp16.  One warp
// per row n of w: lane l takes the 8-element groups k0 = 8 (l + 32 i) in increasing i and accumulates M fp32 sums in that order, the
// warp then adds its lanes in a fixed butterfly, lane 0 adds the bias and rounds once to fp16 (to nearest even).  Palettes and index
// bytes are read straight from global memory (through L1); nothing decoded is written.  Groups that lie inside one block and start
// on an 8-index boundary decode from q whole bytes; others (nib or K not multiples of 8, block edges) index by index.
template <int MMAX>
__global__ void __launch_bounds__(256) palettized_gemm_f16_kernel(const __half* const a, const long long lda, const uint8_t* const wq, const int q, const int nib, const int M, const int N, const int K,
	__half* const c, const long long ldc, const float* const bias32, const __half* const bias16)
{
	const int lane = threadIdx.x & 31;
	const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (n >= N)
		return;
	const int entries = 1 << q;
	const size_t pal_bytes = (size_t)entries * 2, idx_bytes = (size_t)nib * q / 8, stride = pal_bytes + idx_bytes;
	const size_t count = (size_t)N * K;
	const long long total_idx = (long long)((count * q + 7) / 8);
	const bool avec = (lda % 8 == 0) && (((uintptr_t)a) % 16 == 0);
	const bool pal2 = stride % 2 == 0 && ((uintptr_t)wq) % 2 == 0;
	float acc[MMAX];
#pragma unroll
	for (int m = 0; m < MMAX; m++)
		acc[m] = 0.f;
	for (int k0 = lane * 8; k0 < K; k0 += 256)
	{
		const size_t e0 = (size_t)n * K + k0;
		const int kn = K - k0 < 8 ? K - k0 : 8;
		size_t b = e0 / nib;
		long long j = (long long)(e0 - b * nib);
		float w[8];
		if (kn == 8 && (j & 7) == 0 && j + 8 <= nib)
		{
			const uint8_t* const base = wq + b * stride;
			const long long avail = total_idx - (long long)(b * idx_bytes) - (j / 8) * q;
			const uint64_t bits = group_bits(base + pal_bytes + (j / 8) * q, q, avail);
#pragma unroll
			for (int e = 0; e < 8; e++)
				w[e] = palette_f16(base, (unsigned)(bits >> (64 - q * (e + 1))) & (entries - 1), pal2);
		} else {
#pragma unroll
			for (int e = 0; e < 8; e++)
			{
				if (e < kn)
				{
					const uint8_t* const base = wq + b * stride;
					const unsigned i = index_at(base + pal_bytes, j, q, total_idx - (long long)(b * idx_bytes));
					w[e] = palette_f16(base, i, pal2);
					if (++j == nib)
						j = 0, b++;
				} else
					w[e] = 0.f;
			}
		}
#pragma unroll
		for (int m = 0; m < MMAX; m++)
		{
			if (m < M)
			{
				const __half* const ar = a + m * lda + k0;
				float x[8];
				if (avec && kn == 8)
				{
					const uint4 u = __ldg((const uint4*)ar);
					const __half2* const h = (const __half2*)&u;
#pragma unroll
					for (int e = 0; e < 4; e++)
					{
						const float2 f = __half22float2(h[e]);
						x[2 * e] = f.x, x[2 * e + 1] = f.y;
					}
				} else {
#pragma unroll
					for (int e = 0; e < 8; e++)
						x[e] = e < kn ? __half2float(ar[e]) : 0.f;
				}
#pragma unroll
				for (int e = 0; e < 8; e++)
					acc[m] = fmaf(x[e], w[e], acc[m]);
			}
		}
	}
#pragma unroll
	for (int m = 0; m < MMAX; m++)
	{
		float v = acc[m];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1)
			v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0 && m < M)
		{
			if (bias32)
				v += bias32[n];
			else if (bias16)
				v += __half2float(bias16[n]);
			c[m * ldc + n] = __float2half_rn(v);
		}
	}
}

} // namespace

int depalettize(cudaStream_t stream, const void* in, const int palette_datatype, const int qbits, const int nib, void* out, const size_t count)
{
	if (!palettize_params_ok(qbits, nib))
		return 1;
	if (count == 0)
		return 0;
	switch (palette_datatype)
	{
		case 0x20000: return launch_depalettize(stream, (const uint8_t*)in, qbits, nib, count, (uint16_t*)out);            // CCV_16F
		case 0x04000: return launch_depalettize(stream, (const uint8_t*)in, qbits, nib, count, (float*)out);               // CCV_32F
		case 0x10000: return launch_depalettize(stream, (const uint8_t*)in, qbits, nib, count, (double*)out);              // CCV_64F
	}
	return 1;
}

int gemm_palettized_f16(cudaStream_t stream, const int M, const int N, const int K, const void* a, const long long lda, const void* wq, const int qbits, const int nib, void* c, const long long ldc, const float* bias32, const void* bias16)
{
	if (!palettize_params_ok(qbits, nib) || M < 1 || M > PALETTIZED_GEMM_M_MAX || N < 1 || K < 1 || lda < K || ldc < N)
		return 1;
	const int warps = 8;
	const dim3 grid((N + warps - 1) / warps);
	palettized_gemm_f16_kernel<PALETTIZED_GEMM_M_MAX><<<grid, warps * 32, 0, stream>>>((const __half*)a, lda, (const uint8_t*)wq, qbits, nib, M, N, K, (__half*)c, ldc, bias32, (const __half*)bias16);
	return launched("palettized_gemm_f16_kernel launch");
}

} // namespace sm100
