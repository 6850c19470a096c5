// sm100_ew.cu -- the HBM-bound kernels: elementwise, pooling, batch norm, softmax, losses, SGD, dtype / layout moves.
// All are coalesced, 128-bit vectorised where the shape allows, grid-stride with the grid sized as a multiple of the
// SM count; reductions use warp shuffles and one atomic per block.  Semantics follow CCV_NNC_BACKEND_CPU_REF
// (file:line cited per kernel, relative to /root/reference/lib/nnc/cmd).
#include "sm100_ew.h"
#include "sm100_elem.cuh"
#include "sm100_cmd.h"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <float.h>

namespace sm100 {

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		v += __shfl_xor_sync(0xffffffff, v, o);
	return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		v = fmaxf(v, __shfl_xor_sync(0xffffffff, v, o));
	return v;
}
// block-wide reductions for blockDim.x <= 1024 (result valid in every thread)
__device__ __forceinline__ float block_sum(float v, float* sh)
{
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	v = warp_sum(v);
	__syncthreads();
	if (lane == 0)
		sh[w] = v;
	__syncthreads();
	v = lane < nw ? sh[lane] : 0.f;
	return warp_sum(v);
}
__device__ __forceinline__ float block_max(float v, float* sh)
{
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	v = warp_max(v);
	__syncthreads();
	if (lane == 0)
		sh[w] = v;
	__syncthreads();
	v = lane < nw ? sh[lane] : -FLT_MAX;
	return warp_max(v);
}

static inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

// =============================================================================================== set / sum / axpby
__global__ void set_f32_kernel(float* __restrict__ p, const size_t n, const float v)
{
	const size_t n4 = n >> 2;
	const float4 v4 = make_float4(v, v, v, v);
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
		reinterpret_cast<float4*>(p)[i] = v4;
	for (size_t i = (n4 << 2) + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		p[i] = v;
}
__global__ void set_f32_scalar_kernel(float* __restrict__ p, const size_t n, const float v)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		p[i] = v;
}
// util/ccv_nnc_util_cpu_ref.c:596-640 (SET)
int ew_set_f32(cudaStream_t s, float* p, size_t n, float v)
{
	if (n == 0)
		return 0;
	if (aligned16(p))
		set_f32_kernel<<<grid_for((n >> 2) + 1, 256, 8), 256, 0, s>>>(p, n, v);
	else
		set_f32_scalar_kernel<<<grid_for(n, 256, 8), 256, 0, s>>>(p, n, v);
	return launched("set_f32");
}
__global__ void set_u16_kernel(uint16_t* __restrict__ p, const size_t n, const uint16_t v)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		p[i] = v;
}
int ew_set_u16(cudaStream_t s, uint16_t* p, size_t n, uint16_t v)
{
	if (n == 0)
		return 0;
	set_u16_kernel<<<grid_for(n, 256, 8), 256, 0, s>>>(p, n, v);
	return launched("set_u16");
}
__global__ void set_u64_kernel(uint64_t* __restrict__ p, const size_t n, const uint64_t v)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		p[i] = v;
}
int ew_set_u64(cudaStream_t s, uint64_t* p, size_t n, uint64_t v)
{
	if (n == 0)
		return 0;
	set_u64_kernel<<<grid_for(n, 256, 8), 256, 0, s>>>(p, n, v);
	return launched("set_u64");
}
// int32 n-ary sum (label / index arithmetic in graphs: small tensors, scalar accesses)
struct SumArgsI32 {
	const int* in[64];
	int k;
};
__global__ void sum_i32_kernel(const SumArgsI32 a, int* __restrict__ out, const size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		int v = 0;
		for (int j = 0; j < a.k; j++)
			v += a.in[j][i];
		out[i] = v;
	}
}
int ew_sum_i32(cudaStream_t s, const int* const* inputs, int k, int* out, size_t n)
{
	if (n == 0)
		return 0;
	if (k < 1 || k > 64)
		return 1;
	SumArgsI32 a;
	for (int j = 0; j < k; j++)
		a.in[j] = inputs[j];
	a.k = k;
	sum_i32_kernel<<<grid_for(n, 256, 8), 256, 0, s>>>(a, out, n);
	return launched("sum_i32");
}

struct SumArgs {
	const float* in[8];
	int k;
};
template <int VEC>
__global__ void sum_kernel(const SumArgs a, float* __restrict__ out, const size_t n, const int accumulate)
{
	if (VEC == 4)
	{
		const size_t n4 = n >> 2;
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
		{
			float4 acc = accumulate ? reinterpret_cast<const float4*>(out)[i] : make_float4(0, 0, 0, 0);
#pragma unroll 8
			for (int j = 0; j < a.k; j++)
			{
				const float4 v = reinterpret_cast<const float4*>(a.in[j])[i];
				acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
			}
			reinterpret_cast<float4*>(out)[i] = acc;
		}
		for (size_t i = (n4 << 2) + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		{
			float acc = accumulate ? out[i] : 0.f;
			for (int j = 0; j < a.k; j++)
				acc += a.in[j][i];
			out[i] = acc;
		}
	} else {
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		{
			float acc = accumulate ? out[i] : 0.f;
			for (int j = 0; j < a.k; j++)
				acc += a.in[j][i];
			out[i] = acc;
		}
	}
}
// ew/ccv_nnc_ew_cpu_ref.c:15-110 (EWSUM): c = a0 + a1 + ...; evaluated left to right like the reference
int ew_sum_f32(cudaStream_t s, const float* const* inputs, int k, float* out, size_t n)
{
	if (n == 0 || k <= 0)
		return 0;
	int done = 0;
	while (done < k)
	{
		SumArgs a;
		a.k = (k - done) > 8 ? 8 : (k - done);
		bool vec = aligned16(out);
		for (int j = 0; j < a.k; j++)
		{
			a.in[j] = inputs[done + j];
			vec = vec && aligned16(a.in[j]);
		}
		if (vec)
			sum_kernel<4><<<grid_for((n >> 2) + 1, 256, 8), 256, 0, s>>>(a, out, n, done > 0);
		else
			sum_kernel<1><<<grid_for(n, 256, 8), 256, 0, s>>>(a, out, n, done > 0);
		if (launched("ew_sum"))
			return -1;
		done += a.k;
	}
	return 0;
}

__global__ void axpby_kernel(const float p, const float* __restrict__ a, const float q, const float* __restrict__ b, float* __restrict__ c, const size_t n, const int vec)
{
	if (vec)
	{
		const size_t n4 = n >> 2;
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
		{
			const float4 x = reinterpret_cast<const float4*>(a)[i];
			float4 r = make_float4(p * x.x, p * x.y, p * x.z, p * x.w);
			if (b)
			{
				const float4 y = reinterpret_cast<const float4*>(b)[i];
				r.x += q * y.x, r.y += q * y.y, r.z += q * y.z, r.w += q * y.w;
			}
			reinterpret_cast<float4*>(c)[i] = r;
		}
		for (size_t i = (n4 << 2) + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			c[i] = b ? p * a[i] + q * b[i] : p * a[i];
	} else
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			c[i] = b ? p * a[i] + q * b[i] : p * a[i];
}
// blas/ccv_nnc_add_cpu_ref.c (ADD: c = p * a + q * b), blas/ccv_nnc_mul_cpu_ref.c (SCALAR_MUL: c = p * a)
int ew_axpby_f32(cudaStream_t s, float p, const float* a, float q, const float* b, float* c, size_t n)
{
	if (n == 0)
		return 0;
	const int vec = aligned16(a) && aligned16(c) && (!b || aligned16(b));
	axpby_kernel<<<grid_for(vec ? (n >> 2) + 1 : n, 256, 8), 256, 0, s>>>(p, a, q, b, c, n, vec);
	return launched("ew_axpby");
}

struct Bcast4 {
	int dim[4];
	int as[4], bs[4], cs[4];
};
template <int OP>
__global__ void bcast_kernel(const float p, const float* __restrict__ a, const float q, const float* __restrict__ b, float* __restrict__ c, const Bcast4 d, const size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		size_t r = i;
		const int i3 = r % d.dim[3];
		r /= d.dim[3];
		const int i2 = r % d.dim[2];
		r /= d.dim[2];
		const int i1 = r % d.dim[1];
		const int i0 = (int)(r / d.dim[1]);
		const float av = a[(size_t)i0 * d.as[0] + (size_t)i1 * d.as[1] + (size_t)i2 * d.as[2] + (size_t)i3 * d.as[3]];
		const size_t co = (size_t)i0 * d.cs[0] + (size_t)i1 * d.cs[1] + (size_t)i2 * d.cs[2] + (size_t)i3 * d.cs[3];
		if (OP == 0)
			c[co] = b ? p * av + q * b[(size_t)i0 * d.bs[0] + (size_t)i1 * d.bs[1] + (size_t)i2 * d.bs[2] + (size_t)i3 * d.bs[3]] : p * av;
		else
			c[co] = p * av * b[(size_t)i0 * d.bs[0] + (size_t)i1 * d.bs[1] + (size_t)i2 * d.bs[2] + (size_t)i3 * d.bs[3]];
	}
}
static Bcast4 make_bcast(const int* as, const int* bs, const int* cs, const int* dim)
{
	Bcast4 d;
	for (int i = 0; i < 4; i++)
		d.dim[i] = dim[i] > 0 ? dim[i] : 1, d.as[i] = as[i], d.bs[i] = bs ? bs[i] : 0, d.cs[i] = cs[i];
	return d;
}
int ew_axpby_bcast_f32(cudaStream_t s, float p, const float* a, const int* astride, float q, const float* b, const int* bstride, float* c, const int* cstride, const int* dim)
{
	const Bcast4 d = make_bcast(astride, bstride, cstride, dim);
	const size_t n = (size_t)d.dim[0] * d.dim[1] * d.dim[2] * d.dim[3];
	if (n == 0)
		return 0;
	bcast_kernel<0><<<grid_for(n, 256, 8), 256, 0, s>>>(p, a, q, b, c, d, n);
	return launched("ew_axpby_bcast");
}
int ew_mul_bcast_f32(cudaStream_t s, float p, const float* a, const int* astride, const float* b, const int* bstride, float* c, const int* cstride, const int* dim)
{
	const Bcast4 d = make_bcast(astride, bstride, cstride, dim);
	const size_t n = (size_t)d.dim[0] * d.dim[1] * d.dim[2] * d.dim[3];
	if (n == 0)
		return 0;
	bcast_kernel<1><<<grid_for(n, 256, 8), 256, 0, s>>>(p, a, 0.f, b, c, d, n);
	return launched("ew_mul_bcast");
}

// =============================================================================================== relu
__global__ void relu_fwd_kernel(const float* __restrict__ a, float* __restrict__ b, const size_t n, const int vec)
{
	if (vec)
	{
		const size_t n4 = n >> 2;
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
		{
			const float4 x = reinterpret_cast<const float4*>(a)[i];
			reinterpret_cast<float4*>(b)[i] = make_float4(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f), fmaxf(x.z, 0.f), fmaxf(x.w, 0.f));
		}
		for (size_t i = (n4 << 2) + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			b[i] = fmaxf(a[i], 0.f);
	} else
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			b[i] = fmaxf(a[i], 0.f);
}
// relu/ccv_nnc_relu_cpu_ref.c:13-31
int ew_relu_fwd_f32(cudaStream_t s, const float* a, float* b, size_t n)
{
	if (n == 0)
		return 0;
	const int vec = aligned16(a) && aligned16(b);
	relu_fwd_kernel<<<grid_for(vec ? (n >> 2) + 1 : n, 256, 8), 256, 0, s>>>(a, b, n, vec);
	return launched("relu_fwd");
}
__global__ void relu_bwd_kernel(const float* __restrict__ g, const float* __restrict__ b, float* __restrict__ h, const size_t n, const int vec)
{
	if (vec)
	{
		const size_t n4 = n >> 2;
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
		{
			const float4 x = reinterpret_cast<const float4*>(b)[i];
			const float4 y = reinterpret_cast<const float4*>(g)[i];
			reinterpret_cast<float4*>(h)[i] = make_float4(x.x > 0 ? y.x : 0.f, x.y > 0 ? y.y : 0.f, x.z > 0 ? y.z : 0.f, x.w > 0 ? y.w : 0.f);
		}
		for (size_t i = (n4 << 2) + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			h[i] = b[i] > 0 ? g[i] : 0.f;
	} else
		for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
			h[i] = b[i] > 0 ? g[i] : 0.f;
}
// relu/ccv_nnc_relu_cpu_ref.c:33-55: the mask is the forward OUTPUT b > 0
int ew_relu_bwd_f32(cudaStream_t s, const float* g, const float* b, float* h, size_t n)
{
	if (n == 0)
		return 0;
	const int vec = aligned16(g) && aligned16(b) && aligned16(h);
	relu_bwd_kernel<<<grid_for(vec ? (n >> 2) + 1 : n, 256, 8), 256, 0, s>>>(g, b, h, n, vec);
	return launched("relu_bwd");
}

// =============================================================================================== column sums
// Each block owns a slab of rows; threads are laid out (column, row-lane); per-column partials are combined across
// the block in shared memory and added to the output with one atomic per (block, column).
__global__ void colsum_kernel(const float* __restrict__ g, const size_t rows, const int cols, const long long ld, float* __restrict__ out, const int cpb)
{
	extern __shared__ float sh[];
	const int tx = threadIdx.x % cpb, ty = threadIdx.x / cpb, rpi = blockDim.x / cpb;
	const int col = blockIdx.x * cpb + tx;
	float acc = 0.f;
	if (ty < rpi && col < cols)
		for (size_t r = (size_t)blockIdx.y * rpi + ty; r < rows; r += (size_t)gridDim.y * rpi)
			acc += g[r * ld + col];
	sh[threadIdx.x] = acc;
	__syncthreads();
	if (ty == 0 && col < cols)
	{
		for (int j = 1; j < rpi; j++)
			acc += sh[j * cpb + tx];
		atomicAdd(out + col, acc);
	}
}
// Vector form (cols, ld multiples of 4, 16-byte aligned): a thread owns one float4 column group and keeps four row loads
// in flight; a block covers `cpb` column groups x (256 / cpb) rows per step.
__global__ void __launch_bounds__(256) colsum_vec_kernel(const float4* __restrict__ g, const size_t rows, const int cols4, const long long ld4, float* __restrict__ out, float* __restrict__ part, const int cpb)
{
	__shared__ float4 sh[256];
	const int tx = threadIdx.x % cpb, ty = threadIdx.x / cpb, rpi = 256 / cpb;
	const int col4 = blockIdx.x * cpb + tx;
	float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
	if (col4 < cols4)
	{
		const size_t step = (size_t)gridDim.y * rpi;
		size_t r = (size_t)blockIdx.y * rpi + ty;
		const float4* p = g + col4;
		for (; r + 3 * step < rows; r += 4 * step)
		{
			const float4 v0 = __ldg(p + r * ld4), v1 = __ldg(p + (r + step) * ld4), v2 = __ldg(p + (r + 2 * step) * ld4), v3 = __ldg(p + (r + 3 * step) * ld4);
			a0.x += v0.x, a0.y += v0.y, a0.z += v0.z, a0.w += v0.w;
			a1.x += v1.x, a1.y += v1.y, a1.z += v1.z, a1.w += v1.w;
			a2.x += v2.x, a2.y += v2.y, a2.z += v2.z, a2.w += v2.w;
			a3.x += v3.x, a3.y += v3.y, a3.z += v3.z, a3.w += v3.w;
		}
		for (; r < rows; r += step)
		{
			const float4 v0 = __ldg(p + r * ld4);
			a0.x += v0.x, a0.y += v0.y, a0.z += v0.z, a0.w += v0.w;
		}
	}
	a0.x += a1.x + a2.x + a3.x, a0.y += a1.y + a2.y + a3.y, a0.z += a1.z + a2.z + a3.z, a0.w += a1.w + a2.w + a3.w;
	sh[threadIdx.x] = a0;
	__syncthreads();
	if (ty == 0 && col4 < cols4)
	{
		for (int j = 1; j < rpi; j++)
		{
			const float4 v = sh[j * cpb + tx];
			a0.x += v.x, a0.y += v.y, a0.z += v.z, a0.w += v.w;
		}
		if (part) // two-stage: per-block partial rows, summed in a fixed order by colsum_partials_kernel
			*reinterpret_cast<float4*>(part + ((size_t)blockIdx.y * cols4 + col4) * 4) = a0;
		else {
			float* const o = out + 4 * (size_t)col4;
			atomicAdd(o, a0.x), atomicAdd(o + 1, a0.y), atomicAdd(o + 2, a0.z), atomicAdd(o + 3, a0.w);
		}
	}
}
// out[col] (+)= sum over y of part[y][col]: 32 columns x 32 row-lanes per block, fixed summation order
__global__ void __launch_bounds__(1024) colsum_partials_kernel(const float* __restrict__ part, const int gy, const int ncols, float* __restrict__ out, const int accumulate)
{
	__shared__ float sh[32][33];
	const int cx = threadIdx.x & 31, yl = threadIdx.x >> 5;
	const int col = blockIdx.x * 32 + cx;
	float acc = 0.f;
	if (col < ncols)
	{
		int y = yl;
		for (; y + 96 < gy; y += 128)
		{
			const float a0 = part[(size_t)y * ncols + col], a1 = part[(size_t)(y + 32) * ncols + col], a2 = part[(size_t)(y + 64) * ncols + col], a3 = part[(size_t)(y + 96) * ncols + col];
			acc += (a0 + a1) + (a2 + a3);
		}
		for (; y < gy; y += 32)
			acc += part[(size_t)y * ncols + col];
	}
	sh[yl][cx] = acc;
	__syncthreads();
	if (yl == 0 && col < ncols)
	{
		float t = 0.f;
#pragma unroll
		for (int j = 0; j < 32; j++)
			t += sh[j][cx];
		out[col] = accumulate ? out[col] + t : t;
	}
}
size_t colsum_workspace_bytes(int cols) { return ((size_t)sm_count() * 8 + 8) * (size_t)((cols + 3) / 4 * 4) * sizeof(float); }
static int colsum_f32(cudaStream_t s, const float* g, size_t rows, int cols, long long ld, float* out, int accumulate, void* workspace)
{
	if (cols <= 0)
		return 0;
	const bool vec = cols % 4 == 0 && ld % 4 == 0 && (((uintptr_t)g) & 15) == 0;
	if (!accumulate && !(vec && workspace && rows > 0))
	{
		const cudaError_t e = cudaMemsetAsync(out, 0, (size_t)cols * 4, s);
		if (e != cudaSuccess)
		{
			set_last_error("memset(colsum)", e);
			return -1;
		}
	}
	if (rows == 0)
		return 0;
	if (vec)
	{
		const int cols4 = cols / 4;
		int cpb = 1;
		while (cpb < cols4 && cpb < 256)
			cpb <<= 1;
		const int rpi = 256 / cpb;
		const int gx = (cols4 + cpb - 1) / cpb;
		size_t gy = (rows + (size_t)rpi * 16 - 1) / ((size_t)rpi * 16);
		const size_t cap = (size_t)(sm_count() * 8 + gx - 1) / gx;
		if (gy > cap)
			gy = cap;
		if (gy < 1)
			gy = 1;
		colsum_vec_kernel<<<dim3(gx, (unsigned)gy), 256, 0, s>>>((const float4*)g, rows, cols4, ld / 4, out, (float*)workspace, cpb);
		if (launched("colsum_vec"))
			return -1;
		if (workspace)
		{
			colsum_partials_kernel<<<(cols + 31) / 32, 1024, 0, s>>>((const float*)workspace, (int)gy, cols, out, accumulate);
			return launched("colsum_partials");
		}
		return 0;
	}
	const int cpb = cols >= 256 ? 256 : (cols >= 128 ? 128 : (cols >= 64 ? 64 : 32));
	const int rpi = 256 / cpb;
	const int gx = (cols + cpb - 1) / cpb;
	size_t gy = (rows + rpi * 8 - 1) / ((size_t)rpi * 8);
	const size_t cap = (size_t)(sm_count() * 4 + gx - 1) / gx;
	if (gy > cap)
		gy = cap;
	if (gy < 1)
		gy = 1;
	colsum_kernel<<<dim3(gx, (unsigned)gy), 256, 256 * sizeof(float), s>>>(g, rows, cols, ld, out, cpb);
	return launched("colsum");
}

// generic <= 4-d reduction to a broadcast shape: one thread block per output element (small outputs only)
struct Reduce4 {
	int adim[4], astride[4], rdim[4];
};
__global__ void reduce_sum_kernel(const float* __restrict__ a, float* __restrict__ out, const Reduce4 d, const float scale, const int accumulate)
{
	__shared__ float sh[32];
	// output index -> (o0, o1, o2, o3)
	int o = blockIdx.x;
	int oi[4];
	for (int k = 3; k >= 0; k--)
		oi[k] = o % d.rdim[k], o /= d.rdim[k];
	int ext[4];
	size_t total = 1;
	for (int k = 0; k < 4; k++)
		ext[k] = d.rdim[k] == 1 ? d.adim[k] : 1, total *= ext[k];
	float acc = 0.f;
	for (size_t i = threadIdx.x; i < total; i += blockDim.x)
	{
		size_t r = i;
		size_t off = 0;
		for (int k = 3; k >= 0; k--)
		{
			const int ik = (int)(r % ext[k]);
			r /= ext[k];
			off += (size_t)(d.rdim[k] == 1 ? ik : oi[k]) * d.astride[k];
		}
		acc += a[off];
	}
	acc = block_sum(acc, sh);
	if (threadIdx.x == 0)
		out[blockIdx.x] = accumulate ? out[blockIdx.x] + acc * scale : acc * scale;
}
int reduce_sum_bcast_f32(cudaStream_t s, const float* a, const int* adim, const int* astride, float* out, const int* rdim, float scale, int accumulate)
{
	Reduce4 d;
	size_t outs = 1;
	for (int i = 0; i < 4; i++)
		d.adim[i] = adim[i] > 0 ? adim[i] : 1, d.astride[i] = astride[i], d.rdim[i] = rdim[i] > 0 ? rdim[i] : 1, outs *= d.rdim[i];
	if (outs > 0x7fffffff)
		return 1;
	reduce_sum_kernel<<<(unsigned)outs, 256, 0, s>>>(a, out, d, scale, accumulate);
	return launched("reduce_sum");
}

// =============================================================================================== pooling (NHWC)
// pool/ccv_nnc_max_pool_cpu_ref.c:13-59, pool/ccv_nnc_avg_pool_cpu_ref.c:13-58: the window is clipped to the input
// (SET_BORDER_OFFSET_SIZE_FOR, ccv_nnc_internal.h:209-213); the average divides by the clipped window size.
// VEC channels of one pixel: one 16-byte access when VEC is the type's vector width, a scalar access when VEC == 1
template <typename T, int VEC>
__device__ __forceinline__ void pool_load(const T* p, float (&v)[VEC])
{
	if constexpr (VEC == 1)
		v[0] = ldf(p);
	else
		ldv(p, v);
}
template <typename T, int VEC>
__device__ __forceinline__ void pool_store(T* p, const float (&v)[VEC])
{
	if constexpr (VEC == 1)
		stf(p, v[0]);
	else
		stv(p, v);
}
template <typename T, int VEC, int IS_MAX>
__global__ void pool_fwd_kernel(const PoolGeom g, const T* __restrict__ a, T* __restrict__ b)
{
	const int CV = g.C / VEC;
	const size_t total = (size_t)g.N * g.P * g.Q * CV;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		int c, q, p, n;
		if (total <= 0xffffffffull)
		{
			// 32-bit index math (a 64-bit divide costs ~5x a 32-bit one and there are three per element)
			const unsigned ii = (unsigned)i;
			unsigned r = ii / (unsigned)CV;
			c = (int)(ii - r * (unsigned)CV) * VEC;
			const unsigned r2 = r / (unsigned)g.Q;
			q = (int)(r - r2 * (unsigned)g.Q);
			n = (int)(r2 / (unsigned)g.P);
			p = (int)(r2 - (unsigned)n * (unsigned)g.P);
		} else {
			c = (int)(i % CV) * VEC;
			size_t r = i / CV;
			q = (int)(r % g.Q);
			r /= g.Q;
			p = (int)(r % g.P);
			n = (int)(r / g.P);
		}
		const int h0 = max(p * g.stride_h - g.pad_h, 0), h1 = min(p * g.stride_h - g.pad_h + g.R, g.H);
		const int w0 = max(q * g.stride_w - g.pad_w, 0), w1 = min(q * g.stride_w - g.pad_w + g.S, g.W);
		float v[VEC];
#pragma unroll
		for (int k = 0; k < VEC; k++)
			v[k] = IS_MAX ? -FLT_MAX : 0.f;
		for (int h = h0; h < h1; h++)
			for (int w = w0; w < w1; w++)
			{
				const T* ap = a + n * g.an + h * g.ah + w * g.aw + c;
				float x[VEC];
				pool_load<T, VEC>(ap, x);
#pragma unroll
				for (int k = 0; k < VEC; k++)
					v[k] = IS_MAX ? fmaxf(v[k], x[k]) : v[k] + x[k];
			}
		if (!IS_MAX)
		{
			const float inv = (float)((h1 - h0) * (w1 - w0));
#pragma unroll
			for (int k = 0; k < VEC; k++)
				v[k] = v[k] / inv;
		}
		T* bp = b + n * g.bn + p * g.bh + q * g.bw + c;
		pool_store<T, VEC>(bp, v);
	}
}
template <typename T>
static bool pool_vec_ok(const PoolGeom& g, const T* a, const T* b)
{
	constexpr int W = Vec16<T>::W; // channels per 16-byte access
	return g.C % W == 0 && aligned_v16(a) && aligned_v16(b) && g.aw % W == 0 && g.ah % W == 0 && g.an % W == 0 && g.bw % W == 0 && g.bh % W == 0 && g.bn % W == 0;
}
template <typename T, int IS_MAX>
static int pool_fwd_t(cudaStream_t s, const PoolGeom& g, const T* a, T* b)
{
	const size_t total = (size_t)g.N * g.P * g.Q * g.C;
	if (total == 0)
		return 0;
	if (pool_vec_ok(g, a, (const T*)b))
		pool_fwd_kernel<T, Vec16<T>::W, IS_MAX><<<grid_for(total / Vec16<T>::W, 256, 8), 256, 0, s>>>(g, a, b);
	else
		pool_fwd_kernel<T, 1, IS_MAX><<<grid_for(total, 256, 8), 256, 0, s>>>(g, a, b);
	return launched(IS_MAX ? "pool_max_fwd" : "pool_avg_fwd");
}
int pool_max_fwd_f32(cudaStream_t s, const PoolGeom& g, const float* a, float* b) { return pool_fwd_t<float, 1>(s, g, a, b); }
int pool_avg_fwd_f32(cudaStream_t s, const PoolGeom& g, const float* a, float* b) { return pool_fwd_t<float, 0>(s, g, a, b); }
int pool_max_fwd_16(cudaStream_t s, int kind, const PoolGeom& g, const void* a, void* b)
{
	return kind == 1 ? pool_fwd_t<__nv_bfloat16, 1>(s, g, (const __nv_bfloat16*)a, (__nv_bfloat16*)b) : pool_fwd_t<__half, 1>(s, g, (const __half*)a, (__half*)b);
}
int pool_avg_fwd_16(cudaStream_t s, int kind, const PoolGeom& g, const void* a, void* b)
{
	return kind == 1 ? pool_fwd_t<__nv_bfloat16, 0>(s, g, (const __nv_bfloat16*)a, (__nv_bfloat16*)b) : pool_fwd_t<__half, 0>(s, g, (const __half*)a, (__half*)b);
}
// Backward as a gather over input positions (no atomics): input (h, w) collects from every window that covers it.
// max: pool/ccv_nnc_max_pool_cpu_ref.c:61-139 -- every position equal to the window max receives the gradient.
// avg: pool/ccv_nnc_avg_pool_cpu_ref.c:60-110 -- gradient / clipped window size.
template <typename T, int VEC, int IS_MAX>
__global__ void pool_bwd_kernel(const PoolGeom g, const T* __restrict__ gb, const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ ga)
{
	const int CV = g.C / VEC;
	const size_t total = (size_t)g.N * g.H * g.W * CV;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		int c, w, h, n;
		if (total <= 0xffffffffull)
		{
			const unsigned ii = (unsigned)i;
			unsigned r = ii / (unsigned)CV;
			c = (int)(ii - r * (unsigned)CV) * VEC;
			const unsigned r2 = r / (unsigned)g.W;
			w = (int)(r - r2 * (unsigned)g.W);
			n = (int)(r2 / (unsigned)g.H);
			h = (int)(r2 - (unsigned)n * (unsigned)g.H);
		} else {
			c = (int)(i % CV) * VEC;
			size_t r = i / CV;
			w = (int)(r % g.W);
			r /= g.W;
			h = (int)(r % g.H);
			n = (int)(r / g.H);
		}
		if (!IS_MAX && VEC > 1 && g.R == g.stride_h && g.S == g.stride_w && g.pad_h == 0 && g.pad_w == 0 && g.P * g.stride_h <= g.H && g.Q * g.stride_w <= g.W)
		{
			// non-overlapping windows (the 2 x 2 / 2 shortcut pools, the global pool): every input position belongs to at most one
			// window, and with P * R <= H, Q * S <= W (no end border) none is clipped -> one load, one divide per lane, one store
			const int p = h / g.stride_h, q = w / g.stride_w;
			float o[VEC];
#pragma unroll
			for (int k = 0; k < VEC; k++)
				o[k] = 0.f;
			if (p < g.P && q < g.Q)
			{
				pool_load<T, VEC>(gb + n * g.bn + p * g.bh + q * g.bw + c, o);
				const float inv = (float)(g.R * g.S);
#pragma unroll
				for (int k = 0; k < VEC; k++)
					o[k] = o[k] / inv;
			}
			pool_store<T, VEC>(ga + n * g.an + h * g.ah + w * g.aw + c, o);
			continue;
		}
		// windows p with p * stride - pad <= h < p * stride - pad + R
		const int p_lo = max((h + g.pad_h - g.R + g.stride_h) / g.stride_h, 0), p_hi = min((h + g.pad_h) / g.stride_h, g.P - 1);
		const int q_lo = max((w + g.pad_w - g.S + g.stride_w) / g.stride_w, 0), q_hi = min((w + g.pad_w) / g.stride_w, g.Q - 1);
		float x[VEC], acc[VEC];
#pragma unroll
		for (int k = 0; k < VEC; k++)
			acc[k] = 0.f, x[k] = 0.f;
		if (IS_MAX)
		{
			pool_load<T, VEC>(a + n * g.an + h * g.ah + w * g.aw + c, x);
		}
		for (int p = p_lo; p <= p_hi; p++)
		{
			if (h + g.pad_h - g.R >= p * g.stride_h) // (h + pad - R + stride) / stride rounds toward zero for negatives
				continue;
			const int h0 = max(p * g.stride_h - g.pad_h, 0), h1 = min(p * g.stride_h - g.pad_h + g.R, g.H);
			for (int q = q_lo; q <= q_hi; q++)
			{
				if (w + g.pad_w - g.S >= q * g.stride_w)
					continue;
				const size_t o = n * g.bn + p * g.bh + q * g.bw + c;
				float gv[VEC], bv[VEC];
				pool_load<T, VEC>(gb + o, gv);
				if (IS_MAX)
					pool_load<T, VEC>(b + o, bv);
				if (IS_MAX)
				{
#pragma unroll
					for (int k = 0; k < VEC; k++)
						if (x[k] == bv[k])
							acc[k] += gv[k];
				} else {
					const int w0 = max(q * g.stride_w - g.pad_w, 0), w1 = min(q * g.stride_w - g.pad_w + g.S, g.W);
					const float inv = (float)((h1 - h0) * (w1 - w0));
#pragma unroll
					for (int k = 0; k < VEC; k++)
						acc[k] += gv[k] / inv;
				}
			}
		}
		T* hp = ga + n * g.an + h * g.ah + w * g.aw + c;
		pool_store<T, VEC>(hp, acc);
	}
}
template <typename T>
static int pool_max_bwd_t(cudaStream_t s, const PoolGeom& g, const T* grad_b, const T* a, const T* b, T* grad_a)
{
	const size_t total = (size_t)g.N * g.H * g.W * g.C;
	if (total == 0)
		return 0;
	if (pool_vec_ok(g, a, b) && aligned_v16(grad_b) && aligned_v16(grad_a))
		pool_bwd_kernel<T, Vec16<T>::W, 1><<<grid_for(total / Vec16<T>::W, 256, 8), 256, 0, s>>>(g, grad_b, a, b, grad_a);
	else
		pool_bwd_kernel<T, 1, 1><<<grid_for(total, 256, 8), 256, 0, s>>>(g, grad_b, a, b, grad_a);
	return launched("pool_max_bwd");
}
// Average-pool backward when the windows tile the input exactly (window = stride, no padding, H = P * R, W = Q * S: the 2 x 2 / 2
// shortcut pools and the global pool of a ResNet): one thread per OUTPUT gradient group -- one 16-byte load, one multiply per
// element, R * S 16-byte stores -- instead of one thread (and three integer divisions) per input group.
// MASK = 1: the pool is the shortcut of a residual block whose input gradient is the sum of both branches behind a ReLU: the store is
// ga = y > 0 ? add + v : 0 with add (the other branch's gradient) and y (the block input) laid out as ga, v rounded to T first as a
// stored pool gradient would be.  add may be ga itself: every element is read before the same thread writes it, so ga is not
// __restrict__.
template <typename T, int MASK>
__global__ void __launch_bounds__(256) avgpool_bwd_tiles_kernel(const PoolGeom g, const T* __restrict__ gb, T* ga, const T* add, const T* y)
{
	constexpr int W = Vec16<T>::W;
	const unsigned CW = (unsigned)g.C / W;
	const size_t total = (size_t)g.N * g.P * g.Q * CW;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		const size_t r = i / CW;
		const int c = (int)(i - r * CW) * W;
		const size_t r2 = r / (unsigned)g.Q;
		const int q = (int)(r - r2 * (unsigned)g.Q);
		const int n = (int)(r2 / (unsigned)g.P), p = (int)(r2 - (size_t)n * (unsigned)g.P);
		float v[W];
		ldv(gb + n * g.bn + p * g.bh + q * g.bw + c, v);
#pragma unroll
		for (int k = 0; k < W; k++)
			v[k] = v[k] / (float)(g.R * g.S); // the reference divides (pool/ccv_nnc_avg_pool_cpu_ref.c:60-110); keep its rounding
		const long long base = n * g.an + (long long)p * g.R * g.ah + (long long)q * g.S * g.aw + c;
		if (MASK)
#pragma unroll
			for (int k = 0; k < W; k++)
				v[k] = rnd(gb, v[k]);
		for (int dh = 0; dh < g.R; dh++)
			for (int dw = 0; dw < g.S; dw++)
			{
				const long long o = base + dh * g.ah + dw * g.aw;
				if (MASK)
				{
					float rv[W], yv[W], ov[W];
					ldv(add + o, rv), ldv(y + o, yv);
#pragma unroll
					for (int k = 0; k < W; k++)
						ov[k] = yv[k] > 0.f ? rv[k] + v[k] : 0.f;
					stv(ga + o, ov);
				} else
					stv(ga + o, v);
			}
	}
}
// the tiles kernel's geometry: every window lies inside the input and no two overlap
template <typename T>
static bool avgpool_tiles_ok(const PoolGeom& g, const T* grad_b, const T* grad_a)
{
	constexpr int W = Vec16<T>::W;
	return g.R == g.stride_h && g.S == g.stride_w && g.pad_h == 0 && g.pad_w == 0 && g.H == g.P * g.R && g.W == g.Q * g.S && g.C % W == 0 && aligned_v16(grad_b) && aligned_v16(grad_a) &&
		g.aw % W == 0 && g.ah % W == 0 && g.an % W == 0 && g.bw % W == 0 && g.bh % W == 0 && g.bn % W == 0;
}
template <typename T>
static int pool_avg_bwd_t(cudaStream_t s, const PoolGeom& g, const T* grad_b, T* grad_a)
{
	const size_t total = (size_t)g.N * g.H * g.W * g.C;
	if (total == 0)
		return 0;
	constexpr int W = Vec16<T>::W;
	if (avgpool_tiles_ok(g, grad_b, grad_a))
	{
		avgpool_bwd_tiles_kernel<T, 0><<<grid_for((size_t)g.N * g.P * g.Q * (g.C / W), 256, 8), 256, 0, s>>>(g, grad_b, grad_a, (const T*)0, (const T*)0);
		return launched("pool_avg_bwd");
	}
	if (pool_vec_ok(g, (const T*)grad_a, grad_b))
		pool_bwd_kernel<T, Vec16<T>::W, 0><<<grid_for(total / Vec16<T>::W, 256, 8), 256, 0, s>>>(g, grad_b, (const T*)0, (const T*)0, grad_a);
	else
		pool_bwd_kernel<T, 1, 0><<<grid_for(total, 256, 8), 256, 0, s>>>(g, grad_b, (const T*)0, (const T*)0, grad_a);
	return launched("pool_avg_bwd");
}
// grad_a = y > 0 ? r + avgpool_backward(grad_b) : 0 in one pass; r and y are addressed with grad_a's strides.  1 (nothing launched)
// when the geometry is not the tiles kernel's
template <typename T>
static int pool_avg_bwd_add_relu_t(cudaStream_t s, const PoolGeom& g, const T* grad_b, const T* r, const T* y, T* grad_a)
{
	if (!avgpool_tiles_ok(g, grad_b, grad_a) || !aligned_v16(r) || !aligned_v16(y))
		return 1;
	if ((size_t)g.N * g.H * g.W * g.C == 0)
		return 0;
	avgpool_bwd_tiles_kernel<T, 1><<<grid_for((size_t)g.N * g.P * g.Q * (g.C / Vec16<T>::W), 256, 8), 256, 0, s>>>(g, grad_b, grad_a, r, y);
	return launched("pool_avg_bwd_add_relu") ? -1 : 0;
}
int pool_avg_bwd_add_relu(cudaStream_t s, int kind, const PoolGeom& g, const void* grad_b, const void* r, const void* y, void* grad_a)
{
	if (kind == 0)
		return pool_avg_bwd_add_relu_t<float>(s, g, (const float*)grad_b, (const float*)r, (const float*)y, (float*)grad_a);
	if (kind == 1)
		return pool_avg_bwd_add_relu_t<__nv_bfloat16>(s, g, (const __nv_bfloat16*)grad_b, (const __nv_bfloat16*)r, (const __nv_bfloat16*)y, (__nv_bfloat16*)grad_a);
	return pool_avg_bwd_add_relu_t<__half>(s, g, (const __half*)grad_b, (const __half*)r, (const __half*)y, (__half*)grad_a);
}
int pool_max_bwd_f32(cudaStream_t s, const PoolGeom& g, const float* grad_b, const float* a, const float* b, float* grad_a) { return pool_max_bwd_t<float>(s, g, grad_b, a, b, grad_a); }
int pool_avg_bwd_f32(cudaStream_t s, const PoolGeom& g, const float* grad_b, float* grad_a) { return pool_avg_bwd_t<float>(s, g, grad_b, grad_a); }
int pool_max_bwd_16(cudaStream_t s, int kind, const PoolGeom& g, const void* grad_b, const void* a, const void* b, void* grad_a)
{
	return kind == 1 ? pool_max_bwd_t<__nv_bfloat16>(s, g, (const __nv_bfloat16*)grad_b, (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, (__nv_bfloat16*)grad_a)
		: pool_max_bwd_t<__half>(s, g, (const __half*)grad_b, (const __half*)a, (const __half*)b, (__half*)grad_a);
}
int pool_avg_bwd_16(cudaStream_t s, int kind, const PoolGeom& g, const void* grad_b, void* grad_a)
{
	return kind == 1 ? pool_avg_bwd_t<__nv_bfloat16>(s, g, (const __nv_bfloat16*)grad_b, (__nv_bfloat16*)grad_a) : pool_avg_bwd_t<__half>(s, g, (const __half*)grad_b, (__half*)grad_a);
}

// =============================================================================================== softmax / losses
// softmax/ccv_nnc_softmax_cpu_ref.c:13-40: per row, b = exp(a - max) / sum; one block per row.  b may be a (in place), so neither
// pointer is __restrict__: each element is read before the same thread writes it
__global__ void softmax_fwd_kernel(const float* a, float* b, const int count)
{
	__shared__ float sh[32];
	const float* ap = a + (size_t)blockIdx.x * count;
	float* bp = b + (size_t)blockIdx.x * count;
	float m = -FLT_MAX;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		m = fmaxf(m, ap[j]);
	m = block_max(m, sh);
	float sum = 0.f;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
	{
		const float e = expf(ap[j] - m);
		bp[j] = e;
		sum += e;
	}
	sum = block_sum(sum, sh);
	const float inv = 1.f / sum;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		bp[j] *= inv;
}
static int softmax_threads(int count) { return count >= 1024 ? 256 : (count >= 256 ? 128 : (count >= 64 ? 64 : 32)); }
int softmax_fwd_f32(cudaStream_t s, const float* a, float* b, int batch, int count)
{
	if (batch <= 0 || count <= 0)
		return 0;
	softmax_fwd_kernel<<<batch, softmax_threads(count), 0, s>>>(a, b, count);
	return launched("softmax_fwd");
}
// softmax/ccv_nnc_softmax_cpu_ref.c:42-75: h = (g - sum(g * b)) * b; h may be g (in place)
__global__ void softmax_bwd_kernel(const float* g, const float* __restrict__ b, float* h, const int count)
{
	__shared__ float sh[32];
	const size_t o = (size_t)blockIdx.x * count;
	float sum = 0.f;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		sum += g[o + j] * b[o + j];
	sum = block_sum(sum, sh);
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		h[o + j] = (g[o + j] - sum) * b[o + j];
}
int softmax_bwd_f32(cudaStream_t s, const float* g, const float* b, float* h, int batch, int count)
{
	if (batch <= 0 || count <= 0)
		return 0;
	softmax_bwd_kernel<<<batch, softmax_threads(count), 0, s>>>(g, b, h, count);
	return launched("softmax_bwd");
}
__device__ __forceinline__ int label_of(const void* label, const int kind, const int i)
{
	return kind == 1 ? reinterpret_cast<const int*>(label)[i] : (int)(reinterpret_cast<const float*>(label)[i] + 0.5f);
}
// loss/ccv_nnc_categorical_crossentropy_cpu_ref.c:13-105
__global__ void cce_fwd_kernel(const float* __restrict__ a, const void* __restrict__ label, const int kind, float* __restrict__ c, const int count, const float trim0, const float trim1)
{
	__shared__ float sh[32];
	const int i = blockIdx.x;
	const float* ap = a + (size_t)i * count;
	float p = 0.f;
	if (kind == 2)
	{
		const float* bp = reinterpret_cast<const float*>(label) + (size_t)i * count;
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			p += -bp[j] * logf(ap[j]);
	} else {
		const int l = label_of(label, kind, i);
		if (trim0 == 0.f && trim1 == 1.f)
		{
			if (threadIdx.x == 0)
				c[i] = -logf(ap[l]);
			return;
		}
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			p += -(j == l ? trim1 : trim0) * logf(ap[j]);
	}
	p = block_sum(p, sh);
	if (threadIdx.x == 0)
		c[i] = p;
}
int cce_fwd_f32(cudaStream_t s, const float* a, const void* label, int label_kind, float* c, int batch, int count, float trim0, float trim1)
{
	if (batch <= 0 || count <= 0)
		return 0;
	cce_fwd_kernel<<<batch, softmax_threads(count), 0, s>>>(a, label, label_kind, c, count, trim0, trim1);
	return launched("cce_fwd");
}
// loss/ccv_nnc_categorical_crossentropy_cpu_ref.c:107-300: h = -g * t / a (g == NULL means 1)
__global__ void cce_bwd_kernel(const float* __restrict__ g, const float* __restrict__ a, const void* __restrict__ label, const int kind, float* __restrict__ h, const int count, const float trim0, const float trim1)
{
	const int i = blockIdx.x;
	const float gp = g ? g[i] : 1.f;
	const float* ap = a + (size_t)i * count;
	float* hp = h + (size_t)i * count;
	if (kind == 2)
	{
		const float* bp = reinterpret_cast<const float*>(label) + (size_t)i * count;
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			hp[j] = -gp * bp[j] / ap[j];
		return;
	}
	const int l = label_of(label, kind, i);
	if (trim0 == 0.f && trim1 == 1.f)
	{
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			hp[j] = j == l ? -gp / ap[j] : 0.f;
	} else {
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			hp[j] = -gp * (j == l ? trim1 : trim0) / ap[j];
	}
}
int cce_bwd_f32(cudaStream_t s, const float* g, const float* a, const void* label, int label_kind, float* h, int batch, int count, float trim0, float trim1)
{
	if (batch <= 0 || count <= 0)
		return 0;
	cce_bwd_kernel<<<batch, softmax_threads(count), 0, s>>>(g, a, label, label_kind, h, count, trim0, trim1);
	return launched("cce_bwd");
}
// softmax_loss/ccv_nnc_softmax_crossentropy_cpu_ref.c:13-170: d = softmax(a); c = sum_j t_j * (max - a_j).
// (The reference's "loss" deliberately leaves out log(sum exp): it is assigned before the exponentials, :46,:71,:98.)
// d may be a (softmax_loss/ccv_nnc_softmax_crossentropy.c:17-20 lets the graph allocator alias them), so neither is __restrict__ and
// the loss term of a_j is taken in the exponential pass, from the value in a register, before d_j overwrites it
__global__ void softmax_cce_fwd_kernel(const float* a, const void* __restrict__ label, const int kind, float* __restrict__ c, float* d, const int count, const float trim0, const float trim1)
{
	__shared__ float sh[32];
	const int i = blockIdx.x;
	const float* ap = a + (size_t)i * count;
	float* dp = d + (size_t)i * count;
	float m = -FLT_MAX;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		m = fmaxf(m, ap[j]);
	m = block_max(m, sh);
	const int l = kind == 2 ? -1 : label_of(label, kind, i);
	const float* bp = kind == 2 ? reinterpret_cast<const float*>(label) + (size_t)i * count : 0;
	float sum = 0.f, p = 0.f;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
	{
		const float x = ap[j];
		if (c)
		{
			const float t = kind == 2 ? bp[j] : (j == l ? trim1 : trim0);
			if (t != 0.f)
				p += t * (m - x);
		}
		const float e = expf(x - m);
		dp[j] = e;
		sum += e;
	}
	sum = block_sum(sum, sh);
	const float inv = 1.f / sum;
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		dp[j] *= inv;
	if (c)
	{
		p = block_sum(p, sh);
		if (threadIdx.x == 0)
			c[i] = p;
	}
}
int softmax_cce_fwd_f32(cudaStream_t s, const float* a, const void* label, int label_kind, float* c, float* d, int batch, int count, float trim0, float trim1)
{
	if (batch <= 0 || count <= 0)
		return 0;
	softmax_cce_fwd_kernel<<<batch, softmax_threads(count), 0, s>>>(a, label, label_kind, c, d, count, trim0, trim1);
	return launched("softmax_cce_fwd");
}
// softmax_loss/ccv_nnc_softmax_crossentropy_cpu_ref.c:172-340: h = g * (d - t); g == NULL means 1.  h may be d
// (softmax_loss/ccv_nnc_softmax_crossentropy.c:31-40)
__global__ void softmax_cce_bwd_kernel(const float* __restrict__ g, const void* __restrict__ label, const int kind, const float* d, float* h, const int count, const float trim0, const float trim1)
{
	const int i = blockIdx.x;
	const float gp = g ? g[i] : 1.f;
	const float* dp = d + (size_t)i * count;
	float* hp = h + (size_t)i * count;
	if (kind == 2)
	{
		const float* bp = reinterpret_cast<const float*>(label) + (size_t)i * count;
		for (int j = threadIdx.x; j < count; j += blockDim.x)
			hp[j] = gp * (dp[j] - bp[j]);
		return;
	}
	const int l = label_of(label, kind, i);
	for (int j = threadIdx.x; j < count; j += blockDim.x)
		hp[j] = gp * (dp[j] - (j == l ? trim1 : trim0));
}
int softmax_cce_bwd_f32(cudaStream_t s, const float* g, const void* label, int label_kind, const float* d, float* h, int batch, int count, float trim0, float trim1)
{
	if (batch <= 0 || count <= 0)
		return 0;
	softmax_cce_bwd_kernel<<<batch, softmax_threads(count), 0, s>>>(g, label, label_kind, d, h, count, trim0, trim1);
	return launched("softmax_cce_bwd");
}

// =============================================================================================== SGD
// sgd/ccv_nnc_sgd_cpu_ref.c:16-126.  b may be a and n may be m (sgd/ccv_nnc_sgd.c:14-19: how models call it), so those are not
// __restrict__
template <int VEC>
__global__ void sgd_kernel(const void* __restrict__ g, const int g_kind, const float* a, const float* m, float* b, float* n, const size_t count, const int nesterov, const float rate, const float scale, const float decay, const float momentum, const float inv_dampening)
{
	const size_t cv = VEC == 4 ? count >> 2 : count;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < cv; i += (size_t)gridDim.x * blockDim.x)
	{
		float gv[VEC], av[VEC], mv[VEC], bv[VEC], nv[VEC];
		if (VEC == 4)
		{
			// the gradient may be 16-bit while parameters and momenta are fp32 (the reference's mixed form, sgd/gpu/ccv_nnc_sgd_gpu_ref.cu:71-74)
			const float4 t = g_kind == 0 ? ld4(reinterpret_cast<const float*>(g) + i * 4) : g_kind == 1 ? ld4(reinterpret_cast<const __nv_bfloat16*>(g) + i * 4) : ld4(reinterpret_cast<const __half*>(g) + i * 4);
			const float4 u = reinterpret_cast<const float4*>(a)[i], w = reinterpret_cast<const float4*>(m)[i];
			gv[0] = t.x, gv[1 % VEC] = t.y, gv[2 % VEC] = t.z, gv[3 % VEC] = t.w;
			av[0] = u.x, av[1 % VEC] = u.y, av[2 % VEC] = u.z, av[3 % VEC] = u.w;
			mv[0] = w.x, mv[1 % VEC] = w.y, mv[2 % VEC] = w.z, mv[3 % VEC] = w.w;
		} else
			gv[0] = ld_kind(g, i, g_kind), av[0] = a[i], mv[0] = m[i];
#pragma unroll
		for (int j = 0; j < VEC; j++)
		{
			if (nesterov)
			{
				float grad = scale * gv[j];
				const float mom = nv[j] = momentum * mv[j] + grad + decay * av[j];
				grad += momentum * mom;
				bv[j] = av[j] - rate * grad;
			} else {
				const float mom = nv[j] = momentum * mv[j] + inv_dampening * (scale * gv[j] + decay * av[j]);
				bv[j] = av[j] - rate * mom;
			}
		}
		if (VEC == 4)
		{
			reinterpret_cast<float4*>(b)[i] = make_float4(bv[0], bv[1 % VEC], bv[2 % VEC], bv[3 % VEC]);
			reinterpret_cast<float4*>(n)[i] = make_float4(nv[0], nv[1 % VEC], nv[2 % VEC], nv[3 % VEC]);
		} else
			b[i] = bv[0], n[i] = nv[0];
	}
}
static inline bool g_aligned(const void* g, int g_kind) { return (((uintptr_t)g) & (g_kind ? 7 : 15)) == 0; }
int sgd_any(cudaStream_t s, int g_kind, const void* g, const float* a, const float* m, float* b, float* n, size_t count, int nesterov, float rate, float scale, float decay, float momentum, float dampening)
{
	if (count == 0)
		return 0;
	const float inv_dampening = 1.f - dampening;
	if (count % 4 == 0 && g_aligned(g, g_kind) && aligned16(a) && aligned16(m) && aligned16(b) && aligned16(n))
		sgd_kernel<4><<<grid_for(count / 4, 256, 8), 256, 0, s>>>(g, g_kind, a, m, b, n, count, nesterov, rate, scale, decay, momentum, inv_dampening);
	else
		sgd_kernel<1><<<grid_for(count, 256, 8), 256, 0, s>>>(g, g_kind, a, m, b, n, count, nesterov, rate, scale, decay, momentum, inv_dampening);
	return launched("sgd");
}

// Many SGD commands with the same hyper-parameters in one launch (the per-parameter SGD nodes of a model are a run of ~200
// small tensors): the tensor table travels in the kernel parameters (<= SGD_MULTI_MAX tensors per launch), a block owns
// one 4096-element chunk of one tensor.  Same arithmetic as sgd_kernel.
constexpr int SGD_MULTI_MAX = 32;
constexpr unsigned SGD_MULTI_CHUNK = 4096;
struct SgdMulti {
	const void* g[SGD_MULTI_MAX];
	int g_kind;
	const float* a[SGD_MULTI_MAX];
	const float* m[SGD_MULTI_MAX];
	float* b[SGD_MULTI_MAX];
	float* n[SGD_MULTI_MAX];
	unsigned count[SGD_MULTI_MAX];
	unsigned block_start[SGD_MULTI_MAX + 1];
	int tensors;
};
__global__ void __launch_bounds__(256) sgd_multi_kernel(const __grid_constant__ SgdMulti t, const int nesterov, const float rate, const float scale, const float decay, const float momentum, const float inv_dampening)
{
	int ti = 0;
	while (ti + 1 < t.tensors && blockIdx.x >= t.block_start[ti + 1])
		ti++;
	const unsigned base = (blockIdx.x - t.block_start[ti]) * SGD_MULTI_CHUNK;
	const unsigned count = t.count[ti];
	const void* const g = t.g[ti];
	const float* const a = t.a[ti];
	const float* const m = t.m[ti];
	float* const b = t.b[ti];
	float* const n = t.n[ti];
#pragma unroll
	for (int it = 0; it < 4; it++)
	{
		const unsigned i = base + (it * 256 + threadIdx.x) * 4;
		if (i >= count)
			break;
		const float4 gv = t.g_kind == 0 ? ld4(reinterpret_cast<const float*>(g) + i) : t.g_kind == 1 ? ld4(reinterpret_cast<const __nv_bfloat16*>(g) + i) : ld4(reinterpret_cast<const __half*>(g) + i);
		const float4 av = *reinterpret_cast<const float4*>(a + i), mv = *reinterpret_cast<const float4*>(m + i);
		const float gs[4] = { gv.x, gv.y, gv.z, gv.w }, as[4] = { av.x, av.y, av.z, av.w }, ms[4] = { mv.x, mv.y, mv.z, mv.w };
		float bs[4], ns[4];
#pragma unroll
		for (int j = 0; j < 4; j++)
		{
			if (nesterov)
			{
				float grad = scale * gs[j];
				const float mom = ns[j] = momentum * ms[j] + grad + decay * as[j];
				grad += momentum * mom;
				bs[j] = as[j] - rate * grad;
			} else {
				const float mom = ns[j] = momentum * ms[j] + inv_dampening * (scale * gs[j] + decay * as[j]);
				bs[j] = as[j] - rate * mom;
			}
		}
		*reinterpret_cast<float4*>(b + i) = make_float4(bs[0], bs[1], bs[2], bs[3]);
		*reinterpret_cast<float4*>(n + i) = make_float4(ns[0], ns[1], ns[2], ns[3]);
	}
}
int sgd_multi_any(cudaStream_t s, int tensors, int g_kind, const void* const* g, const float* const* a, const float* const* m, float* const* b, float* const* n, const size_t* counts, int nesterov, float rate, float scale, float decay, float momentum, float dampening)
{
	const float inv_dampening = 1.f - dampening;
	int i = 0;
	while (i < tensors)
	{
		SgdMulti t;
		t.tensors = 0, t.g_kind = g_kind;
		unsigned blocks = 0;
		while (i < tensors && t.tensors < SGD_MULTI_MAX)
		{
			const bool vec = counts[i] % 4 == 0 && counts[i] < 0xffffffffull && g_aligned(g[i], g_kind) && aligned16(a[i]) && aligned16(m[i]) && aligned16(b[i]) && aligned16(n[i]);
			if (!vec)
			{
				if (t.tensors > 0)
					break; // flush what is batched, then do this one on its own
				if (sgd_any(s, g_kind, g[i], a[i], m[i], b[i], n[i], counts[i], nesterov, rate, scale, decay, momentum, dampening))
					return -1;
				i++;
				continue;
			}
			if (counts[i] > 0)
			{
				const int k = t.tensors++;
				t.g[k] = g[i], t.a[k] = a[i], t.m[k] = m[i], t.b[k] = b[i], t.n[k] = n[i];
				t.count[k] = (unsigned)counts[i];
				t.block_start[k] = blocks;
				blocks += (unsigned)((counts[i] + SGD_MULTI_CHUNK - 1) / SGD_MULTI_CHUNK);
			}
			i++;
		}
		if (t.tensors > 0)
		{
			t.block_start[t.tensors] = blocks;
			sgd_multi_kernel<<<blocks, 256, 0, s>>>(t, nesterov, rate, scale, decay, momentum, inv_dampening);
			if (launched("sgd_multi"))
				return -1;
		}
	}
	return 0;
}

// =============================================================================================== 16-bit elementwise
// relu / n-ary sum / column sums on bf16 / fp16 tensors (fp32 arithmetic, one rounding on the way out)
template <typename T, int BWD>
__global__ void relu16_kernel(const T* __restrict__ g, const T* __restrict__ a, T* __restrict__ out, const size_t n, const int vec)
{
	constexpr int W = Vec16<T>::W;
	const size_t nw = vec ? n / W : 0;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nw; i += (size_t)gridDim.x * blockDim.x)
	{
		float x[W], y[W], o[W];
		ldv(a + i * W, x);
		if (BWD)
			ldv(g + i * W, y);
#pragma unroll
		for (int k = 0; k < W; k++)
			o[k] = BWD ? (x[k] > 0 ? y[k] : 0.f) : fmaxf(x[k], 0.f);
		stv(out + i * W, o);
	}
	for (size_t i = nw * W + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		stf(out + i, BWD ? (ldf(a + i) > 0 ? ldf(g + i) : 0.f) : fmaxf(ldf(a + i), 0.f));
}
template <typename T>
static int relu16_t(cudaStream_t s, const T* g, const T* a, T* out, size_t n, int bwd)
{
	if (n == 0)
		return 0;
	const int vec = aligned_v16(a) && aligned_v16(out) && (!bwd || aligned_v16(g));
	if (bwd)
		relu16_kernel<T, 1><<<grid_for(vec ? n / Vec16<T>::W + 1 : n, 256, 8), 256, 0, s>>>(g, a, out, n, vec);
	else
		relu16_kernel<T, 0><<<grid_for(vec ? n / Vec16<T>::W + 1 : n, 256, 8), 256, 0, s>>>(g, a, out, n, vec);
	return launched("relu16");
}
int ew_relu_fwd_16(cudaStream_t s, int kind, const void* a, void* b, size_t n)
{
	return kind == 1 ? relu16_t<__nv_bfloat16>(s, 0, (const __nv_bfloat16*)a, (__nv_bfloat16*)b, n, 0) : relu16_t<__half>(s, 0, (const __half*)a, (__half*)b, n, 0);
}
int ew_relu_bwd_16(cudaStream_t s, int kind, const void* g, const void* b, void* h, size_t n)
{
	return kind == 1 ? relu16_t<__nv_bfloat16>(s, (const __nv_bfloat16*)g, (const __nv_bfloat16*)b, (__nv_bfloat16*)h, n, 1) : relu16_t<__half>(s, (const __half*)g, (const __half*)b, (__half*)h, n, 1);
}
struct SumArgs16 {
	const void* in[8];
	int k;
};
template <typename T>
__global__ void sum16_kernel(const SumArgs16 a, T* __restrict__ out, const size_t n, const int vec)
{
	constexpr int W = Vec16<T>::W;
	const size_t nw = vec ? n / W : 0;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nw; i += (size_t)gridDim.x * blockDim.x)
	{
		float acc[W];
#pragma unroll
		for (int k = 0; k < W; k++)
			acc[k] = 0.f;
#pragma unroll 8
		for (int j = 0; j < a.k; j++)
		{
			float v[W];
			ldv(reinterpret_cast<const T*>(a.in[j]) + i * W, v);
#pragma unroll
			for (int k = 0; k < W; k++)
				acc[k] += v[k];
		}
		stv(out + i * W, acc);
	}
	for (size_t i = nw * W + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		float acc = 0.f;
		for (int j = 0; j < a.k; j++)
			acc += ldf(reinterpret_cast<const T*>(a.in[j]) + i);
		stf(out + i, acc);
	}
}
// c = a0 + a1 + ... (<= 8 operands per call; the sum is formed in fp32 and rounded once)
int ew_sum_16(cudaStream_t s, int kind, const void* const* inputs, int k, void* out, size_t n)
{
	if (n == 0 || k <= 0)
		return 0;
	if (k > 8)
		return 1;
	SumArgs16 a;
	a.k = k;
	bool vec = (((uintptr_t)out) & 15) == 0;
	for (int j = 0; j < k; j++)
		a.in[j] = inputs[j], vec = vec && (((uintptr_t)inputs[j]) & 15) == 0;
	if (kind == 1)
		sum16_kernel<__nv_bfloat16><<<grid_for(vec ? (n >> 3) + 1 : n, 256, 8), 256, 0, s>>>(a, (__nv_bfloat16*)out, n, vec);
	else
		sum16_kernel<__half><<<grid_for(vec ? (n >> 3) + 1 : n, 256, 8), 256, 0, s>>>(a, (__half*)out, n, vec);
	return launched("ew_sum16");
}

// ew/ccv_nnc_ew_cpu_ref.c:235-334 (EWPROD): c = a0 * a1 * ..., every product rounded on its own, left to right.  fp32 in chunks of
// 8 operands like EWSUM, each later chunk continuing from the output; 16-bit in one launch of <= 8 widened operands, rounded once.
// The running product starts from 1, and 1 * a0 is a0 exactly (signed zeros and NaN payloads included).
template <typename T, int VEC>
__global__ void prod_kernel(const SumArgs16 a, T* __restrict__ out, const size_t n, const int accumulate)
{
	const size_t nv = VEC > 1 ? n / VEC : 0;
	if constexpr (VEC > 1)
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x)
	{
		float acc[VEC];
		if (accumulate)
			ldv(out + i * VEC, acc);
		else
#pragma unroll
			for (int k = 0; k < VEC; k++)
				acc[k] = 1.f;
#pragma unroll 8
		for (int j = 0; j < a.k; j++)
		{
			float v[VEC];
			ldv(reinterpret_cast<const T*>(a.in[j]) + i * VEC, v);
#pragma unroll
			for (int k = 0; k < VEC; k++)
				acc[k] = __fmul_rn(acc[k], v[k]);
		}
		stv(out + i * VEC, acc);
	}
	for (size_t i = nv * VEC + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		float acc = accumulate ? ldf(out + i) : 1.f;
		for (int j = 0; j < a.k; j++)
			acc = __fmul_rn(acc, ldf(reinterpret_cast<const T*>(a.in[j]) + i));
		stf(out + i, acc);
	}
}
template <typename T>
static int prod_t(cudaStream_t s, const void* const* inputs, int k, T* out, size_t n)
{
	constexpr int W = Vec16<T>::W;
	for (int done = 0; done < k;)
	{
		SumArgs16 a;
		a.k = (k - done) > 8 ? 8 : (k - done);
		bool vec = aligned_v16(out);
		for (int j = 0; j < a.k; j++)
			a.in[j] = inputs[done + j], vec = vec && aligned_v16(a.in[j]);
		if (vec)
			prod_kernel<T, W><<<grid_for(n / W + 1, 256, 8), 256, 0, s>>>(a, out, n, done > 0);
		else
			prod_kernel<T, 1><<<grid_for(n, 256, 8), 256, 0, s>>>(a, out, n, done > 0);
		if (launched("ew_prod"))
			return -1;
		done += a.k;
	}
	return 0;
}
int ew_prod(cudaStream_t s, int kind, const void* const* inputs, int k, void* out, size_t n)
{
	if (n == 0 || k <= 0)
		return 0;
	if (k > (kind == 0 ? 64 : 8))
		return 1;
	return kind == 0 ? prod_t<float>(s, inputs, k, (float*)out, n) : kind == 1 ? prod_t<__nv_bfloat16>(s, inputs, k, (__nv_bfloat16*)out, n) : prod_t<__half>(s, inputs, k, (__half*)out, n);
}

// ew/ccv_nnc_ew_cpu_ref.c:336-480 (EWPROD backward): h_z = g * b / a_z, or b / a_z without g, each operation rounded on its own.  One
// launch for every output; a thread reads all operands of its element before it writes any output, so outputs may alias inputs.
template <int MAXK>
struct ProdBackArgs {
	const void* a[MAXK];
	void* h[MAXK];
	const void* g;
	const void* b;
	int k;
};
template <typename T, int MAXK>
__global__ void prod_back_kernel(const ProdBackArgs<MAXK> p, const size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		const float bv = ldf(reinterpret_cast<const T*>(p.b) + i);
		const float num = p.g ? __fmul_rn(ldf(reinterpret_cast<const T*>(p.g) + i), bv) : bv;
		float r[MAXK];
#pragma unroll
		for (int z = 0; z < MAXK; z++)
			if (z < p.k)
				r[z] = __fdiv_rn(num, ldf(reinterpret_cast<const T*>(p.a[z]) + i));
#pragma unroll
		for (int z = 0; z < MAXK; z++)
			if (z < p.k)
				stf(reinterpret_cast<T*>(p.h[z]) + i, r[z]);
	}
}
template <typename T, int MAXK>
static int prod_back_t(cudaStream_t s, const void* g, const void* b, const void* const* a, void* const* h, int k, size_t n)
{
	ProdBackArgs<MAXK> p;
	p.g = g, p.b = b, p.k = k;
	for (int z = 0; z < k; z++)
		p.a[z] = a[z], p.h[z] = h[z];
	prod_back_kernel<T, MAXK><<<grid_for(n, 256, 8), 256, 0, s>>>(p, n);
	return launched("ew_prod_back");
}
int ew_prod_back(cudaStream_t s, int kind, const void* g, const void* b, const void* const* a, void* const* h, int k, size_t n)
{
	if (n == 0 || k <= 0)
		return 0;
	if (k > (kind == 0 ? 64 : 8))
		return 1;
	return kind == 0 ? prod_back_t<float, 64>(s, g, b, a, h, k, n) : kind == 1 ? prod_back_t<__nv_bfloat16, 8>(s, g, b, a, h, k, n) : prod_back_t<__half, 8>(s, g, b, a, h, k, n);
}
// column sums with any input / output element kind: per-block partial rows (fp32) in the workspace, combined in a fixed order
template <typename T>
__global__ void __launch_bounds__(256) colsum_any_kernel(const T* __restrict__ g, const size_t rows, const int cols, const long long ld, float* __restrict__ part)
{
	// thread = (column group of 4, row lane); blockIdx.y = row slab
	__shared__ float4 sh[256];
	const int cols4 = cols >> 2;
	const int cpb = cols4 >= 256 ? 256 : cols4, rpi = 256 / cpb;
	const int tx = threadIdx.x % cpb, ty = threadIdx.x / cpb;
	const int col4 = blockIdx.x * cpb + tx;
	float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
	if (ty < rpi && col4 < cols4)
		for (size_t r = (size_t)blockIdx.y * rpi + ty; r < rows; r += (size_t)gridDim.y * rpi)
		{
			const float4 v = ld4(g + r * ld + col4 * 4);
			acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
		}
	sh[threadIdx.x] = acc;
	__syncthreads();
	if (ty == 0 && col4 < cols4)
	{
		for (int j = 1; j < rpi; j++)
		{
			const float4 v = sh[j * cpb + tx];
			acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
		}
		*reinterpret_cast<float4*>(part + ((size_t)blockIdx.y * cols4 + col4) * 4) = acc;
	}
}
__global__ void __launch_bounds__(1024) colsum_partials_any_kernel(const float* __restrict__ part, const int gy, const int ncols, void* __restrict__ out, const int out_kind, const int accumulate)
{
	__shared__ float sh[32][33];
	const int cx = threadIdx.x & 31, yl = threadIdx.x >> 5;
	const int col = blockIdx.x * 32 + cx;
	float acc = 0.f;
	if (col < ncols)
		for (int y = yl; y < gy; y += 32)
			acc += part[(size_t)y * ncols + col];
	sh[yl][cx] = acc;
	__syncthreads();
	if (yl == 0 && col < ncols)
	{
		float t = 0.f;
#pragma unroll
		for (int j = 0; j < 32; j++)
			t += sh[j][cx];
		st_kind(out, col, accumulate ? ld_kind(out, col, out_kind) + t : t, out_kind);
	}
}
// one block per column, any stride / alignment / element kind (odd shapes: a 10-class head); fixed summation order
__global__ void colsum_scalar_kernel(const void* __restrict__ g, const int g_kind, const size_t rows, const long long ld, void* __restrict__ out, const int out_kind, const int accumulate)
{
	__shared__ float sh[256];
	const int col = blockIdx.x;
	float acc = 0.f;
	for (size_t r = threadIdx.x; r < rows; r += blockDim.x)
		acc += ld_kind(g, r * ld + col, g_kind);
	sh[threadIdx.x] = acc;
	__syncthreads();
	for (int o = 128; o > 0; o >>= 1)
	{
		if ((int)threadIdx.x < o)
			sh[threadIdx.x] += sh[threadIdx.x + o];
		__syncthreads();
	}
	if (threadIdx.x == 0)
		st_kind(out, col, accumulate ? ld_kind(out, col, out_kind) + sh[0] : sh[0], out_kind);
}
int colsum_any(cudaStream_t s, int g_kind, const void* g, size_t rows, int cols, long long ld, void* out, int out_kind, int accumulate, void* workspace)
{
	if (g_kind == 0 && out_kind == 0)
		return colsum_f32(s, (const float*)g, rows, cols, ld, (float*)out, accumulate, workspace);
	if (cols <= 0)
		return 0;
	// the vector kernel loads 4 elements of g at once: 16 bytes of fp32, 8 of bf16 / fp16
	if (cols % 4 || ld % 4 || !workspace || (((uintptr_t)g) & (g_kind == 0 ? 15 : 7)))
	{
		colsum_scalar_kernel<<<cols, 256, 0, s>>>(g, g_kind, rows, ld, out, out_kind, accumulate);
		return launched("colsum_scalar");
	}
	const int cols4 = cols / 4, cpb = cols4 >= 256 ? 256 : cols4, rpi = 256 / cpb;
	const int gx = (cols4 + cpb - 1) / cpb;
	size_t gy = (rows + (size_t)rpi * 32 - 1) / ((size_t)rpi * 32);
	const size_t cap = (size_t)(sm_count() * 8 + gx - 1) / gx;
	if (gy > cap)
		gy = cap;
	if (gy < 1)
		gy = 1;
	float* const part = (float*)workspace;
	if (g_kind == 0)
		colsum_any_kernel<float><<<dim3(gx, (unsigned)gy), 256, 0, s>>>((const float*)g, rows, cols, ld, part);
	else if (g_kind == 1)
		colsum_any_kernel<__nv_bfloat16><<<dim3(gx, (unsigned)gy), 256, 0, s>>>((const __nv_bfloat16*)g, rows, cols, ld, part);
	else
		colsum_any_kernel<__half><<<dim3(gx, (unsigned)gy), 256, 0, s>>>((const __half*)g, rows, cols, ld, part);
	if (launched("colsum_any"))
		return -1;
	colsum_partials_any_kernel<<<(cols + 31) / 32, 1024, 0, s>>>(part, (int)gy, cols, out, out_kind, accumulate);
	return launched("colsum_partials_any");
}

// strided [rows, cols] matrix of element kind `kind` <-> dense fp32 [rows, cols]: the operands of 16-bit GEMMs whose strides the
// tensor-core path cannot take (TMA wants 16-byte multiples) are widened, multiplied on the CUDA cores and narrowed back
__global__ void widen_matrix_kernel(const void* __restrict__ src, const int kind, const long long rs, const long long cs, float* __restrict__ dst, const int rows, const int cols)
{
	const size_t total = (size_t)rows * cols;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		const size_t r = i / cols, c = i - r * cols;
		dst[i] = ld_kind(src, r * rs + c * cs, kind);
	}
}
__global__ void narrow_matrix_kernel(const float* __restrict__ src, void* __restrict__ dst, const int kind, const long long rs, const long long cs, const int rows, const int cols, const int accumulate)
{
	const size_t total = (size_t)rows * cols;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		const size_t r = i / cols, c = i - r * cols;
		const size_t at = r * rs + c * cs;
		st_kind(dst, at, accumulate ? ld_kind(dst, at, kind) + src[i] : src[i], kind);
	}
}
int widen_matrix(cudaStream_t s, const void* src, int kind, long long rs, long long cs, float* dst, int rows, int cols)
{
	if (rows <= 0 || cols <= 0)
		return 0;
	widen_matrix_kernel<<<grid_for((size_t)rows * cols, 256, 8), 256, 0, s>>>(src, kind, rs, cs, dst, rows, cols);
	return launched("widen_matrix");
}
int narrow_matrix(cudaStream_t s, const float* src, void* dst, int kind, long long rs, long long cs, int rows, int cols, int accumulate)
{
	if (rows <= 0 || cols <= 0)
		return 0;
	narrow_matrix_kernel<<<grid_for((size_t)rows * cols, 256, 8), 256, 0, s>>>(src, dst, kind, rs, cs, rows, cols, accumulate);
	return launched("narrow_matrix");
}

// =============================================================================================== dtype conversion
// f32 -> f16 is f32_to_f16_trunc (sm100_elem.cuh): the reference's truncating table method, not __float2half_rn.
template <int AD, int BD>
__global__ void convert_kernel(const void* __restrict__ a, void* __restrict__ b, const size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		if (AD == 0 && BD == 1)
			reinterpret_cast<uint16_t*>(b)[i] = f32_to_f16_trunc(reinterpret_cast<const float*>(a)[i]);
		else if (AD == 1 && BD == 0)
			reinterpret_cast<float*>(b)[i] = __half2float(reinterpret_cast<const __half*>(a)[i]);
		else if (AD == 0 && BD == 2)
			reinterpret_cast<double*>(b)[i] = (double)reinterpret_cast<const float*>(a)[i];
		else if (AD == 2 && BD == 0)
			reinterpret_cast<float*>(b)[i] = (float)reinterpret_cast<const double*>(a)[i];
		else if (AD == 0 && BD == 3)
			reinterpret_cast<__nv_bfloat16*>(b)[i] = __float2bfloat16_rn(reinterpret_cast<const float*>(a)[i]);
		else if (AD == 3 && BD == 0)
			reinterpret_cast<float*>(b)[i] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a)[i]);
		else if (AD == 2 && BD == 1)
			reinterpret_cast<uint16_t*>(b)[i] = f32_to_f16_trunc((float)reinterpret_cast<const double*>(a)[i]);
		else if (AD == 1 && BD == 2)
			reinterpret_cast<double*>(b)[i] = (double)__half2float(reinterpret_cast<const __half*>(a)[i]);
	}
}
int convert_dtype(cudaStream_t s, const void* a, int ad, void* b, int bd, size_t n)
{
	if (n == 0)
		return 0;
	const int grid = grid_for(n, 256, 8);
#define CONV_CASE(A, B) if (ad == A && bd == B) { convert_kernel<A, B><<<grid, 256, 0, s>>>(a, b, n); return launched("convert_dtype"); }
	CONV_CASE(0, 1) CONV_CASE(1, 0) CONV_CASE(0, 2) CONV_CASE(2, 0) CONV_CASE(0, 3) CONV_CASE(3, 0) CONV_CASE(2, 1) CONV_CASE(1, 2)
#undef CONV_CASE
	return 1;
}

// =============================================================================================== strided copy
template <typename T>
__global__ void copy_strided_kernel(const T* __restrict__ a, T* __restrict__ b, const Bcast4 d, const size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		size_t r = i;
		const int i3 = r % d.dim[3];
		r /= d.dim[3];
		const int i2 = r % d.dim[2];
		r /= d.dim[2];
		const int i1 = r % d.dim[1];
		const int i0 = (int)(r / d.dim[1]);
		b[(size_t)i0 * d.cs[0] + (size_t)i1 * d.cs[1] + (size_t)i2 * d.cs[2] + (size_t)i3 * d.cs[3]] = a[(size_t)i0 * d.as[0] + (size_t)i1 * d.as[1] + (size_t)i2 * d.as[2] + (size_t)i3 * d.as[3]];
	}
}
// util/ccv_nnc_util_cpu_ref.c (DATA_TRANSFER / FORMAT_TRANSFORM / TRANSPOSE all reduce to b[index] = a[index] over
// permuted strides).  The index space is enumerated in the order that makes b's writes coalesced.
int copy_strided(cudaStream_t s, const void* a, const int* astride, void* b, const int* bstride, const int* dim, int elem_size)
{
	Bcast4 d = make_bcast(astride, 0, bstride, dim);
	// order the four axes by decreasing output stride so that consecutive threads write consecutive addresses
	int order[4] = { 0, 1, 2, 3 };
	for (int i = 0; i < 4; i++)
		for (int j = i + 1; j < 4; j++)
			if (d.cs[order[j]] > d.cs[order[i]] || (d.cs[order[j]] == d.cs[order[i]] && d.dim[order[j]] < d.dim[order[i]]))
			{
				const int t = order[i];
				order[i] = order[j];
				order[j] = t;
			}
	Bcast4 e;
	for (int i = 0; i < 4; i++)
		e.dim[i] = d.dim[order[i]], e.as[i] = d.as[order[i]], e.cs[i] = d.cs[order[i]], e.bs[i] = 0;
	const size_t n = (size_t)e.dim[0] * e.dim[1] * e.dim[2] * e.dim[3];
	if (n == 0)
		return 0;
	const int grid = grid_for(n, 256, 8);
	if (elem_size == 4)
		copy_strided_kernel<uint32_t><<<grid, 256, 0, s>>>((const uint32_t*)a, (uint32_t*)b, e, n);
	else if (elem_size == 2)
		copy_strided_kernel<uint16_t><<<grid, 256, 0, s>>>((const uint16_t*)a, (uint16_t*)b, e, n);
	else if (elem_size == 8)
		copy_strided_kernel<uint64_t><<<grid, 256, 0, s>>>((const uint64_t*)a, (uint64_t*)b, e, n);
	else if (elem_size == 1)
		copy_strided_kernel<uint8_t><<<grid, 256, 0, s>>>((const uint8_t*)a, (uint8_t*)b, e, n);
	else
		return 1;
	return launched("copy_strided");
}

} // namespace sm100
