// sm100_norm.cu -- layer norm, rms norm (row reductions with warp shuffles) and upsample (coalesced over channels).
// Semantics: norm/ccv_nnc_layer_norm_cpu_ref.c:16-420, norm/ccv_nnc_rmsnorm_cpu_ref.c:16-330,
// upsample/ccv_nnc_upsample_cpu_ref.c:16-509 (paths relative to /root/reference/lib/nnc/cmd).
#include "sm100_ew.h"
#include "sm100_contract.h"
#include <float.h>

namespace sm100 {

static int check(const char* what)
{
	count_launch();
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		set_last_error(what, e);
		return -1;
	}
	return 0;
}

__device__ __forceinline__ float wsum(float v)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		v += __shfl_xor_sync(0xffffffff, v, o);
	return v;
}
__device__ __forceinline__ float bsum(float v, float* sh)
{
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	v = wsum(v);
	__syncthreads();
	if (lane == 0)
		sh[w] = v;
	__syncthreads();
	v = lane < nw ? sh[lane] : 0.f;
	return wsum(v);
}
static int row_threads(int inner) { return inner >= 2048 ? 512 : (inner >= 512 ? 256 : (inner >= 128 ? 128 : (inner >= 64 ? 64 : 32))); }

// one block per row: mean, biased variance of (x - mean) (two passes over a row that sits in L1/L2), y = xhat * scale + bias
template <int RMS>
__global__ void norm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ bias, float* __restrict__ y, float* __restrict__ saved_mean, float* __restrict__ saved_inv_std, const int inner, const float epsilon)
{
	__shared__ float sh[32];
	const float* xp = x + (size_t)blockIdx.x * inner;
	float* yp = y + (size_t)blockIdx.x * inner;
	float mean = 0.f;
	if (!RMS)
	{
		float s = 0.f;
		for (int j = threadIdx.x; j < inner; j += blockDim.x)
			s += xp[j];
		mean = bsum(s, sh) * (1.f / inner);
	}
	float v = 0.f;
	for (int j = threadIdx.x; j < inner; j += blockDim.x)
	{
		const float d = xp[j] - mean;
		v += d * d;
	}
	v = bsum(v, sh);
	const float inv_std = 1.f / sqrtf(v * (1.f / inner) + epsilon);
	if (threadIdx.x == 0)
	{
		if (!RMS && saved_mean)
			saved_mean[blockIdx.x] = mean;
		if (saved_inv_std)
			saved_inv_std[blockIdx.x] = inv_std;
	}
	for (int j = threadIdx.x; j < inner; j += blockDim.x)
	{
		float o = (xp[j] - mean) * inv_std;
		if (scale)
			o *= scale[j];
		if (bias)
			o += bias[j];
		yp[j] = o;
	}
}
int layer_norm_fwd_f32(cudaStream_t s, const float* x, const float* scale, const float* bias, float* y, float* saved_mean, float* saved_inv_std, int rows, int inner, float epsilon)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	norm_fwd_kernel<0><<<rows, row_threads(inner), 0, s>>>(x, scale, bias, y, saved_mean, saved_inv_std, inner, epsilon);
	return check("layer_norm_fwd");
}
int rmsnorm_fwd_f32(cudaStream_t s, const float* x, const float* scale, float* y, float* saved_inv_std, int rows, int inner, float epsilon)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	norm_fwd_kernel<1><<<rows, row_threads(inner), 0, s>>>(x, scale, 0, y, 0, saved_inv_std, inner, epsilon);
	return check("rmsnorm_fwd");
}
// dx per row.  layer norm: r * (gs - mean(gs) - xhat * mean(gs * xhat)); rms norm: r * (gs - xhat * mean(gs * xhat)), gs = g * scale
template <int RMS>
__global__ void norm_bwd_dx_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, float* __restrict__ dx, const int inner)
{
	__shared__ float sh[32];
	const size_t o = (size_t)blockIdx.x * inner;
	const float mean = RMS ? 0.f : saved_mean[blockIdx.x], r = saved_inv_std[blockIdx.x];
	float s1 = 0.f, s2 = 0.f;
	for (int j = threadIdx.x; j < inner; j += blockDim.x)
	{
		const float gs = g[o + j] * (scale ? scale[j] : 1.f);
		s1 += gs;
		s2 += gs * (x[o + j] - mean) * r;
	}
	s1 = RMS ? 0.f : bsum(s1, sh) * (1.f / inner);
	s2 = bsum(s2, sh) * (1.f / inner);
	for (int j = threadIdx.x; j < inner; j += blockDim.x)
	{
		const float gs = g[o + j] * (scale ? scale[j] : 1.f);
		dx[o + j] = r * (gs - s1 - (x[o + j] - mean) * r * s2);
	}
}
// dscale[j] = sum_rows g * xhat, dbias[j] = sum_rows g.  Row block y (rows y, y + gridDim.y, ..) leaves its two partial sums of column j
// in part[y][j] and part[y][inner + j]; norm_bwd_dparam_rows_kernel then adds the gridDim.y rows in a fixed order, so the result does
// not depend on the order in which blocks finish (one atomicAdd per (block, column) did).
static int dparam_row_blocks(int rows) { return rows < 296 ? rows : 296; }
size_t norm_bwd_workspace_bytes(int rows, int inner) { return rows <= 0 || inner <= 0 ? 0 : (size_t)dparam_row_blocks(rows) * 2 * (size_t)inner * sizeof(float); }
template <int RMS>
__global__ void norm_bwd_dparam_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, float* __restrict__ part, const int rows, const int inner)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= inner)
		return;
	float a = 0.f, b = 0.f;
	for (int r = blockIdx.y; r < rows; r += gridDim.y)
	{
		const float gv = g[(size_t)r * inner + j];
		a += gv * (x[(size_t)r * inner + j] - (RMS ? 0.f : saved_mean[r])) * saved_inv_std[r];
		b += gv;
	}
	float* const row = part + (size_t)blockIdx.y * 2 * inner;
	row[j] = a;
	if (!RMS)
		row[inner + j] = b;
}
// 32 columns x 32 row-lanes per block: lane l adds rows l, l + 32, .. in order, then the 32 lane sums are added in order
__global__ void __launch_bounds__(1024) norm_bwd_dparam_rows_kernel(const float* __restrict__ part, const int gy, const int inner, float* __restrict__ dscale, float* __restrict__ dbias)
{
	__shared__ float sh[2][32][33];
	const int cx = threadIdx.x & 31, yl = threadIdx.x >> 5;
	const int j = blockIdx.x * 32 + cx;
	float a = 0.f, b = 0.f;
	if (j < inner)
		for (int y = yl; y < gy; y += 32)
		{
			const float* const row = part + (size_t)y * 2 * inner;
			if (dscale)
				a += row[j];
			if (dbias)
				b += row[inner + j];
		}
	sh[0][yl][cx] = a, sh[1][yl][cx] = b;
	__syncthreads();
	if (yl != 0 || j >= inner)
		return;
	a = b = 0.f;
#pragma unroll
	for (int l = 0; l < 32; l++)
		a += sh[0][l][cx], b += sh[1][l][cx];
	if (dscale)
		dscale[j] = a;
	if (dbias)
		dbias[j] = b;
}
template <int RMS>
static int norm_bwd(cudaStream_t s, const float* g, const float* x, const float* scale, const float* saved_mean, const float* saved_inv_std, float* dx, float* dscale, float* dbias, int rows, int inner, void* workspace)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	if ((dscale || dbias) && !workspace)
		return -1;
	if (dx)
	{
		norm_bwd_dx_kernel<RMS><<<rows, row_threads(inner), 0, s>>>(g, x, scale, saved_mean, saved_inv_std, dx, inner);
		if (check("norm_bwd_dx"))
			return -1;
	}
	if (dscale || dbias)
	{
		const int gy = dparam_row_blocks(rows);
		norm_bwd_dparam_kernel<RMS><<<dim3((inner + 127) / 128, gy), 128, 0, s>>>(g, x, saved_mean, saved_inv_std, (float*)workspace, rows, inner);
		if (check("norm_bwd_dparam"))
			return -1;
		norm_bwd_dparam_rows_kernel<<<(inner + 31) / 32, 1024, 0, s>>>((const float*)workspace, gy, inner, dscale, dbias);
		if (check("norm_bwd_dparam_rows"))
			return -1;
	}
	return 0;
}
int layer_norm_bwd_f32(cudaStream_t s, const float* g, const float* x, const float* scale, const float* saved_mean, const float* saved_inv_std, float* dx, float* dscale, float* dbias, int rows, int inner, void* workspace)
{
	return norm_bwd<0>(s, g, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, inner, workspace);
}
int rmsnorm_bwd_f32(cudaStream_t s, const float* g, const float* x, const float* scale, const float* saved_inv_std, float* dx, float* dscale, int rows, int inner, void* workspace)
{
	return norm_bwd<1>(s, g, x, scale, 0, saved_inv_std, dx, dscale, 0, rows, inner, workspace);
}

// ------------------------------------------------------------------------------------------------ upsample
struct Coef {
	int i0, i1;
	float c0, c1;
};
// _ccv_nnc_init_bi_coeffs (upsample/ccv_nnc_upsample_cpu_ref.c:220-243), same float arithmetic
__device__ __forceinline__ Coef bi_coef(const int i, const int ss, const float s, const int align_corners)
{
	const float xs = align_corners ? i * s : (i + 0.5f) * s - 0.5f;
	Coef c;
	c.i0 = (int)xs;
	c.i1 = min((int)(xs + 1), ss - 1);
	c.c1 = xs - c.i0;
	c.c0 = 1.0f - c.c1;
	return c;
}
__device__ __forceinline__ int nearest_idx(const int i, const int ss, const float s, const int align_corners)
{
	return min(align_corners ? (int)(i * s + 0.5f) : (int)((i + 0.5f) * s), ss - 1);
}
// thread per output element; NHWC: channels fastest (coalesced); NCHW: width fastest
template <int BWD>
__global__ void upsample_kernel(const float* __restrict__ src, float* __restrict__ dst, const int N, const int H, const int W, const int C, const int OH, const int OW, const int type, const int align_corners, const int nchw, const float rh, const float rw)
{
	const size_t total = (size_t)N * OH * OW * C;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		int n, c, oy, ox;
		size_t r = i;
		if (nchw)
			ox = r % OW, r /= OW, oy = r % OH, r /= OH, c = r % C, n = (int)(r / C);
		else
			c = r % C, r /= C, ox = r % OW, r /= OW, oy = r % OH, n = (int)(r / OH);
		auto in_at = [&](int y, int x) -> size_t { return nchw ? (((size_t)n * C + c) * H + y) * W + x : (((size_t)n * H + y) * W + x) * C + c; };
		// forward: dst = output (upsampled), src = input. backward: src = output gradient (upsampled), dst = input gradient
		if (type == 0)
		{
			const int y = nearest_idx(oy, H, rh, align_corners), x = nearest_idx(ox, W, rw, align_corners);
			if (BWD)
				atomicAdd(dst + in_at(y, x), src[i]);
			else
				dst[i] = src[in_at(y, x)];
		} else {
			const Coef cy = bi_coef(oy, H, rh, align_corners), cx = bi_coef(ox, W, rw, align_corners);
			if (BWD)
			{
				const float v = src[i];
				atomicAdd(dst + in_at(cy.i0, cx.i0), v * cy.c0 * cx.c0);
				atomicAdd(dst + in_at(cy.i0, cx.i1), v * cy.c0 * cx.c1);
				atomicAdd(dst + in_at(cy.i1, cx.i0), v * cy.c1 * cx.c0);
				atomicAdd(dst + in_at(cy.i1, cx.i1), v * cy.c1 * cx.c1);
			} else
				dst[i] = src[in_at(cy.i0, cx.i0)] * cx.c0 * cy.c0 + src[in_at(cy.i0, cx.i1)] * cx.c1 * cy.c0 + src[in_at(cy.i1, cx.i0)] * cx.c0 * cy.c1 + src[in_at(cy.i1, cx.i1)] * cx.c1 * cy.c1;
		}
	}
}
static void ratios(int H, int W, int OH, int OW, int align_corners, float& rh, float& rw)
{
	rh = align_corners ? (float)(H - 1) / (OH - 1 > 1 ? OH - 1 : 1) : (float)H / OH;
	rw = align_corners ? (float)(W - 1) / (OW - 1 > 1 ? OW - 1 : 1) : (float)W / OW;
}
int upsample_fwd_f32(cudaStream_t s, const float* a, float* b, int N, int H, int W, int C, int OH, int OW, int type, int align_corners, int nchw)
{
	const size_t total = (size_t)N * OH * OW * C;
	if (total == 0)
		return 0;
	float rh, rw;
	ratios(H, W, OH, OW, align_corners, rh, rw);
	size_t blocks = (total + 255) / 256;
	if (blocks > 132 * 16)
		blocks = 132 * 16;
	upsample_kernel<0><<<(unsigned)blocks, 256, 0, s>>>(a, b, N, H, W, C, OH, OW, type, align_corners, nchw, rh, rw);
	return check("upsample_fwd");
}
int upsample_bwd_f32(cudaStream_t s, const float* g, float* h, int N, int H, int W, int C, int OH, int OW, int type, int align_corners, int nchw)
{
	const size_t total = (size_t)N * OH * OW * C;
	if (cudaMemsetAsync(h, 0, (size_t)N * H * W * C * 4, s) != cudaSuccess)
		return -1;
	if (total == 0)
		return 0;
	float rh, rw;
	ratios(H, W, OH, OW, align_corners, rh, rw);
	size_t blocks = (total + 255) / 256;
	if (blocks > 132 * 16)
		blocks = 132 * 16;
	upsample_kernel<1><<<(unsigned)blocks, 256, 0, s>>>(g, h, N, H, W, C, OH, OW, type, align_corners, nchw, rh, rw);
	return check("upsample_bwd");
}


// ---- group norm (norm/ccv_nnc_group_norm_cpu_ref.c) ------------------------------------------------------------------
// Everything is a <= 4-d index space `dim`; a statistic / scale / bias tensor has dims rdim with rdim[d] <= dim[d] and the
// element i of axis d belongs to slot i * rdim[d] / dim[d] (:64-76), i.e. slot g owns the contiguous range
// [ceil(g * dim / rdim), ceil((g + 1) * dim / rdim)).  One thread block walks the box of one slot.
struct GnBox {
	int lo[4], ext[4];
	long long count;
};

__device__ __forceinline__ GnBox gn_box(const GroupNormGeom& g, const int* const rdim, long long slot)
{
	GnBox b;
	b.count = 1;
#pragma unroll
	for (int d = 3; d >= 0; d--)
	{
		const int gd = (int)(slot % rdim[d]);
		slot /= rdim[d];
		const int lo = (int)(((long long)gd * g.dim[d] + rdim[d] - 1) / rdim[d]);
		const int hi = (int)(((long long)(gd + 1) * g.dim[d] + rdim[d] - 1) / rdim[d]);
		b.lo[d] = lo, b.ext[d] = hi - lo;
		b.count *= hi - lo;
	}
	return b;
}

__device__ __forceinline__ void gn_coord(const GnBox& b, long long i, int c[4])
{
#pragma unroll
	for (int d = 3; d >= 0; d--)
	{
		c[d] = b.lo[d] + (int)(i % b.ext[d]);
		i /= b.ext[d];
	}
}

__device__ __forceinline__ long long gn_offset(const int c[4], const long long stride[4])
{
	return c[0] * stride[0] + c[1] * stride[1] + c[2] * stride[2] + c[3] * stride[3];
}

// slot of coordinate c in a tensor of dims rdim (packed)
__device__ __forceinline__ long long gn_slot(const GroupNormGeom& g, const int c[4], const int rdim[4])
{
	long long s = 0;
#pragma unroll
	for (int d = 0; d < 4; d++)
		s = s * rdim[d] + (long long)c[d] * rdim[d] / g.dim[d];
	return s;
}

__device__ __forceinline__ float gn_block_sum(float v, float* const red) { return bsum(v, red); }

__global__ void gn_stats_kernel(const GroupNormGeom g, const float* __restrict__ x, float* __restrict__ saved_mean, float* __restrict__ saved_inv_std, const float epsilon)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.rdim, blockIdx.x);
	int c[4];
	float sum = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		sum += x[gn_offset(c, g.xstride)];
	}
	const float inv_n = 1.f / (float)b.count;
	const float mean = gn_block_sum(sum, red) * inv_n;
	float sq = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const float w = x[gn_offset(c, g.xstride)] - mean;
		sq += w * w;
	}
	const float var = gn_block_sum(sq, red) * inv_n;
	if (threadIdx.x == 0)
	{
		saved_mean[blockIdx.x] = mean;
		saved_inv_std[blockIdx.x] = 1.f / sqrtf(var + epsilon);
	}
}

__global__ void gn_apply_kernel(const GroupNormGeom g, const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ bias, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, float* __restrict__ y, const long long total)
{
	GnBox all;
	for (int d = 0; d < 4; d++)
		all.lo[d] = 0, all.ext[d] = g.dim[d];
	int c[4];
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		gn_coord(all, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		float v = (x[gn_offset(c, g.xstride)] - saved_mean[r]) * saved_inv_std[r];
		if (scale)
			v = v * scale[gn_slot(g, c, g.sdim)] + bias[gn_slot(g, c, g.sdim)];
		y[gn_offset(c, g.ystride)] = v;
	}
}

// per statistic slot: gssr = sum g * scale * inv_std, ahgssr = sum xhat * g * scale * inv_std (:412-470)
__global__ void gn_bwd_stats_kernel(const GroupNormGeom g, const float* __restrict__ grad, const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, float* __restrict__ sums)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.rdim, blockIdx.x);
	const float mean = saved_mean[blockIdx.x], inv_std = saved_inv_std[blockIdx.x];
	int c[4];
	float s0 = 0, s1 = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const float ah = (x[gn_offset(c, g.xstride)] - mean) * inv_std;
		float gss = grad[gn_offset(c, g.ystride)] * inv_std;
		if (scale)
			gss *= scale[gn_slot(g, c, g.sdim)];
		s0 += gss, s1 += ah * gss;
	}
	s0 = gn_block_sum(s0, red), s1 = gn_block_sum(s1, red);
	if (threadIdx.x == 0)
		sums[2 * blockIdx.x] = s0, sums[2 * blockIdx.x + 1] = s1;
}

// h = gss - (gssr + xhat * ahgssr) / n (:472-500)
__global__ void gn_bwd_apply_kernel(const GroupNormGeom g, const float* __restrict__ grad, const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, const float* __restrict__ sums, float* __restrict__ h, const long long total, const float inv_n)
{
	GnBox all;
	for (int d = 0; d < 4; d++)
		all.lo[d] = 0, all.ext[d] = g.dim[d];
	int c[4];
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		gn_coord(all, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		const float inv_std = saved_inv_std[r];
		const float ah = (x[gn_offset(c, g.xstride)] - saved_mean[r]) * inv_std;
		float gss = grad[gn_offset(c, g.ystride)] * inv_std;
		if (scale)
			gss *= scale[gn_slot(g, c, g.sdim)];
		h[gn_offset(c, g.hstride)] = gss - (sums[2 * r] + ah * sums[2 * r + 1]) * inv_n;
	}
}

// per scale / bias slot: dscale = sum xhat * g, dbias = sum g (:322-345, :254)
__global__ void gn_bwd_dparam_kernel(const GroupNormGeom g, const float* __restrict__ grad, const float* __restrict__ x, const float* __restrict__ saved_mean, const float* __restrict__ saved_inv_std, float* __restrict__ dscale, float* __restrict__ dbias)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.sdim, blockIdx.x);
	int c[4];
	float s0 = 0, s1 = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		const float gv = grad[gn_offset(c, g.ystride)];
		s0 += (x[gn_offset(c, g.xstride)] - saved_mean[r]) * saved_inv_std[r] * gv;
		s1 += gv;
	}
	s0 = gn_block_sum(s0, red), s1 = gn_block_sum(s1, red);
	if (threadIdx.x == 0)
	{
		if (dscale)
			dscale[blockIdx.x] = s0;
		if (dbias)
			dbias[blockIdx.x] = s1;
	}
}

static long long gn_count(const int* d) { return (long long)d[0] * d[1] * d[2] * d[3]; }

int group_norm_fwd_f32(cudaStream_t s, const GroupNormGeom& g, const float* x, const float* scale, const float* bias, float* y, float* saved_mean, float* saved_inv_std, float epsilon)
{
	const long long total = gn_count(g.dim), slots = gn_count(g.rdim);
	if (total == 0)
		return 0;
	gn_stats_kernel<<<(unsigned)slots, 512, 0, s>>>(g, x, saved_mean, saved_inv_std, epsilon);
	count_launch();
	long long blocks = (total + 255) / 256;
	if (blocks > 132 * 16)
		blocks = 132 * 16;
	gn_apply_kernel<<<(unsigned)blocks, 256, 0, s>>>(g, x, scale, bias, saved_mean, saved_inv_std, y, total);
	return check("group_norm_fwd");
}

size_t group_norm_bwd_workspace_bytes(const GroupNormGeom& g) { return (size_t)gn_count(g.rdim) * 2 * sizeof(float); }

int group_norm_bwd_f32(cudaStream_t s, const GroupNormGeom& g, const float* grad, const float* x, const float* scale, const float* saved_mean, const float* saved_inv_std, float* h, float* dscale, float* dbias, void* workspace)
{
	const long long total = gn_count(g.dim), slots = gn_count(g.rdim);
	if (total == 0)
		return 0;
	if (h)
	{
		float* const sums = (float*)workspace;
		gn_bwd_stats_kernel<<<(unsigned)slots, 512, 0, s>>>(g, grad, x, scale, saved_mean, saved_inv_std, sums);
		if (check("group_norm_bwd_stats"))
			return -1;
		long long blocks = (total + 255) / 256;
		if (blocks > 132 * 16)
			blocks = 132 * 16;
		gn_bwd_apply_kernel<<<(unsigned)blocks, 256, 0, s>>>(g, grad, x, scale, saved_mean, saved_inv_std, sums, h, total, (float)slots / (float)total);
		if (check("group_norm_bwd_apply"))
			return -1;
	}
	if (dscale || dbias)
	{
		gn_bwd_dparam_kernel<<<(unsigned)gn_count(g.sdim), 256, 0, s>>>(g, grad, x, saved_mean, saved_inv_std, dscale, dbias);
		if (check("group_norm_bwd_dparam"))
			return -1;
	}
	return 0;
}

} // namespace sm100
