// sm100_norm.cu -- layer norm, rms norm (row reductions with warp shuffles) and upsample (coalesced over channels).
// Semantics: norm/ccv_nnc_layer_norm_cpu_ref.c:16-420, norm/ccv_nnc_rmsnorm_cpu_ref.c:16-330,
// upsample/ccv_nnc_upsample_cpu_ref.c:16-509 (paths relative to /root/reference/lib/nnc/cmd).
#include "sm100_ew.h"
#include "sm100_contract.h"
#include "sm100_elem.cuh"
#include <float.h>
#include <type_traits>

namespace sm100 {

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

// Element types.  The activations (x, y / g, x, dx) are TX: float, __nv_bfloat16 or __half.  Every other operand has its own type,
// float or TX: TP scale, TB bias, TS both statistics, TDS dscale, TDB dbias.  16-bit values are widened exactly, all arithmetic is
// fp32 in the order of the fp32 kernels, and every output is rounded to its type once (round to nearest even, stf / stv).
//
// Rows of a 16-bit TX take 16-byte accesses (8 elements) when inner % 8 == 0 and every row operand is 16-byte aligned; every other
// row, and every fp32 row, takes single-element accesses.  The choice is the same for every row of a call and for a single row.
template <typename TX>
__device__ __forceinline__ bool row_vec(const int inner, const void* a, const void* b, const void* c, const void* d)
{
	return sizeof(TX) == 2 && inner % 8 == 0 && ((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)c) | ((uintptr_t)d)) & 15) == 0;
}
// 8 consecutive elements: one 16-byte access of a 16-bit type, two of fp32
__device__ __forceinline__ void ld8(const float* p, float (&v)[8])
{
	float a[4], b[4];
	ldv(p, a), ldv(p + 4, b);
#pragma unroll
	for (int k = 0; k < 4; k++)
		v[k] = a[k], v[4 + k] = b[k];
}
__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) { ldv(p, v); }
__device__ __forceinline__ void ld8(const __half* p, float (&v)[8]) { ldv(p, v); }
__device__ __forceinline__ void st8(float* p, const float (&v)[8])
{
	const float a[4] = { v[0], v[1], v[2], v[3] }, b[4] = { v[4], v[5], v[6], v[7] };
	stv(p, a), stv(p + 4, b);
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&v)[8]) { stv(p, v); }
__device__ __forceinline__ void st8(__half* p, const float (&v)[8]) { stv(p, v); }
// the value v has once stored as T and read back (v itself for fp32)
template <typename T>
__device__ __forceinline__ float stored(const float v)
{
	T t;
	stf(&t, v);
	return ldf(&t);
}

// one block per row: mean, biased variance of (x - mean) (two passes over a row that sits in L1/L2), y = xhat * scale + bias.
// y is computed from the statistics as stored (rounded to TS when they are 16-bit), which is what the backward reads.
template <int RMS, typename TX, typename TP, typename TB, typename TS>
__global__ void norm_fwd_kernel(const TX* __restrict__ x, const TP* __restrict__ scale, const TB* __restrict__ bias, TX* __restrict__ y, TS* __restrict__ saved_mean, TS* __restrict__ saved_inv_std, const int inner, const float epsilon)
{
	__shared__ float sh[32];
	const TX* xp = x + (size_t)blockIdx.x * inner;
	TX* yp = y + (size_t)blockIdx.x * inner;
	const bool vec = row_vec<TX>(inner, x, y, scale, bias);
	float mean = 0.f;
	if (!RMS)
	{
		float s = 0.f;
		if (vec)
			for (int j = 8 * threadIdx.x; j < inner; j += 8 * blockDim.x)
			{
				float xv[8];
				ld8(xp + j, xv);
#pragma unroll
				for (int k = 0; k < 8; k++)
					s += xv[k];
			}
		else
			for (int j = threadIdx.x; j < inner; j += blockDim.x)
				s += ldf(xp + j);
		mean = bsum(s, sh) * (1.f / inner);
	}
	float v = 0.f;
	if (vec)
		for (int j = 8 * threadIdx.x; j < inner; j += 8 * blockDim.x)
		{
			float xv[8];
			ld8(xp + j, xv);
#pragma unroll
			for (int k = 0; k < 8; k++)
			{
				const float d = xv[k] - mean;
				v += d * d;
			}
		}
	else
		for (int j = threadIdx.x; j < inner; j += blockDim.x)
		{
			const float d = ldf(xp + j) - mean;
			v += d * d;
		}
	v = bsum(v, sh);
	const float inv_std = 1.f / sqrtf(v * (1.f / inner) + epsilon);
	if (threadIdx.x == 0)
	{
		if (!RMS && saved_mean)
			stf(saved_mean + blockIdx.x, mean);
		if (saved_inv_std)
			stf(saved_inv_std + blockIdx.x, inv_std);
	}
	const float ym = saved_mean ? stored<TS>(mean) : mean, yr = saved_inv_std ? stored<TS>(inv_std) : inv_std;
	if (vec)
		for (int j = 8 * threadIdx.x; j < inner; j += 8 * blockDim.x)
		{
			float o[8], sc[8], b[8];
			ld8(xp + j, o);
			if (scale)
				ld8(scale + j, sc);
			if (bias)
				ld8(bias + j, b);
#pragma unroll
			for (int k = 0; k < 8; k++)
			{
				o[k] = (o[k] - ym) * yr;
				if (scale)
					o[k] *= sc[k];
				if (bias)
					o[k] += b[k];
			}
			st8(yp + j, o);
		}
	else
		for (int j = threadIdx.x; j < inner; j += blockDim.x)
		{
			float o = (ldf(xp + j) - ym) * yr;
			if (scale)
				o *= ldf(scale + j);
			if (bias)
				o += ldf(bias + j);
			stf(yp + j, o);
		}
}

// calls f with a null pointer whose element type is that of `kind` (0 fp32, 1 bf16, 2 fp16: ElemKind)
template <typename F>
static int with_kind(const int kind, F&& f)
{
	return kind == 1 ? f((__nv_bfloat16*)0) : kind == 2 ? f((__half*)0) : f((float*)0);
}
// the same for an operand that is either fp32 (kind 0) or of the activations' type TX
template <typename TX, typename F>
static int with_kind_of(const int kind, F&& f)
{
	return kind ? f((TX*)0) : f((float*)0);
}
template <typename P> using elem_t = typename std::remove_pointer<P>::type;

template <int RMS, typename TX, typename TP, typename TB, typename TS>
static int norm_fwd(cudaStream_t s, const void* x, const void* scale, const void* bias, void* y, void* saved_mean, void* saved_inv_std, int rows, int inner, float epsilon)
{
	norm_fwd_kernel<RMS, TX, TP, TB, TS><<<rows, row_threads(inner), 0, s>>>((const TX*)x, (const TP*)scale, (const TB*)bias, (TX*)y, (TS*)saved_mean, (TS*)saved_inv_std, inner, epsilon);
	return launched(RMS ? "rmsnorm_fwd" : "layer_norm_fwd");
}
int layer_norm_fwd(cudaStream_t s, const NormKinds& k, const void* x, const void* scale, const void* bias, void* y, void* saved_mean, void* saved_inv_std, int rows, int inner, float epsilon)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	return with_kind(k.x, [&](auto tx) {
		using TX = elem_t<decltype(tx)>;
		return with_kind_of<TX>(k.scale, [&](auto tp) {
			return with_kind_of<TX>(k.bias, [&](auto tb) {
				return with_kind_of<TX>(k.stat, [&](auto ts) {
					return norm_fwd<0, TX, elem_t<decltype(tp)>, elem_t<decltype(tb)>, elem_t<decltype(ts)> >(s, x, scale, bias, y, saved_mean, saved_inv_std, rows, inner, epsilon);
				});
			});
		});
	});
}
int rmsnorm_fwd(cudaStream_t s, const NormKinds& k, const void* x, const void* scale, void* y, void* saved_inv_std, int rows, int inner, float epsilon)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	return with_kind(k.x, [&](auto tx) {
		using TX = elem_t<decltype(tx)>;
		return with_kind_of<TX>(k.scale, [&](auto tp) {
			return with_kind_of<TX>(k.stat, [&](auto ts) {
				return norm_fwd<1, TX, elem_t<decltype(tp)>, float, elem_t<decltype(ts)> >(s, x, scale, 0, y, 0, saved_inv_std, rows, inner, epsilon);
			});
		});
	});
}
// dx per row.  layer norm: r * (gs - mean(gs) - xhat * mean(gs * xhat)); rms norm: r * (gs - xhat * mean(gs * xhat)), gs = g * scale
template <int RMS, typename TX, typename TP, typename TS>
__global__ void norm_bwd_dx_kernel(const TX* __restrict__ g, const TX* __restrict__ x, const TP* __restrict__ scale, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, TX* __restrict__ dx, const int inner)
{
	__shared__ float sh[32];
	const size_t o = (size_t)blockIdx.x * inner;
	const float mean = RMS ? 0.f : ldf(saved_mean + blockIdx.x), r = ldf(saved_inv_std + blockIdx.x);
	const bool vec = row_vec<TX>(inner, g, x, scale, dx);
	float s1 = 0.f, s2 = 0.f;
	if (vec)
		for (int j = 8 * threadIdx.x; j < inner; j += 8 * blockDim.x)
		{
			float gv[8], xv[8], sc[8];
			ld8(g + o + j, gv), ld8(x + o + j, xv);
			if (scale)
				ld8(scale + j, sc);
#pragma unroll
			for (int k = 0; k < 8; k++)
			{
				const float gs = gv[k] * (scale ? sc[k] : 1.f);
				s1 += gs;
				s2 += gs * (xv[k] - mean) * r;
			}
		}
	else
		for (int j = threadIdx.x; j < inner; j += blockDim.x)
		{
			const float gs = ldf(g + o + j) * (scale ? ldf(scale + j) : 1.f);
			s1 += gs;
			s2 += gs * (ldf(x + o + j) - mean) * r;
		}
	s1 = RMS ? 0.f : bsum(s1, sh) * (1.f / inner);
	s2 = bsum(s2, sh) * (1.f / inner);
	if (vec)
		for (int j = 8 * threadIdx.x; j < inner; j += 8 * blockDim.x)
		{
			float gv[8], xv[8], sc[8];
			ld8(g + o + j, gv), ld8(x + o + j, xv);
			if (scale)
				ld8(scale + j, sc);
#pragma unroll
			for (int k = 0; k < 8; k++)
			{
				const float gs = gv[k] * (scale ? sc[k] : 1.f);
				gv[k] = r * (gs - s1 - (xv[k] - mean) * r * s2);
			}
			st8(dx + o + j, gv);
		}
	else
		for (int j = threadIdx.x; j < inner; j += blockDim.x)
		{
			const float gs = ldf(g + o + j) * (scale ? ldf(scale + j) : 1.f);
			const float d = r * (gs - s1 - (ldf(x + o + j) - mean) * r * s2);
			stf(dx + o + j, d);
		}
}
// dscale[j] = sum_rows g * xhat, dbias[j] = sum_rows g.  Row block y (rows y, y + gridDim.y, ..) leaves its two partial sums of column j
// in part[y][j] and part[y][inner + j] (fp32 whatever the operands' types); norm_bwd_dparam_rows_kernel then adds the gridDim.y rows in a
// fixed order and rounds once, so the result does not depend on the order in which blocks finish (one atomicAdd per (block, column) did).
static int dparam_row_blocks(int rows) { return rows < 296 ? rows : 296; }
size_t norm_bwd_workspace_bytes(int rows, int inner) { return rows <= 0 || inner <= 0 ? 0 : (size_t)dparam_row_blocks(rows) * 2 * (size_t)inner * sizeof(float); }
template <int RMS, typename TX, typename TS>
__global__ void norm_bwd_dparam_kernel(const TX* __restrict__ g, const TX* __restrict__ x, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, float* __restrict__ part, const int rows, const int inner)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= inner)
		return;
	float a = 0.f, b = 0.f;
	for (int r = blockIdx.y; r < rows; r += gridDim.y)
	{
		const float gv = ldf(g + (size_t)r * inner + j);
		a += gv * (ldf(x + (size_t)r * inner + j) - (RMS ? 0.f : ldf(saved_mean + r))) * ldf(saved_inv_std + r);
		b += gv;
	}
	float* const row = part + (size_t)blockIdx.y * 2 * inner;
	row[j] = a;
	if (!RMS)
		row[inner + j] = b;
}
// 32 columns x 32 row-lanes per block: lane l adds rows l, l + 32, .. in order, then the 32 lane sums are added in order
template <typename TDS, typename TDB>
__global__ void __launch_bounds__(1024) norm_bwd_dparam_rows_kernel(const float* __restrict__ part, const int gy, const int inner, TDS* __restrict__ dscale, TDB* __restrict__ dbias)
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
		stf(dscale + j, a);
	if (dbias)
		stf(dbias + j, b);
}
template <int RMS, typename TX, typename TP, typename TS, typename TDS, typename TDB>
static int norm_bwd(cudaStream_t s, const void* g, const void* x, const void* scale, const void* saved_mean, const void* saved_inv_std, void* dx, void* dscale, void* dbias, int rows, int inner, void* workspace)
{
	if (dx)
	{
		norm_bwd_dx_kernel<RMS, TX, TP, TS><<<rows, row_threads(inner), 0, s>>>((const TX*)g, (const TX*)x, (const TP*)scale, (const TS*)saved_mean, (const TS*)saved_inv_std, (TX*)dx, inner);
		if (launched("norm_bwd_dx"))
			return -1;
	}
	if (dscale || dbias)
	{
		const int gy = dparam_row_blocks(rows);
		norm_bwd_dparam_kernel<RMS, TX, TS><<<dim3((inner + 127) / 128, gy), 128, 0, s>>>((const TX*)g, (const TX*)x, (const TS*)saved_mean, (const TS*)saved_inv_std, (float*)workspace, rows, inner);
		if (launched("norm_bwd_dparam"))
			return -1;
		norm_bwd_dparam_rows_kernel<TDS, TDB><<<(inner + 31) / 32, 1024, 0, s>>>((const float*)workspace, gy, inner, (TDS*)dscale, (TDB*)dbias);
		if (launched("norm_bwd_dparam_rows"))
			return -1;
	}
	return 0;
}
template <int RMS>
static int norm_bwd_any(cudaStream_t s, const NormKinds& k, const void* g, const void* x, const void* scale, const void* saved_mean, const void* saved_inv_std, void* dx, void* dscale, void* dbias, int rows, int inner, void* workspace)
{
	if (rows <= 0 || inner <= 0)
		return 0;
	if ((dscale || dbias) && !workspace)
		return -1;
	return with_kind(k.x, [&](auto tx) {
		using TX = elem_t<decltype(tx)>;
		return with_kind_of<TX>(k.scale, [&](auto tp) {
			return with_kind_of<TX>(k.stat, [&](auto ts) {
				return with_kind_of<TX>(k.dscale, [&](auto tds) {
					return with_kind_of<TX>(RMS ? 0 : k.dbias, [&](auto tdb) {
						return norm_bwd<RMS, TX, elem_t<decltype(tp)>, elem_t<decltype(ts)>, elem_t<decltype(tds)>, elem_t<decltype(tdb)> >(s, g, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, inner, workspace);
					});
				});
			});
		});
	});
}
int layer_norm_bwd(cudaStream_t s, const NormKinds& k, const void* g, const void* x, const void* scale, const void* saved_mean, const void* saved_inv_std, void* dx, void* dscale, void* dbias, int rows, int inner, void* workspace)
{
	return norm_bwd_any<0>(s, k, g, x, scale, saved_mean, saved_inv_std, dx, dscale, dbias, rows, inner, workspace);
}
int rmsnorm_bwd(cudaStream_t s, const NormKinds& k, const void* g, const void* x, const void* scale, const void* saved_inv_std, void* dx, void* dscale, int rows, int inner, void* workspace)
{
	return norm_bwd_any<1>(s, k, g, x, scale, 0, saved_inv_std, dx, dscale, 0, rows, inner, workspace);
}

// ------------------------------------------------------------------------------------------------ upsample
// Every result is the reference's bit for bit: the source indices and coefficients use its arithmetic (double where it computes in
// double, each intermediate rounded where it rounds, nothing contracted into an FMA), the forward its association, and the
// backward sums each input element's contributions in the reference's order.
struct Coef {
	int i0, i1;
	float c0, c1;
};
// _ccv_nnc_init_bi_coeffs (upsample/ccv_nnc_upsample_cpu_ref.c:220-243): xs = i * s in float, or (i + 0.5) * s - 0.5 in double
// rounded to float once
__device__ __forceinline__ Coef bi_coef(const int i, const int ss, const float s, const int align_corners)
{
	const float xs = align_corners ? __fmul_rn((float)i, s) : (float)__dsub_rn(__dmul_rn(i + 0.5, (double)s), 0.5);
	Coef c;
	c.i0 = (int)xs;
	c.i1 = min((int)__fadd_rn(xs, 1.f), ss - 1);
	c.c1 = __fsub_rn(xs, (float)c.i0);
	c.c0 = __fsub_rn(1.f, c.c1);
	return c;
}
// upsample_cpu_ref.c:48,62: (int)((i + 0.5) * s) in double, or (int)(i * s + 0.5) with i * s in float and the sum in double.  In float
// alone (i + 0.5) * s can round up to an integer k that the double product stays below (6 -> 19 rows at i = 9).
__device__ __forceinline__ int nearest_idx(const int i, const int ss, const float s, const int align_corners)
{
	return min(align_corners ? (int)((double)__fmul_rn((float)i, s) + 0.5) : (int)__dmul_rn(i + 0.5, (double)s), ss - 1);
}
// thread per output element; NHWC: channels fastest (coalesced); NCHW: width fastest
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
		if (type == 0)
		{
			dst[i] = src[in_at(nearest_idx(oy, H, rh, align_corners), nearest_idx(ox, W, rw, align_corners))];
			continue;
		}
		const Coef cy = bi_coef(oy, H, rh, align_corners), cx = bi_coef(ox, W, rw, align_corners);
		const float a00 = src[in_at(cy.i0, cx.i0)], a01 = src[in_at(cy.i0, cx.i1)], a10 = src[in_at(cy.i1, cx.i0)], a11 = src[in_at(cy.i1, cx.i1)];
		float t00, t01, t10, t11;
		if (nchw) // ap1[si0] * sc0 * ysc0 + ... (upsample_cpu_ref.c:304-305)
			t00 = __fmul_rn(__fmul_rn(a00, cx.c0), cy.c0), t01 = __fmul_rn(__fmul_rn(a01, cx.c1), cy.c0), t10 = __fmul_rn(__fmul_rn(a10, cx.c0), cy.c1), t11 = __fmul_rn(__fmul_rn(a11, cx.c1), cy.c1);
		else // c00 = sc0 * ysc0, ap00[cd] * c00 + ... (:345-355)
			t00 = __fmul_rn(a00, __fmul_rn(cx.c0, cy.c0)), t01 = __fmul_rn(a01, __fmul_rn(cx.c1, cy.c0)), t10 = __fmul_rn(a10, __fmul_rn(cx.c0, cy.c1)), t11 = __fmul_rn(a11, __fmul_rn(cx.c1, cy.c1));
		dst[i] = __fadd_rn(__fadd_rn(__fadd_rn(t00, t01), t10), t11);
	}
}
// The output rows (columns) that read input row y form one range: f, the source row of an output row, is non-decreasing.  From an
// estimate o, the least o with f(o) >= y (O when there is none) and the greatest o with f(o) <= y (-1 when there is none).
template <typename F>
__device__ __forceinline__ int first_at_least(const F& f, const int y, int o, const int O)
{
	while (o > 0 && f(o - 1) >= y)
		o--;
	while (o < O && f(o) < y)
		o++;
	return o;
}
template <typename F>
__device__ __forceinline__ int last_at_most(const F& f, const int y, int o, const int O)
{
	while (o < O - 1 && f(o + 1) <= y)
		o++;
	while (o >= 0 && f(o) > y)
		o--;
	return o;
}
// where output row y / s lies, clamped to [0, O]
__device__ __forceinline__ int estimate(const double y, const float s, const int O)
{
	return s > 0 ? (int)fmin(fmax(y / s, 0.0), (double)O) : 0;
}
// thread per input element: the sum of the output gradients that read it, in output raster order and, within one output, over the
// corners 00, 01, 10, 11 -- the order the reference adds them in (upsample_cpu_ref.c:168-169, 204-205, 425-428, 478-481).  No atomics:
// the result is the same on every run.
__global__ void upsample_back_kernel(const float* __restrict__ g, float* __restrict__ h, const int N, const int H, const int W, const int C, const int OH, const int OW, const int type, const int align_corners, const int nchw, const float rh, const float rw)
{
	const size_t total = (size_t)N * H * W * C;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		int n, c, y, x;
		size_t r = i;
		if (nchw)
			x = r % W, r /= W, y = r % H, r /= H, c = r % C, n = (int)(r / C);
		else
			c = r % C, r /= C, x = r % W, r /= W, y = r % H, n = (int)(r / H);
		auto out_at = [&](int oy, int ox) -> size_t { return nchw ? (((size_t)n * C + c) * OH + oy) * OW + ox : (((size_t)n * OH + oy) * OW + ox) * C + c; };
		float acc = 0.f;
		if (type == 0)
		{
			auto fy = [&](int o) { return nearest_idx(o, H, rh, align_corners); };
			auto fx = [&](int o) { return nearest_idx(o, W, rw, align_corners); };
			const int y0 = first_at_least(fy, y, estimate(y, rh, OH), OH), y1 = last_at_most(fy, y, estimate(y + 1, rh, OH) - 1, OH);
			const int x0 = first_at_least(fx, x, estimate(x, rw, OW), OW), x1 = last_at_most(fx, x, estimate(x + 1, rw, OW) - 1, OW);
			for (int oy = y0; oy <= y1; oy++)
				for (int ox = x0; ox <= x1; ox++)
					acc = __fadd_rn(acc, g[out_at(oy, ox)]);
		} else {
			// an output reads row y when its i1 >= y and its i0 <= y, and then through one or both of its corner rows
			auto fy0 = [&](int o) { return bi_coef(o, H, rh, align_corners).i0; };
			auto fy1 = [&](int o) { return bi_coef(o, H, rh, align_corners).i1; };
			auto fx0 = [&](int o) { return bi_coef(o, W, rw, align_corners).i0; };
			auto fx1 = [&](int o) { return bi_coef(o, W, rw, align_corners).i1; };
			const int y0 = first_at_least(fy1, y, estimate(y - 1, rh, OH), OH), y1 = last_at_most(fy0, y, estimate(y + 1, rh, OH) - 1, OH);
			const int x0 = first_at_least(fx1, x, estimate(x - 1, rw, OW), OW), x1 = last_at_most(fx0, x, estimate(x + 1, rw, OW) - 1, OW);
			for (int oy = y0; oy <= y1; oy++)
			{
				const Coef cy = bi_coef(oy, H, rh, align_corners);
				for (int ox = x0; ox <= x1; ox++)
				{
					const Coef cx = bi_coef(ox, W, rw, align_corners);
					const float v = g[out_at(oy, ox)];
					for (int ry = 0; ry < 2; ry++)
						if ((ry ? cy.i1 : cy.i0) == y)
							for (int rx = 0; rx < 2; rx++)
								if ((rx ? cx.i1 : cx.i0) == x)
								{
									const float ysc = ry ? cy.c1 : cy.c0, xsc = rx ? cx.c1 : cx.c0;
									// NCHW: bp1[xd] * ysc * sc; NHWC: bp1[cd] * (sc * ysc)
									acc = __fadd_rn(acc, nchw ? __fmul_rn(__fmul_rn(v, ysc), xsc) : __fmul_rn(v, __fmul_rn(xsc, ysc)));
								}
				}
			}
		}
		h[i] = acc;
	}
}
static void ratios(int H, int W, int OH, int OW, int align_corners, float& rh, float& rw)
{
	rh = align_corners ? (float)(H - 1) / (OH - 1 > 1 ? OH - 1 : 1) : (float)H / OH;
	rw = align_corners ? (float)(W - 1) / (OW - 1 > 1 ? OW - 1 : 1) : (float)W / OW;
}
static unsigned upsample_blocks(const size_t total)
{
	const size_t blocks = (total + 255) / 256;
	return (unsigned)(blocks > 132 * 16 ? 132 * 16 : blocks);
}
int upsample_fwd_f32(cudaStream_t s, const float* a, float* b, int N, int H, int W, int C, int OH, int OW, int type, int align_corners, int nchw)
{
	const size_t total = (size_t)N * OH * OW * C;
	if (total == 0)
		return 0;
	float rh, rw;
	ratios(H, W, OH, OW, align_corners, rh, rw);
	upsample_kernel<<<upsample_blocks(total), 256, 0, s>>>(a, b, N, H, W, C, OH, OW, type, align_corners, nchw, rh, rw);
	return launched("upsample_fwd");
}
int upsample_bwd_f32(cudaStream_t s, const float* g, float* h, int N, int H, int W, int C, int OH, int OW, int type, int align_corners, int nchw)
{
	const size_t total = (size_t)N * H * W * C;
	if (total == 0)
		return 0;
	float rh, rw;
	ratios(H, W, OH, OW, align_corners, rh, rw);
	upsample_back_kernel<<<upsample_blocks(total), 256, 0, s>>>(g, h, N, H, W, C, OH, OW, type, align_corners, nchw, rh, rw);
	return launched("upsample_bwd");
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

// element types as for the row norms: TX x / y / grad / h, TP scale, TB bias, TS statistics, TDS dscale, TDB dbias
template <typename TX, typename TS>
__global__ void gn_stats_kernel(const GroupNormGeom g, const TX* __restrict__ x, TS* __restrict__ saved_mean, TS* __restrict__ saved_inv_std, const float epsilon)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.rdim, blockIdx.x);
	int c[4];
	float sum = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		sum += ldf(x + gn_offset(c, g.xstride));
	}
	const float inv_n = 1.f / (float)b.count;
	const float mean = gn_block_sum(sum, red) * inv_n;
	float sq = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const float w = ldf(x + gn_offset(c, g.xstride)) - mean;
		sq += w * w;
	}
	const float var = gn_block_sum(sq, red) * inv_n;
	if (threadIdx.x == 0)
	{
		stf(saved_mean + blockIdx.x, mean);
		stf(saved_inv_std + blockIdx.x, 1.f / sqrtf(var + epsilon));
	}
}

// y from the statistics as stored (what the backward reads)
template <typename TX, typename TP, typename TB, typename TS>
__global__ void gn_apply_kernel(const GroupNormGeom g, const TX* __restrict__ x, const TP* __restrict__ scale, const TB* __restrict__ bias, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, TX* __restrict__ y, const long long total)
{
	GnBox all;
	for (int d = 0; d < 4; d++)
		all.lo[d] = 0, all.ext[d] = g.dim[d];
	int c[4];
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		gn_coord(all, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		float v = (ldf(x + gn_offset(c, g.xstride)) - ldf(saved_mean + r)) * ldf(saved_inv_std + r);
		if (scale)
			v = v * ldf(scale + gn_slot(g, c, g.sdim)) + ldf(bias + gn_slot(g, c, g.sdim));
		stf(y + gn_offset(c, g.ystride), v);
	}
}

// per statistic slot: gssr = sum g * scale * inv_std, ahgssr = sum xhat * g * scale * inv_std (:412-470)
template <typename TX, typename TP, typename TS>
__global__ void gn_bwd_stats_kernel(const GroupNormGeom g, const TX* __restrict__ grad, const TX* __restrict__ x, const TP* __restrict__ scale, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, float* __restrict__ sums)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.rdim, blockIdx.x);
	const float mean = ldf(saved_mean + blockIdx.x), inv_std = ldf(saved_inv_std + blockIdx.x);
	int c[4];
	float s0 = 0, s1 = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const float ah = (ldf(x + gn_offset(c, g.xstride)) - mean) * inv_std;
		float gss = ldf(grad + gn_offset(c, g.ystride)) * inv_std;
		if (scale)
			gss *= ldf(scale + gn_slot(g, c, g.sdim));
		s0 += gss, s1 += ah * gss;
	}
	s0 = gn_block_sum(s0, red), s1 = gn_block_sum(s1, red);
	if (threadIdx.x == 0)
		sums[2 * blockIdx.x] = s0, sums[2 * blockIdx.x + 1] = s1;
}

// h = gss - (gssr + xhat * ahgssr) / n (:472-500)
template <typename TX, typename TP, typename TS>
__global__ void gn_bwd_apply_kernel(const GroupNormGeom g, const TX* __restrict__ grad, const TX* __restrict__ x, const TP* __restrict__ scale, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, const float* __restrict__ sums, TX* __restrict__ h, const long long total, const float inv_n)
{
	GnBox all;
	for (int d = 0; d < 4; d++)
		all.lo[d] = 0, all.ext[d] = g.dim[d];
	int c[4];
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		gn_coord(all, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		const float inv_std = ldf(saved_inv_std + r);
		const float ah = (ldf(x + gn_offset(c, g.xstride)) - ldf(saved_mean + r)) * inv_std;
		float gss = ldf(grad + gn_offset(c, g.ystride)) * inv_std;
		if (scale)
			gss *= ldf(scale + gn_slot(g, c, g.sdim));
		stf(h + gn_offset(c, g.hstride), gss - (sums[2 * r] + ah * sums[2 * r + 1]) * inv_n);
	}
}

// per scale / bias slot: dscale = sum xhat * g, dbias = sum g (:322-345, :254); fp32 sums in a fixed order, rounded once
template <typename TX, typename TS, typename TDS, typename TDB>
__global__ void gn_bwd_dparam_kernel(const GroupNormGeom g, const TX* __restrict__ grad, const TX* __restrict__ x, const TS* __restrict__ saved_mean, const TS* __restrict__ saved_inv_std, TDS* __restrict__ dscale, TDB* __restrict__ dbias)
{
	__shared__ float red[32];
	const GnBox b = gn_box(g, g.sdim, blockIdx.x);
	int c[4];
	float s0 = 0, s1 = 0;
	for (long long i = threadIdx.x; i < b.count; i += blockDim.x)
	{
		gn_coord(b, i, c);
		const long long r = gn_slot(g, c, g.rdim);
		const float gv = ldf(grad + gn_offset(c, g.ystride));
		s0 += (ldf(x + gn_offset(c, g.xstride)) - ldf(saved_mean + r)) * ldf(saved_inv_std + r) * gv;
		s1 += gv;
	}
	s0 = gn_block_sum(s0, red), s1 = gn_block_sum(s1, red);
	if (threadIdx.x == 0)
	{
		if (dscale)
			stf(dscale + blockIdx.x, s0);
		if (dbias)
			stf(dbias + blockIdx.x, s1);
	}
}

static long long gn_count(const int* d) { return (long long)d[0] * d[1] * d[2] * d[3]; }

template <typename TX, typename TP, typename TB, typename TS>
static int gn_fwd(cudaStream_t s, const GroupNormGeom& g, const void* x, const void* scale, const void* bias, void* y, void* saved_mean, void* saved_inv_std, float epsilon, long long total, long long slots)
{
	gn_stats_kernel<TX, TS><<<(unsigned)slots, 512, 0, s>>>(g, (const TX*)x, (TS*)saved_mean, (TS*)saved_inv_std, epsilon);
	count_launch();
	long long blocks = (total + 255) / 256;
	if (blocks > 132 * 16)
		blocks = 132 * 16;
	gn_apply_kernel<TX, TP, TB, TS><<<(unsigned)blocks, 256, 0, s>>>(g, (const TX*)x, (const TP*)scale, (const TB*)bias, (const TS*)saved_mean, (const TS*)saved_inv_std, (TX*)y, total);
	return launched("group_norm_fwd");
}

int group_norm_fwd(cudaStream_t s, const NormKinds& k, const GroupNormGeom& g, const void* x, const void* scale, const void* bias, void* y, void* saved_mean, void* saved_inv_std, float epsilon)
{
	const long long total = gn_count(g.dim), slots = gn_count(g.rdim);
	if (total == 0)
		return 0;
	return with_kind(k.x, [&](auto tx) {
		using TX = elem_t<decltype(tx)>;
		return with_kind_of<TX>(k.scale, [&](auto tp) {
			return with_kind_of<TX>(k.bias, [&](auto tb) {
				return with_kind_of<TX>(k.stat, [&](auto ts) {
					return gn_fwd<TX, elem_t<decltype(tp)>, elem_t<decltype(tb)>, elem_t<decltype(ts)> >(s, g, x, scale, bias, y, saved_mean, saved_inv_std, epsilon, total, slots);
				});
			});
		});
	});
}

size_t group_norm_bwd_workspace_bytes(const GroupNormGeom& g) { return (size_t)gn_count(g.rdim) * 2 * sizeof(float); }

template <typename TX, typename TP, typename TS, typename TDS, typename TDB>
static int gn_bwd(cudaStream_t s, const GroupNormGeom& g, const void* grad, const void* x, const void* scale, const void* saved_mean, const void* saved_inv_std, void* h, void* dscale, void* dbias, void* workspace, long long total, long long slots)
{
	if (h)
	{
		float* const sums = (float*)workspace;
		gn_bwd_stats_kernel<TX, TP, TS><<<(unsigned)slots, 512, 0, s>>>(g, (const TX*)grad, (const TX*)x, (const TP*)scale, (const TS*)saved_mean, (const TS*)saved_inv_std, sums);
		if (launched("group_norm_bwd_stats"))
			return -1;
		long long blocks = (total + 255) / 256;
		if (blocks > 132 * 16)
			blocks = 132 * 16;
		gn_bwd_apply_kernel<TX, TP, TS><<<(unsigned)blocks, 256, 0, s>>>(g, (const TX*)grad, (const TX*)x, (const TP*)scale, (const TS*)saved_mean, (const TS*)saved_inv_std, sums, (TX*)h, total, (float)slots / (float)total);
		if (launched("group_norm_bwd_apply"))
			return -1;
	}
	if (dscale || dbias)
	{
		gn_bwd_dparam_kernel<TX, TS, TDS, TDB><<<(unsigned)gn_count(g.sdim), 256, 0, s>>>(g, (const TX*)grad, (const TX*)x, (const TS*)saved_mean, (const TS*)saved_inv_std, (TDS*)dscale, (TDB*)dbias);
		if (launched("group_norm_bwd_dparam"))
			return -1;
	}
	return 0;
}

int group_norm_bwd(cudaStream_t s, const NormKinds& k, const GroupNormGeom& g, const void* grad, const void* x, const void* scale, const void* saved_mean, const void* saved_inv_std, void* h, void* dscale, void* dbias, void* workspace)
{
	const long long total = gn_count(g.dim), slots = gn_count(g.rdim);
	if (total == 0)
		return 0;
	return with_kind(k.x, [&](auto tx) {
		using TX = elem_t<decltype(tx)>;
		return with_kind_of<TX>(k.scale, [&](auto tp) {
			return with_kind_of<TX>(k.stat, [&](auto ts) {
				return with_kind_of<TX>(k.dscale, [&](auto tds) {
					return with_kind_of<TX>(k.dbias, [&](auto tdb) {
						return gn_bwd<TX, elem_t<decltype(tp)>, elem_t<decltype(ts)>, elem_t<decltype(tds)>, elem_t<decltype(tdb)> >(s, g, grad, x, scale, saved_mean, saved_inv_std, h, dscale, dbias, workspace, total, slots);
					});
				});
			});
		});
	});
}

} // namespace sm100
