// sm100_ffma.cu -- CUDA-core fp32 contractions (CCV_NNC_SM100_ALGO_FFMA): the shape-agnostic companions of the
// wgmma path.  They take any stride / alignment / channel count (e.g. the 3-channel stem convolution, grouped
// convolutions, tensor views) and compute exact fp32 products, so they also serve as the on-device cross-check of
// the tensor-core kernels.  One tiled SIMT GEMM (64 x 64 x 16, 4 x 4 register micro-tiles) is instantiated with
// different operand "views" (functors mapping (row, k) / (k, col) to memory), which is how implicit-GEMM
// convolution forward / data-gradient / weight-gradient reuse it.
// Reference semantics: lib/nnc/cmd/blas/ccv_nnc_gemm_cpu_ref.c:110-448, lib/nnc/cmd/convolution/ccv_nnc_conv_cpu_ref.c:13-345.
#include "sm100_contract.h"

namespace sm100 {

struct StridedView {
	const float* p;
	long long rs, cs;
	int rows, cols;
	__device__ __forceinline__ float operator()(int r, int c) const { return (r < rows && c < cols) ? __ldg(p + r * rs + c * cs) : 0.f; }
};

// A(m, k) for convolution forward: m = output pixel (n, p, q), k = (r, s, c) of one group
struct Im2colRows {
	const float* x;
	int H, W, Cg, R, S, P, Q, M;
	int sh, sw, ph, pw, dh, dw;
	long long xn, xh, xw;
	__device__ __forceinline__ float operator()(int m, int k) const
	{
		if (m >= M || k >= R * S * Cg)
			return 0.f;
		const int c = k % Cg;
		const int t = k / Cg;
		const int s = t % S, r = t / S;
		const int q = m % Q;
		const int u = m / Q;
		const int pp = u % P, n = u / P;
		const int h = pp * sh - ph + r * dh, w = q * sw - pw + s * dw;
		if (h < 0 || h >= H || w < 0 || w >= W)
			return 0.f;
		return __ldg(x + n * xn + h * xh + w * xw + c);
	}
};

// A(m, k) for the data gradient: m = input pixel (n, h, w), k = (r, s, ko); reads grad_b where the stride divides
struct DgradRows {
	const float* g;
	int H, W, Kg, R, S, P, Q, M;
	int sh, sw, ph, pw, dh, dw;
	long long gn, gh, gw;
	__device__ __forceinline__ float operator()(int m, int k) const
	{
		if (m >= M || k >= R * S * Kg)
			return 0.f;
		const int ko = k % Kg;
		const int t = k / Kg;
		const int s = t % S, r = t / S;
		const int w = m % W;
		const int u = m / W;
		const int h = u % H, n = u / H;
		const int hn = h + ph - r * dh, wn = w + pw - s * dw;
		if (hn < 0 || wn < 0 || hn % sh || wn % sw)
			return 0.f;
		const int pp = hn / sh, q = wn / sw;
		if (pp >= P || q >= Q)
			return 0.f;
		return __ldg(g + n * gn + pp * gh + q * gw + ko);
	}
};

// B(k, n) for the data gradient: k = (r, s, ko), n = c ; filters w[K, R, S, Cg]
struct DgradFilter {
	const float* w;
	int Kg, R, S, Cg;
	__device__ __forceinline__ float operator()(int k, int n) const
	{
		if (k >= R * S * Kg || n >= Cg)
			return 0.f;
		const int ko = k % Kg;
		const int t = k / Kg;
		return __ldg(w + ((long long)ko * R * S + t) * Cg + n);
	}
};

// B(k, n) for the weight gradient: k = output pixel, n = (r, s, c)
struct Im2colCols {
	Im2colRows v;
	__device__ __forceinline__ float operator()(int k, int n) const { return v(k, n); }
};

template <class AV, class BV>
__global__ void __launch_bounds__(256) ffma_gemm_kernel(const AV A, const BV B, float* __restrict__ C, const long long ldc, const float* __restrict__ bias, const int M, const int N, const int K, const int k_per_split, const int accumulate, const long long split_stride)
{
	C += blockIdx.z * split_stride;
	__shared__ float As[16][64 + 4];
	__shared__ float Bs[16][64 + 4];
	const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
	const int k_begin = blockIdx.z * k_per_split;
	const int k_end = min(K, k_begin + k_per_split);
	float acc[4][4];
#pragma unroll
	for (int i = 0; i < 4; i++)
#pragma unroll
		for (int j = 0; j < 4; j++)
			acc[i][j] = 0.f;
	for (int k0 = k_begin; k0 < k_end; k0 += 16)
	{
		// 64 x 16 of A and 16 x 64 of B, 4 elements per thread each
#pragma unroll
		for (int i = 0; i < 4; i++)
		{
			const int e = threadIdx.x + i * 256;
			const int ak = e & 15, am = e >> 4;
			As[ak][am] = (k0 + ak < k_end) ? A(m0 + am, k0 + ak) : 0.f;
			const int bn = e & 63, bk = e >> 6;
			Bs[bk][bn] = (k0 + bk < k_end) ? B(k0 + bk, n0 + bn) : 0.f;
		}
		__syncthreads();
#pragma unroll
		for (int kk = 0; kk < 16; kk++)
		{
			float a[4], b[4];
#pragma unroll
			for (int i = 0; i < 4; i++)
				a[i] = As[kk][ty * 4 + i], b[i] = Bs[kk][tx * 4 + i];
#pragma unroll
			for (int i = 0; i < 4; i++)
#pragma unroll
				for (int j = 0; j < 4; j++)
					acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
		}
		__syncthreads();
	}
#pragma unroll
	for (int i = 0; i < 4; i++)
	{
		const int m = m0 + ty * 4 + i;
		if (m >= M)
			continue;
#pragma unroll
		for (int j = 0; j < 4; j++)
		{
			const int n = n0 + tx * 4 + j;
			if (n >= N)
				continue;
			float v = acc[i][j];
			if (bias && blockIdx.z == 0)
				v += bias[n];
			float* o = C + m * ldc + n;
			*o = accumulate ? *o + v : v;
		}
	}
}

// splits > 1: each split writes its partial products to its own fp32 slice [M, ldp] of the scratch, and splitk_reduce adds the
// slices into C in split order (bit-identical from run to run, unlike atomic adds); as many splits as the scratch holds
template <class AV, class BV>
static int launch_ffma(cudaStream_t stream, const AV& A, const BV& B, float* C, long long ldc, const float* bias, int M, int N, int K, int accumulate, int splits, const Scratch& scratch)
{
	if (M <= 0 || N <= 0)
		return 0;
	const long long ldp = ((long long)N + 3) & ~3ll;
	const size_t slice = (size_t)M * ldp * sizeof(float);
	if (splits > 1 && (long long)splits > (long long)((scratch.ptr ? scratch.bytes : 0) / slice))
		splits = (int)((scratch.ptr ? scratch.bytes : 0) / slice);
	int k_per = K;
	if (splits > 1)
	{
		k_per = ((K + splits - 1) / splits + 15) / 16 * 16;
		splits = (K + k_per - 1) / k_per;
	}
	if (splits < 1)
		splits = 1;
	dim3 grid((N + 63) / 64, (M + 63) / 64, splits);
	if (splits > 1)
		ffma_gemm_kernel<AV, BV><<<grid, 256, 0, stream>>>(A, B, (float*)scratch.ptr, ldp, bias, M, N, K, k_per, 0, (long long)M * ldp);
	else
		ffma_gemm_kernel<AV, BV><<<grid, 256, 0, stream>>>(A, B, C, ldc, bias, M, N, K, k_per, accumulate, 0);
	count_launch();
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		set_last_error("ffma_gemm_kernel launch", e);
		return -1;
	}
	return splits > 1 ? splitk_reduce(stream, (const float*)scratch.ptr, splits, (long long)M * ldp, M, N, ldp, C, ldc, accumulate) : 0;
}

int gemm_ffma(cudaStream_t stream, int M, int N, int K, const float* a, long long a_rs, long long a_cs, const float* b, long long b_rs, long long b_cs, float* c, long long ldc, const float* bias, int accumulate, const Scratch& scratch)
{
	StridedView A = { a, a_rs, a_cs, M, K };
	StridedView B = { b, b_rs, b_cs, K, N };
	const long long tiles = (long long)((M + 63) / 64) * ((N + 63) / 64);
	int splits = 1;
	if (tiles < 132 && K >= 1024)
		splits = (int)((264 + tiles - 1) / tiles);
	if (splits > K / 256)
		splits = K / 256 > 0 ? K / 256 : 1;
	return launch_ffma(stream, A, B, c, ldc, bias, M, N, K, accumulate, splits, scratch);
}

static Im2colRows im2col_view(const ConvGeom& g, int groups, const float* a, int group)
{
	Im2colRows v;
	v.x = a + (long long)group * (g.C / groups);
	v.H = g.H, v.W = g.W, v.Cg = g.C / groups, v.R = g.R, v.S = g.S, v.P = g.P, v.Q = g.Q, v.M = g.N * g.P * g.Q;
	v.sh = g.stride_h, v.sw = g.stride_w, v.ph = g.pad_h0, v.pw = g.pad_w0, v.dh = g.dil_h, v.dw = g.dil_w;
	v.xn = g.an, v.xh = g.ah, v.xw = g.aw;
	return v;
}

int conv_fprop_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* a, const float* w, const float* bias, float* b)
{
	const int Cg = g.C / groups, Kg = g.K / groups;
	if (g.bh != (long long)g.Q * g.bw || g.bn != (long long)g.P * g.bh) // outputs are rows of a pitched [NPQ, K] matrix
		return 1;
	for (int gr = 0; gr < groups; gr++)
	{
		Im2colRows A = im2col_view(g, groups, a, gr);
		// w[K, R, S, Cg]: B(k, n) = w[(gr * Kg + n), k]
		StridedView B = { w + (long long)gr * Kg * g.R * g.S * Cg, 1, (long long)g.R * g.S * Cg, g.R * g.S * Cg, Kg };
		const int rc = launch_ffma(stream, A, B, b + gr * Kg, g.bw, bias ? bias + gr * Kg : 0, g.N * g.P * g.Q, Kg, g.R * g.S * Cg, 0, 1, Scratch());
		if (rc)
			return rc;
	}
	return 0;
}

int conv_dgrad_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* grad_b, const float* w, float* grad_a)
{
	const int Cg = g.C / groups, Kg = g.K / groups;
	if (g.ah != (long long)g.W * g.aw || g.an != (long long)g.H * g.ah)
		return 1;
	for (int gr = 0; gr < groups; gr++)
	{
		DgradRows A;
		A.g = grad_b + gr * Kg;
		A.H = g.H, A.W = g.W, A.Kg = Kg, A.R = g.R, A.S = g.S, A.P = g.P, A.Q = g.Q, A.M = g.N * g.H * g.W;
		A.sh = g.stride_h, A.sw = g.stride_w, A.ph = g.pad_h0, A.pw = g.pad_w0, A.dh = g.dil_h, A.dw = g.dil_w;
		A.gn = g.bn, A.gh = g.bh, A.gw = g.bw;
		DgradFilter B = { w + (long long)gr * Kg * g.R * g.S * Cg, Kg, g.R, g.S, Cg };
		const int rc = launch_ffma(stream, A, B, grad_a + gr * Cg, g.aw, 0, g.N * g.H * g.W, Cg, g.R * g.S * Kg, 0, 1, Scratch());
		if (rc)
			return rc;
	}
	return 0;
}

int conv_wgrad_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* grad_b, const float* a, float* grad_w, int accumulate, const Scratch& scratch)
{
	const int Cg = g.C / groups, Kg = g.K / groups;
	const int npq = g.N * g.P * g.Q;
	for (int gr = 0; gr < groups; gr++)
	{
		// A(m = ko, k = pixel) = grad_b[pixel, gr * Kg + ko]; requires grad_b rows at a constant pitch
		if (g.bh != (long long)g.Q * g.bw || g.bn != (long long)g.P * g.bh)
			return 1;
		StridedView A = { grad_b + gr * Kg, 1, g.bw, Kg, npq };
		Im2colCols B = { im2col_view(g, groups, a, gr) };
		const int rsc = g.R * g.S * Cg;
		const long long tiles = (long long)((Kg + 63) / 64) * ((rsc + 63) / 64);
		int splits = (int)((592 + tiles - 1) / tiles);
		if (splits > npq / 512)
			splits = npq / 512 > 0 ? npq / 512 : 1;
		const int rc = launch_ffma(stream, A, B, grad_w + (long long)gr * Kg * rsc, rsc, 0, Kg, rsc, npq, accumulate, splits, scratch);
		if (rc)
			return rc;
	}
	return 0;
}

} // namespace sm100
