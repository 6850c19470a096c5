// sm100_sdpa.cu -- SCALED_DOT_PRODUCT_ATTENTION forward / backward, composed per (batch, head) from the tensor-core GEMM
// (wgmma TF32) and two row kernels (masked / causal softmax, softmax gradient), i.e. the same decomposition the
// reference's own unit test checks the fused op against (test/unit/nnc/attention.tests.c:14-468).  The score matrix of
// one (batch, head) lives in the stream workspace.  Semantics: scaled_dot_product_attention/
// ccv_nnc_scaled_dot_product_attention_cpu_ref.c:16-257 (forward), :259-479 (backward); causal masks are aligned to
// the bottom-right (x_end = max(x - Sq + Sk + 1, 0), :147); GQA maps query head h to kv head h / (Hq / Hk).
// 16-bit tensors take the single-kernel flash attention of sm100_fmha.cu instead.
#include "sm100_contract.h"
#include "sm100_ew.h"
#include <float.h>

namespace sm100 {

// the attention scores already occupy the command's workspace: these products run without split-K slices
static const Scratch no_scratch = { 0, 0 };

__device__ __forceinline__ float wsum_(float v)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		v += __shfl_xor_sync(0xffffffff, v, o);
	return v;
}
__device__ __forceinline__ float wmax_(float v)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		v = fmaxf(v, __shfl_xor_sync(0xffffffff, v, o));
	return v;
}
__device__ __forceinline__ float bsum_(float v, float* sh)
{
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	v = wsum_(v);
	__syncthreads();
	if (lane == 0)
		sh[w] = v;
	__syncthreads();
	return wsum_(lane < nw ? sh[lane] : 0.f);
}
__device__ __forceinline__ float bmax_(float v, float* sh)
{
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
	v = wmax_(v);
	__syncthreads();
	if (lane == 0)
		sh[w] = v;
	__syncthreads();
	return wmax_(lane < nw ? sh[lane] : -FLT_MAX);
}

// one block per query row x: s[x, :] <- softmax(scale * s[x, :] + mask[x, :]) over y < x_end, 0 beyond (causal)
__global__ void sdpa_softmax_kernel(float* __restrict__ s, const int sq, const int sk, const float scale, const float* __restrict__ mask, const long long mask_row_stride, const int mask_col_stride, const int is_causal)
{
	__shared__ float sh[32];
	const int x = blockIdx.x;
	float* const row = s + (size_t)x * sk;
	const int x_end = is_causal ? max(x - sq + sk + 1, 0) : sk;
	const float* const mrow = mask ? mask + (size_t)x * mask_row_stride : 0;
	float m = -FLT_MAX;
	for (int y = threadIdx.x; y < x_end; y += blockDim.x)
	{
		const float v = scale * row[y] + (mrow ? mrow[(size_t)y * mask_col_stride] : 0.f);
		row[y] = v;
		m = fmaxf(m, v);
	}
	m = bmax_(m, sh);
	float sum = 0.f;
	for (int y = threadIdx.x; y < x_end; y += blockDim.x)
	{
		const float e = expf(row[y] - m);
		row[y] = e;
		sum += e;
	}
	sum = bsum_(sum, sh);
	const float inv = 1.f / sum;
	for (int y = threadIdx.x; y < sk; y += blockDim.x)
		row[y] = y < x_end ? row[y] * inv : 0.f;
}

// ds[x, y] = scale * (dp[x, y] - sum_y dp[x, y] * p[x, y]) * p[x, y]   (written over dp)
__global__ void sdpa_dsoftmax_kernel(const float* __restrict__ p, float* __restrict__ dp, const int sk, const float scale)
{
	__shared__ float sh[32];
	const size_t o = (size_t)blockIdx.x * sk;
	float sum = 0.f;
	for (int y = threadIdx.x; y < sk; y += blockDim.x)
		sum += dp[o + y] * p[o + y];
	sum = bsum_(sum, sh);
	for (int y = threadIdx.x; y < sk; y += blockDim.x)
		dp[o + y] = scale * (dp[o + y] - sum) * p[o + y];
}

static int row_threads(int n) { return n >= 2048 ? 512 : (n >= 512 ? 256 : (n >= 128 ? 128 : 64)); }

size_t sdpa_workspace_bytes(int sq, int sk, int backward) { return (size_t)sq * sk * sizeof(float) * (backward ? 2 : 1) + 256; }

// strides are in elements; q: [B, Sq, H, D], k/v: [B, Sk, Hk, D / Dv], o: [B, Sq, H, Dv]
int sdpa_forward_f32(cudaStream_t s, const SdpaGeom& g, const float* q, const float* k, const float* v, const float* mask, float* o, void* workspace)
{
	float* const S = (float*)workspace;
	const int ratio = g.H / g.Hk;
	for (int b = 0; b < g.B; b++)
		for (int h = 0; h < g.H; h++)
		{
			const float* qp = q + b * g.q_b + h * g.q_h;
			const float* kp = k + b * g.k_b + (h / ratio) * g.k_h;
			const float* vp = v + b * g.v_b + (h / ratio) * g.v_h;
			float* op = o + b * g.o_b + h * g.o_h;
			// S = Q K^T
			int rc = gemm_any(s, 0, g.Sq, g.Sk, g.D, qp, g.q_s, 0, kp, g.k_s, 1, S, g.Sk, 0, 0, 0, no_scratch);
			if (rc > 0)
				rc = gemm_ffma(s, g.Sq, g.Sk, g.D, qp, g.q_s, 1, kp, 1, g.k_s, S, g.Sk, 0, 0);
			if (rc)
				return rc;
			const float* mp = mask ? mask + (g.mask_b ? b * g.mask_b : 0) + (g.mask_h ? h * g.mask_h : 0) : 0;
			sdpa_softmax_kernel<<<g.Sq, row_threads(g.Sk), 0, s>>>(S, g.Sq, g.Sk, g.scale, mp, g.mask_s, g.mask_c, g.is_causal);
			if (launched("sdpa_softmax"))
				return -1;
			// O = P V
			rc = gemm_any(s, 0, g.Sq, g.Dv, g.Sk, S, g.Sk, 0, vp, g.v_s, 0, op, g.o_s, 0, 0, 0, no_scratch);
			if (rc > 0)
				rc = gemm_ffma(s, g.Sq, g.Dv, g.Sk, S, g.Sk, 1, vp, g.v_s, 1, op, g.o_s, 0, 0);
			if (rc)
				return rc;
		}
	return 0;
}

static int mm(cudaStream_t s, int M, int N, int K, const float* a, long long lda, int ta, const float* b, long long ldb, int tb, float* c, long long ldc, int accumulate)
{
	int rc = gemm_any(s, 0, M, N, K, a, lda, ta, b, ldb, tb, c, ldc, 0, 0, accumulate, no_scratch);
	if (rc > 0)
		rc = gemm_ffma(s, M, N, K, a, ta ? 1 : lda, ta ? lda : 1, b, tb ? 1 : ldb, tb ? ldb : 1, c, ldc, 0, accumulate);
	return rc;
}

// dq, dk, dv from dO, q, k, v; the softmax is recomputed (the reference does the same, :261); no mask support (:262)
int sdpa_backward_f32(cudaStream_t s, const SdpaGeom& g, const float* dout, const float* q, const float* k, const float* v, float* dq, float* dk, float* dv, const SdpaGeom& dg, void* workspace)
{
	float* const P = (float*)workspace;
	float* const dP = P + (size_t)g.Sq * g.Sk;
	const int ratio = g.H / g.Hk;
	for (int b = 0; b < g.B; b++)
		for (int h = 0; h < g.H; h++)
		{
			const int hk = h / ratio;
			const int first = (h % ratio) == 0; // the first query head of a kv group overwrites dk / dv, the rest accumulate (:388-401)
			const float* qp = q + b * g.q_b + h * g.q_h;
			const float* kp = k + b * g.k_b + hk * g.k_h;
			const float* vp = v + b * g.v_b + hk * g.v_h;
			const float* gp = dout + b * g.o_b + h * g.o_h;
			float* dqp = dq + b * dg.q_b + h * dg.q_h;
			float* dkp = dk + b * dg.k_b + hk * dg.k_h;
			float* dvp = dv + b * dg.v_b + hk * dg.v_h;
			int rc = mm(s, g.Sq, g.Sk, g.D, qp, g.q_s, 0, kp, g.k_s, 1, P, g.Sk, 0); // S = Q K^T
			if (rc)
				return rc;
			sdpa_softmax_kernel<<<g.Sq, row_threads(g.Sk), 0, s>>>(P, g.Sq, g.Sk, g.scale, 0, 0, 0, g.is_causal);
			if (launched("sdpa_softmax(bwd)"))
				return -1;
			rc = mm(s, g.Sk, g.Dv, g.Sq, P, g.Sk, 1, gp, g.o_s, 0, dvp, dg.v_s, !first); // dV (+)= P^T dO
			if (rc)
				return rc;
			rc = mm(s, g.Sq, g.Sk, g.Dv, gp, g.o_s, 0, vp, g.v_s, 1, dP, g.Sk, 0); // dP = dO V^T
			if (rc)
				return rc;
			sdpa_dsoftmax_kernel<<<g.Sq, row_threads(g.Sk), 0, s>>>(P, dP, g.Sk, g.scale);
			if (launched("sdpa_dsoftmax"))
				return -1;
			rc = mm(s, g.Sq, g.D, g.Sk, dP, g.Sk, 0, kp, g.k_s, 0, dqp, dg.q_s, 0); // dQ = dS K
			if (rc)
				return rc;
			rc = mm(s, g.Sk, g.D, g.Sq, dP, g.Sk, 1, qp, g.q_s, 0, dkp, dg.k_s, !first); // dK (+)= dS^T Q
			if (rc)
				return rc;
		}
	return 0;
}

} // namespace sm100
