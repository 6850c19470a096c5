// sm100_backend.cu -- group (A) of include/ccv_nnc_sm100.h: the command layer of CCV_NNC_BACKEND_GPU_SM100.
//
// One exec function per command, with the reference's signature (lib/nnc/ccv_nnc.h:315) and positional tensor
// conventions (lib/nnc/ccv_nnc.h:308-314), and one registration function per command spelled exactly as
// REGISTER_COMMAND_BACKEND(cmd, CCV_NNC_BACKEND_GPU_SM100) would (lib/nnc/ccv_nnc_internal.h:196-202).  An exec only
// validates shapes, pulls the CUDA stream / workspace from the stream context and enqueues kernels; it never
// synchronises and there is no CPU path: anything it cannot run returns CCV_NNC_EXEC_INVALID.
#include "sm100_cmd.h"
#include "sm100_ew.h"
#include <cuda_runtime.h>
#include <string.h>
#include <algorithm>
#include <vector>

using namespace sm100;

namespace {

struct TV {
	unsigned char* p;
	int nd;
	int dim[CCV_NNC_MAX_DIM_ALLOC];
	int stride[CCV_NNC_MAX_DIM_ALLOC];
	int contiguous;
	int datatype;
	int format;
	size_t count;
};

// ccv_nnc_tensor_view_get_stride (lib/nnc/ccv_nnc_easy.h): a view carries its strides, a plain tensor is packed
TV view_of(const ccv_nnc_tensor_t* const t)
{
	TV v;
	memset(&v, 0, sizeof(v));
	v.p = t->data.u8;
	v.nd = nd_of(t);
	v.datatype = CCV_GET_DATA_TYPE(t->info.datatype);
	v.format = t->info.format;
	v.count = 1;
	int i;
	for (i = 0; i < v.nd; i++)
		v.dim[i] = t->info.dim[i], v.count *= (size_t)t->info.dim[i];
	if (CCV_IS_TENSOR_VIEW(t))
	{
		const ccv_nnc_tensor_view_t* const tv = (const ccv_nnc_tensor_view_t*)t;
		int packed = 1;
		v.contiguous = 1;
		for (i = v.nd - 1; i >= 0; i--)
		{
			v.stride[i] = tv->stride[i];
			if (v.dim[i] != 1 && tv->stride[i] != packed)
				v.contiguous = 0;
			packed *= v.dim[i];
		}
	} else {
		int packed = 1;
		for (i = v.nd - 1; i >= 0; i--)
			v.stride[i] = packed, packed *= v.dim[i];
		v.contiguous = 1;
	}
	return v;
}

// ccv_nnc_tensor_view_get_dim: right-align into 4 dims with leading 1s
void dims4(const TV& v, int dim[4], int stride[4])
{
	const int off = 4 - v.nd;
	int i;
	for (i = 0; i < 4; i++)
	{
		if (i < off)
			dim[i] = 1, stride[i] = 0;
		else
			dim[i] = v.dim[i - off], stride[i] = v.stride[i - off];
	}
}

// split-K scratch of a command that no staging layer wraps: the stream workspace (grow-only, one buffer per stream:
// lib/nnc/gpu/ccv_nnc_compat.cu:438-471).  The wrapped commands carve it out of their one workspace request (scratch_at).
inline Scratch scratch_of(ccv_nnc_stream_context_t* const stream_context)
{
	void* const p = ccv_nnc_stream_context_get_workspace(stream_context, CONTRACT_SCRATCH_BYTES, CCV_TENSOR_GPU_MEMORY);
	const Scratch s = { p, p ? CONTRACT_SCRATCH_BYTES : 0 };
	return s;
}
inline Scratch scratch_at(void* const p, const size_t bytes)
{
	const Scratch s = { p, p ? bytes : 0 };
	return s;
}

inline bool is_f32(const ccv_nnc_tensor_t* const t) { return CCV_GET_DATA_TYPE(t->info.datatype) == CCV_32F; }
inline uint16_t f32_to_16(const float v, const int kind); // host-side rounding of a fill value (defined with exec_via_f32)

bool same_shape(const TV& a, const TV& b)
{
	if (a.nd != b.nd)
		return false;
	for (int i = 0; i < a.nd; i++)
		if (a.dim[i] != b.dim[i])
			return false;
	return true;
}

int dtype_code(const int datatype)
{
	switch (CCV_GET_DATA_TYPE(datatype))
	{
		case CCV_32F: return 0;
		case CCV_16F: return 1;
		case CCV_64F: return 2;
		case CCV_16BF: return 3;
	}
	return -1;
}

size_t dtype_size(const int datatype)
{
	switch (CCV_GET_DATA_TYPE(datatype))
	{
		case CCV_8U: return 1;
		case CCV_16F: case CCV_16BF: return 2;
		case CCV_32F: case CCV_32S: return 4;
		case CCV_64F: case CCV_64S: return 8;
	}
	return 0;
}

#define RC(x) do { const int rc_ = (x); if (rc_ < 0) return CCV_NNC_EXEC_INVALID; if (rc_ > 0) return CCV_NNC_EXEC_INVALID; } while (0)

// ================================================================================================ GEMM
struct Mat {
	unsigned char* p;
	size_t esz; // bytes per element
	int batch, rows, cols;
	long long batch_inc, rs, cs;
};
// the matrix of batch entry i
inline unsigned char* at(const Mat& m, const int i) { return m.p + i * m.batch_inc * (long long)m.esz; }

// ccv_nnc_tensor_get_matrix_params (lib/nnc/ccv_nnc_easy.h:421-444) for nd <= 3
bool mat_of(const TV& v, const int transpose[2], Mat& m)
{
	if (v.nd < 1 || v.nd > 3)
		return false;
	m.p = v.p;
	m.esz = dtype_size(v.datatype);
	m.batch = v.nd < 3 ? 1 : v.dim[v.nd - 3];
	m.batch_inc = v.nd < 3 ? 0 : v.stride[v.nd - 3];
	m.rows = v.nd == 1 ? 1 : v.dim[v.nd - 2];
	m.rs = v.nd >= 2 ? v.stride[v.nd - 2] : (long long)v.stride[0] * v.dim[0];
	m.cols = v.dim[v.nd - 1];
	m.cs = v.stride[v.nd - 1];
	if (transpose[0] != transpose[1])
	{
		const int t = m.rows;
		m.rows = m.cols, m.cols = t;
		const long long u = m.rs;
		m.rs = m.cs, m.cs = u;
	}
	return true;
}

// Algorithm of a GEMM command.  An explicit cmd.algorithm (what ccv_nnc_cmd_autotune stores) wins; otherwise fp32 data means
// fp32-grade products -- the reference's cuBLAS path computes fp32 GEMMs in CUBLAS_COMPUTE_32F
// (lib/nnc/gpu/ccv_nnc_compat.cu:786-803) -- i.e. the error-compensated 3xTF32 kernel, unless the caller opted into TF32 with
// CCV_NNC_GEMM_32TF (lib/nnc/ccv_nnc.h:103-105).
int gemm_algorithm(const ccv_nnc_cmd_t& cmd)
{
	if (cmd.algorithm >= 0 && cmd.algorithm < CCV_NNC_SM100_ALGO_COUNT)
		return cmd.algorithm;
	return (cmd.info.blas.flags & CCV_NNC_GEMM_32TF) ? CCV_NNC_SM100_ALGO_TF32 : CCV_NNC_SM100_ALGO_3XTF32;
}
// Algorithm of a CONVOLUTION command: explicit, else one-pass TF32 -- the reference's own GPU convolution sets
// CUDNN_TENSOR_OP_MATH on every convolution descriptor (lib/nnc/gpu/ccv_nnc_compat.cu:1393), which is TF32 tensor-core math
// for fp32 data; CCV_NNC_SM100_ALGO_3XTF32 / _FFMA are there for callers that need fp32-grade convolutions.
int conv_algorithm(const ccv_nnc_cmd_t& cmd)
{
	if (cmd.algorithm >= 0 && cmd.algorithm < CCV_NNC_SM100_ALGO_COUNT)
		return cmd.algorithm;
	return CCV_NNC_SM100_ALGO_TF32;
}

// C[M, N] (+)= A[M, K] * B[K, N] + bias over arbitrary (row, col) element strides, element kind `kind` (0 = fp32, 1 = bf16,
// 2 = fp16; the algorithm only matters for fp32); bias fp32 (bias32) or of the 16-bit kind (bias16)
int gemm_dispatch(cudaStream_t s, const Scratch& scratch, const int kind, const int algorithm, const int M, const int N, const int K, const void* a, long long a_rs, long long a_cs, const void* b, long long b_rs, long long b_cs, void* c, long long c_rs, long long c_cs, const float* bias32, const void* bias16, const int accumulate)
{
	if (M <= 0 || N <= 0)
		return 0;
	if (K <= 0)
		return 1;
	if (c_cs != 1 && N > 1)
	{
		if ((c_rs != 1 && M > 1) || bias32 || bias16)
			return 1;
		return gemm_dispatch(s, scratch, kind, algorithm, N, M, K, b, b_cs, b_rs, a, a_cs, a_rs, c, c_cs, 1, 0, 0, accumulate); // C^T = B^T A^T
	}
	if (kind != 0 || algorithm != CCV_NNC_SM100_ALGO_FFMA)
	{
		int ta = -1, tb = -1;
		long long lda = 0, ldb = 0;
		if (a_cs == 1 || K == 1)
			ta = 0, lda = a_rs;
		else if (a_rs == 1 || M == 1)
			ta = 1, lda = a_cs;
		if (b_cs == 1 || N == 1)
			tb = 0, ldb = b_rs;
		else if (b_rs == 1 || K == 1)
			tb = 1, ldb = b_cs;
		if (ta >= 0 && tb >= 0)
		{
			const int rc = gemm_any(s, kind, M, N, K, a, lda, ta, b, ldb, tb, c, c_rs, bias32, bias16, accumulate, scratch, algorithm == CCV_NNC_SM100_ALGO_3XTF32);
			if (rc <= 0)
				return rc;
		}
	}
	if (kind == 0)
		return gemm_ffma(s, M, N, K, (const float*)a, a_rs, a_cs, (const float*)b, b_rs, b_cs, (float*)c, c_rs, bias32, accumulate, scratch);
	// 16-bit shapes the tensor-core path cannot take (a leading dimension that is not a multiple of 16 bytes, e.g. a 10-class head):
	// widen the operands into the command's scratch, multiply in fp32 on the CUDA cores, narrow the result (one rounding).  Small
	// by construction: anything large has TMA-friendly strides.
	const size_t need = ((size_t)M * K + (size_t)K * N + (size_t)M * N + (size_t)N) * sizeof(float) + 1024;
	if (!scratch.ptr || scratch.bytes < need)
		return 1;
	float* const a32 = (float*)scratch.ptr;
	float* const b32 = a32 + (((size_t)M * K + 63) & ~(size_t)63);
	float* const c32 = b32 + (((size_t)K * N + 63) & ~(size_t)63);
	float* const bias_w = c32 + (((size_t)M * N + 63) & ~(size_t)63);
	if (widen_matrix(s, a, kind, a_rs, a_cs, a32, M, K) || widen_matrix(s, b, kind, b_rs, b_cs, b32, K, N))
		return -1;
	const float* bias_f = bias32;
	if (!bias_f && bias16)
	{
		if (widen_matrix(s, bias16, kind, 0, 1, bias_w, 1, N))
			return -1;
		bias_f = bias_w;
	}
	const int rc = gemm_ffma(s, M, N, K, a32, K, 1, b32, N, 1, c32, N, bias_f, 0);
	if (rc)
		return rc;
	return narrow_matrix(s, c32, c, kind, c_rs, c_cs, M, N, accumulate) ? -1 : 0;
}

// Workspace function of a command that a staging layer may wrap: the exact size of the one workspace request the command makes for
// these operands (0: none), or (size_t)-1 when it refuses them.  The command asks for that size before its first launch and hands
// slices of it to the helpers under it, which never ask themselves.
typedef size_t (*staged_inner_f)(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* in, int input_size, ccv_nnc_tensor_t* const* out, int output_size);
size_t no_workspace(const ccv_nnc_cmd_t&, const ccv_nnc_hint_t&, ccv_nnc_tensor_t* const*, int, ccv_nnc_tensor_t* const*, int) { return 0; }

// GEMM: the contraction scratch; the backward's column sum of the bias gradient shares it
size_t gemm_forw_workspace(const ccv_nnc_cmd_t&, const ccv_nnc_hint_t&, ccv_nnc_tensor_t* const*, int, ccv_nnc_tensor_t* const*, int) { return CONTRACT_SCRATCH_BYTES; }
size_t gemm_back_workspace(const ccv_nnc_cmd_t&, const ccv_nnc_hint_t&, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	size_t need = (output_size > 0 && out[0]) || (output_size > 1 && out[1]) ? CONTRACT_SCRATCH_BYTES : 0;
	if (output_size > 2 && out[2] && input_size > 0 && in[0])
	{
		const TV g = view_of(in[0]);
		need = std::max(need, colsum_workspace_bytes(g.nd > 0 ? g.dim[g.nd - 1] : 1));
	}
	return need;
}

// blas/ccv_nnc_gemm_cpu_ref.c:110-184
int exec_gemm_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 2 || output_size < 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const bias_t = input_size > 2 ? inputs[2] : 0;
	const int kind = kind_of(inputs[0]);
	if (kind < 0 || kind_of(inputs[1]) != kind || kind_of(outputs[0]) != kind || (bias_t && kind_of(bias_t) != kind && !is_f32(bias_t)))
		return CCV_NNC_EXEC_INVALID;
	const int no_transpose[2] = { 0, 0 };
	Mat a, w, b, bias;
	if (!mat_of(view_of(inputs[0]), cmd.info.blas.transpose_a, a) || !mat_of(view_of(inputs[1]), cmd.info.blas.transpose_b, w) || !mat_of(view_of(outputs[0]), no_transpose, b))
		return CCV_NNC_EXEC_INVALID;
	if (a.rows != b.rows || a.cols != w.rows || w.cols != b.cols)
		return CCV_NNC_EXEC_INVALID;
	if ((a.batch != b.batch && a.batch != 1) || (w.batch != b.batch && w.batch != 1))
		return CCV_NNC_EXEC_INVALID;
	if (a.batch == 1)
		a.batch_inc = 0;
	if (w.batch == 1)
		w.batch_inc = 0;
	bool matrix_bias = false;
	if (bias_t)
	{
		if (!mat_of(view_of(bias_t), no_transpose, bias) || bias.cols != b.cols || bias.cs != 1)
			return CCV_NNC_EXEC_INVALID;
		// the third operand is a row vector added to every row, or (blas/gpu/ccv_nnc_gemm_gpu_cublas.cu; test/int/nnc/cublas.tests.c:164-211)
		// a full [M, N] matrix: then c = a w + d, applied as a second pass
		matrix_bias = bias.rows == b.rows && bias.rows != 1;
		if ((bias.rows != 1 && !matrix_bias) || (matrix_bias && (kind != 0 || b.cs != 1)))
			return CCV_NNC_EXEC_INVALID;
		if (bias.batch == 1)
			bias.batch_inc = 0;
	}
	cudaStream_t s = stream_of(stream_context);
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, gemm_forw_workspace(cmd, hint, inputs, input_size, outputs, output_size), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	const Scratch scratch = scratch_at(ws, CONTRACT_SCRATCH_BYTES);
	const int algorithm = gemm_algorithm(cmd);
	if (matrix_bias)
	{
		for (int i = 0; i < b.batch; i++)
		{
			RC(gemm_dispatch(s, scratch, 0, algorithm, b.rows, b.cols, a.cols, at(a, i), a.rs, a.cs, at(w, i), w.rs, w.cs, at(b, i), b.rs, b.cs, 0, 0, 0));
			const int d4[4] = { 1, 1, b.rows, b.cols }, cs4[4] = { 0, 0, (int)b.rs, 1 }, ds4[4] = { 0, 0, (int)bias.rs, 1 };
			RC(ew_axpby_bcast_f32(s, 1.f, (const float*)at(b, i), cs4, 1.f, (const float*)at(bias, i), ds4, (float*)at(b, i), cs4, d4));
		}
		return CCV_NNC_EXEC_SUCCESS;
	}
	// the bias is fp32 or in the operands' type
	const bool bias32 = bias_t && is_f32(bias_t);
	for (int i = 0; i < b.batch; i++)
		RC(gemm_dispatch(s, scratch, kind, algorithm, b.rows, b.cols, a.cols, at(a, i), a.rs, a.cs, at(w, i), w.rs, w.cs, at(b, i), b.rs, b.cs, bias32 ? (const float*)at(bias, i) : 0, bias_t && !bias32 ? at(bias, i) : 0, 0));
	return CCV_NNC_EXEC_SUCCESS;
}

// blas/ccv_nnc_gemm_cpu_ref.c:318-448: inputs (g, a, w), outputs (h, dw, dbias), each optional
int exec_gemm_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 2 || output_size < 1 || !inputs[0])
		return CCV_NNC_EXEC_INVALID;
	const int no_transpose[2] = { 0, 0 };
	const int accumulate = (flags & CCV_NNC_ACCUMULATE_OUTPUT) ? 1 : 0;
	Mat g;
	const int kind = kind_of(inputs[0]);
	if (kind < 0 || !mat_of(view_of(inputs[0]), no_transpose, g))
		return CCV_NNC_EXEC_INVALID;
	const int algorithm = gemm_algorithm(cmd);
	cudaStream_t s = stream_of(stream_context);
	const size_t ws_bytes = gemm_back_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	void* const ws = ws_bytes ? ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !ws)
		return CCV_NNC_EXEC_OOM;
	const Scratch scratch = scratch_at(ws, CONTRACT_SCRATCH_BYTES);
	ccv_nnc_tensor_t* const dbias_t = output_size > 2 ? outputs[2] : 0;
	ccv_nnc_tensor_t* const dw_t = output_size > 1 ? outputs[1] : 0;
	ccv_nnc_tensor_t* const h_t = outputs[0];
	if (dbias_t)
	{
		Mat db;
		if (!mat_of(view_of(dbias_t), no_transpose, db) || db.cols != g.cols || db.cs != 1 || g.cs != 1 || db.rows != 1)
			return CCV_NNC_EXEC_INVALID;
		if (db.batch != 1 && db.batch != g.batch)
			return CCV_NNC_EXEC_INVALID;
		const int db_kind = kind_of(dbias_t);
		if (db_kind < 0)
			return CCV_NNC_EXEC_INVALID;
		if (db.batch == 1)
			db.batch_inc = 0;
		for (int i = 0; i < g.batch; i++)
			RC(colsum_any(s, kind, at(g, i), g.rows, g.cols, g.rs, at(db, i), db_kind, accumulate || (db.batch == 1 && i > 0), ws));
	}
	if (dw_t)
	{
		if (!inputs[1] || kind_of(inputs[1]) != kind || kind_of(dw_t) != kind)
			return CCV_NNC_EXEC_INVALID;
		Mat a, dw;
		if (!mat_of(view_of(inputs[1]), cmd.info.blas.transpose_a, a) || !mat_of(view_of(dw_t), cmd.info.blas.transpose_b, dw))
			return CCV_NNC_EXEC_INVALID;
		if (a.rows != g.rows || a.cols != dw.rows || dw.cols != g.cols)
			return CCV_NNC_EXEC_INVALID;
		if (a.batch == 1)
			a.batch_inc = 0;
		if (dw.batch == 1)
			dw.batch_inc = 0;
		// dw[K, N] = a^T[K, M] * g[M, N]; a shared dw sums over the batch
		for (int i = 0; i < g.batch; i++)
			RC(gemm_dispatch(s, scratch, kind, algorithm, dw.rows, dw.cols, g.rows, at(a, i), a.cs, a.rs, at(g, i), g.rs, g.cs, at(dw, i), dw.rs, dw.cs, 0, 0, accumulate || (dw.batch == 1 && i > 0)));
	}
	if (h_t)
	{
		if (input_size < 3 || !inputs[2] || kind_of(inputs[2]) != kind || kind_of(h_t) != kind)
			return CCV_NNC_EXEC_INVALID;
		Mat h, w;
		if (!mat_of(view_of(h_t), cmd.info.blas.transpose_a, h) || !mat_of(view_of(inputs[2]), cmd.info.blas.transpose_b, w))
			return CCV_NNC_EXEC_INVALID;
		if (h.cols != w.rows || w.cols != g.cols || h.rows != g.rows)
			return CCV_NNC_EXEC_INVALID;
		if (w.batch == 1)
			w.batch_inc = 0;
		if (h.batch == 1)
			h.batch_inc = 0;
		// h[M, K] = g[M, N] * w^T[N, K]
		for (int i = 0; i < g.batch; i++)
			RC(gemm_dispatch(s, scratch, kind, algorithm, h.rows, h.cols, g.cols, at(g, i), g.rs, g.cs, at(w, i), w.cs, w.rs, at(h, i), h.rs, h.cs, 0, 0, accumulate || (h.batch == 1 && i > 0)));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ GEMM with two batch axes
// ccv_nnc_tensor_get_matrix_params (lib/nnc/ccv_nnc_easy.h:421-444) and the reference GEMMs take up to 4-d operands
// [b0, b1, rows, cols] (attention-style "batch (2, 4)" products, test/int/nnc/cublas.tests.c:1801-2100), any of them possibly a
// view, an operand with fewer axes being shared by every outer batch.  The 3-d commands above are run once per outer index on
// sub-views; an output that is shared across the outer axis accumulates from the second index on (in a call of its own, so
// that per-index outputs are still overwritten).
struct Slice4 {
	ccv_nnc_tensor_view_t v;
	int is4;
};
inline void slice4_make(ccv_nnc_tensor_t* const t, Slice4& sl)
{
	sl.is4 = t && nd_of(t) == 4;
	if (!sl.is4)
		return;
	const TV tv = view_of(t);
	memset(&sl.v, 0, sizeof(sl.v));
	memcpy(&sl.v, t, sizeof(ccv_nnc_tensor_t));
	sl.v.type |= CCV_TENSOR_VIEW;
	memset(sl.v.info.dim, 0, sizeof(sl.v.info.dim));
	int packed = 1, contiguous = 1;
	for (int i = 2; i >= 0; i--)
	{
		sl.v.info.dim[i] = tv.dim[i + 1], sl.v.stride[i] = tv.stride[i + 1];
		if (tv.dim[i + 1] != 1 && tv.stride[i + 1] != packed)
			contiguous = 0;
		packed *= tv.dim[i + 1];
	}
	sl.v.contiguous = contiguous;
}
template <ccv_nnc_cmd_exec_f F>
int exec_gemm_nd4(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	enum { MAXT = 4 };
	int outer = 0;
	for (int i = 0; i < input_size; i++)
		if (inputs[i] && nd_of(inputs[i]) == 4)
			outer = std::max(outer, inputs[i]->info.dim[0]);
	for (int i = 0; i < output_size; i++)
		if (outputs[i] && nd_of(outputs[i]) == 4)
			outer = std::max(outer, outputs[i]->info.dim[0]);
	if (outer == 0)
		return F(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	if (input_size > MAXT || output_size > MAXT)
		return CCV_NNC_EXEC_INVALID;
	Slice4 si[MAXT], so[MAXT];
	ccv_nnc_tensor_t* in[MAXT];
	ccv_nnc_tensor_t* out[MAXT];
	ccv_nnc_tensor_t* out_shared[MAXT];
	int any_shared = 0, any_sliced = 0;
	for (int i = 0; i < input_size; i++)
	{
		slice4_make(inputs[i], si[i]);
		if (si[i].is4 && inputs[i]->info.dim[0] != outer && inputs[i]->info.dim[0] != 1)
			return CCV_NNC_EXEC_INVALID;
	}
	for (int i = 0; i < output_size; i++)
	{
		slice4_make(outputs[i], so[i]);
		if (so[i].is4 && outputs[i]->info.dim[0] != outer && outputs[i]->info.dim[0] != 1)
			return CCV_NNC_EXEC_INVALID;
		if (outputs[i])
		{
			const int shared = !so[i].is4 || outputs[i]->info.dim[0] == 1;
			any_shared |= shared, any_sliced |= !shared;
		}
	}
	for (int o = 0; o < outer; o++)
	{
		for (int i = 0; i < input_size; i++)
		{
			in[i] = inputs[i];
			if (si[i].is4)
			{
				const size_t step = inputs[i]->info.dim[0] == 1 ? 0 : (size_t)o * view_of(inputs[i]).stride[0];
				si[i].v.data.u8 = inputs[i]->data.u8 + step * dtype_size(inputs[i]->info.datatype);
				in[i] = (ccv_nnc_tensor_t*)&si[i].v;
			}
		}
		for (int i = 0; i < output_size; i++)
		{
			out[i] = outputs[i], out_shared[i] = 0;
			if (!outputs[i])
				continue;
			const int shared = !so[i].is4 || outputs[i]->info.dim[0] == 1;
			if (so[i].is4)
			{
				const size_t step = outputs[i]->info.dim[0] == 1 ? 0 : (size_t)o * view_of(outputs[i]).stride[0];
				so[i].v.data.u8 = outputs[i]->data.u8 + step * dtype_size(outputs[i]->info.datatype);
				out[i] = (ccv_nnc_tensor_t*)&so[i].v;
			}
			if (shared && o > 0 && any_sliced)
				out_shared[i] = out[i], out[i] = 0; // second call, accumulating
		}
		if (o == 0 || any_sliced)
		{
			const int rc = F(cmd, hint, (o > 0 && !any_sliced) ? (flags | CCV_NNC_ACCUMULATE_OUTPUT) : flags, in, input_size, out, output_size, stream_context);
			if (rc != CCV_NNC_EXEC_SUCCESS)
				return rc;
		}
		if (o > 0 && any_shared)
		{
			const int rc = F(cmd, hint, flags | CCV_NNC_ACCUMULATE_OUTPUT, in, input_size, any_sliced ? out_shared : out, output_size, stream_context);
			if (rc != CCV_NNC_EXEC_SUCCESS)
				return rc;
		}
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ CONVOLUTION
// NHWC activations ([N,] H, W, C), filters [K, R, S, C / groups] (convolution/ccv_nnc_conv_cpu_ref.c:47-65)
bool conv_geom(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, const TV& a, const TV& w, const TV& b, ConvGeom& g)
{
	if (a.format != CCV_TENSOR_FORMAT_NHWC || b.format != CCV_TENSOR_FORMAT_NHWC)
		return false;
	if ((a.nd != 3 && a.nd != 4) || (b.nd != 3 && b.nd != 4) || w.nd != 4 || !w.contiguous)
		return false;
	const int ao = a.nd - 3, bo = b.nd - 3;
	memset(&g, 0, sizeof(g));
	g.N = a.nd == 4 ? a.dim[0] : 1;
	if ((b.nd == 4 ? b.dim[0] : 1) != g.N)
		return false;
	g.H = a.dim[ao], g.W = a.dim[ao + 1], g.C = a.dim[ao + 2];
	g.P = b.dim[bo], g.Q = b.dim[bo + 1], g.K = b.dim[bo + 2];
	g.R = w.dim[1], g.S = w.dim[2];
	if (a.stride[ao + 2] != 1 || b.stride[bo + 2] != 1)
		return false;
	g.an = a.nd == 4 ? a.stride[0] : (long long)g.H * a.stride[ao];
	g.ah = a.stride[ao], g.aw = a.stride[ao + 1];
	g.bn = b.nd == 4 ? b.stride[0] : (long long)g.P * b.stride[bo];
	g.bh = b.stride[bo], g.bw = b.stride[bo + 1];
	g.stride_h = hint.stride.dim[0] > 0 ? hint.stride.dim[0] : 1;
	g.stride_w = hint.stride.dim[1] > 0 ? hint.stride.dim[1] : 1;
	g.dil_h = cmd.info.convolution.dilation[0] > 1 ? cmd.info.convolution.dilation[0] : 1;
	g.dil_w = cmd.info.convolution.dilation[1] > 1 ? cmd.info.convolution.dilation[1] : 1;
	g.pad_h0 = hint.border.begin[0], g.pad_w0 = hint.border.begin[1];
	// CPU_REF clips the window at the far edge (SET_BORDER_OFFSET_SIZE_FOR), i.e. the effective end padding is whatever
	// the output extent implies, not hint.border.end
	g.pad_h1 = (g.P - 1) * g.stride_h + (g.R - 1) * g.dil_h + 1 - g.H - g.pad_h0;
	g.pad_w1 = (g.Q - 1) * g.stride_w + (g.S - 1) * g.dil_w + 1 - g.W - g.pad_w0;
	const int groups = cmd.info.convolution.groups > 0 ? cmd.info.convolution.groups : 1;
	if (w.dim[0] != g.K || g.K != cmd.info.convolution.count || w.dim[3] * groups != g.C || g.K % groups != 0)
		return false;
	if (cmd.info.size.dim[0] != g.R || cmd.info.size.dim[1] != g.S)
		return false;
	return true;
}

// ------------------------------------------------------------------------------------------------ grouped convolution on tensor cores
// groups > 1 (convolution/ccv_nnc_conv_cpu_ref.c:47-65; the reference's GPU path hands groups to cuDNN,
// convolution/gpu/ccv_nnc_conv_gpu_cudnn.cu:204-357): group i contracts channels [i C/g, (i+1) C/g) against filters
// [i K/g, (i+1) K/g) -- `groups` independent dense convolutions whose operands are channel SLICES of the NHWC tensors (pixel stride
// C, not C/g) except for the filters, whose rows are contiguous per group.  When a group is wide enough to fill tensor-core tiles
// (C/g and K/g multiples of the 16-byte vector and >= 16) each group's slices are made dense in the stream workspace (one strided
// copy in, one out), and the dense wgmma kernels above do the arithmetic; narrower groups (depthwise and the like) stay on the
// FFMA kernels, where the contraction is too short for a 64-deep MMA anyway.  PASS 0 = fprop, 1 = wgrad, 2 = dgrad.
// The workspace of one pass is [contraction workspace | one group's dense activations | its results]; false when the groups are too
// narrow or unaligned for it (the caller falls back).
struct GroupPlan {
	ConvGeom gg; // one group as a dense convolution
	size_t inner, xb, yb;
};
bool group_plan(const ConvGeom& g, const int kind, const int groups, const int pass, GroupPlan& p)
{
	const int align = kind == 0 ? 4 : 8;
	const size_t es = elem_size(kind);
	if (groups <= 1 || g.C % groups || g.K % groups)
		return false;
	const int Cg = g.C / groups, Kg = g.K / groups;
	if (Cg % align || Kg % align || Cg < 16 || Kg < 16)
		return false;
	const long long lim = 0x7fffffffll;
	if ((long long)g.N * g.an > lim || (long long)g.N * g.bn > lim)
		return false; // copy_strided walks int strides
	ConvGeom& gg = p.gg;
	gg = g;
	gg.C = Cg, gg.K = Kg;
	gg.aw = Cg, gg.ah = (long long)g.W * Cg, gg.an = (long long)g.H * g.W * Cg;
	gg.bw = Kg, gg.bh = (long long)g.Q * Kg, gg.bn = (long long)g.P * g.Q * Kg;
	const size_t nx = (size_t)g.N * g.H * g.W * Cg, ny = (size_t)g.N * g.P * g.Q * Kg;
	p.xb = (nx * es + 255) & ~(size_t)255, p.yb = (ny * es + 255) & ~(size_t)255;
	// the fp32 data gradient's workspace, else the split-K scratch
	p.inner = pass == 2 ? conv_dgrad_workspace_bytes(gg, kind) : CONTRACT_SCRATCH_BYTES;
	return true;
}
// returns 0 done, 1 not applicable (caller falls back), < 0 error; ws holds the group plan's bytes
template <int PASS>
int conv_grouped_tc(cudaStream_t s, unsigned char* const ws, const int kind, const ConvGeom& g, const int groups, const int x3, const int accumulate,
	const void* const act, const void* const filt, const float* const bias32, const void* const bias16, const void* const res, void* const out)
{
	GroupPlan p;
	if (!group_plan(g, kind, groups, PASS, p))
		return 1;
	const ConvGeom& gg = p.gg;
	const int Cg = gg.C, Kg = gg.K;
	const size_t es = elem_size(kind);
	const Scratch scratch = scratch_at(ws, CONTRACT_SCRATCH_BYTES);
	unsigned char* const xg = ws + p.inner;
	unsigned char* const yg = xg + p.xb;
	const int xd[4] = { g.N, g.H, g.W, Cg }, xs_t[4] = { (int)g.an, (int)g.ah, (int)g.aw, 1 }, xs_d[4] = { g.H * g.W * Cg, g.W * Cg, Cg, 1 };
	const int yd[4] = { g.N, g.P, g.Q, Kg }, ys_t[4] = { (int)g.bn, (int)g.bh, (int)g.bw, 1 }, ys_d[4] = { g.P * g.Q * Kg, g.Q * Kg, Kg, 1 };
	const size_t wstep = (size_t)Kg * g.R * g.S * Cg * es;
	for (int i = 0; i < groups; i++)
	{
		// (an operand a pass does not use is NULL: no arithmetic on it)
		const unsigned char* const act_i = act ? (const unsigned char*)act + (size_t)i * Cg * es : 0;
		const unsigned char* const res_i = res ? (const unsigned char*)res + (size_t)i * Kg * es : 0;
		const unsigned char* const w_i = filt ? (const unsigned char*)filt + (size_t)i * wstep : 0;
		int rc;
		if (PASS == 0)
		{
			// y_i = conv(x_i, w_i) + bias_i
			if (copy_strided(s, act_i, xs_t, xg, xs_d, xd, (int)es))
				return -1;
			rc = conv_fprop_any(s, kind, gg, xg, w_i, bias32 ? bias32 + (size_t)i * Kg : 0, bias16 ? (const unsigned char*)bias16 + (size_t)i * Kg * 2 : 0, yg, scratch, x3);
			if (rc)
				return i == 0 ? rc : -1;
			if (copy_strided(s, yg, ys_d, (unsigned char*)out + (size_t)i * Kg * es, ys_t, yd, (int)es))
				return -1;
		} else if (PASS == 1) {
			// dw_i (+)= wgrad(g_i, x_i): the filter gradient's rows of a group are contiguous
			if (copy_strided(s, act_i, xs_t, xg, xs_d, xd, (int)es) || copy_strided(s, res_i, ys_t, yg, ys_d, yd, (int)es))
				return -1;
			rc = conv_wgrad_any(s, kind, gg, yg, xg, (unsigned char*)out + (size_t)i * wstep, accumulate, scratch, x3);
			if (rc)
				return i == 0 ? rc : -1;
		} else {
			// h_i = dgrad(g_i, w_i) (+ bias_i: the forward of a transposed convolution, whose outputs are the C side)
			if (copy_strided(s, res_i, ys_t, yg, ys_d, yd, (int)es))
				return -1;
			rc = conv_dgrad_any(s, kind, gg, yg, w_i, bias32 ? bias32 + (size_t)i * Cg : 0, bias16 ? (const unsigned char*)bias16 + (size_t)i * Cg * 2 : 0, xg, ws, x3);
			if (rc)
				return i == 0 ? rc : -1;
			if (copy_strided(s, xg, xs_d, (unsigned char*)out + (size_t)i * Cg * es, xs_t, xd, (int)es))
				return -1;
		}
	}
	return 0;
}

// h = dgrad(gb, w) (+ bias[C]) on the geometry gh, returns a CCV_NNC_EXEC_* status: the data gradient of CONVOLUTION_BACKWARD (no
// bias) and the forward of CONVOLUTION_TRANSPOSE (bias32 fp32, or bias16 of the tensors' 16-bit type).  Tensor cores for one group,
// per-group dense launches for wide groups (fp32 unless ALGO_FFMA; 16-bit always).  Where they decline, fp32 runs on FFMA (also
// narrow groups and unaligned channels); 16-bit groups they cannot take run on the direct grouped kernels (sm100_conv_grouped.cu),
// 16-bit single-group shapes they cannot take (3-channel pixels) in the functional form -- widen g, w and the bias, fp32 FFMA data
// gradient + bias, one rounding on the way back.
// workspace of the 16-bit functional form below: fp32 copies of g, w, h and the bias, 256-byte aligned
size_t dgrad16_fallback_bytes(const ConvGeom& gh)
{
	return ((size_t)gh.N * gh.P * gh.Q * gh.K + (size_t)gh.K * gh.R * gh.S * gh.C + (size_t)gh.N * gh.H * gh.W * gh.C + gh.C) * sizeof(float) + 1280;
}
// ws holds conv_workspace(gh, kind, groups, algo, CONV_DGRAD)
int dgrad_nhwc(cudaStream_t s, unsigned char* const ws, const int kind, const int algo, const int groups, const ConvGeom& gh, const void* const gb, const void* const w, const float* const bias32, const void* const bias16, void* const h)
{
	const int x3 = algo == CCV_NNC_SM100_ALGO_3XTF32;
	int rc = 1;
	if (kind > 0 || algo != CCV_NNC_SM100_ALGO_FFMA)
		rc = groups > 1 ? conv_grouped_tc<2>(s, ws, kind, gh, groups, x3, 0, 0, w, bias32, bias16, gb, h) : conv_dgrad_any(s, kind, gh, gb, w, bias32, bias16, h, ws, x3);
	if (rc < 0)
		return CCV_NNC_EXEC_INVALID;
	if (rc == 0)
		return CCV_NNC_EXEC_SUCCESS;
	if (kind == 0)
	{
		RC(conv_dgrad_ffma(s, gh, groups, (const float*)gb, (const float*)w, bias32, (float*)h));
		return CCV_NNC_EXEC_SUCCESS;
	}
	if (groups > 1) // groups the tensor cores do not take: the direct CUDA-core kernels
	{
		RC(conv_dgrad_grouped16(s, kind, gh, groups, gb, w, bias32, bias16, h));
		return CCV_NNC_EXEC_SUCCESS;
	}
	// (the image gradient of a stem, test/int/nnc/cudnn.tests.c:499-577; the RGB head of a transposed convolution)  Dense tensors.
	const size_t ng = (size_t)gh.N * gh.P * gh.Q * gh.K, nw = (size_t)gh.K * gh.R * gh.S * gh.C, nh = (size_t)gh.N * gh.H * gh.W * gh.C, nb = bias16 ? gh.C : 0;
	if (gh.bw != gh.K || gh.bh != (long long)gh.Q * gh.K || gh.bn != (long long)gh.P * gh.Q * gh.K || gh.aw != gh.C || gh.ah != (long long)gh.W * gh.C || gh.an != (long long)gh.H * gh.W * gh.C || ng > 0x7fffffffull || nh > 0x7fffffffull)
		return CCV_NNC_EXEC_INVALID;
	float* const g32 = (float*)ws;
	float* const w32 = (float*)(((uintptr_t)(g32 + ng) + 255) & ~(uintptr_t)255);
	float* const h32 = (float*)(((uintptr_t)(w32 + nw) + 255) & ~(uintptr_t)255);
	float* const b32 = (float*)(((uintptr_t)(h32 + nh) + 255) & ~(uintptr_t)255);
	RC(widen_matrix(s, gb, kind, (long long)ng, 1, g32, 1, (int)ng));
	RC(widen_matrix(s, w, kind, (long long)nw, 1, w32, 1, (int)nw));
	if (nb)
		RC(widen_matrix(s, bias16, kind, (long long)nb, 1, b32, 1, (int)nb));
	RC(conv_dgrad_ffma(s, gh, 1, g32, w32, nb ? b32 : bias32, h32));
	RC(narrow_matrix(s, h32, h, kind, (long long)nh, 1, 1, (int)nh, 0));
	return CCV_NNC_EXEC_SUCCESS;
}

// The workspace of the products `which` of a convolution on g: the most any path the shapes permit uses -- the split-K scratch or
// the fp32 data gradient's workspace, the grouped [contraction | group activations | group results], im2col for unaligned channels,
// the 16-bit functional data gradient where the tensor cores may decline.  The FFMA kernels use none, except the weight gradient's
// split-K scratch; the direct 16-bit grouped kernels likewise (their weight gradient's pixel-chunk slices).
enum { CONV_FPROP = 1, CONV_WGRAD = 2, CONV_DGRAD = 4 };
size_t conv_workspace(const ConvGeom& g, const int kind, const int groups, const int algo, const unsigned which)
{
	size_t need = 0;
	GroupPlan gp;
	for (int pass = 0; pass < 3; pass++)
	{
		if (!(which & (1u << pass)))
			continue;
		if (kind == 0 && algo == CCV_NNC_SM100_ALGO_FFMA)
			need = std::max(need, pass == 1 ? CONTRACT_SCRATCH_BYTES : 0);
		else if (groups > 1)
		{
			need = std::max(need, group_plan(g, kind, groups, pass, gp) ? gp.inner + gp.xb + gp.yb : kind == 0 && pass == 1 ? CONTRACT_SCRATCH_BYTES : 0);
			if (kind > 0 && pass == 1) // where the tensor cores decline, the direct kernels' weight gradient
				need = std::max(need, conv_grouped16_wgrad_bytes(g, groups));
		}
		else {
			need = std::max(need, pass == 2 ? conv_dgrad_workspace_bytes(g, kind) : CONTRACT_SCRATCH_BYTES);
			if (pass < 2 && g.C % (kind == 0 ? 4 : 8) != 0)
				need = std::max(need, conv_im2col_workspace_bytes(g, kind));
			if (pass == 2 && kind > 0 && conv_dgrad_may_decline(g, kind))
				need = std::max(need, dgrad16_fallback_bytes(g));
		}
	}
	return need;
}
inline int conv_groups(const ccv_nnc_cmd_t& cmd) { return cmd.info.convolution.groups > 0 ? cmd.info.convolution.groups : 1; }

size_t conv_forw_workspace(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	ConvGeom g;
	if (input_size < 2 || output_size < 1 || !in[0] || !in[1] || !out[0] || kind_of(in[0]) < 0 || !conv_geom(cmd, hint, view_of(in[0]), view_of(in[1]), view_of(out[0]), g))
		return (size_t)-1;
	return conv_workspace(g, kind_of(in[0]), conv_groups(cmd), conv_algorithm(cmd), CONV_FPROP);
}

// inputs (g, a, w), outputs (h, dw, dbias): the weight gradient and the column sum on the geometry of a, the data gradient on h's
size_t conv_back_workspace(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	if (input_size < 2 || output_size < 1 || !in[0] || !in[1])
		return (size_t)-1;
	ccv_nnc_tensor_t* const h_t = out[0];
	ccv_nnc_tensor_t* const dw_t = output_size > 1 ? out[1] : 0;
	ccv_nnc_tensor_t* const w_t = input_size > 2 ? in[2] : 0;
	ccv_nnc_tensor_t* const filt = dw_t ? dw_t : w_t;
	const int kind = kind_of(in[0]), groups = conv_groups(cmd), algo = conv_algorithm(cmd);
	ConvGeom g, gh;
	if (!filt || kind < 0 || !conv_geom(cmd, hint, view_of(in[1]), view_of(filt), view_of(in[0]), g))
		return (size_t)-1;
	size_t need = conv_workspace(g, kind, groups, algo, dw_t ? CONV_WGRAD : 0);
	if (output_size > 2 && out[2])
		need = std::max(need, colsum_workspace_bytes(g.K));
	if (h_t && w_t && conv_geom(cmd, hint, view_of(h_t), view_of(w_t), view_of(in[0]), gh))
		need = std::max(need, conv_workspace(gh, kind, groups, algo, CONV_DGRAD));
	return need;
}

int conv_forw_nhwc(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const size_t ws_bytes = conv_forw_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	if (ws_bytes == (size_t)-1)
		return CCV_NNC_EXEC_INVALID;
	unsigned char* const ws = ws_bytes ? (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !ws)
		return CCV_NNC_EXEC_OOM;
	// every tensor of one kind; the bias fp32 or of that kind
	const ccv_nnc_tensor_t* const bias_t = input_size > 2 ? inputs[2] : 0;
	const int kind = kind_of(inputs[0]);
	if (kind_of(inputs[1]) != kind || kind_of(outputs[0]) != kind || (bias_t && ((kind_of(bias_t) != kind && !is_f32(bias_t)) || CCV_IS_TENSOR_VIEW(bias_t))))
		return CCV_NNC_EXEC_INVALID;
	ConvGeom g;
	if (!conv_geom(cmd, hint, view_of(inputs[0]), view_of(inputs[1]), view_of(outputs[0]), g) || (bias_t && bias_t->info.dim[0] != g.K))
		return CCV_NNC_EXEC_INVALID;
	const int groups = conv_groups(cmd), algo = conv_algorithm(cmd), x3 = algo == CCV_NNC_SM100_ALGO_3XTF32;
	cudaStream_t s = stream_of(stream_context);
	const void* const a = inputs[0]->data.u8;
	const void* const w = inputs[1]->data.u8;
	const float* const bias32 = bias_t && is_f32(bias_t) ? bias_t->data.f32 : 0;
	const void* const bias16 = bias_t && !is_f32(bias_t) ? (const void*)bias_t->data.u8 : 0;
	void* const b = outputs[0]->data.u8;
	int rc = 1;
	if (kind > 0 || algo != CCV_NNC_SM100_ALGO_FFMA)
	{
		if (groups > 1)
			rc = conv_grouped_tc<0>(s, ws, kind, g, groups, x3, 0, a, w, bias32, bias16, 0, b);
		else {
			rc = conv_fprop_any(s, kind, g, a, w, bias32, bias16, b, scratch_at(ws, CONTRACT_SCRATCH_BYTES), x3);
			if (rc > 0 && g.C % (16 / elem_size(kind)) != 0) // TMA cannot address pixels of other sizes (the 3-channel stem): explicit im2col + tensor-core GEMM
				rc = conv_fprop_im2col_any(s, kind, g, a, w, bias32, bias16, b, ws, x3);
		}
	}
	if (rc < 0)
		return CCV_NNC_EXEC_INVALID;
	if (rc > 0)
	{
		if (kind > 0 && groups > 1) // groups the tensor cores do not take: the direct CUDA-core kernels
			RC(conv_fprop_grouped16(s, kind, g, groups, a, w, bias32, bias16, b));
		else if (kind > 0) // there is no 16-bit FFMA kernel to fall back to
			return CCV_NNC_EXEC_INVALID;
		else
			RC(conv_fprop_ffma(s, g, groups, (const float*)a, (const float*)w, bias32, (float*)b));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// convolution/ccv_nnc_conv_cpu_ref.c:174-345: inputs (g, a, w), outputs (h, dw, dbias); dw / dbias honour
// CCV_NNC_ACCUMULATE_OUTPUT, h is always overwritten (:286)
int conv_back_nhwc(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const size_t ws_bytes = conv_back_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	if (ws_bytes == (size_t)-1)
		return CCV_NNC_EXEC_INVALID;
	unsigned char* const ws = ws_bytes ? (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !ws)
		return CCV_NNC_EXEC_OOM;
	ccv_nnc_tensor_t* const h_t = outputs[0];
	ccv_nnc_tensor_t* const dw_t = output_size > 1 ? outputs[1] : 0;
	ccv_nnc_tensor_t* const dbias_t = output_size > 2 ? outputs[2] : 0;
	const ccv_nnc_tensor_t* const w_t = input_size > 2 ? inputs[2] : 0;
	const ccv_nnc_tensor_t* const filt = dw_t ? dw_t : w_t;
	// every operand is checked before the first launch: a refused call leaves the outputs as they were
	const int kind = kind_of(inputs[0]);
	if (!filt || kind_of(inputs[1]) != kind || kind_of(filt) != kind || (h_t && kind_of(h_t) != kind) || (w_t && kind_of(w_t) != kind))
		return CCV_NNC_EXEC_INVALID;
	ConvGeom g, gh;
	if (!conv_geom(cmd, hint, view_of(inputs[1]), view_of(filt), view_of(inputs[0]), g))
		return CCV_NNC_EXEC_INVALID;
	if (h_t && (!w_t || !conv_geom(cmd, hint, view_of(h_t), view_of(w_t), view_of(inputs[0]), gh)))
		return CCV_NNC_EXEC_INVALID;
	// dbias in fp32, or for 16-bit gradients also in their type
	const int db_kind = dbias_t ? kind_of(dbias_t) : 0;
	if (dbias_t && (db_kind < 0 || (kind == 0 && db_kind != 0) || dbias_t->info.dim[0] != g.K || g.bh != (long long)g.Q * g.bw || g.bn != (long long)g.P * g.bh))
		return CCV_NNC_EXEC_INVALID;
	const int groups = conv_groups(cmd);
	const int accumulate = (flags & CCV_NNC_ACCUMULATE_OUTPUT) ? 1 : 0;
	const int algo = conv_algorithm(cmd), x3 = algo == CCV_NNC_SM100_ALGO_3XTF32;
	cudaStream_t s = stream_of(stream_context);
	const void* const gb = inputs[0]->data.u8;
	const void* const a = inputs[1]->data.u8;
	if (dbias_t)
		RC(colsum_any(s, kind, gb, (size_t)g.N * g.P * g.Q, g.K, g.bw, dbias_t->data.u8, db_kind, accumulate, ws));
	if (dw_t)
	{
		int rc = 1;
		if (kind > 0 || algo != CCV_NNC_SM100_ALGO_FFMA)
		{
			if (groups > 1)
				rc = conv_grouped_tc<1>(s, ws, kind, g, groups, x3, accumulate, a, 0, 0, 0, gb, dw_t->data.u8);
			else {
				rc = conv_wgrad_any(s, kind, g, gb, a, dw_t->data.u8, accumulate, scratch_at(ws, CONTRACT_SCRATCH_BYTES), x3);
				if (rc > 0 && g.C % (16 / elem_size(kind)) != 0)
					rc = conv_wgrad_im2col_any(s, kind, g, gb, a, dw_t->data.u8, accumulate, ws, x3);
			}
		}
		if (rc > 0 && kind > 0 && groups > 1) // groups the tensor cores do not take: the direct CUDA-core kernels
			rc = conv_wgrad_grouped16(s, kind, g, groups, gb, a, dw_t->data.u8, accumulate, scratch_at(ws, ws_bytes));
		if (rc < 0 || (rc > 0 && kind > 0))
			return CCV_NNC_EXEC_INVALID;
		if (rc > 0)
			RC(conv_wgrad_ffma(s, g, groups, (const float*)gb, (const float*)a, dw_t->data.f32, accumulate, scratch_at(ws, CONTRACT_SCRATCH_BYTES)));
	}
	if (h_t)
		return dgrad_nhwc(s, ws, kind, algo, groups, gh, gb, w_t->data.u8, 0, 0, h_t->data.u8);
	return CCV_NNC_EXEC_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ staged operands
// Some operands reach a command in a form its kernels do not take.  The command then runs in its dense form on shadow copies in
// the stream workspace, and results are copied back:
//   - STAGE_NCHW: the convolution, transposed convolution and pooling kernels are NHWC.  The reference's GPU convolution takes any
//     mix of formats -- its tests run NHWC activations against NCHW filters and all-NCHW forward and backward
//     (convolution/gpu/ccv_nnc_conv_gpu_cudnn.cu:204-357; test/int/nnc/cudnn.tests.c:24-85, 87-140, 417-497), and so do its pools
//     (pool/gpu/ccv_nnc_max_pool_gpu_cudnn.cu; test/int/nnc/cudnn.tests.c:2772-2870) -- so every NCHW operand is re-laid out (one
//     strided copy each way).  Outputs that accumulate are staged in as well.
//   - STAGE_F32: the commands with fp32 kernels only take bf16 / fp16 tensors in their functional form (widen every 16-bit tensor,
//     round every 16-bit result once, to nearest even).  Aliased 16-bit tensors share one shadow.
//   - STAGE_QX: a palettized weight (CCV_QX) is decoded, so the result is the dense command's, bit for bit.
// The workspace is one grow-only buffer per stream, and growing it frees the old one.  So the layer makes one request,
// [inner | staging], `inner` being the wrapped command's workspace function on the shadows: the command's own request is then
// the same size or smaller and returns the same base.  Layers compose (a palettized filter of an NCHW convolution): a layer's own
// workspace function is inner(shadows) + staging.
enum { STAGE_NCHW, STAGE_F32, STAGE_QX };

inline bool is_nchw(const ccv_nnc_tensor_t* const t) { return t && t->info.format == CCV_TENSOR_FORMAT_NCHW && nd_of(t) >= 3; }
inline bool is_qx(const ccv_nnc_tensor_t* const t) { return t && CCV_GET_DATA_TYPE(t->info.datatype) == CCV_QX; }
inline int qx_palette(const ccv_nnc_tensor_t* const t) { return (t->info.datatype & 0xff) << 12; }
inline int qx_bits(const ccv_nnc_tensor_t* const t) { return (t->info.datatype >> 8) & 0xf; }
// a palettized operand the decoder takes, with a palette of the command's dense type: not a view, qbits 4..8, whole index bytes per
// block, fp16 / fp32 palettes
bool qx_ok(const ccv_nnc_tensor_t* const t, const int dense)
{
	const int pal = qx_palette(t);
	return !CCV_IS_TENSOR_VIEW(t) && palettize_params_ok(qx_bits(t), t->info.reserved) && (pal == CCV_16F || pal == CCV_32F) && pal == dense;
}
inline int qx_decode(cudaStream_t s, const ccv_nnc_tensor_t* const t, void* const out)
{
	return depalettize(s, t->data.u8, qx_palette(t), qx_bits(t), t->info.reserved, out, view_of(t).count);
}

struct Shadow {
	ccv_nnc_tensor_t t; // what the wrapped command sees
	ccv_nnc_tensor_t* orig;
	size_t bytes;
	int in, out; // filled before the command runs / copied back after it
	int d[4], src[4], dst[4], elem; // STAGE_NCHW: index space N, H, W, C with the NCHW and the NHWC strides
};
struct StagePlan {
	enum { MAXT = 16 };
	Shadow sh[2 * MAXT];
	int n;
	size_t staging;
	ccv_nnc_tensor_t* in[MAXT];
	ccv_nnc_tensor_t* out[MAXT];
};

inline bool is_staged(const int transform, const ccv_nnc_tensor_t* const t)
{
	return t && (transform == STAGE_NCHW ? is_nchw(t) : transform == STAGE_F32 ? kind_of(t) > 0 : is_qx(t));
}

// the shadow of one operand, t itself when the transform leaves it alone, NULL when the call is refused
ccv_nnc_tensor_t* stage_operand(StagePlan& p, const int transform, ccv_nnc_tensor_t* const t, const int is_out, const int stage_in, const int dense)
{
	if (!is_staged(transform, t))
		return t;
	if (transform == STAGE_F32)
		for (int j = 0; j < p.n; j++)
			if (p.sh[j].orig == t || p.sh[j].orig->data.u8 == t->data.u8)
			{
				p.sh[j].out |= is_out;
				return &p.sh[j].t;
			}
	const TV v = view_of(t);
	Shadow& x = p.sh[p.n];
	memcpy(&x.t, t, sizeof(ccv_nnc_tensor_t));
	x.t.type &= ~CCV_TENSOR_VIEW;
	x.orig = t, x.in = stage_in, x.out = is_out;
	size_t elem;
	if (transform == STAGE_NCHW)
	{
		elem = dtype_size(t->info.datatype);
		if (!v.contiguous || (v.nd != 3 && v.nd != 4) || elem == 0)
			return 0;
		const int N = v.nd == 4 ? v.dim[0] : 1, C = v.dim[v.nd - 3], H = v.dim[v.nd - 2], W = v.dim[v.nd - 1];
		const int d[4] = { N, H, W, C }, src[4] = { C * H * W, W, 1, H * W }, dst[4] = { H * W * C, W * C, C, 1 };
		memcpy(x.d, d, sizeof(d)), memcpy(x.src, src, sizeof(src)), memcpy(x.dst, dst, sizeof(dst));
		x.elem = (int)elem;
		x.t.info.format = CCV_TENSOR_FORMAT_NHWC;
		memset(x.t.info.dim, 0, sizeof(x.t.info.dim));
		if (v.nd == 4)
			x.t.info.dim[0] = N, x.t.info.dim[1] = H, x.t.info.dim[2] = W, x.t.info.dim[3] = C;
		else
			x.t.info.dim[0] = H, x.t.info.dim[1] = W, x.t.info.dim[2] = C;
	} else if (transform == STAGE_F32) {
		if (!v.contiguous || v.count > 0x7fffffffull)
			return 0;
		elem = sizeof(float);
		x.t.info.datatype = CCV_32F;
		x.in = 1; // an output may be read by the command too (in-place forms)
	} else {
		if (is_out || !qx_ok(t, dense))
			return 0;
		const int pal = qx_palette(t);
		elem = dtype_size(pal);
		x.t.info.datatype = pal;
		x.t.info.reserved = 0;
		x.t.type = (x.t.type & ~0xFF000) | pal;
		x.t.data_size = 0;
	}
	x.bytes = (v.count * elem + 255) & ~(size_t)255;
	p.staging += x.bytes;
	p.n++;
	return &x.t;
}

// `select`: STAGE_NCHW, non-zero when outputs[1..] accumulate under CCV_NNC_ACCUMULATE_OUTPUT; STAGE_QX, bit i set when inputs[i]
// may be palettized.  false: the call is refused (outputs untouched).  p.n == 0: nothing to stage, the command runs on the
// caller's operands, whatever their number.
bool stage_plan(const int transform, const unsigned select, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, StagePlan& p)
{
	p.n = 0, p.staging = 0;
	bool any = false;
	for (int i = 0; i < input_size; i++)
		any = any || is_staged(transform, inputs[i]);
	for (int i = 0; i < output_size; i++)
		any = any || is_staged(transform, outputs[i]);
	if (!any)
		return true;
	if (input_size > StagePlan::MAXT || output_size > StagePlan::MAXT || (transform == STAGE_NCHW && (input_size > 3 || output_size > 3)))
		return false;
	int dense = 0; // the type of the command's other tensors, which a palette must have
	for (int i = 0; i < output_size && !dense; i++)
		if (outputs[i])
			dense = CCV_GET_DATA_TYPE(outputs[i]->info.datatype);
	for (int i = 0; i < input_size && !dense; i++)
		if (inputs[i] && !is_qx(inputs[i]))
			dense = CCV_GET_DATA_TYPE(inputs[i]->info.datatype);
	for (int i = 0; i < input_size; i++)
		if ((transform == STAGE_QX && is_qx(inputs[i]) && !(select & (1u << i))) || (!(p.in[i] = stage_operand(p, transform, inputs[i], 0, 1, dense)) && inputs[i]))
			return false;
	const int accumulating = transform == STAGE_NCHW && select && (flags & CCV_NNC_ACCUMULATE_OUTPUT);
	for (int i = 0; i < output_size; i++)
		if (!(p.out[i] = stage_operand(p, transform, outputs[i], 1, accumulating && i > 0, dense)) && outputs[i])
			return false;
	return true;
}

// one operand into its shadow, or (!in) the shadow's result back
int stage(cudaStream_t s, const int transform, const Shadow& x, const int in)
{
	const ccv_nnc_tensor_t* const t = x.orig;
	const size_t n = view_of(t).count;
	if (transform == STAGE_NCHW)
		return in ? copy_strided(s, t->data.u8, x.src, x.t.data.u8, x.dst, x.d, x.elem) : copy_strided(s, x.t.data.u8, x.dst, t->data.u8, x.src, x.d, x.elem);
	if (transform == STAGE_F32)
		return in ? widen_matrix(s, t->data.u8, kind_of(t), (long long)n, 1, x.t.data.f32, 1, (int)n) : narrow_matrix(s, x.t.data.f32, t->data.u8, kind_of(t), (long long)n, 1, 1, (int)n, 0);
	return qx_decode(s, t, x.t.data.u8);
}

// `exec` runs on the shadows, `inner_of` is its workspace function
int staged(const int transform, const unsigned select, const ccv_nnc_cmd_exec_f exec, const staged_inner_f inner_of, const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	StagePlan p;
	if (!stage_plan(transform, select, flags, inputs, input_size, outputs, output_size, p))
		return CCV_NNC_EXEC_INVALID;
	if (!p.n)
		return exec(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	const size_t inner = inner_of(cmd, hint, p.in, input_size, p.out, output_size);
	if (inner == (size_t)-1)
		return CCV_NNC_EXEC_INVALID;
	const size_t at = (inner + 255) & ~(size_t)255;
	unsigned char* const ws = (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, at + p.staging, CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	cudaStream_t s = stream_of(stream_context);
	unsigned char* q = ws + at;
	for (int j = 0; j < p.n; j++)
		p.sh[j].t.data.u8 = q, q += p.sh[j].bytes;
	for (int j = 0; j < p.n; j++)
		if (p.sh[j].in)
			RC(stage(s, transform, p.sh[j], 1));
	const int rc = exec(cmd, hint, flags, p.in, input_size, p.out, output_size, stream_context);
	if (rc != CCV_NNC_EXEC_SUCCESS)
		return rc;
	if (ccv_nnc_stream_context_get_workspace(stream_context, 1, CCV_TENSOR_GPU_MEMORY) != (void*)ws)
	{
		// the wrapped command asked for more than its workspace function said: the staged tensors moved with the workspace
		set_last_error("staged operands: the workspace moved under them", cudaErrorInvalidValue);
		return CCV_NNC_EXEC_INVALID;
	}
	for (int j = 0; j < p.n; j++)
		if (p.sh[j].out)
			RC(stage(s, transform, p.sh[j], 0));
	return CCV_NNC_EXEC_SUCCESS;
}

size_t staged_workspace(const int transform, const unsigned select, const staged_inner_f inner_of, const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size)
{
	StagePlan p;
	if (!stage_plan(transform, select, 0, inputs, input_size, outputs, output_size, p))
		return (size_t)-1;
	if (!p.n)
		return inner_of(cmd, hint, inputs, input_size, outputs, output_size);
	const size_t inner = inner_of(cmd, hint, p.in, input_size, p.out, output_size);
	return inner == (size_t)-1 ? inner : ((inner + 255) & ~(size_t)255) + p.staging;
}

// the NHWC command EXEC (workspace function WS) on any mix of formats; ACCUMULATING: outputs[1..] may be read before written
template <ccv_nnc_cmd_exec_f EXEC, staged_inner_f WS, int ACCUMULATING>
int exec_nchw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return staged(STAGE_NCHW, ACCUMULATING, EXEC, WS, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}
template <staged_inner_f WS>
size_t nchw_workspace(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	return staged_workspace(STAGE_NCHW, 0, WS, cmd, hint, in, input_size, out, output_size);
}

// ================================================================================================ CONVOLUTION_TRANSPOSE
// convolution/ccv_nnc_conv_transpose_cpu_ref.c:13-197.  y = T(a) is the data gradient of the "mirrored" convolution, the one that
// maps y's extent onto a's: y plays its input (C = Cout = count), a its output (K = Cin), and w[Cin, R, S, Cout / groups] has its
// filter layout [K, R, S, C / groups]; the hint means what it means for that convolution (CPU_REF walks the same clipped windows).
// Pixels of y that no tap reaches hold the bias.  The backward (which the reference leaves undefined) is the mirrored convolution's
// forward for da = conv(g, w), its weight gradient with the activations swapped for dw = wgrad(grad = a, x = g), and the column sum
// of g for dbias: the same launches as CONVOLUTION_FORWARD / _BACKWARD, bit for bit.
// The mirrored CONVOLUTION command: count = Cin (convolution_transpose.count is Cout; groups and dilation sit at the same offsets)
bool conv_mirror(const ccv_nnc_cmd_t& cmd, const TV& w, const uint32_t mirror_id, ccv_nnc_cmd_t& mirror)
{
	const int groups = cmd.info.convolution_transpose.groups > 0 ? cmd.info.convolution_transpose.groups : 1;
	if (w.nd != 4 || w.dim[3] * groups != cmd.info.convolution_transpose.count)
		return false;
	mirror = cmd;
	mirror.cmd = mirror_id;
	mirror.info.convolution.count = w.dim[0];
	return true;
}
// geometry of the mirrored convolution from (big = y or its gradient, w, small = a or its gradient)
bool conv_transpose_geom(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, const TV& big, const TV& w, const TV& small, ConvGeom& g)
{
	ccv_nnc_cmd_t mirror;
	return conv_mirror(cmd, w, CCV_NNC_CONVOLUTION_BACKWARD, mirror) && conv_geom(mirror, hint, big, w, small, g);
}

// workspace functions: the mirrored convolution's data gradient; for the backward its forward (da), weight gradient (dw) and the
// column sum over Cout (dbias)
size_t conv_transpose_forw_workspace(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	ConvGeom g;
	if (input_size < 2 || output_size < 1 || !in[0] || !in[1] || !out[0] || kind_of(in[0]) < 0 || !conv_transpose_geom(cmd, hint, view_of(out[0]), view_of(in[1]), view_of(in[0]), g))
		return (size_t)-1;
	return conv_workspace(g, kind_of(in[0]), conv_groups(cmd), conv_algorithm(cmd), CONV_DGRAD);
}
size_t conv_transpose_back_workspace(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	ccv_nnc_tensor_t* const g_t = input_size > 0 ? in[0] : 0;
	ccv_nnc_tensor_t* const a_t = input_size > 1 ? in[1] : 0;
	ccv_nnc_tensor_t* const w_t = input_size > 2 ? in[2] : 0;
	ccv_nnc_tensor_t* const da_t = output_size > 0 ? out[0] : 0;
	ccv_nnc_tensor_t* const dw_t = output_size > 1 ? out[1] : 0;
	ccv_nnc_tensor_t* const filt = dw_t ? dw_t : w_t;
	ccv_nnc_tensor_t* const small = a_t ? a_t : da_t;
	const int kind = g_t ? kind_of(g_t) : -1, groups = conv_groups(cmd), algo = conv_algorithm(cmd);
	ConvGeom g;
	if (kind < 0 || !filt || !small || !conv_transpose_geom(cmd, hint, view_of(g_t), view_of(filt), view_of(small), g))
		return (size_t)-1;
	size_t need = output_size > 2 && out[2] ? colsum_workspace_bytes(g.C) : 0;
	if (da_t && w_t && conv_transpose_geom(cmd, hint, view_of(g_t), view_of(w_t), view_of(da_t), g))
		need = std::max(need, conv_workspace(g, kind, groups, algo, CONV_FPROP));
	if (dw_t && a_t && conv_transpose_geom(cmd, hint, view_of(g_t), view_of(dw_t), view_of(a_t), g))
		need = std::max(need, conv_workspace(g, kind, groups, algo, CONV_WGRAD));
	return need;
}

// inputs (a, w, bias?), output y (always overwritten)
int conv_transpose_forw_nhwc(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 2 || output_size < 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const bias_t = input_size > 2 ? inputs[2] : 0;
	const int kind = kind_of(inputs[0]);
	if (kind < 0 || kind_of(inputs[1]) != kind || kind_of(outputs[0]) != kind || (bias_t && ((kind_of(bias_t) != kind && !is_f32(bias_t)) || CCV_IS_TENSOR_VIEW(bias_t))))
		return CCV_NNC_EXEC_INVALID;
	ConvGeom g;
	if (!conv_transpose_geom(cmd, hint, view_of(outputs[0]), view_of(inputs[1]), view_of(inputs[0]), g) || (bias_t && bias_t->info.dim[0] != g.C))
		return CCV_NNC_EXEC_INVALID;
	const size_t ws_bytes = conv_transpose_forw_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	unsigned char* const ws = ws_bytes ? (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !ws)
		return CCV_NNC_EXEC_OOM;
	const float* const bias32 = bias_t && is_f32(bias_t) ? bias_t->data.f32 : 0;
	const void* const bias16 = bias_t && !is_f32(bias_t) ? (const void*)bias_t->data.u8 : 0;
	return dgrad_nhwc(stream_of(stream_context), ws, kind, conv_algorithm(cmd), conv_groups(cmd), g, inputs[0]->data.u8, inputs[1]->data.u8, bias32, bias16, outputs[0]->data.u8);
}

// inputs (g, a, w), outputs (da, dw, dbias), any output may be NULL; dw / dbias honour CCV_NNC_ACCUMULATE_OUTPUT, da is overwritten
int conv_transpose_back_nhwc(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	ccv_nnc_tensor_t* const g_t = input_size > 0 ? inputs[0] : 0;
	ccv_nnc_tensor_t* const a_t = input_size > 1 ? inputs[1] : 0;
	ccv_nnc_tensor_t* const w_t = input_size > 2 ? inputs[2] : 0;
	ccv_nnc_tensor_t* const da_t = output_size > 0 ? outputs[0] : 0;
	ccv_nnc_tensor_t* const dw_t = output_size > 1 ? outputs[1] : 0;
	ccv_nnc_tensor_t* const dbias_t = output_size > 2 ? outputs[2] : 0;
	const ccv_nnc_tensor_t* const filt = dw_t ? dw_t : w_t;
	const ccv_nnc_tensor_t* const small = a_t ? a_t : da_t;
	const int kind = g_t ? kind_of(g_t) : -1;
	if (kind < 0 || !filt || !small || (dw_t && !a_t) || (da_t && !w_t))
		return CCV_NNC_EXEC_INVALID;
	ConvGeom g, gchk;
	if (!conv_transpose_geom(cmd, hint, view_of(g_t), view_of(filt), view_of(small), g))
		return CCV_NNC_EXEC_INVALID;
	// every operand is checked before the first launch: a refused call leaves the outputs as they were
	const int groups = conv_groups(cmd);
	if ((a_t && kind_of(a_t) != kind) || (w_t && kind_of(w_t) != kind) || (da_t && kind_of(da_t) != kind) || (dw_t && kind_of(dw_t) != kind))
		return CCV_NNC_EXEC_INVALID;
	if ((dw_t && !conv_transpose_geom(cmd, hint, view_of(g_t), view_of(dw_t), view_of(a_t), gchk)) || (da_t && !conv_transpose_geom(cmd, hint, view_of(g_t), view_of(w_t), view_of(da_t), gchk)))
		return CCV_NNC_EXEC_INVALID;
	// 16-bit forwards and weight gradients of one group run on the tensor cores only: Cin a multiple of 8 (grouped ones also on the
	// direct kernels)
	if (kind > 0 && (da_t || dw_t) && groups == 1 && g.K % 8)
		return CCV_NNC_EXEC_INVALID;
	const int db_kind = dbias_t ? kind_of(dbias_t) : 0;
	if (dbias_t && (db_kind < 0 || (kind == 0 && db_kind != 0) || dbias_t->info.dim[0] != g.C || g.ah != (long long)g.W * g.aw || g.an != (long long)g.H * g.ah))
		return CCV_NNC_EXEC_INVALID;
	// one request for the whole call: the mirrored commands below then get the same buffer
	const size_t ws_bytes = conv_transpose_back_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	void* const ws = ws_bytes ? ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !ws)
		return CCV_NNC_EXEC_OOM;
	if (da_t)
	{
		// da = conv(g, w), the mirrored convolution's forward
		ccv_nnc_cmd_t mirror;
		conv_mirror(cmd, view_of(w_t), CCV_NNC_CONVOLUTION_FORWARD, mirror);
		ccv_nnc_tensor_t* const in[2] = { g_t, w_t };
		ccv_nnc_tensor_t* const out[1] = { da_t };
		const int rc = conv_forw_nhwc(mirror, hint, 0, in, 2, out, 1, stream_context);
		if (rc != CCV_NNC_EXEC_SUCCESS)
			return rc;
	}
	if (dw_t)
	{
		// dw (+)= wgrad(grad = a, x = g) of the mirrored convolution
		ccv_nnc_cmd_t mirror;
		conv_mirror(cmd, view_of(dw_t), CCV_NNC_CONVOLUTION_BACKWARD, mirror);
		ccv_nnc_tensor_t* const in[3] = { a_t, g_t, 0 };
		ccv_nnc_tensor_t* const out[2] = { 0, dw_t };
		const int rc = conv_back_nhwc(mirror, hint, flags, in, 3, out, 2, stream_context);
		if (rc != CCV_NNC_EXEC_SUCCESS)
			return rc;
	}
	if (dbias_t)
	{
		// dbias[c] (+)= sum over the pixels of g, which are the mirrored convolution's input pixels
		const int accumulate = (flags & CCV_NNC_ACCUMULATE_OUTPUT) ? 1 : 0;
		cudaStream_t s = stream_of(stream_context);
		RC(colsum_any(s, kind, g_t->data.u8, (size_t)g.N * g.H * g.W, g.C, g.aw, dbias_t->data.u8, db_kind, accumulate, ws));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ BATCH NORM
// norm/ccv_nnc_batch_norm_cpu_ref.c:16-250.  Supported reduction shapes: per-channel statistics of an NHWC
// ([.., C], scale dims [1,1,1,C]) or NCHW ([N, C, H, W], scale dims [1,C,1,1]) tensor.
bool bn_layout(const TV& a, const TV& scale, size_t& outer, int& C, size_t& inner)
{
	int ad[4], as[4], rd[4], rs[4];
	if (a.nd > 4 || scale.nd > 4 || !a.contiguous || !scale.contiguous)
		return false;
	dims4(a, ad, as);
	dims4(scale, rd, rs);
	int axis = -1;
	for (int i = 0; i < 4; i++)
		if (rd[i] != 1)
		{
			if (axis >= 0 || rd[i] != ad[i])
				return false;
			axis = i;
		}
	if (axis < 0)
		axis = 3; // a single statistic over everything: C = 1
	if (rd[axis] == 1 && ad[axis] != 1)
	{
		// scale has one element but the tensor does not: treat the whole tensor as one channel
		outer = 1, C = 1, inner = a.count;
		return true;
	}
	outer = 1, inner = 1;
	for (int i = 0; i < axis; i++)
		outer *= ad[i];
	for (int i = axis + 1; i < 4; i++)
		inner *= ad[i];
	C = ad[axis];
	return true;
}

// resid (training only): y = relu(bn(x) + resid), the batch norm at the end of a residual block fused with the block's sum and ReLU
int bnorm_forw(const int fuse_relu, const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context, const ccv_nnc_tensor_t* const resid = 0)
{
	// a 6th input is the statistics tensor of a fused convolution -> batch norm pair (ccv_nnc_sm100_graph_fuse): its `sig`
	// field carries the number of valid partial rows the convolution produced for this issue (0 = none: reduce here)
	const ccv_nnc_tensor_t* const stats_t = input_size == 6 ? inputs[5] : 0;
	if ((input_size != 5 && input_size != 6) || output_size < 1)
		return CCV_NNC_EXEC_INVALID;
	// x / y may be fp32, bf16 or fp16; scale, bias and the statistics are fp32 (lib/nnc/ccv_cnnp_model_addons.c:954-956)
	for (int i = 1; i < 5; i++)
		if (!inputs[i] || !is_f32(inputs[i]))
			return CCV_NNC_EXEC_INVALID;
	const int kind = inputs[0] ? kind_of(inputs[0]) : -1;
	if (kind < 0 || !outputs[0] || kind_of(outputs[0]) != kind)
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), scale = view_of(inputs[1]), b = view_of(outputs[0]);
	size_t outer, inner;
	int C;
	if (!same_shape(a, b) || !b.contiguous || !bn_layout(a, scale, outer, C, inner))
		return CCV_NNC_EXEC_INVALID;
	if (resid && (fuse_relu || cmd.info.bnorm.is_test || kind_of(resid) != kind || !view_of(resid).contiguous || view_of(resid).count != b.count))
		return CCV_NNC_EXEC_INVALID;
	for (int i = 2; i < 5; i++)
		if (view_of(inputs[i]).count != (size_t)C)
			return CCV_NNC_EXEC_INVALID;
	cudaStream_t s = stream_of(stream_context);
	if (cmd.info.bnorm.is_test)
	{
		if (fuse_relu)
			return CCV_NNC_EXEC_INVALID;
		void* const tws = ccv_nnc_stream_context_get_workspace(stream_context, bn_workspace_bytes(C), CCV_TENSOR_GPU_MEMORY);
		if (!tws)
			return CCV_NNC_EXEC_OOM;
		if (kind == 0)
			RC(bn_fwd_test_f32(s, inputs[0]->data.f32, outputs[0]->data.f32, inputs[1]->data.f32, inputs[2]->data.f32, inputs[3]->data.f32, inputs[4]->data.f32, outer, C, inner, cmd.info.bnorm.epsilon, tws));
		else
			RC(bn_fwd_test_16(s, kind, inputs[0]->data.u8, outputs[0]->data.u8, inputs[1]->data.f32, inputs[2]->data.f32, inputs[3]->data.f32, inputs[4]->data.f32, outer, C, inner, cmd.info.bnorm.epsilon, tws));
		return CCV_NNC_EXEC_SUCCESS;
	}
	if (output_size != 5 || !outputs[1] || !outputs[2] || !outputs[3] || !outputs[4])
		return CCV_NNC_EXEC_INVALID;
	// running mean / var are updated in place (:45-46)
	if (inputs[3]->data.f32 != outputs[1]->data.f32 || inputs[4]->data.f32 != outputs[2]->data.f32)
		return CCV_NNC_EXEC_INVALID;
	if (view_of(outputs[3]).count != (size_t)C || view_of(outputs[4]).count != (size_t)C)
		return CCV_NNC_EXEC_INVALID;
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, bn_workspace_bytes(C), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	for (int i = 1; i < 5; i++)
		if (!is_f32(outputs[i]))
			return CCV_NNC_EXEC_INVALID;
	if (kind == 0)
		RC(bn_fwd_train_f32(s, inputs[0]->data.f32, outputs[0]->data.f32, inputs[1]->data.f32, inputs[2]->data.f32, outputs[1]->data.f32, outputs[2]->data.f32, outputs[3]->data.f32, outputs[4]->data.f32, outer, C, inner, cmd.info.bnorm.epsilon, cmd.info.bnorm.momentum, ws, fuse_relu,
			stats_t && inner == 1 ? stats_t->data.f32 : 0, stats_t ? (int)stats_t->sig : 0, resid ? resid->data.f32 : 0));
	else
		RC(bn_fwd_train_16(s, kind, inputs[0]->data.u8, outputs[0]->data.u8, inputs[1]->data.f32, inputs[2]->data.f32, outputs[1]->data.f32, outputs[2]->data.f32, outputs[3]->data.f32, outputs[4]->data.f32, outer, C, inner, cmd.info.bnorm.epsilon, cmd.info.bnorm.momentum, ws, fuse_relu,
			stats_t && inner == 1 ? stats_t->data.f32 : 0, stats_t ? (int)stats_t->sig : 0, resid ? resid->data.u8 : 0));
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_bnorm_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_forw(0, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

static inline bool h_t_ok(const ccv_nnc_tensor_t* const h) { return h != 0; }

// norm/ccv_nnc_batch_norm_cpu_ref.c:312-470: inputs[0] = g, [5] = a, [6] = scale, [13] = saved_mean, [14] = saved_inv_std;
// outputs (h, dscale, dbias)
int bnorm_back(const int fused_relu, const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 15 || output_size < 1)
		return CCV_NNC_EXEC_INVALID;
	// the fused form carries the forward bias in slot 7 (unused by BATCH_NORM_BACKWARD, norm/ccv_nnc_norm.c:28-37)
	const ccv_nnc_tensor_t* const bias_t = fused_relu ? inputs[7] : 0;
	if (fused_relu && !bias_t)
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const g_t = inputs[0];
	const ccv_nnc_tensor_t* const a_t = inputs[5];
	const ccv_nnc_tensor_t* const scale_t = inputs[6];
	const ccv_nnc_tensor_t* const mean_t = inputs[13];
	const ccv_nnc_tensor_t* const istd_t = inputs[14];
	if (!g_t || !a_t || !scale_t || !mean_t || !istd_t)
		return CCV_NNC_EXEC_INVALID;
	ccv_nnc_tensor_t* const h_t = outputs[0];
	ccv_nnc_tensor_t* const dscale_t = output_size > 1 ? outputs[1] : 0;
	ccv_nnc_tensor_t* const dbias_t = output_size > 2 ? outputs[2] : 0;
	// a 4th output is the bias gradient of the convolution that produced this batch norm's input (graph rewrite (g) of
	// ccv_nnc_sm100_graph_fuse): sum over pixels of the dx written here
	ccv_nnc_tensor_t* const conv_dbias_t = output_size > 3 ? outputs[3] : 0;
	const TV a = view_of(a_t), g = view_of(g_t), scale = view_of(scale_t);
	size_t outer, inner;
	int C;
	if (!same_shape(a, g) || !g.contiguous || !bn_layout(a, scale, outer, C, inner))
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(g_t);
	if (kind < 0 || kind_of(a_t) != kind || (h_t && kind_of(h_t) != kind) || !is_f32(scale_t) || !is_f32(mean_t) || !is_f32(istd_t) || (bias_t && !is_f32(bias_t)) || (dscale_t && !is_f32(dscale_t)) || (dbias_t && !is_f32(dbias_t)))
		return CCV_NNC_EXEC_INVALID;
	if (conv_dbias_t && (!h_t_ok(outputs[0]) || kind_of(conv_dbias_t) < 0 || view_of(conv_dbias_t).count != (size_t)C || !view_of(conv_dbias_t).contiguous))
		return CCV_NNC_EXEC_INVALID;
	if (h_t && (!same_shape(view_of(h_t), a) || !view_of(h_t).contiguous))
		return CCV_NNC_EXEC_INVALID;
	// every per-channel tensor is read or written as C packed floats
	for (const ccv_nnc_tensor_t* const t : { (const ccv_nnc_tensor_t*)mean_t, (const ccv_nnc_tensor_t*)istd_t, bias_t, (const ccv_nnc_tensor_t*)dscale_t, (const ccv_nnc_tensor_t*)dbias_t })
		if (t && (view_of(t).count != (size_t)C || !view_of(t).contiguous))
			return CCV_NNC_EXEC_INVALID;
	cudaStream_t s = stream_of(stream_context);
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, bn_workspace_bytes(C), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	if (kind == 0 && (!conv_dbias_t || is_f32(conv_dbias_t)))
		RC(bn_bwd_f32(s, g_t->data.f32, a_t->data.f32, scale_t->data.f32, bias_t ? bias_t->data.f32 : 0, mean_t->data.f32, istd_t->data.f32, h_t ? h_t->data.f32 : 0, dscale_t ? dscale_t->data.f32 : 0, dbias_t ? dbias_t->data.f32 : 0, outer, C, inner, ws, conv_dbias_t ? conv_dbias_t->data.f32 : 0));
	else if (kind != 0)
		RC(bn_bwd_16(s, kind, g_t->data.u8, a_t->data.u8, scale_t->data.f32, bias_t ? bias_t->data.f32 : 0, mean_t->data.f32, istd_t->data.f32, h_t ? (void*)h_t->data.u8 : 0, dscale_t ? dscale_t->data.f32 : 0, dbias_t ? dbias_t->data.f32 : 0, outer, C, inner, ws,
			conv_dbias_t ? (void*)conv_dbias_t->data.u8 : 0, conv_dbias_t ? kind_of(conv_dbias_t) : 0));
	else
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_bnorm_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_back(0, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// ================================================================================================ RELU / EW
int exec_relu_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || kind_of(inputs[0]) < 0 || kind_of(outputs[0]) != kind_of(inputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), b = view_of(outputs[0]);
	if (!a.contiguous || !b.contiguous || a.count != b.count)
		return CCV_NNC_EXEC_INVALID;
	if (kind_of(inputs[0]) == 0)
		RC(ew_relu_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, outputs[0]->data.f32, a.count));
	else
		RC(ew_relu_fwd_16(stream_of(stream_context), kind_of(inputs[0]), inputs[0]->data.u8, outputs[0]->data.u8, a.count));
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_relu_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 3 || output_size < 1 || !inputs[0] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const TV g = view_of(inputs[0]), b = view_of(inputs[2]), h = view_of(outputs[0]);
	if (!g.contiguous || !b.contiguous || !h.contiguous || g.count != b.count || g.count != h.count)
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(inputs[0]);
	if (kind < 0 || kind_of(inputs[2]) != kind || kind_of(outputs[0]) != kind)
		return CCV_NNC_EXEC_INVALID;
	if (kind == 0)
		RC(ew_relu_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[2]->data.f32, outputs[0]->data.f32, g.count));
	else
		RC(ew_relu_bwd_16(stream_of(stream_context), kind, inputs[0]->data.u8, inputs[2]->data.u8, outputs[0]->data.u8, g.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// the order EWSUM adds its operands in (ew/ccv_nnc_ew_cpu_ref.c:29-45): when the output is the storage of an operand z >= 1, that
// operand comes first and the rest follow left to right; otherwise plain left to right.  Starting from the aliased operand also keeps
// it from being overwritten before it is read: the fp32 sum runs in chunks of 8 operands, and every chunk after the first adds onto
// the output.
void ewsum_order(ccv_nnc_tensor_t* const* const inputs, const int input_size, const void* const out, int* const order)
{
	int k = 0;
	for (int z = 1; z < input_size && !k; z++)
		if (inputs[z]->data.u8 == out)
			k = z;
	order[0] = k;
	for (int z = 0, j = 1; z < input_size; z++)
		if (z != k)
			order[j++] = z;
}

// ew/ccv_nnc_ew_cpu_ref.c:15-110,207-214
int exec_ewsum_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size >= 1 && output_size >= 1 && outputs[0] && CCV_GET_DATA_TYPE(outputs[0]->info.datatype) == CCV_32S)
	{
		// int32 tensors (ew/gpu/ccv_nnc_ew_gpu_cudnn.cu registers CCV_32S; test/int/nnc/cudnn.tests.c:4817-4850)
		const TV ci = view_of(outputs[0]);
		const int* iptrs[64];
		if (!ci.contiguous || input_size > 64)
			return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < input_size; i++)
		{
			if (!inputs[i] || CCV_GET_DATA_TYPE(inputs[i]->info.datatype) != CCV_32S || !view_of(inputs[i]).contiguous || view_of(inputs[i]).count != ci.count)
				return CCV_NNC_EXEC_INVALID;
			iptrs[i] = inputs[i]->data.i32;
		}
		RC(ew_sum_i32(stream_of(stream_context), iptrs, input_size, outputs[0]->data.i32, ci.count));
		return CCV_NNC_EXEC_SUCCESS;
	}
	if (input_size < 1 || output_size < 1 || !outputs[0] || kind_of(outputs[0]) < 0)
		return CCV_NNC_EXEC_INVALID;
	const TV c = view_of(outputs[0]);
	if (!c.contiguous || input_size > 64)
		return CCV_NNC_EXEC_INVALID;
	if (kind_of(outputs[0]) > 0)
	{
		// bf16 / fp16: up to 8 operands, summed in fp32 and rounded once
		const int kind = kind_of(outputs[0]);
		const void* p16[8];
		if (input_size > 8)
			return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < input_size; i++)
		{
			if (!inputs[i] || kind_of(inputs[i]) != kind || !view_of(inputs[i]).contiguous || view_of(inputs[i]).count != c.count)
				return CCV_NNC_EXEC_INVALID;
		}
		int order[8];
		ewsum_order(inputs, input_size, outputs[0]->data.u8, order);
		for (int i = 0; i < input_size; i++)
			p16[i] = inputs[order[i]]->data.u8;
		if (input_size == 1)
		{
			if (p16[0] != outputs[0]->data.u8 && cudaMemcpyAsync(outputs[0]->data.u8, p16[0], c.count * 2, cudaMemcpyDeviceToDevice, stream_of(stream_context)) != cudaSuccess)
				return CCV_NNC_EXEC_INVALID;
			return CCV_NNC_EXEC_SUCCESS;
		}
		RC(ew_sum_16(stream_of(stream_context), kind, p16, input_size, outputs[0]->data.u8, c.count));
		return CCV_NNC_EXEC_SUCCESS;
	}
	const float* ptrs[64];
	for (int i = 0; i < input_size; i++)
	{
		if (!inputs[i] || !is_f32(inputs[i]))
			return CCV_NNC_EXEC_INVALID;
		const TV a = view_of(inputs[i]);
		if (!a.contiguous || a.count != c.count)
			return CCV_NNC_EXEC_INVALID;
	}
	int order[64];
	ewsum_order(inputs, input_size, outputs[0]->data.u8, order);
	for (int i = 0; i < input_size; i++)
		ptrs[i] = inputs[order[i]]->data.f32;
	cudaStream_t s = stream_of(stream_context);
	if (input_size == 1)
	{
		if (ptrs[0] != outputs[0]->data.f32 && cudaMemcpyAsync(outputs[0]->data.f32, ptrs[0], c.count * 4, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
			return CCV_NNC_EXEC_INVALID;
		return CCV_NNC_EXEC_SUCCESS;
	}
	RC(ew_sum_f32(s, ptrs, input_size, outputs[0]->data.f32, c.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// ew/ccv_nnc_ew_cpu_ref.c:216-233: every output receives the incoming gradient (or ones if it is absent)
int exec_ewsum_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	for (int i = 0; i < output_size; i++)
	{
		if (!outputs[i])
			continue;
		const TV h = view_of(outputs[i]);
		const int kind = kind_of(outputs[i]);
		if (!h.contiguous || kind < 0)
			return CCV_NNC_EXEC_INVALID;
		if (input_size < 1 || !inputs[0])
		{
			if (kind == 0)
				RC(ew_set_f32(s, outputs[i]->data.f32, h.count, 1.f));
			else
				RC(ew_set_u16(s, (uint16_t*)outputs[i]->data.u8, h.count, kind == 1 ? (uint16_t)0x3f80 : (uint16_t)0x3c00));
		} else if (inputs[0]->data.u8 != outputs[i]->data.u8) {
			const TV g = view_of(inputs[0]);
			if (!g.contiguous || g.count != h.count || kind_of(inputs[0]) != kind)
				return CCV_NNC_EXEC_INVALID;
			if (cudaMemcpyAsync(outputs[i]->data.u8, inputs[0]->data.u8, h.count * elem_size(kind), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
				return CCV_NNC_EXEC_INVALID;
		}
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// EWPROD operands: one floating-point kind, packed, the dims of `like` (no broadcasting), at most 4-d (ew/ccv_nnc_ew_cpu_ref.c:262-264)
bool ewprod_operand(const ccv_nnc_tensor_t* const t, const int kind, const TV& like)
{
	if (!t || kind_of(t) != kind)
		return false;
	const TV v = view_of(t);
	return v.contiguous && v.nd <= 4 && same_shape(v, like);
}

// ew/ccv_nnc_ew_cpu_ref.c:235-334,1688-1694: c = a0 * a1 * ... in EWSUM's operand order (ewsum_order), every product rounded on its own
int exec_ewprod_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs || !outputs || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(outputs[0]);
	if (kind < 0 || input_size > (kind == 0 ? 64 : 8))
		return CCV_NNC_EXEC_INVALID;
	const TV c = view_of(outputs[0]);
	if (!ewprod_operand(outputs[0], kind, c))
		return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < input_size; i++)
		if (!ewprod_operand(inputs[i], kind, c))
			return CCV_NNC_EXEC_INVALID;
	int order[64];
	const void* ptrs[64];
	ewsum_order(inputs, input_size, outputs[0]->data.u8, order);
	for (int i = 0; i < input_size; i++)
		ptrs[i] = inputs[order[i]]->data.u8;
	cudaStream_t s = stream_of(stream_context);
	if (input_size == 1)
	{
		if (ptrs[0] != outputs[0]->data.u8 && c.count && cudaMemcpyAsync(outputs[0]->data.u8, ptrs[0], c.count * elem_size(kind), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
			return CCV_NNC_EXEC_INVALID;
		return CCV_NNC_EXEC_SUCCESS;
	}
	RC(ew_prod(s, kind, ptrs, input_size, outputs[0]->data.u8, c.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// ew/ccv_nnc_ew_cpu_ref.c:336-480: inputs (g, a_1 .. a_n, b), outputs (h_1 .. h_n), h_i = g * b / a_i (b / a_i without g).  Every a, b and h
// is required; all outputs are written by one launch.
int exec_ewprod_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (output_size < 1 || input_size != output_size + 2 || !inputs || !outputs || !inputs[input_size - 1])
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const b = inputs[input_size - 1];
	const int kind = kind_of(b);
	if (kind < 0 || output_size > (kind == 0 ? 64 : 8))
		return CCV_NNC_EXEC_INVALID;
	const TV bv = view_of(b);
	if (!ewprod_operand(b, kind, bv) || (inputs[0] && !ewprod_operand(inputs[0], kind, bv)))
		return CCV_NNC_EXEC_INVALID;
	const void* a[64];
	void* h[64];
	for (int z = 0; z < output_size; z++)
	{
		if (!ewprod_operand(inputs[z + 1], kind, bv) || !ewprod_operand(outputs[z], kind, bv))
			return CCV_NNC_EXEC_INVALID;
		a[z] = inputs[z + 1]->data.u8, h[z] = outputs[z]->data.u8;
	}
	RC(ew_prod_back(stream_of(stream_context), kind, inputs[0] ? inputs[0]->data.u8 : 0, b->data.u8, a, h, output_size, bv.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// broadcasting helper: c's 4-d shape drives the loop; an operand dimension of 1 broadcasts (stride 0)
bool bcast_strides(const TV& c, const TV& x, int xs[4])
{
	int cd[4], cs[4], xd[4], xs0[4];
	if (c.nd > 4 || x.nd > 4)
		return false;
	dims4(c, cd, cs);
	dims4(x, xd, xs0);
	for (int i = 0; i < 4; i++)
	{
		if (xd[i] == cd[i])
			xs[i] = xd[i] == 1 ? 0 : xs0[i];
		else if (xd[i] == 1)
			xs[i] = 0;
		else
			return false;
	}
	return true;
}

// blas/ccv_nnc_add_cpu_ref.c:13-198: c = p * a + q * b, b optional, numpy-style broadcast of a and b into c
int exec_add_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || !is_f32(inputs[0]) || !is_f32(outputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const b_t = input_size > 1 ? inputs[1] : 0;
	const float p = cmd.info.blas.a[0], q = cmd.info.blas.a[1];
	const TV a = view_of(inputs[0]), c = view_of(outputs[0]);
	cudaStream_t s = stream_of(stream_context);
	if (a.contiguous && c.contiguous && same_shape(a, c) && (!b_t || (view_of(b_t).contiguous && same_shape(view_of(b_t), c))))
	{
		RC(ew_axpby_f32(s, p, inputs[0]->data.f32, q, b_t ? b_t->data.f32 : 0, outputs[0]->data.f32, c.count));
		return CCV_NNC_EXEC_SUCCESS;
	}
	int cd[4], cs[4], as[4], bs[4];
	if (c.nd > 4)
		return CCV_NNC_EXEC_INVALID;
	dims4(c, cd, cs);
	if (!bcast_strides(c, a, as) || (b_t && !bcast_strides(c, view_of(b_t), bs)))
		return CCV_NNC_EXEC_INVALID;
	RC(ew_axpby_bcast_f32(s, p, inputs[0]->data.f32, as, q, b_t ? b_t->data.f32 : 0, b_t ? bs : 0, outputs[0]->data.f32, cs, cd));
	return CCV_NNC_EXEC_SUCCESS;
}

// gradient of a broadcast operand: scale * g summed over the broadcast axes
int reduce_to(cudaStream_t s, const float scale, const ccv_nnc_tensor_t* const g_t, ccv_nnc_tensor_t* const out_t)
{
	const TV g = view_of(g_t), o = view_of(out_t);
	if (!o.contiguous || g.nd > 4 || o.nd > 4)
		return 1;
	if (g.contiguous && same_shape(g, o))
		return ew_axpby_f32(s, scale, g_t->data.f32, 0.f, 0, out_t->data.f32, o.count);
	int gd[4], gs[4], od[4], os[4];
	dims4(g, gd, gs);
	dims4(o, od, os);
	for (int i = 0; i < 4; i++)
		if (od[i] != gd[i] && od[i] != 1)
			return 1;
	return reduce_sum_bcast_f32(s, g_t->data.f32, gd, gs, out_t->data.f32, od, scale, 0);
}

// blas/ccv_nnc_add_cpu_ref.c:200-330
int exec_add_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	const float pq[2] = { cmd.info.blas.a[0], cmd.info.blas.a[1] };
	for (int i = 0; i < 2 && i < output_size; i++)
	{
		if (!outputs[i])
			continue;
		if (!is_f32(outputs[i]))
			return CCV_NNC_EXEC_INVALID;
		if (input_size < 1 || !inputs[0])
		{
			const TV o = view_of(outputs[i]);
			if (!o.contiguous)
				return CCV_NNC_EXEC_INVALID;
			RC(ew_set_f32(s, outputs[i]->data.f32, o.count, pq[i]));
		} else
			RC(reduce_to(s, pq[i], inputs[0], outputs[i]));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// blas/ccv_nnc_mul_cpu_ref.c: MUL c = p * a * b (broadcast); SCALAR_MUL c = p * a
int exec_mul_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 2 || output_size < 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	if (!is_f32(inputs[0]) || !is_f32(inputs[1]) || !is_f32(outputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), b = view_of(inputs[1]), c = view_of(outputs[0]);
	int cd[4], cs[4], as[4], bs[4];
	if (c.nd > 4)
		return CCV_NNC_EXEC_INVALID;
	dims4(c, cd, cs);
	if (!bcast_strides(c, a, as) || !bcast_strides(c, b, bs))
		return CCV_NNC_EXEC_INVALID;
	RC(ew_mul_bcast_f32(stream_of(stream_context), cmd.info.blas.a[0], inputs[0]->data.f32, as, inputs[1]->data.f32, bs, outputs[0]->data.f32, cs, cd));
	return CCV_NNC_EXEC_SUCCESS;
}

// blas/ccv_nnc_mul_cpu_ref.c:192-330: d(p a b)/da = p g b, d/db = p g a, each summed over the axes along which that operand was
// broadcast (g == NULL reads as ones).  Same shapes: one fused pass; otherwise the product is formed over the full index space fd
// -- the gradient's shape, or (no gradient) the broadcast of the two operands -- in the stream workspace and reduced onto the
// operand's shape in a fixed order.  mul_back_plan returns that space's element count for outputs[i], 0 for the fused pass,
// (size_t)-1 when refused.
size_t mul_back_plan(ccv_nnc_tensor_t* const* const inputs, ccv_nnc_tensor_t* const* const outputs, const int i, int fd[4], int fs[4], int od[4], int xs[4], int gs[4])
{
	const ccv_nnc_tensor_t* const other = inputs[2 - i]; // ha needs b (inputs[2]), hb needs a (inputs[1])
	if (!other || !is_f32(other) || !is_f32(outputs[i]) || (inputs[0] && !is_f32(inputs[0])))
		return (size_t)-1;
	const TV o = view_of(outputs[i]), x = view_of(other);
	if (!o.contiguous || o.nd > 4 || x.nd > 4)
		return (size_t)-1;
	int os[4], xd[4], gd[4] = { 1, 1, 1, 1 };
	dims4(o, od, os);
	if (x.contiguous && same_shape(o, x) && (!inputs[0] || (view_of(inputs[0]).contiguous && same_shape(view_of(inputs[0]), o))))
	{
		memcpy(fs, os, sizeof(os));
		return 0;
	}
	dims4(x, xd, xs);
	memset(gs, 0, 4 * sizeof(int));
	if (inputs[0])
	{
		const TV g = view_of(inputs[0]);
		if (g.nd > 4)
			return (size_t)-1;
		dims4(g, gd, gs);
	}
	size_t fcount = 1;
	for (int k = 0; k < 4; k++)
	{
		fd[k] = std::max(std::max(od[k], xd[k]), gd[k]);
		if ((od[k] != fd[k] && od[k] != 1) || (xd[k] != fd[k] && xd[k] != 1) || (gd[k] != fd[k] && gd[k] != 1))
			return (size_t)-1;
		if (xd[k] == 1)
			xs[k] = 0;
		if (gd[k] == 1)
			gs[k] = 0;
		fcount *= (size_t)fd[k];
	}
	for (int k = 3, packed = 1; k >= 0; k--)
		fs[k] = packed, packed *= fd[k];
	return fcount;
}
// the largest full index space of the two gradients, in fp32
size_t mul_back_workspace(const ccv_nnc_cmd_t&, const ccv_nnc_hint_t&, ccv_nnc_tensor_t* const* const in, const int input_size, ccv_nnc_tensor_t* const* const out, const int output_size)
{
	if (input_size < 3)
		return (size_t)-1;
	size_t need = 0;
	int fd[4], fs[4], od[4], xs[4], gs[4];
	for (int i = 0; i < 2 && i < output_size; i++)
		if (out[i])
		{
			const size_t n = mul_back_plan(in, out, i, fd, fs, od, xs, gs);
			if (n == (size_t)-1)
				return n;
			need = std::max(need, n * sizeof(float));
		}
	return need;
}
int exec_mul_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const size_t ws_bytes = mul_back_workspace(cmd, hint, inputs, input_size, outputs, output_size);
	if (ws_bytes == (size_t)-1)
		return CCV_NNC_EXEC_INVALID;
	float* const t = ws_bytes ? (float*)ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY) : 0;
	if (ws_bytes && !t)
		return CCV_NNC_EXEC_OOM;
	cudaStream_t s = stream_of(stream_context);
	const float p = cmd.info.blas.a[0];
	for (int i = 0; i < 2 && i < output_size; i++)
	{
		if (!outputs[i])
			continue;
		const ccv_nnc_tensor_t* const other = inputs[2 - i];
		int fd[4], fs[4], od[4], xs[4], gs[4];
		if (!mul_back_plan(inputs, outputs, i, fd, fs, od, xs, gs))
		{
			if (!inputs[0])
				RC(ew_axpby_f32(s, p, other->data.f32, 0.f, 0, outputs[i]->data.f32, view_of(outputs[i]).count));
			else
				RC(ew_mul_bcast_f32(s, p, inputs[0]->data.f32, fs, other->data.f32, fs, outputs[i]->data.f32, fs, od));
			continue;
		}
		if (inputs[0])
			RC(ew_mul_bcast_f32(s, p, inputs[0]->data.f32, gs, other->data.f32, xs, t, fs, fd));
		else
			RC(ew_axpby_bcast_f32(s, p, other->data.f32, xs, 0.f, 0, 0, t, fs, fd));
		RC(reduce_sum_bcast_f32(s, t, fd, fs, outputs[i]->data.f32, od, 1.f, 0));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_scalar_mul_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || !is_f32(inputs[0]) || !is_f32(outputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), c = view_of(outputs[0]);
	if (!a.contiguous || !c.contiguous || a.count != c.count)
		return CCV_NNC_EXEC_INVALID;
	RC(ew_axpby_f32(stream_of(stream_context), cmd.info.blas.a[0], inputs[0]->data.f32, 0.f, 0, outputs[0]->data.f32, c.count));
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_scalar_mul_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (output_size < 1 || !outputs[0] || !is_f32(outputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const TV h = view_of(outputs[0]);
	if (!h.contiguous)
		return CCV_NNC_EXEC_INVALID;
	cudaStream_t s = stream_of(stream_context);
	if (input_size < 1 || !inputs[0])
		RC(ew_set_f32(s, outputs[0]->data.f32, h.count, cmd.info.blas.a[0]));
	else {
		if (!view_of(inputs[0]).contiguous || view_of(inputs[0]).count != h.count)
			return CCV_NNC_EXEC_INVALID;
		RC(ew_axpby_f32(s, cmd.info.blas.a[0], inputs[0]->data.f32, 0.f, 0, outputs[0]->data.f32, h.count));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ POOLING
bool pool_geom(const ccv_nnc_cmd_t& cmd, const ccv_nnc_hint_t& hint, const TV& a, const TV& b, PoolGeom& g)
{
	if (a.format != CCV_TENSOR_FORMAT_NHWC || b.format != CCV_TENSOR_FORMAT_NHWC)
		return false;
	if ((a.nd != 3 && a.nd != 4) || a.nd != b.nd)
		return false;
	const int ao = a.nd - 3, bo = b.nd - 3;
	memset(&g, 0, sizeof(g));
	g.N = a.nd == 4 ? a.dim[0] : 1;
	if (b.nd == 4 && b.dim[0] != g.N)
		return false;
	g.H = a.dim[ao], g.W = a.dim[ao + 1], g.C = a.dim[ao + 2];
	g.P = b.dim[bo], g.Q = b.dim[bo + 1];
	if (b.dim[bo + 2] != g.C || a.stride[ao + 2] != 1 || b.stride[bo + 2] != 1)
		return false;
	g.an = a.nd == 4 ? a.stride[0] : 0, g.ah = a.stride[ao], g.aw = a.stride[ao + 1];
	g.bn = b.nd == 4 ? b.stride[0] : 0, g.bh = b.stride[bo], g.bw = b.stride[bo + 1];
	g.R = cmd.info.size.dim[0], g.S = cmd.info.size.dim[1];
	g.stride_h = hint.stride.dim[0] > 0 ? hint.stride.dim[0] : 1;
	g.stride_w = hint.stride.dim[1] > 0 ? hint.stride.dim[1] : 1;
	g.pad_h = hint.border.begin[0], g.pad_w = hint.border.begin[1];
	return g.R > 0 && g.S > 0;
}

// pool/ccv_nnc_max_pool_cpu_ref.c:13-59 / pool/ccv_nnc_avg_pool_cpu_ref.c:13-58 (all N images, unlike CPU_REF which
// only walks image 0 -- SURVEY.md 0.6)
template <int IS_MAX>
int exec_pool_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || kind_of(inputs[0]) < 0 || kind_of(outputs[0]) != kind_of(inputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(inputs[0]);
	PoolGeom g;
	if (!pool_geom(cmd, hint, view_of(inputs[0]), view_of(outputs[0]), g))
		return CCV_NNC_EXEC_INVALID;
	if (kind != 0)
		RC(IS_MAX ? pool_max_fwd_16(stream_of(stream_context), kind, g, inputs[0]->data.u8, outputs[0]->data.u8) : pool_avg_fwd_16(stream_of(stream_context), kind, g, inputs[0]->data.u8, outputs[0]->data.u8));
	else if (IS_MAX)
		RC(pool_max_fwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, outputs[0]->data.f32));
	else
		RC(pool_avg_fwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, outputs[0]->data.f32));
	return CCV_NNC_EXEC_SUCCESS;
}

// max: inputs (g, a, b) -> h; avg: inputs (g, ...) -> h
template <int IS_MAX>
int exec_pool_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || kind_of(inputs[0]) < 0 || kind_of(outputs[0]) != kind_of(inputs[0]))
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(inputs[0]);
	PoolGeom g;
	if (!pool_geom(cmd, hint, view_of(outputs[0]), view_of(inputs[0]), g))
		return CCV_NNC_EXEC_INVALID;
	if (IS_MAX)
	{
		if (input_size < 3 || !inputs[1] || !inputs[2])
			return CCV_NNC_EXEC_INVALID;
		const TV a = view_of(inputs[1]), b = view_of(inputs[2]), gv = view_of(inputs[0]), h = view_of(outputs[0]);
		// the kernel addresses a with h's strides and b with g's strides
		if (!same_shape(a, h) || !same_shape(b, gv))
			return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < a.nd; i++)
			if (a.stride[i] != h.stride[i])
				return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < b.nd; i++)
			if (b.stride[i] != gv.stride[i])
				return CCV_NNC_EXEC_INVALID;
		if (kind_of(inputs[1]) != kind || kind_of(inputs[2]) != kind)
			return CCV_NNC_EXEC_INVALID;
		if (kind != 0)
			RC(pool_max_bwd_16(stream_of(stream_context), kind, g, inputs[0]->data.u8, inputs[1]->data.u8, inputs[2]->data.u8, outputs[0]->data.u8));
		else
			RC(pool_max_bwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, inputs[1]->data.f32, inputs[2]->data.f32, outputs[0]->data.f32));
	} else if (kind != 0)
		RC(pool_avg_bwd_16(stream_of(stream_context), kind, g, inputs[0]->data.u8, outputs[0]->data.u8));
	else
		RC(pool_avg_bwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, outputs[0]->data.f32));
	return CCV_NNC_EXEC_SUCCESS;
}

// AVERAGE_POOL_BACKWARD(g -> s) ; EWSUM(r, s -> out) ; RELU_BACKWARD in place on out (mask y), as one pass out = y > 0 ? r + s : 0 that
// never writes s: inputs (g, r, y), outputs (out).  Geometries the one-pass kernel does not take run the three steps with s in the
// workspace.
int exec_avgpool_add_relu_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 3 || output_size != 1 || !inputs[0] || !inputs[1] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(outputs[0]);
	const TV r = view_of(inputs[1]), y = view_of(inputs[2]), o = view_of(outputs[0]);
	if (kind < 0 || kind_of(inputs[0]) != kind || kind_of(inputs[1]) != kind || kind_of(inputs[2]) != kind || !r.contiguous || !y.contiguous || !o.contiguous || !same_shape(r, o) || !same_shape(y, o))
		return CCV_NNC_EXEC_INVALID;
	PoolGeom g;
	if (!pool_geom(cmd, hint, o, view_of(inputs[0]), g))
		return CCV_NNC_EXEC_INVALID;
	cudaStream_t s = stream_of(stream_context);
	const int rc = pool_avg_bwd_add_relu(s, kind, g, inputs[0]->data.u8, inputs[1]->data.u8, inputs[2]->data.u8, outputs[0]->data.u8);
	if (rc <= 0)
		return rc ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, o.count * (kind == 0 ? 4 : 2), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	if (kind != 0)
	{
		RC(pool_avg_bwd_16(s, kind, g, inputs[0]->data.u8, ws));
		RC(ew_add_relu_bwd_16(s, kind, inputs[1]->data.u8, ws, inputs[2]->data.u8, outputs[0]->data.u8, o.count));
	} else {
		RC(pool_avg_bwd_f32(s, g, inputs[0]->data.f32, (float*)ws));
		RC(ew_add_relu_bwd_f32(s, inputs[1]->data.f32, (const float*)ws, inputs[2]->data.f32, outputs[0]->data.f32, o.count));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ SOFTMAX / LOSSES
bool rows_of(const TV& a, int& batch, int& count)
{
	if (!a.contiguous || a.nd < 1)
		return false;
	batch = a.nd < 2 ? 1 : a.dim[0];
	count = (int)(a.count / (size_t)batch);
	return true;
}

int exec_softmax_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0] || !is_f32(inputs[0]) || !is_f32(outputs[0]))
		return CCV_NNC_EXEC_INVALID;
	int batch, count;
	const TV a = view_of(inputs[0]), b = view_of(outputs[0]);
	if (!rows_of(a, batch, count) || !b.contiguous || !same_shape(a, b))
		return CCV_NNC_EXEC_INVALID;
	RC(softmax_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, outputs[0]->data.f32, batch, count));
	return CCV_NNC_EXEC_SUCCESS;
}

int exec_softmax_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 3 || output_size < 1 || !inputs[0] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int batch, count;
	const TV g = view_of(inputs[0]), b = view_of(inputs[2]), h = view_of(outputs[0]);
	if (!rows_of(g, batch, count) || !b.contiguous || !h.contiguous || !same_shape(g, b) || !same_shape(g, h))
		return CCV_NNC_EXEC_INVALID;
	RC(softmax_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[2]->data.f32, outputs[0]->data.f32, batch, count));
	return CCV_NNC_EXEC_SUCCESS;
}

// label tensor -> kind (0 fp32 index, 1 int32 index, 2 fp32 distribution), following the reference's "range" rule
// (loss/ccv_nnc_categorical_crossentropy_cpu_ref.c:27-30)
bool label_kind_of(const ccv_nnc_tensor_t* const b_t, const int batch, int& kind)
{
	const TV b = view_of(b_t);
	if (!b.contiguous)
		return false;
	if (CCV_GET_DATA_TYPE(b_t->info.datatype) == CCV_32S)
	{
		kind = 1;
		return true;
	}
	if (CCV_GET_DATA_TYPE(b_t->info.datatype) != CCV_32F)
		return false;
	int range;
	if (b.nd > 1)
		range = b.dim[b.nd - 1]; // ccv_nnc_tensor_get_c for the 2-d [batch, count] case
	else
		range = batch == 1 ? b.dim[0] : 1;
	kind = range == 1 ? 0 : 2;
	return true;
}

// the label holds one class index per row (kind 0 / 1) or one row of `count` probabilities per row (kind 2)
bool label_fits(const ccv_nnc_tensor_t* const b_t, const int kind, const int batch, const int count)
{
	return view_of(b_t).count == (size_t)batch * (kind == 2 ? (size_t)count : 1);
}

// a loss c or a gradient g of the loss: one fp32 value per row (absent: g reads as ones)
bool per_row_ok(const ccv_nnc_tensor_t* const t, const int batch)
{
	return !t || (is_f32(t) && view_of(t).contiguous && view_of(t).count == (size_t)batch);
}

int exec_cce_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 2 || output_size < 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int batch, count, kind;
	if (!is_f32(inputs[0]) || !rows_of(view_of(inputs[0]), batch, count) || !label_kind_of(inputs[1], batch, kind) || !label_fits(inputs[1], kind, batch, count) || !per_row_ok(outputs[0], batch))
		return CCV_NNC_EXEC_INVALID;
	RC(cce_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[1]->data.ptr, kind, outputs[0]->data.f32, batch, count, cmd.info.label_smoothing.trim0, cmd.info.label_smoothing.trim1));
	return CCV_NNC_EXEC_SUCCESS;
}

// inputs (g, a, b) -> h
int exec_cce_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 3 || output_size < 1 || !inputs[1] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int batch, count, kind;
	if (!is_f32(inputs[1]) || !rows_of(view_of(inputs[1]), batch, count) || !label_kind_of(inputs[2], batch, kind) || !label_fits(inputs[2], kind, batch, count) || !per_row_ok(inputs[0], batch) || !view_of(outputs[0]).contiguous || !same_shape(view_of(inputs[1]), view_of(outputs[0])))
		return CCV_NNC_EXEC_INVALID;
	RC(cce_bwd_f32(stream_of(stream_context), inputs[0] ? inputs[0]->data.f32 : 0, inputs[1]->data.f32, inputs[2]->data.ptr, kind, outputs[0]->data.f32, batch, count, cmd.info.label_smoothing.trim0, cmd.info.label_smoothing.trim1));
	return CCV_NNC_EXEC_SUCCESS;
}

// softmax_loss/ccv_nnc_softmax_crossentropy_cpu_ref.c:13-170: inputs (a, label) -> outputs (c, d)
int exec_softmax_cce_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 2 || output_size != 2 || !inputs[0] || !inputs[1] || !outputs[1])
		return CCV_NNC_EXEC_INVALID;
	int batch, count, kind;
	if (!is_f32(inputs[0]) || !rows_of(view_of(inputs[0]), batch, count) || !label_kind_of(inputs[1], batch, kind) || !label_fits(inputs[1], kind, batch, count) || !per_row_ok(outputs[0], batch) || !view_of(outputs[1]).contiguous || !same_shape(view_of(inputs[0]), view_of(outputs[1])))
		return CCV_NNC_EXEC_INVALID;
	RC(softmax_cce_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[1]->data.ptr, kind, outputs[0] ? outputs[0]->data.f32 : 0, outputs[1]->data.f32, batch, count, cmd.info.label_smoothing.trim0, cmd.info.label_smoothing.trim1));
	return CCV_NNC_EXEC_SUCCESS;
}

// inputs: [0] = g (may be NULL), [3] = label, [5] = d; outputs[0] = h (:172-181)
int exec_softmax_cce_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 6 || output_size < 1 || !inputs[3] || !inputs[5] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int batch, count, kind;
	if (!is_f32(inputs[5]) || !rows_of(view_of(inputs[5]), batch, count) || !label_kind_of(inputs[3], batch, kind) || !label_fits(inputs[3], kind, batch, count) || !per_row_ok(inputs[0], batch) || !view_of(outputs[0]).contiguous || !same_shape(view_of(inputs[5]), view_of(outputs[0])))
		return CCV_NNC_EXEC_INVALID;
	RC(softmax_cce_bwd_f32(stream_of(stream_context), inputs[0] ? inputs[0]->data.f32 : 0, inputs[3]->data.ptr, kind, inputs[5]->data.f32, outputs[0]->data.f32, batch, count, cmd.info.label_smoothing.trim0, cmd.info.label_smoothing.trim1));
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ SGD
// sgd/ccv_nnc_sgd_cpu_ref.c:16-126: inputs (g, a, m) -> outputs (b, n)
int exec_sgd_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 3 || output_size != 2)
		return CCV_NNC_EXEC_INVALID;
	size_t count = 0;
	// the gradient may be fp32, bf16 or fp16; parameters and momenta are fp32 (the reference's GPU kernel takes the mixed form
	// g 16-bit / a, m fp32 too: sgd/gpu/ccv_nnc_sgd_gpu_ref.cu:71-74)
	for (int i = 0; i < 3; i++)
	{
		if (!inputs[i] || (i == 0 ? kind_of(inputs[i]) < 0 : !is_f32(inputs[i])) || !view_of(inputs[i]).contiguous)
			return CCV_NNC_EXEC_INVALID;
		if (i == 0)
			count = view_of(inputs[0]).count;
		else if (view_of(inputs[i]).count != count)
			return CCV_NNC_EXEC_INVALID;
	}
	for (int i = 0; i < 2; i++)
		if (!outputs[i] || !is_f32(outputs[i]) || !view_of(outputs[i]).contiguous || view_of(outputs[i]).count != count)
			return CCV_NNC_EXEC_INVALID;
	if (cmd.info.sgd.nesterov && cmd.info.sgd.dampening != 0)
		return CCV_NNC_EXEC_INVALID;
	RC(sgd_any(stream_of(stream_context), kind_of(inputs[0]), inputs[0]->data.u8, inputs[1]->data.f32, inputs[2]->data.f32, outputs[0]->data.f32, outputs[1]->data.f32, count, cmd.info.sgd.nesterov, cmd.info.sgd.rate, cmd.info.sgd.scale, cmd.info.sgd.decay, cmd.info.sgd.momentum, cmd.info.sgd.dampening));
	return CCV_NNC_EXEC_SUCCESS;
}

// A run of SGD_FORWARD commands with identical parameters, merged by ccv_nnc_sm100_graph_fuse: inputs = (g, a, m) x T,
// outputs = (b, n) x T.  Every triple is validated exactly as exec_sgd_forw validates one command.
int exec_sgd_multi(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size % 3 != 0 || output_size * 3 != input_size * 2 || input_size == 0)
		return CCV_NNC_EXEC_INVALID;
	if (cmd.info.sgd.nesterov && cmd.info.sgd.dampening != 0)
		return CCV_NNC_EXEC_INVALID;
	const int T = input_size / 3;
	std::vector<const void*> g(T);
	std::vector<const float*> a(T), m(T);
	std::vector<float*> b(T), n(T);
	const int g_kind = inputs[0] ? kind_of(inputs[0]) : -1;
	if (g_kind < 0)
		return CCV_NNC_EXEC_INVALID;
	std::vector<size_t> counts(T);
	for (int t = 0; t < T; t++)
	{
		for (int i = 0; i < 3; i++)
			if (!inputs[3 * t + i] || (i == 0 ? kind_of(inputs[3 * t]) != g_kind : !is_f32(inputs[3 * t + i])) || !view_of(inputs[3 * t + i]).contiguous)
				return CCV_NNC_EXEC_INVALID;
		counts[t] = view_of(inputs[3 * t]).count;
		if (view_of(inputs[3 * t + 1]).count != counts[t] || view_of(inputs[3 * t + 2]).count != counts[t])
			return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < 2; i++)
			if (!outputs[2 * t + i] || !is_f32(outputs[2 * t + i]) || !view_of(outputs[2 * t + i]).contiguous || view_of(outputs[2 * t + i]).count != counts[t])
				return CCV_NNC_EXEC_INVALID;
		g[t] = inputs[3 * t]->data.u8, a[t] = inputs[3 * t + 1]->data.f32, m[t] = inputs[3 * t + 2]->data.f32;
		b[t] = outputs[2 * t]->data.f32, n[t] = outputs[2 * t + 1]->data.f32;
	}
	RC(sgd_multi_any(stream_of(stream_context), T, g_kind, g.data(), a.data(), m.data(), b.data(), n.data(), counts.data(), cmd.info.sgd.nesterov, cmd.info.sgd.rate, cmd.info.sgd.scale, cmd.info.sgd.decay, cmd.info.sgd.momentum, cmd.info.sgd.dampening));
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ SET / MOVES
// util/ccv_nnc_util_cpu_ref.c:637-664
int exec_set_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	const float v = cmd.cmd == CCV_NNC_SET_BACKWARD ? 0.f : cmd.info.blas.a[0];
	for (int i = 0; i < output_size; i++)
	{
		if (!outputs[i])
			continue;
		const TV o = view_of(outputs[i]);
		if (!o.contiguous)
			return CCV_NNC_EXEC_INVALID;
		const int dt = CCV_GET_DATA_TYPE(outputs[i]->info.datatype);
		if (v == 0.f)
		{
			if (cudaMemsetAsync(outputs[i]->data.u8, 0, o.count * dtype_size(dt), s) != cudaSuccess)
				return CCV_NNC_EXEC_INVALID;
		} else if (dt == CCV_32F)
			RC(ew_set_f32(s, outputs[i]->data.f32, o.count, v));
		else if (dt == CCV_32S) {
			const int iv = (int)v;
			float fv;
			memcpy(&fv, &iv, 4);
			RC(ew_set_f32(s, outputs[i]->data.f32, o.count, fv));
		} else if (dt == CCV_64F) {
			// a double is two 32-bit words: fill the word pairs (o.count * 2 words, even / odd word pattern)
			const double dv = (double)v;
			RC(ew_set_u64(s, (uint64_t*)outputs[i]->data.u8, o.count, *(const uint64_t*)&dv));
		} else if (dt == CCV_16F || dt == CCV_16BF)
			RC(ew_set_u16(s, (uint16_t*)outputs[i]->data.u8, o.count, f32_to_16(v, dt == CCV_16BF ? 1 : 2)));
		else
			return CCV_NNC_EXEC_INVALID;
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// copy between two tensors of equal shape and datatype: memcpy when both are packed, strided kernel otherwise
int copy_tensor(cudaStream_t s, const ccv_nnc_tensor_t* const a_t, ccv_nnc_tensor_t* const b_t)
{
	const TV a = view_of(a_t), b = view_of(b_t);
	if (a.datatype != b.datatype || a.count != b.count)
		return 1;
	const size_t es = dtype_size(a.datatype);
	const int a_gpu = CCV_TENSOR_GET_MEMORY(a_t->info.type) == CCV_TENSOR_GPU_MEMORY, b_gpu = CCV_TENSOR_GET_MEMORY(b_t->info.type) == CCV_TENSOR_GPU_MEMORY;
	if (a.contiguous && b.contiguous)
	{
		const cudaMemcpyKind kind = a_gpu ? (b_gpu ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost) : (b_gpu ? cudaMemcpyHostToDevice : cudaMemcpyHostToHost);
		const cudaError_t e = cudaMemcpyAsync(b.p, a.p, a.count * es, kind, s);
		if (e != cudaSuccess)
		{
			set_last_error("cudaMemcpyAsync(data transfer)", e);
			return -1;
		}
		count_launch(0);
		return 0;
	}
	if (!a_gpu || !b_gpu || a.nd > 4 || !same_shape(a, b))
		return 1;
	int ad[4], as[4], bd[4], bs[4];
	dims4(a, ad, as);
	dims4(b, bd, bs);
	return copy_strided(s, a.p, as, b.p, bs, ad, (int)es);
}

// util/ccv_nnc_util_cpu_ref.c:596-617
int exec_data_transfer(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	const int n = input_size < output_size ? input_size : output_size;
	for (int i = 0; i < n; i++)
		if (inputs[i] && outputs[i] && inputs[i] != outputs[i])
			RC(copy_tensor(s, inputs[i], outputs[i]));
	// Without a stream context the reference's transfer is the BLOCKING cudaMemcpy (util/gpu/ccv_nnc_util_gpu_ref.cu:44-60): the
	// caller reads a pinned host tensor right after the call (test/int/nnc/schedule.tests.c:56-59).  The copies above were enqueued
	// on the default stream; wait for them.
	if (!stream_context && cudaStreamSynchronize(s) != cudaSuccess)
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// util/ccv_nnc_util_cpu_ref.c:996-1082: same format = copy; NHWC <-> NCHW = copy over permuted strides
int exec_format_transform(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	for (int i = 0; i < output_size && i < input_size; i++)
	{
		if (!inputs[i] || !outputs[i])
			continue;
		const TV a = view_of(inputs[i]), b = view_of(outputs[i]);
		if (a.dim[0] == 0 || b.dim[0] == 0)
			continue;
		if (a.format == b.format)
		{
			RC(copy_tensor(s, inputs[i], outputs[i]));
			continue;
		}
		if (a.nd == b.nd && a.nd < 3)
		{
			// a vector / matrix tagged with another format (the bias gradient of an NCHW convolution, test/int/nnc/cudnn.tests.c:455-471): plain copy
			RC(copy_tensor(s, inputs[i], outputs[i]));
			continue;
		}
		if (a.datatype != b.datatype || a.nd != b.nd || (a.nd != 3 && a.nd != 4))
			return CCV_NNC_EXEC_INVALID;
		// express both in (n, c, h, w) index order
		int d[4], as[4], bs[4];
		const int o = a.nd - 3;
		auto nchw_of = [&](const TV& t, int dim[4], int st[4]) -> bool {
			dim[0] = t.nd == 4 ? t.dim[0] : 1, st[0] = t.nd == 4 ? t.stride[0] : 0;
			if (t.format == CCV_TENSOR_FORMAT_NHWC)
				dim[1] = t.dim[o + 2], st[1] = t.stride[o + 2], dim[2] = t.dim[o], st[2] = t.stride[o], dim[3] = t.dim[o + 1], st[3] = t.stride[o + 1];
			else if (t.format == CCV_TENSOR_FORMAT_NCHW)
				dim[1] = t.dim[o], st[1] = t.stride[o], dim[2] = t.dim[o + 1], st[2] = t.stride[o + 1], dim[3] = t.dim[o + 2], st[3] = t.stride[o + 2];
			else
				return false;
			return true;
		};
		int bd[4];
		if (!nchw_of(a, d, as) || !nchw_of(b, bd, bs))
			return CCV_NNC_EXEC_INVALID;
		for (int k = 0; k < 4; k++)
			if (d[k] != bd[k])
				return CCV_NNC_EXEC_INVALID;
		RC(copy_strided(s, a.p, as, b.p, bs, d, (int)dtype_size(a.datatype)));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// util/ccv_nnc_util_cpu_ref.c:1102-1180: swap two axes
int exec_transpose(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	for (int i = 0; i < output_size && i < input_size; i++)
	{
		if (!inputs[i] || !outputs[i])
			continue;
		const TV a = view_of(inputs[i]), b = view_of(outputs[i]);
		if (a.nd != b.nd || a.nd > 4 || a.datatype != b.datatype)
			return CCV_NNC_EXEC_INVALID;
		const int ax0 = cmd.info.transpose.axis[0], ax1 = cmd.info.transpose.axis[1];
		if (ax0 < 0 || ax1 < 0 || ax0 >= a.nd || ax1 >= a.nd)
			return CCV_NNC_EXEC_INVALID;
		int d[4], as[4], bs[4];
		const int off = 4 - a.nd;
		for (int k = 0; k < 4; k++)
		{
			if (k < off)
			{
				d[k] = 1, as[k] = bs[k] = 0;
				continue;
			}
			const int bk = k - off; // index in b
			const int ak = bk == ax0 ? ax1 : (bk == ax1 ? ax0 : bk);
			if (b.dim[bk] != a.dim[ak])
				return CCV_NNC_EXEC_INVALID;
			d[k] = b.dim[bk], bs[k] = b.stride[bk], as[k] = a.stride[ak];
		}
		RC(copy_strided(s, a.p, as, b.p, bs, d, (int)dtype_size(a.datatype)));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// util/ccv_nnc_util_cpu_ref.c:1200-1260
int exec_datatype_conversion(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	for (int i = 0; i < output_size && i < input_size; i++)
	{
		if (!inputs[i] || !outputs[i])
			continue;
		const TV a = view_of(inputs[i]), b = view_of(outputs[i]);
		if (a.count != b.count)
			return CCV_NNC_EXEC_INVALID;
		if (a.datatype == b.datatype)
		{
			RC(copy_tensor(s, inputs[i], outputs[i]));
			continue;
		}
		if (!a.contiguous || !b.contiguous || dtype_code(a.datatype) < 0 || dtype_code(b.datatype) < 0)
			return CCV_NNC_EXEC_INVALID;
		RC(convert_dtype(s, a.p, dtype_code(a.datatype), b.p, dtype_code(b.datatype), a.count));
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// ================================================================================================ 16-bit tensors on fp32-only commands
// The commands below have fp32 kernels only; the reference's GPU backends register them for CCV_16F as well (e.g.
// softmax/gpu/ccv_nnc_softmax_gpu_cudnn.cu, blas/gpu/ccv_nnc_add_gpu_cudnn.cu) and its half-precision tests run them
// (test/int/nnc/cudnn.tests.c:3504-3678, 4151-4323, 4363-4735).  For bf16 / fp16 tensors the command runs in its functional form
// (STAGE_F32).
inline uint16_t f32_to_16(const float v, const int kind)
{
	uint32_t u;
	memcpy(&u, &v, 4);
	if (kind == 1)
		return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16); // bf16, round to nearest even
	// fp16, round to nearest even (finite range; the fill values this is used for are small)
	const uint32_t sign = (u >> 16) & 0x8000u;
	const int32_t e = (int32_t)((u >> 23) & 0xff) - 127 + 15;
	uint32_t m = u & 0x7fffffu;
	if (e >= 31)
		return (uint16_t)(sign | 0x7c00u);
	if (e <= 0)
	{
		if (e < -10)
			return (uint16_t)sign;
		m |= 0x800000u;
		const int shift = 14 - e;
		const uint32_t r = m >> shift, rem = m & ((1u << shift) - 1), half = 1u << (shift - 1);
		return (uint16_t)(sign | (r + (rem > half || (rem == half && (r & 1)))));
	}
	const uint32_t r = (uint32_t)(e << 10) | (m >> 13), rem = m & 0x1fffu;
	return (uint16_t)(sign | (r + (rem > 0x1000u || (rem == 0x1000u && (r & 1)))));
}

template <ccv_nnc_cmd_exec_f F32, staged_inner_f WS = no_workspace>
int exec_via_f32(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return staged(STAGE_F32, 0, F32, WS, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// SGD: fp32 parameters / momenta with gradients of any type run natively (the mixed-precision form); 16-bit PARAMETERS
// (sgd/gpu/ccv_nnc_sgd_gpu_ref.cu:75-77, test/int/nnc/sgd.tests.c:73-137) go through the functional form
int exec_sgd_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size >= 2 && inputs[1] && kind_of(inputs[1]) > 0)
		return exec_via_f32<exec_sgd_forw>(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	return exec_sgd_forw(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// ================================================================================================ palettized (CCV_QX) operands
// lib/nnc/cmd/blas/gpu/ccv_nnc_gemm_gpu_cublas.cu:291-334, convolution/gpu/ccv_nnc_conv_gpu_cudnn.cu:79,328,
// convolution/gpu/ccv_nnc_conv_transpose_gpu_cudnn.cu:72,127: a weight operand may be a palettized tensor (STAGE_QX).
bool any_qx(ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size)
{
	for (int i = 0; i < input_size; i++)
		if (is_qx(inputs[i]))
			return true;
	for (int i = 0; i < output_size; i++)
		if (is_qx(outputs[i]))
			return true;
	return false;
}

// The few-row dense layer on a palettized weight, without decoding it: c[M, N] = a[M, K] w[N, K]^T (+ bias), a / c fp16, w with fp16
// palettes and no batch axis, M = every row of a up to PALETTIZED_GEMM_M_MAX.  Returns false when the call is not of that form.
bool gemm_fused_qx_plan(const ccv_nnc_cmd_t& cmd, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, int& M, int& N, int& K)
{
	if (input_size < 2 || output_size < 1 || !inputs[0] || !is_qx(inputs[1]) || !outputs[0] || is_qx(inputs[0]) || CCV_IS_TENSOR_VIEW(inputs[1]))
		return false;
	const ccv_nnc_tensor_t* const bias_t = input_size > 2 ? inputs[2] : 0;
	if (CCV_GET_DATA_TYPE(inputs[0]->info.datatype) != CCV_16F || CCV_GET_DATA_TYPE(outputs[0]->info.datatype) != CCV_16F || qx_palette(inputs[1]) != CCV_16F ||
		!palettize_params_ok(qx_bits(inputs[1]), inputs[1]->info.reserved))
		return false;
	const int* const ta = cmd.info.blas.transpose_a;
	const int* const tb = cmd.info.blas.transpose_b;
	const TV a = view_of(inputs[0]), w = view_of(inputs[1]), c = view_of(outputs[0]);
	if (w.nd != 2 || tb[0] == tb[1] || ta[0] != ta[1] || a.nd < 1 || a.nd > 3 || c.nd != a.nd || !a.contiguous || !c.contiguous)
		return false;
	K = w.dim[1], N = w.dim[0];
	if (a.dim[a.nd - 1] != K || c.dim[c.nd - 1] != N)
		return false;
	const size_t rows = a.count / K;
	if (rows < 1 || rows > (size_t)PALETTIZED_GEMM_M_MAX || c.count / N != rows)
		return false;
	if (bias_t)
	{
		const TV b = view_of(bias_t);
		if (b.nd != 1 || b.dim[0] != N || is_qx(bias_t) || (CCV_GET_DATA_TYPE(bias_t->info.datatype) != CCV_16F && CCV_GET_DATA_TYPE(bias_t->info.datatype) != CCV_32F))
			return false;
	}
	M = (int)rows;
	return true;
}

int exec_gemm_forw_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	int M, N, K;
	if (gemm_fused_qx_plan(cmd, inputs, input_size, outputs, output_size, M, N, K))
	{
		const ccv_nnc_tensor_t* const bias_t = input_size > 2 ? inputs[2] : 0;
		const bool b32 = bias_t && is_f32(bias_t);
		RC(gemm_palettized_f16(stream_of(stream_context), M, N, K, inputs[0]->data.u8, K, inputs[1]->data.u8, qx_bits(inputs[1]), inputs[1]->info.reserved, outputs[0]->data.u8, N,
			b32 ? bias_t->data.f32 : 0, bias_t && !b32 ? (const void*)bias_t->data.u8 : 0));
		return CCV_NNC_EXEC_SUCCESS;
	}
	return staged(STAGE_QX, 0x3, exec_gemm_nd4<exec_gemm_forw>, gemm_forw_workspace, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

int exec_gemm_back_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	// inputs (g, a, w): a is palettized only for dw, w only for h
	const unsigned mask = (output_size > 1 && outputs[1] ? 0x2u : 0u) | (output_size > 0 && outputs[0] ? 0x4u : 0u);
	return staged(STAGE_QX, mask, exec_gemm_nd4<exec_gemm_back>, gemm_back_workspace, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// convolutions (EXEC: the NHWC command, WS: its workspace function): palettized filters, inputs[1] of the forwards and inputs[2] of the
// backwards when the data gradient (outputs[0]) is asked for, decoded around the NCHW staging
template <ccv_nnc_cmd_exec_f EXEC, staged_inner_f WS, int BACKWARD>
int exec_conv_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const unsigned mask = BACKWARD ? (output_size > 0 && outputs[0] ? 0x4u : 0u) : 0x2u;
	return staged(STAGE_QX, mask, exec_nchw<EXEC, WS, BACKWARD>, nchw_workspace<WS>, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// util/gpu/ccv_nnc_util_gpu_ref.cu:22-24: a palettized tensor moves as its bytes; both sides carry the same datatype word and block size
int exec_data_transfer_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (!any_qx(inputs, input_size, outputs, output_size))
		return exec_data_transfer(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	const int n = input_size < output_size ? input_size : output_size;
	for (int i = 0; i < n; i++)
		if (inputs[i] && outputs[i] && (is_qx(inputs[i]) || is_qx(outputs[i])))
		{
			const ccv_nnc_tensor_t* const a = inputs[i];
			const ccv_nnc_tensor_t* const b = outputs[i];
			if (a->info.datatype != b->info.datatype || a->info.reserved != b->info.reserved || CCV_IS_TENSOR_VIEW(a) || CCV_IS_TENSOR_VIEW(b) || view_of(a).count != view_of(b).count ||
				!palettize_params_ok(qx_bits(a), a->info.reserved))
				return CCV_NNC_EXEC_INVALID;
		}
	cudaStream_t s = stream_of(stream_context);
	for (int i = 0; i < n; i++)
	{
		if (!inputs[i] || !outputs[i] || inputs[i] == outputs[i])
			continue;
		if (!is_qx(inputs[i]))
		{
			RC(copy_tensor(s, inputs[i], outputs[i]));
			continue;
		}
		const size_t bytes = palettize_data_bytes(view_of(inputs[i]).count, qx_bits(inputs[i]), inputs[i]->info.reserved, dtype_size(qx_palette(inputs[i])));
		const cudaError_t e = cudaMemcpyAsync(outputs[i]->data.u8, inputs[i]->data.u8, bytes, cudaMemcpyDefault, s);
		if (e != cudaSuccess)
		{
			set_last_error("data transfer (palettized)", e);
			return CCV_NNC_EXEC_INVALID;
		}
	}
	if (!stream_context && cudaStreamSynchronize(s) != cudaSuccess)
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// registry->autotune of the contraction commands (lib/nnc/ccv_nnc.h:323; called by ccv_nnc_cmd_autotune, ccv_nnc_cmd.c:519-531, on
// scratch copies of the operands): every algorithm of this backend that accepts the shapes is timed on the device (CUDA
// events on the caller's stream, best of 3 after a warm-up) and the index of the fastest one is returned.  The generic
// fallback of the reference times the asynchronous *enqueue* with a host clock (ccv_nnc_cmd.c:549-555), which says nothing
// about a GPU kernel -- hence a real autotune function.  The attention commands use it too: algorithm 0 refuses some calls algorithm 1
// runs (a 16-bit D = 160 forward that asks for the log-sum-exp), so the tuned command is the one that runs.
template <ccv_nnc_cmd_exec_f EXEC, int COUNT>
int autotune_algorithms(const ccv_nnc_cmd_t cmd, const size_t max_workspace_size, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	cudaStream_t s = stream_of(stream_context);
	cudaEvent_t e0, e1;
	if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess)
		return 0;
	int best = 0;
	float best_ms = -1.f;
	for (int k = 0; k < COUNT; k++) // the contractions: TF32, 3XTF32, FFMA; attention: COMPOSED, FLASH
	{
		ccv_nnc_cmd_t c = cmd;
		c.algorithm = k;
		if (EXEC(c, hint, flags, inputs, input_size, outputs, output_size, stream_context) != CCV_NNC_EXEC_SUCCESS) // warm-up + applicability
			continue;
		float ms = -1.f;
		for (int rep = 0; rep < 3; rep++)
		{
			cudaEventRecord(e0, s);
			EXEC(c, hint, flags, inputs, input_size, outputs, output_size, stream_context);
			cudaEventRecord(e1, s);
			float t = 0.f;
			if (cudaEventSynchronize(e1) != cudaSuccess || cudaEventElapsedTime(&t, e0, e1) != cudaSuccess)
				continue;
			if (ms < 0.f || t < ms)
				ms = t;
		}
		if (ms >= 0.f && (best_ms < 0.f || ms < best_ms))
			best_ms = ms, best = k;
	}
	cudaEventDestroy(e0);
	cudaEventDestroy(e1);
	return best;
}

} // namespace

namespace sm100 {
int backend_gemm_nt_bias(void* stream_context, int kind, int M, int N, int K, const void* a, const void* w, void* c, const void* bias, int bias_is_f32)
{
	ccv_nnc_stream_context_t* const ctx = (ccv_nnc_stream_context_t*)stream_context;
	const Scratch scratch = scratch_of(ctx);
	cudaStream_t s = stream_of(ctx);
	return gemm_dispatch(s, scratch, kind, CCV_NNC_SM100_ALGO_3XTF32, M, N, K, a, K, 1, w, 1, K, c, N, 1, bias && bias_is_f32 ? (const float*)bias : 0, bias && !bias_is_f32 ? bias : 0, 0);
}
bool backend_qx_ok(const void* const tensor, const int dense)
{
	return qx_ok((const ccv_nnc_tensor_t*)tensor, dense);
}
int backend_qx_decode(void* const stream_context, const void* const tensor, void* const out)
{
	return qx_decode(stream_of((ccv_nnc_stream_context_t*)stream_context), (const ccv_nnc_tensor_t*)tensor, out);
}
// GEMM_BACKWARD(NO_TRANSPOSE, TRANSPOSE(0, 1)) as ccv_nnc_cmd() makes it: algorithm -1, no blas flags
static ccv_nnc_cmd_t gemm_back_nt_cmd()
{
	ccv_nnc_cmd_t cmd;
	memset(&cmd, 0, sizeof(cmd));
	cmd.cmd = CCV_NNC_GEMM_BACKWARD;
	cmd.backend = CCV_NNC_BACKEND_GPU_SM100;
	cmd.algorithm = -1;
	cmd.info.blas.a[0] = 1, cmd.info.blas.a[1] = 1;
	cmd.info.blas.transpose_b[0] = 0, cmd.info.blas.transpose_b[1] = 1;
	return cmd;
}
size_t backend_gemm_back_workspace(void* const* const inputs, void* const* const outputs)
{
	ccv_nnc_hint_t hint;
	memset(&hint, 0, sizeof(hint));
	return gemm_back_workspace(gemm_back_nt_cmd(), hint, (ccv_nnc_tensor_t* const*)inputs, 3, (ccv_nnc_tensor_t* const*)outputs, 3);
}
int backend_gemm_back(void* const stream_context, const int flags, void* const* const inputs, void* const* const outputs)
{
	ccv_nnc_hint_t hint;
	memset(&hint, 0, sizeof(hint));
	return exec_gemm_back_any(gemm_back_nt_cmd(), hint, flags, (ccv_nnc_tensor_t* const*)inputs, 3, (ccv_nnc_tensor_t* const*)outputs, 3, (ccv_nnc_stream_context_t*)stream_context);
}
} // namespace sm100

// implemented in sm100_backend_ext.cu (attention, layer / rms norm, upsample, allreduce)
extern "C" {
int ccv_nnc_sm100_exec_sdpa_forw(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_sdpa_back(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_lnorm_forw(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_lnorm_back(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_rmsnorm_forw(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_rmsnorm_back(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_upsample_forw(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_upsample_back(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_gnorm_forw(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_gnorm_back(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
int ccv_nnc_sm100_exec_allreduce(const ccv_nnc_cmd_t, const ccv_nnc_hint_t, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_tensor_t* const*, const int, ccv_nnc_stream_context_t*);
}

// ================================================================================================ fused pairs
// Used by the flat graph runner's peephole pass (ccv_nnc_sm100_graph_fuse): each stands for two adjacent reference
// commands and produces what the pair would have produced.
extern "C" int ccv_nnc_sm100_fused_bn_relu_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_forw(1, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// BATCH_NORM_FORWARD with the statistics tensor of its producing convolution as a 6th input (no ReLU)
extern "C" int ccv_nnc_sm100_fused_bn_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_forw(0, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// BATCH_NORM_FORWARD(train) ; EWSUM(bn output, s -> y) ; RELU_FORWARD in place on y, as one pass y = relu(bn(x) + s) that never
// writes the batch norm's own output.  inputs: the batch norm's five (and the statistics tensor of a linked convolution); outputs: y,
// the batch norm's four statistics outputs, then s (read only).
extern "C" int ccv_nnc_sm100_fused_bn_add_relu_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (output_size != 6 || !outputs[5])
		return CCV_NNC_EXEC_INVALID;
	return bnorm_forw(0, cmd, hint, flags, inputs, input_size, outputs, 5, stream_context, outputs[5]);
}

// AVERAGE_POOL_BACKWARD ; EWSUM ; RELU_BACKWARD at the shortcut of a strided residual block (exec_avgpool_add_relu_back)
extern "C" int ccv_nnc_sm100_fused_avgpool_add_relu_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return exec_avgpool_add_relu_back(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// BATCH_NORM_BACKWARD with the bias gradient of the producing convolution as a 4th output (no ReLU in front)
extern "C" int ccv_nnc_sm100_fused_bn_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_back(0, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

extern "C" int ccv_nnc_sm100_fused_relu_bn_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return bnorm_back(1, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// inputs (a, b) -> y = relu(a + b)
extern "C" int ccv_nnc_sm100_fused_add_relu_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 2 || output_size != 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), b = view_of(inputs[1]), y = view_of(outputs[0]);
	const int kind = kind_of(outputs[0]);
	if (!a.contiguous || !b.contiguous || !y.contiguous || a.count != y.count || b.count != y.count || kind < 0 || kind_of(inputs[0]) != kind || kind_of(inputs[1]) != kind)
		return CCV_NNC_EXEC_INVALID;
	if (kind != 0)
		RC(ew_add_relu_fwd_16(stream_of(stream_context), kind, inputs[0]->data.u8, inputs[1]->data.u8, outputs[0]->data.u8, y.count));
	else
		RC(ew_add_relu_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[1]->data.f32, outputs[0]->data.f32, y.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// inputs (a, b, y) -> out = y > 0 ? a + b : 0   (EWSUM of two branch gradients followed by RELU_BACKWARD)
extern "C" int ccv_nnc_sm100_fused_add_relu_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 3 || output_size != 1 || !inputs[0] || !inputs[1] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const TV a = view_of(inputs[0]), b = view_of(inputs[1]), y = view_of(inputs[2]), o = view_of(outputs[0]);
	const int kind = kind_of(outputs[0]);
	if (!a.contiguous || !b.contiguous || !y.contiguous || !o.contiguous || a.count != o.count || b.count != o.count || y.count != o.count || kind < 0 || kind_of(inputs[0]) != kind || kind_of(inputs[1]) != kind || kind_of(inputs[2]) != kind)
		return CCV_NNC_EXEC_INVALID;
	if (kind != 0)
		RC(ew_add_relu_bwd_16(stream_of(stream_context), kind, inputs[0]->data.u8, inputs[1]->data.u8, inputs[2]->data.u8, outputs[0]->data.u8, o.count));
	else
		RC(ew_add_relu_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[1]->data.f32, inputs[2]->data.f32, outputs[0]->data.f32, o.count));
	return CCV_NNC_EXEC_SUCCESS;
}

// CONVOLUTION_FORWARD whose output feeds a training BATCH_NORM_FORWARD: outputs[1] is the statistics tensor
// ([4 planes x rows, K] fp32: count, shift, shifted sum, shifted sum of squares per (CTA, warp quarter) row) shared with the
// batch-norm node; the tensor-core epilogue folds its output into it and the number of rows in use lands in the `sig` field
// (0 when the launch took a path without that epilogue).
extern "C" int ccv_nnc_sm100_fused_conv_stats_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (output_size != 2 || !outputs[1])
		return CCV_NNC_EXEC_INVALID;
	ccv_nnc_tensor_t* const stats_t = outputs[1];
	int rows = 0;
	const int max_rows = stats_t->info.dim[0] / 4;
	if (outputs[0] && stats_t->info.dim[1] == cmd.info.convolution.count)
		conv_stats_request(stats_t->data.f32, max_rows, &rows);
	const int rc = exec_nchw<conv_forw_nhwc, conv_forw_workspace, 0>(cmd, hint, flags, inputs, input_size, outputs, 1, stream_context);
	conv_stats_request(0, 0, 0); // never leave a request pending for an unrelated launch
	stats_t->sig = rc == CCV_NNC_EXEC_SUCCESS ? (uint64_t)rows : 0;
	return rc;
}

// T SGD_FORWARD commands with identical parameters as one command: inputs (g, a, m) x T -> outputs (b, n) x T
extern "C" int ccv_nnc_sm100_fused_sgd_multi(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return exec_sgd_multi(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

// ================================================================================================ registration
namespace sm100 {
int exec_via_f32_rt(ccv_nnc_cmd_exec_f f32, const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return staged(STAGE_F32, 0, f32, no_workspace, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}
}

REGISTER_SM100(CCV_NNC_GEMM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_gemm_forw_any); registry->autotune = autotune_algorithms<exec_gemm_forw_any, CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_GEMM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_gemm_back_any); registry->autotune = autotune_algorithms<exec_gemm_back_any, CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_CONVOLUTION_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_conv_any<conv_forw_nhwc, conv_forw_workspace, 0>); registry->autotune = autotune_algorithms<exec_conv_any<conv_forw_nhwc, conv_forw_workspace, 0> , CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_CONVOLUTION_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_conv_any<conv_back_nhwc, conv_back_workspace, 1>); registry->autotune = autotune_algorithms<exec_conv_any<conv_back_nhwc, conv_back_workspace, 1> , CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_conv_any<conv_transpose_forw_nhwc, conv_transpose_forw_workspace, 0>); registry->autotune = autotune_algorithms<exec_conv_any<conv_transpose_forw_nhwc, conv_transpose_forw_workspace, 0> , CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_CONVOLUTION_TRANSPOSE_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_ALGO_COUNT, exec_conv_any<conv_transpose_back_nhwc, conv_transpose_back_workspace, 1>); registry->autotune = autotune_algorithms<exec_conv_any<conv_transpose_back_nhwc, conv_transpose_back_workspace, 1> , CCV_NNC_SM100_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_QX, CCV_NNC_SM100_SDPA_ALGO_COUNT, ccv_nnc_sm100_exec_sdpa_forw); registry->autotune = autotune_algorithms<ccv_nnc_sm100_exec_sdpa_forw, CCV_NNC_SM100_SDPA_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, CCV_NNC_SM100_SDPA_ALGO_COUNT, ccv_nnc_sm100_exec_sdpa_back); registry->autotune = autotune_algorithms<ccv_nnc_sm100_exec_sdpa_back, CCV_NNC_SM100_SDPA_ALGO_COUNT>; }
REGISTER_SM100(CCV_NNC_SOFTMAX_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_softmax_forw>); }
REGISTER_SM100(CCV_NNC_SOFTMAX_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_softmax_back>); }
REGISTER_SM100(CCV_NNC_BATCH_NORM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_bnorm_forw); }
REGISTER_SM100(CCV_NNC_BATCH_NORM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_bnorm_back); }
REGISTER_SM100(CCV_NNC_LAYER_NORM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_lnorm_forw); }
REGISTER_SM100(CCV_NNC_LAYER_NORM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_lnorm_back); }
REGISTER_SM100(CCV_NNC_GROUP_NORM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_gnorm_forw); }
REGISTER_SM100(CCV_NNC_GROUP_NORM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_gnorm_back); }
REGISTER_SM100(CCV_NNC_RMSNORM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_rmsnorm_forw); }
REGISTER_SM100(CCV_NNC_RMSNORM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_rmsnorm_back); }
REGISTER_SM100(CCV_NNC_EWSUM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_ewsum_forw); }
REGISTER_SM100(CCV_NNC_EWSUM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_ewsum_back); }
REGISTER_SM100(CCV_NNC_EWPROD_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_ewprod_forw); }
REGISTER_SM100(CCV_NNC_EWPROD_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_ewprod_back); }
REGISTER_SM100(CCV_NNC_ADD_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_add_forw>); }
REGISTER_SM100(CCV_NNC_ADD_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_add_back>); }
REGISTER_SM100(CCV_NNC_MUL_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_mul_forw>); }
REGISTER_SM100(CCV_NNC_MUL_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_mul_back, mul_back_workspace>); }
REGISTER_SM100(CCV_NNC_SCALAR_MUL_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_scalar_mul_forw>); }
REGISTER_SM100(CCV_NNC_SCALAR_MUL_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<exec_scalar_mul_back>); }
REGISTER_SM100(CCV_NNC_RELU_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_relu_forw); }
REGISTER_SM100(CCV_NNC_RELU_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_relu_back); }
REGISTER_SM100(CCV_NNC_MAX_POOL_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_nchw<exec_pool_forw<1>, no_workspace, 0>); }
REGISTER_SM100(CCV_NNC_MAX_POOL_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_nchw<exec_pool_back<1>, no_workspace, 0>); }
REGISTER_SM100(CCV_NNC_AVERAGE_POOL_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_nchw<exec_pool_forw<0>, no_workspace, 0>); }
REGISTER_SM100(CCV_NNC_AVERAGE_POOL_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_nchw<exec_pool_back<0>, no_workspace, 0>); }
REGISTER_SM100(CCV_NNC_UPSAMPLE_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<ccv_nnc_sm100_exec_upsample_forw>); }
REGISTER_SM100(CCV_NNC_UPSAMPLE_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_NCHW, CCV_32F | CCV_16F | CCV_16BF, 1, exec_via_f32<ccv_nnc_sm100_exec_upsample_back>); }
REGISTER_SM100(CCV_NNC_SET_FORWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_set_forw); }
REGISTER_SM100(CCV_NNC_SET_BACKWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_set_forw); }
REGISTER_SM100(CCV_NNC_DATA_TRANSFER_FORWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF | CCV_32S | CCV_8U | CCV_QX, 1, exec_data_transfer_any); registry->tensor_memory = CCV_TENSOR_CPU_MEMORY | CCV_TENSOR_GPU_MEMORY; }
REGISTER_SM100(CCV_NNC_DATA_TRANSFER_BACKWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF | CCV_32S | CCV_8U | CCV_QX, 1, exec_data_transfer_any); registry->tensor_memory = CCV_TENSOR_CPU_MEMORY | CCV_TENSOR_GPU_MEMORY; }
REGISTER_SM100(CCV_NNC_FORMAT_TRANSFORM_FORWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_32S | CCV_16F | CCV_16BF | CCV_8U, 1, exec_format_transform); }
REGISTER_SM100(CCV_NNC_FORMAT_TRANSFORM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_32S | CCV_16F | CCV_16BF | CCV_8U, 1, exec_format_transform); }
REGISTER_SM100(CCV_NNC_TRANSPOSE_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_transpose); }
REGISTER_SM100(CCV_NNC_TRANSPOSE_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_transpose); }
REGISTER_SM100(CCV_NNC_DATATYPE_CONVERSION_FORWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF, 1, exec_datatype_conversion); }
REGISTER_SM100(CCV_NNC_DATATYPE_CONVERSION_BACKWARD) { fill(registry, ALL_FORMATS, CCV_64F | CCV_32F | CCV_16F | CCV_16BF, 1, exec_datatype_conversion); }
REGISTER_SM100(CCV_NNC_SGD_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_sgd_any); }
REGISTER_SM100(CCV_NNC_SGD_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F, 1, exec_invalid); }
REGISTER_SM100(CCV_NNC_CATEGORICAL_CROSSENTROPY_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_via_f32<exec_cce_forw>); }
REGISTER_SM100(CCV_NNC_CATEGORICAL_CROSSENTROPY_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_via_f32<exec_cce_back>); }
REGISTER_SM100(CCV_NNC_SOFTMAX_CROSSENTROPY_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_via_f32<exec_softmax_cce_forw>); }
REGISTER_SM100(CCV_NNC_SOFTMAX_CROSSENTROPY_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_via_f32<exec_softmax_cce_back>); }
REGISTER_SM100(CCV_NNC_COMM_ALLREDUCE_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_allreduce); }
REGISTER_SM100(CCV_NNC_COMM_ALLREDUCE_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, ccv_nnc_sm100_exec_allreduce); }
