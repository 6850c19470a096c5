// sm100_ext_ops.cu -- the commands a transformer block around SCALED_DOT_PRODUCT_ATTENTION needs on the same backend
// (SURVEY.md 8f-4): GELU, SWISH (forward / backward), INDEX_SELECT (forward / backward), ADAMW.  HBM-bound, grid-stride,
// 16-byte accesses; fp32 and, for the activations, bf16 / fp16 tensors (fp32 arithmetic, one rounding on the way out).
// Semantics (paths relative to /root/reference/lib/nnc/cmd):
//   gelu/ccv_nnc_gelu_cpu_ref.c:13-92      erf form x/2 (1 + erf(x / sqrt 2)) or the tanh approximation (cmd.info.gelu.tanh)
//   swish/ccv_nnc_swish_cpu_ref.c:13-86    x / (1 + exp(-x));  backward g (x (y - y^2) + y), y = sigmoid(x)
//   index/ccv_nnc_index_select_cpu_ref.c:13-137  b[i, :] = a[indices[i], :] (int32 indices; fp32 indices interpolate between
//                                          rows j0 and min(j0 + 1, rows - 1)); backward zeroes h and adds g rows in index order
//   adam/ccv_nnc_adamw_cpu_ref.c:13-250    decoupled weight decay: b = a - rate decay a - (m' rate / (1 - beta1^t)) / (sqrt(v' / (1 - beta2^t)) + eps)
//                                          (amsgrad: running maximum of the bias-corrected second moment)
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <cuda_runtime.h>
#include <math.h>

// functional form of an fp32-only command on bf16 / fp16 tensors (sm100_backend.cu: widen into the workspace, run `f32`, round back once)
namespace sm100 {
int exec_via_f32_rt(ccv_nnc_cmd_exec_f f32, const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);
}
using namespace sm100;

namespace {

// ------------------------------------------------------------------------------------------------ activations
// OP 0: gelu (erf), 1: gelu (tanh), 2: swish
template <int OP>
__device__ __forceinline__ float act_fwd(const float x)
{
	if (OP == 0)
		return x * 0.5f * (1.f + erff(x * 0.70710678118654752440f));
	if (OP == 1)
		return 0.5f * x * (1.f + tanhf(0.797884560802865355f * (x + 0.044715f * x * x * x)));
	return x / (1.f + expf(-x));
}
template <int OP>
__device__ __forceinline__ float act_bwd(const float g, const float x)
{
	if (OP == 0)
	{
		const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752440f));
		const float pdf = expf(-0.5f * x * x) * 0.797884560802865355f;
		return g * (cdf + x * pdf); // exactly gelu_cpu_ref.c:83-88, whose `pdf` carries the constant sqrt(2 / pi) (twice the normal density): parity is with CPU_REF
	}
	if (OP == 1)
	{
		const float x_sq = x * x;
		const float inner = 0.797884560802865355f * (x + 0.044715f * x_sq * x);
		const float t = tanhf(inner);
		const float left = 0.5f * x, right = 1.f + t;
		return g * (0.5f * right + left * (1.f - t * t) * 0.797884560802865355f * (1.f + 3.f * 0.044715f * x_sq));
	}
	const float y = 1.f / (1.f + expf(-x));
	return g * (x * (y - y * y) + y);
}
template <typename T, int OP, int BWD>
__global__ void __launch_bounds__(256) act_kernel(const T* __restrict__ g, const T* __restrict__ a, T* __restrict__ out, const size_t n, const int vec)
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
			o[k] = BWD ? act_bwd<OP>(y[k], x[k]) : act_fwd<OP>(x[k]);
		stv(out + i * W, o);
	}
	for (size_t i = nw * W + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
		stf(out + i, BWD ? act_bwd<OP>(ldf(g + i), ldf(a + i)) : act_fwd<OP>(ldf(a + i)));
}
template <typename T, int OP>
int run_act(cudaStream_t s, const void* g, const void* a, void* out, size_t n)
{
	if (n == 0)
		return 0;
	const int vec = aligned_v16((const T*)a) && aligned_v16((const T*)out) && (!g || aligned_v16((const T*)g));
	const int grid = grid_for(vec ? n / Vec16<T>::W + 1 : n, 256, 8);
	if (g)
		act_kernel<T, OP, 1><<<grid, 256, 0, s>>>((const T*)g, (const T*)a, (T*)out, n, vec);
	else
		act_kernel<T, OP, 0><<<grid, 256, 0, s>>>((const T*)0, (const T*)a, (T*)out, n, vec);
	return launched("activation");
}
template <int OP>
int run_act_kind(cudaStream_t s, int kind, const void* g, const void* a, void* out, size_t n)
{
	if (kind == 0)
		return run_act<float, OP>(s, g, a, out, n);
	if (kind == 1)
		return run_act<__nv_bfloat16, OP>(s, g, a, out, n);
	return run_act<__half, OP>(s, g, a, out, n);
}
// forward: inputs (a) -> outputs (b); backward: inputs (g, a, [b]) -> outputs (h)
template <int IS_SWISH, int BWD>
int exec_act(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < (BWD ? 2 : 1) || output_size < 1 || !inputs[0] || (BWD && !inputs[1]) || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const a = BWD ? inputs[1] : inputs[0];
	const ccv_nnc_tensor_t* const g = BWD ? inputs[0] : 0;
	const int kind = kind_of(a);
	if (kind < 0 || kind_of(outputs[0]) != kind || (g && kind_of(g) != kind) || !CCV_IS_TENSOR_CONTIGUOUS(a) || !CCV_IS_TENSOR_CONTIGUOUS(outputs[0]) || (g && !CCV_IS_TENSOR_CONTIGUOUS(g)))
		return CCV_NNC_EXEC_INVALID;
	if (!same_dims(a, outputs[0]) || (g && !same_dims(a, g)))
		return CCV_NNC_EXEC_INVALID;
	const size_t n = count_of(a);
	cudaStream_t s = stream_of(stream_context);
	int rc;
	if (IS_SWISH)
		rc = run_act_kind<2>(s, kind, g ? g->data.u8 : 0, a->data.u8, outputs[0]->data.u8, n);
	else if (cmd.info.gelu.tanh)
		rc = run_act_kind<1>(s, kind, g ? g->data.u8 : 0, a->data.u8, outputs[0]->data.u8, n);
	else
		rc = run_act_kind<0>(s, kind, g ? g->data.u8 : 0, a->data.u8, outputs[0]->data.u8, n);
	return rc ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ index select
// one block per output row; threads stride over the columns (element size 2 or 4 bytes: a plain row copy)
template <typename U>
__global__ void index_select_kernel(const U* __restrict__ a, const int* __restrict__ indices, U* __restrict__ b, const int a_rows, const int cols, const long long a_inc, const long long b_inc)
{
	const int i = blockIdx.x;
	const int idx = indices[i];
	if (idx < 0 || idx >= a_rows)
		return; // the reference asserts; leave the row untouched
	const U* const ap = a + (long long)idx * a_inc;
	U* const bp = b + (long long)i * b_inc;
	for (int j = threadIdx.x; j < cols; j += blockDim.x)
		bp[j] = ap[j];
}
// fp32 indices: linear interpolation between rows j0 and min(j0 + 1, rows - 1) (index_select_cpu_ref.c:47-63)
__global__ void index_select_lerp_kernel(const float* __restrict__ a, const float* __restrict__ indices, float* __restrict__ b, const int a_rows, const int cols, const long long a_inc, const long long b_inc)
{
	const int i = blockIdx.x;
	const float f = indices[i];
	const int j0 = (int)f;
	if (j0 < 0 || j0 >= a_rows)
		return;
	const int j1 = min(j0 + 1, a_rows - 1);
	const float w1 = __fsub_rn(f, (float)j0), w0 = __fsub_rn(1.f, w1);
	const float* const ap0 = a + (long long)j0 * a_inc;
	const float* const ap1 = a + (long long)j1 * a_inc;
	float* const bp = b + (long long)i * b_inc;
	for (int j = threadIdx.x; j < cols; j += blockDim.x)
		bp[j] = __fadd_rn(__fmul_rn(ap0[j], w0), __fmul_rn(ap1[j], w1)); // the reference's rounding: no FMA
}
// backward: h[r, :] = sum over i with indices[i] == r of g[i, :], added in increasing i (the reference's order: bit-reproducible,
// no atomics).  One block per row of h; every block walks the index list (broadcast loads).
template <typename T>
__global__ void index_select_back_kernel(const T* __restrict__ g, const int* __restrict__ indices, T* __restrict__ h, const int g_rows, const int cols, const long long g_inc, const long long h_inc)
{
	const int r = blockIdx.x;
	for (int j0 = threadIdx.x; j0 < cols; j0 += blockDim.x)
	{
		float acc = 0.f;
		for (int i = 0; i < g_rows; i++)
			if (indices[i] == r)
				acc += ldf(g + (long long)i * g_inc + j0);
		stf(h + (long long)r * h_inc + j0, acc);
	}
}
bool rows_cols(const ccv_nnc_tensor_t* const t, int& rows, int& cols, long long& inc)
{
	int nd = 0;
	while (nd < CCV_NNC_MAX_DIM_ALLOC && t->info.dim[nd] > 0)
		nd++;
	if (nd < 1 || nd > 2)
		return false;
	rows = t->info.dim[0], cols = nd < 2 ? 1 : t->info.dim[1];
	inc = CCV_IS_TENSOR_VIEW(t) ? (nd < 2 ? 1 : ((const ccv_nnc_tensor_view_t*)t)->stride[0]) : cols;
	if (CCV_IS_TENSOR_VIEW(t) && nd == 2 && ((const ccv_nnc_tensor_view_t*)t)->stride[1] != 1)
		return false;
	return true;
}
// inputs (a, indices) -> outputs (b)
int exec_index_select_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size != 2 || output_size != 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int a_rows, a_cols, b_rows, b_cols;
	long long a_inc, b_inc;
	if (!rows_cols(inputs[0], a_rows, a_cols, a_inc) || !rows_cols(outputs[0], b_rows, b_cols, b_inc) || a_cols != b_cols)
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const idx = inputs[1];
	if (idx->info.dim[0] != b_rows || idx->info.dim[1] != 0 || CCV_IS_TENSOR_VIEW(idx) || CCV_GET_DATA_TYPE(inputs[0]->info.datatype) != CCV_GET_DATA_TYPE(outputs[0]->info.datatype))
		return CCV_NNC_EXEC_INVALID;
	if (b_rows == 0 || a_cols == 0)
		return CCV_NNC_EXEC_SUCCESS;
	cudaStream_t s = stream_of(stream_context);
	const int threads = a_cols >= 256 ? 256 : (a_cols >= 64 ? 64 : 32);
	const int dt = CCV_GET_DATA_TYPE(inputs[0]->info.datatype);
	if (CCV_GET_DATA_TYPE(idx->info.datatype) == CCV_32S)
	{
		if (dt == CCV_32F || dt == CCV_32S)
			index_select_kernel<uint32_t><<<b_rows, threads, 0, s>>>((const uint32_t*)inputs[0]->data.u8, idx->data.i32, (uint32_t*)outputs[0]->data.u8, a_rows, a_cols, a_inc, b_inc);
		else if (dt == CCV_16F || dt == CCV_16BF)
			index_select_kernel<uint16_t><<<b_rows, threads, 0, s>>>((const uint16_t*)inputs[0]->data.u8, idx->data.i32, (uint16_t*)outputs[0]->data.u8, a_rows, a_cols, a_inc, b_inc);
		else
			return CCV_NNC_EXEC_INVALID;
	} else if (CCV_GET_DATA_TYPE(idx->info.datatype) == CCV_32F && dt == CCV_32F)
		index_select_lerp_kernel<<<b_rows, threads, 0, s>>>(inputs[0]->data.f32, idx->data.f32, outputs[0]->data.f32, a_rows, a_cols, a_inc, b_inc);
	else
		return CCV_NNC_EXEC_INVALID;
	return launched("index_select") ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}
// inputs (g, a, indices) -> outputs (h, [zeroed gradient of the indices])
int exec_index_select_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 3 || output_size < 1 || output_size > 2 || !inputs[0] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int g_rows, g_cols, h_rows, h_cols;
	long long g_inc, h_inc;
	if (!rows_cols(inputs[0], g_rows, g_cols, g_inc) || !rows_cols(outputs[0], h_rows, h_cols, h_inc) || g_cols != h_cols)
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const idx = inputs[2];
	const int kind = kind_of(inputs[0]);
	if (idx->info.dim[0] != g_rows || idx->info.dim[1] != 0 || CCV_IS_TENSOR_VIEW(idx) || CCV_GET_DATA_TYPE(idx->info.datatype) != CCV_32S || kind < 0 || kind_of(outputs[0]) != kind)
		return CCV_NNC_EXEC_INVALID;
	cudaStream_t s = stream_of(stream_context);
	if (output_size > 1 && outputs[1] && !CCV_IS_TENSOR_VIEW(outputs[1]))
		if (cudaMemsetAsync(outputs[1]->data.u8, 0, count_of(outputs[1]) * (CCV_GET_DATA_TYPE(outputs[1]->info.datatype) == CCV_32F || CCV_GET_DATA_TYPE(outputs[1]->info.datatype) == CCV_32S ? 4 : 2), s) != cudaSuccess)
			return CCV_NNC_EXEC_INVALID;
	if (h_rows == 0 || h_cols == 0)
		return CCV_NNC_EXEC_SUCCESS;
	const int threads = h_cols >= 256 ? 256 : (h_cols >= 64 ? 64 : 32);
	if (kind == 0)
		index_select_back_kernel<float><<<h_rows, threads, 0, s>>>(inputs[0]->data.f32, idx->data.i32, outputs[0]->data.f32, g_rows, g_cols, g_inc, h_inc);
	else if (kind == 1)
		index_select_back_kernel<__nv_bfloat16><<<h_rows, threads, 0, s>>>((const __nv_bfloat16*)inputs[0]->data.u8, idx->data.i32, (__nv_bfloat16*)outputs[0]->data.u8, g_rows, g_cols, g_inc, h_inc);
	else
		index_select_back_kernel<__half><<<h_rows, threads, 0, s>>>((const __half*)inputs[0]->data.u8, idx->data.i32, (__half*)outputs[0]->data.u8, g_rows, g_cols, g_inc, h_inc);
	return launched("index_select_back") ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ AdamW
// inputs (g, a, m, v, [vm]) -> outputs (b, n, u, [um]); g fp32 / bf16 / fp16, everything else fp32; contiguous.  Every product and
// sum is rounded on its own, in CPU_REF's association (adam/ccv_nnc_adam{,w}_cpu_ref.c), so b, n, u and um equal CPU_REF's bit for
// bit; the amsgrad maximum is CPU_REF's ccv_max(vm, v_hat) = vm > v_hat ? vm : v_hat, which keeps a NaN v_hat.  No operand is
// __restrict__: models call the command in place (b = a, n = m, u = v, um = vm).
template <int L2>
__global__ void __launch_bounds__(256) adamw_kernel(const void* g, const int g_kind, const float* a, const float* m, const float* v, const float* vm,
	float* b, float* n, float* u, float* um, const size_t count, const float scale, const float beta1, const float beta2, const float rate_inv_bias_correction1,
	const float inv_bias_correction2, const float rate_decay, const float epsilon)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x)
	{
		const float av = a[i];
		float grad = __fmul_rn(scale, ld_kind(g, i, g_kind));
		if (L2)
			grad = __fadd_rn(grad, __fmul_rn(rate_decay, av)); // ADAM: the decay is an L2 term of the gradient (adam/ccv_nnc_adam_cpu_ref.c:117-118); rate_decay carries `decay` itself
		const float mom = __fadd_rn(__fmul_rn(beta1, m[i]), __fmul_rn(1.f - beta1, grad));
		const float vel = __fadd_rn(__fmul_rn(beta2, v[i]), __fmul_rn(__fmul_rn(1.f - beta2, grad), grad));
		float vel_hat = __fmul_rn(vel, inv_bias_correction2);
		if (vm)
		{
			const float vmax = vm[i];
			vel_hat = vmax > vel_hat ? vmax : vel_hat;
		}
		n[i] = mom, u[i] = vel;
		if (vm)
			um[i] = vel_hat;
		const float q = __fdiv_rn(__fmul_rn(mom, rate_inv_bias_correction1), __fadd_rn(__fsqrt_rn(vel_hat), epsilon));
		b[i] = __fsub_rn(L2 ? av : __fsub_rn(av, __fmul_rn(rate_decay, av)), q);
	}
}
template <int L2>
int exec_adam_f32(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 4 || output_size < 3 || cmd.info.adam.step < 1)
		return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < 4; i++)
		if (!inputs[i] || !CCV_IS_TENSOR_CONTIGUOUS(inputs[i]) || (i > 0 && CCV_GET_DATA_TYPE(inputs[i]->info.datatype) != CCV_32F))
			return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < 3; i++)
		if (!outputs[i] || !CCV_IS_TENSOR_CONTIGUOUS(outputs[i]) || CCV_GET_DATA_TYPE(outputs[i]->info.datatype) != CCV_32F)
			return CCV_NNC_EXEC_INVALID;
	const int g_kind = kind_of(inputs[0]);
	if (g_kind < 0)
		return CCV_NNC_EXEC_INVALID;
	const size_t count = count_of(inputs[1]);
	for (int i = 0; i < 4; i++)
		if (count_of(inputs[i]) != count)
			return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < 3; i++)
		if (count_of(outputs[i]) != count)
			return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const vm = input_size >= 5 ? inputs[4] : 0;
	ccv_nnc_tensor_t* const um = output_size >= 4 ? outputs[3] : 0;
	const bool ams = cmd.info.adam.amsgrad && vm && um;
	if (ams && (CCV_GET_DATA_TYPE(vm->info.datatype) != CCV_32F || CCV_GET_DATA_TYPE(um->info.datatype) != CCV_32F || count_of(vm) != count || count_of(um) != count || !CCV_IS_TENSOR_CONTIGUOUS(vm) || !CCV_IS_TENSOR_CONTIGUOUS(um)))
		return CCV_NNC_EXEC_INVALID;
	if (count == 0)
		return CCV_NNC_EXEC_SUCCESS;
	const float rate = cmd.info.adam.rate, beta1 = cmd.info.adam.beta1, beta2 = cmd.info.adam.beta2;
	const float rate_inv_bias_correction1 = rate / (1 - powf(beta1, cmd.info.adam.step));
	const float inv_bias_correction2 = 1. / (1 - powf(beta2, cmd.info.adam.step)); // the quotient in double, rounded once, as CPU_REF
	adamw_kernel<L2><<<grid_for(count, 256, 8), 256, 0, stream_of(stream_context)>>>(inputs[0]->data.u8, g_kind, inputs[1]->data.f32, inputs[2]->data.f32, inputs[3]->data.f32, ams ? vm->data.f32 : 0,
		outputs[0]->data.f32, outputs[1]->data.f32, outputs[2]->data.f32, ams ? um->data.f32 : 0, count, cmd.info.adam.scale, beta1, beta2, rate_inv_bias_correction1, inv_bias_correction2, L2 ? cmd.info.adam.decay : rate * cmd.info.adam.decay, cmd.info.adam.epsilon);
	return launched("adamw") ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}
// parameters / moments in half precision (adam/gpu/ccv_nnc_adamw_gpu_ref.cu registers CCV_16F; test/int/nnc/adam.tests.c:300-360): functional form
template <int L2>
int exec_adam_any(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size >= 2 && inputs[1] && kind_of(inputs[1]) > 0)
		return exec_via_f32_rt(exec_adam_f32<L2>, cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	return exec_adam_f32<L2>(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
}

} // namespace

REGISTER_SM100(CCV_NNC_GELU_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_act<0, 0>); }
REGISTER_SM100(CCV_NNC_GELU_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_act<0, 1>); }
REGISTER_SM100(CCV_NNC_SWISH_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_act<1, 0>); }
REGISTER_SM100(CCV_NNC_SWISH_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_act<1, 1>); }
REGISTER_SM100(CCV_NNC_INDEX_SELECT_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_index_select_forw); }
REGISTER_SM100(CCV_NNC_INDEX_SELECT_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_index_select_back); }
REGISTER_SM100(CCV_NNC_ADAMW_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_adam_any<0>); }
REGISTER_SM100(CCV_NNC_ADAM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_adam_any<1>); }
// an optimizer has no backward (adam/ccv_nnc_adamw_cpu_ref.c: _ccv_nnc_adamw_back)
REGISTER_SM100(CCV_NNC_ADAM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_invalid); }
REGISTER_SM100(CCV_NNC_ADAMW_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_invalid); }
