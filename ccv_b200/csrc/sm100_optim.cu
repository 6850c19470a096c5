// sm100_optim.cu -- the LAMB and RMSPROP optimizers (forward; their backward is INVALID, as the reference's).  Semantics are CPU_REF's
// (paths relative to lib/nnc/cmd of the reference):
//   lamb/ccv_nnc_lamb_cpu_ref.c        grad = scale g;  n = beta1 m + (1 - beta1) grad;  u = beta2 v + (1 - beta2) grad grad;
//                                      update = (n ibc1) / (sqrt(u ibc2) + epsilon) + a decay;  b = a - (rate trust) update, where
//                                      trust = |a| / |update| over the whole tensor (sums of float squares kept in double), 1 when
//                                      either norm is not > 0
//   rmsprop/ccv_nnc_rmsprop_cpu_ref.c  grad = scale g + decay a;  u = alpha v + (1 - alpha) grad grad;  n = momentum m + grad / (sqrt(u)
//                                      + epsilon);  b = a - rate n
// Inputs (g, a, m, v) -> outputs (b, n, u); b = a, n = m, u = v (in place, or any subset of it) are allowed.  g is fp32, bf16 or fp16;
// a, m, v, b, n, u share one type, fp32, bf16 or fp16.  16-bit values are widened on load, the arithmetic is fp32 with every product
// and sum rounded on its own in CPU_REF's association (no FMA contraction), and each output is rounded once on store.  Operands are
// contiguous; counts are 64-bit.
//
// Both optimizers run from one table of tensors (OptimTable, in the kernel parameters, <= OPTIM_MULTI_MAX tensors per launch): a single
// command is a table of one, a fused graph run (ccv_nnc_sm100_graph_fuse) a longer one.  A CTA owns one OPTIM_CHUNK-element chunk of
// one tensor, with 4-element vectors when the tensor's count and every pointer allow it, single elements otherwise.
//   RMSPROP: one streaming launch per table.
//   LAMB:    three launches per table, and no workspace the size of a tensor:
//            1. norms: each CTA computes update from (g, a, m, v) and writes its chunk's (sum a^2, sum update^2) as two doubles to a
//               small workspace.  It writes no output, so every in-place or partial-alias form is safe.
//            2. trust: one CTA per tensor adds that tensor's partials in a fixed order and writes r = rate * trust (float).
//            3. apply: each CTA recomputes n, u and update with the same device function (so the update behind the norm is, bit for
//               bit, the update applied) and writes b = a - r update, n and u.
//            Every sum is a fixed tree (per thread in element order, warp butterfly, warps in order, partials per thread then the same
//            tree): the same inputs give the same bits on every run.  Traffic: pass 1 reads g, a, m, v; pass 3 reads them again and
//            writes b, n, u (44 B per element with fp32 state and gradient).
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <vector>

using namespace sm100;

namespace {

constexpr int OPTIM_MULTI_MAX = 32;
constexpr int OPTIM_THREADS = 256;
constexpr unsigned OPTIM_CHUNK = 4096; // elements per CTA: ResNet-50's largest parameter (2 359 296) is 576 chunks

struct OptimTable {
	const void* g[OPTIM_MULTI_MAX];
	const void* a[OPTIM_MULTI_MAX];
	const void* m[OPTIM_MULTI_MAX];
	const void* v[OPTIM_MULTI_MAX];
	void* b[OPTIM_MULTI_MAX];
	void* n[OPTIM_MULTI_MAX];
	void* u[OPTIM_MULTI_MAX];
	unsigned long long count[OPTIM_MULTI_MAX];
	unsigned block_start[OPTIM_MULTI_MAX + 1];
	unsigned char vec[OPTIM_MULTI_MAX];
	int tensors;
};

struct LambArgs {
	float scale, beta1, one_minus_beta1, beta2, one_minus_beta2, ibc1, ibc2, epsilon, decay, rate;
};
struct RmspropArgs {
	float rate, scale, decay, alpha, one_minus_alpha, momentum, epsilon;
};

// ------------------------------------------------------------------------------------------------ arithmetic (CPU_REF's order)
__device__ __forceinline__ float lamb_update(const LambArgs& p, const float g, const float a, const float m, const float v, float& n, float& u)
{
	const float grad = __fmul_rn(p.scale, g);
	n = __fadd_rn(__fmul_rn(p.beta1, m), __fmul_rn(p.one_minus_beta1, grad));
	u = __fadd_rn(__fmul_rn(p.beta2, v), __fmul_rn(__fmul_rn(p.one_minus_beta2, grad), grad));
	return __fadd_rn(__fdiv_rn(__fmul_rn(n, p.ibc1), __fadd_rn(__fsqrt_rn(__fmul_rn(u, p.ibc2)), p.epsilon)), __fmul_rn(a, p.decay));
}
__device__ __forceinline__ void rmsprop_step(const RmspropArgs& p, const float g, const float a, const float m, const float v, float& b, float& n, float& u)
{
	const float grad = __fadd_rn(__fmul_rn(p.scale, g), __fmul_rn(p.decay, a));
	u = __fadd_rn(__fmul_rn(p.alpha, v), __fmul_rn(__fmul_rn(p.one_minus_alpha, grad), grad));
	n = __fadd_rn(__fmul_rn(p.momentum, m), __fdiv_rn(grad, __fadd_rn(__fsqrt_rn(u), p.epsilon)));
	b = __fsub_rn(a, __fmul_rn(p.rate, n));
}

// ------------------------------------------------------------------------------------------------ table walk
__device__ __forceinline__ int tensor_of(const OptimTable& t)
{
	int ti = 0;
	while (ti + 1 < t.tensors && blockIdx.x >= t.block_start[ti + 1])
		ti++;
	return ti;
}
template <int W, typename T>
__device__ __forceinline__ void ldw(const T* p, float (&x)[W])
{
	if (W == 4)
	{
		const float4 q = ld4(p);
		x[0] = q.x, x[1 % W] = q.y, x[2 % W] = q.z, x[3 % W] = q.w;
	} else
		x[0] = ldf(p);
}
template <int W, typename T>
__device__ __forceinline__ void stw(T* p, const float (&x)[W])
{
	if (W == 4)
		st4(p, make_float4(x[0], x[1 % W], x[2 % W], x[3 % W]));
	else
		stf(p, x[0]);
}
// calls f(i, g[W], a[W], m[W], v[W]) for this CTA's elements of tensor ti, W at a time, in element order per thread
template <int W, typename TG, typename TS, typename F>
__device__ __forceinline__ void walk_chunk(const OptimTable& t, const int ti, F&& f)
{
	const TG* const g = (const TG*)t.g[ti];
	const TS* const a = (const TS*)t.a[ti];
	const TS* const m = (const TS*)t.m[ti];
	const TS* const v = (const TS*)t.v[ti];
	const unsigned long long count = t.count[ti];
	const unsigned long long base = (unsigned long long)(blockIdx.x - t.block_start[ti]) * OPTIM_CHUNK;
#pragma unroll
	for (int it = 0; it < (int)(OPTIM_CHUNK / (OPTIM_THREADS * W)); it++)
	{
		const unsigned long long i = base + ((unsigned long long)it * OPTIM_THREADS + threadIdx.x) * W;
		if (i >= count)
			break; // vector tensors have count % 4 == 0, so i < count covers the whole vector
		float gv[W], av[W], mv[W], vv[W];
		ldw<W>(g + i, gv);
		ldw<W>(a + i, av);
		ldw<W>(m + i, mv);
		ldw<W>(v + i, vv);
		f(i, gv, av, mv, vv);
	}
}

// the CTA's sum of (x, y) in a fixed tree: warp butterfly, then warp 0 adds the warps in order; valid in thread 0
__device__ __forceinline__ void block_sum2(double& x, double& y)
{
	__shared__ double sx[OPTIM_THREADS / 32], sy[OPTIM_THREADS / 32];
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
	{
		x = __dadd_rn(x, __shfl_xor_sync(0xffffffffu, x, o));
		y = __dadd_rn(y, __shfl_xor_sync(0xffffffffu, y, o));
	}
	if ((threadIdx.x & 31) == 0)
		sx[threadIdx.x >> 5] = x, sy[threadIdx.x >> 5] = y;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		x = sx[0], y = sy[0];
		for (int w = 1; w < OPTIM_THREADS / 32; w++)
			x = __dadd_rn(x, sx[w]), y = __dadd_rn(y, sy[w]);
	}
}

// ------------------------------------------------------------------------------------------------ LAMB
template <int W, typename TG, typename TS>
__device__ __forceinline__ void lamb_norm_chunk(const OptimTable& t, const int ti, const LambArgs& p, double& sa, double& su)
{
	walk_chunk<W, TG, TS>(t, ti, [&](const unsigned long long, const float (&g)[W], const float (&a)[W], const float (&m)[W], const float (&v)[W]) {
#pragma unroll
		for (int j = 0; j < W; j++)
		{
			float n, u;
			const float update = lamb_update(p, g[j], a[j], m[j], v[j], n, u);
			sa = __dadd_rn(sa, (double)__fmul_rn(a[j], a[j]));
			su = __dadd_rn(su, (double)__fmul_rn(update, update));
		}
	});
}
template <typename TG, typename TS>
__global__ void __launch_bounds__(OPTIM_THREADS) lamb_norm_kernel(const __grid_constant__ OptimTable t, const LambArgs p, double2* __restrict__ partial)
{
	const int ti = tensor_of(t);
	double sa = 0, su = 0;
	if (t.vec[ti])
		lamb_norm_chunk<4, TG, TS>(t, ti, p, sa, su);
	else
		lamb_norm_chunk<1, TG, TS>(t, ti, p, sa, su);
	block_sum2(sa, su);
	if (threadIdx.x == 0)
		partial[blockIdx.x] = make_double2(sa, su);
}
// one CTA per tensor: its partials in a fixed order, then r = rate * trust as CPU_REF forms it
__global__ void __launch_bounds__(OPTIM_THREADS) lamb_trust_kernel(const __grid_constant__ OptimTable t, const float rate, const double2* __restrict__ partial, float* __restrict__ r)
{
	const unsigned ti = blockIdx.x;
	double sa = 0, su = 0;
	for (unsigned k = t.block_start[ti] + threadIdx.x; k < t.block_start[ti + 1]; k += OPTIM_THREADS)
		sa = __dadd_rn(sa, partial[k].x), su = __dadd_rn(su, partial[k].y);
	block_sum2(sa, su);
	if (threadIdx.x == 0)
	{
		const double w_norm = __dsqrt_rn(sa), update_norm = __dsqrt_rn(su);
		const float trust = w_norm > 0 && update_norm > 0 ? __double2float_rn(__ddiv_rn(w_norm, update_norm)) : 1.f; // NaN: 1
		r[ti] = __fmul_rn(rate, trust);
	}
}
template <int W, typename TG, typename TS>
__device__ __forceinline__ void lamb_apply_chunk(const OptimTable& t, const int ti, const LambArgs& p, const float r)
{
	TS* const b = (TS*)t.b[ti];
	TS* const n = (TS*)t.n[ti];
	TS* const u = (TS*)t.u[ti];
	walk_chunk<W, TG, TS>(t, ti, [&](const unsigned long long i, const float (&g)[W], const float (&a)[W], const float (&m)[W], const float (&v)[W]) {
		float bv[W], nv[W], uv[W];
#pragma unroll
		for (int j = 0; j < W; j++)
			bv[j] = __fsub_rn(a[j], __fmul_rn(r, lamb_update(p, g[j], a[j], m[j], v[j], nv[j], uv[j])));
		stw<W>(b + i, bv);
		stw<W>(n + i, nv);
		stw<W>(u + i, uv);
	});
}
template <typename TG, typename TS>
__global__ void __launch_bounds__(OPTIM_THREADS) lamb_apply_kernel(const __grid_constant__ OptimTable t, const LambArgs p, const float* __restrict__ r)
{
	const int ti = tensor_of(t);
	if (t.vec[ti])
		lamb_apply_chunk<4, TG, TS>(t, ti, p, r[ti]);
	else
		lamb_apply_chunk<1, TG, TS>(t, ti, p, r[ti]);
}

// ------------------------------------------------------------------------------------------------ RMSPROP
template <int W, typename TG, typename TS>
__device__ __forceinline__ void rmsprop_chunk(const OptimTable& t, const int ti, const RmspropArgs& p)
{
	TS* const b = (TS*)t.b[ti];
	TS* const n = (TS*)t.n[ti];
	TS* const u = (TS*)t.u[ti];
	walk_chunk<W, TG, TS>(t, ti, [&](const unsigned long long i, const float (&g)[W], const float (&a)[W], const float (&m)[W], const float (&v)[W]) {
		float bv[W], nv[W], uv[W];
#pragma unroll
		for (int j = 0; j < W; j++)
			rmsprop_step(p, g[j], a[j], m[j], v[j], bv[j], nv[j], uv[j]);
		stw<W>(b + i, bv);
		stw<W>(n + i, nv);
		stw<W>(u + i, uv);
	});
}
template <typename TG, typename TS>
__global__ void __launch_bounds__(OPTIM_THREADS) rmsprop_kernel(const __grid_constant__ OptimTable t, const RmspropArgs p)
{
	const int ti = tensor_of(t);
	if (t.vec[ti])
		rmsprop_chunk<4, TG, TS>(t, ti, p);
	else
		rmsprop_chunk<1, TG, TS>(t, ti, p);
}

// ------------------------------------------------------------------------------------------------ host

// f(TG(), TS()) with the element types of the gradient and of the state
template <typename F>
int with_types(const int g_kind, const int s_kind, F&& f)
{
	auto state = [&](auto tg) {
		if (s_kind == 0)
			return f(tg, float());
		if (s_kind == 1)
			return f(tg, __nv_bfloat16());
		return f(tg, __half());
	};
	if (g_kind == 0)
		return state(float());
	if (g_kind == 1)
		return state(__nv_bfloat16());
	return state(__half());
}

// T commands' operands, inputs (g, a, m, v) x T -> outputs (b, n, u) x T, checked and split into launch tables.  Returns false (and
// launches nothing) when any operand is refused.
bool plan(ccv_nnc_tensor_t* const* const inputs, ccv_nnc_tensor_t* const* const outputs, const int T, int& g_kind, int& s_kind, std::vector<OptimTable>& tables, unsigned& max_blocks)
{
	g_kind = inputs[0] ? kind_of(inputs[0]) : -1;
	s_kind = inputs[1] ? kind_of(inputs[1]) : -1;
	if (g_kind < 0 || s_kind < 0)
		return false;
	tables.clear();
	max_blocks = 0;
	OptimTable cur;
	cur.tensors = 0;
	unsigned long long blocks = 0;
	auto flush = [&]() {
		if (cur.tensors == 0)
			return;
		cur.block_start[cur.tensors] = (unsigned)blocks;
		tables.push_back(cur);
		max_blocks = max_blocks > (unsigned)blocks ? max_blocks : (unsigned)blocks;
		cur.tensors = 0;
		blocks = 0;
	};
	for (int t = 0; t < T; t++)
	{
		ccv_nnc_tensor_t* const ops[7] = { inputs[4 * t], inputs[4 * t + 1], inputs[4 * t + 2], inputs[4 * t + 3], outputs[3 * t], outputs[3 * t + 1], outputs[3 * t + 2] };
		for (int i = 0; i < 7; i++)
			if (!ops[i] || !CCV_IS_TENSOR_CONTIGUOUS(ops[i]) || kind_of(ops[i]) != (i == 0 ? g_kind : s_kind))
				return false;
		const size_t count = count_of(ops[1]);
		bool vec = count % 4 == 0 && (((uintptr_t)ops[0]->data.u8) & (4 * elem_size(g_kind) - 1)) == 0;
		for (int i = 0; i < 7; i++)
		{
			if (count_of(ops[i]) != count)
				return false;
			if (i > 0 && (((uintptr_t)ops[i]->data.u8) & (4 * elem_size(s_kind) - 1)) != 0)
				vec = false;
		}
		const unsigned long long chunks = (count + OPTIM_CHUNK - 1) / OPTIM_CHUNK;
		if (chunks > (unsigned long long)INT_MAX)
			return false; // more than 2^43 elements in one tensor: beyond one grid
		if (cur.tensors == OPTIM_MULTI_MAX || blocks + chunks > (unsigned long long)INT_MAX)
			flush();
		const int k = cur.tensors++;
		cur.g[k] = ops[0]->data.u8, cur.a[k] = ops[1]->data.u8, cur.m[k] = ops[2]->data.u8, cur.v[k] = ops[3]->data.u8;
		cur.b[k] = ops[4]->data.u8, cur.n[k] = ops[5]->data.u8, cur.u[k] = ops[6]->data.u8;
		cur.count[k] = count;
		cur.vec[k] = vec;
		cur.block_start[k] = (unsigned)blocks;
		blocks += chunks;
	}
	flush();
	return true;
}

int run_lamb(const ccv_nnc_cmd_t cmd, ccv_nnc_tensor_t* const* const inputs, ccv_nnc_tensor_t* const* const outputs, const int T, ccv_nnc_stream_context_t* const stream_context)
{
	const int step = cmd.info.lamb.step;
	if (step < 1)
		return CCV_NNC_EXEC_INVALID;
	int g_kind, s_kind;
	unsigned max_blocks;
	std::vector<OptimTable> tables;
	if (!plan(inputs, outputs, T, g_kind, s_kind, tables, max_blocks))
		return CCV_NNC_EXEC_INVALID;
	LambArgs p;
	p.scale = cmd.info.lamb.scale;
	p.beta1 = cmd.info.lamb.beta1, p.one_minus_beta1 = 1 - p.beta1;
	p.beta2 = cmd.info.lamb.beta2, p.one_minus_beta2 = 1 - p.beta2;
	p.ibc1 = (float)(1. / (1 - powf(p.beta1, step)));
	p.ibc2 = (float)(1. / (1 - powf(p.beta2, step)));
	p.epsilon = cmd.info.lamb.epsilon, p.decay = cmd.info.lamb.decay, p.rate = cmd.info.lamb.rate;
	// partials of the largest table, then one r per tensor; tables run in stream order, so each reuses the same bytes
	unsigned char* const ws = (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, (size_t)max_blocks * sizeof(double2) + OPTIM_MULTI_MAX * sizeof(float), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	double2* const partial = (double2*)ws;
	float* const r = (float*)(ws + (size_t)max_blocks * sizeof(double2));
	cudaStream_t s = (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context);
	for (const OptimTable& t : tables)
	{
		const unsigned blocks = t.block_start[t.tensors];
		const int rc = with_types(g_kind, s_kind, [&](auto tg, auto ts) {
			using TG = decltype(tg);
			using TS = decltype(ts);
			lamb_norm_kernel<TG, TS><<<blocks, OPTIM_THREADS, 0, s>>>(t, p, partial);
			if (launched("lamb_norm"))
				return -1;
			lamb_trust_kernel<<<t.tensors, OPTIM_THREADS, 0, s>>>(t, p.rate, partial, r);
			if (launched("lamb_trust"))
				return -1;
			lamb_apply_kernel<TG, TS><<<blocks, OPTIM_THREADS, 0, s>>>(t, p, r);
			return launched("lamb_apply");
		});
		if (rc)
			return CCV_NNC_EXEC_INVALID;
	}
	return CCV_NNC_EXEC_SUCCESS;
}

int run_rmsprop(const ccv_nnc_cmd_t cmd, ccv_nnc_tensor_t* const* const inputs, ccv_nnc_tensor_t* const* const outputs, const int T, ccv_nnc_stream_context_t* const stream_context)
{
	int g_kind, s_kind;
	unsigned max_blocks;
	std::vector<OptimTable> tables;
	if (!plan(inputs, outputs, T, g_kind, s_kind, tables, max_blocks))
		return CCV_NNC_EXEC_INVALID;
	RmspropArgs p;
	p.rate = cmd.info.rmsprop.rate, p.scale = cmd.info.rmsprop.scale, p.decay = cmd.info.rmsprop.decay;
	p.alpha = cmd.info.rmsprop.alpha, p.one_minus_alpha = 1 - p.alpha;
	p.momentum = cmd.info.rmsprop.momentum, p.epsilon = cmd.info.rmsprop.epsilon;
	cudaStream_t s = (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context);
	for (const OptimTable& t : tables)
	{
		const int rc = with_types(g_kind, s_kind, [&](auto tg, auto ts) {
			rmsprop_kernel<decltype(tg), decltype(ts)><<<t.block_start[t.tensors], OPTIM_THREADS, 0, s>>>(t, p);
			return launched("rmsprop");
		});
		if (rc)
			return CCV_NNC_EXEC_INVALID;
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// one command: inputs (g, a, m, v) -> outputs (b, n, u)
template <int IS_LAMB>
int exec_optim(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 4 || output_size < 3)
		return CCV_NNC_EXEC_INVALID;
	return IS_LAMB ? run_lamb(cmd, inputs, outputs, 1, stream_context) : run_rmsprop(cmd, inputs, outputs, 1, stream_context);
}
// T commands with identical parameters (a fused graph run): inputs (g, a, m, v) x T -> outputs (b, n, u) x T
template <int IS_LAMB>
int exec_optim_multi(const ccv_nnc_cmd_t cmd, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const int T = input_size / 4;
	if (T < 1 || input_size != 4 * T || output_size != 3 * T)
		return CCV_NNC_EXEC_INVALID;
	return IS_LAMB ? run_lamb(cmd, inputs, outputs, T, stream_context) : run_rmsprop(cmd, inputs, outputs, T, stream_context);
}

} // namespace

extern "C" int ccv_nnc_sm100_fused_lamb_multi(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return exec_optim_multi<1>(cmd, inputs, input_size, outputs, output_size, stream_context);
}
extern "C" int ccv_nnc_sm100_fused_rmsprop_multi(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return exec_optim_multi<0>(cmd, inputs, input_size, outputs, output_size, stream_context);
}

REGISTER_SM100(CCV_NNC_LAMB_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_optim<1>); }
REGISTER_SM100(CCV_NNC_LAMB_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_invalid); }
REGISTER_SM100(CCV_NNC_RMSPROP_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_optim<0>); }
REGISTER_SM100(CCV_NNC_RMSPROP_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_invalid); }
