// sm100_loss.cu -- BINARY_CROSSENTROPY, SIGMOID_BINARY_CROSSENTROPY, MSE and SMOOTH_L1 (forward / backward) over [batch, count]
// rows of fp32, bf16 or fp16 tensors (b may be fp32 under 16-bit a).  Semantics (paths relative to lib/nnc/cmd of the reference):
//   loss/ccv_nnc_binary_crossentropy_cpu_ref.c          c = sum (b - 1) log(1 - a) - pw b log(a)    h = g (a b (pw - 1) + a - pw b) / max((1 - a) a, 1e-12)
//   sigmoid_loss/ccv_nnc_sigmoid_binary_crossentropy_cpu_ref.c   c = sum (1 - b) a + (1 + b (pw - 1)) log(1 + e^-a), d = sigmoid(a);  h = g ((d - 1) b pw + d (1 - b))
//   loss/ccv_nnc_mse_cpu_ref.c                          c = sum (b - a)^2 (/ count);  ha = (2 / count | 2) g (a - b), hb = the same with (b - a)
//   loss/ccv_nnc_smooth_l1_cpu_ref.c                    s = sum |b - a|; c = s < beta ? sum (b - a)^2 0.5 / beta : s - 0.5 beta;  h from c against beta / 2
// pw = 1 takes the reference's shorter forms.  Outputs are overwritten (CCV_NNC_ACCUMULATE_OUTPUT is ignored, as in CPU_REF).
//
// Forward: a per-row reduction (loss_plan) fixed by batch, count and the element size alone.  A row is cut into units of one 16-byte
// vector of a (4 fp32 / 8 16-bit elements; the last unit of a row may be short), a unit's elements are added in order by one thread,
// and a group of G threads (G a power of two <= 32, or a whole CTA of 256) takes a segment of a row: units lane, lane + G, ...; the
// group's sums are added by a fixed shuffle tree (and, for G = 256, the 8 warp sums in warp order).  Short rows pack 256 / G to a
// CTA; a row longer than LOSS_CHUNK_UNITS units is split into chunks of that many units, whose fp32 partials go to the workspace and
// are added per row by loss_combine_kernel, which applies the loss's finish (mean scale, smooth-L1 branch, pos_weight) before the
// single rounding.  Unaligned operands load element by element in the same unit order, so the bits depend on the shape only.  No
// atomics: two runs give the same bits.
// Backward: one element-wise pass (16-byte vectors on aligned rows, one element per thread otherwise) in CPU_REF's operations and
// order, each product / sum rounded on its own (no FMA contraction): fp32 gradients equal CPU_REF's bit for bit, 16-bit ones CPU_REF's
// on the widened inputs, rounded once.  BCE divides by the clamped denominator in double as CPU_REF does.
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <cuda_runtime.h>
#include <string.h>

using namespace sm100;

namespace {

enum { L_BCE, L_SBCE, L_MSE, L_SL1 };
constexpr int THREADS = 256;
constexpr int LOSS_CHUNK_UNITS = 2048; // units per chunk of a split row: 8 per thread of a 256-thread CTA

struct LossArg {
	int batch, count;
	long long xs, bs, os, o2s; // row pitches (elements): a (backward of SBCE: d), b, the element-wise output (h / ha; forward: d), hb
	long long cstep, gstep;    // element step between rows of c and g
	int pw1;                   // pos_weight == 1: the reference's short forms
	float pw, pwm1;            // pos_weight, pos_weight - 1 (fp32, as CPU_REF)
	float scale;               // MSE: (float)(1 / count) (forward) / (float)(2 / count) (backward) for the mean, 1 / 2 for the sum
	float beta, beta_2, beta_inv_2, inv_beta; // smooth L1: beta, (float)(0.5 beta), (float)(0.5 / beta), (float)(1 / beta)
	// forward plan
	int units, group, chunk_units, chunks, np;
};

// the forward plan: a function of (batch, count, element size) only
struct LossPlan {
	int units, group, chunk_units, chunks, np;
	size_t blocks;    // CTAs of the reduction launch
	size_t ws_bytes;  // fp32 partials of split rows
	int launches;
};
LossPlan loss_plan(const int op, const int pw1, const int batch, const int count, const int elem_size, const int with_c)
{
	LossPlan p;
	const int V = 16 / elem_size;
	p.units = (count + V - 1) / V;
	p.np = (op == L_BCE && !pw1) || op == L_SL1 ? 2 : 1;
	if (p.units <= 32)
	{
		p.group = 1;
		while (p.group < p.units)
			p.group *= 2;
	} else
		p.group = p.units <= 256 ? 32 : THREADS;
	p.chunk_units = p.units > LOSS_CHUNK_UNITS ? LOSS_CHUNK_UNITS : p.units;
	p.chunks = (p.units + p.chunk_units - 1) / p.chunk_units;
	const size_t segs = (size_t)batch * p.chunks, per_cta = THREADS / p.group;
	p.blocks = (segs + per_cta - 1) / per_cta;
	p.ws_bytes = with_c && p.chunks > 1 ? segs * p.np * sizeof(float) : 0;
	p.launches = with_c && p.chunks > 1 ? 2 : 1;
	return p;
}

// how a unit of V elements is read / written: element by element up to `n`; in groups of 4 (ld4 / st4: 16 bytes in fp32, 8 in 16-bit;
// rows of a multiple of 4 elements, such as [N, 4] boxes); or as one 16-byte vector (two for fp32 b under 16-bit a).  The values and
// the order they are used in are the same in every mode.
enum { M_ELEM, M_QUAD, M_VEC };
template <int V, int MODE, typename T>
__device__ __forceinline__ void ld_unit(const T* p, float (&v)[V], const int n)
{
	if constexpr (MODE == M_VEC && sizeof(T) * V == 16)
		ldv(p, v);
	else if constexpr (MODE == M_VEC) {
#pragma unroll
		for (int j = 0; j < V; j += 4)
			ldv(p + j, *reinterpret_cast<float(*)[4]>(&v[j]));
	} else if constexpr (MODE == M_QUAD) {
#pragma unroll
		for (int j = 0; j < V; j += 4)
		{
			const float4 t = j < n ? ld4(p + j) : make_float4(0.f, 0.f, 0.f, 0.f);
			v[j] = t.x, v[j + 1] = t.y, v[j + 2] = t.z, v[j + 3] = t.w;
		}
	} else {
#pragma unroll
		for (int j = 0; j < V; j++)
			v[j] = j < n ? ldf(p + j) : 0.f;
	}
}
template <int V, int MODE, typename T>
__device__ __forceinline__ void st_unit(T* p, const float (&v)[V], const int n)
{
	if constexpr (MODE == M_VEC)
		stv(p, v);
	else if constexpr (MODE == M_QUAD) {
#pragma unroll
		for (int j = 0; j < V; j += 4)
			if (j < n)
				st4(p + j, make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]));
	} else {
#pragma unroll
		for (int j = 0; j < V; j++)
			if (j < n)
				stf(p + j, v[j]);
	}
}

// one element's contribution to the row sums (s0, s1); SBCE also gives d = sigmoid(a)
template <int OP>
__device__ __forceinline__ void loss_term(const float a, const float b, const LossArg& p, float& s0, float& s1, float& d)
{
	if (OP == L_BCE)
	{
		const float t1 = (b - 1.f) * logf(1.f - a), t2 = b * logf(a);
		if (p.pw1)
			s0 += t1 - t2;
		else
			s0 += t1, s1 += t2;
	} else if (OP == L_SBCE) {
		// log(1 + e^-a) = max(-a, 0) + log1p(e^-|a|): finite for every finite a (the direct form overflows below a = -88.7)
		const float e = expf(-fabsf(a));
		const float sp = fmaxf(-a, 0.f) + log1pf(e);
		s0 += (1.f - b) * a + (1.f + b * p.pwm1) * sp;
		d = a >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
	} else if (OP == L_MSE) {
		const float t = b - a;
		s0 += t * t;
	} else {
		const float t = b - a;
		s0 += fabsf(t), s1 += t * t;
	}
}
template <int OP>
__device__ __forceinline__ float loss_finish(const float s0, const float s1, const LossArg& p)
{
	if (OP == L_BCE)
		return p.pw1 ? s0 : s0 - s1 * p.pw;
	if (OP == L_MSE)
		return s0 * p.scale;
	if (OP == L_SL1)
		return s0 < p.beta ? s1 * p.beta_inv_2 : s0 - p.beta_2;
	return s0;
}
// the sum of a group of G threads (power of two <= 32) by a fixed xor tree; lane 0 of the group holds it
__device__ __forceinline__ float group_sum(float v, const int G)
{
	for (int o = G >> 1; o > 0; o >>= 1)
		v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

// forward: each group of p.group threads reduces one segment (row, chunk); c == NULL (SBCE without c) only writes d
template <int OP, typename T, typename TB, int MODE>
__global__ void __launch_bounds__(THREADS) loss_fwd_kernel(const T* a, const TB* b, T* c, T* d, float* part, const LossArg p)
{
	constexpr int V = Vec16<T>::W;
	__shared__ float red[2][THREADS / 32];
	const int G = p.group, lane = threadIdx.x & (G - 1);
	const long long per_cta = THREADS / G, segs = (long long)p.batch * p.chunks;
	for (long long seg0 = blockIdx.x * per_cta; seg0 < segs; seg0 += (long long)gridDim.x * per_cta)
	{
		const long long seg = seg0 + threadIdx.x / G;
		float s0 = 0.f, s1 = 0.f;
		long long row = 0;
		if (seg < segs)
		{
			row = seg / p.chunks;
			const int k = (int)(seg - row * p.chunks);
			const int u1 = min((k + 1) * p.chunk_units, p.units);
			const T* const ap = a + row * p.xs;
			const TB* const bp = b + row * p.bs;
			for (int u = k * p.chunk_units + lane; u < u1; u += G)
			{
				const int n = min(V, p.count - u * V);
				float av[V], bv[V], dv[V];
				ld_unit<V, MODE>(ap + u * V, av, n);
				ld_unit<V, MODE>(bp + u * V, bv, n);
				float t0 = 0.f, t1 = 0.f;
#pragma unroll
				for (int j = 0; j < V; j++)
					if (MODE == M_VEC || j < n)
						loss_term<OP>(av[j], bv[j], p, t0, t1, dv[j]);
				s0 += t0, s1 += t1;
				if (OP == L_SBCE)
					st_unit<V, MODE>(d + row * p.os + u * V, dv, n);
			}
		}
		if (!c)
			continue;
		if (G <= 32)
			s0 = group_sum(s0, G), s1 = group_sum(s1, G);
		else {
			s0 = group_sum(s0, 32), s1 = group_sum(s1, 32);
			if ((threadIdx.x & 31) == 0)
				red[0][threadIdx.x >> 5] = s0, red[1][threadIdx.x >> 5] = s1;
			__syncthreads();
			if (threadIdx.x == 0)
			{
				s0 = red[0][0], s1 = red[1][0];
				for (int w = 1; w < THREADS / 32; w++)
					s0 += red[0][w], s1 += red[1][w];
			}
			__syncthreads();
		}
		if (lane == 0 && seg < segs)
		{
			if (p.chunks == 1)
				stf(c + row * p.cstep, loss_finish<OP>(s0, s1, p));
			else {
				part[seg * p.np] = s0;
				if (p.np == 2)
					part[seg * p.np + 1] = s1;
			}
		}
	}
}
// split rows: one warp per row adds the row's chunk partials (lane-strided in chunk order, then the xor tree), finishes and rounds once
template <int OP, typename T>
__global__ void __launch_bounds__(THREADS) loss_combine_kernel(const float* part, T* c, const LossArg p)
{
	const long long row = ((long long)blockIdx.x * THREADS + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (row >= p.batch)
		return;
	const float* const q = part + row * p.chunks * p.np;
	float s0 = 0.f, s1 = 0.f;
	for (int k = lane; k < p.chunks; k += 32)
	{
		s0 += q[k * p.np];
		if (p.np == 2)
			s1 += q[k * p.np + 1];
	}
	s0 = group_sum(s0, 32), s1 = group_sum(s1, 32);
	if (lane == 0)
		stf(c + row * p.cstep, loss_finish<OP>(s0, s1, p));
}

// backward, one element: x = a (d for SBCE), y = b; per-row g (1 when absent: gv is then unused) and c (smooth L1)
template <int OP>
__device__ __forceinline__ void loss_grad(const float x, const float y, const bool has_g, const float gv, const float cv, const LossArg& p, float& h0, float& h1)
{
	if (OP == L_BCE)
	{
		const float num0 = p.pw1 ? __fsub_rn(x, y) : __fsub_rn(__fadd_rn(__fmul_rn(__fmul_rn(x, y), p.pwm1), x), __fmul_rn(p.pw, y));
		const float num = has_g ? __fmul_rn(gv, num0) : num0;
		const float den = __fmul_rn(__fsub_rn(1.f, x), x);
		// ccv_max((1 - a) a, 1e-12): a double; the quotient of a float by a float is the same in float as in double rounded to float
		h0 = (double)den > 1e-12 ? __fdiv_rn(num, den) : __double2float_rn(__ddiv_rn((double)num, 1e-12));
	} else if (OP == L_SBCE) {
		const float v = p.pw1 ? __fsub_rn(x, y) : __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(x, 1.f), y), p.pw), __fmul_rn(x, __fsub_rn(1.f, y)));
		h0 = has_g ? __fmul_rn(gv, v) : v;
	} else if (OP == L_MSE) {
		const float gs = has_g ? __fmul_rn(p.scale, gv) : p.scale;
		h0 = __fmul_rn(gs, __fsub_rn(x, y)), h1 = __fmul_rn(gs, __fsub_rn(y, x));
	} else {
		const float t = __fsub_rn(x, y);
		if (cv < p.beta_2)
			h0 = __fmul_rn(has_g ? __fmul_rn(p.inv_beta, gv) : p.inv_beta, t);
		else {
			const float gs = has_g ? gv : 1.f;
			h0 = t > 0.f ? gs : -gs;
		}
	}
}
// B_ELEM: one element per work item; B_ROWVEC: one 16-byte vector of a row (count a whole number of vectors, aligned rows); B_FLAT:
// one 16-byte vector of the packed [batch, count] tensors taken as one flat array, whatever count is (a vector may span rows: g and c
// are read per element)
enum { B_ELEM, B_ROWVEC, B_FLAT };
template <int OP, typename T, typename TB, int MODE>
__global__ void __launch_bounds__(THREADS) loss_bwd_kernel(const T* g, const T* x, const TB* y, const T* c, T* h0, T* h1, const LossArg p, const size_t n)
{
	constexpr int V = MODE == B_ELEM ? 1 : Vec16<T>::W;
	constexpr int LM = MODE == B_ELEM ? M_ELEM : M_VEC;
	const size_t per_row = (size_t)(p.count / V);
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
	{
		float xv[V], yv[V], o0[V], o1[V];
		size_t row, xo, bo, oo, o2o;
		if (MODE == B_FLAT)
		{
			xo = bo = oo = o2o = i * V;
			row = xo / (size_t)p.count;
		} else {
			row = i / per_row;
			const size_t col = (i - row * per_row) * V;
			xo = row * p.xs + col, bo = row * p.bs + col, oo = row * p.os + col, o2o = row * p.o2s + col;
		}
		ld_unit<V, LM>(x + xo, xv, V);
		ld_unit<V, LM>(y + bo, yv, V);
		int col = (int)(xo - row * (size_t)p.count); // B_FLAT: the column of element 0 of the vector
#pragma unroll
		for (int j = 0; j < V; j++)
		{
			if (MODE == B_FLAT && j > 0 && ++col == p.count)
				col = 0, row++;
			const float gv = g ? ldf(g + row * p.gstep) : 1.f;
			const float cv = OP == L_SL1 ? ldf(c + row * p.cstep) : 0.f;
			loss_grad<OP>(xv[j], yv[j], g != 0, gv, cv, p, o0[j], o1[j]);
		}
		if (h0)
			st_unit<V, LM>(h0 + oo, o0, V);
		if (OP == L_MSE && h1)
			st_unit<V, LM>(h1 + o2o, o1, V);
	}
}

// one call's operands (device pointers; NULL where absent)
struct LossCall {
	const void *g, *x, *y, *c;
	void *out, *out2, *part; // forward: out = c, out2 = d; backward: out = h / ha, out2 = hb
};
template <typename T>
bool v16(const void* p, const long long pitch) { return !p || (aligned_v16((const char*)p) && pitch % Vec16<T>::W == 0); }
template <typename T>
bool v4(const void* p, const long long pitch) { return !p || ((((uintptr_t)p) & (4 * sizeof(T) - 1)) == 0 && pitch % 4 == 0); }

template <int OP, typename T, typename TB, int MODE>
int launch_fwd(cudaStream_t s, const LossCall& k, const LossArg& p, const LossPlan& plan)
{
	const unsigned blocks = (unsigned)(plan.blocks < (1u << 30) ? plan.blocks : (1u << 30));
	loss_fwd_kernel<OP, T, TB, MODE><<<blocks, THREADS, 0, s>>>((const T*)k.x, (const TB*)k.y, (T*)k.out, (T*)k.out2, (float*)k.part, p);
	if (launched("loss forward"))
		return -1;
	if (plan.launches == 1)
		return 0;
	loss_combine_kernel<OP, T><<<(unsigned)(((size_t)p.batch * 32 + THREADS - 1) / THREADS), THREADS, 0, s>>>((const float*)k.part, (T*)k.out, p);
	return launched("loss combine");
}
template <int OP, typename T, typename TB, int MODE>
int launch_bwd(cudaStream_t s, const LossCall& k, const LossArg& p)
{
	const size_t n = MODE == B_FLAT ? (size_t)p.batch * p.count / Vec16<T>::W : (size_t)p.batch * (p.count / (MODE == B_ROWVEC ? Vec16<T>::W : 1));
	size_t blocks = (n + THREADS - 1) / THREADS;
	if (blocks > (size_t)sm_count() * 16)
		blocks = (size_t)sm_count() * 16;
	loss_bwd_kernel<OP, T, TB, MODE><<<(unsigned)blocks, THREADS, 0, s>>>((const T*)k.g, (const T*)k.x, (const TB*)k.y, (const T*)k.c, (T*)k.out, (T*)k.out2, p, n);
	return launched("loss backward");
}
template <int OP, typename T, typename TB>
int run_t(cudaStream_t s, const int forward, const LossCall& k, const LossArg& p, const LossPlan& plan)
{
	const bool vec = p.count % Vec16<T>::W == 0 && v16<T>(k.x, p.xs) && v16<TB>(k.y, p.bs) && (forward ? v16<T>(k.out2, p.os) : v16<T>(k.out, p.os) && v16<T>(k.out2, p.o2s));
	if (forward)
	{
		const bool quad = p.count % 4 == 0 && v4<T>(k.x, p.xs) && v4<TB>(k.y, p.bs) && v4<T>(k.out2, p.os);
		return vec ? launch_fwd<OP, T, TB, M_VEC>(s, k, p, plan) : quad ? launch_fwd<OP, T, TB, M_QUAD>(s, k, p, plan) : launch_fwd<OP, T, TB, M_ELEM>(s, k, p, plan);
	}
	if (vec)
		return launch_bwd<OP, T, TB, B_ROWVEC>(s, k, p);
	// packed operands whose rows are not whole vectors (16-bit [N, 4] boxes): stream the tensors flat
	const long long cnt = p.count;
	const bool flat = ((long long)p.batch * cnt) % Vec16<T>::W == 0 && p.xs == cnt && p.bs == cnt && (!k.out || p.os == cnt) && (!k.out2 || p.o2s == cnt) &&
		v16<T>(k.x, 0) && v16<TB>(k.y, 0) && v16<T>(k.out, 0) && v16<T>(k.out2, 0);
	return flat ? launch_bwd<OP, T, TB, B_FLAT>(s, k, p) : launch_bwd<OP, T, TB, B_ELEM>(s, k, p);
}
template <int OP>
int run_loss(cudaStream_t s, const int kind, const int bkind, const int forward, const LossCall& k, const LossArg& p, const LossPlan& plan)
{
	if (kind == 0)
		return run_t<OP, float, float>(s, forward, k, p, plan);
	if (kind == 1)
		return bkind == 0 ? run_t<OP, __nv_bfloat16, float>(s, forward, k, p, plan) : run_t<OP, __nv_bfloat16, __nv_bfloat16>(s, forward, k, p, plan);
	return bkind == 0 ? run_t<OP, __half, float>(s, forward, k, p, plan) : run_t<OP, __half, __half>(s, forward, k, p, plan);
}

// ------------------------------------------------------------------------------------------------ command layer
// a [batch, count] operand (1-d: one row) whose inner axis is contiguous; its row pitch in elements
struct Rows {
	int batch, count;
	long long pitch;
};
bool rows_of(const ccv_nnc_tensor_t* const t, Rows& r)
{
	const int nd = nd_of(t);
	if (nd < 1 || nd > 2)
		return false;
	const bool view = CCV_IS_TENSOR_VIEW(t);
	const int* const stride = ((const ccv_nnc_tensor_view_t*)t)->stride;
	r.batch = nd == 2 ? t->info.dim[0] : 1;
	r.count = t->info.dim[nd - 1];
	if (view && stride[nd - 1] != 1)
		return false;
	r.pitch = nd == 2 && view ? stride[0] : r.count;
	return true;
}
bool same_rows(const Rows& a, const Rows& b) { return a.batch == b.batch && a.count == b.count; }
// c / g: `batch` elements, 1-d or [batch, 1]; the element step between rows as CPU_REF takes it (1 for 1-d, the outer stride for 2-d)
bool per_row(const ccv_nnc_tensor_t* const t, const int batch, long long& step)
{
	const int nd = nd_of(t);
	if (nd < 1 || nd > 2 || t->info.dim[0] != batch || (nd == 2 && t->info.dim[1] != 1))
		return false;
	step = nd == 2 && CCV_IS_TENSOR_VIEW(t) ? ((const ccv_nnc_tensor_view_t*)t)->stride[0] : 1;
	return true;
}
void* data_of(const ccv_nnc_tensor_t* const t) { return t ? t->data.u8 : 0; }

LossArg loss_arg(const ccv_nnc_cmd_t& cmd, const int op, const int forward, const Rows& r)
{
	LossArg p;
	memset(&p, 0, sizeof(p));
	p.batch = r.batch, p.count = r.count;
	p.pw = cmd.info.binary_crossentropy.pos_weight;
	p.pw1 = p.pw == 1;
	p.pwm1 = p.pw - 1;
	if (op == L_MSE)
	{
		const int mean = cmd.info.mse.reduce_op == CCV_NNC_MSE_REDUCE_MEAN;
		p.scale = forward ? (mean ? (float)(1.0 / (float)r.count) : 1.f) : (mean ? (float)(2.0 / (float)r.count) : 2.f);
	}
	if (op == L_SL1)
	{
		const float beta = cmd.info.smooth_l1.beta;
		p.beta = beta, p.beta_2 = (float)(0.5 * beta), p.beta_inv_2 = (float)(0.5 / beta), p.inv_beta = (float)(1.0 / beta);
	}
	return p;
}
bool b_kind_ok(const ccv_nnc_tensor_t* const b, const int kind)
{
	const int bk = kind_of(b);
	return bk == kind || (kind != 0 && bk == 0);
}

// inputs (a, b) -> outputs (c) or, for SBCE, (c | NULL, d)
template <int OP>
int exec_loss_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const ccv_nnc_tensor_t* const a = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const b = input_size > 1 ? inputs[1] : 0;
	const ccv_nnc_tensor_t* const c = output_size > 0 ? outputs[0] : 0;
	const ccv_nnc_tensor_t* const d = OP == L_SBCE && output_size > 1 ? outputs[1] : 0;
	if (!a || !b || (OP == L_SBCE ? !d : !c))
		return CCV_NNC_EXEC_INVALID;
	if (OP == L_MSE && cmd.info.mse.reduce_op != CCV_NNC_MSE_REDUCE_MEAN && cmd.info.mse.reduce_op != CCV_NNC_MSE_REDUCE_SUM)
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(a);
	Rows ra, rb, rd;
	long long cstep = 0;
	if (kind < 0 || !b_kind_ok(b, kind) || !rows_of(a, ra) || !rows_of(b, rb) || !same_rows(ra, rb))
		return CCV_NNC_EXEC_INVALID;
	if (c && (kind_of(c) != kind || !per_row(c, ra.batch, cstep)))
		return CCV_NNC_EXEC_INVALID;
	if (d && (kind_of(d) != kind || !rows_of(d, rd) || !same_rows(ra, rd)))
		return CCV_NNC_EXEC_INVALID;
	LossArg p = loss_arg(cmd, OP, 1, ra);
	p.xs = ra.pitch, p.bs = rb.pitch, p.os = d ? rd.pitch : 0, p.cstep = cstep;
	const LossPlan plan = loss_plan(OP, p.pw1, ra.batch, ra.count, kind == 0 ? 4 : 2, c != 0);
	p.units = plan.units, p.group = plan.group, p.chunk_units = plan.chunk_units, p.chunks = plan.chunks, p.np = plan.np;
	void* ws = 0;
	if (plan.ws_bytes)
	{
		ws = ccv_nnc_stream_context_get_workspace(stream_context, plan.ws_bytes, CCV_TENSOR_GPU_MEMORY);
		if (!ws)
			return CCV_NNC_EXEC_OOM;
	}
	const LossCall k = { 0, a->data.u8, b->data.u8, 0, data_of(c), data_of(d), ws };
	return run_loss<OP>(stream_of(stream_context), kind, kind_of(b), 1, k, p, plan) ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

// BCE (g | NULL, a, b) -> h;  SBCE (g | NULL, -, -, b, -, d) -> h;  MSE (g | NULL, a, b) -> (ha | NULL, hb | NULL);  SL1 (g | NULL, a, b, c) -> h
template <int OP>
int exec_loss_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const int xi = OP == L_SBCE ? 5 : 1, yi = OP == L_SBCE ? 3 : 2;
	const ccv_nnc_tensor_t* const g = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const x = input_size > xi ? inputs[xi] : 0;
	const ccv_nnc_tensor_t* const y = input_size > yi ? inputs[yi] : 0;
	const ccv_nnc_tensor_t* const c = OP == L_SL1 && input_size > 3 ? inputs[3] : 0;
	const ccv_nnc_tensor_t* const h0 = output_size > 0 ? outputs[0] : 0;
	const ccv_nnc_tensor_t* const h1 = OP == L_MSE && output_size > 1 ? outputs[1] : 0;
	if (!x || !y || (OP == L_SL1 && !c) || (OP == L_MSE ? !h0 && !h1 : !h0))
		return CCV_NNC_EXEC_INVALID;
	if (OP == L_MSE && cmd.info.mse.reduce_op != CCV_NNC_MSE_REDUCE_MEAN && cmd.info.mse.reduce_op != CCV_NNC_MSE_REDUCE_SUM)
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(x);
	Rows rx, ry, r0, r1;
	long long gstep = 0, cstep = 0;
	if (kind < 0 || !b_kind_ok(y, kind) || !rows_of(x, rx) || !rows_of(y, ry) || !same_rows(rx, ry))
		return CCV_NNC_EXEC_INVALID;
	if (h0 && (kind_of(h0) != kind || !rows_of(h0, r0) || !same_rows(rx, r0)))
		return CCV_NNC_EXEC_INVALID;
	if (h1 && (kind_of(h1) != kind || !rows_of(h1, r1) || !same_rows(rx, r1)))
		return CCV_NNC_EXEC_INVALID;
	// g is a packed tensor (CPU_REF asserts it is not a view)
	if (g && (kind_of(g) != kind || CCV_IS_TENSOR_VIEW(g) || !per_row(g, rx.batch, gstep)))
		return CCV_NNC_EXEC_INVALID;
	if (c && (kind_of(c) != kind || !per_row(c, rx.batch, cstep)))
		return CCV_NNC_EXEC_INVALID;
	LossArg p = loss_arg(cmd, OP, 0, rx);
	p.xs = rx.pitch, p.bs = ry.pitch, p.os = h0 ? r0.pitch : 0, p.o2s = h1 ? r1.pitch : 0, p.gstep = gstep, p.cstep = cstep;
	const LossPlan plan = {};
	const LossCall k = { data_of(g), x->data.u8, y->data.u8, data_of(c), data_of(h0), data_of(h1), 0 };
	return run_loss<OP>(stream_of(stream_context), kind, kind_of(y), 0, k, p, plan) ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

} // namespace

REGISTER_SM100(CCV_NNC_BINARY_CROSSENTROPY_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_forw<L_BCE>); }
REGISTER_SM100(CCV_NNC_BINARY_CROSSENTROPY_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_back<L_BCE>); }
REGISTER_SM100(CCV_NNC_SIGMOID_BINARY_CROSSENTROPY_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_forw<L_SBCE>); }
REGISTER_SM100(CCV_NNC_SIGMOID_BINARY_CROSSENTROPY_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_back<L_SBCE>); }
REGISTER_SM100(CCV_NNC_MSE_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_forw<L_MSE>); }
REGISTER_SM100(CCV_NNC_MSE_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_back<L_MSE>); }
REGISTER_SM100(CCV_NNC_SMOOTH_L1_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_forw<L_SL1>); }
REGISTER_SM100(CCV_NNC_SMOOTH_L1_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF, 1, exec_loss_back<L_SL1>); }
