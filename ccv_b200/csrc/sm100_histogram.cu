// sm100_histogram.cu -- HISTOGRAM_FORWARD / _BACKWARD on fp32, bf16 and fp16 tensors.  Semantics are CPU_REF's
// (lib/nnc/cmd/histogram/ccv_nnc_histogram_cpu_ref.c of the reference; DESIGN.md §2 restates them).  Inputs (a, [bounds]), outputs
// (b, [s]): b is a packed int32 tensor of bin counts, zeroed and then counted whatever CCV_NNC_ACCUMULATE_OUTPUT says; s, when given,
// receives (min, max, (float)sum, (float)sum of squares) of a.  16-bit values are widened exactly; bounds and statistics stay fp32.
//
//   EVEN    NaN -> b[bins + 2]; v < min -> b[0]; v >= max -> b[bins + 1]; else clamp((int)((v - min) * range) + 1, 1, bins), range =
//           (float)bins / (max - min), each operation rounded on its own; a product outside int range (or NaN) converts to INT_MIN as
//           x86-64's cvttss2si does, which the clamp sends to bin 1.
//   LOG     NaN -> b[2u + 1]; v >= max -> b[2u]; v <= -max -> b[0]; -min < v < min -> b[u]; else idx = ceilf(logf(|v| min_inv) log_base),
//           u + idx or u - idx by the sign of v, clamped to [0, 2u].  log_base, u and min_inv are computed on the host as CPU_REF does.
//           The bins are those of the correctly rounded logf: the device's logf (1 ulp) decides every element whose scaled logarithm is
//           not within 2^-19 (relative) of an integer; those few are recomputed from (float)log((double)y).
//   BINS    NaN -> b[n + 1]; else CPU_REF's own _upper_bound over the n bounds (the same midpoints, the same `v < bounds[mid]`), so
//           unsorted, repeated and NaN bounds give its bins too.
//
// Statistics.  min / max are the scans m = m < v ? m : v and m = m > v ? m : v from the first element in the view's row-major order.
// A NaN sets m to NaN and the next element replaces it, so the result is the last element when that is NaN, and otherwise the extreme
// of the elements after the last NaN, where of equal values (+0 / -0) the later one wins.  That is what each CTA computes for its chunk
// of consecutive elements: the index and value of its last NaN, and the extreme of the elements after it together with its index.  The
// finalize kernel keeps the elements after the last NaN of the whole tensor and takes the extreme with the same tie rule.  sum and sum
// of squares are double accumulations of v and of (float)(v * v), in a fixed order (per thread, then fixed shuffle and CTA trees), so
// two runs give the same bits.
//
// Launches: a memset of b, one counting pass over a, and (only when s is given) one single-CTA finalize.  Counts go to per-CTA shared
// memory when the bins fit (HIST_SHARED_WORDS), with increments aggregated per warp over lanes of the same bin (__match_any_sync), and
// are added to b at the end; otherwise straight to b with the same aggregated integer atomics.  Integer counts are exact in any order.
// The per-CTA statistic slots are one workspace request made before the first launch.
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <climits>
#include <cmath>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

using namespace sm100;

namespace {

constexpr int HIST_THREADS = 256;
constexpr int HIST_CTAS_PER_SM = 4;
// A CTA's static and dynamic shared memory together stay within the 48 KB a launch may use without opting in: HIST_STATIC_BYTES
// covers the static part (the per-warp reduction slots, checked against sizeof(Acc) below), and the rest holds counts and bounds.
constexpr int HIST_STATIC_BYTES = 1024;
constexpr int HIST_SHARED_WORDS = (48 * 1024 - HIST_STATIC_BYTES) / 4;
constexpr int FINAL_THREADS = 1024;

struct HistParams {
	int nbins; // counts the rule addresses: EVEN bins + 3, LOG 2u + 2, BINS n + 2 (the last one is NaN's)
	int bins;  // EVEN
	float min, max, range; // EVEN, LOG (range: EVEN only)
	int upper; // LOG: u
	float min_inv, log_base; // LOG
	const float* bounds; // BINS, in global memory
	int nbounds;
};

// the view of a in row-major order, adjacent packed dimensions merged
struct HistView {
	long long count;
	int nd;
	long long dim[CCV_NNC_MAX_DIM_ALLOC];
	long long stride[CCV_NNC_MAX_DIM_ALLOC];
};

// what a chunk of consecutive elements contributes to the statistics (see the head of the file); index -1: none
struct StatSlot {
	long long last_nan;
	long long imin, imax;
	double sum, sq;
	float nan_v, vmin, vmax;
};

// x86-64 cvttss2si: truncation toward zero, INT_MIN for NaN and anything outside int range
__device__ __forceinline__ int cvtt(const float t) { return (t >= -2147483648.f && t < 2147483648.f) ? __float2int_rz(t) : INT_MIN; }

template <int TYPE>
__device__ __forceinline__ int bin_of(const float v, const HistParams& p, const float* const bounds)
{
	if (isnan(v))
		return p.nbins - 1;
	if (TYPE == CCV_NNC_HISTOGRAM_EVEN)
	{
		if (v < p.min)
			return 0;
		if (v >= p.max)
			return p.bins + 1;
		const int i = (int)((unsigned)cvtt(__fmul_rn(__fsub_rn(v, p.min), p.range)) + 1u);
		return min(max(i, 1), p.bins);
	} else if (TYPE == CCV_NNC_HISTOGRAM_LOGARITHMIC) {
		const int u = p.upper;
		if (v >= p.max)
			return 2 * u;
		if (v <= -p.max)
			return 0;
		if (v < p.min && v > -p.min)
			return u;
		const float y = __fmul_rn(fabsf(v), p.min_inv);
		float t = __fmul_rn(logf(y), p.log_base);
		if (fabsf(__fsub_rn(t, rintf(t))) <= __fmul_rn(fmaxf(fabsf(t), 1.f), 0x1p-19f))
			t = __fmul_rn((float)log((double)y), p.log_base); // near a bin edge: the correctly rounded logarithm decides
		const int idx = cvtt(ceilf(t));
		const int i = v > 0 ? (int)((unsigned)u + (unsigned)idx) : (int)((unsigned)u - (unsigned)idx);
		return min(max(i, 0), 2 * u);
	} else {
		int hi = p.nbounds, lo = -1;
		while (lo + 1 < hi)
		{
			const int mid = ((hi - lo) >> 1) + lo;
			if (v < bounds[mid])
				hi = mid;
			else
				lo = mid;
		}
		return hi;
	}
}

// one increment per group of lanes that hit the same bin.  Every lane of the warp calls this (the loops below keep the warp's trip
// count uniform); a lane without an element passes bin -1 and adds nothing.
__device__ __forceinline__ void count_bin(int* const cnt, const int bin)
{
	const unsigned peers = __match_any_sync(0xffffffffu, bin);
	if (bin >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1)
		atomicAdd(cnt + bin, __popc(peers));
}

struct Acc {
	long long last_nan, imin, imax;
	double sum, sq;
	float nan_v, vmin, vmax;

	__device__ void init()
	{
		last_nan = imin = imax = -1;
		sum = sq = 0;
		nan_v = vmin = vmax = 0.f;
	}
	// elements arrive in increasing index: a later equal value replaces the held one, as the scans do
	__device__ __forceinline__ void extremes(const float x, const long long i)
	{
		if (imin < 0 || !(vmin < x))
			vmin = x, imin = i;
		if (imax < 0 || !(vmax > x))
			vmax = x, imax = i;
	}
	__device__ __forceinline__ void add(const float x, const long long i)
	{
		if (isnan(x))
			last_nan = i, nan_v = x, imin = imax = -1;
		else
			extremes(x, i);
		sum += (double)x;
		sq += (double)__fmul_rn(x, x);
	}
};

// extremes of two disjoint sets: the smaller (larger) value, of equal ones the later element
__device__ __forceinline__ void merge_min(float& v, long long& i, const float w, const long long j)
{
	if (j < 0)
		return;
	if (i < 0 || w < v || (!(v < w) && j > i))
		v = w, i = j;
}
__device__ __forceinline__ void merge_max(float& v, long long& i, const float w, const long long j)
{
	if (j < 0)
		return;
	if (i < 0 || w > v || (!(v > w) && j > i))
		v = w, i = j;
}
static_assert(sizeof(Acc) * (HIST_THREADS / 32) + sizeof(long long) + 16 <= HIST_STATIC_BYTES, "histogram_kernel's static shared memory");

__device__ __forceinline__ void merge(Acc& a, const Acc& b, const bool sums)
{
	if (b.last_nan > a.last_nan)
		a.last_nan = b.last_nan, a.nan_v = b.nan_v;
	merge_min(a.vmin, a.imin, b.vmin, b.imin);
	merge_max(a.vmax, a.imax, b.vmax, b.imax);
	if (sums)
		a.sum += b.sum, a.sq += b.sq;
}
__device__ __forceinline__ Acc shfl_down(const Acc& a, const int d)
{
	Acc b;
	b.last_nan = __shfl_down_sync(0xffffffffu, a.last_nan, d);
	b.imin = __shfl_down_sync(0xffffffffu, a.imin, d);
	b.imax = __shfl_down_sync(0xffffffffu, a.imax, d);
	b.sum = __shfl_down_sync(0xffffffffu, a.sum, d);
	b.sq = __shfl_down_sync(0xffffffffu, a.sq, d);
	b.nan_v = __shfl_down_sync(0xffffffffu, a.nan_v, d);
	b.vmin = __shfl_down_sync(0xffffffffu, a.vmin, d);
	b.vmax = __shfl_down_sync(0xffffffffu, a.vmax, d);
	return b;
}
// fixed-order reduction over the CTA; the result is valid in thread 0.  `red` holds one Acc per warp.
__device__ Acc block_reduce(Acc a, Acc* const red, const bool sums)
{
	for (int d = 16; d > 0; d >>= 1)
	{
		const Acc b = shfl_down(a, d);
		merge(a, b, sums);
	}
	const int warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
	__syncthreads();
	if ((threadIdx.x & 31) == 0)
		red[warp] = a;
	__syncthreads();
	if (threadIdx.x == 0)
		for (int w = 1; w < warps; w++)
			merge(a, red[w], sums);
	return a;
}

template <typename T, int LAYOUT>
__device__ __forceinline__ float load1(const T* const a, const HistView& v, long long i)
{
	if (LAYOUT == 2)
	{
		long long off = 0;
		for (int d = v.nd - 1; d > 0; d--)
		{
			off += (i % v.dim[d]) * v.stride[d];
			i /= v.dim[d];
		}
		return ldf(a + off + i * v.stride[0]);
	}
	return ldf(a + i);
}

// LAYOUT 0: packed, 16-byte aligned, chunk a multiple of the vector width; 1: packed; 2: strided.  Each CTA owns the elements
// [blockIdx.x chunk, (blockIdx.x + 1) chunk) and each thread visits its elements in increasing index.
template <typename T, int TYPE, int LAYOUT>
__global__ void __launch_bounds__(HIST_THREADS, HIST_CTAS_PER_SM) histogram_kernel(const T* __restrict__ a, const HistView v, const HistParams p, int* __restrict__ b, const int shared_bins, const int shared_bounds, StatSlot* __restrict__ slots, const long long chunk)
{
	extern __shared__ int smem[];
	__shared__ Acc red[HIST_THREADS / 32];
	__shared__ long long chunk_nan;
	int* const cnt = shared_bins ? smem : b;
	const float* bounds = p.bounds;
	if (shared_bins)
		for (int i = threadIdx.x; i < p.nbins; i += blockDim.x)
			smem[i] = 0;
	if (shared_bounds)
	{
		float* const sb = reinterpret_cast<float*>(smem + (shared_bins ? p.nbins : 0));
		for (int i = threadIdx.x; i < p.nbounds; i += blockDim.x)
			sb[i] = p.bounds[i];
		bounds = sb;
	}
	__syncthreads();
	const long long s = blockIdx.x * chunk, e = min(s + chunk, v.count);
	const bool stats = slots != 0;
	Acc acc;
	acc.init();
	// the trip counts depend only on the tile start, so every lane of a warp reaches each count_bin
	if (LAYOUT == 0)
	{
		constexpr int W = Vec16<T>::W;
		for (long long tile = s; tile < e; tile += (long long)blockDim.x * W)
		{
			const long long base = tile + (long long)threadIdx.x * W;
			float x[W];
			if (base + W <= e)
				ldv(a + base, x);
			else
#pragma unroll
				for (int k = 0; k < W; k++)
					x[k] = base + k < e ? ldf(a + base + k) : 0.f;
#pragma unroll
			for (int k = 0; k < W; k++)
			{
				const bool in = base + k < e;
				if (in && stats)
					acc.add(x[k], base + k);
				count_bin(cnt, in ? bin_of<TYPE>(x[k], p, bounds) : -1);
			}
		}
	} else {
		for (long long tile = s; tile < e; tile += blockDim.x)
		{
			const long long i = tile + threadIdx.x;
			const bool in = i < e;
			const float x = in ? load1<T, LAYOUT>(a, v, i) : 0.f;
			if (in && stats)
				acc.add(x, i);
			count_bin(cnt, in ? bin_of<TYPE>(x, p, bounds) : -1);
		}
	}
	if (stats)
	{
		Acc r = block_reduce(acc, red, true);
		if (threadIdx.x == 0)
			chunk_nan = r.last_nan;
		__syncthreads();
		const long long last = chunk_nan;
		if (last >= 0)
		{
			// the chunk holds a NaN: its extremes come from the elements after the chunk's last NaN only
			Acc t;
			t.init();
			for (long long i = last + 1 + threadIdx.x; i < e; i += blockDim.x)
				t.extremes(load1<T, LAYOUT == 2 ? 2 : 1>(a, v, i), i);
			const Acc q = block_reduce(t, red, false);
			r.imin = q.imin, r.vmin = q.vmin, r.imax = q.imax, r.vmax = q.vmax;
		}
		if (threadIdx.x == 0)
		{
			StatSlot o;
			o.last_nan = r.last_nan, o.nan_v = r.nan_v;
			o.imin = r.imin, o.vmin = r.vmin, o.imax = r.imax, o.vmax = r.vmax;
			o.sum = r.sum, o.sq = r.sq;
			slots[blockIdx.x] = o;
		}
	}
	if (shared_bins)
	{
		__syncthreads();
		for (int i = threadIdx.x; i < p.nbins; i += blockDim.x)
			if (smem[i])
				atomicAdd(b + i, smem[i]);
	}
}

// one CTA: combine the slots in CTA order and store (min, max, (float)sum, (float)sum of squares)
__global__ void __launch_bounds__(FINAL_THREADS) histogram_stats_kernel(const StatSlot* __restrict__ slots, const int nslots, const long long count, float* __restrict__ s)
{
	__shared__ Acc red[FINAL_THREADS / 32];
	__shared__ long long last_nan;
	Acc a;
	a.init();
	// every thread's slots are consecutive, so the sums are combined in one fixed order
	const int per = (nslots + FINAL_THREADS - 1) / FINAL_THREADS;
	for (int c = threadIdx.x * per; c < min(nslots, (int)(threadIdx.x + 1) * per); c++)
	{
		Acc b;
		b.last_nan = slots[c].last_nan, b.nan_v = slots[c].nan_v;
		b.imin = slots[c].imin, b.vmin = slots[c].vmin, b.imax = slots[c].imax, b.vmax = slots[c].vmax;
		b.sum = slots[c].sum, b.sq = slots[c].sq;
		merge(a, b, true);
	}
	Acc r = block_reduce(a, red, true);
	if (threadIdx.x == 0)
		last_nan = r.last_nan;
	__syncthreads();
	// only the extremes after the tensor's last NaN count
	Acc t;
	t.init();
	for (int c = threadIdx.x * per; c < min(nslots, (int)(threadIdx.x + 1) * per); c++)
	{
		if (slots[c].imin > last_nan)
			merge_min(t.vmin, t.imin, slots[c].vmin, slots[c].imin);
		if (slots[c].imax > last_nan)
			merge_max(t.vmax, t.imax, slots[c].vmax, slots[c].imax);
	}
	const Acc q = block_reduce(t, red, false);
	if (threadIdx.x == 0)
	{
		const bool nan_last = r.last_nan == count - 1;
		s[0] = nan_last ? r.nan_v : q.vmin;
		s[1] = nan_last ? r.nan_v : q.vmax;
		s[2] = (float)r.sum;
		s[3] = (float)r.sq;
	}
}

// ------------------------------------------------------------------------------------------------ host side
bool packed(const ccv_nnc_tensor_t* const t) { return t && CCV_IS_TENSOR_CONTIGUOUS(t) && t->data.u8; }

// element kind of a: 0 fp32, 1 bf16, 2 fp16; -1 otherwise (CCV_GET_DATA_TYPE keeps the CCV_QX bit, so palettized tensors are refused)

HistView view_of(const ccv_nnc_tensor_t* const t)
{
	HistView v;
	memset(&v, 0, sizeof(v));
	int nd = 0;
	while (nd < CCV_NNC_MAX_DIM_ALLOC && t->info.dim[nd] > 0)
		nd++;
	long long dim[CCV_NNC_MAX_DIM_ALLOC], stride[CCV_NNC_MAX_DIM_ALLOC];
	long long packed_stride = 1;
	for (int i = nd - 1; i >= 0; i--)
	{
		dim[i] = t->info.dim[i];
		stride[i] = CCV_IS_TENSOR_VIEW(t) ? ((const ccv_nnc_tensor_view_t*)t)->stride[i] : packed_stride;
		packed_stride *= dim[i];
	}
	v.count = packed_stride;
	// merge a dimension into the next inner one when it steps over exactly that one's extent; size-1 dimensions vanish
	for (int i = 0; i < nd; i++)
	{
		if (dim[i] == 1)
			continue;
		if (v.nd > 0 && v.stride[v.nd - 1] == stride[i] * dim[i])
		{
			v.dim[v.nd - 1] *= dim[i];
			v.stride[v.nd - 1] = stride[i];
		} else
			v.dim[v.nd] = dim[i], v.stride[v.nd] = stride[i], v.nd++;
	}
	if (v.nd == 0)
		v.dim[0] = 1, v.stride[0] = 1, v.nd = 1;
	return v;
}

template <typename T, int TYPE>
int launch(const T* a, const HistView& v, const HistParams& p, int* b, StatSlot* slots, const int grid, const long long chunk, const int shared_bins, const int shared_bounds, const int layout, cudaStream_t s)
{
	const size_t shm = ((shared_bins ? p.nbins : 0) + (shared_bounds ? p.nbounds : 0)) * sizeof(int);
	if (layout == 0)
		histogram_kernel<T, TYPE, 0><<<grid, HIST_THREADS, shm, s>>>(a, v, p, b, shared_bins, shared_bounds, slots, chunk);
	else if (layout == 1)
		histogram_kernel<T, TYPE, 1><<<grid, HIST_THREADS, shm, s>>>(a, v, p, b, shared_bins, shared_bounds, slots, chunk);
	else
		histogram_kernel<T, TYPE, 2><<<grid, HIST_THREADS, shm, s>>>(a, v, p, b, shared_bins, shared_bounds, slots, chunk);
	return launched("histogram");
}

template <typename T>
int launch_type(const int type, const T* a, const HistView& v, const HistParams& p, int* b, StatSlot* slots, const int grid, const long long chunk, const int shared_bins, const int shared_bounds, const int layout, cudaStream_t s)
{
	if (type == CCV_NNC_HISTOGRAM_EVEN)
		return launch<T, CCV_NNC_HISTOGRAM_EVEN>(a, v, p, b, slots, grid, chunk, shared_bins, shared_bounds, layout, s);
	if (type == CCV_NNC_HISTOGRAM_LOGARITHMIC)
		return launch<T, CCV_NNC_HISTOGRAM_LOGARITHMIC>(a, v, p, b, slots, grid, chunk, shared_bins, shared_bounds, layout, s);
	return launch<T, CCV_NNC_HISTOGRAM_BINS>(a, v, p, b, slots, grid, chunk, shared_bins, shared_bounds, layout, s);
}

// inputs (a, [bounds]) -> outputs (b, [s]).  Everything is checked before the first launch; a refused call returns INVALID and
// leaves the outputs untouched.
int exec_histogram_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	if (input_size < 1 || output_size < 1 || !inputs || !outputs || !inputs[0] || !inputs[0]->data.u8 || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const a = inputs[0];
	ccv_nnc_tensor_t* const b = outputs[0];
	ccv_nnc_tensor_t* const st = output_size > 1 ? outputs[1] : 0;
	const int kind = kind_of(a);
	const long long count = nd_of(a) ? (long long)count_of(a) : 0;
	if (kind < 0 || count < 1 || count > INT_MAX)
		return CCV_NNC_EXEC_INVALID;
	if (!packed(b) || b->info.datatype != CCV_32S)
		return CCV_NNC_EXEC_INVALID;
	const long long bcount = (long long)count_of(b);
	if (st && (!packed(st) || st->info.datatype != CCV_32F || count_of(st) < 4))
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_cmd_param_t& info = cmd.info;
	HistParams p;
	memset(&p, 0, sizeof(p));
	const int type = info.histogram.type;
	if (type == CCV_NNC_HISTOGRAM_EVEN)
	{
		const float min = info.histogram.min, max = info.histogram.max;
		if (!(max > min) || info.histogram.bins < 1 || info.histogram.bins > INT_MAX - 3 || bcount != (long long)info.histogram.bins + 3)
			return CCV_NNC_EXEC_INVALID;
		p.bins = info.histogram.bins, p.min = min, p.max = max;
		p.range = (float)p.bins / (max - min);
		p.nbins = p.bins + 3;
	} else if (type == CCV_NNC_HISTOGRAM_LOGARITHMIC) {
		const float min = info.histogram.min, max = info.histogram.max, rate = info.histogram.rate;
		if (!(min > 0) || !(max > min) || !(rate > 1))
			return CCV_NNC_EXEC_INVALID;
		const float log_base = 1.0 / logf(rate);
		const float min_inv = 1.0 / min;
		const float top = max * min_inv;
		if (!std::isfinite(top) || !std::isfinite(log_base))
			return CCV_NNC_EXEC_INVALID;
		const float upper = ceilf(logf(max / min) * log_base);
		if (!(upper >= 0) || upper > (float)((INT_MAX - 2) / 2))
			return CCV_NNC_EXEC_INVALID;
		p.upper = (int)upper, p.min = min, p.max = max, p.min_inv = min_inv, p.log_base = log_base;
		p.nbins = 2 * p.upper + 2;
		if (bcount < p.nbins)
			return CCV_NNC_EXEC_INVALID;
	} else if (type == CCV_NNC_HISTOGRAM_BINS) {
		const ccv_nnc_tensor_t* const h = input_size > 1 ? inputs[1] : 0;
		if (!packed(h) || h->info.datatype != CCV_32F || CCV_TENSOR_GET_MEMORY(h->info.type) != CCV_TENSOR_GPU_MEMORY)
			return CCV_NNC_EXEC_INVALID;
		const long long n = nd_of(h) ? (long long)count_of(h) : 0;
		if (n < 1 || n > INT_MAX - 2 || bcount != n + 2)
			return CCV_NNC_EXEC_INVALID;
		p.bounds = h->data.f32, p.nbounds = (int)n, p.nbins = (int)n + 2;
	} else
		return CCV_NNC_EXEC_INVALID;
	const HistView v = view_of(a);
	const bool contiguous = v.nd == 1 && v.stride[0] == 1;
	const int W = kind == 0 ? 4 : 8;
	const int layout = !contiguous ? 2 : ((uintptr_t)a->data.u8 & 15) == 0 ? 0 : 1;
	// consecutive chunks of whole vectors, at most HIST_CTAS_PER_SM CTAs per SM
	const long long tile = (long long)HIST_THREADS * W;
	long long grid = (count + tile - 1) / tile;
	if (grid > (long long)sm_count() * HIST_CTAS_PER_SM)
		grid = (long long)sm_count() * HIST_CTAS_PER_SM;
	long long chunk = (count + grid - 1) / grid;
	chunk = (chunk + W - 1) / W * W;
	grid = (count + chunk - 1) / chunk;
	const int shared_bins = p.nbins <= HIST_SHARED_WORDS;
	const int shared_bounds = type == CCV_NNC_HISTOGRAM_BINS && p.nbounds <= HIST_SHARED_WORDS - (shared_bins ? p.nbins : 0);
	StatSlot* slots = 0;
	if (st)
	{
		slots = (StatSlot*)ccv_nnc_stream_context_get_workspace(stream_context, grid * sizeof(StatSlot), CCV_TENSOR_GPU_MEMORY);
		if (!slots)
			return CCV_NNC_EXEC_OOM;
	}
	cudaStream_t s = (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context);
	cudaMemsetAsync(b->data.i32, 0, bcount * sizeof(int), s);
	if (launched("histogram_zero"))
		return CCV_NNC_EXEC_INVALID;
	int rc;
	if (kind == 0)
		rc = launch_type<float>(type, a->data.f32, v, p, b->data.i32, slots, (int)grid, chunk, shared_bins, shared_bounds, layout, s);
	else if (kind == 1)
		rc = launch_type<__nv_bfloat16>(type, (const __nv_bfloat16*)a->data.u8, v, p, b->data.i32, slots, (int)grid, chunk, shared_bins, shared_bounds, layout, s);
	else
		rc = launch_type<__half>(type, (const __half*)a->data.u8, v, p, b->data.i32, slots, (int)grid, chunk, shared_bins, shared_bounds, layout, s);
	if (rc)
		return CCV_NNC_EXEC_INVALID;
	if (st)
	{
		histogram_stats_kernel<<<1, FINAL_THREADS, 0, s>>>(slots, (int)grid, count, st->data.f32);
		if (launched("histogram_stats"))
			return CCV_NNC_EXEC_INVALID;
	}
	return CCV_NNC_EXEC_SUCCESS;
}

} // namespace

REGISTER_SM100(CCV_NNC_HISTOGRAM_FORWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_histogram_forw); }
// the reference has no histogram gradient (_ccv_nnc_histogram_back returns CCV_NNC_EXEC_INVALID)
REGISTER_SM100(CCV_NNC_HISTOGRAM_BACKWARD) { fill(registry, ALL_FORMATS, CCV_32F | CCV_16F | CCV_16BF | CCV_32S, 1, exec_invalid); }
