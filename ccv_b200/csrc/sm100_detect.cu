// sm100_detect.cu -- ROI_ALIGN and NMS (forward / backward), the two commands of a two-stage detector's head.  Semantics are CPU_REF's
// (paths relative to lib/nnc/cmd of the reference), quirks included (DESIGN.md §2):
//   roi/ccv_nnc_roi_align_cpu_ref.c   c[n, r, j] = inv * sum over the bin's live samples (y, x) of a00 c00 + a01 c01 + a10 c10 + a11 c11,
//                                     where bin i = r + start_h (CPU_REF writes the first live bin row to output row 0) and
//                                     inv = 1.0 / (live rows * live columns); backward: o[pixel] += (g c) inv over n, i, j, y, x, corners
//   nms/ccv_nnc_nms_cpu_ref.c         rows (score, x, y, w, h) sorted by score, greedy suppression at IoU >= threshold, kept rows first
//
// ROI_ALIGN.  Features are fp32, bf16 or fp16 in NHWC or NCHW (any strides: the kernels take an element step per axis), ROIs fp32 rows
// (x, y, w, h) normalised to the map, as a packed [4] / [k, 4] tensor or a view with unit column step.  A ROI's sample positions along an
// axis are ay(k) = (float)(roi + (k + 0.5) scale - 0.5) (double, as the reference's 0.5 literals make it), k < bin * pool.  They are
// non-decreasing in k, so the live samples (-1 <= ay < size) are one index range [lo, hi), found by a bounded search, and so are the
// samples that touch one pixel row (py - 1 <= ay < py + 1).  Every product and sum is rounded on its own (no FMA contraction): fp32
// results equal CPU_REF's source order bit for bit, 16-bit ones that arithmetic on the widened inputs, rounded once on store.
//   forward:  one CTA per (ROI, output row); threads along (column, channel).  No workspace.
//   backward: a gather, pixel-stationary: a warp owns RB_PIX pixels of one image and 32 * RB_CPL channels (lane c, c + 32, ...), a CTA
//             stages the per-ROI axis parameters of RB_CHUNK ROIs at a time in shared memory, and each warp skips every ROI whose live
//             sample span misses its pixel.  Each pixel adds its terms in CPU_REF's order (ROI ascending, bins, samples, corners 00, 01,
//             10, 11).  No atomics and no workspace: two runs give the same bits.
// A ROI with a non-finite value, or with more than ROI_MAX_BINS_PER_PIXEL * size samples per bin (or ROI_MAX_SAMPLES samples in all)
// along an axis, is read as an empty ROI
// (zeros): the coordinates live on the GPU, so exec cannot refuse them, and CPU_REF is undefined there.
//
// NMS.  fp32 [m, 5] or [n, m, 5] (row and batch steps from views), d = 5 only.  Per batch item, in one launch per phase:
//   rank:   the stable descending rank of each row's score on the order-preserving 32-bit key (-0 folded onto +0, NaNs ordered by their
//           bits): greater keys plus equal keys at lower index.  A permutation for every input.  Rows are scattered to the workspace.
//   mask:   the upper triangle of "IoU(i, j) >= threshold" for sorted i < j, 64-bit words, CPU_REF's fp32 formula term by term.
//   sweep:  one CTA per item holds the "removed" bit vector in shared memory, resolves each 64-row block serially and ORs its kept rows'
//           masks into the later words; then it writes the kept rows in score order, the tail with c = -1 and score -FLT_MAX.  No CTA
//           waits on another CTA.
// The workspace is (5 + 1) * 4 * m + 8 * m * ceil(m / 64) bytes per item; the batch runs in groups that fit NMS_WORKSPACE_CAP.
// Backward: one CTA per item zeroes the output and scatters g's rows to c's indices up to the first negative one.
#include "sm100_cmd.h"
#include "sm100_elem.cuh"
#include <cuda_runtime.h>
#include <float.h>
#include <string.h>

using namespace sm100;

namespace {

constexpr int ROI_MAX_BINS_PER_PIXEL = 4;  // per axis: ceil(roi_size / pool) <= 4 * size, else the ROI is read as empty
constexpr int ROI_MAX_SAMPLES = 1 << 30;   // per axis: bin * pool <= 2^30, so sample indices stay ints
constexpr int RF_THREADS = 256;
constexpr int RB_PIX = 4, RB_CPL = 8, RB_WARPS = 8, RB_CHUNK = 128;
constexpr int NMS_THREADS = 256;
constexpr size_t NMS_WORKSPACE_CAP = (size_t)1 << 30;

// ------------------------------------------------------------------------------------------------ ROI_ALIGN
// one axis of one ROI: sample k sits at ay(k); live samples are [lo, hi); bins of `bin` samples, `pool` of them
struct RoiAxis {
	float roi, scale;
	int bin, n, lo, hi; // n = bin * pool samples; bin == 0: empty ROI
};

__device__ __forceinline__ float roi_pos(const float roi, const float scale, const int k)
{
	return __double2float_rn(__dsub_rn(__dadd_rn((double)roi, __dmul_rn(__dadd_rn((double)k, 0.5), (double)scale)), 0.5));
}
// the first k in [lo, hi] with roi_pos(k) >= t (hi when none): an estimate, then unit steps (roi_pos is non-decreasing in k, so the
// result is exact; the steps are bounded by hi - lo)
__device__ __forceinline__ int roi_lower_bound(const RoiAxis& ax, const float t, const int lo, const int hi)
{
	float e = __fsub_rn(__fdiv_rn(__fsub_rn(__fadd_rn(t, 0.5f), ax.roi), ax.scale), 0.5f);
	e = e != e ? (float)lo : fminf(fmaxf(e, (float)lo), (float)hi);
	int k = min(max((int)e, lo), hi); // (float)hi may round above hi once hi > 2^24
	while (k > lo && roi_pos(ax.roi, ax.scale, k - 1) >= t)
		k--;
	while (k < hi && roi_pos(ax.roi, ax.scale, k) < t)
		k++;
	return k;
}
// _ccv_nnc_bilinear_coeffs (roi/ccv_nnc_roi_align_cpu_ref.c:18-99) for one axis: v = normalised start, vs = normalised size
__device__ __forceinline__ RoiAxis roi_axis(const float v, const float vs, const int size, const int pool)
{
	RoiAxis ax;
	ax.roi = __fmul_rn(v, (float)size);
	const float rs = __fmul_rn(vs, (float)size);
	const float bins = ceilf(__fdiv_rn(rs, (float)pool));
	ax.bin = 0, ax.n = 0, ax.lo = 0, ax.hi = 0, ax.scale = 0.f;
	if (!isfinite(ax.roi) || !isfinite(rs) || !(bins >= 1.f) || bins > (float)ROI_MAX_BINS_PER_PIXEL * (float)size || (double)bins * pool > (double)ROI_MAX_SAMPLES)
		return ax;
	ax.bin = (int)bins;
	ax.n = ax.bin * pool;
	ax.scale = __fdiv_rn(rs, (float)ax.n);
	ax.lo = roi_lower_bound(ax, -1.f, 0, ax.n);
	ax.hi = roi_lower_bound(ax, (float)size, ax.lo, ax.n);
	return ax;
}
// live samples in bin i
__device__ __forceinline__ int roi_live(const RoiAxis& ax, const int i) { return max(0, min(ax.hi, (i + 1) * ax.bin) - max(ax.lo, i * ax.bin)); }
// sample k: corner rows i0, i1 and weight r (CPU_REF: iy = floorf(ay), r = ay - iy, i0 / i1 = iy / iy + 1 clamped; live samples only)
__device__ __forceinline__ void roi_sample(const RoiAxis& ax, const int k, const int size, int& i0, int& i1, float& r)
{
	const float a = roi_pos(ax.roi, ax.scale, k);
	const int i = (int)floorf(a);
	r = __fsub_rn(a, (float)i);
	i0 = max(i, 0), i1 = min(i + 1, size - 1);
}

struct RoiArg {
	int h, w, ch, pool_h, pool_w;
	int a_n, b_n, n; // n: output ROIs (forward) / g's ROIs (backward)
	long long bstep; // element step between ROIs of b (0: one ROI)
	long long fn, fy, fx, fc; // the feature map (a / o): element steps per axis
	long long pn, py, px, pc; // the pooled tensor (c / g)
};

template <typename T>
__global__ void __launch_bounds__(RF_THREADS) roi_align_fwd_kernel(const T* __restrict__ a, const float* __restrict__ b, T* __restrict__ c, const RoiArg p)
{
	const int n = blockIdx.x, r = blockIdx.y;
	const float* const box = b + (n % p.b_n) * p.bstep;
	const RoiAxis ay = roi_axis(box[1], box[3], p.h, p.pool_h), ax = roi_axis(box[0], box[2], p.w, p.pool_w);
	const bool live = ay.bin > 0 && ax.bin > 0 && ay.lo < ay.hi && ax.lo < ax.hi;
	const int start_h = live ? ay.lo / ay.bin : p.pool_h, end_h = live ? (ay.hi - 1) / ay.bin + 1 : 0;
	const int start_w = live ? ax.lo / ax.bin : p.pool_w, end_w = live ? (ax.hi - 1) / ax.bin + 1 : 0;
	const int i = r + start_h; // CPU_REF writes bin rows [start_h, end_h) to output rows 0, 1, ...
	const T* const an = a + (long long)(n % p.a_n) * p.fn;
	T* const cn = c + (long long)n * p.pn + (long long)r * p.py;
	const int total = p.pool_w * p.ch;
	for (int t = threadIdx.x; t < total; t += RF_THREADS)
	{
		const int j = t / p.ch, k = t - j * p.ch;
		float acc = 0.f;
		if (i < end_h && j >= start_w && j < end_w)
		{
			const T* const ak = an + k * p.fc;
			const int y1 = min(ay.hi, (i + 1) * ay.bin), x1 = min(ax.hi, (j + 1) * ax.bin);
			for (int y = max(ay.lo, i * ay.bin); y < y1; y++)
			{
				int iy0, iy1;
				float ry;
				roi_sample(ay, y, p.h, iy0, iy1, ry);
				const T* const r0 = ak + iy0 * p.fy;
				const T* const r1 = ak + iy1 * p.fy;
				for (int x = max(ax.lo, j * ax.bin); x < x1; x++)
				{
					int ix0, ix1;
					float rx;
					roi_sample(ax, x, p.w, ix0, ix1, rx);
					const float c00 = __fmul_rn(__fsub_rn(1.f, ry), __fsub_rn(1.f, rx)), c01 = __fmul_rn(__fsub_rn(1.f, ry), rx);
					const float c10 = __fmul_rn(ry, __fsub_rn(1.f, rx)), c11 = __fmul_rn(ry, rx);
					const float a00 = ldf(r0 + ix0 * p.fx), a01 = ldf(r0 + ix1 * p.fx), a10 = ldf(r1 + ix0 * p.fx), a11 = ldf(r1 + ix1 * p.fx);
					const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a00, c00), __fmul_rn(a01, c01)), __fmul_rn(a10, c10)), __fmul_rn(a11, c11));
					acc = __fadd_rn(acc, s);
				}
			}
			const float inv = __double2float_rn(__ddiv_rn(1.0, (double)(roi_live(ay, i) * roi_live(ax, j))));
			acc = __fmul_rn(acc, inv);
		}
		stf(cn + j * p.px + k * p.pc, acc);
	}
}

// per-ROI parameters a backward CTA stages in shared memory
struct RoiStage {
	RoiAxis y, x;
	float y_first, y_last, x_first, x_last; // positions of the first / last live sample
	int n;                                  // the ROI's index in g
};

template <typename T>
__global__ void __launch_bounds__(RB_WARPS * 32) roi_align_bwd_kernel(const T* __restrict__ g, const float* __restrict__ b, T* __restrict__ o, const RoiArg p, const int o_n)
{
	__shared__ RoiStage st[RB_CHUNK];
	const int img = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int c0 = blockIdx.z * 32 * RB_CPL;
	const long long hw = (long long)p.h * p.w;
	const long long pix0 = ((long long)blockIdx.x * RB_WARPS + warp) * RB_PIX;
	float acc[RB_PIX][RB_CPL];
#pragma unroll
	for (int q = 0; q < RB_PIX; q++)
#pragma unroll
		for (int u = 0; u < RB_CPL; u++)
			acc[q][u] = 0.f;
	// ROIs of this image: n = img, img + o_n, ... < p.n
	const int rois = img < p.n ? (p.n - img + o_n - 1) / o_n : 0;
	for (int base = 0; base < rois; base += RB_CHUNK)
	{
		const int cnt = min(RB_CHUNK, rois - base);
		__syncthreads();
		for (int t = threadIdx.x; t < cnt; t += RB_WARPS * 32)
		{
			RoiStage s;
			s.n = img + (base + t) * o_n;
			const float* const box = b + (s.n % p.b_n) * p.bstep;
			s.y = roi_axis(box[1], box[3], p.h, p.pool_h), s.x = roi_axis(box[0], box[2], p.w, p.pool_w);
			const bool live = s.y.bin > 0 && s.x.bin > 0 && s.y.lo < s.y.hi && s.x.lo < s.x.hi;
			s.y_first = live ? roi_pos(s.y.roi, s.y.scale, s.y.lo) : 1.f, s.y_last = live ? roi_pos(s.y.roi, s.y.scale, s.y.hi - 1) : -1.f;
			s.x_first = live ? roi_pos(s.x.roi, s.x.scale, s.x.lo) : 1.f, s.x_last = live ? roi_pos(s.x.roi, s.x.scale, s.x.hi - 1) : -1.f;
			st[t] = s;
		}
		__syncthreads();
#pragma unroll
		for (int q = 0; q < RB_PIX; q++)
		{
			const long long pix = pix0 + q;
			if (pix >= hw)
				break;
			const int py = (int)(pix / p.w), px = (int)(pix - (long long)py * p.w);
			const float ty0 = (float)(py - 1), ty1 = (float)(py + 1), tx0 = (float)(px - 1), tx1 = (float)(px + 1);
			for (int e = 0; e < cnt; e++)
			{
				const RoiStage& s = st[e];
				// the samples touching row py have ty0 <= ay < ty1 (floor(ay) is py - 1 or py); the same for columns
				if (s.y_last < ty0 || s.y_first >= ty1 || s.x_last < tx0 || s.x_first >= tx1)
					continue;
				const int ylo = roi_lower_bound(s.y, ty0, s.y.lo, s.y.hi), yhi = roi_lower_bound(s.y, ty1, ylo, s.y.hi);
				const int xlo = roi_lower_bound(s.x, tx0, s.x.lo, s.x.hi), xhi = roi_lower_bound(s.x, tx1, xlo, s.x.hi);
				if (ylo >= yhi || xlo >= xhi)
					continue;
				const T* const gn = g + (long long)s.n * p.pn;
				for (int i = ylo / s.y.bin; i * s.y.bin < yhi; i++)
				{
					const int ly = roi_live(s.y, i);
					for (int j = xlo / s.x.bin; j * s.x.bin < xhi; j++)
					{
						const float inv = __double2float_rn(__ddiv_rn(1.0, (double)(ly * roi_live(s.x, j))));
						const T* const gz = gn + i * p.py + j * p.px;
						float gv[RB_CPL];
#pragma unroll
						for (int u = 0; u < RB_CPL; u++)
						{
							const int k = c0 + lane + 32 * u;
							gv[u] = k < p.ch ? ldf(gz + k * p.pc) : 0.f;
						}
						const int y1 = min(yhi, (i + 1) * s.y.bin), x1 = min(xhi, (j + 1) * s.x.bin);
						for (int y = max(ylo, i * s.y.bin); y < y1; y++)
						{
							int iy0, iy1;
							float ry;
							roi_sample(s.y, y, p.h, iy0, iy1, ry);
							const bool y0 = iy0 == py, y1m = iy1 == py;
							for (int x = max(xlo, j * s.x.bin); x < x1; x++)
							{
								int ix0, ix1;
								float rx;
								roi_sample(s.x, x, p.w, ix0, ix1, rx);
								const bool x0 = ix0 == px, x1m = ix1 == px;
								const float c00 = __fmul_rn(__fsub_rn(1.f, ry), __fsub_rn(1.f, rx)), c01 = __fmul_rn(__fsub_rn(1.f, ry), rx);
								const float c10 = __fmul_rn(ry, __fsub_rn(1.f, rx)), c11 = __fmul_rn(ry, rx);
#pragma unroll
								for (int u = 0; u < RB_CPL; u++)
								{
									if (y0 && x0)
										acc[q][u] = __fadd_rn(acc[q][u], __fmul_rn(__fmul_rn(gv[u], c00), inv));
									if (y0 && x1m)
										acc[q][u] = __fadd_rn(acc[q][u], __fmul_rn(__fmul_rn(gv[u], c01), inv));
									if (y1m && x0)
										acc[q][u] = __fadd_rn(acc[q][u], __fmul_rn(__fmul_rn(gv[u], c10), inv));
									if (y1m && x1m)
										acc[q][u] = __fadd_rn(acc[q][u], __fmul_rn(__fmul_rn(gv[u], c11), inv));
								}
							}
						}
					}
				}
			}
		}
	}
	if (img >= o_n)
		return;
#pragma unroll
	for (int q = 0; q < RB_PIX; q++)
	{
		const long long pix = pix0 + q;
		if (pix >= hw)
			break;
		const int py = (int)(pix / p.w), px = (int)(pix - (long long)py * p.w);
		T* const oz = o + (long long)img * p.fn + py * p.fy + px * p.fx;
#pragma unroll
		for (int u = 0; u < RB_CPL; u++)
		{
			const int k = c0 + lane + 32 * u;
			if (k < p.ch)
				stf(oz + k * p.fc, acc[q][u]);
		}
	}
}

// ------------------------------------------------------------------------------------------------ NMS
struct NmsArg {
	int m, words;              // rows per item, ceil(m / 64)
	long long an, am, bn, bm;  // element steps: a / b between items and rows
	long long cn;              // c: between items
	float thr;
};

// order-preserving key of a score: larger score, larger key; -0 folded onto +0; NaNs ordered by their bits
__device__ __forceinline__ uint32_t score_key(const float s)
{
	uint32_t u = __float_as_uint(s);
	if (u == 0x80000000u)
		u = 0;
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// rank every row of item blockIdx.y (greater keys, then equal keys at lower index) and scatter it to the sorted workspace
__global__ void __launch_bounds__(NMS_THREADS) nms_rank_kernel(const float* __restrict__ a, float* __restrict__ sorted, int* __restrict__ idx, const NmsArg p, const int item0)
{
	__shared__ uint32_t keys[NMS_THREADS * 4];
	const int item = item0 + blockIdx.y;
	const float* const an = a + item * p.an;
	const int i = blockIdx.x * NMS_THREADS + threadIdx.x;
	const uint32_t ki = i < p.m ? score_key(an[(long long)i * p.am]) : 0;
	int rank = 0;
	for (int j0 = 0; j0 < p.m; j0 += NMS_THREADS * 4)
	{
		__syncthreads();
		for (int t = threadIdx.x; t < NMS_THREADS * 4; t += NMS_THREADS)
			keys[t] = j0 + t < p.m ? score_key(an[(long long)(j0 + t) * p.am]) : 0;
		__syncthreads();
		const int jn = min(NMS_THREADS * 4, p.m - j0);
		for (int t = 0; t < jn; t++)
		{
			const uint32_t kj = keys[t];
			rank += kj > ki || (kj == ki && j0 + t < i);
		}
	}
	if (i >= p.m)
		return;
	float* const sn = sorted + ((long long)blockIdx.y * p.m + rank) * 5;
	const float* const ar = an + (long long)i * p.am;
#pragma unroll
	for (int d = 0; d < 5; d++)
		sn[d] = ar[d];
	idx[(long long)blockIdx.y * p.m + rank] = i;
}

// CPU_REF's IoU test of sorted rows x (the higher score) and y (nms/ccv_nnc_nms_cpu_ref.c:77-86), each operation rounded on its own
__device__ __forceinline__ bool nms_overlaps(const float* bx, const float* by, const float thr)
{
	const float area1 = __fmul_rn(bx[3], bx[4]), area2 = __fmul_rn(by[3], by[4]);
	const float xe0 = __fadd_rn(bx[1], bx[3]), xe1 = __fadd_rn(by[1], by[3]);
	const float ye0 = __fadd_rn(bx[2], bx[4]), ye1 = __fadd_rn(by[2], by[4]);
	const float xd = __fsub_rn(xe0 < xe1 ? xe0 : xe1, bx[1] > by[1] ? bx[1] : by[1]);
	const float yd = __fsub_rn(ye0 < ye1 ? ye0 : ye1, bx[2] > by[2] ? bx[2] : by[2]);
	const float xdiff = 0.f > xd ? 0.f : xd, ydiff = 0.f > yd ? 0.f : yd;
	const float inter = __fmul_rn(xdiff, ydiff);
	const float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
	return iou >= thr;
}

// mask[item][i][w] bit t: sorted row w * 64 + t (> i) overlaps row i.  One CTA of 64 threads per (row block, column block >= it)
__global__ void __launch_bounds__(64) nms_mask_kernel(const float* __restrict__ sorted, unsigned long long* __restrict__ mask, const NmsArg p)
{
	const int rb = blockIdx.y, cb = blockIdx.x;
	if (cb < rb)
		return;
	__shared__ float cols[64 * 5];
	const float* const sn = sorted + (long long)blockIdx.z * p.m * 5;
	const int j0 = cb * 64, cn = min(64, p.m - j0);
	for (int t = threadIdx.x; t < cn * 5; t += 64)
		cols[t] = sn[(long long)j0 * 5 + t];
	__syncthreads();
	const int i = rb * 64 + threadIdx.x;
	if (i >= p.m)
		return;
	float bx[5];
#pragma unroll
	for (int d = 0; d < 5; d++)
		bx[d] = sn[(long long)i * 5 + d];
	unsigned long long bits = 0;
	for (int t = cb == rb ? threadIdx.x + 1 : 0; t < cn; t++)
		if (nms_overlaps(bx, cols + t * 5, p.thr))
			bits |= 1ull << t;
	mask[((long long)blockIdx.z * p.m + i) * p.words + cb] = bits;
}

// the greedy sweep and the compaction of one item per CTA
__global__ void __launch_bounds__(NMS_THREADS) nms_sweep_kernel(const float* __restrict__ sorted, const int* __restrict__ idx, const unsigned long long* __restrict__ mask, float* b, int* c, const NmsArg p, const int item0)
{
	extern __shared__ unsigned long long sm[];
	unsigned long long* const removed = sm;          // [words]
	unsigned long long* const kept = sm + p.words;   // [words]
	int* const before = (int*)(sm + 2 * p.words);    // [words]: kept rows in earlier words
	__shared__ unsigned long long diag[64];
	const int item = item0 + blockIdx.x;
	const float* const sn = sorted + (long long)blockIdx.x * p.m * 5;
	const int* const in = idx + (long long)blockIdx.x * p.m;
	const unsigned long long* const mk = mask + (long long)blockIdx.x * p.m * p.words;
	// rows whose score is -FLT_MAX count as suppressed already: never kept, never suppressing (CPU_REF's `== -FLT_MAX` tests)
	for (int w = threadIdx.x; w < p.words; w += NMS_THREADS)
	{
		unsigned long long r = 0;
		for (int t = 0; t < 64 && w * 64 + t < p.m; t++)
			if (sn[(long long)(w * 64 + t) * 5] == -FLT_MAX)
				r |= 1ull << t;
		removed[w] = r;
	}
	for (int w = 0; w < p.words; w++)
	{
		__syncthreads();
		if (threadIdx.x < 64)
			diag[threadIdx.x] = w * 64 + threadIdx.x < p.m ? mk[(long long)(w * 64 + threadIdx.x) * p.words + w] : 0;
		__syncthreads();
		if (threadIdx.x == 0)
		{
			unsigned long long r = removed[w], k = 0;
			const int n = min(64, p.m - w * 64);
			for (int t = 0; t < n; t++)
				if (!((r >> t) & 1))
					k |= 1ull << t, r |= diag[t];
			removed[w] = r, kept[w] = k;
		}
		__syncthreads();
		const unsigned long long k = kept[w];
		for (int v = w + 1 + threadIdx.x; v < p.words; v += NMS_THREADS)
		{
			unsigned long long r = removed[v];
			for (unsigned long long q = k; q; q &= q - 1)
				r |= mk[(long long)(w * 64 + __ffsll((long long)q) - 1) * p.words + v];
			removed[v] = r;
		}
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		int s = 0;
		for (int w = 0; w < p.words; w++)
			before[w] = s, s += __popcll(kept[w]);
		before[p.words] = s;
	}
	__syncthreads();
	const int nkept = before[p.words];
	float* const bn = b + item * p.bn;
	int* const cn = c + item * p.cn;
	for (int x = threadIdx.x; x < p.m; x += NMS_THREADS)
	{
		const int w = x >> 6, t = x & 63;
		const unsigned long long k = kept[w];
		if ((k >> t) & 1)
		{
			const int y = before[w] + __popcll(k & ((1ull << t) - 1));
			float* const row = bn + (long long)y * p.bm;
#pragma unroll
			for (int d = 0; d < 5; d++)
				row[d] = sn[(long long)x * 5 + d];
			cn[y] = in[x];
		}
		if (x >= nkept)
		{
			// the tail keeps the sorted array's coordinates at its own positions
			float* const row = bn + (long long)x * p.bm;
			row[0] = -FLT_MAX;
#pragma unroll
			for (int d = 1; d < 5; d++)
				row[d] = sn[(long long)x * 5 + d];
			cn[x] = -1;
		}
	}
}

// backward: h = 0, then h[c[x]] = g[x] for x before the first negative index (indices outside [0, m) are skipped)
__global__ void __launch_bounds__(NMS_THREADS) nms_bwd_kernel(const float* __restrict__ g, const int* __restrict__ c, float* __restrict__ h, const NmsArg p)
{
	__shared__ int first;
	const int item = blockIdx.x;
	const int* const cn = c + item * p.cn;
	const float* const gn = g + item * p.an;
	float* const hn = h + item * p.bn;
	if (threadIdx.x == 0)
		first = p.m;
	__syncthreads();
	int f = p.m;
	for (int x = threadIdx.x; x < p.m; x += NMS_THREADS)
		if (cn[x] < 0)
		{
			f = x;
			break;
		}
	atomicMin(&first, f); // a shared-memory minimum: the result does not depend on the order
	for (int x = threadIdx.x; x < p.m; x += NMS_THREADS)
	{
		float* const row = hn + (long long)x * p.bm;
#pragma unroll
		for (int d = 0; d < 5; d++)
			row[d] = 0.f;
	}
	__syncthreads();
	const int n = first;
	for (int x = threadIdx.x; x < n; x += NMS_THREADS)
	{
		const int k = cn[x];
		if (k >= p.m)
			continue;
		float* const row = hn + (long long)k * p.bm;
		const float* const gr = gn + (long long)x * p.am;
#pragma unroll
		for (int d = 0; d < 5; d++)
			row[d] = gr[d];
	}
}

// ------------------------------------------------------------------------------------------------ command layer
// element steps of every axis: a view's strides, else packed
void steps_of(const ccv_nnc_tensor_t* const t, const int nd, long long* const s)
{
	if (CCV_IS_TENSOR_VIEW(t))
	{
		for (int i = 0; i < nd; i++)
			s[i] = ((const ccv_nnc_tensor_view_t*)t)->stride[i];
		return;
	}
	long long v = 1;
	for (int i = nd - 1; i >= 0; i--)
		s[i] = v, v *= t->info.dim[i];
}

// a feature-shaped operand [n?, H, W, C] (NHWC) or [n?, C, H, W] (NCHW)
struct Map {
	int n, h, w, c;
	long long sn, sy, sx, sc;
};
bool map_of(const ccv_nnc_tensor_t* const t, Map& m)
{
	const int nd = nd_of(t);
	if (nd != 3 && nd != 4)
		return false;
	const int fmt = t->info.format;
	if (fmt != CCV_TENSOR_FORMAT_NHWC && fmt != CCV_TENSOR_FORMAT_NCHW)
		return false;
	long long s[4];
	steps_of(t, nd, s);
	const int o = nd - 3;
	m.n = nd == 4 ? t->info.dim[0] : 1;
	m.sn = nd == 4 ? s[0] : 0;
	if (fmt == CCV_TENSOR_FORMAT_NHWC)
		m.h = t->info.dim[o], m.w = t->info.dim[o + 1], m.c = t->info.dim[o + 2], m.sy = s[o], m.sx = s[o + 1], m.sc = s[o + 2];
	else
		m.c = t->info.dim[o], m.h = t->info.dim[o + 1], m.w = t->info.dim[o + 2], m.sc = s[o], m.sy = s[o + 1], m.sx = s[o + 2];
	return m.n > 0 && m.h > 0 && m.w > 0 && m.c > 0;
}
// ROIs: fp32 [4] or [k, 4] with a unit column step
bool rois_of(const ccv_nnc_tensor_t* const b, int& bn, long long& bstep)
{
	const int nd = nd_of(b);
	if (CCV_GET_DATA_TYPE(b->info.datatype) != CCV_32F || (nd != 1 && nd != 2) || b->info.dim[nd - 1] != 4)
		return false;
	long long s[2];
	steps_of(b, nd, s);
	if (s[nd - 1] != 1)
		return false;
	bn = nd == 2 ? b->info.dim[0] : 1;
	bstep = nd == 2 ? s[0] : 0;
	return bn > 0;
}

template <typename T>
int roi_fwd_t(cudaStream_t s, const void* a, const float* b, void* c, const RoiArg& p)
{
	roi_align_fwd_kernel<T><<<dim3((unsigned)p.n, (unsigned)p.pool_h), RF_THREADS, 0, s>>>((const T*)a, b, (T*)c, p);
	return launched("roi align forward");
}
template <typename T>
int roi_bwd_t(cudaStream_t s, const void* g, const float* b, void* o, const RoiArg& p, const int o_n)
{
	const long long hw = (long long)p.h * p.w, per = (long long)RB_WARPS * RB_PIX;
	const dim3 grid((unsigned)((hw + per - 1) / per), (unsigned)o_n, (unsigned)((p.ch + 32 * RB_CPL - 1) / (32 * RB_CPL)));
	roi_align_bwd_kernel<T><<<grid, RB_WARPS * 32, 0, s>>>((const T*)g, b, (T*)o, p, o_n);
	return launched("roi align backward");
}

// (a, b) -> c
int exec_roi_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const ccv_nnc_tensor_t* const a = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const b = input_size > 1 ? inputs[1] : 0;
	const ccv_nnc_tensor_t* const c = output_size > 0 ? outputs[0] : 0;
	if (!a || !b || !c)
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(a);
	Map ma, mc;
	RoiArg p;
	if (kind < 0 || kind_of(c) != kind || a->info.format != c->info.format || !map_of(a, ma) || !map_of(c, mc) || !rois_of(b, p.b_n, p.bstep))
		return CCV_NNC_EXEC_INVALID;
	if (ma.c != mc.c || mc.n != (ma.n > p.b_n ? ma.n : p.b_n))
		return CCV_NNC_EXEC_INVALID;
	p.h = ma.h, p.w = ma.w, p.ch = ma.c, p.pool_h = mc.h, p.pool_w = mc.w, p.a_n = ma.n, p.n = mc.n;
	p.fn = ma.sn, p.fy = ma.sy, p.fx = ma.sx, p.fc = ma.sc, p.pn = mc.sn, p.py = mc.sy, p.px = mc.sx, p.pc = mc.sc;
	const cudaStream_t s = stream_of(stream_context);
	const int r = kind == 0 ? roi_fwd_t<float>(s, a->data.u8, b->data.f32, c->data.u8, p) : kind == 1 ? roi_fwd_t<__nv_bfloat16>(s, a->data.u8, b->data.f32, c->data.u8, p) : roi_fwd_t<__half>(s, a->data.u8, b->data.f32, c->data.u8, p);
	return r ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

// (g, -, b) -> o
int exec_roi_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const ccv_nnc_tensor_t* const g = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const b = input_size > 2 ? inputs[2] : 0;
	const ccv_nnc_tensor_t* const o = output_size > 0 ? outputs[0] : 0;
	if (!g || !b || !o)
		return CCV_NNC_EXEC_INVALID;
	const int kind = kind_of(g);
	Map mg, mo;
	RoiArg p;
	if (kind < 0 || kind_of(o) != kind || g->info.format != o->info.format || !map_of(g, mg) || !map_of(o, mo) || !rois_of(b, p.b_n, p.bstep))
		return CCV_NNC_EXEC_INVALID;
	if (mg.c != mo.c || mg.n != (mo.n > p.b_n ? mo.n : p.b_n))
		return CCV_NNC_EXEC_INVALID;
	p.h = mo.h, p.w = mo.w, p.ch = mo.c, p.pool_h = mg.h, p.pool_w = mg.w, p.a_n = mo.n, p.n = mg.n;
	p.fn = mo.sn, p.fy = mo.sy, p.fx = mo.sx, p.fc = mo.sc, p.pn = mg.sn, p.py = mg.sy, p.px = mg.sx, p.pc = mg.sc;
	const cudaStream_t s = stream_of(stream_context);
	const int r = kind == 0 ? roi_bwd_t<float>(s, g->data.u8, b->data.f32, o->data.u8, p, mo.n) : kind == 1 ? roi_bwd_t<__nv_bfloat16>(s, g->data.u8, b->data.f32, o->data.u8, p, mo.n) : roi_bwd_t<__half>(s, g->data.u8, b->data.f32, o->data.u8, p, mo.n);
	return r ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

// an NMS box operand: fp32 [m, 5] or [n, m, 5] with a unit column step; its item and row steps
bool boxes_of(const ccv_nnc_tensor_t* const t, int& n, int& m, long long& sn, long long& sm)
{
	const int nd = nd_of(t);
	if (CCV_GET_DATA_TYPE(t->info.datatype) != CCV_32F || (nd != 2 && nd != 3) || t->info.dim[nd - 1] != 5)
		return false;
	long long s[3];
	steps_of(t, nd, s);
	if (s[nd - 1] != 1)
		return false;
	n = nd == 3 ? t->info.dim[0] : 1, m = t->info.dim[nd - 2];
	sn = nd == 3 ? s[0] : 0, sm = s[nd - 2];
	return n > 0 && m > 0;
}
// the index operand: int32 [m] or [n, m] with a unit step along m
bool index_of(const ccv_nnc_tensor_t* const t, const int n, const int m, long long& sn)
{
	const int nd = nd_of(t);
	if (CCV_GET_DATA_TYPE(t->info.datatype) != CCV_32S || (nd != 1 && nd != 2))
		return false;
	if (nd == 1 ? (n != 1 || t->info.dim[0] != m) : (t->info.dim[0] != n || t->info.dim[1] != m))
		return false;
	long long s[2];
	steps_of(t, nd, s);
	if (s[nd - 1] != 1)
		return false;
	sn = nd == 2 ? s[0] : 0;
	return true;
}
size_t nms_item_bytes(const int m)
{
	const size_t words = ((size_t)m + 63) / 64;
	return (((size_t)m * 6 * sizeof(float) + 255) & ~(size_t)255) + (size_t)m * words * sizeof(unsigned long long);
}

// a -> (b, c)
int exec_nms_forw(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const ccv_nnc_tensor_t* const a = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const b = output_size > 0 ? outputs[0] : 0;
	const ccv_nnc_tensor_t* const c = output_size > 1 ? outputs[1] : 0;
	if (!a || !b || !c)
		return CCV_NNC_EXEC_INVALID;
	int n, m, n2, m2;
	NmsArg p;
	if (!boxes_of(a, n, m, p.an, p.am) || !boxes_of(b, n2, m2, p.bn, p.bm) || n2 != n || m2 != m || nd_of(a) != nd_of(b) || !index_of(c, n, m, p.cn))
		return CCV_NNC_EXEC_INVALID;
	p.m = m, p.words = (m + 63) / 64, p.thr = cmd.info.nms.iou_threshold;
	const size_t per = nms_item_bytes(m);
	size_t fit = per > NMS_WORKSPACE_CAP ? 1 : NMS_WORKSPACE_CAP / per;
	fit = fit < 65535 ? fit : 65535; // items sit on a grid axis
	const int group = (int)(fit < (size_t)n ? fit : n);
	const size_t smem = (size_t)p.words * 2 * sizeof(unsigned long long) + ((size_t)p.words + 1) * sizeof(int);
	if (smem > 200 * 1024)
		return CCV_NNC_EXEC_INVALID; // m > 800 000 rows per item
	char* const ws = (char*)ccv_nnc_stream_context_get_workspace(stream_context, per * group, CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	float* const sorted = (float*)ws;
	int* const idx = (int*)(ws + (size_t)group * m * 5 * sizeof(float));
	unsigned long long* const mask = (unsigned long long*)(ws + (((size_t)group * m * 6 * sizeof(float) + 255) & ~(size_t)255));
	const cudaStream_t s = stream_of(stream_context);
	if (smem > 48 * 1024 && cudaFuncSetAttribute(nms_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
		return CCV_NNC_EXEC_INVALID;
	for (int item0 = 0; item0 < n; item0 += group)
	{
		const int items = n - item0 < group ? n - item0 : group;
		nms_rank_kernel<<<dim3((unsigned)((m + NMS_THREADS - 1) / NMS_THREADS), (unsigned)items), NMS_THREADS, 0, s>>>(a->data.f32, sorted, idx, p, item0);
		if (launched("nms rank"))
			return CCV_NNC_EXEC_INVALID;
		nms_mask_kernel<<<dim3((unsigned)p.words, (unsigned)p.words, (unsigned)items), 64, 0, s>>>(sorted, mask, p);
		if (launched("nms mask"))
			return CCV_NNC_EXEC_INVALID;
		nms_sweep_kernel<<<(unsigned)items, NMS_THREADS, smem, s>>>(sorted, idx, mask, b->data.f32, c->data.i32, p, item0);
		if (launched("nms sweep"))
			return CCV_NNC_EXEC_INVALID;
	}
	return CCV_NNC_EXEC_SUCCESS;
}

// (g, -, -, -, c) -> h
int exec_nms_back(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	const ccv_nnc_tensor_t* const g = input_size > 0 ? inputs[0] : 0;
	const ccv_nnc_tensor_t* const c = input_size > 4 ? inputs[4] : 0;
	const ccv_nnc_tensor_t* const h = output_size > 0 ? outputs[0] : 0;
	if (!g || !c || !h)
		return CCV_NNC_EXEC_INVALID;
	int n, m, n2, m2;
	NmsArg p;
	if (!boxes_of(g, n, m, p.an, p.am) || !boxes_of(h, n2, m2, p.bn, p.bm) || n2 != n || m2 != m || nd_of(g) != nd_of(h) || !index_of(c, n, m, p.cn))
		return CCV_NNC_EXEC_INVALID;
	p.m = m, p.words = (m + 63) / 64, p.thr = 0;
	nms_bwd_kernel<<<(unsigned)n, NMS_THREADS, 0, stream_of(stream_context)>>>(g->data.f32, c->data.i32, h->data.f32, p);
	return launched("nms backward") ? CCV_NNC_EXEC_INVALID : CCV_NNC_EXEC_SUCCESS;
}

} // namespace

REGISTER_SM100(CCV_NNC_ROI_ALIGN_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_32F | CCV_16F | CCV_16BF, 1, exec_roi_forw); }
REGISTER_SM100(CCV_NNC_ROI_ALIGN_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_32F | CCV_16F | CCV_16BF, 1, exec_roi_back); }
REGISTER_SM100(CCV_NNC_NMS_FORWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_32F | CCV_32S, 1, exec_nms_forw); }
REGISTER_SM100(CCV_NNC_NMS_BACKWARD) { fill(registry, CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC, CCV_32F | CCV_32S, 1, exec_nms_back); }
