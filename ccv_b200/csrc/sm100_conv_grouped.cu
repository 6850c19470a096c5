// sm100_conv_grouped.cu -- direct (not implicit-GEMM) grouped NHWC convolutions for bf16 / fp16 tensors on the CUDA cores: the
// groups the tensor-core path cannot take (depthwise, channel multipliers, C / groups or K / groups below 16 or not a multiple of
// the 16-byte vector, tensors past 2^31 elements).  Reference semantics: lib/nnc/cmd/convolution/ccv_nnc_conv_cpu_ref.c:47-65 --
// output channel k = i Kg + j reads input channels [i Cg, (i + 1) Cg), filters w[K, R, S, Cg].
//
// Every output element is one fp32 sum in a fixed order -- taps r, then s, then the group's channels -- plus the bias, rounded
// once to nearest even; results do not depend on the launch shape.  Two forms of the forward and the data gradient:
//   - depthwise (Cg = Kg = 1) with 16-byte channel vectors: a CTA computes a tile of pixels x up to 64 channels from shared memory
//     -- its filter slice (fp32, tap-major) and the input tile with its halo, read from HBM once per CTA as 16-byte vectors --, each
//     thread 8 channels of up to 4 pixels down a column;
//   - any group shape (odd C, Cg = 20, channel multipliers): one thread per output element.
// The data gradient gathers over the taps of the input pixel's residue class only.  The weight gradient is a long reduction over
// N P Q pixels into few filter elements: each CTA sums one chunk of pixels (wgrad_plan; threads of a CTA take interleaved pixels, their
// partial sums are added in lane order) into its own fp32 slice of the scratch, and splitk_reduce adds the slices in order and
// rounds once (old value + sum under ACCUMULATE_OUTPUT).  No atomics: two runs give the same bits.
#include "sm100_contract.h"
#include "sm100_elem.cuh"
#include <algorithm>

namespace sm100 {

namespace {

constexpr int THREADS = 256;
constexpr int VEC = 8; // 16-bit elements per 16-byte vector
constexpr int DW_MAX_SMEM = 48 << 10;

// grid-stride launches: enough CTAs to fill the machine several times over, the rest walks
unsigned grid_for(long long work, int per_cta, int other_dims = 1)
{
	long long b = (work + per_cta - 1) / per_cta;
	const long long cap = std::max(1ll, (long long)sm_count() * 32 / std::max(1, other_dims));
	return (unsigned)std::max(1ll, std::min(b, cap));
}

// (n, y, x) of index m of an [N, Y, X] grid; `small` (the grid has fewer than 2^32 points) takes 32-bit divisions, several times
// cheaper than 64-bit ones
__device__ __forceinline__ void unravel(const long long m, const int X, const int Y, const bool small, int& n, int& y, int& x)
{
	if (small)
	{
		const unsigned u = (unsigned)m, t = u / (unsigned)X;
		x = (int)(u - t * (unsigned)X), y = (int)(t % (unsigned)Y), n = (int)(t / (unsigned)Y);
	} else {
		const long long t = m / X;
		x = (int)(m - t * X), y = (int)(t % Y), n = (int)(t / Y);
	}
}

template <typename T>
__device__ __forceinline__ float bias_at(const float* bias32, const T* bias16, const int c)
{
	return bias32 ? bias32[c] : bias16 ? ldf(bias16 + c) : 0.f;
}

// ------------------------------------------------------------------------------------------------ forward
template <typename T>
__global__ void __launch_bounds__(THREADS) gconv_fprop_kernel(const ConvGeom g, const int Cg, const int Kg, const T* __restrict__ x, const T* __restrict__ w, const float* __restrict__ bias32, const T* __restrict__ bias16, T* __restrict__ y)
{
	const long long total = (long long)g.N * g.P * g.Q * g.K;
	const bool small = total <= 0xffffffffll;
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		int n, p, q, k;
		unravel(i, g.K, g.Q, small, p, q, k); // p holds n * P + p until the next line
		n = p / g.P, p -= n * g.P;
		const T* const xn = x + n * g.an + (long long)(k / Kg) * Cg;
		const T* const wk = w + (long long)k * g.R * g.S * Cg;
		float acc = 0.f;
		for (int r = 0; r < g.R; r++)
		{
			const int h = p * g.stride_h - g.pad_h0 + r * g.dil_h;
			if (h < 0 || h >= g.H)
				continue;
			for (int s = 0; s < g.S; s++)
			{
				const int ww = q * g.stride_w - g.pad_w0 + s * g.dil_w;
				if (ww < 0 || ww >= g.W)
					continue;
				const T* const xp = xn + h * g.ah + ww * g.aw;
				const T* const wp = wk + (r * g.S + s) * Cg;
				for (int c = 0; c < Cg; c++)
					acc = fmaf(ldf(xp + c), ldf(wp + c), acc);
			}
		}
		stf(y + n * g.bn + p * g.bh + q * g.bw + k, acc + bias_at(bias32, bias16, k));
	}
}

// Depthwise tiles: blockDim = (cvb channel vectors, 256 / cvb pixel threads), the pixel threads arranged as rows_t x TILE_W; each
// thread computes `rows` outputs down its column, so a CTA covers (rows_t rows) x TILE_W output pixels of one image and cvb * 8
// channels.  Shared memory: the filter slice as fp32 [R S][cvb * 8], then the activations the tile reads -- its input tile with the
// halo -- as [ih][iw][cvb * 8] 16-bit elements, each read from HBM once per CTA.  Pixels outside the image are never loaded or
// read: the tap tests are the scalar kernels', so the sums (and the bits) are the same.
constexpr int TILE_W = 16;

__device__ __forceinline__ int floor_div(const int a, const int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

template <typename T>
__device__ __forceinline__ void load_filter_slice(const ConvGeom& g, const T* __restrict__ w, float* wsm, const int c0, const int cw)
{
	const int RS = g.R * g.S;
	for (int e = threadIdx.y * blockDim.x + threadIdx.x; e < RS * cw; e += blockDim.x * blockDim.y)
	{
		const int c = c0 + e % cw;
		wsm[e] = c < g.C ? ldf(w + (long long)c * RS + e / cw) : 0.f;
	}
}

// [ih][iw] pixels of a pitched NHWC image from (h0, w0), the CTA's channel vectors; pixels outside [0, H) x [0, W) are skipped
template <typename T>
__device__ __forceinline__ void load_tile(const T* __restrict__ src, const long long sh, const long long sw, const int H, const int W, const int C, const int h0, const int w0, const int ih, const int iw, const int c0, T* tile)
{
	const int cvb = blockDim.x, cw = cvb * VEC;
	for (int e = threadIdx.y * cvb + threadIdx.x; e < ih * iw * cvb; e += cvb * blockDim.y)
	{
		const int cv = e % cvb, pix = e / cvb, ii = pix / iw, jj = pix - ii * iw;
		const int h = h0 + ii, x = w0 + jj, c = c0 + cv * VEC;
		if (h >= 0 && h < H && x >= 0 && x < W && c < C)
			*reinterpret_cast<uint4*>(tile + pix * cw + cv * VEC) = *reinterpret_cast<const uint4*>(src + h * sh + x * sw + c);
	}
}

template <typename T>
__global__ void __launch_bounds__(THREADS) dwconv_fprop_tile_kernel(const ConvGeom g, const int rows, const int ih, const int iw, const T* __restrict__ x, const T* __restrict__ w, const float* __restrict__ bias32, const T* __restrict__ bias16, T* __restrict__ y)
{
	extern __shared__ float smem[];
	const int cw = blockDim.x * VEC, c0 = blockIdx.y * cw, rows_t = blockDim.y / TILE_W, th = rows_t * rows;
	const int tiles_w = (g.Q + TILE_W - 1) / TILE_W, tiles_h = (g.P + th - 1) / th;
	const int tx = blockIdx.x % tiles_w, ty = blockIdx.x / tiles_w % tiles_h, n = blockIdx.x / tiles_w / tiles_h;
	const int p0 = ty * th, q0 = tx * TILE_W, hb = p0 * g.stride_h - g.pad_h0, wb = q0 * g.stride_w - g.pad_w0;
	float* const wsm = smem;
	T* const xs = reinterpret_cast<T*>(smem + g.R * g.S * cw);
	load_filter_slice(g, w, wsm, c0, cw);
	load_tile(x + n * g.an, g.ah, g.aw, g.H, g.W, g.C, hb, wb, ih, iw, c0, xs);
	__syncthreads();
	const int c = c0 + threadIdx.x * VEC, q = q0 + threadIdx.y % TILE_W;
	if (c >= g.C || q >= g.Q)
		return;
	float b[VEC];
#pragma unroll
	for (int j = 0; j < VEC; j++)
		b[j] = bias_at(bias32, bias16, c + j);
	const float* const wt = wsm + threadIdx.x * VEC;
	const T* const xt = xs + threadIdx.x * VEC;
	for (int i = 0; i < rows; i++)
	{
		const int p = p0 + threadIdx.y / TILE_W + i * rows_t;
		if (p >= g.P)
			break;
		float acc[VEC];
#pragma unroll
		for (int j = 0; j < VEC; j++)
			acc[j] = 0.f;
		for (int r = 0; r < g.R; r++)
		{
			const int h = p * g.stride_h - g.pad_h0 + r * g.dil_h;
			if (h < 0 || h >= g.H)
				continue;
			for (int s = 0; s < g.S; s++)
			{
				const int ww = q * g.stride_w - g.pad_w0 + s * g.dil_w;
				if (ww < 0 || ww >= g.W)
					continue;
				float v[VEC];
				ldv(xt + ((h - hb) * iw + (ww - wb)) * cw, v);
				const float* const f = wt + (r * g.S + s) * cw;
#pragma unroll
				for (int j = 0; j < VEC; j++)
					acc[j] = fmaf(v[j], f[j], acc[j]);
			}
		}
#pragma unroll
		for (int j = 0; j < VEC; j++)
			acc[j] += b[j];
		stv(y + n * g.bn + p * g.bh + q * g.bw + c, acc);
	}
}

// ------------------------------------------------------------------------------------------------ data gradient
// h[n, hh, ww, c] = sum over the taps (r, s) whose output pixel p = (hh + pad - r dil) / stride is whole and in range, over the
// group's Kg gradient channels, of g[n, p, q, k] w[k, r, s, c mod Cg]; pixels no tap reaches are 0 (+ bias)
template <typename T>
__global__ void __launch_bounds__(THREADS) gconv_dgrad_kernel(const ConvGeom g, const int Cg, const int Kg, const T* __restrict__ gy, const T* __restrict__ w, const float* __restrict__ bias32, const T* __restrict__ bias16, T* __restrict__ h)
{
	const long long total = (long long)g.N * g.H * g.W * g.C;
	const bool small = total <= 0xffffffffll;
	const int RSC = g.R * g.S * Cg;
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
	{
		int n, hx, wx, c;
		unravel(i, g.C, g.W, small, hx, wx, c); // hx holds n * H + hx until the next line
		n = hx / g.H, hx -= n * g.H;
		const int k0 = c / Cg * Kg, ci = c % Cg;
		const T* const gn = gy + n * g.bn + k0;
		const T* const wc = w + (long long)k0 * RSC + ci;
		float acc = 0.f;
		for (int r = 0; r < g.R; r++)
		{
			const int hn = hx + g.pad_h0 - r * g.dil_h;
			if (hn < 0 || hn % g.stride_h)
				continue;
			const int p = hn / g.stride_h;
			if (p >= g.P)
				continue;
			for (int s = 0; s < g.S; s++)
			{
				const int wn = wx + g.pad_w0 - s * g.dil_w;
				if (wn < 0 || wn % g.stride_w)
					continue;
				const int q = wn / g.stride_w;
				if (q >= g.Q)
					continue;
				const T* const gp = gn + p * g.bh + q * g.bw;
				const T* const wp = wc + (r * g.S + s) * Cg;
				for (int kk = 0; kk < Kg; kk++)
					acc = fmaf(ldf(gp + kk), ldf(wp + (long long)kk * RSC), acc);
			}
		}
		stf(h + n * g.an + hx * g.ah + wx * g.aw + c, acc + bias_at(bias32, bias16, c));
	}
}

// the data gradient's tiles: input pixels [h0, h0 + th) x [w0, w0 + TILE_W) read the gradient pixels from (floor((h0 + pad - (R - 1)
// dil) / stride), ...), ih x iw of them (dw_tile)
template <typename T>
__global__ void __launch_bounds__(THREADS) dwconv_dgrad_tile_kernel(const ConvGeom g, const int rows, const int ih, const int iw, const T* __restrict__ gy, const T* __restrict__ w, const float* __restrict__ bias32, const T* __restrict__ bias16, T* __restrict__ h)
{
	extern __shared__ float smem[];
	const int cw = blockDim.x * VEC, c0 = blockIdx.y * cw, rows_t = blockDim.y / TILE_W, th = rows_t * rows;
	const int tiles_w = (g.W + TILE_W - 1) / TILE_W, tiles_h = (g.H + th - 1) / th;
	const int tx = blockIdx.x % tiles_w, ty = blockIdx.x / tiles_w % tiles_h, n = blockIdx.x / tiles_w / tiles_h;
	const int h0 = ty * th, w0 = tx * TILE_W;
	const int pb = floor_div(h0 + g.pad_h0 - (g.R - 1) * g.dil_h, g.stride_h), qb = floor_div(w0 + g.pad_w0 - (g.S - 1) * g.dil_w, g.stride_w);
	float* const wsm = smem;
	T* const gs = reinterpret_cast<T*>(smem + g.R * g.S * cw);
	load_filter_slice(g, w, wsm, c0, cw);
	load_tile(gy + n * g.bn, g.bh, g.bw, g.P, g.Q, g.C, pb, qb, ih, iw, c0, gs);
	__syncthreads();
	const int c = c0 + threadIdx.x * VEC, wx = w0 + threadIdx.y % TILE_W;
	if (c >= g.C || wx >= g.W)
		return;
	float b[VEC];
#pragma unroll
	for (int j = 0; j < VEC; j++)
		b[j] = bias_at(bias32, bias16, c + j);
	const float* const wt = wsm + threadIdx.x * VEC;
	const T* const gt = gs + threadIdx.x * VEC;
	for (int i = 0; i < rows; i++)
	{
		const int hx = h0 + threadIdx.y / TILE_W + i * rows_t;
		if (hx >= g.H)
			break;
		float acc[VEC];
#pragma unroll
		for (int j = 0; j < VEC; j++)
			acc[j] = 0.f;
		for (int r = 0; r < g.R; r++)
		{
			const int hn = hx + g.pad_h0 - r * g.dil_h;
			if (hn < 0 || hn % g.stride_h)
				continue;
			const int p = hn / g.stride_h;
			if (p >= g.P)
				continue;
			for (int s = 0; s < g.S; s++)
			{
				const int wn = wx + g.pad_w0 - s * g.dil_w;
				if (wn < 0 || wn % g.stride_w)
					continue;
				const int q = wn / g.stride_w;
				if (q >= g.Q)
					continue;
				float v[VEC];
				ldv(gt + ((p - pb) * iw + (q - qb)) * cw, v);
				const float* const f = wt + (r * g.S + s) * cw;
#pragma unroll
				for (int j = 0; j < VEC; j++)
					acc[j] = fmaf(v[j], f[j], acc[j]);
			}
		}
#pragma unroll
		for (int j = 0; j < VEC; j++)
			acc[j] += b[j];
		stv(h + n * g.an + hx * g.ah + wx * g.aw + c, acc);
	}
}

// ------------------------------------------------------------------------------------------------ weight gradient
// CTA (blockIdx.x, blockIdx.y): filter elements [blockIdx.x eb, + eb) over the pixels [blockIdx.y chunk, + chunk); thread t takes
// element t mod eb and pixels lane = t / eb, + lanes, ...; the lanes' sums are added in lane order.  part[blockIdx.y][e] (fp32).
// An element is (k, r, s, ci) with ci fastest (the scalar form) or, depthwise with vectors, (r, s, channel vector) with the vector
// fastest, 8 channels per thread.
template <typename T, int V>
__global__ void __launch_bounds__(THREADS) gconv_wgrad_kernel(const ConvGeom g, const int Cg, const int Kg, const int elems, const int eb, const long long chunk, const T* __restrict__ gy, const T* __restrict__ x, float* __restrict__ part)
{
	__shared__ float red[THREADS * V];
	const int lanes = THREADS / eb, lane = threadIdx.x / eb, e = blockIdx.x * eb + threadIdx.x % eb;
	const bool active = lane < lanes && e < elems;
	float acc[V];
#pragma unroll
	for (int j = 0; j < V; j++)
		acc[j] = 0.f;
	if (active)
	{
		int k, r, s, ci, xc;
		if (V == 1)
		{
			ci = e % Cg;
			const int t = e / Cg;
			s = t % g.S, r = t / g.S % g.R, k = t / (g.S * g.R);
			xc = k / Kg * Cg + ci;
		} else {
			const int cvs = g.C / V;
			k = e % cvs * V, s = e / cvs % g.S, r = e / cvs / g.S;
			xc = k;
		}
		const long long npq = (long long)g.N * g.P * g.Q;
		const long long m0 = blockIdx.y * chunk, m1 = min(npq, m0 + chunk);
		const bool small = npq <= 0xffffffffll;
		for (long long m = m0 + lane; m < m1; m += lanes)
		{
			int n, p, q;
			unravel(m, g.Q, g.P, small, n, p, q);
			const int h = p * g.stride_h - g.pad_h0 + r * g.dil_h, ww = q * g.stride_w - g.pad_w0 + s * g.dil_w;
			if (h < 0 || h >= g.H || ww < 0 || ww >= g.W)
				continue;
			const T* const gp = gy + n * g.bn + p * g.bh + q * g.bw + k;
			const T* const xp = x + n * g.an + h * g.ah + ww * g.aw + xc;
			if constexpr (V == 1)
				acc[0] = fmaf(ldf(gp), ldf(xp), acc[0]);
			else {
				float a[V], b[V];
				ldv(gp, a);
				ldv(xp, b);
#pragma unroll
				for (int j = 0; j < V; j++)
					acc[j] = fmaf(a[j], b[j], acc[j]);
			}
		}
	}
	if (lanes > 1)
	{
#pragma unroll
		for (int j = 0; j < V; j++)
			red[j * THREADS + threadIdx.x] = acc[j];
		__syncthreads();
		if (lane == 0 && active)
			for (int l = 1; l < lanes; l++)
#pragma unroll
				for (int j = 0; j < V; j++)
					acc[j] += red[j * THREADS + threadIdx.x + l * eb];
	}
	if (lane != 0 || !active)
		return;
	float* const out = part + blockIdx.y * (long long)g.K * g.R * g.S * Cg;
	if (V == 1)
		out[e] = acc[0];
	else {
		// dw[c, r, s] (Cg = 1)
		const int cvs = g.C / V, RS = g.R * g.S, c = e % cvs * V, t = e / cvs;
#pragma unroll
		for (int j = 0; j < V; j++)
			out[(long long)(c + j) * RS + t] = acc[j];
	}
}

// depthwise with 16-byte channel vectors: C a multiple of 8, pitches of whole vectors, 16-byte aligned bases
bool depthwise_vec_ok(const ConvGeom& g, const int groups, const void* const a, const void* const b)
{
	return groups == g.C && g.K == g.C && g.C % VEC == 0 && g.an % VEC == 0 && g.ah % VEC == 0 && g.aw % VEC == 0 && g.bn % VEC == 0 && g.bh % VEC == 0 && g.bw % VEC == 0 &&
		((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0;
}

// the tile launch of a depthwise forward (dgrad = 0) or data gradient: up to 8 channel vectors per CTA (a power of two), 4, 2 or 1
// output rows per thread, the most that keeps the filter slice and the input tile within 48 KiB; false when not even one row fits
// (very large or dilated filters), the caller then takes the scalar form
struct DwTile {
	dim3 grid, block;
	int rows, ih, iw;
	size_t smem;
};
bool dw_tile(const ConvGeom& g, const bool dgrad, DwTile& t)
{
	const int cvs = g.C / VEC;
	int cvb = 8;
	while (cvb > cvs)
		cvb >>= 1;
	const int rows_t = THREADS / cvb / TILE_W, oh = dgrad ? g.H : g.P, ow = dgrad ? g.W : g.Q;
	for (int rows = 4; rows >= 1; rows >>= 1)
	{
		const int th = rows_t * rows;
		// the rows / columns of the source a tile reads (for the data gradient a bound: its residue classes start anywhere)
		const int ih = dgrad ? (th - 1 + (g.R - 1) * g.dil_h) / g.stride_h + 2 : (th - 1) * g.stride_h + (g.R - 1) * g.dil_h + 1;
		const int iw = dgrad ? (TILE_W - 1 + (g.S - 1) * g.dil_w) / g.stride_w + 2 : (TILE_W - 1) * g.stride_w + (g.S - 1) * g.dil_w + 1;
		const size_t smem = (size_t)g.R * g.S * cvb * VEC * sizeof(float) + (size_t)ih * iw * cvb * VEC * 2;
		const long long tiles = (long long)g.N * ((oh + th - 1) / th) * ((ow + TILE_W - 1) / TILE_W);
		if (smem <= (size_t)DW_MAX_SMEM && tiles <= 0x7fffffffll)
		{
			t.rows = rows, t.ih = ih, t.iw = iw, t.smem = smem;
			t.block = dim3(cvb, THREADS / cvb);
			t.grid = dim3((unsigned)tiles, (unsigned)((cvs + cvb - 1) / cvb));
			return true;
		}
	}
	return false;
}

// The weight gradient's pixel chunks.  Enough chunks for about WGRAD_CTAS CTAs, but at most WGRAD_MAX_SPLITS, because the ordered
// combine adds `splits` slices per filter element in one thread; at least WGRAD_MIN_CHUNK pixels per chunk; enlarged where the
// slices would not fit CONTRACT_SCRATCH_BYTES.  A function of the geometry alone (constants, not the device's SM count), so the workspace request and
// the launch agree and the bits are the same on every device.
constexpr long long WGRAD_CTAS = 2048, WGRAD_MAX_SPLITS = 512, WGRAD_MIN_CHUNK = 512;
struct WgradPlan {
	long long chunk, splits, elems;
};
WgradPlan wgrad_plan(const ConvGeom& g, const int groups)
{
	WgradPlan w;
	const long long npq = (long long)g.N * g.P * g.Q;
	w.elems = (long long)g.K * g.R * g.S * (g.C / groups);
	// the thread-owned units of the launch: channel vectors for depthwise layers of whole vectors (alignment aside), elements otherwise
	const long long units = groups == g.C && g.K == g.C && g.C % VEC == 0 ? w.elems / VEC : w.elems;
	const long long ctas_x = (units + THREADS - 1) / THREADS;
	long long splits = std::max(1ll, std::min({ (WGRAD_CTAS + ctas_x - 1) / ctas_x, WGRAD_MAX_SPLITS, (npq + WGRAD_MIN_CHUNK - 1) / WGRAD_MIN_CHUNK }));
	// (splits are gridDim.y: at most 65535)
	const long long fit = std::min(65535ll, std::max(1ll, (long long)(CONTRACT_SCRATCH_BYTES / (w.elems * sizeof(float)))));
	splits = std::min(splits, fit);
	w.chunk = (npq + splits - 1) / splits;
	w.splits = std::max(1ll, (npq + w.chunk - 1) / w.chunk);
	return w;
}

template <typename T>
int fprop(cudaStream_t s, const ConvGeom& g, const int groups, const T* a, const T* w, const float* bias32, const T* bias16, T* b)
{
	DwTile t;
	if (depthwise_vec_ok(g, groups, a, b) && dw_tile(g, false, t))
	{
		dwconv_fprop_tile_kernel<T><<<t.grid, t.block, t.smem, s>>>(g, t.rows, t.ih, t.iw, a, w, bias32, bias16, b);
		return launched("dwconv_fprop_tile_kernel");
	}
	gconv_fprop_kernel<T><<<grid_for((long long)g.N * g.P * g.Q * g.K, THREADS), THREADS, 0, s>>>(g, g.C / groups, g.K / groups, a, w, bias32, bias16, b);
	return launched("gconv_fprop_kernel");
}

template <typename T>
int dgrad(cudaStream_t s, const ConvGeom& g, const int groups, const T* gy, const T* w, const float* bias32, const T* bias16, T* h)
{
	DwTile t;
	if (depthwise_vec_ok(g, groups, h, gy) && dw_tile(g, true, t))
	{
		dwconv_dgrad_tile_kernel<T><<<t.grid, t.block, t.smem, s>>>(g, t.rows, t.ih, t.iw, gy, w, bias32, bias16, h);
		return launched("dwconv_dgrad_tile_kernel");
	}
	gconv_dgrad_kernel<T><<<grid_for((long long)g.N * g.H * g.W * g.C, THREADS), THREADS, 0, s>>>(g, g.C / groups, g.K / groups, gy, w, bias32, bias16, h);
	return launched("gconv_dgrad_kernel");
}

template <typename T>
int wgrad(cudaStream_t s, const int kind, const ConvGeom& g, const int groups, const T* gy, const T* a, T* dw, const int accumulate, const Scratch& scratch)
{
	const WgradPlan p = wgrad_plan(g, groups);
	if (!scratch.ptr || scratch.bytes < (size_t)(p.splits * p.elems) * sizeof(float))
	{
		set_last_error("grouped 16-bit weight gradient: scratch smaller than conv_grouped16_wgrad_bytes", cudaErrorInvalidValue);
		return -1;
	}
	float* const part = (float*)scratch.ptr;
	const int vec = depthwise_vec_ok(g, groups, a, gy);
	const long long units = vec ? p.elems / VEC : p.elems;
	const int eb = (int)std::min<long long>(THREADS, units);
	const dim3 grid((unsigned)((units + eb - 1) / eb), (unsigned)p.splits);
	if (vec)
		gconv_wgrad_kernel<T, VEC><<<grid, THREADS, 0, s>>>(g, 1, 1, (int)units, eb, p.chunk, gy, a, part);
	else
		gconv_wgrad_kernel<T, 1><<<grid, THREADS, 0, s>>>(g, g.C / groups, g.K / groups, (int)units, eb, p.chunk, gy, a, part);
	if (launched("gconv_wgrad_kernel"))
		return -1;
	return splitk_reduce(s, part, (int)p.splits, p.elems, 1, (int)p.elems, p.elems, (float*)dw, p.elems, accumulate, kind);
}

bool shape_ok(const ConvGeom& g, const int kind, const int groups)
{
	return (kind == 1 || kind == 2) && groups >= 1 && g.C % groups == 0 && g.K % groups == 0 && g.N > 0 && g.P > 0 && g.Q > 0 && g.H > 0 && g.W > 0;
}

} // namespace

size_t conv_grouped16_wgrad_bytes(const ConvGeom& g, const int groups)
{
	if (groups < 1 || g.C % groups)
		return 0;
	const WgradPlan p = wgrad_plan(g, groups);
	return (size_t)(p.splits * p.elems) * sizeof(float);
}

int conv_fprop_grouped16(cudaStream_t stream, const int kind, const ConvGeom& g, const int groups, const void* a, const void* w, const float* bias32, const void* bias16, void* b)
{
	if (!shape_ok(g, kind, groups))
		return 1;
	if (kind == 1)
		return fprop(stream, g, groups, (const __nv_bfloat16*)a, (const __nv_bfloat16*)w, bias32, (const __nv_bfloat16*)bias16, (__nv_bfloat16*)b);
	return fprop(stream, g, groups, (const __half*)a, (const __half*)w, bias32, (const __half*)bias16, (__half*)b);
}

int conv_dgrad_grouped16(cudaStream_t stream, const int kind, const ConvGeom& g, const int groups, const void* grad_b, const void* w, const float* bias32, const void* bias16, void* grad_a)
{
	if (!shape_ok(g, kind, groups))
		return 1;
	if (kind == 1)
		return dgrad(stream, g, groups, (const __nv_bfloat16*)grad_b, (const __nv_bfloat16*)w, bias32, (const __nv_bfloat16*)bias16, (__nv_bfloat16*)grad_a);
	return dgrad(stream, g, groups, (const __half*)grad_b, (const __half*)w, bias32, (const __half*)bias16, (__half*)grad_a);
}

int conv_wgrad_grouped16(cudaStream_t stream, const int kind, const ConvGeom& g, const int groups, const void* grad_b, const void* a, void* grad_w, const int accumulate, const Scratch& scratch)
{
	if (!shape_ok(g, kind, groups))
		return 1;
	if (kind == 1)
		return wgrad(stream, kind, g, groups, (const __nv_bfloat16*)grad_b, (const __nv_bfloat16*)a, (__nv_bfloat16*)grad_w, accumulate, scratch);
	return wgrad(stream, kind, g, groups, (const __half*)grad_b, (const __half*)a, (__half*)grad_w, accumulate, scratch);
}

} // namespace sm100
