// sm100_contract.h -- internal C++ interface between the command layer (sm100_backend.cu) and the tensor-core
// contraction launchers (sm100_contract.cu).  All pointers are device pointers; shapes in elements.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace sm100 {

struct ConvGeom {
	// NHWC activations a[N, H, W, C] (element strides an, ah, aw; channel stride 1),
	// filters w[K, R, S, C] contiguous, outputs b[N, P, Q, K] (element strides bn, bh, bw).
	int N, H, W, C;
	int K, R, S;
	int P, Q;
	int stride_h, stride_w;
	int pad_h0, pad_h1, pad_w0, pad_w1; // border begin / end
	int dil_h, dil_w;
	long long an, ah, aw;
	long long bn, bh, bw;
};

// Device scratch of the calling command (a slice of the stream workspace, valid for the work this call enqueues).  Split-K
// launches write one partial tile set per split into it and a second kernel adds the slices in a fixed order (deterministic,
// replay-stable results instead of red.global.add); with too little scratch the split factor is reduced, down to no split.
struct Scratch {
	void* ptr;
	size_t bytes;
};
// what a caller should ask the stream workspace for so that no split factor has to be reduced (tiles x splits never exceeds
// ~2 CTAs per SM plus one wave of 128 x 256 fp32 tiles)
constexpr size_t CONTRACT_SCRATCH_BYTES = (size_t)96 << 20;

// x3 (last argument of every entry point): 0 = one-pass TF32, 1 = error-compensated 3xTF32 (fp32-grade products, a third of
// the tensor rate; sm100_umma_gemm.cuh).
// returns 0 on success, 1 if the shape/alignment cannot use the TMA+wgmma path (caller falls back to FFMA), <0 on CUDA error.
// C[M, N] (+)= op(A) * op(B) + bias; A is [M, K] (lda) or, if trans_a, [K, M]; B is [K, N] (ldb) or, if trans_b, [N, K].
int gemm_tf32(cudaStream_t stream, int M, int N, int K, const float* a, long long lda, int trans_a, const float* b, long long ldb, int trans_b, float* c, long long ldc, const float* bias, int accumulate, const Scratch& scratch, int x3 = 0);
int conv_fprop_tf32(cudaStream_t stream, const ConvGeom& g, const float* a, const float* w, const float* bias, float* b, const Scratch& scratch, int x3 = 0);
// the fp32 data gradient works in a workspace of conv_dgrad_workspace_bytes(g) (which includes CONTRACT_SCRATCH_BYTES for split-K slices).
// bias[C] (NULL: none) is added to every pixel of grad_a, also to those no filter tap reaches: that makes the data gradient the
// forward of a transposed convolution (CONVOLUTION_TRANSPOSE_FORWARD).
size_t conv_dgrad_workspace_bytes(const ConvGeom& g);
int conv_dgrad_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* w, const float* bias, float* grad_a, void* workspace, int x3 = 0);
int conv_wgrad_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* a, float* grad_w, int accumulate, const Scratch& scratch, int x3 = 0);

// The same contractions on 16-bit tensors (kind 1 = bf16, 2 = fp16): wgmma bf16 / fp16 with fp32 accumulation in registers, 16-bit
// result (rounded once, to nearest even).  Every leading dimension / channel count must be a multiple of 8 elements (16 bytes).
// bias: fp32 (bias32) or in the tensors' 16-bit type (bias16); at most one of them.  Returns as above (1 = shape not covered).
int gemm_16(cudaStream_t stream, int kind, int M, int N, int K, const void* a, long long lda, int trans_a, const void* b, long long ldb, int trans_b, void* c, long long ldc, const float* bias32, const void* bias16, int accumulate, const Scratch& scratch);
int conv_fprop_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* a, const void* w, const float* bias32, const void* bias16, void* b, const Scratch& scratch);
int conv_dgrad_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* w, const float* bias32, const void* bias16, void* grad_a, const Scratch& scratch);
// true when conv_dgrad_tf32 / conv_dgrad_16 may return 1 for this geometry and element kind on shape grounds (a superset of the shape
// tests they make; operand pointers aside): callers that reserve the workspace of their fallback ahead of the call count it in then
bool conv_dgrad_may_decline(const ConvGeom& g, int kind);
int conv_wgrad_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* a, void* grad_w, int accumulate, const Scratch& scratch);

// Ask the NEXT conv_fprop_tf32 / gemm_tf32 launch of this host thread to also produce per-column statistics of its output
// (batch-norm forward fused into the producing convolution).  `part` holds four planes of max_rows x N floats -- count,
// shift k, sum(v - k), sum((v - k)^2) -- one row per (CTA, epilogue warp quarter); *rows_out = rows in use (the plane
// pitch is *rows_out x N; 0 when the launch took a path without this epilogue; the request is consumed either way).
// Combined by bn_fwd_train_f32 (ext_part / ext_rows) with a Chan merge in double precision.
void conv_stats_request(float* part, int max_rows, int* rows_out);

// Small-channel convolutions (C not a multiple of 4, e.g. the 3-channel stem): explicit im2col into `workspace`
// ([N*P*Q, Kp] with Kp = R*S*C rounded up to 32, zero padded) followed by the tensor-core GEMM.  Returns 1 when not applicable.
size_t conv_im2col_workspace_bytes(const ConvGeom& g, int kind = 0); // kind: 0 = fp32, 1 = bf16, 2 = fp16
// (the workspace must hold conv_im2col_workspace_bytes(g), which includes CONTRACT_SCRATCH_BYTES for the GEMM's split-K slices)
int conv_fprop_im2col_tf32(cudaStream_t stream, const ConvGeom& g, const float* a, const float* w, const float* bias, float* b, void* workspace, int x3 = 0);
int conv_wgrad_im2col_tf32(cudaStream_t stream, const ConvGeom& g, const float* grad_b, const float* a, float* grad_w, int accumulate, void* workspace, int x3 = 0);
int conv_fprop_im2col_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* a, const void* w, const float* bias32, const void* bias16, void* b, void* workspace);
int conv_wgrad_im2col_16(cudaStream_t stream, int kind, const ConvGeom& g, const void* grad_b, const void* a, void* grad_w, int accumulate, void* workspace);

// CUDA-core fp32 versions of the same contractions: any stride/alignment, groups, exact fp32 products.  Long reductions over few
// output tiles split K into slices of `scratch` (none given: no split), combined in split order like the tensor-core path.
int gemm_ffma(cudaStream_t stream, int M, int N, int K, const float* a, long long a_rs, long long a_cs, const float* b, long long b_rs, long long b_cs, float* c, long long ldc, const float* bias, int accumulate, const Scratch& scratch = Scratch());
int conv_fprop_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* a, const float* w, const float* bias, float* b);
int conv_dgrad_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* grad_b, const float* w, const float* bias, float* grad_a);
int conv_wgrad_ffma(cudaStream_t stream, const ConvGeom& g, int groups, const float* grad_b, const float* a, float* grad_w, int accumulate, const Scratch& scratch = Scratch());
// out[r, c] = (accumulate ? out[r, c] : 0) + part[0][r, c] + part[1][r, c] + ... (fp32 slices [rows, cols] of pitch ldp, split_stride apart)
int splitk_reduce(cudaStream_t stream, const float* part, int splits, long long split_stride, int rows, int cols, long long ldp, float* out, long long ldo, int accumulate, int out_kind = 0);

// scaled dot product attention (sm100_sdpa.cu): element strides of q [B, Sq, H, D], k / v [B, Sk, Hk, D | Dv], o [B, Sq, H, Dv]
struct SdpaGeom {
	int B, H, Hk, Sq, Sk, D, Dv;
	float scale;
	int is_causal;
	long long q_b, q_s, q_h, k_b, k_s, k_h, v_b, v_s, v_h, o_b, o_s, o_h;
	long long mask_b, mask_h, mask_s; // additive mask [B | 1, H | 1, Sq, Sk]: 0 strides broadcast
	int mask_c;
};
size_t sdpa_workspace_bytes(int sq, int sk, int backward);
int sdpa_forward_f32(cudaStream_t s, const SdpaGeom& g, const float* q, const float* k, const float* v, const float* mask, float* o, void* workspace);
// dg carries the strides of dq / dk / dv in its q_* / k_* / v_* fields
int sdpa_backward_f32(cudaStream_t s, const SdpaGeom& g, const float* dout, const float* q, const float* k, const float* v, float* dq, float* dk, float* dv, const SdpaGeom& dg, void* workspace);

// 16-bit (bf16 / fp16) flash attention forward on wgmma (sm100_fmha.cu): D = Dv <= 128; lse [B, H, Sq] fp32 or NULL.
// returns 0 on success, 1 when the shape is not covered, < 0 on CUDA errors
int sdpa_forward_f16(cudaStream_t s, const SdpaGeom& g, int is_bf16, const void* q, const void* k, const void* v, void* o, float* lse);

// 16-bit flash attention backward on wgmma (sm100_fmha_bwd.cu), deterministic: D = Dv <= 128.  g carries the strides of q / k / v and, in
// o_*, of dout; dg the strides of dq / dk / dv in q_* / k_* / v_*.  out (strides oo_*) / lse = the forward's saved outputs, or NULL:
// both are then recomputed into the workspace (sdpa_backward_f16_workspace_bytes(g, 1)).  Same return convention as the forward.
size_t sdpa_backward_f16_workspace_bytes(const SdpaGeom& g, int need_forward);
int sdpa_backward_f16(cudaStream_t s, const SdpaGeom& g, const SdpaGeom& dg, int is_bf16, const void* dout, const void* q, const void* k, const void* v, const void* out, long long oo_b, long long oo_s, long long oo_h,
	const float* lse, void* dq, void* dk, void* dv, void* workspace);

// c[M, N] = a[M, K] w[N, K]^T (+ bias[N]) on the stream context's contraction scratch, all operands packed row-major; kind 0 = fp32
// (the GEMM command's default algorithm, 3xTF32), 1 = bf16, 2 = fp16; bias in the operands' type or fp32 (bias_is_f32).  Used by
// commands that end in a dense projection (the attention "unify head" output).  Returns 0, or non-zero like the GEMM launchers.
int backend_gemm_nt_bias(void* stream_context, int kind, int M, int N, int K, const void* a, const void* w, void* c, const void* bias, int bias_is_f32);

// palettized (CCV_QX) tensors (sm100_palettize.cu).  qbits 4..8; nib (elements per palette block) must make the block stride
// nib * qbits / 8 a whole number of bytes.  palette_datatype is CCV_16F, CCV_32F or CCV_64F; out holds `count` decoded elements.
bool palettize_params_ok(int qbits, int nib);
size_t palettize_data_bytes(size_t count, int qbits, int nib, size_t palette_elem);
// returns 0, 1 when the parameters are refused, < 0 on CUDA errors
int depalettize(cudaStream_t stream, const void* in, int palette_datatype, int qbits, int nib, void* out, size_t count);
// c[M, N] (ldc) = a[M, K] (lda) w[N, K]^T (+ bias[N], fp32 or fp16) with fp16 a / c and w palettized with fp16 palettes, packed
// [N, K]; M <= PALETTIZED_GEMM_M_MAX.  Decodes w in registers, fp32 accumulation in a fixed order, no workspace.  Returns as above.
// The bound is measured (tools/bench_palettize.py, DESIGN.md §7.3): on an H100 the kernel beats decode + dense GEMM on every benchmark
// shape at one row only; from 4 rows on it loses on some of them.
constexpr int PALETTIZED_GEMM_M_MAX = 1;
int gemm_palettized_f16(cudaStream_t stream, int M, int N, int K, const void* a, long long lda, const void* wq, int qbits, int nib, void* c, long long ldc, const float* bias32, const void* bias16);

// bookkeeping shared by every launcher in the backend
void count_launch(int n = 1);
unsigned long long launch_count();
void set_last_error(const char* what, cudaError_t err);
const char* last_error();

} // namespace sm100
