// sm100_backend_ext.cu -- command layer for attention, layer / rms norm, upsample and the gradient allreduce.
#include "../../include/ccv_nnc_sm100.h"
#include "sm100_contract.h"
#include "sm100_ew.h"
#include <cuda_runtime.h>
#include <string.h>

using namespace sm100;

namespace {

inline cudaStream_t stream_of(ccv_nnc_stream_context_t* const stream_context) { return (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context); }

int nd_of(const ccv_nnc_tensor_t* const t)
{
	int i;
	for (i = 0; i < CCV_NNC_MAX_DIM_ALLOC; i++)
		if (t->info.dim[i] == 0)
			return i;
	return CCV_NNC_MAX_DIM_ALLOC;
}

size_t count_of(const ccv_nnc_tensor_t* const t)
{
	size_t c = 1;
	for (int i = 0; i < nd_of(t); i++)
		c *= (size_t)t->info.dim[i];
	return c;
}

bool packed_f32(const ccv_nnc_tensor_t* const t)
{
	return CCV_GET_DATA_TYPE(t->info.datatype) == CCV_32F && CCV_IS_TENSOR_CONTIGUOUS(t);
}

// the normalised axes must be the trailing ones: x is then [rows, inner]
bool rows_inner(const ccv_nnc_tensor_t* const x, const int* const axis, const int axis_count, int& rows, int& inner)
{
	if (!packed_f32(x))
		return false;
	const int nd = nd_of(x);
	if (axis_count < 1 || axis_count > nd)
		return false;
	bool reduced[CCV_NNC_MAX_DIM_ALLOC] = { false };
	for (int i = 0; i < axis_count; i++)
	{
		if (axis[i] < 0 || axis[i] >= nd)
			return false;
		reduced[axis[i]] = true;
	}
	long long r = 1, in = 1;
	bool seen_reduced = false;
	for (int i = 0; i < nd; i++)
	{
		if (reduced[i])
			seen_reduced = true, in *= x->info.dim[i];
		else {
			if (seen_reduced && x->info.dim[i] != 1)
				return false; // a kept axis after a reduced one: not a trailing reduction
			r *= x->info.dim[i];
		}
	}
	if (r > 0x7fffffff || in > 0x7fffffff)
		return false;
	rows = (int)r, inner = (int)in;
	return true;
}

} // namespace

#define SM100_EXEC_ARGS const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context

extern "C" {

// ---- scaled dot product attention ----------------------------------------------------------------------------------
// [B, S, H, D] tensors (3-d [B, S, D] = one head), element strides from views; the feature axis must be contiguous
static bool sdpa_axes(const ccv_nnc_tensor_t* const t, const int datatype, int& B, int& S, int& H, int& D, long long& sb, long long& ss, long long& sh)
{
	if (CCV_GET_DATA_TYPE(t->info.datatype) != datatype)
		return false;
	const int nd = nd_of(t);
	if (nd != 3 && nd != 4)
		return false;
	long long stride[4];
	if (CCV_IS_TENSOR_VIEW(t))
		for (int i = 0; i < nd; i++)
			stride[i] = ((const ccv_nnc_tensor_view_t*)t)->stride[i];
	else {
		long long packed = 1;
		for (int i = nd - 1; i >= 0; i--)
			stride[i] = packed, packed *= t->info.dim[i];
	}
	if (stride[nd - 1] != 1)
		return false;
	B = t->info.dim[0], S = t->info.dim[1];
	sb = stride[0], ss = stride[1];
	if (nd == 4)
		H = t->info.dim[2], D = t->info.dim[3], sh = stride[2];
	else
		H = 1, D = t->info.dim[2], sh = 0;
	return true;
}

static bool sdpa_geom(const ccv_nnc_cmd_t& cmd, const ccv_nnc_tensor_t* const q, const ccv_nnc_tensor_t* const k, const ccv_nnc_tensor_t* const v, const ccv_nnc_tensor_t* const o, SdpaGeom& g)
{
	memset(&g, 0, sizeof(g));
	int B2, B3, B4, H3, H4, D2, S3, S4;
	const int dt = CCV_GET_DATA_TYPE(q->info.datatype);
	if (dt != CCV_32F && dt != CCV_16F && dt != CCV_16BF)
		return false;
	if (!sdpa_axes(q, dt, g.B, g.Sq, g.H, g.D, g.q_b, g.q_s, g.q_h) || !sdpa_axes(k, dt, B2, g.Sk, g.Hk, D2, g.k_b, g.k_s, g.k_h) ||
		!sdpa_axes(v, dt, B3, S3, H3, g.Dv, g.v_b, g.v_s, g.v_h) || !sdpa_axes(o, dt, B4, S4, H4, D2, g.o_b, g.o_s, g.o_h))
		return false;
	if (B2 != g.B || B3 != g.B || B4 != g.B || S3 != g.Sk || S4 != g.Sq || H3 != g.Hk || H4 != g.H || D2 != g.Dv || g.Hk <= 0 || g.H % g.Hk != 0)
		return false;
	if (k->info.dim[nd_of(k) - 1] != g.D)
		return false;
	g.scale = cmd.info.scaled_dot_product_attention.scale;
	g.is_causal = cmd.info.scaled_dot_product_attention.is_causal;
	return true;
}

// scaled_dot_product_attention/ccv_nnc_scaled_dot_product_attention_cpu_ref.c:16-183: inputs (q, k, v, [attn_mask]) ->
// outputs (y, [softmax_lse]); `outputs` here already has the per-head attention tensor in slot 0 (see the entry point below)
static int sdpa_forw_core(SM100_EXEC_ARGS)
{
	if (input_size < 3 || output_size < 1 || !inputs[0] || !inputs[1] || !inputs[2] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	SdpaGeom g;
	if (!sdpa_geom(cmd, inputs[0], inputs[1], inputs[2], outputs[0], g))
		return CCV_NNC_EXEC_INVALID;
	const ccv_nnc_tensor_t* const mask_t = input_size > 3 ? inputs[3] : 0;
	const int dt = CCV_GET_DATA_TYPE(inputs[0]->info.datatype);
	const float* mask = 0;
	if (mask_t)
	{
		// [.., Sq, Sk] with optional leading (batch, head) axes of extent 1 or full (:82-86,:104); fp32 also next to 16-bit q / k / v
		const int nd = nd_of(mask_t);
		if (!packed_f32(mask_t) || nd < 2 || nd > 4 || mask_t->info.dim[nd - 1] != g.Sk || mask_t->info.dim[nd - 2] != g.Sq)
			return CCV_NNC_EXEC_INVALID;
		int md[4] = { 1, 1, g.Sq, g.Sk };
		for (int i = 0; i < nd - 2; i++)
			md[2 - (nd - 2) + i] = mask_t->info.dim[i];
		if ((md[0] != 1 && md[0] != g.B) || (md[1] != 1 && md[1] != g.H))
			return CCV_NNC_EXEC_INVALID;
		g.mask_c = 1, g.mask_s = g.Sk;
		g.mask_h = md[1] > 1 ? (long long)g.Sq * g.Sk : 0;
		g.mask_b = md[0] > 1 ? (long long)md[1] * g.Sq * g.Sk : 0;
		mask = mask_t->data.f32;
	}
	if (dt != CCV_32F)
	{
		// 16-bit tensors: the wgmma flash-attention kernel (sm100_fmha.cu) when it covers the call -- no additive mask (like the
		// reference's flash-attention backend), head dimension 128; it also writes the log-sum-exp
		float* lse = 0;
		if (output_size > 1 && outputs[1])
		{
			if (!packed_f32(outputs[1]) || count_of(outputs[1]) != (size_t)g.B * g.H * g.Sq)
				return CCV_NNC_EXEC_INVALID;
			lse = outputs[1]->data.f32;
		}
		int rc = mask ? 1 : sdpa_forward_f16(stream_of(stream_context), g, dt == CCV_16BF, inputs[0]->data.u8, inputs[1]->data.u8, inputs[2]->data.u8, outputs[0]->data.u8, lse);
		if (rc < 0)
			return CCV_NNC_EXEC_INVALID;
		if (rc == 0)
			return CCV_NNC_EXEC_SUCCESS;
		// Everything else the command allows (masks, other head dimensions, the reference trials D in {40, 64, 128, 160, 224},
		// test/int/nnc/cublas.tests.c:2752-2833): the functional form the backward uses too -- widen q, k, v into the stream workspace,
		// run the fp32 path, narrow the result (fp16 with the reference's truncating conversion, bf16 to nearest even).  Slower,
		// never a hard failure.  The fp32 path keeps no log-sum-exp (CPU_REF does not write one either, :16-183).
		if (lse || CCV_IS_TENSOR_VIEW(inputs[0]) || CCV_IS_TENSOR_VIEW(inputs[1]) || CCV_IS_TENSOR_VIEW(inputs[2]) || CCV_IS_TENSOR_VIEW(outputs[0]))
			return CCV_NNC_EXEC_NO_KERNEL;
		const size_t nq = count_of(inputs[0]), nk = count_of(inputs[1]), nv = count_of(inputs[2]), no = count_of(outputs[0]);
		const size_t bytes = (nq + nk + nv + no) * sizeof(float) + 256 + sdpa_workspace_bytes(g.Sq, g.Sk, 0);
		float* const base = (float*)ccv_nnc_stream_context_get_workspace(stream_context, bytes, CCV_TENSOR_GPU_MEMORY);
		if (!base)
			return CCV_NNC_EXEC_OOM;
		float* const q32 = base;
		float* const k32 = q32 + nq;
		float* const v32 = k32 + nk;
		float* const o32 = v32 + nv;
		void* const inner_ws = (void*)(((uintptr_t)(o32 + no) + 255) & ~(uintptr_t)255);
		const int code = dt == CCV_16BF ? 3 : 1;
		cudaStream_t st = stream_of(stream_context);
		if (convert_dtype(st, inputs[0]->data.u8, code, q32, 0, nq) || convert_dtype(st, inputs[1]->data.u8, code, k32, 0, nk) || convert_dtype(st, inputs[2]->data.u8, code, v32, 0, nv))
			return CCV_NNC_EXEC_INVALID;
		if (sdpa_forward_f32(st, g, q32, k32, v32, mask, o32, inner_ws))
			return CCV_NNC_EXEC_INVALID;
		if (convert_dtype(st, o32, 0, outputs[0]->data.u8, code, no))
			return CCV_NNC_EXEC_INVALID;
		return CCV_NNC_EXEC_SUCCESS;
	}
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, sdpa_workspace_bytes(g.Sq, g.Sk, 0), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	if (sdpa_forward_f32(stream_of(stream_context), g, inputs[0]->data.f32, inputs[1]->data.f32, inputs[2]->data.f32, mask, outputs[0]->data.f32, ws))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}


// The command's entry point.  With "unify head" weights (inputs[4] = w [H Dv, H Dv], inputs[5] = bias, :26-27,:184-255) the per-head
// attention goes to outputs[2] and outputs[0] = that tensor seen as [B, Sq, H Dv], times w^T, plus bias: the attention above followed
// by one dense projection on the tensor cores (fp32: the GEMM command's default 3xTF32; 16-bit: kind::f16).
int ccv_nnc_sm100_exec_sdpa_forw(SM100_EXEC_ARGS)
{
	ccv_nnc_tensor_t* const w = input_size > 4 ? inputs[4] : 0;
	ccv_nnc_tensor_t* const bias = input_size > 5 ? inputs[5] : 0;
	if (!w)
	{
		if (bias) // a bias always requires a weight matrix (:27-28)
			return CCV_NNC_EXEC_INVALID;
		return sdpa_forw_core(cmd, hint, flags, inputs, input_size, outputs, output_size, stream_context);
	}
	if (input_size < 3 || output_size < 3 || !outputs[0] || !outputs[2] || !inputs[0])
		return CCV_NNC_EXEC_INVALID;
	ccv_nnc_tensor_t* const c = outputs[2];
	ccv_nnc_tensor_t* const d = outputs[0];
	const int dt = CCV_GET_DATA_TYPE(inputs[0]->info.datatype);
	const int c_nd = nd_of(c), d_nd = nd_of(d);
	if (CCV_IS_TENSOR_VIEW(c) || CCV_IS_TENSOR_VIEW(d) || CCV_IS_TENSOR_VIEW(w) || (c_nd != 3 && c_nd != 4) || d_nd != 3 || nd_of(w) != 2)
		return CCV_NNC_EXEC_INVALID;
	// the weights may be palettized (attention/gpu/ccv_nnc_scaled_dot_product_attention_flash_attn.cu registers CCV_QX), with a
	// palette of the activations' type; no other operand may be
	const bool w_qx = CCV_GET_DATA_TYPE(w->info.datatype) == CCV_QX;
	const int w_dt = w_qx ? (w->info.datatype & 0xff) << 12 : CCV_GET_DATA_TYPE(w->info.datatype);
	const int w_q = (w->info.datatype >> 8) & 0xf;
	if (w_qx && ((dt != CCV_16F && dt != CCV_32F) || !palettize_params_ok(w_q, w->info.reserved)))
		return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < input_size; i++)
		if (i != 4 && inputs[i] && CCV_GET_DATA_TYPE(inputs[i]->info.datatype) == CCV_QX)
			return CCV_NNC_EXEC_INVALID;
	for (int i = 0; i < output_size; i++)
		if (outputs[i] && CCV_GET_DATA_TYPE(outputs[i]->info.datatype) == CCV_QX)
			return CCV_NNC_EXEC_INVALID;
	if (CCV_GET_DATA_TYPE(c->info.datatype) != dt || CCV_GET_DATA_TYPE(d->info.datatype) != dt || w_dt != dt)
		return CCV_NNC_EXEC_INVALID;
	const int B = c->info.dim[0], S = c->info.dim[1];
	const long long hd = c_nd == 4 ? (long long)c->info.dim[2] * c->info.dim[3] : c->info.dim[2];
	if (d->info.dim[0] != B || d->info.dim[1] != S || d->info.dim[2] != hd || w->info.dim[0] != hd || w->info.dim[1] != hd || hd > 0x7fffffff || (long long)B * S > 0x7fffffff)
		return CCV_NNC_EXEC_INVALID;
	int bias_f32 = 0;
	if (bias)
	{
		const int bdt = CCV_GET_DATA_TYPE(bias->info.datatype);
		if (CCV_IS_TENSOR_VIEW(bias) || count_of(bias) != (size_t)hd || (bdt != dt && bdt != CCV_32F))
			return CCV_NNC_EXEC_INVALID;
		bias_f32 = bdt == CCV_32F;
	}
	// the attention proper, into c: inputs (q, k, v, mask), outputs (c, lse)
	ccv_nnc_tensor_t* core_in[4] = { inputs[0], inputs[1], inputs[2], input_size > 3 ? inputs[3] : 0 };
	ccv_nnc_tensor_t* core_out[2] = { c, output_size > 1 ? outputs[1] : 0 };
	const int st = sdpa_forw_core(cmd, hint, flags, core_in, 4, core_out, 2, stream_context);
	if (st != CCV_NNC_EXEC_SUCCESS)
		return st;
	const int kind = dt == CCV_32F ? 0 : (dt == CCV_16BF ? 1 : 2);
	const void* w_data = w->data.u8;
	if (w_qx)
	{
		// one workspace request [the projection's contraction scratch | decoded weights]: the projection's own request does not move it
		unsigned char* const ws = (unsigned char*)ccv_nnc_stream_context_get_workspace(stream_context, CONTRACT_SCRATCH_BYTES + (size_t)hd * hd * (dt == CCV_32F ? 4 : 2), CCV_TENSOR_GPU_MEMORY);
		if (!ws)
			return CCV_NNC_EXEC_OOM;
		if (depalettize(stream_of(stream_context), w->data.u8, dt, w_q, w->info.reserved, ws + CONTRACT_SCRATCH_BYTES, (size_t)hd * hd))
			return CCV_NNC_EXEC_INVALID;
		w_data = ws + CONTRACT_SCRATCH_BYTES;
	}
	if (backend_gemm_nt_bias(stream_context, kind, B * S, (int)hd, (int)hd, c->data.u8, w_data, d->data.u8, bias ? bias->data.u8 : 0, bias_f32))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// :259-479: inputs[0] = g, [3] = q, [4] = k, [5] = v -> outputs (dq, dk, dv); masks are not differentiable here either (:262)
int ccv_nnc_sm100_exec_sdpa_back(SM100_EXEC_ARGS)
{
	if (input_size < 6 || output_size < 3 || !inputs[0] || !inputs[3] || !inputs[4] || !inputs[5] || !outputs[0] || !outputs[1] || !outputs[2])
		return CCV_NNC_EXEC_INVALID;
	if ((input_size > 6 && inputs[6]) || (input_size > 7 && inputs[7]))
		return CCV_NNC_EXEC_INVALID;
	SdpaGeom g, dg;
	const int dt = CCV_GET_DATA_TYPE(inputs[3]->info.datatype);
	if (dt != CCV_32F)
	{
		// 16-bit backward.  Outside the fused kernel's shapes (below) the functional form: widen g, q, k, v to fp32 in the stream
		// workspace, run the fp32 composed backward (TF32 tensor-core GEMMs per (b, h)), narrow dq, dk, dv back.  The fused kernels
		// take every operand through its strides, so views (a slice of a packed QKV tensor, pitched gradients) reach them; only the
		// functional form, which widens whole tensors, refuses views.
		if (!sdpa_geom(cmd, inputs[3], inputs[4], inputs[5], inputs[0], g) || !sdpa_geom(cmd, outputs[0], outputs[1], outputs[2], inputs[0], dg))
			return CCV_NNC_EXEC_INVALID;
		if (dg.B != g.B || dg.H != g.H || dg.Hk != g.Hk || dg.Sq != g.Sq || dg.Sk != g.Sk || dg.D != g.D || dg.Dv != g.Dv)
			return CCV_NNC_EXEC_INVALID;
		// the fused wgmma backward (sm100_fmha_bwd.cu) when it covers the call: head dimension 128, 16-byte aligned rows.  It works
		// from the forward's saved output and log-sum-exp (inputs[9], inputs[10]: ...flash_attn.cu:240-241) and recomputes both itself
		// when the caller does not pass them.
		{
			const ccv_nnc_tensor_t* const o_t = input_size > 9 ? inputs[9] : 0;
			const ccv_nnc_tensor_t* const lse_t = input_size > 10 ? inputs[10] : 0;
			const void* o_ptr = 0;
			const float* lse_ptr = 0;
			long long oo_b = 0, oo_s = 0, oo_h = 0;
			if (o_t && lse_t && packed_f32(lse_t) && count_of(lse_t) == (size_t)g.B * g.H * g.Sq)
			{
				int oB, oS, oH, oD;
				if (sdpa_axes(o_t, dt, oB, oS, oH, oD, oo_b, oo_s, oo_h) && oB == g.B && oS == g.Sq && oH == g.H && oD == g.Dv)
					o_ptr = o_t->data.u8, lse_ptr = lse_t->data.f32;
			}
			const int need_forward = !o_ptr;
			void* const fws = ccv_nnc_stream_context_get_workspace(stream_context, sdpa_backward_f16_workspace_bytes(g, need_forward), CCV_TENSOR_GPU_MEMORY);
			if (!fws)
				return CCV_NNC_EXEC_OOM;
			const int rc = sdpa_backward_f16(stream_of(stream_context), g, dg, dt == CCV_16BF, inputs[0]->data.u8, inputs[3]->data.u8, inputs[4]->data.u8, inputs[5]->data.u8, o_ptr, oo_b, oo_s, oo_h, lse_ptr,
				outputs[0]->data.u8, outputs[1]->data.u8, outputs[2]->data.u8, fws);
			if (rc < 0)
				return CCV_NNC_EXEC_INVALID;
			if (rc == 0)
				return CCV_NNC_EXEC_SUCCESS;
		}
		for (int i : { 0, 3, 4, 5 })
			if (CCV_IS_TENSOR_VIEW(inputs[i]))
				return CCV_NNC_EXEC_INVALID;
		for (int i = 0; i < 3; i++)
			if (CCV_IS_TENSOR_VIEW(outputs[i]))
				return CCV_NNC_EXEC_INVALID;
		const size_t nq = count_of(inputs[3]), nk = count_of(inputs[4]), nv = count_of(inputs[5]), no = count_of(inputs[0]);
		const size_t floats = no + 2 * nq + 2 * nk + 2 * nv;
		const size_t ws_bytes = floats * sizeof(float) + 256 + sdpa_workspace_bytes(g.Sq, g.Sk, 1);
		float* const base = (float*)ccv_nnc_stream_context_get_workspace(stream_context, ws_bytes, CCV_TENSOR_GPU_MEMORY);
		if (!base)
			return CCV_NNC_EXEC_OOM;
		float* const g32 = base;
		float* const q32 = g32 + no;
		float* const k32 = q32 + nq;
		float* const v32 = k32 + nk;
		float* const dq32 = v32 + nv;
		float* const dk32 = dq32 + nq;
		float* const dv32 = dk32 + nk;
		void* const inner_ws = (void*)(((uintptr_t)(dv32 + nv) + 255) & ~(uintptr_t)255);
		const int code = dt == CCV_16BF ? 3 : 1;
		cudaStream_t st = stream_of(stream_context);
		if (convert_dtype(st, inputs[0]->data.u8, code, g32, 0, no) || convert_dtype(st, inputs[3]->data.u8, code, q32, 0, nq) ||
			convert_dtype(st, inputs[4]->data.u8, code, k32, 0, nk) || convert_dtype(st, inputs[5]->data.u8, code, v32, 0, nv))
			return CCV_NNC_EXEC_INVALID;
		if (sdpa_backward_f32(st, g, g32, q32, k32, v32, dq32, dk32, dv32, dg, inner_ws))
			return CCV_NNC_EXEC_INVALID;
		// fp16 narrowing follows the reference's truncating f32 -> f16 (lib/ccv_util.c:1434-1440), bf16 rounds to nearest even
		if (convert_dtype(st, dq32, 0, outputs[0]->data.u8, code, nq) || convert_dtype(st, dk32, 0, outputs[1]->data.u8, code, nk) || convert_dtype(st, dv32, 0, outputs[2]->data.u8, code, nv))
			return CCV_NNC_EXEC_INVALID;
		return CCV_NNC_EXEC_SUCCESS;
	}
	if (!sdpa_geom(cmd, inputs[3], inputs[4], inputs[5], inputs[0], g) || !sdpa_geom(cmd, outputs[0], outputs[1], outputs[2], inputs[0], dg))
		return CCV_NNC_EXEC_INVALID;
	if (dg.B != g.B || dg.H != g.H || dg.Hk != g.Hk || dg.Sq != g.Sq || dg.Sk != g.Sk || dg.D != g.D || dg.Dv != g.Dv)
		return CCV_NNC_EXEC_INVALID;
	void* const ws = ccv_nnc_stream_context_get_workspace(stream_context, sdpa_workspace_bytes(g.Sq, g.Sk, 1), CCV_TENSOR_GPU_MEMORY);
	if (!ws)
		return CCV_NNC_EXEC_OOM;
	if (sdpa_backward_f32(stream_of(stream_context), g, inputs[0]->data.f32, inputs[3]->data.f32, inputs[4]->data.f32, inputs[5]->data.f32, outputs[0]->data.f32, outputs[1]->data.f32, outputs[2]->data.f32, dg, ws))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}
// ---- layer norm / rms norm: statistics over the trailing axes (saved_mean dims [d0, .., 1, .., 1]) -----------------
// norm/ccv_nnc_layer_norm_cpu_ref.c:16-190: inputs (x, [scale, bias]) -> outputs (y, [saved_mean, saved_inv_std])
int ccv_nnc_sm100_exec_lnorm_forw(SM100_EXEC_ARGS)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	const int affine = cmd.info.lnorm.elementwise_affine;
	if (affine && (input_size < 3 || !inputs[1] || !inputs[2]))
		return CCV_NNC_EXEC_INVALID;
	int rows, inner;
	if (!rows_inner(inputs[0], cmd.info.lnorm.axis, cmd.info.lnorm.count, rows, inner) || !packed_f32(outputs[0]) || count_of(outputs[0]) != (size_t)rows * inner)
		return CCV_NNC_EXEC_INVALID;
	if (affine && (!packed_f32(inputs[1]) || !packed_f32(inputs[2]) || count_of(inputs[1]) != (size_t)inner || count_of(inputs[2]) != (size_t)inner))
		return CCV_NNC_EXEC_INVALID;
	float* sm = output_size > 1 && outputs[1] ? outputs[1]->data.f32 : 0;
	float* sis = output_size > 2 && outputs[2] ? outputs[2]->data.f32 : 0;
	if ((sm && count_of(outputs[1]) != (size_t)rows) || (sis && count_of(outputs[2]) != (size_t)rows))
		return CCV_NNC_EXEC_INVALID;
	if (layer_norm_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, affine ? inputs[1]->data.f32 : 0, affine ? inputs[2]->data.f32 : 0, outputs[0]->data.f32, sm, sis, rows, inner, cmd.info.lnorm.epsilon))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// norm/ccv_nnc_layer_norm_cpu_ref.c:192-420: inputs[0] = g, [3] = x, [4] = scale (affine), [7 | 5] = saved_mean, [8 | 6] = saved_inv_std
int ccv_nnc_sm100_exec_lnorm_back(SM100_EXEC_ARGS)
{
	const int affine = cmd.info.lnorm.elementwise_affine;
	const int mi = affine ? 7 : 5, si = affine ? 8 : 6;
	if (input_size <= si || output_size < 1 || !inputs[0] || !inputs[3] || !inputs[mi] || !inputs[si] || (affine && !inputs[4]))
		return CCV_NNC_EXEC_INVALID;
	int rows, inner;
	if (!rows_inner(inputs[3], cmd.info.lnorm.axis, cmd.info.lnorm.count, rows, inner) || !packed_f32(inputs[0]) || count_of(inputs[0]) != (size_t)rows * inner)
		return CCV_NNC_EXEC_INVALID;
	if (count_of(inputs[mi]) != (size_t)rows || count_of(inputs[si]) != (size_t)rows)
		return CCV_NNC_EXEC_INVALID;
	float* h = outputs[0] ? outputs[0]->data.f32 : 0;
	float* ds = output_size > 1 && outputs[1] ? outputs[1]->data.f32 : 0;
	float* db = output_size > 2 && outputs[2] ? outputs[2]->data.f32 : 0;
	if (layer_norm_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[3]->data.f32, affine ? inputs[4]->data.f32 : 0, inputs[mi]->data.f32, inputs[si]->data.f32, h, ds, db, rows, inner, 0))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// ---- group norm -------------------------------------------------------------------------------------------------------
// norm/ccv_nnc_group_norm_cpu_ref.c:16-222: inputs (x, [scale, bias]) -> outputs (y, saved_mean, saved_inv_std).  The
// statistics tensor's own dims say which elements share a slot (group axis -> groups, reduced axes -> 1).
static bool gn_dims(const ccv_nnc_tensor_t* const t, int dim[4], long long stride[4])
{
	if (CCV_GET_DATA_TYPE(t->info.datatype) != CCV_32F)
		return false;
	const int nd = nd_of(t);
	if (nd < 1 || nd > 4)
		return false;
	long long packed = 1;
	for (int i = 3; i >= 0; i--)
	{
		const int src = i - (4 - nd);
		dim[i] = src >= 0 ? t->info.dim[src] : 1;
		if (stride)
			stride[i] = src >= 0 ? (CCV_IS_TENSOR_VIEW(t) ? ((const ccv_nnc_tensor_view_t*)t)->stride[src] : packed) : 0;
		packed *= dim[i];
	}
	return true;
}

static bool gn_geom(const ccv_nnc_tensor_t* const x, const ccv_nnc_tensor_t* const y, const ccv_nnc_tensor_t* const h, const ccv_nnc_tensor_t* const stat, const ccv_nnc_tensor_t* const scale, GroupNormGeom& g)
{
	int d2[4];
	if (!gn_dims(x, g.dim, g.xstride) || !gn_dims(y, d2, g.ystride) || memcmp(d2, g.dim, sizeof(d2)) != 0)
		return false;
	if (h && (!gn_dims(h, d2, g.hstride) || memcmp(d2, g.dim, sizeof(d2)) != 0))
		return false;
	if (!packed_f32(stat) || nd_of(stat) != nd_of(x) || !gn_dims(stat, g.rdim, 0))
		return false;
	for (int i = 0; i < 4; i++)
		g.sdim[i] = 1;
	if (scale && (!packed_f32(scale) || nd_of(scale) != nd_of(x) || !gn_dims(scale, g.sdim, 0)))
		return false;
	for (int i = 0; i < 4; i++)
		if (g.rdim[i] < 1 || g.rdim[i] > g.dim[i] || g.sdim[i] < 1 || g.sdim[i] > g.dim[i])
			return false;
	return true;
}

int ccv_nnc_sm100_exec_gnorm_forw(SM100_EXEC_ARGS)
{
	if (input_size < 1 || output_size < 3 || !inputs[0] || !outputs[0] || !outputs[1] || !outputs[2])
		return CCV_NNC_EXEC_INVALID;
	const int affine = cmd.info.gnorm.elementwise_affine;
	if (affine && (input_size < 3 || !inputs[1] || !inputs[2] || count_of(inputs[1]) != count_of(inputs[2])))
		return CCV_NNC_EXEC_INVALID;
	GroupNormGeom g;
	if (!gn_geom(inputs[0], outputs[0], 0, outputs[1], affine ? inputs[1] : 0, g) || !packed_f32(outputs[2]) || count_of(outputs[2]) != count_of(outputs[1]) || (affine && !packed_f32(inputs[2])))
		return CCV_NNC_EXEC_INVALID;
	// Both reference implementations read the epsilon through the LAYER-norm arm of the parameter union
	// (norm/ccv_nnc_group_norm_cpu_ref.c:46, norm/gpu/ccv_nnc_group_norm_gpu_cudnn.cu:117: `cmd.info.lnorm.epsilon`), which aliases
	// gnorm.reduce_count -- a small integer whose bits read as a denormal float (~0), NOT gnorm.epsilon.  Parity is with what the
	// reference computes, so the same word is read here (its own tests hold the two backends to 1e-5 on statistics over 4 values,
	// test/int/nnc/cudnn.tests.c:1491-1560, where a 1e-5 epsilon would show).
	if (group_norm_fwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, affine ? inputs[1]->data.f32 : 0, affine ? inputs[2]->data.f32 : 0, outputs[0]->data.f32, outputs[1]->data.f32, outputs[2]->data.f32, cmd.info.lnorm.epsilon))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// norm/ccv_nnc_group_norm_cpu_ref.c:224-505: inputs[0] = g, [3] = x, [4] = scale (affine), [7 | 5] = saved_mean, [8 | 6] = saved_inv_std
int ccv_nnc_sm100_exec_gnorm_back(SM100_EXEC_ARGS)
{
	const int affine = cmd.info.gnorm.elementwise_affine;
	const int mi = affine ? 7 : 5, si = affine ? 8 : 6;
	if (input_size <= si || output_size < 1 || !inputs[0] || !inputs[3] || !inputs[mi] || !inputs[si] || (affine && !inputs[4]))
		return CCV_NNC_EXEC_INVALID;
	ccv_nnc_tensor_t* const h = outputs[0];
	ccv_nnc_tensor_t* const ds = output_size > 1 ? outputs[1] : 0;
	ccv_nnc_tensor_t* const db = output_size > 2 ? outputs[2] : 0;
	GroupNormGeom g;
	if (!gn_geom(inputs[3], inputs[0], h, inputs[mi], affine ? inputs[4] : (ds ? ds : db), g) || !packed_f32(inputs[si]) || count_of(inputs[si]) != count_of(inputs[mi]))
		return CCV_NNC_EXEC_INVALID;
	if ((ds && (!packed_f32(ds) || (long long)count_of(ds) != (long long)g.sdim[0] * g.sdim[1] * g.sdim[2] * g.sdim[3])) || (db && (!packed_f32(db) || (long long)count_of(db) != (long long)g.sdim[0] * g.sdim[1] * g.sdim[2] * g.sdim[3])))
		return CCV_NNC_EXEC_INVALID;
	void* const ws = h ? ccv_nnc_stream_context_get_workspace(stream_context, group_norm_bwd_workspace_bytes(g), CCV_TENSOR_GPU_MEMORY) : 0;
	if (h && !ws)
		return CCV_NNC_EXEC_OOM;
	if (group_norm_bwd_f32(stream_of(stream_context), g, inputs[0]->data.f32, inputs[3]->data.f32, affine ? inputs[4]->data.f32 : 0, inputs[mi]->data.f32, inputs[si]->data.f32, h ? h->data.f32 : 0, ds ? ds->data.f32 : 0, db ? db->data.f32 : 0, ws))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// norm/ccv_nnc_rmsnorm_cpu_ref.c:16-130: inputs (x, scale) -> outputs (y, saved_inv_std)
int ccv_nnc_sm100_exec_rmsnorm_forw(SM100_EXEC_ARGS)
{
	if (input_size < 2 || output_size < 1 || !inputs[0] || !inputs[1] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int rows, inner;
	if (!rows_inner(inputs[0], cmd.info.rmsnorm.axis, cmd.info.rmsnorm.count, rows, inner) || !packed_f32(outputs[0]) || !packed_f32(inputs[1]) || count_of(inputs[1]) != (size_t)inner)
		return CCV_NNC_EXEC_INVALID;
	float* sis = output_size > 1 && outputs[1] ? outputs[1]->data.f32 : 0;
	if (sis && count_of(outputs[1]) != (size_t)rows)
		return CCV_NNC_EXEC_INVALID;
	if (rmsnorm_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[1]->data.f32, outputs[0]->data.f32, sis, rows, inner, cmd.info.rmsnorm.epsilon))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// norm/ccv_nnc_rmsnorm_cpu_ref.c:132-330: inputs[0] = g, [2] = x, [3] = scale, [5] = saved_inv_std -> (h, dscale)
int ccv_nnc_sm100_exec_rmsnorm_back(SM100_EXEC_ARGS)
{
	if (input_size < 6 || output_size < 1 || !inputs[0] || !inputs[2] || !inputs[3] || !inputs[5])
		return CCV_NNC_EXEC_INVALID;
	int rows, inner;
	if (!rows_inner(inputs[2], cmd.info.rmsnorm.axis, cmd.info.rmsnorm.count, rows, inner) || !packed_f32(inputs[0]) || count_of(inputs[5]) != (size_t)rows || count_of(inputs[3]) != (size_t)inner)
		return CCV_NNC_EXEC_INVALID;
	float* h = outputs[0] ? outputs[0]->data.f32 : 0;
	float* ds = output_size > 1 && outputs[1] ? outputs[1]->data.f32 : 0;
	if (rmsnorm_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, inputs[2]->data.f32, inputs[3]->data.f32, inputs[5]->data.f32, h, ds, rows, inner, 0))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

// upsample/ccv_nnc_upsample_cpu_ref.c:16-509: nearest / bilinear, align_corners, NHWC and NCHW
static bool upsample_geom(const ccv_nnc_tensor_t* const a, const ccv_nnc_tensor_t* const b, int& N, int& H, int& W, int& C, int& OH, int& OW, int& nchw)
{
	if (!packed_f32(a) || !packed_f32(b) || a->info.format != b->info.format)
		return false;
	int ad[4], bd[4];
	const int and_ = nd_of(a), bnd = nd_of(b);
	if (and_ > 4 || bnd != and_ || and_ < 3)
		return false;
	for (int i = 0; i < 4; i++)
		ad[i] = i < 4 - and_ ? 1 : a->info.dim[i - (4 - and_)], bd[i] = i < 4 - bnd ? 1 : b->info.dim[i - (4 - bnd)];
	nchw = a->info.format == CCV_TENSOR_FORMAT_NCHW;
	N = ad[0];
	if (nchw)
		C = ad[1], H = ad[2], W = ad[3], OH = bd[2], OW = bd[3];
	else
		H = ad[1], W = ad[2], C = ad[3], OH = bd[1], OW = bd[2];
	return bd[0] == N && (nchw ? bd[1] : bd[3]) == C && OH >= H && OW >= W;
}

int ccv_nnc_sm100_exec_upsample_forw(SM100_EXEC_ARGS)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int N, H, W, C, OH, OW, nchw;
	if (!upsample_geom(inputs[0], outputs[0], N, H, W, C, OH, OW, nchw))
		return CCV_NNC_EXEC_INVALID;
	if (upsample_fwd_f32(stream_of(stream_context), inputs[0]->data.f32, outputs[0]->data.f32, N, H, W, C, OH, OW, cmd.info.upsample.type, cmd.info.upsample.align_corners, nchw))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

int ccv_nnc_sm100_exec_upsample_back(SM100_EXEC_ARGS)
{
	if (input_size < 1 || output_size < 1 || !inputs[0] || !outputs[0])
		return CCV_NNC_EXEC_INVALID;
	int N, H, W, C, OH, OW, nchw;
	if (!upsample_geom(outputs[0], inputs[0], N, H, W, C, OH, OW, nchw))
		return CCV_NNC_EXEC_INVALID;
	if (upsample_bwd_f32(stream_of(stream_context), inputs[0]->data.f32, outputs[0]->data.f32, N, H, W, C, OH, OW, cmd.info.upsample.type, cmd.info.upsample.align_corners, nchw))
		return CCV_NNC_EXEC_INVALID;
	return CCV_NNC_EXEC_SUCCESS;
}

}
