/* integration/cnnp_fused_attention_train.c -- an attention block with the fused unify-head projection, trained through the REFERENCE'S OWN
 * model layer: ccv_cnnp_scaled_dot_product_attention(scale, is_causal, 0, 0, fused_unify_head_weights = 1, no_bias = 0, is_trainable = 1)
 * compiled with SGD and run with ccv_cnnp_model_evaluate / _backward / _apply_gradients on GPU tensors.  Linked against
 * integration/_build/libccv_dropin.so, the reference's autograd issues SCALED_DOT_PRODUCT_ATTENTION_BACKWARD with the weights (inputs
 * (g, -, -, q, k, v, -, w, bias, y, lse, c), outputs (dq, dk, dv, -, dw, dbias)) to CCV_NNC_BACKEND_GPU_SM100, the only GPU backend there.
 *
 * The same program also builds the unfused twin -- the attention without weights, a reshape to [B, S, H D], then ccv_cnnp_dense -- with the
 * same initial weights and bias, and compares the step-1 weights gradients of the two.  The loss is 0.5 / (B S) sum (y - t)^2 against a
 * fixed target t; its gradient (y - t) / (B S) is formed on the host and handed to ccv_cnnp_model_backward.
 *
 *   cnnp_fused_attention_train --dtype 32f|16f [--steps K] [--lr R] [--causal 0|1]
 *
 * Prints one JSON object: the fused model's loss per step, and for the step-1 weights gradient the largest |dw_fused - dw_twin| and the
 * largest ratio of that difference to its bound (<= 1 passes):
 *   bound = 2 (C 2^-24 sqrt(B S) s + x3 s) + |g_fused - g_twin|^T |c| + (16-bit: 2^-10 |dw_twin|),  s = |g|^T |c|,  C = 8,
 * x3 = 2^-20 for fp32 (3xTF32 products) and 0 for 16-bit ones: each side's GEMM rounding (contract_ref's bound), the two sides' different
 * loss gradients (their forwards round y apart), and the 16-bit outputs' rounding.  c is the per-head attention, recomputed here with
 * SCALED_DOT_PRODUCT_ATTENTION_FORWARD.  The graph runner's log is switched to CCV_CLI_INFO so that a command returning anything but
 * success prints "Invalid Status" (lib/nnc/ccv_nnc_graph_run.c). */
#include <ccv.h>
#include <nnc/ccv_nnc.h>
#include <nnc/ccv_nnc_easy.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

enum { B = 2, S = 128, H = 4, D = 64, N = H * D };

static int half; /* 16-bit activations and parameters */

static float lcg_uniform(unsigned long long* const s, const float lo, const float hi)
{
	*s = *s * 6364136223846793005ull + 1442695040888963407ull;
	return lo + (hi - lo) * (float)((*s >> 40) * (1.0 / 16777216.0));
}

static ccv_nnc_tensor_param_t gpu_params(const int d0, const int d1, const int d2, const int d3)
{
	ccv_nnc_tensor_param_t p = half ? GPU_TENSOR_NHWC(000, 16F, d0) : GPU_TENSOR_NHWC(000, 32F, d0);
	p.dim[1] = d1, p.dim[2] = d2, p.dim[3] = d3;
	return p;
}

/* host floats <-> a device tensor of the activations' type */
static void upload(ccv_nnc_tensor_t* const t, const float* const f, const size_t n)
{
	ccv_nnc_tensor_param_t p = t->info;
	p.type = CCV_TENSOR_CPU_MEMORY;
	ccv_nnc_tensor_t* const h = ccv_nnc_tensor_new(0, p, 0);
	if (half)
		ccv_float_to_half_precision(f, (uint16_t*)h->data.f16, n);
	else
		memcpy(h->data.f32, f, sizeof(float) * n);
	ccv_nnc_cmd_exec(CMD_DATA_TRANSFER_FORWARD(), ccv_nnc_no_hint, 0, TENSOR_LIST(h), TENSOR_LIST(t), 0);
	ccv_nnc_tensor_free(h);
}

static void download(ccv_nnc_tensor_t* const host, float* const f, const size_t n)
{
	if (half)
		ccv_half_precision_to_float((uint16_t*)host->data.f16, f, n);
	else
		memcpy(f, host->data.f32, sizeof(float) * n);
}

static void fetch(ccv_nnc_tensor_t* const t, float* const f, const size_t n)
{
	ccv_nnc_tensor_param_t p = t->info;
	p.type = CCV_TENSOR_CPU_MEMORY;
	ccv_nnc_tensor_t* const h = ccv_nnc_tensor_new(0, p, 0);
	ccv_nnc_cmd_exec(CMD_DATA_TRANSFER_FORWARD(), ccv_nnc_no_hint, 0, TENSOR_LIST(t), TENSOR_LIST(h), 0);
	download(h, f, n);
	ccv_nnc_tensor_free(h);
}

/* a custom command for ccv_cnnp_model_parameter_gradients_map: copies the gradient it is handed (inputs[0]) to the host tensor in cmd.data */
static int copy_out(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return ccv_nnc_cmd_exec(CMD_DATA_TRANSFER_FORWARD(), ccv_nnc_no_hint, 0, TENSOR_LIST(inputs[0]), TENSOR_LIST((ccv_nnc_tensor_t*)cmd.data), stream_context);
}
static ccv_nnc_cmd_vtab_t copy_out_isa = { .exec = copy_out };

static ccv_cnnp_model_t* attention_block(const int fused, const float scale, const int causal)
{
	const ccv_cnnp_model_io_t q = ccv_cnnp_input(), k = ccv_cnnp_input(), v = ccv_cnnp_input();
	ccv_cnnp_model_io_t y;
	if (fused)
		y = ccv_cnnp_model_apply(ccv_cnnp_scaled_dot_product_attention(scale, causal, 0, 0, 1, 0, 1, "attention"), MODEL_IO_LIST(q, k, v));
	else {
		y = ccv_cnnp_model_apply(ccv_cnnp_scaled_dot_product_attention(scale, causal, 0, 0, 0, 0, 0, "attention"), MODEL_IO_LIST(q, k, v));
		y = ccv_cnnp_model_apply(ccv_cnnp_reshape(CCV_TENSOR_FORMAT_NHWC, DIM_ALLOC(B, S, N), DIM_ALLOC(), DIM_ALLOC(), "heads"), MODEL_IO_LIST(y));
		y = ccv_cnnp_model_apply(ccv_cnnp_dense(N, 0, 0, 1, "unify_head"), MODEL_IO_LIST(y));
	}
	return ccv_cnnp_model_new(MODEL_IO_LIST(q, k, v), MODEL_IO_LIST(y), 1, fused ? "fused" : "twin");
}

/* `steps` SGD steps of one model; losses[i] = the loss at step i, dw = the step-1 weights gradient, g = the step-1 loss gradient */
static void train(const int fused, const float scale, const int causal, const int steps, const float lr, ccv_nnc_tensor_t* const* const qkv, const float* const target,
	const float* const w0, const float* const b0, double* const losses, float* const dw, float* const g, ccv_nnc_stream_context_t* const stream)
{
	ccv_cnnp_model_t* const model = attention_block(fused, scale, causal);
	const ccv_nnc_tensor_param_t in[3] = { qkv[0]->info, qkv[1]->info, qkv[2]->info };
	ccv_cnnp_model_compile(model, in, 3, CMD_SGD_FORWARD(0, lr, 1, 0, 0, 0), CMD_NOOP());
	ccv_nnc_tensor_t* const tw = ccv_nnc_tensor_new(0, gpu_params(N, N, 0, 0), 0);
	ccv_nnc_tensor_t* const tb = ccv_nnc_tensor_new(0, gpu_params(N, 0, 0, 0), 0);
	upload(tw, w0, (size_t)N * N);
	upload(tb, b0, N);
	ccv_cnnp_model_set_parameter(model, ccv_cnnp_model_parameters(model, CCV_CNNP_PARAMETER_SELECT_WEIGHT, 0), tw);
	ccv_cnnp_model_set_parameter(model, ccv_cnnp_model_parameters(model, CCV_CNNP_PARAMETER_SELECT_BIAS, 0), tb);
	ccv_nnc_tensor_t* const y = ccv_nnc_tensor_new(0, gpu_params(B, S, N, 0), 0);
	ccv_nnc_tensor_t* const ty = ccv_nnc_tensor_new(0, gpu_params(B, S, N, 0), 0);
	ccv_nnc_tensor_param_t hp = gpu_params(N, N, 0, 0);
	hp.type = CCV_TENSOR_CPU_MEMORY;
	ccv_nnc_tensor_t* const hdw = ccv_nnc_tensor_new(0, hp, 0);
	const size_t ny = (size_t)B * S * N;
	float* const hy = (float*)malloc(sizeof(float) * ny);
	float* const hg = (float*)malloc(sizeof(float) * ny);
	int i;
	size_t j;
	for (i = 0; i < steps; i++)
	{
		ccv_cnnp_model_evaluate(model, (ccv_cnnp_evaluate_param_t){ .requires_grad = 1 }, qkv, 3, TENSOR_LIST(y), 0, stream);
		ccv_nnc_stream_context_wait(stream);
		fetch(y, hy, ny);
		double loss = 0;
		for (j = 0; j < ny; j++)
		{
			const float d = hy[j] - target[j];
			loss += 0.5 * d * d;
			hg[j] = d / (B * S);
		}
		losses[i] = loss / (B * S);
		upload(ty, hg, ny);
		if (half) /* the gradient as the backward sees it: rounded to the activations' type */
			fetch(ty, hg, ny);
		ccv_cnnp_model_backward(model, TENSOR_LIST(ty), 0, 0, 0, stream);
		if (i == 0)
		{
			ccv_nnc_cmd_t copy = ccv_nnc_cmd(CCV_NNC_CUSTOM_FORWARD, &copy_out_isa, ccv_nnc_cmd_auto, 0);
			copy.data = hdw;
			ccv_cnnp_model_parameter_gradients_map(model, ccv_cnnp_model_parameters(model, CCV_CNNP_PARAMETER_SELECT_WEIGHT, 0), copy, ccv_nnc_no_hint, 0, 0, 0, 0, 0, stream);
			ccv_nnc_stream_context_wait(stream);
			download(hdw, dw, (size_t)N * N);
			memcpy(g, hg, sizeof(float) * ny);
		}
		ccv_cnnp_model_apply_gradients(model, stream);
		ccv_nnc_stream_context_wait(stream);
	}
	free(hy), free(hg);
	ccv_nnc_tensor_free(tw), ccv_nnc_tensor_free(tb), ccv_nnc_tensor_free(y), ccv_nnc_tensor_free(ty), ccv_nnc_tensor_free(hdw);
	ccv_cnnp_model_free(model);
}

int main(int argc, char** argv)
{
	int steps = 4, causal = 1, i;
	float lr = 1;
	for (i = 1; i < argc; i++)
	{
		if (!strcmp(argv[i], "--dtype") && i + 1 < argc) half = !strcmp(argv[++i], "16f");
		else if (!strcmp(argv[i], "--steps") && i + 1 < argc) steps = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--lr") && i + 1 < argc) lr = (float)atof(argv[++i]);
		else if (!strcmp(argv[i], "--causal") && i + 1 < argc) causal = atoi(argv[++i]);
		else { fprintf(stderr, "unknown argument %s\n", argv[i]); return 2; }
	}
	if (steps < 2)
		steps = 2;
	ccv_nnc_init();
	if (ccv_nnc_device_count(CCV_STREAM_CONTEXT_GPU) < 1)
	{
		printf("{\"unavailable\": \"no GPU device\"}\n");
		return 0;
	}
	CCV_CLI_SET_OUTPUT_LEVEL_AND_ABOVE(CCV_CLI_INFO);
	const float scale = 1.0f / sqrtf((float)D);
	unsigned long long s = 88172645463325252ull;
	const size_t nq = (size_t)B * S * H * D, ny = (size_t)B * S * N;
	float* const buf = (float*)malloc(sizeof(float) * nq);
	ccv_nnc_tensor_t* qkv[3];
	size_t j;
	for (i = 0; i < 3; i++)
	{
		qkv[i] = ccv_nnc_tensor_new(0, gpu_params(B, S, H, D), 0);
		for (j = 0; j < nq; j++)
			buf[j] = lcg_uniform(&s, -1, 1);
		upload(qkv[i], buf, nq);
	}
	float* const target = (float*)malloc(sizeof(float) * ny);
	for (j = 0; j < ny; j++)
		target[j] = lcg_uniform(&s, -1, 1);
	/* the layer's own initialisation (lib/nnc/ccv_cnnp_model_addons.c): U(-sqrt(3) sqrt(2 / n), +..), here drawn on the host and given to both
	 * models; a non-zero bias so that dbias is not a trivial sum */
	float* const w0 = (float*)malloc(sizeof(float) * N * N);
	float b0[N];
	const float bound = sqrtf(3.f) * sqrtf(2.f / N);
	for (j = 0; j < (size_t)N * N; j++)
		w0[j] = lcg_uniform(&s, -bound, bound);
	for (j = 0; j < N; j++)
		b0[j] = lcg_uniform(&s, -0.1f, 0.1f);
	ccv_nnc_stream_context_t* const stream = ccv_nnc_stream_context_new(CCV_STREAM_CONTEXT_GPU);
	double* const losses = (double*)malloc(sizeof(double) * steps * 2);
	float* const dw = (float*)malloc(sizeof(float) * N * N * 2);
	float* const g = (float*)malloc(sizeof(float) * ny * 2);
	train(1, scale, causal, steps, lr, qkv, target, w0, b0, losses, dw, g, stream);
	train(0, scale, causal, steps, lr, qkv, target, w0, b0, losses + steps, dw + N * N, g + ny, stream);
	/* c, the per-head attention both models project */
	ccv_nnc_tensor_t* const tc = ccv_nnc_tensor_new(0, gpu_params(B, S, H, D), 0);
	ccv_nnc_cmd_exec(CMD_SCALED_DOT_PRODUCT_ATTENTION_FORWARD(scale, causal), ccv_nnc_no_hint, 0, qkv, 3, TENSOR_LIST(tc), 0);
	float* const c = (float*)malloc(sizeof(float) * nq);
	fetch(tc, c, nq);
	/* dw[o, i] = sum over rows r of g[r, o] c[r, i] */
	double max_diff = 0, max_ratio = 0;
	const double x3 = half ? 0 : 1.0 / (1 << 20), unit = 8.0 * sqrt((double)B * S) / 16777216.0;
	int o, k;
	for (o = 0; o < N; o++)
		for (k = 0; k < N; k++)
		{
			double sum = 0, dg = 0;
			size_t r;
			for (r = 0; r < (size_t)B * S; r++)
			{
				const double cr = fabs(c[r * N + k]);
				sum += fabs(g[r * N + o]) * cr;
				dg += fabs(g[r * N + o] - g[ny + r * N + o]) * cr;
			}
			const double twin = dw[N * N + o * N + k];
			const double e = 2 * (unit * sum + x3 * sum) + dg + (half ? fabs(twin) / 1024 : 0);
			const double diff = fabs(dw[o * N + k] - twin);
			if (diff > max_diff)
				max_diff = diff;
			const double ratio = diff > 0 ? diff / (e > 0 ? e : 1e-300) : 0;
			if (!(ratio <= max_ratio)) /* NaN included */
				max_ratio = ratio;
		}
	printf("{\"workload\": \"ccv_cnnp_scaled_dot_product_attention with fused unify-head weights, evaluate / backward / apply_gradients\", \"dtype\": \"%s\", "
		"\"B\": %d, \"S\": %d, \"H\": %d, \"D\": %d, \"causal\": %d, \"steps\": %d, \"lr\": %g, \"losses\": [",
		half ? "16f" : "32f", B, S, H, D, causal, steps, lr);
	for (i = 0; i < steps; i++)
		printf("%s%.8g", i ? ", " : "", losses[i]);
	printf("], \"twin_losses\": [");
	for (i = 0; i < steps; i++)
		printf("%s%.8g", i ? ", " : "", losses[steps + i]);
	printf("], \"dw_max_abs_diff\": %.6g, \"dw_max_bound_ratio\": %.6g}\n", max_diff, max_ratio);
	fflush(stdout);
	ccv_nnc_stream_context_free(stream);
	for (i = 0; i < 3; i++)
		ccv_nnc_tensor_free(qkv[i]);
	ccv_nnc_tensor_free(tc);
	free(buf), free(target), free(w0), free(losses), free(dw), free(g), free(c);
	return 0;
}
