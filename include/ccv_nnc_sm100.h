/* include/ccv_nnc_sm100.h
 *
 * The drop-in boundary of the CCV_NNC_BACKEND_GPU_SM100 backend: a C ABI that is bit-compatible with the
 * slice of liuliu/ccv's nnc "Level-1" API that the compute-command hot path touches.
 *
 * Everything here restates an interface of the reference (citations are relative to /root/reference/):
 *   - tensor / parameter / command / hint structs .......... lib/nnc/ccv_nnc_tfb.h:76-111, lib/nnc/ccv_nnc.h:111-306
 *   - exec / autotune function types ....................... lib/nnc/ccv_nnc.h:315,323
 *   - backend registry record + registration symbols ....... lib/nnc/ccv_nnc_internal.h:34-42,196-204
 *   - command / backend identifiers ........................ lib/nnc/cmd/ccv_nnc_cmd.h, lib/nnc/cmd/ccv_nnc_backend.h
 *   - dispatch, tensors, stream contexts ................... lib/nnc/ccv_nnc.h:28,574-636,759-842,940-1100
 *
 * Layouts are checked at compile time below and, in tests/test_abi.py, against the reference headers themselves.
 * There are no torch / C++ types anywhere in this file: plain pointers, ints and sizes only.
 *
 * Two groups of symbols:
 *  (A) BACKEND   -- what lib/nnc links when this backend is dropped under lib/nnc/gpu/sm100:
 *                   _register_command_<CMD>_backend_CCV_NNC_BACKEND_GPU_SM100(registry) for each command below.
 *                   The exec functions they install call back into the host for exactly two things,
 *                   ccv_nnc_stream_context_get_stream() and ccv_nnc_stream_context_get_workspace().
 *  (B) HOST      -- a minimal stand-alone implementation of the callers' side (ccv_nnc_init, ccv_nnc_cmd_exec,
 *                   tensors, stream contexts) with the reference's names and semantics so that the backend can be
 *                   exercised, tested and benchmarked without libccv. When linked into ccv these are ccv's own.
 */
#ifndef GUARD_ccv_nnc_sm100_h
#define GUARD_ccv_nnc_sm100_h

#include <stddef.h>
#include <stdint.h>
#include <sys/types.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------------ */
/* enums: lib/ccv.h:45-54, lib/nnc/ccv_nnc_tfb.h:26-58, lib/nnc/ccv_nnc.h:69-106                                  */
/* ------------------------------------------------------------------------------------------------------------ */
enum {
	CCV_8U   = 0x01000,
	CCV_32S  = 0x02000,
	CCV_32F  = 0x04000,
	CCV_64S  = 0x08000,
	CCV_64F  = 0x10000,
	CCV_16F  = 0x20000,
	CCV_QX   = 0x40000,
	CCV_16BF = 0x80000, /* declared by the reference (lib/ccv.h:53) but without kernels; this backend adds them */
};
#define CCV_GET_DATA_TYPE(x) ((x) & 0xFF000)

enum {
	CCV_TENSOR_FORMAT_NCHW = 0x01,
	CCV_TENSOR_FORMAT_NHWC = 0x02,
	CCV_TENSOR_FORMAT_CHWN = 0x04,
};

enum {
	CCV_TENSOR_CPU_MEMORY = 0x1,
	CCV_TENSOR_GPU_MEMORY = 0x2,
};

enum {
	CCV_COMPUTE_DEVICE_000 = 0x00000,
	CCV_COMPUTE_DEVICE_ANY = 0xfff00,
};
#define CCV_TENSOR_GET_MEMORY(type) ((type) & 0x3)
#define CCV_TENSOR_GET_DEVICE(type) ((type) & 0xfff00)
#define CCV_TENSOR_GET_DEVICE_ID(type) (CCV_TENSOR_GET_DEVICE(type) >> 8)
#define CCV_TENSOR_SET_DEVICE_ID(type, device_id) (type) = (((type) & ~0xfff00) | (((device_id) & 0xfff) << 8))

enum {
	CCV_TENSOR_VIEW       = 0x01000000,
	CCV_TENSOR_MULTIVIEW  = 0x02000000,
	CCV_TENSOR_PINNED_MEM = 0x04000000,
};

/* stream context types (lib/nnc/ccv_nnc.h:928-934) */
enum {
	CCV_STREAM_CONTEXT_CPU = 0x1,
	CCV_STREAM_CONTEXT_GPU = 0x2,
};
#define CCV_STREAM_GET_CONTEXT(type) ((type) & 0x3)
#define CCV_STREAM_GET_DEVICE(type) ((type) & 0xfff00)
#define CCV_STREAM_GET_DEVICE_ID(type) (CCV_STREAM_GET_DEVICE(type) >> 8)
#define CCV_STREAM_SET_DEVICE_ID(type, device_id) (type) = (((type) & ~0xfff00) | (((device_id) & 0xfff) << 8))

enum {
	CCV_NNC_ACCUMULATE_OUTPUT = 0x01,
	CCV_NNC_ZERO_MEMORY_ALLOC = 0x02,
};

enum {
	CCV_NNC_EXEC_SUCCESS   = 0,
	CCV_NNC_EXEC_INVALID   = -1,
	CCV_NNC_EXEC_NO_KERNEL = -2,
	CCV_NNC_EXEC_OOM       = -3,
};

enum {
	CCV_NNC_UPSAMPLE_NEAREST = 0,
	CCV_NNC_UPSAMPLE_BILINEAR = 1,
};

enum {
	CCV_NNC_GEMM_32F = 0x1,
	CCV_NNC_GEMM_32TF = 0x2,
	CCV_NNC_GEMM_16F = 0x4,
};

/* ------------------------------------------------------------------------------------------------------------ */
/* structs: lib/nnc/ccv_nnc_tfb.h:60-111                                                                          */
/* ------------------------------------------------------------------------------------------------------------ */
#define CCV_NNC_MAX_DIM_ALLOC (12)
#define CCV_NNC_MAX_DIM (2)

typedef struct {
	short v;
} ccv_float16_t;

typedef union ccv_numeric_data_u {
	char* i8;
	unsigned char* u8;
	int* i32;
	ccv_float16_t* f16;
	float* f32;
	int64_t* i64;
	uint64_t* u64;
	double* f64;
	void* ptr;
} ccv_numeric_data_t;

typedef struct {
	int type;     /* memory kind | device_id << 8 */
	int format;   /* CCV_TENSOR_FORMAT_* */
	int datatype; /* CCV_32F, ... */
	int reserved;
	int dim[CCV_NNC_MAX_DIM_ALLOC]; /* zero-terminated */
} ccv_nnc_tensor_param_t;

typedef struct {
	int type;
	int refcount;
	ccv_numeric_data_t data;
	off_t dataof;
	uintptr_t alias_ref;
	uint64_t data_size;
	uint64_t sig;
	ccv_nnc_tensor_param_t info;
} ccv_nnc_tensor_t;

typedef struct {
	int type;
	int refcount;
	ccv_numeric_data_t data;
	off_t dataof;
	uintptr_t alias_ref;
	uint64_t data_size;
	uint64_t sig;
	ccv_nnc_tensor_param_t info;
	int contiguous;
	off_t off;
	int stride[CCV_NNC_MAX_DIM_ALLOC];
} ccv_nnc_tensor_view_t;

#define CCV_IS_TENSOR_VIEW(x) ((*(int*)(x)) & CCV_TENSOR_VIEW)
#define CCV_IS_TENSOR_CONTIGUOUS(x) (!CCV_IS_TENSOR_VIEW(x) || (((ccv_nnc_tensor_view_t*)x)->contiguous == 1))

/* ------------------------------------------------------------------------------------------------------------ */
/* command parameters: lib/nnc/ccv_nnc.h:111-274.  Only the union arms this backend reads are spelled out;      */
/* gnorm is kept because it is the arm that sets sizeof (120).                                                   */
/* ------------------------------------------------------------------------------------------------------------ */
typedef struct {
	struct {
		int dim[CCV_NNC_MAX_DIM_ALLOC];
	} size;
	union {
		struct {
			int count;
			int groups;
			int dilation[CCV_NNC_MAX_DIM_ALLOC];
		} convolution;
		struct {
			int count;
			int groups;
			int dilation[CCV_NNC_MAX_DIM_ALLOC];
			int output_padding; /* only the output extent (ccv_nnc_hint_tensor_auto) depends on it */
		} convolution_transpose;
		struct {
			int reserved;
		} pool;
		struct {
			int axis[CCV_NNC_MAX_DIM_ALLOC];
			int count;
			float epsilon;
			int is_test;
			float momentum;
		} bnorm;
		struct {
			int axis[CCV_NNC_MAX_DIM_ALLOC];
			int count;
			float epsilon;
			int elementwise_affine;
		} lnorm;
		struct {
			int group_axis;
			int reduce_axis[CCV_NNC_MAX_DIM_ALLOC];
			int reduce_count;
			int groups;
			float epsilon;
			int elementwise_affine;
		} gnorm;
		struct {
			int axis[CCV_NNC_MAX_DIM_ALLOC];
			int count;
			float epsilon;
		} rmsnorm;
		struct {
			int nesterov;
			float rate;
			float scale;
			float decay;
			float momentum;
			float dampening;
		} sgd;
		struct {
			int step;
			float rate;
			float scale;
			float beta1;
			float beta2;
			float decay;
			float epsilon;
			int amsgrad;
		} adam;
		struct {
			int tanh;
		} gelu;
		struct {
			int transpose_a[2];
			int transpose_b[2];
			float a[3];
			int flags;
		} blas;
		struct {
			float trim0;
			float trim1;
		} label_smoothing;
		struct {
			int axis[CCV_NNC_MAX_DIM_ALLOC];
			int count;
		} reduce;
		struct {
			int axis[2];
		} transpose;
		struct {
			int type;
			float width_scale;
			float height_scale;
			int align_corners;
		} upsample;
		struct {
			float min;
			float max;
		} clamp;
		struct {
			float negative_slope;
		} leaky_relu;
		struct {
			float p;
			int entirety;
		} dropout;
		struct {
			float scale;
			int is_causal;
			int flags;
			int deterministic;
		} scaled_dot_product_attention;
		void* userdata;
	};
} ccv_nnc_cmd_param_t;

/* lib/nnc/ccv_nnc.h:279-287 */
typedef struct {
	struct {
		int dim[CCV_NNC_MAX_DIM_ALLOC];
	} stride;
	struct {
		int begin[CCV_NNC_MAX_DIM_ALLOC];
		int end[CCV_NNC_MAX_DIM_ALLOC];
	} border;
} ccv_nnc_hint_t;

typedef struct ccv_nnc_stream_context_s ccv_nnc_stream_context_t;
typedef struct ccv_nnc_cmd_vtab_s ccv_nnc_cmd_vtab_t;

/* lib/nnc/ccv_nnc.h:296-306 */
typedef struct ccv_nnc_cmd_s {
	uint32_t cmd;
	uint32_t backend;
	int algorithm;
	ccv_nnc_cmd_param_t info;
	ccv_nnc_cmd_vtab_t* isa;
	void* data;
} ccv_nnc_cmd_t;

/* lib/nnc/ccv_nnc.h:315,323.  Backward commands take inputs = [grad of outputs..., forward inputs..., forward
 * outputs...] with NULL where unused, outputs = [grad of inputs...] (lib/nnc/ccv_nnc.h:308-314). */
typedef int(*ccv_nnc_cmd_exec_f)(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);
typedef int(*ccv_nnc_cmd_autotune_f)(const ccv_nnc_cmd_t cmd, const size_t max_workspace_size, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);

/* lib/nnc/ccv_nnc_internal.h:34-42 */
typedef struct {
	int tensor_formats;
	int tensor_datatypes;
	int tensor_memory;
	int algorithms;
	ccv_nnc_cmd_exec_f exec;
	ccv_nnc_cmd_autotune_f autotune;
	void* aux;
} ccv_nnc_cmd_backend_registry_t;

#if defined(__cplusplus) && __cplusplus >= 201103L
#define CCV_SM100_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define CCV_SM100_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif
/* SURVEY.md 0.10: sizes probed from the reference on x86-64 */
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_tensor_param_t) == 64, "ccv_nnc_tensor_param_t ABI");
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_tensor_t) == 112, "ccv_nnc_tensor_t ABI");
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_tensor_view_t) == 176, "ccv_nnc_tensor_view_t ABI");
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_cmd_param_t) == 120, "ccv_nnc_cmd_param_t ABI");
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_hint_t) == 144, "ccv_nnc_hint_t ABI");
CCV_SM100_STATIC_ASSERT(sizeof(ccv_nnc_cmd_t) == 152, "ccv_nnc_cmd_t ABI");

/* ------------------------------------------------------------------------------------------------------------ */
/* identifiers: lib/nnc/cmd/ccv_nnc_cmd.h (generated: SHA256(name)[0..3] & ~1, build-cmd.rb:292),                */
/* lib/nnc/cmd/ccv_nnc_backend.h (SHA256(name)[0..3], build-cmd.rb:386)                                          */
/* ------------------------------------------------------------------------------------------------------------ */
enum {
	CCV_NNC_NOOP = 0,
	CCV_NNC_CUSTOM_FORWARD = 2,
	CCV_NNC_CUSTOM_BACKWARD = 3,
	CCV_NNC_ADD_FORWARD = 0x58fb3664,
	CCV_NNC_ADD_BACKWARD = 0x58fb3665,
	CCV_NNC_AVERAGE_POOL_FORWARD = 0x51267ab8,
	CCV_NNC_AVERAGE_POOL_BACKWARD = 0x51267ab9,
	CCV_NNC_BATCH_NORM_FORWARD = 0x5419819c,
	CCV_NNC_BATCH_NORM_BACKWARD = 0x5419819d,
	CCV_NNC_CATEGORICAL_CROSSENTROPY_FORWARD = 0x1eb327a2,
	CCV_NNC_CATEGORICAL_CROSSENTROPY_BACKWARD = 0x1eb327a3,
	CCV_NNC_COMM_ALLREDUCE_FORWARD = 0x75c8d340,
	CCV_NNC_COMM_ALLREDUCE_BACKWARD = 0x75c8d341,
	CCV_NNC_CONVOLUTION_FORWARD = 0x254d05f4,
	CCV_NNC_CONVOLUTION_BACKWARD = 0x254d05f5,
	CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD = 0xd691f78e,
	CCV_NNC_CONVOLUTION_TRANSPOSE_BACKWARD = 0xd691f78f,
	CCV_NNC_DATATYPE_CONVERSION_FORWARD = 0xd873e38c,
	CCV_NNC_DATATYPE_CONVERSION_BACKWARD = 0xd873e38d,
	CCV_NNC_DATA_TRANSFER_FORWARD = 0x12d21e1a,
	CCV_NNC_DATA_TRANSFER_BACKWARD = 0x12d21e1b,
	CCV_NNC_EWSUM_FORWARD = 0xe21a2c4c,
	CCV_NNC_EWSUM_BACKWARD = 0xe21a2c4d,
	CCV_NNC_FORMAT_TRANSFORM_FORWARD = 0xe4a2b192,
	CCV_NNC_FORMAT_TRANSFORM_BACKWARD = 0xe4a2b193,
	CCV_NNC_GEMM_FORWARD = 0x7e87d00c,
	CCV_NNC_GEMM_BACKWARD = 0x7e87d00d,
	CCV_NNC_GROUP_NORM_FORWARD = 0x17deb074,
	CCV_NNC_GROUP_NORM_BACKWARD = 0x17deb075,
	CCV_NNC_LAYER_NORM_FORWARD = 0xbed3c264,
	CCV_NNC_LAYER_NORM_BACKWARD = 0xbed3c265,
	CCV_NNC_MAX_POOL_FORWARD = 0x7bec9360,
	CCV_NNC_MAX_POOL_BACKWARD = 0x7bec9361,
	CCV_NNC_MUL_FORWARD = 0x24721a46,
	CCV_NNC_MUL_BACKWARD = 0x24721a47,
	CCV_NNC_RELU_FORWARD = 0xc51eaa80,
	CCV_NNC_RELU_BACKWARD = 0xc51eaa81,
	CCV_NNC_RMSNORM_FORWARD = 0x6889e9d0,
	CCV_NNC_RMSNORM_BACKWARD = 0x6889e9d1,
	CCV_NNC_SCALAR_MUL_FORWARD = 0x8b4d86aa,
	CCV_NNC_SCALAR_MUL_BACKWARD = 0x8b4d86ab,
	CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD = 0x284ed926,
	CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD = 0x284ed927,
	CCV_NNC_SET_FORWARD = 0x2b070804,
	CCV_NNC_SET_BACKWARD = 0x2b070805,
	CCV_NNC_SGD_FORWARD = 0xe650ad26,
	CCV_NNC_SGD_BACKWARD = 0xe650ad27,
	CCV_NNC_ADAMW_FORWARD = 0x4f5d4870,
	CCV_NNC_ADAMW_BACKWARD = 0x4f5d4871,
	CCV_NNC_DROPOUT_FORWARD = 0x7f2dc3e4,
	CCV_NNC_DROPOUT_BACKWARD = 0x7f2dc3e5,
	CCV_NNC_ADAM_FORWARD = 0xe30099dc,
	CCV_NNC_ADAM_BACKWARD = 0xe30099dd,
	CCV_NNC_GELU_FORWARD = 0xb1527ab8,
	CCV_NNC_GELU_BACKWARD = 0xb1527ab9,
	CCV_NNC_SWISH_FORWARD = 0x583d90c2,
	CCV_NNC_SWISH_BACKWARD = 0x583d90c3,
	CCV_NNC_INDEX_SELECT_FORWARD = 0x7ee7771e,
	CCV_NNC_INDEX_SELECT_BACKWARD = 0x7ee7771f,
	CCV_NNC_SOFTMAX_FORWARD = 0xc969a252,
	CCV_NNC_SOFTMAX_BACKWARD = 0xc969a253,
	CCV_NNC_SOFTMAX_CROSSENTROPY_FORWARD = 0xc26b7b5e,
	CCV_NNC_SOFTMAX_CROSSENTROPY_BACKWARD = 0xc26b7b5f,
	CCV_NNC_TRANSPOSE_FORWARD = 0xb4d506e0,
	CCV_NNC_TRANSPOSE_BACKWARD = 0xb4d506e1,
	CCV_NNC_UPSAMPLE_FORWARD = 0x73875556,
	CCV_NNC_UPSAMPLE_BACKWARD = 0x73875557,
	/* feeder commands added with the drop-in proof (same rule; each value checked against lib/nnc/cmd/ccv_nnc_cmd.inc when it was added):
	 * cmd/sigmoid, cmd/tanh, cmd/leaky_relu, cmd/ew (EWEXP / EWLOG / EWSQRT / CLAMP / EWDIV), cmd/reduce, cmd/util (MASKED_FILL), cmd/rand,
	 * cmd/dropout, cmd/adam */
	CCV_NNC_SIGMOID_FORWARD = 0xf2f69650,
	CCV_NNC_SIGMOID_BACKWARD = 0xf2f69651,
	CCV_NNC_TANH_FORWARD = 0x6a62be30,
	CCV_NNC_TANH_BACKWARD = 0x6a62be31,
	CCV_NNC_LEAKY_RELU_FORWARD = 0x507144e0,
	CCV_NNC_LEAKY_RELU_BACKWARD = 0x507144e1,
	CCV_NNC_EWEXP_FORWARD = 0xd784b170,
	CCV_NNC_EWEXP_BACKWARD = 0xd784b171,
	CCV_NNC_EWLOG_FORWARD = 0xf4191bf2,
	CCV_NNC_EWLOG_BACKWARD = 0xf4191bf3,
	CCV_NNC_EWSQRT_FORWARD = 0x8870a61e,
	CCV_NNC_EWSQRT_BACKWARD = 0x8870a61f,
	CCV_NNC_CLAMP_FORWARD = 0x2640d854,
	CCV_NNC_CLAMP_BACKWARD = 0x2640d855,
	CCV_NNC_EWDIV_FORWARD = 0x1cd2fa18,
	CCV_NNC_EWDIV_BACKWARD = 0x1cd2fa19,
	CCV_NNC_REDUCE_SUM_FORWARD = 0x52970f06,
	CCV_NNC_REDUCE_SUM_BACKWARD = 0x52970f07,
	CCV_NNC_REDUCE_MEAN_FORWARD = 0xf23556c6,
	CCV_NNC_REDUCE_MEAN_BACKWARD = 0xf23556c7,
	CCV_NNC_REDUCE_MAX_FORWARD = 0x80f1a506,
	CCV_NNC_REDUCE_MAX_BACKWARD = 0x80f1a507,
	CCV_NNC_REDUCE_MIN_FORWARD = 0x6785ef96,
	CCV_NNC_REDUCE_MIN_BACKWARD = 0x6785ef97,
	CCV_NNC_REDUCE_NORM2_FORWARD = 0xb3034e16,
	CCV_NNC_REDUCE_NORM2_BACKWARD = 0xb3034e17,
	CCV_NNC_MASKED_FILL_FORWARD = 0x7f992d84,
	CCV_NNC_MASKED_FILL_BACKWARD = 0x7f992d85,
	CCV_NNC_RANDOM_UNIFORM_FORWARD = 0xa0cd1d5e,
	CCV_NNC_RANDOM_UNIFORM_BACKWARD = 0xa0cd1d5f,
	CCV_NNC_RANDOM_NORMAL_FORWARD = 0x7062c8b4,
	CCV_NNC_RANDOM_NORMAL_BACKWARD = 0x7062c8b5,
};

enum {
	CCV_NNC_NO_BACKEND = 0,
	CCV_NNC_BACKEND_CPU_OPT = 0x46deb194,
	CCV_NNC_BACKEND_CPU_REF = 0x3d9883e5,
	CCV_NNC_BACKEND_GPU_CUBLAS = 0x9b8cfed,
	CCV_NNC_BACKEND_GPU_CUDNN = 0x854b679a,
	CCV_NNC_BACKEND_GPU_NCCL = 0x7afed9c7,
	CCV_NNC_BACKEND_GPU_REF = 0x5f19790a,
	CCV_NNC_BACKEND_MPS = 0xb2f325e2,
	/* new: SHA256("CCV_NNC_BACKEND_GPU_SM100")[0..3] (same rule as build-cmd.rb:386; checked in tests/test_abi.py) */
	CCV_NNC_BACKEND_GPU_SM100 = 0xdbfb784c,
};

/* algorithm selectors of this backend for the contraction commands (cmd.algorithm; -1 = backend default) */
enum {
	CCV_NNC_SM100_ALGO_TF32 = 0,   /* one wgmma tf32 pass, fp32 accumulate */
	CCV_NNC_SM100_ALGO_3XTF32 = 1, /* error-compensated: three tf32 passes on (hi, lo) splits */
	CCV_NNC_SM100_ALGO_FFMA = 2,   /* CUDA-core fp32 FMA (exact fp32 products; any shape / stride) */
	CCV_NNC_SM100_ALGO_COUNT = 3,
};

/* ------------------------------------------------------------------------------------------------------------ */
/* (A) BACKEND registration surface.  One symbol per (command, backend) pair, spelled exactly as                */
/* REGISTER_COMMAND_BACKEND(x, y) does (lib/nnc/ccv_nnc_internal.h:196-202); called by the generated            */
/* _ccv_nnc_cmd_init() (lib/nnc/cmd/ccv_nnc_cmd.inc:670-1149).  Each fills the registry record; exec == NULL     */
/* means "not available" (lib/nnc/ccv_nnc_cmd.c:117-131).                                                        */
/* ------------------------------------------------------------------------------------------------------------ */
#define CCV_NNC_SM100_COMMANDS(X) \
	X(CCV_NNC_GEMM_FORWARD) X(CCV_NNC_GEMM_BACKWARD) \
	X(CCV_NNC_CONVOLUTION_FORWARD) X(CCV_NNC_CONVOLUTION_BACKWARD) \
	X(CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD) X(CCV_NNC_CONVOLUTION_TRANSPOSE_BACKWARD) \
	X(CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_FORWARD) X(CCV_NNC_SCALED_DOT_PRODUCT_ATTENTION_BACKWARD) \
	X(CCV_NNC_SOFTMAX_FORWARD) X(CCV_NNC_SOFTMAX_BACKWARD) \
	X(CCV_NNC_BATCH_NORM_FORWARD) X(CCV_NNC_BATCH_NORM_BACKWARD) \
	X(CCV_NNC_LAYER_NORM_FORWARD) X(CCV_NNC_LAYER_NORM_BACKWARD) X(CCV_NNC_GROUP_NORM_FORWARD) X(CCV_NNC_GROUP_NORM_BACKWARD) \
	X(CCV_NNC_RMSNORM_FORWARD) X(CCV_NNC_RMSNORM_BACKWARD) \
	X(CCV_NNC_EWSUM_FORWARD) X(CCV_NNC_EWSUM_BACKWARD) \
	X(CCV_NNC_ADD_FORWARD) X(CCV_NNC_ADD_BACKWARD) \
	X(CCV_NNC_MUL_FORWARD) X(CCV_NNC_MUL_BACKWARD) \
	X(CCV_NNC_SCALAR_MUL_FORWARD) X(CCV_NNC_SCALAR_MUL_BACKWARD) \
	X(CCV_NNC_RELU_FORWARD) X(CCV_NNC_RELU_BACKWARD) \
	X(CCV_NNC_MAX_POOL_FORWARD) X(CCV_NNC_MAX_POOL_BACKWARD) \
	X(CCV_NNC_AVERAGE_POOL_FORWARD) X(CCV_NNC_AVERAGE_POOL_BACKWARD) \
	X(CCV_NNC_UPSAMPLE_FORWARD) X(CCV_NNC_UPSAMPLE_BACKWARD) \
	X(CCV_NNC_SET_FORWARD) X(CCV_NNC_SET_BACKWARD) \
	X(CCV_NNC_DATA_TRANSFER_FORWARD) X(CCV_NNC_DATA_TRANSFER_BACKWARD) \
	X(CCV_NNC_FORMAT_TRANSFORM_FORWARD) X(CCV_NNC_FORMAT_TRANSFORM_BACKWARD) \
	X(CCV_NNC_TRANSPOSE_FORWARD) X(CCV_NNC_TRANSPOSE_BACKWARD) \
	X(CCV_NNC_DATATYPE_CONVERSION_FORWARD) X(CCV_NNC_DATATYPE_CONVERSION_BACKWARD) \
	X(CCV_NNC_SGD_FORWARD) X(CCV_NNC_SGD_BACKWARD) \
	X(CCV_NNC_ADAMW_FORWARD) X(CCV_NNC_ADAMW_BACKWARD) \
	X(CCV_NNC_GELU_FORWARD) X(CCV_NNC_GELU_BACKWARD) X(CCV_NNC_SWISH_FORWARD) X(CCV_NNC_SWISH_BACKWARD) \
	X(CCV_NNC_INDEX_SELECT_FORWARD) X(CCV_NNC_INDEX_SELECT_BACKWARD) \
	X(CCV_NNC_CATEGORICAL_CROSSENTROPY_FORWARD) X(CCV_NNC_CATEGORICAL_CROSSENTROPY_BACKWARD) \
	X(CCV_NNC_SOFTMAX_CROSSENTROPY_FORWARD) X(CCV_NNC_SOFTMAX_CROSSENTROPY_BACKWARD) \
	X(CCV_NNC_COMM_ALLREDUCE_FORWARD) X(CCV_NNC_COMM_ALLREDUCE_BACKWARD) \
	X(CCV_NNC_SIGMOID_FORWARD) X(CCV_NNC_SIGMOID_BACKWARD) X(CCV_NNC_TANH_FORWARD) X(CCV_NNC_TANH_BACKWARD) X(CCV_NNC_LEAKY_RELU_FORWARD) X(CCV_NNC_LEAKY_RELU_BACKWARD) X(CCV_NNC_EWEXP_FORWARD) X(CCV_NNC_EWEXP_BACKWARD) X(CCV_NNC_EWLOG_FORWARD) X(CCV_NNC_EWLOG_BACKWARD) X(CCV_NNC_EWSQRT_FORWARD) X(CCV_NNC_EWSQRT_BACKWARD) X(CCV_NNC_CLAMP_FORWARD) X(CCV_NNC_CLAMP_BACKWARD) \
	X(CCV_NNC_EWDIV_FORWARD) X(CCV_NNC_EWDIV_BACKWARD) X(CCV_NNC_REDUCE_SUM_FORWARD) X(CCV_NNC_REDUCE_SUM_BACKWARD) X(CCV_NNC_REDUCE_MEAN_FORWARD) X(CCV_NNC_REDUCE_MEAN_BACKWARD) X(CCV_NNC_REDUCE_MAX_FORWARD) X(CCV_NNC_REDUCE_MAX_BACKWARD) X(CCV_NNC_REDUCE_MIN_FORWARD) X(CCV_NNC_REDUCE_MIN_BACKWARD) X(CCV_NNC_REDUCE_NORM2_FORWARD) X(CCV_NNC_REDUCE_NORM2_BACKWARD) X(CCV_NNC_MASKED_FILL_FORWARD) X(CCV_NNC_MASKED_FILL_BACKWARD) \
	X(CCV_NNC_RANDOM_UNIFORM_FORWARD) X(CCV_NNC_RANDOM_UNIFORM_BACKWARD) X(CCV_NNC_RANDOM_NORMAL_FORWARD) X(CCV_NNC_RANDOM_NORMAL_BACKWARD) X(CCV_NNC_ADAM_FORWARD) X(CCV_NNC_ADAM_BACKWARD) X(CCV_NNC_DROPOUT_FORWARD) X(CCV_NNC_DROPOUT_BACKWARD)

#define CCV_SM100_DECLARE_REGISTER(cmd) void _register_command_ ## cmd ## _backend_CCV_NNC_BACKEND_GPU_SM100(ccv_nnc_cmd_backend_registry_t* const registry);
CCV_NNC_SM100_COMMANDS(CCV_SM100_DECLARE_REGISTER)
#undef CCV_SM100_DECLARE_REGISTER

/* What the backend needs back from its host (ccv's own when linked into libccv: lib/nnc/gpu/ccv_nnc_compat.h:95-97,
 * lib/nnc/ccv_nnc.h:955).  get_stream returns the cudaStream_t as void* so that this header stays plain C. */
void* ccv_nnc_stream_context_get_stream(const ccv_nnc_stream_context_t* const stream_context);
int ccv_nnc_stream_context_get_device(const ccv_nnc_stream_context_t* const stream_context);
void* ccv_nnc_stream_context_get_workspace(ccv_nnc_stream_context_t* const stream_context, const size_t workspace_size, const int mem);
/* lib/nnc/ccv_nnc.h / ccv_nnc_stream.c:247-281: the per-stream-context generator the random-fill commands draw their seed from */
uint32_t ccv_nnc_stream_context_genrand_uint32(ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_stream_context_set_seed(ccv_nnc_stream_context_t* const stream_context, uint32_t seed);

/* ------------------------------------------------------------------------------------------------------------ */
/* (B) HOST side, reference names and semantics.                                                                 */
/* ------------------------------------------------------------------------------------------------------------ */
/* lib/nnc/ccv_nnc.h:28 / ccv_nnc_cmd.c:27-30. Idempotent; runs every _register_command_*_backend_GPU_SM100.     */
void ccv_nnc_init(void);
/* lib/nnc/ccv_nnc.h:759 */
ccv_nnc_cmd_t ccv_nnc_cmd(const uint32_t cmd, ccv_nnc_cmd_vtab_t* const isa, const ccv_nnc_cmd_param_t params, const int flags);
/* lib/nnc/ccv_nnc.h:750: 1 if (cmd, backend) has an exec */
int ccv_nnc_cmd_ok(const uint32_t cmd, const uint32_t backend);
/* lib/nnc/ccv_nnc.h:795 / ccv_nnc_cmd.c:307-328 */
uint32_t ccv_nnc_cmd_find_backend(const ccv_nnc_cmd_t cmd, const int tensor_memory, const int tensor_formats, const int tensor_datatypes);
/* lib/nnc/ccv_nnc.h:842 / ccv_nnc_cmd.c:651-693. Returns CCV_NNC_EXEC_*.  Only enqueues; with stream_context == NULL
 * the per-thread default stream context is used and drained (workspace released) before returning. */
int ccv_nnc_cmd_exec(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);
/* lib/nnc/ccv_nnc.h:776 / ccv_nnc_cmd.c: guess stride/border from the shapes of a and b */
ccv_nnc_hint_t ccv_nnc_hint_auto(const ccv_nnc_cmd_param_t cmd, const ccv_nnc_tensor_param_t a, const ccv_nnc_tensor_param_t b);
uint64_t ccv_nnc_cmd_mono_time(void);

/* lib/nnc/ccv_nnc.h:574-636.  ptr == NULL allocates (cudaMalloc for GPU memory, 64-byte aligned host memory, pinned
 * on request); ptr != NULL wraps caller memory.  flags is accepted for source compatibility and ignored. */
ccv_nnc_tensor_t* ccv_nnc_tensor_new(const void* const ptr, const ccv_nnc_tensor_param_t params, const int flags);
void ccv_nnc_tensor_free(ccv_nnc_tensor_t* const tensor);
ccv_nnc_tensor_view_t* ccv_nnc_tensor_view_new(const ccv_nnc_tensor_t* const tensor, const ccv_nnc_tensor_param_t params, const int ofs[CCV_NNC_MAX_DIM_ALLOC], const int stride[CCV_NNC_MAX_DIM_ALLOC]);
void ccv_nnc_tensor_view_free(ccv_nnc_tensor_view_t* const tensor_view);
int ccv_nnc_tensor_pin_memory(ccv_nnc_tensor_t* const tensor);
size_t ccv_nnc_tensor_data_size(const ccv_nnc_tensor_param_t params);
size_t ccv_nnc_tensor_data_size_without_padding(const ccv_nnc_tensor_param_t params);
/* lib/nnc/ccv_nnc_easy.h:210-217 (an inline function there): the parameters of a palettized (CCV_QX) copy of a CCV_16F / CCV_32F / CCV_64F
 * tensor: the datatype word carries qbits (4..8) and the palette type, `reserved` the number of elements that share one palette */
ccv_nnc_tensor_param_t ccv_nnc_tensor_palettize(const ccv_nnc_tensor_param_t params, const int qbits, const int number_in_blocks);
/* lib/nnc/ccv_nnc.h:916: decode output_length elements of `datatype` (CCV_16F, CCV_32F or CCV_64F) from a palettized buffer of
 * input_length bytes.  This library decodes GPU memory only (memory_type CCV_TENSOR_GPU_MEMORY), on the calling thread's default
 * stream; invalid parameters leave the output untouched and set ccv_nnc_sm100_last_error(). */
void ccv_nnc_depalettize(const void* input, const int datatype, const int memory_type, const size_t input_length, const int qbits, const int number_in_blocks, void* output, const size_t output_length);

/* lib/nnc/ccv_nnc.h:940-1100 */
ccv_nnc_stream_context_t* ccv_nnc_stream_context_new(const int type);
int ccv_nnc_stream_context_type(const ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_stream_context_drain(ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_stream_context_wait(const ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_stream_context_free(ccv_nnc_stream_context_t* const stream_context);
int ccv_nnc_device_count(const int type);
/* lib/nnc/ccv_nnc.h:1022-1064: a signal is emitted on one stream and waited for on another (device-side ordering, no host block) */
typedef struct ccv_nnc_stream_signal_s ccv_nnc_stream_signal_t;
ccv_nnc_stream_signal_t* ccv_nnc_stream_signal_new(const int type);
int ccv_nnc_stream_signal_type(const ccv_nnc_stream_signal_t* const signal);
void ccv_nnc_stream_context_emit_signal(ccv_nnc_stream_context_t* const stream, ccv_nnc_stream_signal_t* const signal);
void ccv_nnc_stream_context_wait_signal(const ccv_nnc_stream_context_t* const stream, const ccv_nnc_stream_signal_t* const signal);
ccv_nnc_stream_context_t* ccv_nnc_stream_signal_get_emitter(const ccv_nnc_stream_signal_t* const signal);
void ccv_nnc_stream_signal_free(ccv_nnc_stream_signal_t* const signal);
typedef ccv_nnc_stream_context_t*(*ccv_nnc_stream_context_neighbor_discovery_f)(const int device_id, void* const context);
void ccv_nnc_stream_context_set_neighbor_discovery(ccv_nnc_stream_context_t* const stream_context, ccv_nnc_stream_context_neighbor_discovery_f discovery, void* const context);
ccv_nnc_stream_context_t* ccv_nnc_stream_context_find_neighbor(ccv_nnc_stream_context_t* const stream_context, const int device_id);

/* ------------------------------------------------------------------------------------------------------------ */
/* FFI conveniences (not in the reference): the same calls with every struct passed by pointer, for bindings      */
/* that cannot pass 152-byte structs by value (ctypes, cgo, JNI).                                                 */
/* ------------------------------------------------------------------------------------------------------------ */
/* lib/nnc/ccv_nnc.h:829 / ccv_nnc_cmd.c:399-600: pick the fastest algorithm of the backend for these operands (device-timed);
 * inputs / outputs are scratch.  The _sm100_ form takes the structs by pointer and returns the algorithm index.                */
ccv_nnc_cmd_t ccv_nnc_cmd_autotune(const ccv_nnc_cmd_t cmd, const size_t max_workspace_size, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_sm100_cmd_autotune(const uint32_t cmd, const ccv_nnc_cmd_param_t* const info, const ccv_nnc_hint_t* const hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context, int* const algorithm);
int ccv_nnc_sm100_cmd_exec(const uint32_t cmd, const uint32_t backend, const int algorithm, const ccv_nnc_cmd_param_t* const info, const ccv_nnc_hint_t* const hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context);
ccv_nnc_tensor_t* ccv_nnc_sm100_tensor_new(const void* const ptr, const ccv_nnc_tensor_param_t* const params);
ccv_nnc_tensor_view_t* ccv_nnc_sm100_tensor_view_new(const ccv_nnc_tensor_t* const tensor, const ccv_nnc_tensor_param_t* const params, const int* const ofs, const int* const stride);
void ccv_nnc_sm100_hint_auto(const ccv_nnc_cmd_param_t* const info, const ccv_nnc_tensor_param_t* const a, const ccv_nnc_tensor_param_t* const b, ccv_nnc_hint_t* const hint);
/* blocking copies between host memory and a GPU tensor's storage (what tests use to stage data) */
int ccv_nnc_sm100_memcpy_h2d(void* const dst_device, const void* const src_host, const size_t bytes, ccv_nnc_stream_context_t* const stream_context);
int ccv_nnc_sm100_memcpy_d2h(void* const dst_host, const void* const src_device, const size_t bytes, ccv_nnc_stream_context_t* const stream_context);
/* CUDA events on a stream context's stream, for device-side timing */
void* ccv_nnc_sm100_event_new(void);
int ccv_nnc_sm100_event_record(void* const event, ccv_nnc_stream_context_t* const stream_context);
float ccv_nnc_sm100_event_elapsed_ms(void* const begin, void* const end);
void ccv_nnc_sm100_event_free(void* const event);
/* ccv_nnc_depalettize of GPU memory on a stream context's stream (NULL: the calling thread's default stream); 0, or -1 when the
 * parameters are refused (the output is then untouched) or the launch failed */
int ccv_nnc_sm100_depalettize(const void* input, const int datatype, const size_t input_length, const int qbits, const int number_in_blocks, void* output, const size_t output_length, ccv_nnc_stream_context_t* const stream_context);
/* number of kernels this backend has launched since process start (bench.py's gpu_launches) */
uint64_t ccv_nnc_sm100_launch_count(void);
/* last CUDA error string seen by the backend (empty if none) */
const char* ccv_nnc_sm100_last_error(void);

/* Communicators behind CCV_NNC_COMM_ALLREDUCE_* (replaces ccv_nnc_nccl_get_comm, lib/nnc/gpu/ccv_nnc_compat.cu:1415-1445).
 * One process per GPU: rank 0 calls _comm_unique_id (128 bytes), ships the id to the other ranks over the host's own side
 * channel, every rank calls _comm_init_rank after selecting its device; COMM_ALLREDUCE on tensors of this device then
 * sums across ranks.  One process, P devices (the reference's shape: tensor i on device i) needs no call at all, the
 * communicators are created on first use.  NCCL is dlopen'ed on first use.  Return 0 on success.                       */
int ccv_nnc_sm100_comm_unique_id(void* const id, const size_t size);
int ccv_nnc_sm100_comm_init_rank(const void* const id, const size_t size, const int world, const int rank);
int ccv_nnc_sm100_comm_rank(void);
int ccv_nnc_sm100_comm_world(void);
void ccv_nnc_sm100_comm_destroy(void);

/* A flat, topologically ordered command list: the slice of ccv_nnc_graph_t that ccv_nnc_graph_run's sync path
 * executes (lib/nnc/ccv_nnc_graph_run.c:911-979: for each exec_info -> ccv_nnc_cmd_exec).  Optionally captured into
 * a CUDA graph so that a whole forward+backward step is one launch from the host's point of view. */
typedef struct ccv_nnc_sm100_graph_s ccv_nnc_sm100_graph_t;
ccv_nnc_sm100_graph_t* ccv_nnc_sm100_graph_new(void);
int ccv_nnc_sm100_graph_exec_new(ccv_nnc_sm100_graph_t* const graph, const uint32_t cmd, const uint32_t backend, const int algorithm, const ccv_nnc_cmd_param_t* const info, const ccv_nnc_hint_t* const hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size);
int ccv_nnc_sm100_graph_size(const ccv_nnc_sm100_graph_t* const graph);
/* node i runs on the graph's side stream: forked after everything issued before it, joined at the end of the run (gradient-bucket allreduce) */
int ccv_nnc_sm100_graph_exec_set_side_stream(ccv_nnc_sm100_graph_t* const graph, const int i, const int side);
/* runs nodes [begin, end) in order on the stream; returns the first non-zero exec status */
int ccv_nnc_sm100_graph_run(ccv_nnc_sm100_graph_t* const graph, const int begin, const int end, ccv_nnc_stream_context_t* const stream_context);
/* peephole fusion of adjacent nodes (BN+ReLU forward, ReLU+BN backward, residual add + ReLU forward / backward); node
 * indices change, so call it before choosing capture ranges. Returns the number of pairs fused. */
int ccv_nnc_sm100_graph_fuse(ccv_nnc_sm100_graph_t* const graph);
/* introspection and per-node device timing (CUDA events, best of reps) of the (possibly fused) node list;
 * fused_kind: 0 plain command, 1 bn+relu forward, 2 relu+bn backward, 3 add+relu forward, 4 add+relu backward,
 * 5 a run of SGD commands as one multi-tensor launch, 6 convolution forward that also produces the batch-norm statistics of
 * its output (extra output: the statistics tensor), 7 batch-norm forward consuming them (extra input), 8 batch-norm backward
 * that also writes the bias gradient of the convolution in front of it (extra output; kind 2 may carry it too) */
int ccv_nnc_sm100_graph_node(const ccv_nnc_sm100_graph_t* const graph, const int i, uint32_t* const cmd, int* const fused_kind, int* const input_size, int* const output_size);
void* ccv_nnc_sm100_graph_node_tensor(const ccv_nnc_sm100_graph_t* const graph, const int i, const int is_output, const int k);
int ccv_nnc_sm100_graph_profile(ccv_nnc_sm100_graph_t* const graph, ccv_nnc_stream_context_t* const stream_context, const int reps, float* const ms);
/* capture nodes [begin, end) into a CUDA graph (id returned, <0 on failure) / replay it */
int ccv_nnc_sm100_graph_capture(ccv_nnc_sm100_graph_t* const graph, const int begin, const int end, ccv_nnc_stream_context_t* const stream_context);
int ccv_nnc_sm100_graph_replay(ccv_nnc_sm100_graph_t* const graph, const int capture_id, ccv_nnc_stream_context_t* const stream_context);
void ccv_nnc_sm100_graph_free(ccv_nnc_sm100_graph_t* const graph);

#ifdef __cplusplus
}
#endif

#endif
