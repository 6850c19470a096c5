// sm100_cmd.h -- host helpers shared by the files that implement commands on include/ccv_nnc_sm100.h: tensor queries, grid sizing
// and the registry entry of a command.
#pragma once
#include "../../include/ccv_nnc_sm100.h"
#include "sm100_contract.h"
#include <cuda_runtime.h>

namespace sm100 {

inline cudaStream_t stream_of(ccv_nnc_stream_context_t* const stream_context) { return (cudaStream_t)ccv_nnc_stream_context_get_stream(stream_context); }

// element kind of the kernels that exist for three floating-point types (ElemKind): 0 = fp32, 1 = bf16, 2 = fp16; -1 for every other
// type, palettized ones included (CCV_GET_DATA_TYPE keeps the CCV_QX bit)
inline int kind_of(const ccv_nnc_tensor_t* const t)
{
	switch (CCV_GET_DATA_TYPE(t->info.datatype))
	{
		case CCV_32F: return 0;
		case CCV_16BF: return 1;
		case CCV_16F: return 2;
	}
	return -1;
}
inline size_t elem_size(const int kind) { return kind == 0 ? 4 : 2; }

// the axes of t: its leading positive dimensions
inline int nd_of(const ccv_nnc_tensor_t* const t)
{
	int i;
	for (i = 0; i < CCV_NNC_MAX_DIM_ALLOC && t->info.dim[i] > 0; i++) {}
	return i;
}
// elements of t (1 for a tensor with no axes)
inline size_t count_of(const ccv_nnc_tensor_t* const t)
{
	size_t n = 1;
	for (int i = 0; i < CCV_NNC_MAX_DIM_ALLOC && t->info.dim[i] > 0; i++)
		n *= (size_t)t->info.dim[i];
	return n;
}
inline bool same_dims(const ccv_nnc_tensor_t* const a, const ccv_nnc_tensor_t* const b)
{
	for (int i = 0; i < CCV_NNC_MAX_DIM_ALLOC; i++)
	{
		if (a->info.dim[i] != b->info.dim[i])
			return false;
		if (a->info.dim[i] == 0)
			break;
	}
	return true;
}

// blocks of a grid-stride launch over `work` items, `threads` items per block: at most `waves` blocks per SM, at least one
inline int grid_for(const size_t work, const int threads, const int waves)
{
	size_t blocks = (work + threads - 1) / threads;
	const size_t cap = (size_t)sm_count() * waves;
	if (blocks > cap)
		blocks = cap;
	return blocks < 1 ? 1 : (int)blocks;
}

// the exec of a command the reference computes nothing for (the backward of an optimizer, an index or a histogram)
inline int exec_invalid(const ccv_nnc_cmd_t cmd, const ccv_nnc_hint_t hint, const int flags, ccv_nnc_tensor_t* const* const inputs, const int input_size, ccv_nnc_tensor_t* const* const outputs, const int output_size, ccv_nnc_stream_context_t* const stream_context)
{
	return CCV_NNC_EXEC_INVALID;
}

constexpr int ALL_FORMATS = CCV_TENSOR_FORMAT_NCHW | CCV_TENSOR_FORMAT_NHWC | CCV_TENSOR_FORMAT_CHWN;
// a registry entry of this backend: GPU memory, no autotune function, no aux
inline void fill(ccv_nnc_cmd_backend_registry_t* const registry, const int formats, const int datatypes, const int algorithms, const ccv_nnc_cmd_exec_f exec)
{
	registry->tensor_formats = formats;
	registry->tensor_datatypes = datatypes;
	registry->tensor_memory = CCV_TENSOR_GPU_MEMORY;
	registry->algorithms = algorithms;
	registry->exec = exec;
	registry->autotune = 0;
	registry->aux = 0;
}

} // namespace sm100

#define REGISTER_SM100(cmd) extern "C" void _register_command_ ## cmd ## _backend_CCV_NNC_BACKEND_GPU_SM100(ccv_nnc_cmd_backend_registry_t* const registry)
