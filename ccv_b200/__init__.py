"""ccv_b200: an H100-native (sm_90a) compute-command backend, CCV_NNC_BACKEND_GPU_SM100, behind liuliu/ccv's own nnc
command API (ccv_nnc_cmd_exec / ccv_nnc_tensor_t / ccv_nnc_stream_context_t).  The product is the C-ABI shared library
ccv_b200/libccv_nnc_sm100.so (sources in ccv_b200/csrc, interface in include/ccv_nnc_sm100.h); this package is the
thin ctypes host-side mirror used by the tests and the benchmark.  There is no CPU fallback anywhere in here."""
from . import abi  # noqa: F401
