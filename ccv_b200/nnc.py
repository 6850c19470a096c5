"""Host-side mirror of the reference's Level-1 API (lib/nnc/ccv_nnc.h) over libccv_nnc_sm100.so.

Names follow the reference: init / tensor_new / cmd_exec / stream_context_new ... plus CMD_* constructors in the
spirit of the generated lib/nnc/cmd/ccv_nnc_cmd_easy.h macros.  Everything here enqueues GPU work through the C ABI;
if the shared library (or a GPU) is missing the import/exec fails loudly - nothing is ever computed on the CPU."""
import ctypes as C
import os

import numpy as np

from . import abi
from .abi import *  # noqa: F401,F403  (re-export the constants)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libccv_nnc_sm100.so")
_lib = None


def lib():
    """Load the backend library; raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("ccv_b200: %s is missing - build it with __graft_entry__.build(); there is no fallback path" % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        vp, i32, u32, sz = C.c_void_p, C.c_int, C.c_uint32, C.c_size_t
        l.ccv_nnc_init.restype = None
        l.ccv_nnc_sm100_cmd_exec.restype = i32
        l.ccv_nnc_sm100_cmd_exec.argtypes = [u32, u32, i32, C.POINTER(abi.CmdParam), C.POINTER(abi.Hint), i32, C.POINTER(vp), i32, C.POINTER(vp), i32, vp]
        l.ccv_nnc_sm100_tensor_new.restype = vp
        l.ccv_nnc_sm100_tensor_new.argtypes = [vp, C.POINTER(abi.TensorParam)]
        l.ccv_nnc_sm100_tensor_view_new.restype = vp
        l.ccv_nnc_sm100_tensor_view_new.argtypes = [vp, C.POINTER(abi.TensorParam), C.POINTER(i32), C.POINTER(i32)]
        l.ccv_nnc_tensor_free.argtypes = [vp]
        l.ccv_nnc_tensor_view_free.argtypes = [vp]
        l.ccv_nnc_tensor_pin_memory.argtypes = [vp]
        l.ccv_nnc_cmd_ok.restype = i32
        l.ccv_nnc_cmd_ok.argtypes = [u32, u32]
        l.ccv_nnc_stream_context_new.restype = vp
        l.ccv_nnc_stream_context_new.argtypes = [i32]
        l.ccv_nnc_stream_context_wait.argtypes = [vp]
        l.ccv_nnc_stream_context_free.argtypes = [vp]
        l.ccv_nnc_stream_context_drain.argtypes = [vp]
        l.ccv_nnc_stream_context_get_stream.restype = vp
        l.ccv_nnc_stream_context_get_stream.argtypes = [vp]
        l.ccv_nnc_device_count.restype = i32
        l.ccv_nnc_device_count.argtypes = [i32]
        l.ccv_nnc_sm100_memcpy_h2d.restype = i32
        l.ccv_nnc_sm100_memcpy_h2d.argtypes = [vp, vp, sz, vp]
        l.ccv_nnc_sm100_memcpy_d2h.restype = i32
        l.ccv_nnc_sm100_memcpy_d2h.argtypes = [vp, vp, sz, vp]
        l.ccv_nnc_sm100_event_new.restype = vp
        l.ccv_nnc_sm100_event_record.argtypes = [vp, vp]
        l.ccv_nnc_sm100_event_elapsed_ms.restype = C.c_float
        l.ccv_nnc_sm100_event_elapsed_ms.argtypes = [vp, vp]
        l.ccv_nnc_sm100_event_free.argtypes = [vp]
        l.ccv_nnc_sm100_launch_count.restype = C.c_uint64
        l.ccv_nnc_sm100_last_error.restype = C.c_char_p
        l.ccv_nnc_sm100_hint_auto.argtypes = [C.POINTER(abi.CmdParam), C.POINTER(abi.TensorParam), C.POINTER(abi.TensorParam), C.POINTER(abi.Hint)]
        l.ccv_nnc_sm100_graph_new.restype = vp
        l.ccv_nnc_sm100_graph_exec_new.restype = i32
        l.ccv_nnc_sm100_graph_exec_new.argtypes = [vp, u32, u32, i32, C.POINTER(abi.CmdParam), C.POINTER(abi.Hint), i32, C.POINTER(vp), i32, C.POINTER(vp), i32]
        l.ccv_nnc_sm100_graph_size.restype = i32
        l.ccv_nnc_sm100_graph_size.argtypes = [vp]
        l.ccv_nnc_sm100_graph_run.restype = i32
        l.ccv_nnc_sm100_graph_run.argtypes = [vp, i32, i32, vp]
        l.ccv_nnc_sm100_graph_fuse.restype = i32
        l.ccv_nnc_sm100_graph_fuse.argtypes = [vp]
        l.ccv_nnc_sm100_graph_node.restype = i32
        l.ccv_nnc_sm100_graph_node.argtypes = [vp, i32, C.POINTER(u32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
        l.ccv_nnc_sm100_graph_node_tensor.restype = vp
        l.ccv_nnc_sm100_graph_node_tensor.argtypes = [vp, i32, i32, i32]
        l.ccv_nnc_sm100_graph_profile.restype = i32
        l.ccv_nnc_sm100_graph_profile.argtypes = [vp, vp, i32, C.POINTER(C.c_float)]
        l.ccv_nnc_sm100_graph_capture.restype = i32
        l.ccv_nnc_sm100_graph_capture.argtypes = [vp, i32, i32, vp]
        l.ccv_nnc_sm100_graph_replay.restype = i32
        l.ccv_nnc_sm100_graph_replay.argtypes = [vp, i32, vp]
        l.ccv_nnc_sm100_graph_free.argtypes = [vp]
        l.ccv_nnc_stream_signal_new.restype = vp
        l.ccv_nnc_stream_signal_new.argtypes = [i32]
        l.ccv_nnc_stream_context_emit_signal.argtypes = [vp, vp]
        l.ccv_nnc_stream_context_wait_signal.argtypes = [vp, vp]
        l.ccv_nnc_stream_signal_free.argtypes = [vp]
        l.ccv_nnc_sm100_cmd_autotune.restype = None
        l.ccv_nnc_sm100_cmd_autotune.argtypes = [u32, C.POINTER(abi.CmdParam), C.POINTER(abi.Hint), i32, C.POINTER(vp), i32, C.POINTER(vp), i32, vp, C.POINTER(i32)]
        l.ccv_nnc_sm100_comm_unique_id.restype = i32
        l.ccv_nnc_sm100_comm_unique_id.argtypes = [vp, sz]
        l.ccv_nnc_sm100_comm_init_rank.restype = i32
        l.ccv_nnc_sm100_comm_init_rank.argtypes = [vp, sz, i32, i32]
        l.ccv_nnc_sm100_comm_rank.restype = i32
        l.ccv_nnc_sm100_comm_world.restype = i32
        l.ccv_nnc_tensor_palettize.restype = abi.TensorParam
        l.ccv_nnc_tensor_palettize.argtypes = [abi.TensorParam, i32, i32]
        l.ccv_nnc_tensor_data_size.restype = sz
        l.ccv_nnc_tensor_data_size.argtypes = [abi.TensorParam]
        l.ccv_nnc_tensor_data_size_without_padding.restype = sz
        l.ccv_nnc_tensor_data_size_without_padding.argtypes = [abi.TensorParam]
        l.ccv_nnc_depalettize.restype = None
        l.ccv_nnc_depalettize.argtypes = [vp, i32, i32, sz, i32, i32, vp, sz]
        l.ccv_nnc_sm100_depalettize.restype = i32
        l.ccv_nnc_sm100_depalettize.argtypes = [vp, i32, sz, i32, i32, vp, sz, vp]
        _lib = l
    return _lib


def init():
    lib().ccv_nnc_init()


NP_DTYPE = {abi.CCV_32F: np.float32, abi.CCV_32S: np.int32, abi.CCV_64F: np.float64, abi.CCV_16F: np.float16, abi.CCV_8U: np.uint8, abi.CCV_16BF: np.uint16}


class Tensor(object):
    """A ccv_nnc_tensor_t* (or view) owned by the backend library."""

    def __init__(self, ptr, params, is_view=False, owner=None):
        self.ptr = ptr
        self.params = params
        self.is_view = is_view
        self._owner = owner  # keep the viewed tensor alive
        self.dims = [d for d in params.dim if d > 0] if params.dim[0] > 0 else []
        nd = 0
        while nd < abi.MAX_DIM_ALLOC and params.dim[nd] > 0:
            nd += 1
        self.dims = [params.dim[i] for i in range(nd)]

    @property
    def struct(self):
        return C.cast(self.ptr, C.POINTER(abi.TensorView if self.is_view else abi.Tensor)).contents

    @property
    def data_ptr(self):
        return self.struct.data

    @property
    def count(self):
        n = 1
        for d in self.dims:
            n *= d
        return n

    @property
    def is_palettized(self):
        return (self.params.datatype & 0xFF000) == abi.CCV_QX

    @property
    def nbytes(self):
        if self.is_palettized:
            return lib().ccv_nnc_tensor_data_size_without_padding(self.params)
        return self.count * abi.DTYPE_SIZE[self.params.datatype & 0xFF000]

    @property
    def on_gpu(self):
        return (self.params.type & 0x3) == abi.CCV_TENSOR_GPU_MEMORY

    def free(self):
        if self.ptr:
            if self.is_view:
                lib().ccv_nnc_tensor_view_free(self.ptr)
            else:
                lib().ccv_nnc_tensor_free(self.ptr)
            self.ptr = None

    # --- staging helpers (blocking copies; tests and benchmark set-up only) -------------------------------
    def upload(self, array, stream=None):
        """A palettized tensor takes its packed bytes (a uint8 array of nbytes, tests/palette_ref.py makes them)."""
        if self.is_palettized:
            a = np.ascontiguousarray(array, dtype=np.uint8).reshape(-1)
            assert a.size == self.nbytes, (a.size, self.nbytes)
        else:
            a = np.ascontiguousarray(array, dtype=NP_DTYPE[self.params.datatype & 0xFF000])
            assert a.size == self.count, (a.shape, self.dims)
        if self.on_gpu:
            rc = lib().ccv_nnc_sm100_memcpy_h2d(self.data_ptr, a.ctypes.data, a.nbytes, stream.ptr if stream else None)
            if rc != 0:
                raise RuntimeError("h2d copy failed: %s" % lib().ccv_nnc_sm100_last_error())
        else:
            C.memmove(self.data_ptr, a.ctypes.data, a.nbytes)
        return self

    def download(self, stream=None):
        if self.is_palettized:
            out = np.empty(self.nbytes, dtype=np.uint8)
        else:
            out = np.empty(self.dims, dtype=NP_DTYPE[self.params.datatype & 0xFF000])
        if self.on_gpu:
            rc = lib().ccv_nnc_sm100_memcpy_d2h(out.ctypes.data, self.data_ptr, out.nbytes, stream.ptr if stream else None)
            if rc != 0:
                raise RuntimeError("d2h copy failed: %s" % lib().ccv_nnc_sm100_last_error())
        else:
            C.memmove(out.ctypes.data, self.data_ptr, out.nbytes)
        return out


def tensor_new(params, ptr=None):
    """ccv_nnc_tensor_new (lib/nnc/ccv_nnc.h:574)."""
    p = lib().ccv_nnc_sm100_tensor_new(ptr, C.byref(params))
    if not p:
        raise MemoryError("ccv_nnc_tensor_new failed: %s" % lib().ccv_nnc_sm100_last_error())
    return Tensor(p, params)


def gpu_tensor(dims, fmt=abi.CCV_TENSOR_FORMAT_NHWC, datatype=abi.CCV_32F, device=0, ptr=None):
    return tensor_new(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, fmt, datatype, dims, device), ptr)


def cpu_tensor(dims, fmt=abi.CCV_TENSOR_FORMAT_NHWC, datatype=abi.CCV_32F):
    return tensor_new(abi.tensor_param(abi.CCV_TENSOR_CPU_MEMORY, fmt, datatype, dims))


def palettize_param(params, qbits, number_in_blocks):
    """ccv_nnc_tensor_palettize (lib/nnc/ccv_nnc_easy.h:210-217): the parameters of a palettized copy of a CCV_16F / CCV_32F /
    CCV_64F tensor, qbits 4..8, `number_in_blocks` elements per palette."""
    return lib().ccv_nnc_tensor_palettize(params, qbits, number_in_blocks)


def gpu_palettized_tensor(dims, datatype, qbits, number_in_blocks, fmt=abi.CCV_TENSOR_FORMAT_NHWC, device=0):
    """A GPU tensor holding a palettized copy of a `datatype` tensor of `dims`; fill it with Tensor.upload(packed bytes)."""
    return tensor_new(palettize_param(abi.tensor_param(abi.CCV_TENSOR_GPU_MEMORY, fmt, datatype, dims, device), qbits, number_in_blocks))


def cpu_palettized_tensor(dims, datatype, qbits, number_in_blocks, fmt=abi.CCV_TENSOR_FORMAT_NHWC):
    return tensor_new(palettize_param(abi.tensor_param(abi.CCV_TENSOR_CPU_MEMORY, fmt, datatype, dims), qbits, number_in_blocks))


def tensor_data_size(params):
    """ccv_nnc_tensor_data_size: the bytes ccv_nnc_tensor_new allocates for `params` (64-byte padded)."""
    return lib().ccv_nnc_tensor_data_size(params)


def depalettize(src, dst, stream=None):
    """ccv_nnc_depalettize on GPU memory (ccv_nnc_sm100_depalettize on `stream`): decode palettized tensor `src` into the dense
    tensor `dst` of its palette type.  Returns 0, or -1 when the parameters are refused."""
    p = src.params
    return lib().ccv_nnc_sm100_depalettize(src.data_ptr, (p.datatype & 0xff) << 12, src.nbytes, (p.datatype >> 8) & 0xf, p.reserved, dst.data_ptr, src.count, stream.ptr if stream else None)


def tensor_view_new(tensor, dims, ofs, stride):
    """ccv_nnc_tensor_view_new (lib/nnc/ccv_nnc.h:622)."""
    params = abi.tensor_param(tensor.params.type & 0x3, tensor.params.format, tensor.params.datatype, dims, (tensor.params.type >> 8) & 0xfff)
    o = (C.c_int * abi.MAX_DIM_ALLOC)(*list(ofs))
    s = (C.c_int * abi.MAX_DIM_ALLOC)(*list(stride))
    p = lib().ccv_nnc_sm100_tensor_view_new(tensor.ptr, C.byref(params), o, s)
    return Tensor(p, params, is_view=True, owner=tensor)


class Stream(object):
    """ccv_nnc_stream_context_t* (lib/nnc/ccv_nnc.h:940)."""

    def __init__(self, device=0):
        self.ptr = lib().ccv_nnc_stream_context_new(abi.CCV_STREAM_CONTEXT_GPU | ((device & 0xfff) << 8))
        if not self.ptr:
            raise RuntimeError("ccv_nnc_stream_context_new failed: %s" % lib().ccv_nnc_sm100_last_error())

    def wait(self):
        lib().ccv_nnc_stream_context_wait(self.ptr)

    @property
    def cuda_stream(self):
        return lib().ccv_nnc_stream_context_get_stream(self.ptr)

    def set_neighbors(self, streams):
        """ccv_nnc_stream_context_set_neighbor_discovery (lib/nnc/ccv_nnc.h:1009-1020): `streams` maps device id -> Stream; the
        multi-device COMM_ALLREDUCE looks its per-device streams up through this, as the graph runner wires it
        (lib/nnc/ccv_nnc_graph_run.c:507-512)."""
        table = dict((int(d), st.ptr) for d, st in streams.items())
        cb_t = C.CFUNCTYPE(C.c_void_p, C.c_int, C.c_void_p)
        self._neighbor_cb = cb_t(lambda device, ctx: table.get(int(device)))
        lib().ccv_nnc_stream_context_set_neighbor_discovery.argtypes = [C.c_void_p, cb_t, C.c_void_p]
        lib().ccv_nnc_stream_context_set_neighbor_discovery(self.ptr, self._neighbor_cb, None)

    def free(self):
        if self.ptr:
            lib().ccv_nnc_stream_context_free(self.ptr)
            self.ptr = None


class Signal(object):
    """ccv_nnc_stream_signal_t (lib/nnc/ccv_nnc.h:1022-1064): emitted on one stream, waited for on another."""

    def __init__(self, device=0):
        self.ptr = lib().ccv_nnc_stream_signal_new(abi.CCV_STREAM_CONTEXT_GPU | (device << 8))
        if not self.ptr:
            raise RuntimeError("ccv_nnc_stream_signal_new failed")

    def emit(self, stream):
        lib().ccv_nnc_stream_context_emit_signal(stream.ptr, self.ptr)

    def wait(self, stream):
        lib().ccv_nnc_stream_context_wait_signal(stream.ptr, self.ptr)

    def free(self):
        if self.ptr:
            lib().ccv_nnc_stream_signal_free(self.ptr)
            self.ptr = None


class Event(object):
    """A CUDA event recorded on a Stream (device-side timing)."""

    def __init__(self):
        self.ptr = lib().ccv_nnc_sm100_event_new()

    def record(self, stream):
        if lib().ccv_nnc_sm100_event_record(self.ptr, stream.ptr if stream else None) != 0:
            raise RuntimeError("cudaEventRecord failed")
        return self

    def elapsed_ms(self, end):
        """milliseconds from this event to `end` (waits for `end`)."""
        return float(lib().ccv_nnc_sm100_event_elapsed_ms(self.ptr, end.ptr))

    def free(self):
        if self.ptr:
            lib().ccv_nnc_sm100_event_free(self.ptr)
            self.ptr = None


class Command(object):
    """ccv_nnc_cmd_t: identifier + backend + algorithm + parameters (lib/nnc/ccv_nnc.h:296-306)."""

    def __init__(self, cmd, info=None, backend=abi.CCV_NNC_BACKEND_GPU_SM100, algorithm=-1):
        self.cmd = cmd
        self.info = info if info is not None else abi.CmdParam()
        self.backend = backend
        self.algorithm = algorithm


def _ptr_array(tensors):
    arr = (C.c_void_p * max(len(tensors), 1))()
    for i, t in enumerate(tensors):
        arr[i] = t.ptr if t is not None else None
    return arr


def cmd_exec(cmd, hint, flags, inputs, outputs, stream=None):
    """ccv_nnc_cmd_exec (lib/nnc/ccv_nnc.h:842). Returns the CCV_NNC_EXEC_* status."""
    return lib().ccv_nnc_sm100_cmd_exec(cmd.cmd, cmd.backend, cmd.algorithm, C.byref(cmd.info), C.byref(hint if hint is not None else abi.NO_HINT), flags,
                                        _ptr_array(inputs), len(inputs), _ptr_array(outputs), len(outputs), stream.ptr if stream else None)


def comm_unique_id():
    """128-byte NCCL id made by rank 0 (ccv_nnc_sm100_comm_unique_id); ship it to the other ranks, then comm_init_rank."""
    buf = C.create_string_buffer(128)
    if lib().ccv_nnc_sm100_comm_unique_id(buf, 128) != 0:
        raise RuntimeError("comm_unique_id failed: %s" % lib().ccv_nnc_sm100_last_error())
    return buf.raw


def comm_init_rank(unique_id, world, rank):
    """Binds this process's current CUDA device into the communicator CCV_NNC_COMM_ALLREDUCE_* uses."""
    buf = C.create_string_buffer(bytes(unique_id), 128)
    if lib().ccv_nnc_sm100_comm_init_rank(buf, 128, world, rank) != 0:
        raise RuntimeError("comm_init_rank failed: %s" % lib().ccv_nnc_sm100_last_error())


def cmd_autotune(cmd, hint, flags, inputs, outputs, stream=None):
    """ccv_nnc_cmd_autotune (lib/nnc/ccv_nnc.h:829): the backend times its algorithms on these (scratch) operands; returns
    a copy of `cmd` with .algorithm set to the fastest."""
    algo = C.c_int(-1)
    lib().ccv_nnc_sm100_cmd_autotune(cmd.cmd, C.byref(cmd.info), C.byref(hint if hint is not None else abi.NO_HINT), flags, _ptr_array(inputs), len(inputs),
                                     _ptr_array(outputs), len(outputs), stream.ptr if stream else None, C.byref(algo))
    return Command(cmd.cmd, info=cmd.info, backend=cmd.backend, algorithm=algo.value)


def launch_count():
    return int(lib().ccv_nnc_sm100_launch_count())


class Graph(object):
    """A flat, topologically ordered command list executed as lib/nnc/ccv_nnc_graph_run.c:911-979 does (one
    ccv_nnc_cmd_exec per node), optionally captured into CUDA graphs."""

    def __init__(self):
        self.ptr = lib().ccv_nnc_sm100_graph_new()
        self._keep = []

    def exec_new(self, cmd, hint, flags, inputs, outputs):
        self._keep.append((inputs, outputs))
        return lib().ccv_nnc_sm100_graph_exec_new(self.ptr, cmd.cmd, cmd.backend, cmd.algorithm, C.byref(cmd.info), C.byref(hint if hint is not None else abi.NO_HINT), flags,
                                                  _ptr_array(inputs), len(inputs), _ptr_array(outputs), len(outputs))

    def __len__(self):
        return lib().ccv_nnc_sm100_graph_size(self.ptr)

    def set_side_stream(self, node, side=True):
        """node runs on the graph's side stream (forked after what precedes it, joined at the end of the run)"""
        lib().ccv_nnc_sm100_graph_exec_set_side_stream.argtypes = [C.c_void_p, C.c_int, C.c_int]
        if lib().ccv_nnc_sm100_graph_exec_set_side_stream(self.ptr, node, 1 if side else 0) != 0:
            raise RuntimeError("set_side_stream: bad node index or graph already captured")

    def fuse(self):
        """Peephole fusion of adjacent commands (BN+ReLU, ReLU+BN backward, residual add + ReLU); returns the number of pairs."""
        return lib().ccv_nnc_sm100_graph_fuse(self.ptr)

    def nodes(self):
        """[(cmd id, fused kind, [input tensor pointers], [output tensor pointers])] of the current (possibly fused) list"""
        out = []
        for i in range(len(self)):
            cmd, fk, ni, no = C.c_uint32(), C.c_int(), C.c_int(), C.c_int()
            lib().ccv_nnc_sm100_graph_node(self.ptr, i, C.byref(cmd), C.byref(fk), C.byref(ni), C.byref(no))
            ins = [lib().ccv_nnc_sm100_graph_node_tensor(self.ptr, i, 0, k) for k in range(ni.value)]
            outs = [lib().ccv_nnc_sm100_graph_node_tensor(self.ptr, i, 1, k) for k in range(no.value)]
            out.append((cmd.value, fk.value, ins, outs))
        return out

    def profile(self, stream, reps=3):
        """per-node device milliseconds (CUDA events around each node, best of reps)"""
        ms = (C.c_float * max(len(self), 1))()
        lib().ccv_nnc_sm100_graph_profile(self.ptr, stream.ptr, reps, ms)
        return [float(x) for x in ms][:len(self)]

    def run(self, stream, begin=0, end=-1):
        return lib().ccv_nnc_sm100_graph_run(self.ptr, begin, end, stream.ptr)

    def capture(self, stream, begin=0, end=-1):
        cid = lib().ccv_nnc_sm100_graph_capture(self.ptr, begin, end, stream.ptr)
        if cid < 0:
            raise RuntimeError("CUDA graph capture failed: %s" % lib().ccv_nnc_sm100_last_error())
        return cid

    def replay(self, capture_id, stream):
        return lib().ccv_nnc_sm100_graph_replay(self.ptr, capture_id, stream.ptr)

    def free(self):
        if self.ptr:
            lib().ccv_nnc_sm100_graph_free(self.ptr)
            self.ptr = None


# ------------------------------------------------------------------------------------------------------------
# CMD_* constructors (lib/nnc/cmd/ccv_nnc_cmd_easy.h)
# ------------------------------------------------------------------------------------------------------------
def _size(info, dims):
    for i, d in enumerate(dims):
        info.size.dim[i] = int(d)


def CMD_GEMM_FORWARD(transpose_a=(0, 0), transpose_b=(0, 0), **kw):
    info = abi.CmdParam()
    _size(info, (1, 1, 1))
    info.blas.a[0], info.blas.a[1] = 1.0, 1.0
    info.blas.transpose_a[0], info.blas.transpose_a[1] = transpose_a
    info.blas.transpose_b[0], info.blas.transpose_b[1] = transpose_b
    return Command(abi.CCV_NNC_GEMM_FORWARD, info, **kw)


def CMD_GEMM_BACKWARD(transpose_a=(0, 0), transpose_b=(0, 0), **kw):
    c = CMD_GEMM_FORWARD(transpose_a, transpose_b, **kw)
    c.cmd = abi.CCV_NNC_GEMM_BACKWARD
    return c


def CMD_CONVOLUTION_FORWARD(groups, count, kh, kw_, channels, dilation=(1, 1), **kw):
    info = abi.CmdParam()
    _size(info, (kh, kw_, channels))
    info.convolution.count = count
    info.convolution.groups = groups
    info.convolution.dilation[0], info.convolution.dilation[1] = dilation
    return Command(abi.CCV_NNC_CONVOLUTION_FORWARD, info, **kw)


def CMD_CONVOLUTION_BACKWARD(groups, count, kh, kw_, channels, dilation=(1, 1), **kw):
    c = CMD_CONVOLUTION_FORWARD(groups, count, kh, kw_, channels, dilation, **kw)
    c.cmd = abi.CCV_NNC_CONVOLUTION_BACKWARD
    return c


def CMD_CONVOLUTION_TRANSPOSE_FORWARD(groups, count, output_padding, kh, kw_, channels, dilation=(1, 1), **kw):
    """Argument order of the reference macro (cmd/convolution/ccv_nnc_convolution.c:119): count = output channels."""
    info = abi.CmdParam()
    _size(info, (kh, kw_, channels))
    info.convolution_transpose.count = count
    info.convolution_transpose.groups = groups
    info.convolution_transpose.dilation[0], info.convolution_transpose.dilation[1] = dilation
    info.convolution_transpose.output_padding = output_padding
    return Command(abi.CCV_NNC_CONVOLUTION_TRANSPOSE_FORWARD, info, **kw)


def CMD_CONVOLUTION_TRANSPOSE_BACKWARD(groups, count, output_padding, kh, kw_, channels, dilation=(1, 1), **kw):
    c = CMD_CONVOLUTION_TRANSPOSE_FORWARD(groups, count, output_padding, kh, kw_, channels, dilation, **kw)
    c.cmd = abi.CCV_NNC_CONVOLUTION_TRANSPOSE_BACKWARD
    return c


def CMD_BATCH_NORM_FORWARD(epsilon, is_test, momentum, axes=(0, 1, 2), **kw):
    info = abi.CmdParam()
    _size(info, (1, 1, 1))
    for i, a in enumerate(axes):
        info.bnorm.axis[i] = a
    info.bnorm.count = len(axes)
    info.bnorm.epsilon = epsilon
    info.bnorm.is_test = is_test
    info.bnorm.momentum = momentum
    return Command(abi.CCV_NNC_BATCH_NORM_FORWARD, info, **kw)


def CMD_BATCH_NORM_BACKWARD(epsilon, is_test, momentum, axes=(0, 1, 2), **kw):
    c = CMD_BATCH_NORM_FORWARD(epsilon, is_test, momentum, axes, **kw)
    c.cmd = abi.CCV_NNC_BATCH_NORM_BACKWARD
    return c


def _simple(cmd_id, size=(1, 1, 1), **kw):
    info = abi.CmdParam()
    _size(info, size)
    return Command(cmd_id, info, **kw)


def CMD_RELU_FORWARD(**kw):
    return _simple(abi.CCV_NNC_RELU_FORWARD, **kw)


def CMD_RELU_BACKWARD(**kw):
    return _simple(abi.CCV_NNC_RELU_BACKWARD, **kw)


def CMD_EWSUM_FORWARD(**kw):
    return _simple(abi.CCV_NNC_EWSUM_FORWARD, **kw)


def CMD_EWSUM_BACKWARD(**kw):
    return _simple(abi.CCV_NNC_EWSUM_BACKWARD, **kw)


def CMD_MAX_POOL_FORWARD(kh, kw_, **kw):
    return _simple(abi.CCV_NNC_MAX_POOL_FORWARD, (kh, kw_, 1), **kw)


def CMD_MAX_POOL_BACKWARD(kh, kw_, **kw):
    return _simple(abi.CCV_NNC_MAX_POOL_BACKWARD, (kh, kw_, 1), **kw)


def CMD_AVERAGE_POOL_FORWARD(kh, kw_, **kw):
    return _simple(abi.CCV_NNC_AVERAGE_POOL_FORWARD, (kh, kw_, 1), **kw)


def CMD_AVERAGE_POOL_BACKWARD(kh, kw_, **kw):
    return _simple(abi.CCV_NNC_AVERAGE_POOL_BACKWARD, (kh, kw_, 1), **kw)


def CMD_SOFTMAX_FORWARD(**kw):
    return _simple(abi.CCV_NNC_SOFTMAX_FORWARD, **kw)


def CMD_SOFTMAX_BACKWARD(**kw):
    return _simple(abi.CCV_NNC_SOFTMAX_BACKWARD, **kw)


def _label_smoothing(cmd_id, trim0, trim1, **kw):
    c = _simple(cmd_id, **kw)
    c.info.label_smoothing.trim0 = trim0
    c.info.label_smoothing.trim1 = trim1
    return c


def CMD_CATEGORICAL_CROSSENTROPY_FORWARD(trim0=0.0, trim1=1.0, **kw):
    return _label_smoothing(abi.CCV_NNC_CATEGORICAL_CROSSENTROPY_FORWARD, trim0, trim1, **kw)


def CMD_CATEGORICAL_CROSSENTROPY_BACKWARD(trim0=0.0, trim1=1.0, **kw):
    return _label_smoothing(abi.CCV_NNC_CATEGORICAL_CROSSENTROPY_BACKWARD, trim0, trim1, **kw)


def CMD_SOFTMAX_CROSSENTROPY_FORWARD(trim0=0.0, trim1=1.0, **kw):
    return _label_smoothing(abi.CCV_NNC_SOFTMAX_CROSSENTROPY_FORWARD, trim0, trim1, **kw)


def CMD_SOFTMAX_CROSSENTROPY_BACKWARD(trim0=0.0, trim1=1.0, **kw):
    return _label_smoothing(abi.CCV_NNC_SOFTMAX_CROSSENTROPY_BACKWARD, trim0, trim1, **kw)


def CMD_GELU_FORWARD(tanh=0, **kw):
    c = _simple(abi.CCV_NNC_GELU_FORWARD, **kw)
    c.info.gelu.tanh = tanh
    return c


def CMD_GELU_BACKWARD(tanh=0, **kw):
    c = _simple(abi.CCV_NNC_GELU_BACKWARD, **kw)
    c.info.gelu.tanh = tanh
    return c


def CMD_SWISH_FORWARD(**kw):
    return _simple(abi.CCV_NNC_SWISH_FORWARD, **kw)


def CMD_SWISH_BACKWARD(**kw):
    return _simple(abi.CCV_NNC_SWISH_BACKWARD, **kw)


def CMD_INDEX_SELECT_FORWARD(**kw):
    return _simple(abi.CCV_NNC_INDEX_SELECT_FORWARD, **kw)


def CMD_INDEX_SELECT_BACKWARD(**kw):
    return _simple(abi.CCV_NNC_INDEX_SELECT_BACKWARD, **kw)


def CMD_ADAMW_FORWARD(step, rate, beta1, beta2, decay, epsilon, amsgrad=0, scale=1.0, **kw):
    c = _simple(abi.CCV_NNC_ADAMW_FORWARD, **kw)
    a = c.info.adam
    a.step, a.rate, a.scale, a.beta1, a.beta2, a.decay, a.epsilon, a.amsgrad = step, rate, scale, beta1, beta2, decay, epsilon, amsgrad
    return c


def CMD_SGD_FORWARD(nesterov, rate, scale, decay, momentum, dampening, **kw):
    c = _simple(abi.CCV_NNC_SGD_FORWARD, **kw)
    s = c.info.sgd
    s.nesterov, s.rate, s.scale, s.decay, s.momentum, s.dampening = nesterov, rate, scale, decay, momentum, dampening
    return c


def _blas(cmd_id, a0=1.0, a1=1.0, **kw):
    c = _simple(cmd_id, **kw)
    c.info.blas.a[0], c.info.blas.a[1] = a0, a1
    return c


def CMD_SET_FORWARD(value, **kw):
    return _blas(abi.CCV_NNC_SET_FORWARD, value, 0.0, **kw)


def CMD_ADD_FORWARD(p, q, **kw):
    return _blas(abi.CCV_NNC_ADD_FORWARD, p, q, **kw)


def CMD_ADD_BACKWARD(p, q, **kw):
    return _blas(abi.CCV_NNC_ADD_BACKWARD, p, q, **kw)


def CMD_MUL_FORWARD(p, **kw):
    return _blas(abi.CCV_NNC_MUL_FORWARD, p, 0.0, **kw)


def CMD_MUL_BACKWARD(p, **kw):
    return _blas(abi.CCV_NNC_MUL_BACKWARD, p, 0.0, **kw)


def CMD_SCALAR_MUL_FORWARD(p, **kw):
    return _blas(abi.CCV_NNC_SCALAR_MUL_FORWARD, p, 0.0, **kw)


def CMD_SCALAR_MUL_BACKWARD(p, **kw):
    return _blas(abi.CCV_NNC_SCALAR_MUL_BACKWARD, p, 0.0, **kw)


def CMD_COMM_ALLREDUCE_FORWARD(**kw):
    return _simple(abi.CCV_NNC_COMM_ALLREDUCE_FORWARD, **kw)


def CMD_DATA_TRANSFER_FORWARD(**kw):
    return _simple(abi.CCV_NNC_DATA_TRANSFER_FORWARD, **kw)


def CMD_FORMAT_TRANSFORM_FORWARD(**kw):
    return _simple(abi.CCV_NNC_FORMAT_TRANSFORM_FORWARD, **kw)


def CMD_DATATYPE_CONVERSION_FORWARD(**kw):
    return _simple(abi.CCV_NNC_DATATYPE_CONVERSION_FORWARD, **kw)


def CMD_TRANSPOSE_FORWARD(axis_a, axis_b, **kw):
    c = _simple(abi.CCV_NNC_TRANSPOSE_FORWARD, **kw)
    c.info.transpose.axis[0], c.info.transpose.axis[1] = axis_a, axis_b
    return c


# ---- element-wise family, reductions, masked fill (cmd/ew/ccv_nnc_ew.c, cmd/sigmoid, cmd/tanh, cmd/leaky_relu, cmd/reduce, cmd/util) ----
def _make_simple(name):
    def fwd(**kw):
        return _simple(getattr(abi, "CCV_NNC_%s_FORWARD" % name), **kw)

    def bwd(**kw):
        return _simple(getattr(abi, "CCV_NNC_%s_BACKWARD" % name), **kw)
    return fwd, bwd


CMD_SIGMOID_FORWARD, CMD_SIGMOID_BACKWARD = _make_simple("SIGMOID")
CMD_TANH_FORWARD, CMD_TANH_BACKWARD = _make_simple("TANH")
CMD_EWEXP_FORWARD, CMD_EWEXP_BACKWARD = _make_simple("EWEXP")
CMD_EWLOG_FORWARD, CMD_EWLOG_BACKWARD = _make_simple("EWLOG")
CMD_EWSQRT_FORWARD, CMD_EWSQRT_BACKWARD = _make_simple("EWSQRT")
CMD_EWDIV_FORWARD, CMD_EWDIV_BACKWARD = _make_simple("EWDIV")


def CMD_LEAKY_RELU_FORWARD(negative_slope, **kw):
    c = _simple(abi.CCV_NNC_LEAKY_RELU_FORWARD, **kw)
    c.info.leaky_relu.negative_slope = negative_slope
    return c


def CMD_LEAKY_RELU_BACKWARD(negative_slope, **kw):
    c = _simple(abi.CCV_NNC_LEAKY_RELU_BACKWARD, **kw)
    c.info.leaky_relu.negative_slope = negative_slope
    return c


def CMD_CLAMP_FORWARD(lo, hi, **kw):
    """lo / hi may be float('nan') for an open side (CMD_CLAMP_FORWARD(min, max), cmd/ew/ccv_nnc_ew.c)"""
    c = _simple(abi.CCV_NNC_CLAMP_FORWARD, **kw)
    c.info.clamp.min, c.info.clamp.max = lo, hi
    return c


def CMD_CLAMP_BACKWARD(lo, hi, **kw):
    c = _simple(abi.CCV_NNC_CLAMP_BACKWARD, **kw)
    c.info.clamp.min, c.info.clamp.max = lo, hi
    return c


def _reduce(cmd_id, axes, **kw):
    c = _simple(cmd_id, **kw)
    for i, a in enumerate(axes):
        c.info.reduce.axis[i] = a
    c.info.reduce.count = len(axes)
    return c


def _make_reduce(name):
    def fwd(*axes, **kw):
        return _reduce(getattr(abi, "CCV_NNC_REDUCE_%s_FORWARD" % name), axes, **kw)

    def bwd(*axes, **kw):
        return _reduce(getattr(abi, "CCV_NNC_REDUCE_%s_BACKWARD" % name), axes, **kw)
    return fwd, bwd


CMD_REDUCE_SUM_FORWARD, CMD_REDUCE_SUM_BACKWARD = _make_reduce("SUM")
CMD_REDUCE_MEAN_FORWARD, CMD_REDUCE_MEAN_BACKWARD = _make_reduce("MEAN")
CMD_REDUCE_MAX_FORWARD, CMD_REDUCE_MAX_BACKWARD = _make_reduce("MAX")
CMD_REDUCE_MIN_FORWARD, CMD_REDUCE_MIN_BACKWARD = _make_reduce("MIN")
CMD_REDUCE_NORM2_FORWARD, CMD_REDUCE_NORM2_BACKWARD = _make_reduce("NORM2")


def CMD_MASKED_FILL_FORWARD(eq, fill, **kw):
    c = _simple(abi.CCV_NNC_MASKED_FILL_FORWARD, **kw)
    c.info.blas.a[0], c.info.blas.a[1] = eq, fill
    return c


def CMD_MASKED_FILL_BACKWARD(eq, fill, **kw):
    c = _simple(abi.CCV_NNC_MASKED_FILL_BACKWARD, **kw)
    c.info.blas.a[0], c.info.blas.a[1] = eq, fill
    return c


def CMD_RANDOM_UNIFORM_FORWARD(lb, ub, **kw):
    c = _simple(abi.CCV_NNC_RANDOM_UNIFORM_FORWARD, **kw)
    c.info.blas.a[0], c.info.blas.a[1] = lb, ub
    return c


def CMD_RANDOM_NORMAL_FORWARD(std, mean, **kw):
    c = _simple(abi.CCV_NNC_RANDOM_NORMAL_FORWARD, **kw)
    c.info.blas.a[0], c.info.blas.a[1] = std, mean
    return c


def CMD_ADAM_FORWARD(step, rate, beta1, beta2, decay, epsilon, amsgrad=0, scale=1.0, **kw):
    c = CMD_ADAMW_FORWARD(step, rate, beta1, beta2, decay, epsilon, amsgrad, scale, **kw)
    c.cmd = abi.CCV_NNC_ADAM_FORWARD
    return c


def CMD_DROPOUT_FORWARD(p, entirety=0, **kw):
    c = _simple(abi.CCV_NNC_DROPOUT_FORWARD, **kw)
    c.info.dropout.p, c.info.dropout.entirety = p, entirety
    return c


def CMD_DROPOUT_BACKWARD(p, entirety=0, **kw):
    c = _simple(abi.CCV_NNC_DROPOUT_BACKWARD, **kw)
    c.info.dropout.p, c.info.dropout.entirety = p, entirety
    return c
