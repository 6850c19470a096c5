"""ctypes mirror of include/ccv_nnc_sm100.h (which itself restates lib/nnc/ccv_nnc.h:111-306 and
lib/nnc/ccv_nnc_tfb.h:60-111 of the reference).  Sizes are asserted against SURVEY.md 0.10."""
import ctypes as C

MAX_DIM_ALLOC = 12

# datatypes (lib/ccv.h:45-54)
CCV_8U, CCV_32S, CCV_32F, CCV_64S, CCV_64F, CCV_16F, CCV_QX, CCV_16BF = 0x01000, 0x02000, 0x04000, 0x08000, 0x10000, 0x20000, 0x40000, 0x80000
# formats / memory (lib/nnc/ccv_nnc_tfb.h:26-36)
CCV_TENSOR_FORMAT_NCHW, CCV_TENSOR_FORMAT_NHWC, CCV_TENSOR_FORMAT_CHWN = 0x01, 0x02, 0x04
CCV_TENSOR_CPU_MEMORY, CCV_TENSOR_GPU_MEMORY = 0x1, 0x2
CCV_TENSOR_VIEW = 0x01000000
CCV_STREAM_CONTEXT_CPU, CCV_STREAM_CONTEXT_GPU = 0x1, 0x2
# exec flags / status (lib/nnc/ccv_nnc.h:69-79)
CCV_NNC_ACCUMULATE_OUTPUT, CCV_NNC_ZERO_MEMORY_ALLOC = 0x01, 0x02
CCV_NNC_EXEC_SUCCESS, CCV_NNC_EXEC_INVALID, CCV_NNC_EXEC_NO_KERNEL, CCV_NNC_EXEC_OOM = 0, -1, -2, -3
CCV_NNC_UPSAMPLE_NEAREST, CCV_NNC_UPSAMPLE_BILINEAR = 0, 1
CCV_NNC_MSE_REDUCE_MEAN, CCV_NNC_MSE_REDUCE_SUM = 0, 1  # lib/nnc/ccv_nnc.h:81-84 (cmd.info.mse.reduce_op)
CCV_NNC_PAD_ZERO, CCV_NNC_PAD_REPLICATE = 0, 1  # lib/nnc/ccv_nnc.h:97-100 (cmd.info.pad.type)
CCV_NNC_HISTOGRAM_EVEN, CCV_NNC_HISTOGRAM_LOGARITHMIC, CCV_NNC_HISTOGRAM_BINS = 0, 1, 2  # lib/nnc/ccv_nnc.h:86-90 (cmd.info.histogram.type)

# backends (lib/nnc/cmd/ccv_nnc_backend.h + the new one)
CCV_NNC_BACKEND_CPU_OPT = 0x46deb194
CCV_NNC_BACKEND_CPU_REF = 0x3d9883e5
CCV_NNC_BACKEND_GPU_SM100 = 0xdbfb784c
CCV_NNC_SM100_ALGO_TF32, CCV_NNC_SM100_ALGO_3XTF32, CCV_NNC_SM100_ALGO_FFMA = 0, 1, 2
CCV_NNC_SM100_SDPA_ALGO_COMPOSED, CCV_NNC_SM100_SDPA_ALGO_FLASH, CCV_NNC_SM100_SDPA_ALGO_FLASH_MASK = 0, 1, 2  # SCALED_DOT_PRODUCT_ATTENTION
CCV_NNC_SM100_SDPA_ALGO_COUNT = 3
CCV_NNC_GEMM_32F, CCV_NNC_GEMM_32TF, CCV_NNC_GEMM_16F = 0x1, 0x2, 0x4  # lib/nnc/ccv_nnc.h:102-106 (cmd.info.blas.flags)

# commands (lib/nnc/cmd/ccv_nnc_cmd.h)
CMD_IDS = dict(
    ADD=0x58fb3664, AVERAGE_POOL=0x51267ab8, BATCH_NORM=0x5419819c, CATEGORICAL_CROSSENTROPY=0x1eb327a2,
    COMM_ALLREDUCE=0x75c8d340, CONVOLUTION=0x254d05f4, CONVOLUTION_TRANSPOSE=0xd691f78e, DATATYPE_CONVERSION=0xd873e38c, DATA_TRANSFER=0x12d21e1a,
    EWSUM=0xe21a2c4c, FORMAT_TRANSFORM=0xe4a2b192, GEMM=0x7e87d00c, GROUP_NORM=0x17deb074, LAYER_NORM=0xbed3c264, MAX_POOL=0x7bec9360,
    MUL=0x24721a46, RELU=0xc51eaa80, RMSNORM=0x6889e9d0, SCALAR_MUL=0x8b4d86aa,
    SCALED_DOT_PRODUCT_ATTENTION=0x284ed926, SET=0x2b070804, SGD=0xe650ad26, SOFTMAX=0xc969a252,
    SOFTMAX_CROSSENTROPY=0xc26b7b5e, TRANSPOSE=0xb4d506e0, UPSAMPLE=0x73875556,
    ADAMW=0x4f5d4870, GELU=0xb1527ab8, SWISH=0x583d90c2, INDEX_SELECT=0x7ee7771e,
    SIGMOID=0xf2f69650, TANH=0x6a62be30, LEAKY_RELU=0x507144e0, EWEXP=0xd784b170, EWLOG=0xf4191bf2, EWSQRT=0x8870a61e, CLAMP=0x2640d854,
    EWDIV=0x1cd2fa18, REDUCE_SUM=0x52970f06, REDUCE_MEAN=0xf23556c6, REDUCE_MAX=0x80f1a506, REDUCE_MIN=0x6785ef96, REDUCE_NORM2=0xb3034e16,
    MASKED_FILL=0x7f992d84, DROPOUT=0x7f2dc3e4, ADAM=0xe30099dc, RANDOM_UNIFORM=0xa0cd1d5e, RANDOM_NORMAL=0x7062c8b4,
    CMUL=0xead486e6, BINARY_CROSSENTROPY=0xcd2107ec, SIGMOID_BINARY_CROSSENTROPY=0xd9e0e4a, MSE=0x6904a9a2, SMOOTH_L1=0x4e428e,
    PAD=0xd8aaca60, MIN=0x972fbd26, MAX=0xdf6f014c, ARGMAX=0x68af2804, ARGMIN=0xeb8747f2, REDUCE_ISNAN=0xee0a4ade,
    ROI_ALIGN=0xfef55168, NMS=0xdba26106, LAMB=0x450edb1a, RMSPROP=0x9c886b1c,
    COMPRESSION_LSSC=0x17ea8f72, HISTOGRAM=0xc5473e44, EWPROD=0xee07e8fe,
)
for _k, _v in CMD_IDS.items():
    globals()["CCV_NNC_%s_FORWARD" % _k] = _v
    globals()["CCV_NNC_%s_BACKWARD" % _k] = _v | 1


class TensorParam(C.Structure):
    _fields_ = [("type", C.c_int), ("format", C.c_int), ("datatype", C.c_int), ("reserved", C.c_int), ("dim", C.c_int * MAX_DIM_ALLOC)]


class Tensor(C.Structure):
    _fields_ = [("type", C.c_int), ("refcount", C.c_int), ("data", C.c_void_p), ("dataof", C.c_long), ("alias_ref", C.c_size_t),
                ("data_size", C.c_uint64), ("sig", C.c_uint64), ("info", TensorParam)]


class TensorView(C.Structure):
    _fields_ = Tensor._fields_ + [("contiguous", C.c_int), ("off", C.c_long), ("stride", C.c_int * MAX_DIM_ALLOC)]


class _Size(C.Structure):
    _fields_ = [("dim", C.c_int * MAX_DIM_ALLOC)]


class _Convolution(C.Structure):
    _fields_ = [("count", C.c_int), ("groups", C.c_int), ("dilation", C.c_int * MAX_DIM_ALLOC)]


class _ConvolutionTranspose(C.Structure):
    _fields_ = [("count", C.c_int), ("groups", C.c_int), ("dilation", C.c_int * MAX_DIM_ALLOC), ("output_padding", C.c_int)]


class _Pool(C.Structure):
    _fields_ = [("reserved", C.c_int)]


class _Bnorm(C.Structure):
    _fields_ = [("axis", C.c_int * MAX_DIM_ALLOC), ("count", C.c_int), ("epsilon", C.c_float), ("is_test", C.c_int), ("momentum", C.c_float)]


class _Lnorm(C.Structure):
    _fields_ = [("axis", C.c_int * MAX_DIM_ALLOC), ("count", C.c_int), ("epsilon", C.c_float), ("elementwise_affine", C.c_int)]


class _Gnorm(C.Structure):
    _fields_ = [("group_axis", C.c_int), ("reduce_axis", C.c_int * MAX_DIM_ALLOC), ("reduce_count", C.c_int), ("groups", C.c_int),
                ("epsilon", C.c_float), ("elementwise_affine", C.c_int)]


class _Rmsnorm(C.Structure):
    _fields_ = [("axis", C.c_int * MAX_DIM_ALLOC), ("count", C.c_int), ("epsilon", C.c_float)]


class _Sgd(C.Structure):
    _fields_ = [("nesterov", C.c_int), ("rate", C.c_float), ("scale", C.c_float), ("decay", C.c_float), ("momentum", C.c_float), ("dampening", C.c_float)]


class _Adam(C.Structure):
    _fields_ = [("step", C.c_int), ("rate", C.c_float), ("scale", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("decay", C.c_float), ("epsilon", C.c_float), ("amsgrad", C.c_int)]


class _Lamb(C.Structure):
    _fields_ = [("step", C.c_int), ("rate", C.c_float), ("scale", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("decay", C.c_float), ("epsilon", C.c_float)]


class _Rmsprop(C.Structure):
    _fields_ = [("rate", C.c_float), ("scale", C.c_float), ("decay", C.c_float), ("alpha", C.c_float), ("momentum", C.c_float), ("epsilon", C.c_float)]


class _Gelu(C.Structure):
    _fields_ = [("tanh", C.c_int)]


class _Blas(C.Structure):
    _fields_ = [("transpose_a", C.c_int * 2), ("transpose_b", C.c_int * 2), ("a", C.c_float * 3), ("flags", C.c_int)]


class _LabelSmoothing(C.Structure):
    _fields_ = [("trim0", C.c_float), ("trim1", C.c_float)]


class _Reduce(C.Structure):
    _fields_ = [("axis", C.c_int * MAX_DIM_ALLOC), ("count", C.c_int)]


class _Transpose(C.Structure):
    _fields_ = [("axis", C.c_int * 2)]


class _Upsample(C.Structure):
    _fields_ = [("type", C.c_int), ("width_scale", C.c_float), ("height_scale", C.c_float), ("align_corners", C.c_int)]


class _Sdpa(C.Structure):
    _fields_ = [("scale", C.c_float), ("is_causal", C.c_int), ("flags", C.c_int), ("deterministic", C.c_int)]


class _Clamp(C.Structure):
    _fields_ = [("min", C.c_float), ("max", C.c_float)]


class _Histogram(C.Structure):
    _fields_ = [("type", C.c_int), ("bins", C.c_int), ("min", C.c_float), ("max", C.c_float), ("rate", C.c_float)]


class _LeakyRelu(C.Structure):
    _fields_ = [("negative_slope", C.c_float)]


class _BinaryCrossentropy(C.Structure):
    _fields_ = [("pos_weight", C.c_float)]


class _SmoothL1(C.Structure):
    _fields_ = [("beta", C.c_float)]


class _Mse(C.Structure):
    _fields_ = [("reduce_op", C.c_int)]


class _Dropout(C.Structure):
    _fields_ = [("p", C.c_float), ("entirety", C.c_int)]


class _Nms(C.Structure):
    _fields_ = [("iou_threshold", C.c_float)]


class _Pad(C.Structure):
    _fields_ = [("type", C.c_int), ("end", C.c_int * MAX_DIM_ALLOC)]


class _CmdUnion(C.Union):
    _fields_ = [("convolution", _Convolution), ("convolution_transpose", _ConvolutionTranspose), ("pool", _Pool), ("bnorm", _Bnorm), ("lnorm", _Lnorm), ("gnorm", _Gnorm), ("rmsnorm", _Rmsnorm),
                ("sgd", _Sgd), ("adam", _Adam), ("lamb", _Lamb), ("rmsprop", _Rmsprop), ("gelu", _Gelu), ("blas", _Blas), ("label_smoothing", _LabelSmoothing), ("reduce", _Reduce), ("transpose", _Transpose),
                ("upsample", _Upsample), ("clamp", _Clamp), ("histogram", _Histogram), ("leaky_relu", _LeakyRelu), ("dropout", _Dropout), ("scaled_dot_product_attention", _Sdpa),
                ("binary_crossentropy", _BinaryCrossentropy), ("smooth_l1", _SmoothL1), ("mse", _Mse), ("nms", _Nms), ("pad", _Pad), ("userdata", C.c_void_p)]


class CmdParam(C.Structure):
    _anonymous_ = ("u",)
    _fields_ = [("size", _Size), ("u", _CmdUnion)]


class _Stride(C.Structure):
    _fields_ = [("dim", C.c_int * MAX_DIM_ALLOC)]


class _Border(C.Structure):
    _fields_ = [("begin", C.c_int * MAX_DIM_ALLOC), ("end", C.c_int * MAX_DIM_ALLOC)]


class Hint(C.Structure):
    _fields_ = [("stride", _Stride), ("border", _Border)]


class Cmd(C.Structure):
    _fields_ = [("cmd", C.c_uint32), ("backend", C.c_uint32), ("algorithm", C.c_int), ("info", CmdParam), ("isa", C.c_void_p), ("data", C.c_void_p)]


assert C.sizeof(TensorParam) == 64 and C.sizeof(Tensor) == 112 and C.sizeof(TensorView) == 176
assert C.sizeof(CmdParam) == 120 and C.sizeof(Hint) == 144 and C.sizeof(Cmd) == 152

DTYPE_SIZE = {CCV_8U: 1, CCV_32S: 4, CCV_32F: 4, CCV_64S: 8, CCV_64F: 8, CCV_16F: 2, CCV_16BF: 2}


def tensor_param(memory, fmt, datatype, dims, device=0):
    p = TensorParam()
    p.type = memory | ((device & 0xfff) << 8)
    p.format = fmt
    p.datatype = datatype
    for i, d in enumerate(dims):
        p.dim[i] = int(d)
    return p


def hint(stride=(1, 1), border=(0, 0), border_end=None):
    """HINT((sh, sw), (bh, bw)) of lib/nnc/ccv_nnc_easy.h: border applies to begin and end unless border_end is given."""
    h = Hint()
    for i, s in enumerate(stride):
        h.stride.dim[i] = int(s)
    for i, b in enumerate(border):
        h.border.begin[i] = int(b)
        h.border.end[i] = int(b)
    if border_end is not None:
        for i, b in enumerate(border_end):
            h.border.end[i] = int(b)
    return h


NO_HINT = Hint()
