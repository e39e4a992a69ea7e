"""ctypes binding of libcds.so (the C ABI declared in include/cds.h).

No torch types cross this boundary: operators carry raw device pointers (``tensor.data_ptr()``),
sizes and strides; the stream is the integer ``cudaStream_t`` of ``torch.cuda.current_stream()``.
The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is NO fallback:
if the shared object is missing, ``load()`` raises and the CUDA sampling path fails loudly.
"""
import ctypes as C
import os

_LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "libcds.so")

ABI_VERSION = 12
OPF_BRANCH_SHIFT = 8   # cds_op.flags bits 8..15: branch index (independent chains run on parallel streams)
OPF_ONCE = 1          # cds_op.flags: run once per plan run (before its first iteration), not in every iteration
OP_CONV, OP_UPDATE, OP_LNMOD, OP_ATTN, OP_PREP, OP_CAST, OP_MHA = range(7)
OP_STASH, OP_UPDATE_BWD, OP_DGRAD, OP_WGRAD = 7, 8, 9, 10      # backward operators of a differentiable loop (csrc/grad.cuh)
OP_GN, OP_GN_BWD, OP_GUIDE = 11, 12, 13       # classifier guidance inside the loop (csrc/classifier.cuh)
OP_HEAD_GRAD = 14                             # QGPOClassifier's energy head and the seed of its backward (csrc/classifier.cuh)
ACT_NONE, ACT_MISH, ACT_SILU, ACT_GELU_TANH, ACT_MISH_SILU, ACT_LEAKY_RELU, ACT_GELU_ERF = range(7)
ACT_RELU = 7                                  # nn.ReLU (MLPNNClassifier's default activation): CDS_OP_STASH / CDS_OP_DGRAD
MATH_FP32, MATH_BF16_TC, MATH_TF32_TC = 0, 1, 2
TC_MODES = (MATH_BF16_TC, MATH_TF32_TC)
F32, BF16, TF32 = 0, 1, 2      # cds_dtype; TF32 = fp32 storage, values rounded to TF32 when written
ROW_FLOATS = 12

_f32p = C.c_void_p   # device pointers are passed as integers


class Vec(C.Structure):
    _fields_ = [("step", _f32p), ("step_stride", C.c_int64), ("sample", _f32p), ("sample_stride", C.c_int64)]


class ConvOp(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("L_in", C.c_int32), ("L_out", C.c_int32), ("C_in", C.c_int32), ("C_out", C.c_int32),
        ("taps", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32), ("phases", C.c_int32),
        ("in_batch_mod", C.c_int32),
        ("in_", _f32p), ("in_bstride", C.c_int64), ("in_lstride", C.c_int32),
        ("w", C.c_void_p),
        ("bias", Vec),
        ("groups", C.c_int32), ("gn_gamma", _f32p), ("gn_beta", _f32p), ("gn_eps", C.c_float),
        ("act", C.c_int32),
        ("scale", Vec), ("shift", Vec),
        ("res", _f32p), ("res_bstride", C.c_int64), ("res_lstride", C.c_int32), ("res_batch_mod", C.c_int32),
        ("res_in", _f32p), ("res_in_bstride", C.c_int64), ("res_in_lstride", C.c_int32), ("res_C", C.c_int32),
        ("res_w", C.c_void_p), ("res_bias", _f32p),
        ("out", _f32p), ("out_bstride", C.c_int64), ("out_lstride", C.c_int32),
        ("math", C.c_int32),
        ("in_dtype", C.c_int32), ("out_dtype", C.c_int32), ("res_dtype", C.c_int32), ("res_in_dtype", C.c_int32),
        ("sample_row_div", C.c_int32),
    ]


class LnModOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("eps", C.c_float),
                ("in_", _f32p), ("out", C.c_void_p), ("shift", _f32p), ("scale", _f32p), ("mod_bstride", C.c_int64),
                ("out_dtype", C.c_int32),
                # backward mode (dout != NULL)
                ("dout", _f32p), ("dout_bstride", C.c_int64), ("dout_lstride", C.c_int32), ("res", _f32p),
                ("gate", _f32p), ("gate_bstride", C.c_int64), ("gated", _f32p), ("gated_dtype", C.c_int32)]


class AttnOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("heads", C.c_int32),
                ("qkv", _f32p), ("out", C.c_void_p), ("out_dtype", C.c_int32), ("qkv_dtype", C.c_int32),
                ("dout", _f32p)]                      # backward mode (dout != NULL)


class MhaOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("Lq", C.c_int32), ("Lk", C.c_int32), ("C", C.c_int32), ("heads", C.c_int32),
                ("masked", C.c_int32), ("diag", C.c_int32),
                ("q", C.c_void_p), ("q_bstride", C.c_int64), ("q_lstride", C.c_int32),
                ("kv_step", C.c_void_p), ("kv_step_stride", C.c_int64), ("kv_step_lstride", C.c_int32),
                ("kv_sample", C.c_void_p), ("kv_sample_bstride", C.c_int64), ("kv_sample_lstride", C.c_int32),
                ("out", C.c_void_p), ("out_bstride", C.c_int64), ("out_lstride", C.c_int32),
                ("in_dtype", C.c_int32), ("out_dtype", C.c_int32)]


class PrepOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("row", C.c_int32), ("x", _f32p), ("xin", _f32p), ("noise", _f32p),
                ("coef", _f32p),
                ("gxin", _f32p), ("coef_iter_stride", C.c_int64)]      # backward mode (gxin != NULL): x += K3 * gxin


class CastOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C_in", C.c_int32), ("C_out", C.c_int32),
                ("in_", _f32p), ("out", C.c_void_p), ("out_dtype", C.c_int32)]


class UpdateOp(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("row", C.c_int32), ("x", _f32p),
        ("pred", _f32p), ("pred_uncond", _f32p), ("w_cfg", C.c_float), ("w_uncond", C.c_float),
        ("noise", _f32p), ("noise_slot_stride", C.c_int64), ("prior", _f32p), ("mask", _f32p), ("x_min", _f32p),
        ("x_max", _f32p),
        ("xhat_prev", _f32p), ("aux", _f32p), ("coef", _f32p), ("predict_noise", C.c_int32), ("final_clip", C.c_int32),
        ("x_cast", C.c_void_p), ("cast_C_in", C.c_int32), ("cast_C_out", C.c_int32), ("x_cast_dtype", C.c_int32),
        ("guide", _f32p), ("guide_s", _f32p),      # EDM kinds: D += guide_s[iter] * guide (NULL: no guidance term)
    ]


class StashOp(C.Structure):
    _fields_ = [("n", C.c_int64), ("act", C.c_int32), ("src", _f32p), ("dst", _f32p), ("dst_iter_stride", C.c_int64),
                ("act_out", _f32p), ("grad", _f32p)]          # backward mode: act_out = grad * act'(src)


class UpdateBwdOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("row", C.c_int32), ("gx", _f32p), ("gpred", _f32p),
                ("x", _f32p), ("x_iter_stride", C.c_int64), ("pred", _f32p), ("pred_iter_stride", C.c_int64),
                ("mask", _f32p), ("x_min", _f32p), ("x_max", _f32p), ("coef", _f32p), ("coef_iter_stride", C.c_int64),
                ("predict_noise", C.c_int32)]


class DgradOp(C.Structure):
    _fields_ = [("rows", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("dz", _f32p), ("ldz", C.c_int32),
                ("w", _f32p), ("ldw", C.c_int32), ("z", _f32p), ("z_iter_stride", C.c_int64),
                ("act", C.c_int32), ("accumulate", C.c_int32), ("out", _f32p), ("ldo", C.c_int32), ("out_sum", _f32p)]


class WgradOp(C.Structure):
    _fields_ = [("rows", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("dz", _f32p), ("ldz", C.c_int32),
                ("h", _f32p), ("h_iter_stride", C.c_int64), ("ldh", C.c_int32), ("act", C.c_int32),
                ("dw", _f32p), ("lddw", C.c_int32), ("db", _f32p), ("db_iter_stride", C.c_int64), ("accumulate", C.c_int32)]


class GnOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("groups", C.c_int32), ("eps", C.c_float),
                ("act", C.c_int32), ("h", _f32p), ("h_bstride", C.c_int64), ("h_lstride", C.c_int32),
                ("gamma", _f32p), ("beta", _f32p), ("vec", Vec),
                ("res", _f32p), ("res_bstride", C.c_int64), ("res_lstride", C.c_int32),
                ("out", _f32p), ("out_bstride", C.c_int64), ("out_lstride", C.c_int32), ("out_dtype", C.c_int32)]


class GnBwdOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("groups", C.c_int32), ("eps", C.c_float),
                ("act", C.c_int32), ("h", _f32p), ("h_bstride", C.c_int64), ("h_lstride", C.c_int32),
                ("gamma", _f32p), ("beta", _f32p),
                ("dout", _f32p), ("dout_bstride", C.c_int64), ("dout_lstride", C.c_int32),
                ("dh", _f32p), ("dh_bstride", C.c_int64), ("dh_lstride", C.c_int32), ("dh_dtype", C.c_int32)]


class GuideOp(C.Structure):
    _fields_ = [("batch", C.c_int32), ("L", C.c_int32), ("C", C.c_int32), ("pred", _f32p),
                ("g", _f32p), ("g_bstride", C.c_int64), ("g_lstride", C.c_int32), ("s", _f32p)]


class HeadGradOp(C.Structure):
    _fields_ = [("rows", C.c_int32), ("K", C.c_int32), ("h", _f32p), ("ldh", C.c_int32), ("act", C.c_int32),
                ("w", _f32p), ("b", _f32p), ("scale", C.c_float), ("seed", _f32p)]


class _OpUnion(C.Union):
    _fields_ = [("conv", ConvOp), ("update", UpdateOp), ("lnmod", LnModOp), ("attn", AttnOp), ("prep", PrepOp),
                ("cast", CastOp), ("mha", MhaOp), ("stash", StashOp), ("update_bwd", UpdateBwdOp), ("dgrad", DgradOp),
                ("wgrad", WgradOp), ("gn", GnOp), ("gn_bwd", GnBwdOp), ("guide", GuideOp), ("head_grad", HeadGradOp)]


class Op(C.Structure):
    _fields_ = [("kind", C.c_int32), ("flags", C.c_int32), ("u", _OpUnion)]


class CdsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libcds error {code}: {msg}")
        self.code = code


_lib = None

# every symbol include/cds.h declares (tests check that the built library exports all of them)
EXPORTS = ["cds_version", "cds_op_size", "cds_conv_tc_supported", "cds_conv_choice", "cds_attn_choice", "cds_mha_choice", "cds_last_error", "cds_device_sm_count", "cds_plan_create", "cds_plan_destroy",
           "cds_plan_append", "cds_plan_finalize", "cds_plan_run", "cds_plan_run_range", "cds_plan_profile", "cds_plan_launches_per_iter",
           "cds_run_op", "cds_debug_trace"]


def lib_path():
    return _LIB_PATH


def load():
    """dlopen libcds.so (once) and set the prototypes.  Raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} is missing: the sm_90a extension has not been built "
            "(run `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU/PyTorch fallback "
            "for the CUDA sampling path.")
    lib = C.CDLL(_LIB_PATH)
    lib.cds_version.restype = C.c_int
    lib.cds_last_error.restype = C.c_char_p
    lib.cds_device_sm_count.argtypes = [C.c_int]
    lib.cds_conv_tc_supported.argtypes = [C.POINTER(ConvOp)]
    lib.cds_conv_choice.argtypes = [C.POINTER(ConvOp), C.POINTER(C.c_int32)]
    lib.cds_attn_choice.argtypes = [C.POINTER(AttnOp), C.POINTER(C.c_int32)]
    lib.cds_mha_choice.argtypes = [C.POINTER(MhaOp), C.POINTER(C.c_int32)]
    lib.cds_plan_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.cds_plan_destroy.argtypes = [C.c_void_p]
    lib.cds_plan_append.argtypes = [C.c_void_p, C.POINTER(Op), C.c_int32]
    lib.cds_plan_finalize.argtypes = [C.c_void_p, C.c_int32]
    lib.cds_plan_run.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    lib.cds_plan_run_range.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.cds_plan_profile.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_float), C.c_int32]
    lib.cds_plan_launches_per_iter.argtypes = [C.c_void_p]
    lib.cds_run_op.argtypes = [C.c_int, C.POINTER(Op), C.c_int32, C.c_void_p]
    lib.cds_debug_trace.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
    if lib.cds_version() != ABI_VERSION:
        raise RuntimeError(f"libcds ABI {lib.cds_version()} != binding ABI {ABI_VERSION}: rebuild the extension")
    if lib.cds_op_size() != C.sizeof(Op):
        raise RuntimeError(f"cds_op layout mismatch: library {lib.cds_op_size()} B, binding {C.sizeof(Op)} B")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise CdsError(rc, load().cds_last_error().decode("utf-8", "replace"))


class Plan:
    """RAII wrapper over ``cds_plan*``."""

    def __init__(self, device_index: int):
        self._lib = load()
        self._h = C.c_void_p()
        check(self._lib.cds_plan_create(int(device_index), C.byref(self._h)))

    def append(self, ops):
        arr = (Op * len(ops))(*ops)
        check(self._lib.cds_plan_append(self._h, arr, len(ops)))

    def finalize(self, n_iters: int):
        check(self._lib.cds_plan_finalize(self._h, int(n_iters)))

    def run(self, first: int, count: int, stream: int, use_graph: bool = True):
        check(self._lib.cds_plan_run(self._h, int(first), int(count), C.c_void_p(stream), 1 if use_graph else 0))

    def run_range(self, it: int, op_first: int, op_count: int, stream: int):
        """operators [op_first, op_first + op_count) of iteration ``it`` with direct launches (the single-step entry)"""
        check(self._lib.cds_plan_run_range(self._h, int(it), int(op_first), int(op_count), C.c_void_p(stream)))

    def profile(self, it: int, stream: int, n_ops: int):
        ms = (C.c_float * n_ops)()
        check(self._lib.cds_plan_profile(self._h, int(it), C.c_void_p(stream), ms, n_ops))
        return list(ms)

    def launches_per_iter(self) -> int:
        return int(self._lib.cds_plan_launches_per_iter(self._h))

    def close(self):
        if self._h:
            self._lib.cds_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


CONV_SIMT, CONV_TC, CONV_PS = 0, 1, 2      # cds_conv_choice info[0]


def conv_choice(conv: ConvOp):
    """The kernel the library would run ``conv`` on (cds_conv_choice): a dict with the family ("simt" / "tc" / "ps") and
    its template parameters.  Raises CdsError if the op would be refused."""
    info = (C.c_int32 * 8)()
    check(load().cds_conv_choice(C.byref(conv), info))
    fam = {CONV_SIMT: "simt", CONV_TC: "tc", CONV_PS: "ps"}[info[0]]
    if fam == "simt":
        return {"family": fam, "bn": info[2]}
    return {"family": fam, "kc": info[1], "n": info[2], "split": info[3], "col_tiles": info[4], "has_res": bool(info[5]),
            "tf32": bool(info[6])}


ATTN_F32, ATTN_BF16_MMA, ATTN_TF32_TMA = 0, 1, 3     # cds_attn_choice info[0]


def attn_choice(attn: AttnOp):
    """The kernel the library would run ``attn`` on (cds_attn_choice): a dict with the family ("f32" / "bf16_mma" /
    "tma"), its template parameter (HD of "f32", NT of "tma", else 0), the head dim and the dynamic shared memory of the
    launch.  Raises CdsError if the op would be refused."""
    info = (C.c_int32 * 4)()
    check(load().cds_attn_choice(C.byref(attn), info))
    fam = {ATTN_F32: "f32", ATTN_BF16_MMA: "bf16_mma", ATTN_TF32_TMA: "tma"}[info[0]]
    return {"family": fam, "param": info[1], "hd": info[2], "smem": info[3]}


def mha_choice(mha: MhaOp):
    """The instantiation the library would run ``mha`` on (cds_mha_choice): a dict with ``hpl`` (head_dim / 32, the template
    parameter of mha_f32_kernel) and ``bf16`` (q / k / v read as bf16).  Raises CdsError if the op would be refused."""
    info = (C.c_int32 * 2)()
    check(load().cds_mha_choice(C.byref(mha), info))
    return {"hpl": info[0], "bf16": bool(info[1])}


def run_op(device_index: int, op: Op, it: int, stream: int):
    check(load().cds_run_op(int(device_index), C.byref(op), int(it), C.c_void_p(stream)))
