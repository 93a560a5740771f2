"""ctypes binding of roc_b200/lib/libroc_b200.so (include/roc_b200.h + include/roc_host.h).

The product has no CPU fallback: if the library is missing this module raises at
import, and on a machine without a CUDA device every compute entry point returns
ROC_ERR_NO_DEVICE (-4) / aborts instead of silently running somewhere else.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libroc_b200.so")

ROC_OK = 0
ROC_ERR_INVALID, ROC_ERR_UNSUPPORTED, ROC_ERR_NOMEM, ROC_ERR_NO_DEVICE, ROC_ERR_IO = -1, -2, -3, -4, -5
AC_MODE_NONE, AC_MODE_RELU, AC_MODE_SIGMOID, AC_MODE_ELU = 0, 1, 2, 3
MASK_TRAIN, MASK_VAL, MASK_TEST, MASK_NONE = 0, 1, 2, 3
SG_EPI_NONE, SG_EPI_NORM, SG_EPI_RELU = 0, 1, 2
SG_EPI_NORM_OUT = 4                                        # roc_sg_forward_teleport_planned: the next hop's norm
AGGR_AVG, AGGR_MAX, AGGR_MIN, AGGR_SUM = 0, 1, 2, 3        # AggrType (gnn.h:75-80); ROC_SG_AGGR_MAX / _MIN = 1 / 2
SG_NOARG = 0xFFFFFFFF                                      # arg of a row with no in-edge
LINEAR_NORM_EPILOGUE = 1
LINEAR_Y_BF16 = 2                                          # Y holds bf16 bits
SG_RED_BSUM = 12                                           # roc_sg_launch.red of the sum over bf16 rows
SG_RED_TELE = 13                                           # roc_sg_launch.red of the teleport sum
SG_RED_BF16 = 16                                           # + r: roc_sg_launch.red of reduction r's bf16 form
SG_RED_DROP = 32                                           # + r: the main kernel of reduction r with (edge) dropout
HOST_DTYPES = ("float32", "bfloat16", "int32")             # ROC_HOST_DTYPE_* by value
LINEAR_BWD_ONLY_DX, LINEAR_BWD_ONLY_DW = 1, 2
GEMM_FWD, GEMM_DW, GEMM_DX = 0, 1, 2                       # `which` of roc_last_gemm_path / roc_last_gemm_info


class LinearBwdArgs(C.Structure):
    """roc_linear_bwd_args (include/roc_b200.h)."""
    _fields_ = [("rows", C.c_int64), ("inDim", C.c_int), ("outDim", C.c_int),
                ("X", C.c_void_p), ("ldX", C.c_int64), ("W", C.c_void_p),
                ("Y", C.c_void_p), ("ldY", C.c_int64), ("dY", C.c_void_p), ("ldDY", C.c_int64),
                ("dW", C.c_void_p), ("dX", C.c_void_p), ("ldDX", C.c_int64),
                ("activation", C.c_int), ("accumulate_dX", C.c_int),
                ("workspace", C.c_void_p), ("workspaceBytes", C.c_size_t),
                ("dropMask", C.c_void_p), ("ldMask", C.c_int64), ("dropRate", C.c_float),
                ("dxReluOf", C.c_void_p), ("ldReluOf", C.c_int64),
                ("dxNormRowEnd", C.c_void_p), ("colLeft", C.c_uint64), ("parts", C.c_int)]


class GemmInfo(C.Structure):
    """roc_gemm_info (include/roc_b200.h): how the last Linear GEMM of one kind was launched."""
    _fields_ = [("path", C.c_int), ("nc", C.c_int), ("epi", C.c_int), ("grid_x", C.c_int), ("grid_y", C.c_int),
                ("stages", C.c_int), ("splits", C.c_int), ("v_per_split", C.c_int64),
                ("w_resident", C.c_int), ("epi_bufs", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


SG_LAUNCH_MAIN, SG_LAUNCH_RING, SG_LAUNCH_FIXUP, SG_LAUNCH_BIG_FIXUP = 0, 1, 2, 3      # roc_sg_launch.kind
SG_LAUNCH_STAT_FIXUP, SG_LAUNCH_RECORD, SG_LAUNCH_HEADS_FIXUP, SG_LAUNCH_HEADS_BIG_FIXUP = 4, 5, 6, 7
SG_LAUNCH_PERMUTE, SG_LAUNCH_KEEP_MASK = 8, 9
SG_LAUNCH_KINDS = ("main", "ring", "fixup", "big_fixup", "stat_fixup", "record", "heads_fixup", "heads_big_fixup",
                   "permute", "keep_mask", "colsum")
SG_MAX_LAUNCHES = 32


class SgLaunch(C.Structure):
    """roc_sg_launch (include/roc_b200.h): one kernel launch of a planned ScatterGather call."""
    _fields_ = [("kind", C.c_int), ("red", C.c_int), ("vec", C.c_int), ("lanes", C.c_int), ("nch", C.c_int),
                ("grid", C.c_int64)]


class SgCallInfo(C.Structure):
    """roc_sg_call_info (include/roc_b200.h): the launches of the calling thread's last planned ScatterGather call."""
    _fields_ = [("count", C.c_int), ("launch", SgLaunch * SG_MAX_LAUNCHES)]


class PerfMetrics(C.Structure):
    """PerfMetrics, softmax_kernel.cu:35-39."""
    _fields_ = [("trainLoss", C.c_float), ("trainAll", C.c_int), ("testAll", C.c_int), ("valAll", C.c_int),
                ("trainCorrect", C.c_int), ("testCorrect", C.c_int), ("valCorrect", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class MultilabelMetrics(C.Structure):
    """roc_multilabel_metrics (include/roc_b200.h): each field indexed [0] train, [1] val, [2] test."""
    _fields_ = [("loss", C.c_double * 3), ("rows", C.c_uint64 * 3), ("exact", C.c_uint64 * 3),
                ("tp", C.c_uint64 * 3), ("fp", C.c_uint64 * 3), ("fn", C.c_uint64 * 3)]

    def as_dict(self):
        return {k: list(getattr(self, k)) for k, _ in self._fields_}


HOST_OPS = ("linear", "indegree_norm", "scatter_gather", "scatter_gather_max", "scatter_gather_min",
            "scatter_gather_weighted", "attention_gather", "relu", "sigmoid", "add", "dropout",
            "softmax_cross_entropy", "sigmoid_cross_entropy", "batch_norm", "elu",
            "attention_scores", "scaled_add")   # ROC_HOST_OP_* by value


class HostOpInfo(C.Structure):
    """roc_host_op_info (include/roc_host.h): one layer's kind and the fusion decisions Model::init made."""
    _fields_ = [(k, C.c_int) for k in ("kind", "fusedInto", "bwdFused", "epilogue", "bwdEpilogue", "fwdOut", "bwdOut",
                                       "flags", "dropOp", "dxOut", "dxReluOf", "dxNorm", "gradOut")]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["kind"] = HOST_OPS[self.kind]
        return d


class RocError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "roc_b200: %s is missing - build it with `make` (or __graft_entry__.build()); "
            "there is no Python/CPU fallback for the kernels" % LIB_PATH)
    return C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)


lib = _load()

vp, i32, i64, u32, u64, f32, f64, sz = (C.c_void_p, C.c_int, C.c_int64, C.c_uint32, C.c_uint64, C.c_float,
                                        C.c_double, C.c_size_t)

# name -> (restype, argtypes); every symbol include/roc_b200.h and include/roc_host.h declare
PROTOTYPES = {
    # ---- roc_b200.h
    "roc_version": (C.c_char_p, []),
    "roc_device_count": (i32, []),
    "roc_launch_count": (u64, []),
    "roc_set_sm_reserve": (i32, [i32]),
    "roc_partition": (i32, [u32, u64, i32, vp, vp, vp, vp]),
    "roc_build_csr": (i32, [u32, u32, u64, vp, vp, vp, vp, vp, vp]),
    "roc_sg_plan_create": (i32, [u32, u32, u64, vp, vp, vp, C.POINTER(vp)]),
    "roc_sg_plan_reserve": (i32, [vp, i32]),
    "roc_sg_plan_destroy": (None, [vp]),
    "roc_sg_plan_info": (i32, [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
    "roc_sg_plan_rows_sorted": (i32, [vp, C.POINTER(i32), vp]),
    "roc_sg_forward_planned": (i32, [vp, i32, vp, i64, vp, i64, i32, vp]),
    "roc_sg_forward_planned_bf16": (i32, [vp, i32, vp, i64, vp, i64, i32, vp]),
    "roc_sg_forward_teleport_planned": (i32, [vp, i32, vp, i64, f32, vp, i64, f32, vp, i64, i32, vp]),
    "roc_sg_forward_dropout_planned": (i32, [vp, i32, vp, i64, vp, i64, i32, vp, f32, vp]),
    "roc_sg_forward_teleport_dropout_planned": (i32, [vp, i32, vp, i64, f32, vp, i64, f32, vp, i64, i32, vp, f32, vp]),
    "roc_sg_minmax_forward_planned": (i32, [vp, i32, i32, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_minmax_forward_planned_bf16": (i32, [vp, i32, i32, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_minmax_backward_planned": (i32, [vp, i32, u32, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_forward_planned": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_forward_planned_bf16": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_backward_planned": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                           i64, vp, i64, vp]),
    "roc_sg_attn_backward_planned_bf16": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64,
                                                vp, i64, vp, i64, vp]),
    "roc_sg_weighted_forward_planned": (i32, [vp, i32, vp, i64, vp, vp, i64, vp]),
    "roc_sg_edge_dot_planned": (i32, [vp, i32, vp, i64, vp, i64, vp, i32, vp]),
    "roc_sg_weighted_forward_planned_bf16": (i32, [vp, i32, vp, i64, vp, vp, i64, vp]),
    "roc_sg_edge_dot_planned_bf16": (i32, [vp, i32, vp, i64, vp, i64, vp, i32, vp]),
    "roc_sg_attn_forward_dropout_planned": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp, f32,
                                                  vp]),
    "roc_sg_attn_forward_dropout_planned_bf16": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                                       f32, vp]),
    "roc_sg_attn_backward_dropout_planned": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64,
                                                   vp, i64, vp, i64, vp, vp, f32, vp]),
    "roc_sg_attn_backward_dropout_planned_bf16": (i32, [vp, i32, i32, f32, u32, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                                        i64, vp, i64, vp, i64, vp, vp, f32, vp]),
    "roc_sg_attn_keep_mask": (i32, [vp, u32, i32, f32, u64, u32, vp, vp]),
    "roc_sg_attn_v2_forward_planned": (i32, [vp, i32, i32, f32, vp, i64, vp, i64, vp, vp, i64, vp, i64, vp]),
    "roc_sg_attn_v2_backward_planned": (i32, [vp, i32, i32, f32, vp, i64, vp, i64, vp, vp, i64, vp, i64, vp, i64, vp,
                                              i64, vp, i64, vp, vp]),
    "roc_sg_attn_v2_backward_exact": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, vp, i64, vp, i64, vp, i64,
                                            vp, i64, vp, i64, vp, vp]),
    "roc_sg_attn_dot_forward_planned": (i32, [vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_dot_backward_planned": (i32, [vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64,
                                               vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_dot_backward_exact": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                             i64, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_softmax_forward_planned": (i32, [vp, i32, vp, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_softmax_backward_planned": (i32, [vp, i32, vp, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp, vp]),
    "roc_sg_softmax_backward_exact": (i32, [vp, vp, i32, vp, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp, vp]),
    "roc_sg_transpose_create": (i32, [u32, vp, vp, vp, C.POINTER(vp)]),
    "roc_sg_transpose_info": (i32, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "roc_sg_transpose_destroy": (None, [vp]),
    "roc_sg_weighted_backward_planned": (i32, [vp, i32, vp, i64, vp, vp, i64, vp]),
    "roc_sg_transpose_sum_backward": (i32, [vp, i32, vp, i64, vp, i64, i32, vp, vp]),
    "roc_sg_transpose_sum_backward_dropout": (i32, [vp, i32, vp, i64, vp, i64, i32, vp, vp, f32, vp]),
    "roc_sg_transpose_minmax_backward": (i32, [vp, i32, vp, i64, vp, i64, vp, i64, vp]),
    "roc_sg_attn_backward_exact": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64,
                                         vp, i64, vp]),
    "roc_sg_attn_backward_exact_bf16": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                              i64, vp, i64, vp]),
    "roc_sg_attn_backward_dropout_exact": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp, i64,
                                                 vp, i64, vp, i64, vp, vp, f32, vp]),
    "roc_sg_attn_backward_dropout_exact_bf16": (i32, [vp, vp, i32, i32, f32, vp, i64, vp, i64, vp, i64, vp, i64, vp,
                                                      i64, vp, i64, vp, i64, vp, vp, f32, vp]),
    "roc_sg_forward": (i32, [u32, u32, u64, i32, vp, vp, vp, vp, vp]),
    "roc_sg_backward": (i32, [u32, u32, u64, i32, vp, vp, vp, vp, vp]),
    "roc_sg_last_call_info": (i32, [C.POINTER(SgCallInfo)]),
    "roc_halo_create": (i32, [u32, u32, u64, vp, vp, C.POINTER(vp)]),
    "roc_halo_destroy": (None, [vp]),
    "roc_halo_size": (u32, [vp]),
    "roc_halo_ids": (vp, [vp]),
    "roc_halo_col_local": (vp, [vp]),
    "roc_halo_recv_layout": (i32, [u32, vp, i32, i32, vp, vp, vp]),
    "roc_halo_send_layout": (i32, [i32, i32, vp, vp, vp, vp]),
    "roc_pack_rows": (i32, [i64, i32, vp, vp, i64, vp, i64, vp]),
    "roc_pack_rows_at": (i32, [i64, i32, vp, vp, vp, i64, vp, i64, vp]),
    "roc_push_rows": (i32, [i64, i32, vp, vp, vp, vp, i64, vp, i32, i64, i32, vp]),
    "roc_indegree_norm": (i32, [u32, u32, u64, i32, vp, vp, i64, vp, i64, vp, vp]),
    "roc_activation_fwd": (i32, [i64, i32, i32, vp, i64, vp, i64, vp]),
    "roc_activation_bwd": (i32, [i64, i32, i32, vp, i64, vp, i64, vp, i64, i32, vp]),
    "roc_activation_fwd_y_bf16": (i32, [i64, i32, i32, vp, i64, vp, i64, vp]),
    "roc_activation_bwd_y_bf16": (i32, [i64, i32, i32, vp, i64, vp, i64, vp, i64, i32, vp]),
    "roc_add_fwd": (i32, [i64, i32, vp, i64, vp, i64, vp, i64, vp]),
    "roc_add_bwd": (i32, [i64, i32, vp, i64, vp, i64, i32, vp, i64, i32, vp]),
    "roc_scaled_add_fwd": (i32, [i64, i32, f32, vp, i64, f32, vp, i64, vp, i64, vp]),
    "roc_scaled_add_bwd": (i32, [i64, i32, vp, i64, f32, vp, i64, i32, f32, vp, i64, i32, vp]),
    "roc_dropout_fwd": (i32, [i64, i32, i64, f32, u64, u32, vp, i64, vp, i64, vp]),
    "roc_dropout_bwd": (i32, [i64, i32, i64, f32, u64, u32, vp, i64, vp, i64, vp]),
    "roc_dropout_mask": (i32, [i64, i32, i64, f32, u64, u32, vp, i64, vp]),
    "roc_dropout_fwd_bf16": (i32, [i64, i32, i64, f32, u64, u32, vp, i64, vp, i64, vp]),
    "roc_softmax_xent_bwd": (i32, [i64, i32, vp, i64, vp, i64, vp, vp, i64, vp, vp]),
    "roc_softmax_xent_bwd_idx": (i32, [i64, i32, vp, i64, vp, vp, vp, i64, vp, vp]),
    "roc_softmax_xent_bwd_norm": (i32, [i64, i32, vp, i64, vp, i64, vp, vp, vp, i64, vp, u64, vp, vp]),
    "roc_sigmoid_xent_bwd": (i32, [i64, i32, vp, i64, vp, i64, vp, vp, i64, vp, u64, vp, vp]),
    "roc_batchnorm_workspace_bytes": (sz, [i64, i32]),
    "roc_batchnorm_fwd": (i32, [i64, i32, vp, i64, vp, vp, f64, f64, vp, vp, i32, i32, vp, i64, vp, vp, vp, vp, vp, sz,
                                vp]),
    "roc_batchnorm_bwd": (i32, [i64, i32, vp, i64, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, i32, vp, sz, vp]),
    "roc_layernorm_fwd": (i32, [i64, i32, vp, i64, vp, vp, f32, i32, vp, i64, vp]),
    "roc_layernorm_workspace_bytes": (sz, [i64, i32]),
    "roc_layernorm_bwd": (i32, [i64, i32, vp, i64, vp, i64, i32, vp, vp, f32, vp, vp, vp, i64, i32, vp, sz, vp]),
    "roc_attn_scores_workspace_bytes": (sz, [i64, i32, i32]),
    "roc_attn_scores_fwd": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp]),
    "roc_attn_scores_fwd_bf16": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp]),
    "roc_attn_scores_bwd": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp, i64, i32, vp, vp, sz, vp]),
    "roc_attn_scores_bwd_bf16": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp, i64, i32, vp, vp, sz, vp]),
    "roc_linear_bwd_fused": (i32, [vp, vp]),
    "roc_linear_fwd": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, i32, i32, vp, u64, vp]),
    "roc_linear_bwd_workspace_bytes": (sz, [i64, i32, i32]),
    "roc_linear_bwd": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp, i64, vp, vp, i64, i32, i32, vp, sz, vp]),
    "roc_linear_fwd_dropout": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, i32, i32, vp, u64, vp, i64, f32, vp]),
    "roc_linear_bwd_dropout": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, vp, i64, vp, vp, i64, i32, i32, vp, sz,
                                     vp, i64, f32, vp]),
    "roc_linear_fwd_bf16": (i32, [i64, i32, i32, vp, i64, vp, vp, i64, i32, i32, vp, u64, vp, i64, f32, vp]),
    "roc_linear_dw_bf16": (i32, [i64, i32, i32, vp, i64, vp, i64, vp, i64, vp, i32, vp, sz, vp, i64, f32, vp]),
    "roc_last_gemm_path": (i32, [i32]),
    "roc_last_gemm_info": (i32, [i32, C.POINTER(GemmInfo)]),
    "roc_adam_update": (i32, [i64, f32, f32, f32, f32, f32, vp, vp, vp, vp, vp]),
    "roc_scale": (i32, [i64, f32, f32, vp, vp]),
    "roc_fill": (i32, [i64, i32, f32, vp, i64, vp]),
    "roc_copy2d": (i32, [i64, i32, vp, i64, vp, i64, vp]),
    "roc_f32_to_bf16": (i32, [i64, i32, vp, i64, vp, i64, vp]),
    "roc_bf16_to_f32": (i32, [i64, i32, vp, i64, vp, i64, vp]),
    "roc_selftest_rowdiv": (i32, [f32, u64, u64, vp, vp]),
    # ---- roc_host.h
    "roc_host_create": (vp, [i32, i32, i32]),
    "roc_host_destroy": (None, [vp]),
    "roc_host_nccl_unique_id": (i32, [vp]),
    "roc_host_nccl_init": (i32, [vp, vp]),
    "roc_host_synchronize": (i32, [vp]),
    "roc_host_stream": (vp, [vp]),
    "roc_host_graph_from_lux": (i32, [vp, C.c_char_p]),
    "roc_host_graph_from_arrays": (i32, [vp, u32, u64, vp, vp]),
    "roc_host_graph_info": (i32, [vp, vp]),
    "roc_host_graph_plan": (vp, [vp]),
    "roc_host_create_node_tensor": (i32, [vp, i32, i32]),
    "roc_host_create_node_tensor_bf16": (i32, [vp, i32]),
    "roc_host_dropout": (i32, [vp, i32, f32, i32]),
    "roc_host_linear": (i32, [vp, i32, i32, i32]),
    "roc_host_indegree_norm": (i32, [vp, i32]),
    "roc_host_scatter_gather": (i32, [vp, i32]),
    "roc_host_scatter_gather_aggr": (i32, [vp, i32, i32]),
    "roc_host_attention_gather": (i32, [vp, i32, i32, i32, f32]),
    "roc_host_dynamic_attention_gather": (i32, [vp, i32, i32, i32, f32]),
    "roc_host_softmax_gather": (i32, [vp, i32, f32, i32]),
    "roc_host_dot_attention_gather": (i32, [vp, i32, i32, i32, i32, f32]),
    "roc_host_attention_gather_dropout": (i32, [vp, i32, i32, i32, f32, f32, i32]),
    "roc_host_scatter_gather_dropout": (i32, [vp, i32, f32, i32]),
    "roc_host_get_aggr_index": (i32, [vp, i32, vp]),
    "roc_host_create_edge_tensor": (i32, [vp, i32]),
    "roc_host_scatter_gather_weighted": (i32, [vp, i32, i32]),
    "roc_host_set_edge_grad": (i32, [vp, i32, i32]),
    "roc_host_relu": (i32, [vp, i32]),
    "roc_host_sigmoid": (i32, [vp, i32]),
    "roc_host_add": (i32, [vp, i32, i32]),
    "roc_host_scaled_add": (i32, [vp, i32, i32, f32, f32]),
    "roc_host_elu": (i32, [vp, i32]),
    "roc_host_attention_scores": (i32, [vp, i32, i32]),
    "roc_host_batch_norm": (i32, [vp, i32, f32, f32]),
    "roc_host_get_batch_norm_stats": (i32, [vp, i32, vp, vp]),
    "roc_host_set_batch_norm_stats": (i32, [vp, i32, vp, vp]),
    "roc_host_layer_norm": (i32, [vp, i32, f32]),
    "roc_host_softmax_cross_entropy": (i32, [vp, i32, i32, i32]),
    "roc_host_sigmoid_cross_entropy": (i32, [vp, i32, i32, i32]),
    "roc_host_adam": (i32, [vp, f64, f64]),
    "roc_host_set_lr": (i32, [vp, f64]),
    "roc_host_get_lr": (f64, [vp]),
    "roc_host_srand": (None, [C.c_uint]),
    "roc_host_set_fusion": (i32, [vp, i32]),
    "roc_host_set_exact_backward": (i32, [vp, i32]),
    "roc_host_set_bf16_aggregation": (i32, [vp, i32]),
    "roc_host_init": (i32, [vp]),
    "roc_host_load_features": (i32, [vp, i32, C.c_char_p]),
    "roc_host_load_labels": (i32, [vp, i32, C.c_char_p]),
    "roc_host_load_train_mask": (i32, [vp, i32, C.c_char_p]),
    "roc_host_set_tensor": (i32, [vp, i32, vp, i32]),
    "roc_host_get_tensor": (i32, [vp, i32, vp, i32]),
    "roc_host_set_tensor_bf16": (i32, [vp, i32, vp]),
    "roc_host_get_tensor_bf16": (i32, [vp, i32, vp]),
    "roc_host_set_labels": (i32, [vp, i32, vp]),
    "roc_host_set_multilabels": (i32, [vp, i32, vp]),
    "roc_host_tensor_shape": (i32, [vp, i32, vp]),
    "roc_host_tensor_ptr": (vp, [vp, i32, i32]),
    "roc_host_tensor_dtype": (i32, [vp, i32]),
    "roc_host_num_parameters": (i32, [vp]),
    "roc_host_parameter_shape": (i32, [vp, i32, vp]),
    "roc_host_get_parameter": (i32, [vp, i32, vp, i32]),
    "roc_host_set_parameter": (i32, [vp, i32, vp]),
    "roc_host_num_ops": (i32, [vp]),
    "roc_host_op_info": (i32, [vp, i32, C.POINTER(HostOpInfo)]),
    "roc_host_train_mode": (i32, [vp]),
    "roc_host_infer_mode": (i32, [vp]),
    "roc_host_zero_gradients": (i32, [vp]),
    "roc_host_forward": (i32, [vp]),
    "roc_host_backward": (i32, [vp]),
    "roc_host_update": (i32, [vp]),
    "roc_host_train_epoch": (i32, [vp]),
    "roc_host_metrics": (i32, [vp, vp]),
    "roc_host_multilabel_metrics": (i32, [vp, C.POINTER(MultilabelMetrics)]),
    "roc_host_profile_sg": (i32, [vp, i32]),
    "roc_host_profile_sg_read": (i32, [vp, i32, vp, vp]),
}

for _name, (_res, _args) in PROTOTYPES.items():
    _f = getattr(lib, _name)   # AttributeError here = the library does not export a declared symbol
    _f.restype = _res
    _f.argtypes = _args


def check(rc, what=""):
    if rc != 0:
        names = {-1: "ROC_ERR_INVALID", -2: "ROC_ERR_UNSUPPORTED", -3: "ROC_ERR_NOMEM", -4: "ROC_ERR_NO_DEVICE",
                 -5: "ROC_ERR_IO"}
        raise RocError("%s failed: %s" % (what or "roc call", names.get(rc, "cudaError %d" % rc)))


def last_gemm_info(which):
    """roc_last_gemm_info as a dict; which = 0 forward, 1 dW, 2 dX."""
    info = GemmInfo()
    check(lib.roc_last_gemm_info(which, C.byref(info)), "roc_last_gemm_info")
    return info.as_dict()


def sg_last_call_info():
    """roc_sg_last_call_info: the launches of the calling thread's last planned ScatterGather call, in order, as
    dicts with the kind's name (SG_LAUNCH_KINDS) in "kind"."""
    info = SgCallInfo()
    check(lib.roc_sg_last_call_info(C.byref(info)), "roc_sg_last_call_info")
    assert info.count <= SG_MAX_LAUNCHES, "%d launches, more than the hook stores" % info.count
    return [dict({k: getattr(info.launch[i], k) for k, _ in SgLaunch._fields_},
                 kind=SG_LAUNCH_KINDS[info.launch[i].kind]) for i in range(info.count)]


def device_count():
    return lib.roc_device_count()


def require_device():
    if device_count() <= 0:
        raise RocError("roc_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
