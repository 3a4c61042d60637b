"""ctypes binding of include/dfgpu.h — the only way Python reaches the CUDA path.

There is NO CPU fallback here: if libdfgpu.so is missing or no CUDA device is present, every
entry point raises.  (The CPU restatement lives in oracle/ and is test infrastructure only.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdfgpu.so")
STRINGS_LIB_PATH = os.path.join(_HERE, "libdfgpu_strings.so")   # include/dfgpu_strings.h: string predicates (own library)

# ---- enums (mirror include/dfgpu.h) -------------------------------------------------------
OK, END = 0, 1
BOOL, INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, DATE32, DATE64, TIMESTAMP, DECIMAL128 = range(1, 16)

EXPR_COLUMN, EXPR_LITERAL, EXPR_BINARY, EXPR_NOT, EXPR_IS_NULL, EXPR_IS_NOT_NULL, EXPR_NEGATIVE, EXPR_CAST = range(1, 9)
(OP_EQ, OP_NEQ, OP_LT, OP_LTEQ, OP_GT, OP_GTEQ, OP_PLUS, OP_MINUS, OP_MULTIPLY, OP_DIVIDE, OP_MODULO, OP_AND, OP_OR,
 OP_IS_DISTINCT_FROM, OP_IS_NOT_DISTINCT_FROM, OP_BITAND, OP_BITOR, OP_BITXOR, OP_SHIFT_LEFT, OP_SHIFT_RIGHT) = range(1, 21)

(JOIN_INNER, JOIN_LEFT, JOIN_RIGHT, JOIN_FULL, JOIN_LEFT_SEMI, JOIN_RIGHT_SEMI, JOIN_LEFT_ANTI, JOIN_RIGHT_ANTI,
 JOIN_LEFT_MARK, JOIN_RIGHT_MARK) = range(10)
NULL_EQUALS_NOTHING, NULL_EQUALS_NULL = 0, 1

AGG_PARTIAL, AGG_FINAL, AGG_FINAL_PARTITIONED, AGG_SINGLE, AGG_SINGLE_PARTITIONED, AGG_PARTIAL_REDUCE = range(6)
AGG_SUM, AGG_COUNT, AGG_MIN, AGG_MAX, AGG_AVG, AGG_COUNT_STAR = range(1, 7)
STAGE_INNER, STAGE_SEMI, STAGE_ANTI, STAGE_MAYBE, STAGE_LEFT, STAGE_LEFT_ANTI, STAGE_RIGHT = range(7)
DENSE_MAX_GROUPS = 256   # DFGPU_DENSE_MAX_GROUPS: slots of a dense aggregate's key domain

GEN_SEQ, GEN_UNIFORM, GEN_SPLITMIX, GEN_PERM, GEN_SPARSE_OF = range(5)

NP_OF_TYPE = {
    INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8, UINT16: np.uint16,
    UINT32: np.uint32, UINT64: np.uint64, FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32,
    DATE64: np.int64, TIMESTAMP: np.int64,
}
TYPE_OF_NP = {np.dtype(v): k for k, v in NP_OF_TYPE.items() if k not in (DATE32, DATE64, TIMESTAMP)}
TYPE_OF_NP[np.dtype(np.bool_)] = BOOL
_WIDTH = {BOOL: 0, INT8: 1, UINT8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, DATE32: 4, INT64: 8,
          UINT64: 8, FLOAT64: 8, DATE64: 8, TIMESTAMP: 8, DECIMAL128: 16}


def decimal128(precision: int, scale: int) -> int:
    """DFGPU_DECIMAL128_TYPE(p, s): the type code of Decimal128(precision, scale)"""
    return DECIMAL128 | (int(precision) << 8) | ((int(scale) & 0xff) << 16)


def type_base(t: int) -> int:
    return t & 0xff


def decimal_precision_scale(t: int):
    sc = (t >> 16) & 0xff
    return (t >> 8) & 0xff, sc - 256 if sc >= 128 else sc


class _Width(dict):
    def __missing__(self, t):          # Decimal128(p, s) codes carry p and s in the upper bytes
        return _WIDTH[t & 0xff]


WIDTH = _Width(_WIDTH)


def decimal_to_words(values) -> np.ndarray:
    """Python ints -> the Arrow Decimal128 buffer: [n, 2] uint64 (low word, high word), two's complement"""
    out = np.empty((len(values), 2), np.uint64)
    for i, v in enumerate(values):
        u = int(v) % (1 << 128)
        out[i, 0] = u & 0xFFFFFFFFFFFFFFFF
        out[i, 1] = u >> 64
    return out


def words_to_decimal(words: np.ndarray) -> list:
    """[n, 2] uint64 -> signed Python ints"""
    out = []
    for lo, hi in np.asarray(words, np.uint64).reshape(-1, 2).tolist():
        u = (int(hi) << 64) | int(lo)
        out.append(u - (1 << 128) if u >= (1 << 127) else u)
    return out


class DfgpuError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"dfgpu error {code}: {msg}")
        self.code = code


class Column(C.Structure):
    _fields_ = [("type", C.c_int32), ("flags", C.c_int32), ("length", C.c_int64), ("offset", C.c_int64),
                ("null_count", C.c_int64), ("values", C.c_void_p), ("validity", C.c_void_p)]


class ExprNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("a", C.c_int32), ("type", C.c_int32), ("is_null", C.c_int32),
                ("lit_i64", C.c_int64), ("lit_f64", C.c_double)]


class HashJoinOptions(C.Structure):
    _fields_ = [("join_type", C.c_int32), ("null_equality", C.c_int32), ("batch_size", C.c_int64),
                ("perfect_hash_join_small_build_threshold", C.c_int64), ("perfect_hash_join_min_key_density", C.c_double),
                ("force_hash_collisions", C.c_int32), ("ordered_output", C.c_int32), ("null_aware", C.c_int32), ("membership_filter", C.c_int32)]


class AggDesc(C.Structure):
    _fields_ = [("func", C.c_int32), ("arg_col", C.c_int32), ("filter_col", C.c_int32), ("reserved", C.c_int32)]


class LookupOptions(C.Structure):
    _fields_ = [("expected_rows", C.c_int64), ("key_min", C.c_int64), ("key_max", C.c_int64), ("has_key_range", C.c_int32),
                ("n_acc_words", C.c_int32), ("membership_filter", C.c_int32), ("filter_only", C.c_int32)]


class PipelineStage(C.Structure):
    _fields_ = [("kind", C.c_int32), ("key_col", C.c_int32), ("lookup", C.c_void_p)]


class PipelineAgg(C.Structure):
    _fields_ = [("func", C.c_int32), ("n_nodes", C.c_int32), ("expr", C.c_void_p)]


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                        ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))),
                        ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p), ("private_data", C.c_void_p)]
ArrowArray._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                       ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)),
                       ("children", C.POINTER(C.POINTER(ArrowArray))), ("dictionary", C.POINTER(ArrowArray)),
                       ("release", C.c_void_p), ("private_data", C.c_void_p)]

# every symbol include/dfgpu.h declares (tests check the library exports all of them)
EXPORTS = [
    "dfgpu_ctx_create", "dfgpu_ctx_destroy", "dfgpu_last_error", "dfgpu_version", "dfgpu_device_count", "dfgpu_sync",
    "dfgpu_ctx_stream", "dfgpu_poll_ready", "dfgpu_malloc", "dfgpu_free", "dfgpu_host_alloc", "dfgpu_host_free", "dfgpu_host_register", "dfgpu_host_unregister", "dfgpu_memcpy_h2d",
    "dfgpu_memcpy_d2h", "dfgpu_memset", "dfgpu_flush_l2", "dfgpu_trim_device_cache", "dfgpu_event_create", "dfgpu_event_record",
    "dfgpu_event_elapsed_ms", "dfgpu_event_destroy", "dfgpu_launch_count", "dfgpu_generate_i64",
    "dfgpu_set_kernel_timing", "dfgpu_kernel_time", "dfgpu_kernel_time_reset",
    "dfgpu_filter_create", "dfgpu_filter_push_host", "dfgpu_filter_push_device", "dfgpu_filter_push_arrow",
    "dfgpu_filter_finish", "dfgpu_filter_next", "dfgpu_filter_metric", "dfgpu_filter_destroy",
    "dfgpu_expr_evaluate_device", "dfgpu_expr_evaluate_host",
    "dfgpu_hashjoin_default_options", "dfgpu_hashjoin_create", "dfgpu_hashjoin_set_filter", "dfgpu_hashjoin_push_build_host",
    "dfgpu_hashjoin_push_build_device", "dfgpu_hashjoin_push_build_arrow", "dfgpu_hashjoin_finish_build",
    "dfgpu_hashjoin_push_probe_host", "dfgpu_hashjoin_push_probe_device", "dfgpu_hashjoin_push_probe_arrow",
    "dfgpu_hashjoin_finish_probe", "dfgpu_hashjoin_next", "dfgpu_hashjoin_metric", "dfgpu_hashjoin_destroy",
    "dfgpu_agg_create", "dfgpu_agg_push_host", "dfgpu_agg_push_device", "dfgpu_agg_push_arrow", "dfgpu_agg_set_skip_partial", "dfgpu_agg_finish",
    "dfgpu_agg_next", "dfgpu_agg_metric", "dfgpu_agg_destroy",
    "dfgpu_batch_num_rows", "dfgpu_batch_num_columns", "dfgpu_batch_column", "dfgpu_batch_is_host",
    "dfgpu_batch_export_arrow", "dfgpu_batch_release", "dfgpu_hash_partition_device",
    "dfgpu_partition_plan_create", "dfgpu_partition_plan_scatter_peer", "dfgpu_partition_plan_create_chunked",
    "dfgpu_partition_plan_scatter_peer_chunk", "dfgpu_partition_plan_scatter_peer_chunk_nullable", "dfgpu_partition_plan_destroy",
    "dfgpu_ipc_export", "dfgpu_ipc_import", "dfgpu_ipc_close",
    "dfgpu_comm_unique_id", "dfgpu_comm_init", "dfgpu_comm_rank", "dfgpu_comm_size", "dfgpu_comm_barrier", "dfgpu_comm_allgather_i64", "dfgpu_comm_share",
    "dfgpu_comm_destroy", "dfgpu_exchange_create", "dfgpu_exchange_run", "dfgpu_exchange_columns", "dfgpu_exchange_destroy",
    "dfgpu_lookup_default_options", "dfgpu_lookup_create", "dfgpu_lookup_metric", "dfgpu_lookup_destroy", "dfgpu_lookup_clear",
    "dfgpu_lookup_filter_buffer", "dfgpu_lookup_filter_allreduce_peer", "dfgpu_pipeline_sink_output_unordered", "dfgpu_pipeline_set_name", "dfgpu_pipeline_set_stage_filter", "dfgpu_column_minmax_device", "dfgpu_column_sum_device",
    "dfgpu_pipeline_create", "dfgpu_pipeline_sink_build", "dfgpu_pipeline_sink_aggregate", "dfgpu_pipeline_sink_aggregate_dense",
    "dfgpu_pipeline_sink_aggregate_hash", "dfgpu_pipeline_sink_output",
    "dfgpu_pipeline_push_host", "dfgpu_pipeline_push_device", "dfgpu_pipeline_push_arrow", "dfgpu_pipeline_finish",
    "dfgpu_pipeline_next", "dfgpu_pipeline_metric", "dfgpu_pipeline_destroy",
    "dfgpu_lookup_create_composite", "dfgpu_pipeline_set_stage_keys", "dfgpu_pipeline_sink_build_composite", "dfgpu_pipeline_set_stage_full",
    "dfgpu_dictionary_create", "dfgpu_dictionary_unify", "dfgpu_dictionary_code", "dfgpu_dictionary_size", "dfgpu_dictionary_value",
    "dfgpu_dictionary_remap", "dfgpu_dictionary_destroy",
]

_lib = None


def load_library() -> C.CDLL:
    """dlopen libdfgpu.so (built in-tree by __graft_entry__.build()). Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    P = C.POINTER

    def sig(name, res, args):
        f = getattr(lib, name)
        f.restype = res
        f.argtypes = args

    sig("dfgpu_ctx_create", C.c_int, [C.c_int, vp, P(vp)])
    sig("dfgpu_ctx_destroy", None, [vp])
    sig("dfgpu_last_error", C.c_char_p, [vp])
    sig("dfgpu_version", C.c_char_p, [])
    sig("dfgpu_device_count", C.c_int, [])
    sig("dfgpu_sync", C.c_int, [vp])
    sig("dfgpu_ctx_stream", vp, [vp])
    sig("dfgpu_poll_ready", C.c_int, [vp])
    sig("dfgpu_malloc", C.c_int, [vp, C.c_size_t, P(vp)])
    sig("dfgpu_free", C.c_int, [vp, vp])
    sig("dfgpu_host_alloc", C.c_int, [vp, C.c_size_t, P(vp)])
    sig("dfgpu_host_free", C.c_int, [vp, vp])
    sig("dfgpu_host_register", C.c_int, [vp, vp, C.c_size_t])
    sig("dfgpu_host_unregister", C.c_int, [vp, vp])
    sig("dfgpu_memcpy_h2d", C.c_int, [vp, vp, vp, C.c_size_t])
    sig("dfgpu_memcpy_d2h", C.c_int, [vp, vp, vp, C.c_size_t])
    sig("dfgpu_memset", C.c_int, [vp, vp, C.c_int, C.c_size_t])
    sig("dfgpu_flush_l2", C.c_int, [vp])
    sig("dfgpu_trim_device_cache", C.c_int, [vp])
    sig("dfgpu_event_create", C.c_int, [vp, P(vp)])
    sig("dfgpu_event_record", C.c_int, [vp, vp])
    sig("dfgpu_event_elapsed_ms", C.c_int, [vp, vp, vp, P(C.c_float)])
    sig("dfgpu_event_destroy", C.c_int, [vp, vp])
    sig("dfgpu_launch_count", i64, [vp])
    sig("dfgpu_set_kernel_timing", C.c_int, [vp, C.c_int])
    sig("dfgpu_kernel_time", C.c_int, [vp, C.c_char_p, P(C.c_double), P(i64)])
    sig("dfgpu_kernel_time_reset", C.c_int, [vp])
    sig("dfgpu_generate_i64", C.c_int, [vp, C.c_int, u64, i64, i64, i64, i64, vp])
    sig("dfgpu_filter_create", C.c_int, [vp, P(i32), i32, P(ExprNode), i32, P(i32), i32, i64, i64, P(vp)])
    for n in ("dfgpu_filter_push_host", "dfgpu_filter_push_device", "dfgpu_hashjoin_push_build_host",
              "dfgpu_hashjoin_push_build_device", "dfgpu_hashjoin_push_probe_host", "dfgpu_hashjoin_push_probe_device",
              "dfgpu_agg_push_host", "dfgpu_agg_push_device"):
        sig(n, C.c_int, [vp, P(Column), i32])
    for n in ("dfgpu_filter_push_arrow", "dfgpu_hashjoin_push_build_arrow", "dfgpu_hashjoin_push_probe_arrow",
              "dfgpu_agg_push_arrow"):
        sig(n, C.c_int, [vp, vp, vp])
    for n in ("dfgpu_filter_finish", "dfgpu_hashjoin_finish_build", "dfgpu_hashjoin_finish_probe", "dfgpu_agg_finish"):
        sig(n, C.c_int, [vp])
    for n in ("dfgpu_filter_next", "dfgpu_hashjoin_next", "dfgpu_agg_next"):
        sig(n, C.c_int, [vp, C.c_int, P(vp)])
    for n in ("dfgpu_filter_metric", "dfgpu_hashjoin_metric", "dfgpu_agg_metric"):
        sig(n, i64, [vp, C.c_char_p])
    for n in ("dfgpu_filter_destroy", "dfgpu_hashjoin_destroy", "dfgpu_agg_destroy", "dfgpu_batch_release"):
        sig(n, None, [vp])
    sig("dfgpu_expr_evaluate_device", C.c_int, [vp, P(Column), i32, i64, P(ExprNode), i32, P(vp)])
    sig("dfgpu_expr_evaluate_host", C.c_int, [vp, P(Column), i32, i64, P(ExprNode), i32, P(vp)])
    sig("dfgpu_hashjoin_default_options", None, [P(HashJoinOptions)])
    sig("dfgpu_hashjoin_create", C.c_int, [vp, P(i32), i32, P(i32), i32, P(i32), P(i32), i32, P(i32), P(i32), i32,
                                           P(HashJoinOptions), P(vp)])
    sig("dfgpu_hashjoin_set_filter", C.c_int, [vp, P(i32), P(i32), i32, P(ExprNode), i32])
    sig("dfgpu_agg_create", C.c_int, [vp, P(i32), i32, P(i32), i32, P(AggDesc), i32, i32, i64, i64, P(vp)])
    sig("dfgpu_agg_set_skip_partial", C.c_int, [vp, i64, C.c_double])
    sig("dfgpu_batch_num_rows", i64, [vp])
    sig("dfgpu_batch_num_columns", i32, [vp])
    sig("dfgpu_batch_column", C.c_int, [vp, i32, P(Column)])
    sig("dfgpu_batch_is_host", C.c_int, [vp])
    sig("dfgpu_batch_export_arrow", C.c_int, [vp, vp, vp])
    sig("dfgpu_hash_partition_device", C.c_int, [vp, P(Column), i32, P(i32), i32, i32, P(vp), P(i64)])
    sig("dfgpu_partition_plan_create", C.c_int, [vp, P(Column), i32, P(i32), i32, i32, P(i64), P(vp)])
    sig("dfgpu_partition_plan_scatter_peer", C.c_int, [vp, P(vp), P(i64)])
    sig("dfgpu_partition_plan_create_chunked", C.c_int, [vp, P(Column), i32, P(i32), i32, i32, i32, P(i64), P(vp)])
    sig("dfgpu_partition_plan_scatter_peer_chunk", C.c_int, [vp, i32, P(vp), P(i64)])
    sig("dfgpu_partition_plan_scatter_peer_chunk_nullable", C.c_int, [vp, i32, P(vp), P(vp), P(i64)])
    sig("dfgpu_partition_plan_destroy", None, [vp])
    sig("dfgpu_ipc_export", C.c_int, [vp, vp, C.c_char_p])
    sig("dfgpu_ipc_import", C.c_int, [vp, C.c_char_p, P(vp)])
    sig("dfgpu_ipc_close", C.c_int, [vp, vp])
    sig("dfgpu_comm_unique_id", C.c_int, [C.c_char_p])
    sig("dfgpu_comm_init", C.c_int, [vp, i32, i32, C.c_char_p, P(vp)])
    sig("dfgpu_comm_rank", i32, [vp])
    sig("dfgpu_comm_size", i32, [vp])
    sig("dfgpu_comm_barrier", C.c_int, [vp])
    sig("dfgpu_comm_allgather_i64", C.c_int, [vp, P(i64), i32, P(i64)])
    sig("dfgpu_comm_share", C.c_int, [vp, vp, P(vp)])
    sig("dfgpu_comm_destroy", None, [vp])
    sig("dfgpu_exchange_create", C.c_int, [vp, P(i32), i32, i64, P(vp)])
    sig("dfgpu_exchange_run", C.c_int, [vp, P(Column), i32, P(i32), i32, P(i64)])
    sig("dfgpu_exchange_columns", C.c_int, [vp, P(Column), i32])
    sig("dfgpu_exchange_destroy", None, [vp])
    sig("dfgpu_dictionary_create", C.c_int, [vp, P(vp)])
    sig("dfgpu_dictionary_unify", C.c_int, [vp, vp, vp, vp, i64, vp])
    sig("dfgpu_dictionary_code", i32, [vp, C.c_char_p, i64])
    sig("dfgpu_dictionary_size", i64, [vp])
    sig("dfgpu_dictionary_value", C.c_int, [vp, i32, P(vp), P(i64)])
    sig("dfgpu_dictionary_remap", C.c_int, [vp, P(Column), C.c_int, vp, i64, P(vp)])
    sig("dfgpu_dictionary_destroy", None, [vp])
    sig("dfgpu_lookup_default_options", None, [P(LookupOptions)])
    sig("dfgpu_lookup_create", C.c_int, [vp, i32, P(i32), i32, P(LookupOptions), P(vp)])
    sig("dfgpu_lookup_create_composite", C.c_int, [vp, P(i32), P(i64), P(i64), i32, P(i32), i32, P(LookupOptions), P(vp)])
    sig("dfgpu_lookup_metric", i64, [vp, C.c_char_p])
    sig("dfgpu_lookup_destroy", None, [vp])
    sig("dfgpu_lookup_clear", C.c_int, [vp])
    sig("dfgpu_lookup_filter_buffer", C.c_int, [vp, P(vp), P(u64)])
    sig("dfgpu_lookup_filter_allreduce_peer", C.c_int, [vp, P(vp), i32, i32])
    sig("dfgpu_pipeline_sink_output_unordered", C.c_int, [vp, P(i32), i32, i64])
    sig("dfgpu_column_minmax_device", C.c_int, [vp, P(Column), P(i64), P(i64), P(i64)])
    sig("dfgpu_column_sum_device", C.c_int, [vp, P(Column), P(u64), P(i64)])
    sig("dfgpu_pipeline_create", C.c_int, [vp, P(i32), i32, P(ExprNode), i32, P(PipelineStage), i32, P(vp)])
    sig("dfgpu_pipeline_sink_build", C.c_int, [vp, vp, i32, P(i32), i32])
    sig("dfgpu_pipeline_sink_build_composite", C.c_int, [vp, vp, P(i32), i32, P(i32), i32])
    sig("dfgpu_pipeline_set_stage_keys", C.c_int, [vp, i32, P(i32), i32])
    sig("dfgpu_pipeline_set_stage_full", C.c_int, [vp, i32])
    sig("dfgpu_pipeline_sink_aggregate", C.c_int, [vp, P(i32), i32, P(PipelineAgg), i32, i32, i64])
    sig("dfgpu_pipeline_sink_aggregate_dense", C.c_int, [vp, P(i32), P(i64), P(i64), i32, P(PipelineAgg), i32, i32, i64])
    sig("dfgpu_pipeline_sink_aggregate_hash", C.c_int, [vp, P(i32), P(i32), i32, P(PipelineAgg), i32, i32, i64, i64])
    sig("dfgpu_pipeline_sink_output", C.c_int, [vp, P(i32), i32, i64])
    sig("dfgpu_pipeline_set_name", C.c_int, [vp, C.c_char_p])
    sig("dfgpu_pipeline_set_stage_filter", C.c_int, [vp, i32, P(ExprNode), i32])
    sig("dfgpu_pipeline_push_host", C.c_int, [vp, P(Column), i32])
    sig("dfgpu_pipeline_push_device", C.c_int, [vp, P(Column), i32])
    sig("dfgpu_pipeline_push_arrow", C.c_int, [vp, vp, vp])
    sig("dfgpu_pipeline_finish", C.c_int, [vp])
    sig("dfgpu_pipeline_next", C.c_int, [vp, C.c_int, P(vp)])
    sig("dfgpu_pipeline_metric", i64, [vp, C.c_char_p])
    sig("dfgpu_pipeline_destroy", None, [vp])
    _lib = lib
    return lib


def _i32arr(xs: Sequence[int]):
    return (C.c_int32 * max(len(xs), 1))(*xs)


# ---- context ------------------------------------------------------------------------------
class Context:
    """dfgpu_ctx: one device + one CUDA stream.  stream: an existing cudaStream_t (int) or None."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.dfgpu_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h))
        if rc != OK:
            raise DfgpuError(rc, "cannot create a CUDA context (no GPU / driver?) — there is no CPU fallback")
        self.h = h
        self.device = device

    def check(self, rc: int):
        if rc < 0:
            raise DfgpuError(rc, self.lib.dfgpu_last_error(self.h).decode())
        return rc

    def close(self):
        if self.h:
            self.lib.dfgpu_ctx_destroy(self.h)
            self.h = None

    def sync(self):
        self.check(self.lib.dfgpu_sync(self.h))

    def poll_ready(self) -> bool:
        """non-blocking: has everything queued on this context's stream completed?"""
        return self.check(self.lib.dfgpu_poll_ready(self.h)) == 1

    @property
    def launches(self) -> int:
        return self.lib.dfgpu_launch_count(self.h)

    def set_kernel_timing(self, on: bool):
        self.check(self.lib.dfgpu_set_kernel_timing(self.h, 1 if on else 0))

    def kernel_time(self, name: str):
        """(total device ms, launches) of one kernel family since the last reset"""
        ms, cnt = C.c_double(), C.c_int64()
        self.check(self.lib.dfgpu_kernel_time(self.h, name.encode(), C.byref(ms), C.byref(cnt)))
        return ms.value, cnt.value

    def kernel_time_reset(self):
        self.check(self.lib.dfgpu_kernel_time_reset(self.h))

    def flush_l2(self):
        self.check(self.lib.dfgpu_flush_l2(self.h))

    def trim_device_cache(self):
        """hand the allocator's idle device blocks back to the driver (dfgpu_trim_device_cache)"""
        self.check(self.lib.dfgpu_trim_device_cache(self.h))

    # memory
    def malloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self.check(self.lib.dfgpu_malloc(self.h, nbytes, C.byref(p)))
        return p.value

    def free(self, ptr: int):
        self.check(self.lib.dfgpu_free(self.h, C.c_void_p(ptr)))

    def pinned_empty(self, n: int, dtype) -> np.ndarray:
        """numpy array backed by pinned host memory (kept alive by the returned array's base)."""
        dtype = np.dtype(dtype)
        nbytes = max(int(n) * dtype.itemsize, 8)
        p = C.c_void_p()
        self.check(self.lib.dfgpu_host_alloc(self.h, nbytes, C.byref(p)))
        buf = (C.c_uint8 * nbytes).from_address(p.value)
        owner = _PinnedOwner(self, p.value, buf)
        arr = np.frombuffer(owner, dtype=dtype, count=int(n)) if n else np.empty(0, dtype)
        return arr

    def to_device(self, arr: np.ndarray) -> "DeviceBuffer":
        arr = np.ascontiguousarray(arr)
        d = DeviceBuffer(self, arr.nbytes)
        self.check(self.lib.dfgpu_memcpy_h2d(self.h, C.c_void_p(d.ptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes))
        self.sync()
        return d

    def to_host(self, ptr: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes, np.uint8)
        if nbytes:
            self.check(self.lib.dfgpu_memcpy_d2h(self.h, out.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), nbytes))
            self.sync()
        return out

    # timing
    def event(self) -> int:
        e = C.c_void_p()
        self.check(self.lib.dfgpu_event_create(self.h, C.byref(e)))
        return e.value

    def record(self, ev: int):
        self.check(self.lib.dfgpu_event_record(self.h, C.c_void_p(ev)))

    def elapsed_ms(self, start: int, stop: int) -> float:
        ms = C.c_float()
        self.check(self.lib.dfgpu_event_elapsed_ms(self.h, C.c_void_p(start), C.c_void_p(stop), C.byref(ms)))
        return ms.value

    def generate_i64(self, kind: int, seed: int, a: int, b: int, start: int, n: int) -> "DeviceBuffer":
        d = DeviceBuffer(self, max(n, 1) * 8)
        self.check(self.lib.dfgpu_generate_i64(self.h, kind, seed, a, b, start, n, C.c_void_p(d.ptr)))
        return d


class _PinnedOwner:
    """buffer-protocol object owning a pinned allocation"""

    def __init__(self, ctx: Context, ptr: int, buf):
        self._ctx, self._ptr, self._buf = ctx, ptr, buf

    def __buffer__(self, flags):  # python 3.12 buffer protocol
        return memoryview(self._buf)

    def __del__(self):
        try:
            if self._ctx.h:
                self._ctx.lib.dfgpu_host_free(self._ctx.h, C.c_void_p(self._ptr))
        except Exception:
            pass


class DeviceBuffer:
    def __init__(self, ctx: Context, nbytes: int):
        self.ctx, self.nbytes = ctx, nbytes
        self.ptr = ctx.malloc(max(nbytes, 8))

    def free(self):
        if self.ptr and self.ctx.h:
            self.ctx.free(self.ptr)
        self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def to_numpy(self, dtype, count: Optional[int] = None) -> np.ndarray:
        raw = self.ctx.to_host(self.ptr, self.nbytes)
        a = raw.view(dtype)
        return a if count is None else a[:count]


# ---- columns ------------------------------------------------------------------------------
def pack_bits(mask: np.ndarray) -> np.ndarray:
    """bool array -> Arrow LSB bitmap, padded to 8 bytes"""
    b = np.packbits(np.asarray(mask, dtype=bool), bitorder="little")
    pad = (-len(b)) % 8
    if pad:
        b = np.concatenate([b, np.zeros(pad, np.uint8)])
    return b if len(b) else np.zeros(8, np.uint8)


def unpack_bits(buf: np.ndarray, n: int, offset: int = 0) -> np.ndarray:
    return np.unpackbits(buf, bitorder="little")[offset:offset + n].astype(bool)


class HostColumn:
    """values (+ optional validity mask) in host memory, with the dfgpu_column describing it"""

    def __init__(self, values: np.ndarray, valid: Optional[np.ndarray] = None, type_id: Optional[int] = None):
        values = np.asarray(values)
        self.type = type_id if type_id is not None else TYPE_OF_NP[values.dtype]
        self.length = len(values)
        if self.type == BOOL:
            self._values = pack_bits(values)
        elif type_base(self.type) == DECIMAL128:
            # values: [n, 2] uint64 words (decimal_to_words) or Python ints
            self._values = np.ascontiguousarray(values if values.dtype == np.uint64 and values.ndim == 2 else decimal_to_words(list(values)))
        else:
            self._values = np.ascontiguousarray(values.astype(NP_OF_TYPE[self.type], copy=False))
        self._validity = None if valid is None else pack_bits(valid)
        self.null_count = 0 if valid is None else int(self.length - np.count_nonzero(valid))

    def c(self) -> Column:
        col = Column()
        col.type, col.flags, col.length, col.offset, col.null_count = self.type, 0, self.length, 0, self.null_count
        col.values = self._values.ctypes.data
        col.validity = self._validity.ctypes.data if self._validity is not None else None
        return col


class DeviceColumn:
    """a column resident in HBM (buffers owned by this object)"""

    def __init__(self, ctx: Context, type_id: int, length: int, values: DeviceBuffer, validity: Optional[DeviceBuffer] = None,
                 null_count: int = 0):
        self.ctx, self.type, self.length, self.values, self.validity, self.null_count = ctx, type_id, length, values, validity, null_count

    @staticmethod
    def from_host(ctx: Context, hc: HostColumn) -> "DeviceColumn":
        v = ctx.to_device(hc._values)
        val = ctx.to_device(hc._validity) if hc._validity is not None else None
        return DeviceColumn(ctx, hc.type, hc.length, v, val, hc.null_count)

    def c(self) -> Column:
        col = Column()
        col.type, col.flags, col.length, col.offset = self.type, 0, self.length, 0
        col.null_count = self.null_count
        col.values = self.values.ptr
        col.validity = self.validity.ptr if self.validity is not None else None
        return col


def _cols(columns) -> "C.Array":
    arr = (Column * max(len(columns), 1))()
    for i, c in enumerate(columns):
        arr[i] = c.c() if not isinstance(c, Column) else c
    return arr


class Batch:
    """library-owned output batch (dfgpu_batch)"""

    def __init__(self, ctx: Context, handle: int):
        self.ctx, self.h = ctx, C.c_void_p(handle)
        lib = ctx.lib
        self.num_rows = lib.dfgpu_batch_num_rows(self.h)
        self.num_columns = lib.dfgpu_batch_num_columns(self.h)
        self.is_host = bool(lib.dfgpu_batch_is_host(self.h))

    def column(self, i: int) -> Column:
        c = Column()
        rc = self.ctx.lib.dfgpu_batch_column(self.h, i, C.byref(c))
        if rc != OK:
            raise DfgpuError(rc, "bad column index")
        return c

    def column_numpy(self, i: int):
        """(values ndarray, valid bool ndarray or None) — copies D2H when the batch is on the device"""
        c = self.column(i)
        n = c.length
        if c.type == BOOL:
            nbytes = (c.offset + n + 7) // 8
            raw = self._read(c.values, nbytes)
            vals = unpack_bits(raw, n, c.offset)
        else:
            w = WIDTH[c.type]
            off = c.offset if (c.validity and not self.is_host) else 0
            raw = self._read((c.values or 0) + off * w, n * w)
            if type_base(c.type) == DECIMAL128:
                vals = raw.view(np.uint64).reshape(-1, 2)
            else:
                vals = raw.view(NP_OF_TYPE[c.type]).copy()
        valid = None
        if c.validity:
            nbytes = (c.offset + n + 7) // 8
            valid = unpack_bits(self._read(c.validity, nbytes), n, c.offset)
        return vals, valid

    def _read(self, ptr, nbytes) -> np.ndarray:
        if nbytes == 0:
            return np.zeros(0, np.uint8)
        if self.is_host:
            return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr)).copy()
        return self.ctx.to_host(ptr, nbytes)

    def to_arrow(self):
        """export a HOST batch through the Arrow C Data Interface -> pyarrow.RecordBatch"""
        import pyarrow as pa
        assert self.is_host, "to_arrow needs a host batch (next(host=True))"
        arr, sch = ArrowArray(), ArrowSchema()
        rc = self.ctx.lib.dfgpu_batch_export_arrow(self.h, C.byref(arr), C.byref(sch))
        if rc != OK:
            raise DfgpuError(rc, "export failed")
        return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))

    def release(self):
        if self.h:
            self.ctx.lib.dfgpu_batch_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class _Operator:
    _next_fn = ""
    _destroy_fn = ""
    _metric_fn = ""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.h = C.c_void_p()

    def _push(self, fn: str, columns):
        arr = _cols(columns)
        self.ctx.check(getattr(self.ctx.lib, fn)(self.h, arr, len(columns)))

    def _push_arrow(self, fn: str, record_batch):
        import pyarrow as pa
        sa = pa.StructArray.from_arrays(record_batch.columns, fields=list(record_batch.schema))
        arr, sch = ArrowArray(), ArrowSchema()
        sa._export_to_c(C.addressof(arr), C.addressof(sch))
        try:
            rc = getattr(self.ctx.lib, fn)(self.h, C.addressof(arr), C.addressof(sch))
        finally:
            for obj in (arr, sch):  # we own the exported structs: call their release callbacks
                if obj.release:
                    C.CFUNCTYPE(None, C.c_void_p)(obj.release)(C.addressof(obj))
        self.ctx.check(rc)

    def next(self, host: bool = True) -> Optional[Batch]:
        out = C.c_void_p()
        rc = self.ctx.check(getattr(self.ctx.lib, self._next_fn)(self.h, 1 if host else 0, C.byref(out)))
        if rc == END:
            return None
        return Batch(self.ctx, out.value)

    def drain(self, host: bool = True) -> List[Batch]:
        res = []
        while True:
            b = self.next(host)
            if b is None:
                return res
            res.append(b)

    def metric(self, name: str) -> int:
        return getattr(self.ctx.lib, self._metric_fn)(self.h, name.encode())

    def close(self):
        if self.h:
            getattr(self.ctx.lib, self._destroy_fn)(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def expr_nodes(nodes: Sequence[tuple]):
    """[(kind, a, type, is_null, lit_i64, lit_f64), ...] -> ExprNode array"""
    arr = (ExprNode * len(nodes))()
    for i, nd in enumerate(nodes):
        if nd[0] == EXPR_LITERAL and type_base(nd[2]) == DECIMAL128:
            # Decimal128 literal: lit_i64 = the value as a Python int; the low word goes to lit_i64, the high word into the bytes of lit_f64
            u = int(nd[4]) % (1 << 128)
            lo, hi = u & 0xFFFFFFFFFFFFFFFF, u >> 64
            arr[i].kind, arr[i].a, arr[i].type, arr[i].is_null = nd[0], nd[1], nd[2], nd[3]
            arr[i].lit_i64 = lo - (1 << 64) if lo >= (1 << 63) else lo
            C.memmove(C.addressof(arr[i]) + ExprNode.lit_f64.offset, hi.to_bytes(8, "little"), 8)
            continue
        arr[i].kind, arr[i].a, arr[i].type, arr[i].is_null, arr[i].lit_i64, arr[i].lit_f64 = nd
    return arr


class FilterHandle(_Operator):
    _next_fn, _destroy_fn, _metric_fn = "dfgpu_filter_next", "dfgpu_filter_destroy", "dfgpu_filter_metric"

    def __init__(self, ctx, schema_types, nodes, projection=None, batch_size=8192, fetch=-1):
        super().__init__(ctx)
        na = expr_nodes(nodes)
        proj = _i32arr(projection) if projection is not None else None
        ctx.check(ctx.lib.dfgpu_filter_create(ctx.h, _i32arr(schema_types), len(schema_types), na, len(nodes), proj,
                                              len(projection) if projection is not None else 0, batch_size, fetch, C.byref(self.h)))

    def push_host(self, cols): self._push("dfgpu_filter_push_host", cols)
    def push_device(self, cols): self._push("dfgpu_filter_push_device", cols)
    def push_arrow(self, rb): self._push_arrow("dfgpu_filter_push_arrow", rb)
    def finish(self): self.ctx.check(self.ctx.lib.dfgpu_filter_finish(self.h))


class HashJoinHandle(_Operator):
    _next_fn, _destroy_fn, _metric_fn = "dfgpu_hashjoin_next", "dfgpu_hashjoin_destroy", "dfgpu_hashjoin_metric"

    def __init__(self, ctx, build_types, probe_types, on_build, on_probe, out_side, out_index, join_type=JOIN_INNER,
                 null_equality=NULL_EQUALS_NOTHING, batch_size=8192, phj_threshold=None, phj_density=None, force_hash_collisions=False,
                 null_aware=False, ordered_output=True, membership_filter=False):
        super().__init__(ctx)
        opt = HashJoinOptions()
        ctx.lib.dfgpu_hashjoin_default_options(C.byref(opt))
        opt.join_type, opt.null_equality, opt.batch_size = join_type, null_equality, batch_size
        if phj_threshold is not None:
            opt.perfect_hash_join_small_build_threshold = phj_threshold
        if phj_density is not None:
            opt.perfect_hash_join_min_key_density = phj_density
        opt.force_hash_collisions = 1 if force_hash_collisions else 0
        opt.null_aware = 1 if null_aware else 0
        opt.membership_filter = 1 if membership_filter else 0   # Bloom filter over the build keys, tested before the table (low hit rates)
        opt.ordered_output = 1 if ordered_output else 0   # 0: the consumer ignores row order (aggregate / repartition above) -> the radix-partitioned probe may run
        ctx.check(ctx.lib.dfgpu_hashjoin_create(ctx.h, _i32arr(build_types), len(build_types), _i32arr(probe_types), len(probe_types),
                                                _i32arr(on_build), _i32arr(on_probe), len(on_build), _i32arr(out_side), _i32arr(out_index),
                                                len(out_side), C.byref(opt), C.byref(self.h)))

    def set_filter(self, col_side, col_index, nodes):
        """JoinFilter: intermediate column c = column col_index[c] of side col_side[c] (0 build / 1 probe); nodes = RPN over them"""
        na = expr_nodes(nodes)
        self.ctx.check(self.ctx.lib.dfgpu_hashjoin_set_filter(self.h, _i32arr(col_side), _i32arr(col_index), len(col_side), na, len(nodes)))

    def push_build_host(self, cols): self._push("dfgpu_hashjoin_push_build_host", cols)
    def push_build_device(self, cols): self._push("dfgpu_hashjoin_push_build_device", cols)
    def push_build_arrow(self, rb): self._push_arrow("dfgpu_hashjoin_push_build_arrow", rb)
    def finish_build(self): self.ctx.check(self.ctx.lib.dfgpu_hashjoin_finish_build(self.h))
    def push_probe_host(self, cols): self._push("dfgpu_hashjoin_push_probe_host", cols)
    def push_probe_device(self, cols): self._push("dfgpu_hashjoin_push_probe_device", cols)
    def push_probe_arrow(self, rb): self._push_arrow("dfgpu_hashjoin_push_probe_arrow", rb)
    def finish_probe(self): self.ctx.check(self.ctx.lib.dfgpu_hashjoin_finish_probe(self.h))


class AggHandle(_Operator):
    _next_fn, _destroy_fn, _metric_fn = "dfgpu_agg_next", "dfgpu_agg_destroy", "dfgpu_agg_metric"

    def __init__(self, ctx, input_types, group_cols, aggs, mode=AGG_SINGLE, batch_size=8192, capacity_hint=0):
        """aggs: [(func, arg_col, filter_col)]"""
        super().__init__(ctx)
        descs = (AggDesc * max(len(aggs), 1))()
        for i, (f, a, fc) in enumerate(aggs):
            descs[i].func, descs[i].arg_col, descs[i].filter_col, descs[i].reserved = f, a, fc, 0
        ctx.check(ctx.lib.dfgpu_agg_create(ctx.h, _i32arr(input_types), len(input_types), _i32arr(group_cols), len(group_cols),
                                           descs, len(aggs), mode, batch_size, capacity_hint, C.byref(self.h)))

    def set_skip_partial(self, probe_rows_threshold: int, probe_ratio_threshold: float = 0.8):
        self.ctx.check(self.ctx.lib.dfgpu_agg_set_skip_partial(self.h, int(probe_rows_threshold), float(probe_ratio_threshold)))

    def push_host(self, cols): self._push("dfgpu_agg_push_host", cols)
    def push_device(self, cols): self._push("dfgpu_agg_push_device", cols)
    def push_arrow(self, rb): self._push_arrow("dfgpu_agg_push_arrow", rb)
    def finish(self): self.ctx.check(self.ctx.lib.dfgpu_agg_finish(self.h))


def evaluate_device(ctx: Context, cols, n_rows: int, nodes) -> "Batch":
    """PhysicalExpr::evaluate on device columns -> a one-column device batch"""
    na = expr_nodes(nodes)
    out = C.c_void_p()
    ctx.check(ctx.lib.dfgpu_expr_evaluate_device(ctx.h, _cols(cols), len(cols), int(n_rows), na, len(nodes), C.byref(out)))
    return Batch(ctx, out.value)


def hash_partition_device(ctx: Context, cols, key_cols, n_parts: int):
    arr = _cols(cols)
    out = C.c_void_p()
    offs = (C.c_int64 * (n_parts + 1))()
    ctx.check(ctx.lib.dfgpu_hash_partition_device(ctx.h, arr, len(cols), _i32arr(key_cols), len(key_cols), n_parts, C.byref(out), offs))
    return Batch(ctx, out.value), list(offs)


def column_minmax_device(ctx: Context, col) -> tuple:
    """(min, max, non-null count) of an integer column resident in HBM — the bounds collect_left_input tracks (exec.rs:2585-2619)"""
    c = col.c() if not isinstance(col, Column) else col
    mn, mx, cnt = C.c_int64(), C.c_int64(), C.c_int64()
    ctx.check(ctx.lib.dfgpu_column_minmax_device(ctx.h, C.byref(c), C.byref(mn), C.byref(mx), C.byref(cnt)))
    return mn.value, mx.value, cnt.value


def column_sum_device(ctx: Context, col) -> int:
    """wrapping (mod 2^64) sum of the non-NULL values of an integer column resident in HBM"""
    c = col.c() if not isinstance(col, Column) else col
    s, cnt = C.c_uint64(), C.c_int64()
    ctx.check(ctx.lib.dfgpu_column_sum_device(ctx.h, C.byref(c), C.byref(s), C.byref(cnt)))
    return s.value


class Lookup:
    """dfgpu_lookup: the build side of a fused join (unique keys, <= 64 bits of payload, optional accumulator words).
    A composite key (dfgpu_lookup_create_composite): key_types = the 2..4 component types and key_ranges = their declared (min, max),
    instead of key_type / key_range"""

    def __init__(self, ctx: Context, key_type: Optional[int] = None, payload_types=(), expected_rows: int = 0, key_range=None, n_acc_words: int = 0,
                 membership_filter: int = -1, filter_only: bool = False, key_types=None, key_ranges=None):
        self.ctx = ctx
        self.h = C.c_void_p()
        opt = LookupOptions()
        ctx.lib.dfgpu_lookup_default_options(C.byref(opt))
        opt.expected_rows, opt.n_acc_words, opt.membership_filter = int(expected_rows), int(n_acc_words), int(membership_filter)
        opt.filter_only = 1 if filter_only else 0
        if key_range is not None:
            opt.has_key_range, opt.key_min, opt.key_max = 1, int(key_range[0]), int(key_range[1])
        pay = _i32arr(list(payload_types))
        if key_types is not None:
            if key_type is not None or key_ranges is None or len(key_ranges) != len(key_types):
                raise ValueError("Lookup: a composite key takes key_types and one (min, max) per component in key_ranges, and no key_type")
            n = len(key_types)
            kmin = (C.c_int64 * n)(*[int(lo) for lo, _ in key_ranges])
            kmax = (C.c_int64 * n)(*[int(hi) for _, hi in key_ranges])
            ctx.check(ctx.lib.dfgpu_lookup_create_composite(ctx.h, _i32arr(list(key_types)), kmin, kmax, n, pay, len(payload_types), C.byref(opt),
                                                            C.byref(self.h)))
        else:
            ctx.check(ctx.lib.dfgpu_lookup_create(ctx.h, key_type, pay, len(payload_types), C.byref(opt), C.byref(self.h)))

    def metric(self, name: str) -> int:
        return self.ctx.lib.dfgpu_lookup_metric(self.h, name.encode())

    def clear(self):
        self.ctx.check(self.ctx.lib.dfgpu_lookup_clear(self.h))

    def filter_buffer(self):
        """(device pointer, bytes) of the membership filter"""
        p, n = C.c_void_p(), C.c_uint64()
        self.ctx.check(self.ctx.lib.dfgpu_lookup_filter_buffer(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def filter_allreduce_peer(self, peer_ptrs, rank: int):
        arr = (C.c_void_p * len(peer_ptrs))(*peer_ptrs)
        self.ctx.check(self.ctx.lib.dfgpu_lookup_filter_allreduce_peer(self.h, arr, rank, len(peer_ptrs)))

    def close(self):
        if self.h:
            self.ctx.lib.dfgpu_lookup_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Pipeline(_Operator):
    """dfgpu_pipeline: predicate -> probe stage(s) -> sink, one pass.  stages: [(kind, key_col, Lookup)]; key_col may be a list of input
    columns, the components of a composite-key lookup (set_stage_keys)
    metric(): the names dfgpu.h lists at dfgpu_pipeline_metric, e.g. "partitioned_records", the {key, value} records the partitioned
    aggregate's first pass wrote (the rows that passed the folded membership filter and fit the record buffer)"""
    _next_fn, _destroy_fn, _metric_fn = "dfgpu_pipeline_next", "dfgpu_pipeline_destroy", "dfgpu_pipeline_metric"

    def __init__(self, ctx, input_types, predicate=None, stages=(), name=None):
        super().__init__(ctx)
        self._name = name
        self._keep = [st[2] for st in stages]
        na = expr_nodes(predicate) if predicate else None
        sa = (PipelineStage * max(len(stages), 1))()
        for i, (kind, key_col, lk) in enumerate(stages):
            sa[i].kind, sa[i].key_col, sa[i].lookup = kind, key_col[0] if isinstance(key_col, (list, tuple)) else key_col, lk.h
        ctx.check(ctx.lib.dfgpu_pipeline_create(ctx.h, _i32arr(input_types), len(input_types), na, len(predicate) if predicate else 0,
                                                sa, len(stages), C.byref(self.h)))
        if name:
            ctx.check(ctx.lib.dfgpu_pipeline_set_name(self.h, name.encode()))
        for i, (_, key_col, _) in enumerate(stages):
            if isinstance(key_col, (list, tuple)):
                self.set_stage_keys(i, key_col)

    def set_stage_keys(self, stage: int, key_cols):
        """composite key of probe stage `stage`: the input columns of the lookup's components, in order"""
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_set_stage_keys(self.h, int(stage), _i32arr(list(key_cols)), len(key_cols)))

    def set_stage_full(self, stage: int):
        """turn RIGHT stage `stage` into a Full join: at finish, the build rows no probe row matched follow as rows whose input columns are
        NULL (the lookup needs payload and n_acc_words >= 1; call before the sink)"""
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_set_stage_full(self.h, int(stage)))

    def set_stage_filter(self, stage: int, nodes):
        """JoinFilter of probe stage `stage`: RPN over the input columns, the payload fields of the INNER / LEFT / LEFT_ANTI stages up to
        this one, then (SEMI / ANTI stages) this stage's own payload fields; a candidate pair matches only when it is TRUE"""
        na = expr_nodes(nodes)
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_set_stage_filter(self.h, int(stage), na, len(nodes)))

    def sink_build(self, target: Lookup, key_col: Optional[int] = None, payload_cols=(), key_cols=None):
        """key_col: the key's input column; key_cols instead: the input columns of a composite-key lookup's components"""
        self._keep.append(target)
        pay = _i32arr(list(payload_cols))
        if key_cols is not None:
            self.ctx.check(self.ctx.lib.dfgpu_pipeline_sink_build_composite(self.h, target.h, _i32arr(list(key_cols)), len(key_cols), pay,
                                                                            len(payload_cols)))
        else:
            self.ctx.check(self.ctx.lib.dfgpu_pipeline_sink_build(self.h, target.h, key_col, pay, len(payload_cols)))

    def _agg_array(self, aggs):
        arr = (PipelineAgg * max(len(aggs), 1))()
        self._agg_nodes = []
        for i, (f, nodes) in enumerate(aggs):
            arr[i].func = f
            if nodes:
                na = expr_nodes(nodes)
                self._agg_nodes.append(na)
                arr[i].n_nodes, arr[i].expr = len(nodes), C.addressof(na)
            else:
                arr[i].n_nodes, arr[i].expr = 0, None
        return arr

    def sink_aggregate(self, group_cols, aggs, mode=AGG_SINGLE, batch_size=0):
        """aggs: [(func, nodes or None)]"""
        arr = self._agg_array(aggs)
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_sink_aggregate(self.h, _i32arr(list(group_cols)), len(group_cols), arr, len(aggs), mode, batch_size))

    def sink_aggregate_dense(self, group_cols, key_range, aggs, mode=AGG_SINGLE, batch_size=0):
        """GROUP BY keys in small declared domains: key_range = [(min, max)] per group column (inclusive, NULL is a group of its
        own), at most DENSE_MAX_GROUPS slots in all; no group columns = one output row.  aggs: [(func, nodes or None)]"""
        group_cols, key_range = list(group_cols), list(key_range)
        if len(key_range) != len(group_cols):
            raise ValueError("sink_aggregate_dense: one (min, max) per group column")
        arr = self._agg_array(aggs)
        kmin = (C.c_int64 * max(len(key_range), 1))(*[int(lo) for lo, _ in key_range])
        kmax = (C.c_int64 * max(len(key_range), 1))(*[int(hi) for _, hi in key_range])
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_sink_aggregate_dense(self.h, _i32arr(group_cols), kmin, kmax, len(group_cols), arr, len(aggs),
                                                                        mode, batch_size))

    def sink_aggregate_hash(self, group_cols, aggs, mode=AGG_SINGLE, batch_size=0, capacity_hint=0, nullable=None):
        """GROUP BY any integer-like virtual columns packed into at most 128 bits (one extra bit per nullable column); the sink owns its
        group table, capacity_hint (expected groups, 0 = unknown) sizes only the first one.  nullable: the declared nullability of each
        group column (None = none is nullable).  aggs: [(func, nodes or None)]"""
        group_cols = list(group_cols)
        if nullable is not None and len(nullable) != len(group_cols):
            raise ValueError("sink_aggregate_hash: one nullability flag per group column")
        arr = self._agg_array(aggs)
        nul = _i32arr([1 if x else 0 for x in nullable]) if nullable is not None else None
        self.ctx.check(self.ctx.lib.dfgpu_pipeline_sink_aggregate_hash(self.h, _i32arr(group_cols), nul, len(group_cols), arr, len(aggs), mode,
                                                                       batch_size, capacity_hint))

    def sink_output(self, out_cols, batch_size=0, ordered=True):
        fn = self.ctx.lib.dfgpu_pipeline_sink_output if ordered else self.ctx.lib.dfgpu_pipeline_sink_output_unordered
        self.ctx.check(fn(self.h, _i32arr(list(out_cols)), len(out_cols), batch_size))

    def push_host(self, cols): self._push("dfgpu_pipeline_push_host", cols)
    def push_device(self, cols): self._push("dfgpu_pipeline_push_device", cols)
    def push_arrow(self, rb): self._push_arrow("dfgpu_pipeline_push_arrow", rb)
    def finish(self): self.ctx.check(self.ctx.lib.dfgpu_pipeline_finish(self.h))


def comm_unique_id() -> bytes:
    """128-byte rendezvous id (the role of ncclUniqueId): create on one rank, hand to every rank by any means"""
    buf = C.create_string_buffer(128)
    if load_library().dfgpu_comm_unique_id(buf) != OK:
        raise DfgpuError(-1, "cannot create a communicator id")
    return buf.raw


class Dictionary:
    """dfgpu_dictionary: one code space for the string keys of every batch (and of both join sides); the operators see INT32 codes"""

    def __init__(self, ctx: Context):
        self.ctx, self.h = ctx, C.c_void_p()
        ctx.check(ctx.lib.dfgpu_dictionary_create(ctx.h, C.byref(self.h)))

    def unify(self, offsets: np.ndarray, data: np.ndarray, valid: Optional[np.ndarray] = None) -> np.ndarray:
        """one batch's dictionary values (Arrow Utf8 layout) -> remap table local code -> unified code (-1 for a NULL value)"""
        offsets = np.ascontiguousarray(offsets, np.int32)
        data = np.ascontiguousarray(data, np.uint8)
        n = len(offsets) - 1
        vbits = None if valid is None else pack_bits(np.asarray(valid, bool))
        remap = np.empty(max(n, 1), np.int32)
        self.ctx.check(self.ctx.lib.dfgpu_dictionary_unify(self.h, offsets.ctypes.data, data.ctypes.data if len(data) else None,
                                                           vbits.ctypes.data if vbits is not None else None, n, remap.ctypes.data))
        return remap[:n]

    def code(self, value: bytes) -> int:
        return int(self.ctx.lib.dfgpu_dictionary_code(self.h, value, len(value)))

    def size(self) -> int:
        return int(self.ctx.lib.dfgpu_dictionary_size(self.h))

    def value(self, code: int) -> bytes:
        ptr, ln = C.c_void_p(), C.c_int64()
        rc = self.ctx.lib.dfgpu_dictionary_value(self.h, int(code), C.byref(ptr), C.byref(ln))
        if rc != OK:
            raise DfgpuError(rc, "dictionary: no such code")
        return C.string_at(ptr.value, ln.value) if ln.value else b""

    def remap(self, codes, remap: np.ndarray, on_host: bool = False) -> "Batch":
        """device INT32 column of unified codes for one batch's keys column"""
        remap = np.ascontiguousarray(remap, np.int32)
        col = codes.c() if not isinstance(codes, Column) else codes
        out = C.c_void_p()
        self.ctx.check(self.ctx.lib.dfgpu_dictionary_remap(self.h, C.byref(col), 1 if on_host else 0, remap.ctypes.data if len(remap) else None,
                                                           len(remap), C.byref(out)))
        self._keep = codes
        return Batch(self.ctx, out.value)

    def close(self):
        if self.h:
            self.ctx.lib.dfgpu_dictionary_destroy(self.h)
            self.h = C.c_void_p()


class Comm:
    """dfgpu_comm: the ranks (one process per GPU) of one box — barrier, count all-gather, buffer sharing over CUDA IPC; no NCCL"""

    def __init__(self, ctx: Context, n_ranks: int, rank: int, unique_id: bytes):
        self.ctx, self.h = ctx, C.c_void_p()
        ctx.check(ctx.lib.dfgpu_comm_init(ctx.h, n_ranks, rank, unique_id, C.byref(self.h)))
        self.rank, self.size = rank, n_ranks

    def barrier(self):
        self.ctx.check(self.ctx.lib.dfgpu_comm_barrier(self.h))

    def allgather_i64(self, mine: Sequence[int]) -> List[List[int]]:
        n = len(mine)
        a = (C.c_int64 * n)(*mine); out = (C.c_int64 * (n * self.size))()
        self.ctx.check(self.ctx.lib.dfgpu_comm_allgather_i64(self.h, a, n, out))
        return [list(out[r * n:(r + 1) * n]) for r in range(self.size)]

    def close(self):
        if self.h:
            self.ctx.lib.dfgpu_comm_destroy(self.h)
            self.h = C.c_void_p()


class Exchange:
    """dfgpu_exchange: RepartitionExec Hash across the ranks of a Comm, entirely inside the library"""

    def __init__(self, comm: Comm, col_types: Sequence[int], cap_rows: int):
        self.comm, self.ctx, self.types, self.h = comm, comm.ctx, list(col_types), C.c_void_p()
        self.ctx.check(self.ctx.lib.dfgpu_exchange_create(comm.h, _i32arr(self.types), len(self.types), int(cap_rows), C.byref(self.h)))

    def run(self, cols, key_cols: Sequence[int]) -> List[Column]:
        rows = C.c_int64()
        self.ctx.check(self.ctx.lib.dfgpu_exchange_run(self.h, _cols(cols), len(cols), _i32arr(list(key_cols)), len(key_cols), C.byref(rows)))
        out = (Column * len(self.types))()
        self.ctx.check(self.ctx.lib.dfgpu_exchange_columns(self.h, out, len(self.types)))
        self.rows = rows.value
        return [out[i] for i in range(len(self.types))]

    def close(self):
        if self.h:
            self.ctx.lib.dfgpu_exchange_destroy(self.h)
            self.h = C.c_void_p()


# ---- string predicates: libdfgpu_strings.so (include/dfgpu_strings.h) -------------------------
STRING_UTF8, STRING_LARGE_UTF8, STRING_UTF8_VIEW = 1, 2, 3
LIKE_NEGATED, LIKE_CASE_INSENSITIVE = 1, 2
LIKE_MAX_PATTERN_BYTES, LIKE_MAX_SEGMENTS = 256, 16
STRING_EQ, STRING_NE, STRING_LT, STRING_LE, STRING_GT, STRING_GE = range(6)
STRING_CMP_OPS = {"=": STRING_EQ, "<>": STRING_NE, "!=": STRING_NE, "<": STRING_LT, "<=": STRING_LE, ">": STRING_GT, ">=": STRING_GE}
STRING_MAX_LITERAL_BYTES, STRING_IN_MAX_VALUES, STRING_IN_MAX_BYTES = 256, 64, 1024
ERR_INVALID = -1   # DFGPU_ERR_INVALID

# every symbol include/dfgpu_strings.h declares
STRINGS_EXPORTS = ["dfgpu_like", "dfgpu_like_codes", "dfgpu_string_compare", "dfgpu_string_in_list", "dfgpu_string_take_data",
                   "dfgpu_string_take_offsets", "dfgpu_string_take_scratch_bytes", "dfgpu_string_take_views", "dfgpu_strings_last_error"]


class StringColumn(C.Structure):
    _fields_ = [("layout", C.c_int32), ("n_data_buffers", C.c_int32), ("length", C.c_int64), ("offset", C.c_int64),
                ("null_count", C.c_int64), ("offsets_or_views", C.c_void_p), ("data_buffers", C.POINTER(C.c_void_p)),
                ("validity", C.c_void_p)]


_strings_lib = None


def load_strings_library() -> C.CDLL:
    """dlopen libdfgpu_strings.so (built next to libdfgpu.so by __graft_entry__.build()). Raises if absent."""
    global _strings_lib
    if _strings_lib is not None:
        return _strings_lib
    if not os.path.exists(STRINGS_LIB_PATH):
        raise ImportError(f"{STRINGS_LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
    lib = C.CDLL(STRINGS_LIB_PATH)
    vp = C.c_void_p
    lib.dfgpu_like.restype = C.c_int
    lib.dfgpu_like.argtypes = [vp, C.POINTER(StringColumn), C.c_char_p, C.c_int64, C.c_int32, vp, vp]
    lib.dfgpu_like_codes.restype = C.c_int
    lib.dfgpu_like_codes.argtypes = [vp, C.POINTER(Column), vp, C.c_int64, vp, vp]
    lib.dfgpu_string_compare.restype = C.c_int
    lib.dfgpu_string_compare.argtypes = [vp, C.POINTER(StringColumn), C.c_int32, C.c_char_p, C.c_int64, vp, vp]
    lib.dfgpu_string_in_list.restype = C.c_int
    lib.dfgpu_string_in_list.argtypes = [vp, C.POINTER(StringColumn), C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.c_int64, C.c_int32,
                                         C.c_int32, vp, vp]
    lib.dfgpu_string_take_scratch_bytes.restype = C.c_int64
    lib.dfgpu_string_take_scratch_bytes.argtypes = [C.c_int64]
    lib.dfgpu_string_take_offsets.restype = C.c_int
    lib.dfgpu_string_take_offsets.argtypes = [vp, C.POINTER(StringColumn), C.c_int32, C.POINTER(Column), vp, vp, vp]
    lib.dfgpu_string_take_data.restype = C.c_int
    lib.dfgpu_string_take_data.argtypes = [vp, C.c_int32, C.c_int64, C.c_int64, vp, vp, vp, vp]
    lib.dfgpu_string_take_views.restype = C.c_int
    lib.dfgpu_string_take_views.argtypes = [vp, C.POINTER(StringColumn), C.c_int32, C.POINTER(Column), vp, vp, vp]
    lib.dfgpu_strings_last_error.restype = C.c_char_p
    lib.dfgpu_strings_last_error.argtypes = []
    _strings_lib = lib
    return lib


def _strings_check(rc: int):
    if rc < 0:
        raise DfgpuError(rc, load_strings_library().dfgpu_strings_last_error().decode())


class DeviceStrings:
    """a pyarrow string / large_string / string_view array copied to HBM buffer for buffer, so the array's slice offset (rows into the
    offsets or views and the validity bitmap) is kept as it is"""

    def __init__(self, ctx: Context, arr):
        import pyarrow as pa
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        t = arr.type
        if pa.types.is_string(t):
            self.layout, width = STRING_UTF8, 4
        elif pa.types.is_large_string(t):
            self.layout, width = STRING_LARGE_UTF8, 8
        elif pa.types.is_string_view(t):
            self.layout, width = STRING_UTF8_VIEW, 16
        else:
            raise NotImplementedError(f"This feature is not implemented: string predicates on the GPU over Arrow type {t}")
        self.ctx, self.length, self.offset, self.null_count = ctx, len(arr), arr.offset, arr.null_count
        bufs = arr.buffers()

        def up(buf, nbytes=None):
            raw = np.frombuffer(buf, np.uint8) if buf is not None else np.zeros(0, np.uint8)
            return ctx.to_device(raw if nbytes is None else raw[:nbytes])
        nel = arr.offset + len(arr) + (0 if self.layout == STRING_UTF8_VIEW else 1)
        self.index = up(bufs[1], nel * width)                  # offsets or views of rows [0, offset + length)
        self.validity = up(bufs[0]) if bufs[0] is not None and arr.null_count > 0 else None
        self.data = [up(b) for b in bufs[2:]]
        self.host_data = list(bufs[2:])     # the host data buffers, which string_take's Utf8View output reuses
        self._ptrs = (C.c_void_p * max(len(self.data), 1))(*[d.ptr for d in self.data])

    @property
    def nbytes(self) -> int:
        """device bytes this array holds"""
        return sum(b.nbytes for b in [self.index] + self.data + ([self.validity] if self.validity is not None else []))

    def c(self) -> StringColumn:
        s = StringColumn()
        s.layout, s.n_data_buffers, s.length, s.offset, s.null_count = self.layout, len(self.data), self.length, self.offset, self.null_count
        s.offsets_or_views = self.index.ptr
        s.data_buffers = C.cast(self._ptrs, C.POINTER(C.c_void_p))
        s.validity = self.validity.ptr if self.validity is not None else None
        return s


def _pattern_bytes(pattern) -> bytes:
    return pattern if isinstance(pattern, (bytes, bytearray)) else str(pattern).encode("utf-8")


def like(ctx: Context, strings, pattern, negated: bool = False, case_insensitive: bool = False) -> DeviceColumn:
    """`strings [NOT] LIKE pattern` (dfgpu_like) -> a UINT8 DeviceColumn in {0, 1}, NULL where the string is NULL.  strings: a
    DeviceStrings or a pyarrow string / large_string / string_view array.  DfgpuError(DFGPU_ERR_UNSUPPORTED) for what the GPU refuses."""
    ds = strings if isinstance(strings, DeviceStrings) else DeviceStrings(ctx, strings)
    lib = load_strings_library()
    n = ds.length
    values = DeviceBuffer(ctx, n)
    validity = DeviceBuffer(ctx, (n + 7) // 8) if ds.validity is not None else None
    pat = _pattern_bytes(pattern)
    flags = (LIKE_NEGATED if negated else 0) | (LIKE_CASE_INSENSITIVE if case_insensitive else 0)
    col = ds.c()
    _strings_check(lib.dfgpu_like(ctx.lib.dfgpu_ctx_stream(ctx.h), C.byref(col), pat, len(pat), flags, C.c_void_p(values.ptr),
                                  C.c_void_p(validity.ptr) if validity is not None else None))
    return DeviceColumn(ctx, UINT8, n, values, validity, ds.null_count if validity is not None else 0)


def string_compare(ctx: Context, strings, op, literal) -> DeviceColumn:
    """`strings op literal` (dfgpu_string_compare) -> a UINT8 DeviceColumn in {0, 1}, NULL where the string is NULL.  op: one of "=",
    "<>" ("!="), "<", "<=", ">", ">=" or a STRING_* code; literal: str or UTF-8 bytes.  strings as in like()."""
    ds = strings if isinstance(strings, DeviceStrings) else DeviceStrings(ctx, strings)
    code = STRING_CMP_OPS[op] if isinstance(op, str) else int(op)
    lib = load_strings_library()
    n = ds.length
    values = DeviceBuffer(ctx, n)
    validity = DeviceBuffer(ctx, (n + 7) // 8) if ds.validity is not None else None
    lit = _pattern_bytes(literal)
    col = ds.c()
    _strings_check(lib.dfgpu_string_compare(ctx.lib.dfgpu_ctx_stream(ctx.h), C.byref(col), code, lit, len(lit), C.c_void_p(values.ptr),
                                            C.c_void_p(validity.ptr) if validity is not None else None))
    return DeviceColumn(ctx, UINT8, n, values, validity, ds.null_count if validity is not None else 0)


def string_in_list(ctx: Context, strings, values, negated: bool = False) -> DeviceColumn:
    """`strings [NOT] IN (values)` (dfgpu_string_in_list) -> a UINT8 DeviceColumn in {0, 1} with SQL's three-valued IN: NULL where the
    string is NULL, and where it is found nowhere while `values` holds a None.  values: str / UTF-8 bytes / None.  strings as in like()."""
    ds = strings if isinstance(strings, DeviceStrings) else DeviceStrings(ctx, strings)
    lib = load_strings_library()
    vals = [_pattern_bytes(v) for v in values if v is not None]
    has_null = any(v is None for v in values)
    n = ds.length
    out = DeviceBuffer(ctx, n)
    validity = DeviceBuffer(ctx, (n + 7) // 8) if ds.validity is not None or has_null else None
    ptrs = (C.c_char_p * max(len(vals), 1))(*vals)
    lens = (C.c_int64 * max(len(vals), 1))(*[len(v) for v in vals])
    col = ds.c()
    _strings_check(lib.dfgpu_string_in_list(ctx.lib.dfgpu_ctx_stream(ctx.h), C.byref(col), ptrs, lens, len(vals), int(has_null), int(bool(negated)),
                                            C.c_void_p(out.ptr), C.c_void_p(validity.ptr) if validity is not None else None))
    return DeviceColumn(ctx, UINT8, n, out, validity, -1 if validity is not None else 0)


def like_codes(ctx: Context, codes, code_match: DeviceColumn, n_codes: int) -> DeviceColumn:
    """the predicate over dictionary codes (dfgpu_like_codes): codes is an INT32 DeviceColumn / Column, code_match the UINT8 value of
    each distinct string (like(), string_compare() or string_in_list() over the dictionary values) -> a UINT8 DeviceColumn, NULL where
    the code is NULL"""
    col = codes.c() if not isinstance(codes, Column) else codes
    lib = load_strings_library()
    n = int(col.length)
    values = DeviceBuffer(ctx, n)
    validity = DeviceBuffer(ctx, (n + 7) // 8) if col.validity else None
    _strings_check(lib.dfgpu_like_codes(ctx.lib.dfgpu_ctx_stream(ctx.h), C.byref(col), C.c_void_p(code_match.values.ptr), int(n_codes),
                                        C.c_void_p(values.ptr), C.c_void_p(validity.ptr) if validity is not None else None))
    return DeviceColumn(ctx, UINT8, n, values, validity, int(col.null_count) if validity is not None else 0)


class TakenStrings:
    """string_take's output: a string array of the sources' layout resident in HBM.  index: the offsets (Utf8 int32, LargeUtf8 int64)
    or the views; data: the one data buffer of a Utf8 / LargeUtf8 array, or the Utf8View output's buffer list (the sources' buffers)."""

    def __init__(self, ctx: Context, layout: int, length: int, null_count: int, index: DeviceBuffer, validity: DeviceBuffer, data, host_data,
                 keep=()):
        self.ctx, self.layout, self.length, self.null_count = ctx, layout, length, null_count
        self.index, self.validity, self.data, self._host_data = index, validity, data, host_data
        self._keep = keep     # the device buffers the enqueued gather still reads (sources, ids, scratch)

    def to_arrow(self):
        """the pyarrow array of the sources' type.  Utf8View copies back the views only and reuses the sources' host data buffers."""
        import pyarrow as pa
        n = self.length
        t = {STRING_UTF8: pa.string(), STRING_LARGE_UTF8: pa.large_string(), STRING_UTF8_VIEW: pa.string_view()}[self.layout]
        validity = pa.py_buffer(self.validity.to_numpy(np.uint8)[:(n + 7) // 8]) if self.null_count and n else None
        if self.layout == STRING_UTF8_VIEW:
            views = pa.py_buffer(self.index.to_numpy(np.uint8)[:n * 16])
            return pa.Array.from_buffers(t, n, [validity, views] + list(self._host_data), null_count=self.null_count)
        w = 4 if self.layout == STRING_UTF8 else 8
        offsets = pa.py_buffer(self.index.to_numpy(np.uint8)[:(n + 1) * w])
        return pa.Array.from_buffers(t, n, [validity, offsets, pa.py_buffer(self.data.to_numpy(np.uint8)[:self.data.nbytes])],
                                     null_count=self.null_count)


def _ids_column(ctx: Context, ids):
    """ids -> (dfgpu Column, owner): a DeviceColumn / Column as it is; a pyarrow uint32 / int64 array or numpy array uploaded"""
    if isinstance(ids, Column):
        return ids, None
    if isinstance(ids, DeviceColumn):
        return ids.c(), ids
    import pyarrow as pa
    if isinstance(ids, (pa.Array, pa.ChunkedArray)):
        if isinstance(ids, pa.ChunkedArray):
            ids = ids.combine_chunks()
        if not (pa.types.is_uint32(ids.type) or pa.types.is_int64(ids.type)):
            raise TypeError(f"string ids are uint32 or int64, not {ids.type}")
        valid = None if ids.null_count == 0 else np.asarray(ids.is_valid())
        hc = HostColumn(np.asarray(ids.fill_null(0)), valid)
    else:
        hc = HostColumn(np.asarray(ids))
    if hc.type not in (UINT32, INT64):
        raise TypeError("string ids are uint32 or int64")
    dc = DeviceColumn.from_host(ctx, hc)
    return dc.c(), dc


def string_take(ctx: Context, sources, ids) -> TakenStrings:
    """arrow-select's `take` over string arrays on the GPU (dfgpu_string_take_*): output row i is the string the id names.
    sources: DeviceStrings or pyarrow string / large_string / string_view arrays, all of one type; ids: UINT32 rows of sources[0], or
    INT64 ids packed as source << 32 | row (DeviceColumn, Column, pyarrow or numpy array).  A NULL id gives NULL.  DfgpuError
    (DFGPU_ERR_INVALID) for an id outside its source, and for a Utf8 output beyond 2^31 - 1 bytes ("offset overflow")."""
    srcs = [s if isinstance(s, DeviceStrings) else DeviceStrings(ctx, s) for s in sources]
    if not srcs:
        raise ValueError("string_take needs a source")
    layout = srcs[0].layout
    if any(s.layout != layout for s in srcs):
        raise TypeError("string_take: the sources differ in type")
    cols = (StringColumn * len(srcs))(*[s.c() for s in srcs])
    idc, owner = _ids_column(ctx, ids)
    lib = load_strings_library()
    stream = ctx.lib.dfgpu_ctx_stream(ctx.h)
    n = int(idc.length)
    if layout == STRING_UTF8_VIEW:
        views = DeviceBuffer(ctx, n * 16)
        validity = DeviceBuffer(ctx, (n + 31) // 32 * 4)
        status = DeviceBuffer(ctx, 16)
        _strings_check(lib.dfgpu_string_take_views(stream, cols, len(srcs), C.byref(idc), C.c_void_p(views.ptr), C.c_void_p(validity.ptr),
                                                   C.c_void_p(status.ptr)))
        bad, nulls = (int(x) for x in status.to_numpy(np.int64, 2))
        if bad:
            raise DfgpuError(ERR_INVALID, f"string_take: {bad} ids outside their source")
        host = [b for s in srcs for b in s.host_data]
        return TakenStrings(ctx, layout, n, nulls, views, validity, [d for s in srcs for d in s.data], host, (srcs, owner))
    offsets = DeviceBuffer(ctx, (n + 3) * 8)
    scratch = DeviceBuffer(ctx, lib.dfgpu_string_take_scratch_bytes(n))
    validity = DeviceBuffer(ctx, (n + 7) // 8)
    _strings_check(lib.dfgpu_string_take_offsets(stream, cols, len(srcs), C.byref(idc), C.c_void_p(scratch.ptr), C.c_void_p(offsets.ptr),
                                                 C.c_void_p(validity.ptr)))
    total, bad, nulls = (int(x) for x in ctx.to_host(offsets.ptr + n * 8, 24).view(np.int64))
    if bad:
        raise DfgpuError(ERR_INVALID, f"string_take: {bad} ids outside their source")
    if layout == STRING_UTF8 and total > 2**31 - 1:      # arrow's take refuses it the same way
        raise DfgpuError(ERR_INVALID, f"string_take: offset overflow ({total} bytes do not fit a Utf8 array)")
    data = DeviceBuffer(ctx, total)
    out_offsets = DeviceBuffer(ctx, (n + 1) * 4) if layout == STRING_UTF8 else offsets
    _strings_check(lib.dfgpu_string_take_data(stream, layout, n, total, C.c_void_p(scratch.ptr), C.c_void_p(offsets.ptr),
                                              C.c_void_p(out_offsets.ptr), C.c_void_p(data.ptr)))
    return TakenStrings(ctx, layout, n, nulls, out_offsets, validity, data, None, (srcs, owner, scratch, offsets))


def device_column_numpy(col: DeviceColumn):
    """(values, valid mask or None) of a DeviceColumn on the host"""
    v = col.values.to_numpy(NP_OF_TYPE[col.type], col.length) if col.length else np.zeros(0, NP_OF_TYPE[col.type])
    valid = None if col.validity is None else unpack_bits(col.validity.to_numpy(np.uint8), col.length)
    return v, valid
