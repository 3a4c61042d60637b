/*
 * dfgpu.h — C ABI of libdfgpu.so: the H100 (sm_90a) kernel layer behind DataFusion's
 * FilterExec / HashJoinExec / AggregateExec hot paths.
 *
 * This is boundary "b3" of SURVEY.md §8(b): the thin `extern "C"` library that a Rust
 * `GpuFilterExec` / `GpuHashJoinExec` / `GpuAggregateExec` (each implementing
 * `trait ExecutionPlan`, reference datafusion/physical-plan/src/execution_plan.rs:102, `execute` :696)
 * binds with `extern "C" { ... }` + `arrow::ffi::{to_ffi, from_ffi}`.  Record batches cross as Arrow
 * C Data Interface structs — the same structs DataFusion's own FFI layer wraps
 * (reference datafusion/ffi/src/arrow_wrappers.rs:31,72; record_batch_stream.rs:101-167).
 *
 * Conventions
 *   - every function returns 0 on success, a negative dfgpu_status on error; the message is
 *     retrievable with dfgpu_last_error(ctx).  Nothing unwinds across the boundary
 *     (mirrors `Err` items in the stream, execution_plan.rs:529-537).
 *   - plain pointers and sizes only.  `dfgpu_column` describes one Arrow primitive array
 *     (values buffer + optional LSB validity bitmap + logical offset), either in host memory
 *     (`*_host` / Arrow entry points) or already resident in HBM (`*_device` entry points).
 *   - one handle per (operator, partition); a handle is not re-entrant; different handles are
 *     independent (each ctx owns one CUDA stream) — the threading contract of
 *     `ExecutionPlan::execute(partition, ..)` (execution_plan.rs:696).
 *   - outputs are library-owned until dfgpu_batch_release.
 *   - input lifetime: HOST buffers (`*_host`, `*_arrow`) belong to the caller again as soon as the call returns (the
 *     library has finished its H2D copies by then, also from pinned memory).  DEVICE inputs (`*_device`) are read on
 *     the ctx stream: they must be complete in that stream's order (or on the legacy stream) and stay unmodified until
 *     the next call on the same handle that synchronises — dfgpu_sync, finish_*, next — returns.
 */
#ifndef DFGPU_H
#define DFGPU_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif

/* ---- status codes ---- */
enum dfgpu_status {
  DFGPU_OK = 0,
  DFGPU_END = 1,              /* next_output: stream exhausted                                  */
  DFGPU_ERR_INVALID = -1,     /* bad argument / unsupported shape (DataFusionError::Plan/Internal) */
  DFGPU_ERR_CUDA = -2,        /* CUDA runtime error (DataFusionError::Execution)                */
  DFGPU_ERR_UNSUPPORTED = -3, /* type / expression not handled on the GPU: caller keeps the CPU operator */
  DFGPU_ERR_ARITH = -4,       /* e.g. integer division by zero (ArrowError::DivideByZero)        */
  DFGPU_ERR_STATE = -5,       /* call sequence violation (push after finish, ...)               */
  DFGPU_ERR_OOM = -6          /* device allocation failed (ResourcesExhausted)                   */
};

/* ---- physical types (Arrow primitive layouts) ---- */
enum dfgpu_type {
  DFGPU_BOOL = 1,   /* bit-packed values buffer */
  DFGPU_INT8 = 2,
  DFGPU_INT16 = 3,
  DFGPU_INT32 = 4,
  DFGPU_INT64 = 5,
  DFGPU_UINT8 = 6,
  DFGPU_UINT16 = 7,
  DFGPU_UINT32 = 8,
  DFGPU_UINT64 = 9,
  DFGPU_FLOAT32 = 10,
  DFGPU_FLOAT64 = 11,
  DFGPU_DATE32 = 12,     /* int32 days  (TPC-H dates, benchmarks/src/tpch/mod.rs:52-122) */
  DFGPU_DATE64 = 13,     /* int64 ms    */
  DFGPU_TIMESTAMP = 14,  /* int64; unit and time zone live in the caller's schema only: any "ts?:tz" is accepted on import and
                          * dfgpu_batch_export_arrow writes "tsn:" — the shim builds its arrays with the DataType of the operator's own
                          * output schema (known at plan time) instead of trusting the exported format string */
  DFGPU_DECIMAL128 = 15  /* 16-byte little-endian two's complement (TPC-H money)           */
};
/* Decimal128(precision, scale) (arrow DataType::Decimal128; the TPC-H money columns are Decimal128(15, 2),
 * benchmarks/src/tpch/mod.rs:52-122): wherever a type code is passed or returned, the precision and the scale ride in the
 * upper bytes — DFGPU_DECIMAL128_TYPE(15, 2).  Arithmetic, comparison, CAST and SUM need them (result types follow
 * arrow-arith's decimal rules, see dfgpu_expr_node); the bare DFGPU_DECIMAL128 code (precision 0) is an opaque 16-byte value
 * that can only be carried, compared for equality as a key, and counted. */
#define DFGPU_DECIMAL128_TYPE(p, s) ((int32_t)(DFGPU_DECIMAL128 | ((int32_t)(p) << 8) | (((int32_t)(s) & 0xff) << 16)))
#define DFGPU_TYPE_BASE(t) ((int32_t)(t) & 0xff)
#define DFGPU_DECIMAL_PRECISION(t) (((int32_t)(t) >> 8) & 0xff)
#define DFGPU_DECIMAL_SCALE(t) ((int32_t)(int8_t)(((int32_t)(t) >> 16) & 0xff))

typedef struct dfgpu_column {
  int32_t type;            /* enum dfgpu_type */
  int32_t flags;           /* reserved, 0 */
  int64_t length;          /* rows */
  int64_t offset;          /* logical offset (elements) into values and validity */
  int64_t null_count;      /* -1 = unknown */
  const void* values;      /* values buffer */
  const uint8_t* validity; /* Arrow LSB-numbered validity bitmap, or NULL = all valid */
} dfgpu_column;

typedef struct dfgpu_ctx dfgpu_ctx;       /* device + stream + allocator + last error */
typedef struct dfgpu_batch dfgpu_batch;   /* library-owned output record batch (device or host) */
typedef struct dfgpu_filter dfgpu_filter;       /* GpuFilterExec stream state    */
typedef struct dfgpu_hashjoin dfgpu_hashjoin;   /* GpuHashJoinExec stream state  */
typedef struct dfgpu_agg dfgpu_agg;             /* GpuAggregateExec stream state */

/* ===================================================================================== */
/* context, memory, timing                                                               */
/* ===================================================================================== */

/* stream: a cudaStream_t created by the caller (e.g. torch's current stream) or NULL to let the
 * library create its own non-blocking stream. */
int dfgpu_ctx_create(int device, void* stream, dfgpu_ctx** out);
void dfgpu_ctx_destroy(dfgpu_ctx* ctx);
const char* dfgpu_last_error(dfgpu_ctx* ctx);
const char* dfgpu_version(void);
int dfgpu_device_count(void);
int dfgpu_sync(dfgpu_ctx* ctx);
/* non-blocking readiness of the ctx stream: 1 = all queued work done, 0 = still running, < 0 = error.  What a Gpu*Exec stream's
 * poll_next consults before returning Poll::Pending — ExecutionPlan streams must never block a tokio worker (execution_plan.rs:549-563) */
int dfgpu_poll_ready(dfgpu_ctx* ctx);
void* dfgpu_ctx_stream(dfgpu_ctx* ctx);

int dfgpu_malloc(dfgpu_ctx* ctx, size_t bytes, void** out);     /* stream-ordered device allocation */
int dfgpu_free(dfgpu_ctx* ctx, void* p);
int dfgpu_host_alloc(dfgpu_ctx* ctx, size_t bytes, void** out); /* pinned host memory */
int dfgpu_host_free(dfgpu_ctx* ctx, void* p);
/* page-lock / release caller-owned host memory in place (e.g. the Arrow buffers of a batch that will be pushed repeatedly or is large):
 * H2D copies from pageable memory run at roughly a third of the pinned PCIe rate (bench.py `boundary_costs`) */
int dfgpu_host_register(dfgpu_ctx* ctx, void* p, size_t bytes);
int dfgpu_host_unregister(dfgpu_ctx* ctx, void* p);
int dfgpu_memcpy_h2d(dfgpu_ctx* ctx, void* dst, const void* src, size_t bytes); /* async on ctx stream */
int dfgpu_memcpy_d2h(dfgpu_ctx* ctx, void* dst, const void* src, size_t bytes);
int dfgpu_memset(dfgpu_ctx* ctx, void* dst, int value, size_t bytes);
int dfgpu_flush_l2(dfgpu_ctx* ctx);  /* writes a >L2 scratch buffer (bench hygiene) */
/* return the idle blocks of the context's caching device allocator to the driver (synchronises the stream); the cache otherwise
 * keeps freed blocks for reuse up to half of the device memory (DFGPU_DEV_CACHE_GB).  What a MemoryPool adapter calls under
 * memory pressure (execution/src/memory_pool). */
int dfgpu_trim_device_cache(dfgpu_ctx* ctx);

/* CUDA-event timing on the ctx stream (torch.cuda.Event only sees torch's stream). */
int dfgpu_event_create(dfgpu_ctx* ctx, void** out);
int dfgpu_event_record(dfgpu_ctx* ctx, void* ev);
int dfgpu_event_elapsed_ms(dfgpu_ctx* ctx, void* start, void* stop, float* ms); /* syncs on stop */
int dfgpu_event_destroy(dfgpu_ctx* ctx, void* ev);

/* optional per-kernel-family CUDA-event timing on the ctx stream (bench.py's roofline numbers):
 * when enabled, the dominant kernels are bracketed by events; dfgpu_kernel_time returns the
 * accumulated device time and launch count of one family ("join_probe", "join_build", "agg_update",
 * "filter_eval", "take", ...). */
int dfgpu_set_kernel_timing(dfgpu_ctx* ctx, int enabled);
int dfgpu_kernel_time(dfgpu_ctx* ctx, const char* name, double* total_ms, int64_t* count);
int dfgpu_kernel_time_reset(dfgpu_ctx* ctx);

/* number of kernels this ctx has launched so far (bench.py's gpu_launches) */
int64_t dfgpu_launch_count(dfgpu_ctx* ctx);

/* deterministic counter-based synthetic column generators, identical on host (oracle) and device
 * so that billion-row inputs never cross PCIe (SURVEY.md §7 step 0).  kind: see dfgpu_gen_kind. */
enum dfgpu_gen_kind {
  DFGPU_GEN_SEQ = 0,        /* v = a + i                                    */
  DFGPU_GEN_UNIFORM = 1,    /* v = a + splitmix64(seed, i) % b              */
  DFGPU_GEN_SPLITMIX = 2,   /* v = splitmix64(seed, i)  (sparse unique-ish) */
  DFGPU_GEN_PERM = 3,       /* v = a + bijection_b(i) over [0,b)  (dense unique) */
  DFGPU_GEN_SPARSE_OF = 4   /* v = splitmix64(seed, splitmix64(seed2=a, i) % b): draws from the SPLITMIX key set */
};
int dfgpu_generate_i64(dfgpu_ctx* ctx, int kind, uint64_t seed, int64_t a, int64_t b, int64_t start,
                       int64_t n, int64_t* out_device);

/* ===================================================================================== */
/* expressions: PhysicalExpr::evaluate (physical-expr-common/src/physical_expr.rs:88)     */
/* ===================================================================================== */

/* An expression is a post-order ("RPN") program of nodes, mirroring the tree walk of
 * BinaryExpr::evaluate (physical-expr/src/expressions/binary.rs:536-676),
 * Column::evaluate (column.rs:121) and Literal::evaluate (literal.rs:106). */
enum dfgpu_expr_kind {
  DFGPU_EXPR_COLUMN = 1,   /* a = column index in the input schema                 */
  DFGPU_EXPR_LITERAL = 2,  /* type + value bits (lit_i64 / lit_f64) or is_null     */
  DFGPU_EXPR_BINARY = 3,   /* a = dfgpu_op ; pops right then left                  */
  DFGPU_EXPR_NOT = 4,
  DFGPU_EXPR_IS_NULL = 5,
  DFGPU_EXPR_IS_NOT_NULL = 6,
  DFGPU_EXPR_NEGATIVE = 7,
  DFGPU_EXPR_CAST = 8      /* type = target type                                    */
};

/* datafusion_expr::Operator (expr-common/src/operator.rs) subset on the hot path */
enum dfgpu_op {
  DFGPU_OP_EQ = 1, DFGPU_OP_NEQ = 2, DFGPU_OP_LT = 3, DFGPU_OP_LTEQ = 4, DFGPU_OP_GT = 5, DFGPU_OP_GTEQ = 6,
  DFGPU_OP_PLUS = 7, DFGPU_OP_MINUS = 8, DFGPU_OP_MULTIPLY = 9, DFGPU_OP_DIVIDE = 10, DFGPU_OP_MODULO = 11,
  DFGPU_OP_AND = 12, DFGPU_OP_OR = 13,
  DFGPU_OP_IS_DISTINCT_FROM = 14, DFGPU_OP_IS_NOT_DISTINCT_FROM = 15,
  DFGPU_OP_BITAND = 16, DFGPU_OP_BITOR = 17, DFGPU_OP_BITXOR = 18, DFGPU_OP_SHIFT_LEFT = 19, DFGPU_OP_SHIFT_RIGHT = 20
};

typedef struct dfgpu_expr_node {
  int32_t kind;     /* dfgpu_expr_kind */
  int32_t a;        /* column index or dfgpu_op */
  int32_t type;     /* literal type / cast target */
  int32_t is_null;  /* literal is NULL */
  int64_t lit_i64;  /* integer / date / bool literal; Decimal128 literal: the low 64 bits */
  double lit_f64;   /* float literal; Decimal128 literal: these 8 bytes hold the HIGH 64 bits (two's complement) */
} dfgpu_expr_node;
/* Decimal128 in expressions (arrow-arith 59.2 arithmetic.rs `decimal_op`, arrow-cast 59.2 cast/decimal.rs — third-party crates
 * pinned by the reference's Cargo.lock and absent from its tree; anchored on the reference's own vectors
 * binary.rs:4355-5000 comparison_decimal_expr_test / arithmetic_decimal_expr_test / arithmetic_divide_zero):
 *   - both operands of a binary node are Decimal128 (the planner's coercion inserted the CASTs, type_coercion/binary.rs:1257);
 *     comparisons need equal (precision, scale);
 *   - PLUS / MINUS : scale max(s1, s2), precision min(38, scale + max(p1 - s1, p2 - s2) + 1); operands rescaled by 10^(scale - s_i)
 *   - MULTIPLY     : precision min(38, p1 + p2 + 1), scale s1 + s2
 *   - DIVIDE       : scale min(38, s1 + 4), precision min(38, p1 + scale - s1 + s2); (l * 10^(scale - s1 + s2)) / r, truncating
 *   - MODULO       : scale max(s1, s2), precision min(38, scale + min(p1 - s1, p2 - s2))
 *   every step is checked on the 128-bit value: overflow = "Arithmetic overflow", zero divisor = "Divide by zero" (DFGPU_ERR_ARITH);
 *   - CAST int -> decimal, decimal -> decimal (rescale, round half away from zero, precision checked), decimal -> int
 *     (truncating), decimal <-> float64 (scale <= 22). */

/* ===================================================================================== */
/* FilterExec (physical-plan/src/filter.rs:85; hot loop poll_next :1364-1445)             */
/* ===================================================================================== */

/* schema: column types of the input batches; predicate: RPN program yielding Boolean;
 * projection: column indices kept in the output (NULL = all, filter.rs:1402);
 * batch_size: coalescer target (coalesce/mod.rs:61-65); fetch: row limit or -1 (filter.rs:623). */
int dfgpu_filter_create(dfgpu_ctx* ctx, const int32_t* schema_types, int32_t n_cols,
                        const dfgpu_expr_node* predicate, int32_t n_nodes,
                        const int32_t* projection, int32_t n_projection,
                        int64_t batch_size, int64_t fetch, dfgpu_filter** out);
int dfgpu_filter_push_host(dfgpu_filter* f, const dfgpu_column* cols, int32_t n_cols);   /* H2D inside */
int dfgpu_filter_push_device(dfgpu_filter* f, const dfgpu_column* cols, int32_t n_cols); /* HBM-resident */
int dfgpu_filter_push_arrow(dfgpu_filter* f, const struct ArrowArray* batch, const struct ArrowSchema* schema);
int dfgpu_filter_finish(dfgpu_filter* f);
/* host=1: output buffers in pinned host memory (D2H inside); host=0: device pointers.
 * returns DFGPU_OK with *out set, DFGPU_END when drained, <0 on error. */
int dfgpu_filter_next(dfgpu_filter* f, int host, dfgpu_batch** out);
int64_t dfgpu_filter_metric(dfgpu_filter* f, const char* name); /* "output_rows","input_rows","selectivity_num" … (filter.rs:1312-1330) */
void dfgpu_filter_destroy(dfgpu_filter* f);

/* stand-alone PhysicalExpr::evaluate on one batch → one output column (device) */
int dfgpu_expr_evaluate_device(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, int64_t n_rows,
                               const dfgpu_expr_node* expr, int32_t n_nodes, dfgpu_batch** out);
int dfgpu_expr_evaluate_host(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, int64_t n_rows,
                             const dfgpu_expr_node* expr, int32_t n_nodes, dfgpu_batch** out);

/* ===================================================================================== */
/* HashJoinExec (physical-plan/src/joins/hash_join/exec.rs:752; stream.rs:295)            */
/* ===================================================================================== */

/* datafusion_common::JoinType (common/src/join_type.rs) */
enum dfgpu_join_type {
  DFGPU_JOIN_INNER = 0, DFGPU_JOIN_LEFT = 1, DFGPU_JOIN_RIGHT = 2, DFGPU_JOIN_FULL = 3,
  DFGPU_JOIN_LEFT_SEMI = 4, DFGPU_JOIN_RIGHT_SEMI = 5, DFGPU_JOIN_LEFT_ANTI = 6, DFGPU_JOIN_RIGHT_ANTI = 7,
  DFGPU_JOIN_LEFT_MARK = 8, DFGPU_JOIN_RIGHT_MARK = 9
};
enum dfgpu_null_equality { DFGPU_NULL_EQUALS_NOTHING = 0, DFGPU_NULL_EQUALS_NULL = 1 };

typedef struct dfgpu_hashjoin_options {
  int32_t join_type;       /* dfgpu_join_type */
  int32_t null_equality;   /* dfgpu_null_equality (joins/utils.rs:2122-2158) */
  int64_t batch_size;      /* execution.batch_size, config.rs:904 — accepted for parity with the reference's options; the join emits ONE output
                            * batch per pushed probe batch (results do not depend on it: the MapOffset resumption of the reference is
                            * batch-size independent, tests/test_gpu_join.py runs the 8192/10/5/2/1 matrix) and the shim slices zero-copy */
  /* perfect-hash (ArrayMap) selection — exec.rs:172-179, config.rs:913,923 */
  int64_t perfect_hash_join_small_build_threshold; /* default 1024 */
  double perfect_hash_join_min_key_density;        /* default 0.15 */
  int32_t force_hash_collisions; /* mirror of cargo feature force_hash_collisions (hash_utils.rs:1185-1205) */
  int32_t ordered_output;  /* 1 (default) = the reference's order: probe order x ascending build index for Inner / RightSemi / RightAnti /
                            * RightMark; Right / Full put unmatched probe rows in probe order between the matches without a JoinFilter and
                            * after them with one (the reference's own order depends on batch_size and `right_side_ordered`, utils.rs:1449-1460:
                            * compare sorted).  0 = the consumer ignores row order (an aggregate or a repartition above): a join whose
                            * table exceeds L2 then takes the radix-partitioned probe and returns rows partition-major */
  int32_t null_aware;      /* NOT IN semantics (HashJoinExec::null_aware, exec.rs:429-455, stream.rs:755-806, 1016-1072): LeftAnti /
                            * RightAnti on ONE key column; a NULL on the other side empties the result, NULL keys of the
                            * preserved side are never emitted (unless the other side is empty) */
  int32_t membership_filter; /* 1 = also build a split-block Bloom filter over the build keys (16 bits per key) and test it before the table
                            * in the ordered probe of the inline (unique-key Inner) path: the stand-alone join's dynamic filter pushdown
                            * (hash_join/shared_bounds.rs, partitioned_hash_eval.rs).  Pays when most probe rows have no partner — a miss
                            * then costs an L2-resident filter probe instead of a DRAM table access; with every row matching it only adds
                            * the filter probe.  0 (default) = off; ignored by the other probe paths */
} dfgpu_hashjoin_options;
void dfgpu_hashjoin_default_options(dfgpu_hashjoin_options* o);

/* build = left child, probe = right child (exec.rs:768-776).  on_build/on_probe: key column indices.
 * out_side[j]/out_index[j]: output column j is column out_index[j] of side out_side[j]
 * (0 = build/left, 1 = probe/right, 2 = mark column) — ColumnIndex of joins/utils.rs:1332-1387.
 * Keys: up to 4 columns of <= 64 bits together are stored exactly in the table (one probe = one compare); anything else — up to 8
 * columns, wider together, a Decimal128 / Boolean key — is looked up by a hash of the key columns and verified on the candidate
 * pairs like the reference's equal_rows_arr (joins/utils.rs:2191-2257): same results, generic probe path.
 * Float key components compare by their bits on both paths, as the reference hashes them (hash_utils.rs hash_float_value): -0.0 does
 * not join +0.0, and a NaN joins a NaN with the same bits only.  (GROUP BY folds -0.0 into +0.0: a different rule.) */
int dfgpu_hashjoin_create(dfgpu_ctx* ctx,
                          const int32_t* build_types, int32_t n_build_cols,
                          const int32_t* probe_types, int32_t n_probe_cols,
                          const int32_t* on_build, const int32_t* on_probe, int32_t n_on,
                          const int32_t* out_side, const int32_t* out_index, int32_t n_out,
                          const dfgpu_hashjoin_options* opts, dfgpu_hashjoin** out);
/* optional JoinFilter (joins/utils.rs:1248-1320 apply_join_filter_to_indices; hash_join/stream.rs:896-906): a Boolean
 * expression over an intermediate batch whose column c is column col_index[c] of side col_side[c] (0 build, 1 probe).
 * Must be called before the first push.  NULL / false filter results drop the candidate pair. */
int dfgpu_hashjoin_set_filter(dfgpu_hashjoin* j, const int32_t* col_side, const int32_t* col_index, int32_t n_cols,
                              const dfgpu_expr_node* expr, int32_t n_nodes);
int dfgpu_hashjoin_push_build_host(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_hashjoin_push_build_device(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_hashjoin_push_build_arrow(dfgpu_hashjoin* j, const struct ArrowArray* batch, const struct ArrowSchema* schema);
int dfgpu_hashjoin_finish_build(dfgpu_hashjoin* j);  /* collect_left_input, exec.rs:2569-2776 */
int dfgpu_hashjoin_push_probe_host(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_hashjoin_push_probe_device(dfgpu_hashjoin* j, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_hashjoin_push_probe_arrow(dfgpu_hashjoin* j, const struct ArrowArray* batch, const struct ArrowSchema* schema);
int dfgpu_hashjoin_finish_probe(dfgpu_hashjoin* j);  /* ExhaustedProbeSide → process_unmatched_build_batch, stream.rs:1002 */
/* A host push probed by the pipelined host probe (see "pipelined_host_probes") yields a host batch: next with host = 0 returns
 * DFGPU_ERR_STATE for it and leaves it queued for next with host = 1. */
int dfgpu_hashjoin_next(dfgpu_hashjoin* j, int host, dfgpu_batch** out);
/* "build_input_rows","input_rows","output_rows","array_map_created_count","probe_hits","radix_partitioned_probes",
 * "pipelined_host_probes" (host pushes of >= 16 Mi rows probed chunk by chunk with overlapped copies) …
 * (joins/utils.rs:1756-1778, exec.rs:108) */
int64_t dfgpu_hashjoin_metric(dfgpu_hashjoin* j, const char* name);
void dfgpu_hashjoin_destroy(dfgpu_hashjoin* j);

/* ===================================================================================== */
/* AggregateExec (physical-plan/src/aggregates/mod.rs:839; modes :289-362)                */
/* ===================================================================================== */

enum dfgpu_agg_mode {
  DFGPU_AGG_PARTIAL = 0,           /* raw → state   (PartialHashAggregateStream, hash_stream.rs:141) */
  DFGPU_AGG_FINAL = 1,             /* state → value (FinalHashAggregateStream, hash_stream.rs:236)   */
  DFGPU_AGG_FINAL_PARTITIONED = 2,
  DFGPU_AGG_SINGLE = 3,            /* raw → value   (SingleHashAggregateStream, single_stream.rs:88)  */
  DFGPU_AGG_SINGLE_PARTITIONED = 4,
  DFGPU_AGG_PARTIAL_REDUCE = 5     /* state → state */
};
enum dfgpu_agg_func {
  DFGPU_AGG_SUM = 1,    /* functions-aggregate/src/sum.rs:308-321 (add_wrapping)      */
  DFGPU_AGG_COUNT = 2,  /* functions-aggregate/src/count.rs:631-780                   */
  DFGPU_AGG_MIN = 3,
  DFGPU_AGG_MAX = 4,
  DFGPU_AGG_AVG = 5,    /* state = [count:u64, sum] (aggregates/mod.rs:3591-3700); over Decimal128(p, s): Single modes only, see below */
  DFGPU_AGG_COUNT_STAR = 6
};
typedef struct dfgpu_agg_desc {
  int32_t func;        /* dfgpu_agg_func */
  int32_t arg_col;     /* input column (raw modes) — in state modes the state columns follow the group columns in order */
  int32_t filter_col;  /* Boolean FILTER (WHERE ..) column or -1 (accumulate.rs:373-470)  */
  int32_t reserved;
} dfgpu_agg_desc;

/* input schema: raw modes = the child's columns; state modes = [group cols..., state cols...] as emitted
 * by a Partial aggregate (sum: [sum]; count: [count]; avg: [count,sum]; min/max: [value]).
 * Arguments: SUM over integers (wrapping), floats and Decimal128(p, s) (-> Decimal128(min(38, p+10), s)); MIN / MAX over integers,
 * floats and Decimal128 (the argument's type, signed i128 order; state = [value], every mode); AVG over integers and floats (-> Float64)
 * and over Decimal128(p, s) -> Decimal128(min(38, p+4), min(38, s+4)) = sum * 10^(ts - s) / count truncated toward zero (DataFusion's
 * DecimalAverager::avg).  DFGPU_ERR_ARITH ("Arithmetic Overflow in AvgAccumulator") from dfgpu_agg_finish when that multiply overflows
 * i128 or the value exceeds the target precision.  AVG over Decimal128 has no defined Partial state: DFGPU_AGG_PARTIAL,
 * DFGPU_AGG_PARTIAL_REDUCE and the Final modes reject it with DFGPU_ERR_UNSUPPORTED; without GROUP BY it runs in the Single modes.
 * Float MIN / MAX, here and in every pipeline aggregate sink, order by IEEE totalOrder on the value's bits: -NaN < -inf < ... < -0.0 <
 * +0.0 < ... < +inf < +NaN, NaNs of one sign ordered by their payload bits.  The result is one of the group's input values bit for bit,
 * it does not depend on row order, batch boundaries or thread timing, and a group without a non-NULL value is NULL. */
int dfgpu_agg_create(dfgpu_ctx* ctx, const int32_t* input_types, int32_t n_cols,
                     const int32_t* group_cols, int32_t n_group,
                     const dfgpu_agg_desc* aggs, int32_t n_aggs,
                     int32_t mode, int64_t batch_size, int64_t capacity_hint, dfgpu_agg** out);
/* skip-partial-aggregation probe (aggregates/skip_partial.rs:69-110; execution.skip_partial_aggregation_probe_rows_threshold = 100000,
 * ..._ratio_threshold = 0.8, both the defaults here): in Partial mode, once that many rows have been aggregated and groups / rows
 * exceeds the ratio, the handle emits its groups and converts every later batch row by row into state rows (convert_to_state).
 * probe_rows_threshold = 0 switches the probe off.  Call before the first push. */
int dfgpu_agg_set_skip_partial(dfgpu_agg* a, int64_t probe_rows_threshold, double probe_ratio_threshold);
int dfgpu_agg_push_host(dfgpu_agg* a, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_agg_push_device(dfgpu_agg* a, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_agg_push_arrow(dfgpu_agg* a, const struct ArrowArray* batch, const struct ArrowSchema* schema);
int dfgpu_agg_finish(dfgpu_agg* a);
int dfgpu_agg_next(dfgpu_agg* a, int host, dfgpu_batch** out);
int64_t dfgpu_agg_metric(dfgpu_agg* a, const char* name); /* "num_groups","input_rows","output_rows","table_capacity","rehashes","skipped_aggregation_rows" */
void dfgpu_agg_destroy(dfgpu_agg* a);

/* ===================================================================================== */
/* Fused pipeline (SURVEY.md §8f rank 3): FilterExec -> HashJoinExec probe side(s) -> sink, ONE pass over HBM.
 *
 * The reference streams 8192-row batches FilterExec (filter.rs:1364-1445) -> HashJoinStream::process_probe_batch
 * (hash_join/stream.rs:740) -> AggregateHashTable::aggregate_batch_inner (aggregate_hash_table/common.rs:205-236) so
 * intermediates stay in cache.  The GPU analogue is one kernel per pipeline (the operators between two pipeline
 * breakers): every input row is read once, filtered, probed and either inserted into the next join's build table,
 * aggregated, or emitted — no intermediate batch round-trips HBM.  A physical-optimizer rule replaces
 *   AggregateExec(HashJoinExec(build, FilterExec(scan)))   /   HashJoinExec build side = HashJoinExec(RightSemi ..)
 * by these handles where the shapes below apply and keeps the unfused Gpu*Exec operators (DFGPU_ERR_UNSUPPORTED) otherwise.
 *
 * dfgpu_lookup  = the build side of a fused join: unique keys (<= 64 bits), <= 64 bits of payload columns, optional
 *                 membership filter (the GPU form of dynamic filter pushdown: PartitionBounds + hash-table membership,
 *                 joins/hash_join/shared_bounds.rs, partitioned_hash_eval.rs, join_hash_map.rs:486 contain_hashes) and
 *                 optional accumulator words per record for an aggregation whose group keys are functionally
 *                 determined by the join key (group id == build row).
 * dfgpu_pipeline= source batch -> predicate -> probe stage(s) -> sink.
 * "virtual columns" of a pipeline: the input columns [0, n_cols) followed by the payload fields of every INNER, LEFT, LEFT_ANTI and
 * RIGHT stage in stage order; expressions, group columns, build payloads and outputs address this space.  A RIGHT stage's payload
 * fields are the only nullable ones (NULL on a probe row that matched nothing; the slot then holds 0). */
/* ===================================================================================== */
typedef struct dfgpu_lookup dfgpu_lookup;
typedef struct dfgpu_pipeline dfgpu_pipeline;

typedef struct dfgpu_lookup_options {
  int64_t expected_rows;   /* 0 = unknown: the first build push counts its survivors first; the table grows by rehash */
  int64_t key_min, key_max;/* valid when has_key_range (column statistics, or dfgpu_column_minmax_device — the bounds
                            * collect_left_input tracks, exec.rs:2585-2619) */
  int32_t has_key_range;
  int32_t n_acc_words;     /* 8-byte accumulator words reserved in every record for a downstream fused aggregation (0..12; what each
                            * aggregate costs: dfgpu_pipeline_sink_aggregate) */
  int32_t membership_filter; /* 1 = build a blocked Bloom filter next to the table, 0 = never, -1 = when the table exceeds L2 */
  int32_t filter_only;       /* 1 = membership filter WITHOUT a table (16 bits per expected_rows key): the pushed-down dynamic filter of a join
                              * whose exact probe happens downstream of an exchange; backs DFGPU_STAGE_MAYBE stages only */
} dfgpu_lookup_options;
void dfgpu_lookup_default_options(dfgpu_lookup_options* o);
/* payload_types: the non-key build columns carried by a match (<= 64 bits together, no NULLs); none = key set only
 * (semi / anti joins; duplicates allowed).  Dense key ranges without payload become a bitmap (the reference's
 * ArrayMap idea, exec.rs:111-191, at one bit per key). */
int dfgpu_lookup_create(dfgpu_ctx* ctx, int32_t key_type, const int32_t* payload_types, int32_t n_payload,
                        const dfgpu_lookup_options* opts, dfgpu_lookup** out);
/* Composite keys: a join on n_keys = 2..4 key columns (TPC-H Q9's (ps_partkey, ps_suppkey)) whose values have declared domains
 * [key_min[g], key_max[g]] (column statistics: the per-column bounds collect_left_input tracks, exec.rs:2585-2619).
 *  Components: integer-like types (Int8..Int64, UInt8..UInt64, Date32, Date64, Timestamp, dictionary codes as Int32); key_min[g] <=
 *    key_max[g] (an unsigned component's key_min >= 0), else DFGPU_ERR_INVALID.
 *  Packing: r_g = key_max[g] - key_min[g] + 1, D = prod_g r_g; the packed key is sum_g (v_g - key_min[g]) * stride_g with stride_0 = 1,
 *    stride_{g+1} = stride_g * r_g, a bijection of the in-domain tuples onto [0, D - 1].  D > 2^63 - 1 is DFGPU_ERR_UNSUPPORTED (such
 *    joins stay on dfgpu_hashjoin's wide-key path).  The lookup is a lookup of that Int64 key: the bitmap / hash / Bloom rules of
 *    dfgpu_lookup_create apply to the range [0, D - 1] (a key set with a small D becomes a bitmap); "unique keys" means unique tuples.
 *    opts->has_key_range must be 0 (DFGPU_ERR_INVALID).  dfgpu_lookup_metric(l, "key_domain") returns D (-1 for a one-column key).
 *  Probe side (dfgpu_pipeline_set_stage_keys): a row with a NULL component, or a component outside its domain, packs to the sentinel D,
 *    which no lookup holds: it matches nothing in INNER / SEMI / LEFT / LEFT_ANTI / MAYBE stages and is kept by ANTI stages, as a NULL
 *    key is (NullEqualsNothing, utils.rs:2146-2155).
 *  Build side (dfgpu_pipeline_sink_build_composite): a row with a NULL component has a NULL key: not inserted, counted in "null_keys".
 *    A row with a non-NULL component outside its domain is not inserted either, and the build pipeline's dfgpu_pipeline_finish returns
 *    DFGPU_ERR_INVALID (like the dense sink's key outside its declared range).  Both are judged on every pushed row, before the predicate.
 *  Each push packs its keys in one extra pass (timed as "pipe_keys:<name>", next to "pipe:<name>"): 8 bytes per row and key are written
 *    and read again by the pipeline kernel. */
int dfgpu_lookup_create_composite(dfgpu_ctx* ctx, const int32_t* key_types, const int64_t* key_min, const int64_t* key_max, int32_t n_keys,
                                  const int32_t* payload_types, int32_t n_payload, const dfgpu_lookup_options* opts, dfgpu_lookup** out);
/* forget every record / key / filter bit, keep the allocations (a persistent build side refilled per query).  Every accumulator word
 * (a FULL stage's visited marks included) is 0 again, and "rows" and "null_keys" restart at 0.  DFGPU_ERR_STATE while a pipeline with the
 * join-keyed aggregate sink over this lookup is alive.  A clear is not needed between two aggregates or Full joins over the same build
 * rows: dfgpu_pipeline_sink_aggregate zeroes words an earlier one wrote (one FULL stage per lookup still needs a clear, see
 * dfgpu_pipeline_set_stage_full). */
int dfgpu_lookup_clear(dfgpu_lookup* l);
/* the membership filter as raw 64-bit blocks (device pointer + size): exported with dfgpu_ipc_export for the peer all-reduce below */
int dfgpu_lookup_filter_buffer(dfgpu_lookup* l, void** words_dev, uint64_t* n_bytes);
/* OR-all-reduce of the membership filters of n_ranks lookups of IDENTICAL geometry (same expected_rows) over peer memory (NVLink):
 * peer_words[r] = rank r's filter buffer (mapped with dfgpu_ipc_import; this lookup's own buffer for r == rank).  This rank merges
 * slice `rank` of every filter and writes the merged slice back into every rank's filter — a reduce-scatter + all-gather in one
 * kernel, no NCCL payload (NCCL has no bitwise OR).  The caller places a barrier before (all filters built) and after (all slices
 * merged) the call.  Reference analogue: SharedBuildAccumulator merging per-partition bounds / membership (shared_bounds.rs). */
int dfgpu_lookup_filter_allreduce_peer(dfgpu_lookup* l, void* const* peer_words, int32_t rank, int32_t n_ranks);
int64_t dfgpu_lookup_metric(dfgpu_lookup* l, const char* name); /* "rows","capacity","mode"(0 hash,1 bitmap),"table_bytes","filter_bytes","rehashes",
                                                                  "null_keys": rows pushed into the build sink with a NULL key (never
                                                                  inserted), counted from the key column before the predicate */
void dfgpu_lookup_destroy(dfgpu_lookup* l);
/* min / max / non-null count of one integer column (device resident): feeds dfgpu_lookup_options.key_min/key_max */
int dfgpu_column_minmax_device(dfgpu_ctx* ctx, const dfgpu_column* col, int64_t* min_out, int64_t* max_out, int64_t* valid_out);
/* wrapping (mod 2^64) sum of the non-NULL values of an integer column, device resident: order-independent fingerprints of
 * results too large to compare row by row (SURVEY.md §8d "Large-config verification"); a Decimal128 column contributes
 * low word + 3 x high word per value */
int dfgpu_column_sum_device(dfgpu_ctx* ctx, const dfgpu_column* col, uint64_t* sum_out, int64_t* valid_out);

enum dfgpu_stage_kind {
  DFGPU_STAGE_INNER = 0, DFGPU_STAGE_SEMI = 1, DFGPU_STAGE_ANTI = 2,
  DFGPU_STAGE_MAYBE = 3,  /* membership pre-filter only (may have false positives, never false negatives): the dynamic filter a downstream
                           * join pushes into this scan (joins/hash_join/shared_bounds.rs); the exact join runs after the exchange */
  DFGPU_STAGE_LEFT = 4,   /* Left join (every build row, NULL-padded when no probe row matches) and LeftAnti join (the build rows no     */
  DFGPU_STAGE_LEFT_ANTI = 5, /* probe row matches): the last stage only, with dfgpu_pipeline_sink_aggregate grouped on it (see there); the
                           * probe runs as for INNER (unmatched probe rows are dropped, the payload fields are virtual columns) */
  DFGPU_STAGE_RIGHT = 6   /* Right join (every probe row, NULL-padded when no build row matches): every row reaching the stage continues,
                           * a matched one with its build row's payload fields, an unmatched one (no partner, a NULL key, a composite key
                           * that packs to the sentinel D) with every payload field of the stage NULL.  The row count never changes, so the
                           * lookup must hold unique keys: it needs payload (its build refuses duplicate keys), and a key-only, bitmap or
                           * filter-only lookup is DFGPU_ERR_UNSUPPORTED at dfgpu_pipeline_create.  Sinks: output (ordered: probe order,
                           * unmatched rows where they occur, as dfgpu_hashjoin's Right join), dense and hash aggregates; the build, pack
                           * and join-keyed aggregate sinks are DFGPU_ERR_UNSUPPORTED, and so is dfgpu_pipeline_set_stage_filter on any
                           * stage of a pipeline with a RIGHT stage.  An aggregate argument reading a RIGHT payload field skips its NULLs.
                           * dfgpu_pipeline_set_stage_full turns a RIGHT stage into a Full join (see there). */
};
typedef struct dfgpu_pipeline_stage {
  int32_t kind;          /* dfgpu_stage_kind: the pipeline input is the PROBE (right) side — Inner / RightSemi / RightAnti / Right, and Left /
                          * LeftAnti (LEFT / LEFT_ANTI) through the join-keyed aggregate sink.  LeftSemi is an INNER stage + the join-keyed
                          * aggregate sink with no aggregates, grouped on the key and payload of a lookup with unique keys */
  int32_t key_col;       /* input column holding the probe key (NULL keys never match, utils.rs:2146-2155) */
  dfgpu_lookup* lookup;  /* must be completely built before the first push */
} dfgpu_pipeline_stage;
typedef struct dfgpu_pipeline_agg {
  int32_t func;                 /* dfgpu_agg_func */
  int32_t n_nodes;              /* argument expression over the virtual columns (RPN); 0 for COUNT(*) */
  const dfgpu_expr_node* expr;
} dfgpu_pipeline_agg;

/* predicate: Boolean RPN over the INPUT columns, or NULL (no FilterExec below the probe) */
int dfgpu_pipeline_create(dfgpu_ctx* ctx, const int32_t* input_types, int32_t n_cols,
                          const dfgpu_expr_node* predicate, int32_t n_pred_nodes,
                          const dfgpu_pipeline_stage* stages, int32_t n_stages, dfgpu_pipeline** out);
/* exactly one sink, chosen before the first push:
 *  build     : surviving rows become records of `target` (key = virtual column key_col, payload = payload_cols in
 *              the order of the lookup's payload_types) — the pipeline IS the build side of the next join;
 *  aggregate : AggregateExec over the surviving rows; group_cols must be the probe key of one INNER (or LEFT / LEFT_ANTI)
 *              stage plus payload fields of that stage (group id == build row; anything else -> DFGPU_ERR_UNSUPPORTED, use dfgpu_agg);
 *              mode = DFGPU_AGG_SINGLE* or DFGPU_AGG_PARTIAL (state columns as dfgpu_agg emits them);
 *              the accumulators are words of the lookup's records (n_acc_words): 1 row counter, then per aggregate
 *                COUNT(x), and SUM / MIN / MAX over a 64-bit type: 1;  AVG over Float64: 2;
 *                Decimal128 SUM: 2;  Decimal128 MIN / MAX: 2, one 16-byte aligned {lo, hi} pair;  Decimal128 AVG: 3;
 *              plus 1 non-null counter for a SUM / MIN / MAX whose argument can be NULL (without it such an argument is
 *              DFGPU_ERR_UNSUPPORTED at the push); spare words become non-null counters.
 *              Over Decimal128: COUNT, SUM, MIN, MAX in every mode; AVG -> Decimal128(min(38, p+4), min(38, s+4)) in Single
 *              modes only (DFGPU_ERR_ARITH at finish when a group's value overflows, as in the dense sink).  A Decimal128 MIN /
 *              MAX needs a record of an even number of words: with payload it always is; a lookup without payload needs an odd
 *              n_acc_words (else DFGPU_ERR_UNSUPPORTED).  The pairs take even words after the row counter, behind at most one
 *              padding word, which may serve as a non-null counter; without pairs the words are taken in aggregate order.
 *              A LEFT / LEFT_ANTI stage must be the last stage and the one grouped on (else DFGPU_ERR_UNSUPPORTED); its key column
 *              then means the BUILD key, emitted from the record (never NULL).  Output in slot order (unspecified) either way:
 *                LEFT: one row per build row; a row no probe row reached is the NULL-padded row: COUNT(*) 1, COUNT(x) 0, SUM / MIN /
 *                  MAX / AVG NULL (and their Partial states: AVG [count 0, sum NULL]), so these columns are nullable.  Every
 *                  argument reads at least one input (probe) column and no payload field of the LEFT stage, and each of its nodes
 *                  propagates NULL (column, literal, arithmetic, comparison, CAST, NOT, negation: no IS [NOT] NULL, IS [NOT]
 *                  DISTINCT FROM, AND, OR), else DFGPU_ERR_UNSUPPORTED;
 *                LEFT_ANTI: no aggregates; one row per build row no probe row reached;
 *                and for both, a lookup whose build pushes held a NULL key ("null_keys" > 0) is DFGPU_ERR_UNSUPPORTED at the first
 *                push (those rows are not in the lookup, but the join emits them);
 *              every other sink over a LEFT / LEFT_ANTI stage is DFGPU_ERR_UNSUPPORTED;
 *              one such sink per lookup at a time (a second one, or a FULL stage, while it is alive: DFGPU_ERR_STATE).  A lookup
 *              serves any number of them in a row: each starts from zero.  When an earlier aggregate sink or FULL stage pushed into
 *              the words, this call zeroes the accumulator words of every record first (kernel-timing family "lookup_acc_reset",
 *              one write pass over capacity x stride x 8 bytes, not measured); a lookup fresh from creation or
 *              dfgpu_lookup_clear launches nothing;
 *  output    : surviving rows, columns = out_cols of the virtual schema, input order preserved. */
int dfgpu_pipeline_sink_build(dfgpu_pipeline* p, dfgpu_lookup* target, int32_t key_col, const int32_t* payload_cols, int32_t n_payload);
/* the build sink of a composite-key lookup (dfgpu_lookup_create_composite): key = the packed tuple of the INPUT columns key_cols[0..n_keys),
 * of the lookup's component types in order (else DFGPU_ERR_INVALID); payload as for dfgpu_pipeline_sink_build.  The packed keys are
 * hidden columns behind the inputs: input columns plus packed keys (this one and one per composite stage) must not exceed 16
 * (DFGPU_ERR_UNSUPPORTED). */
int dfgpu_pipeline_sink_build_composite(dfgpu_pipeline* p, dfgpu_lookup* target, const int32_t* key_cols, int32_t n_keys,
                                        const int32_t* payload_cols, int32_t n_payload);
int dfgpu_pipeline_sink_aggregate(dfgpu_pipeline* p, const int32_t* group_cols, int32_t n_group,
                                  const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size);
/* dense aggregate: AggregateExec over the surviving rows whose 0..8 group columns (virtual columns: input columns or payload
 * fields of INNER and RIGHT stages — an unmatched RIGHT row's field takes its column's NULL slot —, integer-like, <= 64 bits) take
 * values in small declared domains [key_min[g], key_max[g]] (column statistics).  The group of a row is arithmetic, slot = sum_g stride_g * idx_g with idx_g = key - key_min[g] for a value and
 * key_max[g] - key_min[g] + 1 for NULL (a group of its own), row-major strides; no hash table.  The domain may have at most
 * DFGPU_DENSE_MAX_GROUPS slots, prod_g (key_max[g] - key_min[g] + 2), else DFGPU_ERR_UNSUPPORTED; a key outside its range at run
 * time is DFGPU_ERR_INVALID.  n_group = 0 is AggregateStream: exactly one output row, also for empty input (COUNT 0; SUM, MIN, MAX,
 * AVG NULL).  Output: one row per slot that received a row, in slot order (ascending keys, NULL after the values of its column).
 * Up to 8 aggregates: COUNT(*), COUNT(x); SUM over integers (wrapping), Float64, Decimal128 (-> Decimal128(min(38, p+10), s));
 * MIN / MAX over integers, Date32, Float64, Decimal128; AVG over Float64 and Decimal128(p, s) -> Decimal128(min(38, p+4),
 * min(38, s+4)) = sum * 10^(ts - s) / count truncated toward zero, DFGPU_ERR_ARITH when that overflows i128 or the target
 * precision (DataFusion's DecimalAverager::avg).  mode = DFGPU_AGG_SINGLE* or DFGPU_AGG_PARTIAL (state columns as dfgpu_agg emits
 * them; Decimal128 AVG: Single modes only).  MAYBE stages are rejected (their false positives would be counted). */
#define DFGPU_DENSE_MAX_GROUPS 256
int dfgpu_pipeline_sink_aggregate_dense(dfgpu_pipeline* p, const int32_t* group_cols, const int64_t* key_min, const int64_t* key_max,
                                        int32_t n_group, const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size);
/* hash aggregate: AggregateExec over the surviving rows whose GROUP BY keys the join key does not determine (TPC-H Q15's revenue0:
 * l_suppkey; Q3 grouped by o_custkey).  The sink owns its group table.
 *  group_cols: 1..8 virtual columns (input columns or payload fields of INNER and RIGHT stages), integer-like, <= 8 bytes (Int8..Int64,
 *    UInt8..UInt64, Date32, Date64, Timestamp; dictionary-coded strings as their Int32 codes).  group_nullable[g] is the column's
 *    declared nullability (DataFusion's Field::is_nullable); NULL = none is nullable.  The columns are packed into a 128-bit tag,
 *    each at its width followed by one NULL bit when it is nullable; a key wider than 128 bits is DFGPU_ERR_UNSUPPORTED (dfgpu_agg
 *    carries wide keys).  NULL is a group of its own; a NULL in a column declared non-nullable is DFGPU_ERR_INVALID at the push
 *    (a RIGHT stage's payload field is NULL on every unmatched row, so it is declared nullable).
 *  aggs: the functions, limits and result / state types of dfgpu_pipeline_sink_aggregate (<= 4; COUNT(*), COUNT, SUM, MIN, MAX, AVG
 *    over Float64 and Decimal128; Decimal128 AVG in Single modes only; MIN / MAX over Float32 rejected).  The sink sizes the record
 *    words itself: {tag_lo | tag_hi | row counter | the aggregates' words as dfgpu_pipeline_sink_aggregate lays them out, every SUM /
 *    MIN / MAX with a non-null counter}.
 *  mode: DFGPU_AGG_SINGLE, DFGPU_AGG_SINGLE_PARTITIONED or DFGPU_AGG_PARTIAL (the state columns dfgpu_agg emits: its Final consumes them).
 *  MAYBE stages are rejected (their false positives would be counted).
 *  Output: one row per group, group columns then aggregates, in slot order (unspecified), sliced by batch_size.
 *  capacity_hint: the expected number of groups (0 = unknown); it sizes the first table only, results never depend on it.
 *  Growth: a push runs in row chunks of at most 2^26 rows (the first one max(2^20, capacity / 2) rows, then x4); before a chunk the
 *    table grows x4 when groups x 2 > capacity.  Inside the kernel claims stop at 5/8 of the capacity: a row whose group cannot be
 *    claimed is deferred (its row number goes to an overflow list bounded by the chunk's rows) before it touches any accumulator; the
 *    table grows x4 and the deferred rows are pushed again until none is left.  A table beyond 2^32 records is DFGPU_ERR_UNSUPPORTED.
 *  Metrics: "num_groups", "sink_rows" (every surviving row once, replayed rows included), "group_rehashes" (times the table grew),
 *    "replayed_rows" (rows deferred and pushed again). */
int dfgpu_pipeline_sink_aggregate_hash(dfgpu_pipeline* p, const int32_t* group_cols, const int32_t* group_nullable, int32_t n_group,
                                       const dfgpu_pipeline_agg* aggs, int32_t n_aggs, int32_t mode, int64_t batch_size,
                                       int64_t capacity_hint);
/* output: the surviving rows, columns = out_cols (1..16) of the virtual schema, input order preserved, sliced by batch_size (0 = one
 * batch).  Any input column may leave: widths 1, 2, 4, 8 and 16 bytes (Decimal128(p, s) included), with or without a validity bitmap
 * at any Arrow bit offset; payload fields leave too: those of a RIGHT stage always with a bitmap (bit = the row matched), the others
 * never nullable.  An input column leaves with a bitmap exactly when it had one in that push (a column pushed with null_count 0 has
 * none); once several pushes are merged, a column has one when any push gave it one.  Returned bitmap columns report null_count = -1 (unknown), as dfgpu_exchange_columns does.  Boolean input
 * columns are refused by the push (DFGPU_ERR_UNSUPPORTED), so they cannot be output. */
int dfgpu_pipeline_sink_output(dfgpu_pipeline* p, const int32_t* out_cols, int32_t n_out, int64_t batch_size);
/* the same, row order unspecified (what a RepartitionExec consumer sees anyway, repartition/mod.rs:1320-1400): runs on the two-phase
 * kernel and is several times faster than the ordered sink on selective pipelines; it takes the same columns, bitmaps and
 * Decimal128 values as the ordered sink */
int dfgpu_pipeline_sink_output_unordered(dfgpu_pipeline* p, const int32_t* out_cols, int32_t n_out, int64_t batch_size);
/* JoinFilter of probe stage `stage` (joins/utils.rs:1248-1320 apply_join_filter_to_indices; hash_join/stream.rs:896-906): a Boolean RPN
 * program evaluated on each probe row whose key matched at that stage (a candidate pair).  NULL or false means the pair does not match:
 *   INNER (Inner; LeftSemi as an INNER stage under the join-keyed sink), SEMI: the row continues when its key matches and the filter is TRUE;
 *   ANTI: the row continues unless its key matches and the filter is TRUE;
 *   LEFT: a record's row counter and accumulators take only the rows with filter TRUE; a build row no such row reached is the NULL-padded row;
 *   LEFT_ANTI: emits the records that no row with filter TRUE reached;
 *   MAYBE: DFGPU_ERR_UNSUPPORTED (a membership pre-filter has no candidate row to test).
 * Columns of stage s's filter: the input columns, then the payload fields of the INNER / LEFT / LEFT_ANTI stages 0..s in virtual-column
 * order, then, for a SEMI / ANTI stage only, that stage's own payload fields (seen by its filter only, not by later stages or sinks).
 * A lookup with payload has unique keys; a filter that reads no payload field also works over key sets and bitmaps with duplicates.
 * An error inside the filter (÷ 0, % 0, a failing CAST, Decimal128 overflow) is raised only on candidate pairs: a row without a key match,
 * or one an earlier stage dropped, never raises.  NULL probe keys never match.
 * Call after dfgpu_pipeline_create and before the first push; a call after the first push or a second one for the same stage is
 * DFGPU_ERR_STATE.  DFGPU_ERR_INVALID: a result that is not Boolean, a column index out of range (a later stage's payload field
 * included).  DFGPU_ERR_UNSUPPORTED: a MAYBE stage; an AND / OR whose right operand can raise (÷, %, CAST, Decimal128 arithmetic:
 * the per-batch short-circuit cannot be decided for payload fields; comparisons, wrapping integer + - *, Kleene AND / OR / NOT and
 * IS [NOT] NULL are accepted anywhere); more than 128 nodes over all filters of the pipeline.  A pipeline with a stage filter runs
 * neither the ring-fed nor the partitioned aggregate pass ("ring_launches" and "partitioned_launches" stay 0). */
int dfgpu_pipeline_set_stage_filter(dfgpu_pipeline* p, int32_t stage, const dfgpu_expr_node* expr, int32_t n_nodes);
/* Composite key of probe stage `stage`, whose lookup came from dfgpu_lookup_create_composite: the stage probes with the packed tuple of
 * the INPUT columns key_cols[0..n_keys) (components taken from payload fields of earlier stages are not supported).  Their types must be
 * the lookup's component types in order, and the stage's key_col must be key_cols[0] (DFGPU_ERR_INVALID); input columns plus packed keys
 * must not exceed 16 (DFGPU_ERR_UNSUPPORTED).  Call after dfgpu_pipeline_create, before the join-keyed aggregate sink and before the
 * first push (DFGPU_ERR_STATE otherwise, and for a second call on the stage); a push through a composite-key stage without its keys is
 * DFGPU_ERR_STATE.  The join-keyed aggregate sink then groups on ALL the components (plus payload fields of the stage): they are
 * decoded from the record's packed key, (key / stride_g) % r_g + key_min[g], at the component's type; for LEFT / LEFT_ANTI they are the
 * build key's components, never NULL.  The dense, hash and output sinks take the components as ordinary input columns. */
int dfgpu_pipeline_set_stage_keys(dfgpu_pipeline* p, int32_t stage, const int32_t* key_cols, int32_t n_keys);
/* Full join (HashJoinExec(Full), NullEqualsNothing, no JoinFilter): RIGHT stage `stage` also emits the build rows no probe row matched.
 * The output is (1) every probe row reaching the stage exactly as a RIGHT stage produces it, then (2) at dfgpu_pipeline_finish, one row per
 * build record that no surviving probe row matched: every input column NULL, the stage's payload fields the record's values.  The
 * ordered output sink keeps probe order for (1) and appends (2) in the lookup's slot order (DataFusion emits them in build order); both
 * output sinks emit (2) as batches of their own, after those of (1), each sliced by batch_size (batch_size 0: one batch each).  The
 * rows of (2) go through the same sink as any row: the output sinks write them with bitmaps, the dense sink puts their NULL input group
 * columns in the NULL slot, the hash sink sets their NULL bits (declare such group columns nullable), and every aggregate argument is
 * evaluated on them.  They are not counted in "input_rows"; "unmatched_build_rows" counts them.  With kernel timing on, the family
 * "pipe_full_tail:<name>" ("pipe_full_tail" without a name) times their selection and their push; "pipe:<name>" does not count them.
 * A finish whose push of (2) fails leaves the pipeline finished (a second dfgpu_pipeline_finish is DFGPU_ERR_STATE).
 * Each matched record is marked visited in the lookup's first accumulator word.  Call after dfgpu_pipeline_create, before the sink and
 * the first push (DFGPU_ERR_STATE otherwise).  DFGPU_ERR_INVALID: the stage is not RIGHT.  DFGPU_ERR_UNSUPPORTED: the stage is not the
 * pipeline's only stage; its lookup was not created with payload and n_acc_words >= 1; the inputs take all 16 column slots (the build
 * keys of (2) need one); the build side had a NULL key (at push or finish: such a row is not in the lookup).  DFGPU_ERR_STATE: the
 * lookup's marks (or accumulators) are already taken by another pipeline — one FULL pipeline per lookup until dfgpu_lookup_clear.  Words
 * an earlier join-keyed aggregate sink wrote are zeroed by this call, as dfgpu_pipeline_sink_aggregate does.  The
 * build, pack and join-keyed aggregate sinks and stage filters stay DFGPU_ERR_UNSUPPORTED, as for any RIGHT stage. */
int dfgpu_pipeline_set_stage_full(dfgpu_pipeline* p, int32_t stage);
/* optional label: this pipeline's kernel is timed under the family "pipe:<name>" (dfgpu_set_kernel_timing / dfgpu_kernel_time) —
 * the per-operator metrics set of a plan node (metrics(), execution_plan.rs:713) */
int dfgpu_pipeline_set_name(dfgpu_pipeline* p, const char* name);
int dfgpu_pipeline_push_host(dfgpu_pipeline* p, const dfgpu_column* cols, int32_t n_cols);    /* H2D inside, overlapped with the kernel in row chunks */
int dfgpu_pipeline_push_device(dfgpu_pipeline* p, const dfgpu_column* cols, int32_t n_cols);
int dfgpu_pipeline_push_arrow(dfgpu_pipeline* p, const struct ArrowArray* batch, const struct ArrowSchema* schema);
int dfgpu_pipeline_finish(dfgpu_pipeline* p);
int dfgpu_pipeline_next(dfgpu_pipeline* p, int host, dfgpu_batch** out);
int64_t dfgpu_pipeline_metric(dfgpu_pipeline* p, const char* name); /* "input_rows","sink_rows","output_rows","num_groups","ring_launches","dense_block_launches","partitioned_launches",
                                                                      "group_rehashes","replayed_rows","unmatched_build_rows",
                                                                      "partitioned_inserts": build sink pushes whose records went into a
                                                                      table larger than 40 MB (more than L2 holds) radix-partitioned by
                                                                      slot range, one L2-sized range at a time,
                                                                      "partitioned_records": {key, value} records the partitioned
                                                                      aggregate's first pass wrote (rows that passed the join key's
                                                                      membership filter, folded to 8 bits per key, and fit the record
                                                                      buffer) */
void dfgpu_pipeline_destroy(dfgpu_pipeline* p);

/* ===================================================================================== */
/* output batches                                                                        */
/* ===================================================================================== */
int64_t dfgpu_batch_num_rows(const dfgpu_batch* b);
int32_t dfgpu_batch_num_columns(const dfgpu_batch* b);
int dfgpu_batch_column(const dfgpu_batch* b, int32_t i, dfgpu_column* out);
int dfgpu_batch_is_host(const dfgpu_batch* b);
/* export a host batch as an Arrow C Data struct array; ownership of the buffers moves to the
 * ArrowArray's release callback (record_batch_stream.rs:101-110 is the consumer side). */
int dfgpu_batch_export_arrow(dfgpu_batch* b, struct ArrowArray* out_array, struct ArrowSchema* out_schema);
void dfgpu_batch_release(dfgpu_batch* b);

/* ===================================================================================== */
/* exchange: RepartitionExec hash partitioning (physical-plan/src/repartition/mod.rs:1097-1145)
 * — the local pass that precedes the NCCL all-to-all.                                    */
/* ===================================================================================== */

/* Scatter the rows of `cols` (device) into n_parts contiguous regions by
 * partition = exchange_hash(key columns) % n_parts.  Output columns are library-owned device
 * buffers of the same types, with a validity bitmap wherever the input column had one;
 * part_offsets_host[n_parts+1] receives the region boundaries.  Keys: 1..4 fixed-width columns
 * of <= 128 bits each (Decimal128 included); a NULL key leaves the running hash untouched. */
int dfgpu_hash_partition_device(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols,
                                const int32_t* key_cols, int32_t n_keys, int32_t n_parts,
                                dfgpu_batch** out, int64_t* part_offsets_host);

/* Fused partition + exchange over peer memory (NVLink): the scatter writes each row straight into the receive
 * buffer of the GPU that owns its partition — no staging copy, no NCCL payload transfer.  Phase 1 counts rows per
 * destination (the caller all-gathers the counts to learn where its block starts in every receiver), phase 2
 * scatters.  dst_bases[p * n_cols + c] points at column c of rank p's receive buffer (mapped with dfgpu_ipc_import;
 * the local pointer for p == own rank); dst_row_offset[p] is the first row this rank owns in that buffer.
 * Columns: <= 16, fixed-width or Boolean, nullable or not; keys as for dfgpu_hash_partition_device.  A plan with a
 * nullable (validity bitmap) or Boolean column is scattered with dfgpu_partition_plan_scatter_peer_chunk_nullable
 * only: the two calls below refuse it with DFGPU_ERR_INVALID rather than drop its bits. */
typedef struct dfgpu_partition_plan dfgpu_partition_plan;
int dfgpu_partition_plan_create(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys,
                                int32_t n_parts, int64_t* counts_host, dfgpu_partition_plan** out);
int dfgpu_partition_plan_scatter_peer(dfgpu_partition_plan* plan, void* const* dst_bases, const int64_t* dst_row_offset);
/* Chunked form, for overlapping the exchange with the consumer (RepartitionExec streams batches to HashJoinExec the
 * same way, repartition/mod.rs:1320-1400): the input is cut into n_chunks contiguous row ranges, counts_host is
 * [n_chunks][n_parts], and each chunk is scattered by its own call (dst_row_offset[p] = first row of this rank's
 * (chunk, p) block at receiver p) so the receiver can start on chunk c while chunk c+1 is still on the wire. */
int dfgpu_partition_plan_create_chunked(dfgpu_ctx* ctx, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys,
                                        int32_t n_parts, int32_t n_chunks, int64_t* counts_host, dfgpu_partition_plan** out);
int dfgpu_partition_plan_scatter_peer_chunk(dfgpu_partition_plan* plan, int32_t chunk, void* const* dst_bases, const int64_t* dst_row_offset);
/* The same with bit-packed data.  dst_validity[p * n_cols + c] is rank p's receive bitmap for column c, or NULL when column c
 * keeps no bitmap at the receivers (then for every p; a column whose input has NULLs needs one).  dst_validity itself may be
 * NULL: no column keeps a bitmap.  A source column without a bitmap writes all-ones into its block of a receive bitmap, so
 * senders may disagree on nullability.  A Boolean column's dst_bases entry is its receive bitmap, addressed in bits like the
 * validity (row r = bit r).  Bitmap pointers must be 4-byte aligned and readable and writable in whole 32-bit words.  Only
 * the bits of this rank's block change, with atomic updates (system scope in peer memory) of the words it shares with a
 * neighbouring block: receive bitmaps need no zeroing, and several ranks may scatter into one bitmap at the same time. */
int dfgpu_partition_plan_scatter_peer_chunk_nullable(dfgpu_partition_plan* plan, int32_t chunk, void* const* dst_bases, void* const* dst_validity,
                                                     const int64_t* dst_row_offset);
void dfgpu_partition_plan_destroy(dfgpu_partition_plan* plan);
/* CUDA IPC: export a device allocation made with dfgpu_malloc (64-byte handle) / map a peer's allocation */
int dfgpu_ipc_export(dfgpu_ctx* ctx, void* dev_ptr, uint8_t* handle_out);
int dfgpu_ipc_import(dfgpu_ctx* ctx, const uint8_t* handle, void** peer_ptr_out);
int dfgpu_ipc_close(dfgpu_ctx* ctx, void* peer_ptr);

/* ===================================================================================== */
/* dictionary-coded string keys.  The reference joins / groups on Utf8, Utf8View and Dictionary(_, Utf8) columns by hashing and
 * comparing bytes (common/src/hash_utils.rs create_hashes; aggregates/group_values/mod.rs:139-217 GroupValuesBytes /
 * GroupValuesBytesView; the TPC-H string columns, benchmarks/src/tpch/mod.rs:52-122).  On the GPU path a string key is an INT32
 * code — every integer-key operator applies — provided all batches (and both join sides) share ONE code space.  Arrow
 * dictionaries are per batch: a dfgpu_dictionary unifies them on the host (the distinct values are few next to the rows),
 * dfgpu_dictionary_remap rewrites a batch's codes on the device.  A literal (`c_mktsegment = 'BUILDING'`) becomes
 * `codes = dfgpu_dictionary_code(...)`; a string never seen matches nothing (-1).               */
/* ===================================================================================== */
typedef struct dfgpu_dictionary dfgpu_dictionary;
int dfgpu_dictionary_create(dfgpu_ctx* ctx, dfgpu_dictionary** out);
/* merge one batch's dictionary values (Arrow Utf8 layout: offsets[n_values + 1], data; validity = LSB bitmap or NULL) into the
 * unified dictionary; remap_out[i] = unified code of local value i, -1 for a NULL value.  Host-side. */
int dfgpu_dictionary_unify(dfgpu_dictionary* d, const int32_t* offsets, const uint8_t* data, const uint8_t* validity, int64_t n_values, int32_t* remap_out);
int32_t dfgpu_dictionary_code(dfgpu_dictionary* d, const uint8_t* bytes, int64_t len);   /* -1 = not present */
int64_t dfgpu_dictionary_size(dfgpu_dictionary* d);
int dfgpu_dictionary_value(dfgpu_dictionary* d, int32_t code, const uint8_t** bytes, int64_t* len);   /* valid until the next unify */
/* codes: the batch's keys column (any integer type; host buffers when codes_on_host != 0, else device pointers); out: one INT32
 * device column with out[i] = remap[codes[i]], NULL where the input is NULL or the dictionary value is NULL.  A code outside
 * [0, n_remap) is DFGPU_ERR_INVALID. */
int dfgpu_dictionary_remap(dfgpu_dictionary* d, const dfgpu_column* codes, int codes_on_host, const int32_t* remap, int64_t n_remap, dfgpu_batch** out);
void dfgpu_dictionary_destroy(dfgpu_dictionary* d);

/* ===================================================================================== */
/* multi-GPU control inside the ABI (one process or thread per GPU of ONE box): what a Rust host needs to drive the partition
 * exchange without NCCL / torch.distributed.  Control plane: a POSIX shared-memory segment named after a 128-byte unique id the
 * application hands to every rank (the role of ncclUniqueId); data plane: CUDA IPC — every rank maps every peer's receive buffers
 * and the scatter kernel stores rows straight into the owner's HBM over NVLink.  Reference analogue: the channels of RepartitionExec
 * (physical-plan/src/repartition/mod.rs:618-648, 1320-1400).                              */
/* ===================================================================================== */
typedef struct dfgpu_comm dfgpu_comm;
typedef struct dfgpu_exchange dfgpu_exchange;
int dfgpu_comm_unique_id(uint8_t* id_out /* 128 bytes */);      /* call once, broadcast to every rank by any means */
int dfgpu_comm_init(dfgpu_ctx* ctx, int32_t n_ranks, int32_t rank, const uint8_t* id /* 128 bytes */, dfgpu_comm** out); /* collective */
int32_t dfgpu_comm_rank(dfgpu_comm* c);
int32_t dfgpu_comm_size(dfgpu_comm* c);
/* collective: returns once every rank's ctx stream has drained and every rank has arrived */
int dfgpu_comm_barrier(dfgpu_comm* c);
/* collective: all[r][0..n) = rank r's `mine` (n <= 64): the count matrix of an exchange */
int dfgpu_comm_allgather_i64(dfgpu_comm* c, const int64_t* mine, int32_t n, int64_t* all);
/* collective: share a device allocation made with dfgpu_malloc; peer_ptrs_out[r] = rank r's buffer mapped here (own pointer for r == rank) */
int dfgpu_comm_share(dfgpu_comm* c, void* dev_ptr, void** peer_ptrs_out);
void dfgpu_comm_destroy(dfgpu_comm* c);
/* RepartitionExec Hash(key columns) across the ranks (repartition/mod.rs:1097-1145): persistent receive buffers of cap_rows rows per
 * column and a receive validity bitmap of cap_rows bits per column, shared once; one run = histogram -> count all-gather (which also
 * tells every rank which columns some sender holds with a validity bitmap) -> fused partition + peer-memory scatter -> barrier.  Rows
 * arrive grouped by source rank, in source order.  Column types: fixed-width up to 16 bytes (Decimal128(p, s) included) or Boolean,
 * nullable or not.  All three calls are collective. */
int dfgpu_exchange_create(dfgpu_comm* c, const int32_t* col_types, int32_t n_cols, int64_t cap_rows, dfgpu_exchange** out);
int dfgpu_exchange_run(dfgpu_exchange* x, const dfgpu_column* cols, int32_t n_cols, const int32_t* key_cols, int32_t n_keys, int64_t* recv_rows_out);
/* device views of the received rows (valid until the next run); a column some sender held with a validity bitmap comes with the
 * receive bitmap and null_count -1, the others with validity NULL */
int dfgpu_exchange_columns(dfgpu_exchange* x, dfgpu_column* out, int32_t n_cols);
void dfgpu_exchange_destroy(dfgpu_exchange* x);

#ifdef __cplusplus
}
#endif
#endif /* DFGPU_H */
