/*
 * dfgpu_strings.h — C ABI of libdfgpu_strings.so: string predicates on the H100 (sm_90a) that turn a string column into a one-byte
 * mask column, for DataFusion's `LikeExpr` (reference datafusion/physical-expr/src/expressions/like.rs, whose `evaluate` calls
 * arrow-string's `like` / `nlike` kernels, arrow-string/src/like.rs), for a `BinaryExpr` comparing a string column with a Utf8 literal
 * (expressions/binary.rs -> arrow-ord's `eq` / `neq` / `lt` / `lt_eq` / `gt` / `gt_eq`, arrow-ord/src/cmp.rs) and for an `InListExpr`
 * of a string column over a static list of Utf8 literals (expressions/in_list.rs).
 *
 * The library stands apart from libdfgpu.so and does not link it: it includes dfgpu.h only for `dfgpu_column` and the status codes.
 * Every call enqueues its kernels on the caller's CUDA stream (a libdfgpu ctx's `dfgpu_ctx_stream(ctx)`) and returns; it makes no
 * device allocation and no stream synchronise.  Inputs and outputs are device buffers the caller owns (e.g. from `dfgpu_malloc`); they
 * must stay valid until the stream has run the call's work.  The output mask is an ordinary DFGPU_UINT8 column at offset 0, so it
 * feeds dfgpu_filter, dfgpu_expr_evaluate_* and dfgpu_pipeline like any other input column (a predicate `mask = 1` keeps SQL's
 * three-valued logic: a NULL mask gives NULL).
 *
 * Semantics of `s LIKE p` (anchored whole-string match over Unicode code points):
 *   - `%` matches any run of zero or more code points, `_` exactly one code point (1 to 4 bytes of UTF-8); every other character matches
 *     itself.  Case-sensitive; newline and NUL are ordinary characters.
 *   - a NULL string gives NULL for LIKE and for NOT LIKE; on a non-NULL string NOT LIKE is the negation of LIKE.
 *   - string data is Arrow's: valid UTF-8 (the kernels do not validate it).
 * Refused with DFGPU_ERR_UNSUPPORTED (the caller keeps the CPU LikeExpr):
 *   - a pattern containing `\` (arrow-string's literal fast paths and its regex translation need not agree on an escape);
 *   - DFGPU_LIKE_CASE_INSENSITIVE (ILIKE needs Unicode case folding);
 *   - a pattern longer than DFGPU_LIKE_MAX_PATTERN_BYTES bytes, or with more than DFGPU_LIKE_MAX_SEGMENTS non-empty `%`-separated pieces.
 * Rejected with DFGPU_ERR_INVALID: a pattern that is not valid UTF-8, and malformed arguments.
 * A column pattern (`a LIKE b`) and a custom ESCAPE never reach the library: the planner leaves them on the CPU.
 *
 * Semantics of `s op literal` (dfgpu_string_compare), op one of =, <>, <, <=, >, >=:
 *   - Arrow's order for strings: byte-wise lexicographic over the UTF-8 bytes (which is code-point order), a proper prefix sorts first;
 *     equal means equal length and equal bytes.  No collation, no case folding, no trimming.
 *   - a NULL string gives NULL; on a non-NULL string the result is in {0, 1}.
 * Semantics of `s [NOT] IN (v1, v2, ...)` (dfgpu_string_in_list), SQL's three-valued IN as InListExpr evaluates a static list:
 *   - a NULL string gives NULL;
 *   - a string equal to some vi gives 1 for IN and 0 for NOT IN;
 *   - a string equal to none gives NULL when the list holds a NULL (list_has_null), else 0 for IN and 1 for NOT IN.
 *   So a non-NULL string can give NULL.
 * Refused with DFGPU_ERR_UNSUPPORTED (the caller keeps the CPU expression): a comparison literal longer than
 * DFGPU_STRING_MAX_LITERAL_BYTES; a list of more than DFGPU_STRING_IN_MAX_VALUES distinct values or more than DFGPU_STRING_IN_MAX_BYTES
 * bytes of them; a list holding a NULL over a Utf8View column of more than 240 data buffers (pass the list without its NULL and add the
 * NULL by Kleene logic: IN is `mask OR NULL`, NOT IN is `mask AND NULL`).  Rejected with DFGPU_ERR_INVALID: a literal or list value
 * that is not valid UTF-8, an unknown op, malformed arguments.
 * A column compared with a column never reaches the library.
 *
 * How rows are settled, cheapest bytes first: a Utf8 / LargeUtf8 row's length comes from its two offsets, so `=` / `<>` against a literal
 * of another length, and an IN row whose length is no value's length, read no string bytes; an ordering comparison stops at the first
 * byte that differs.  A Utf8View row is settled from its 16-byte view (the length, the 4-byte prefix, the whole string when it is 12
 * bytes or shorter); its data buffer is read only for a longer string the view leaves open.  An IN row is looked up by a hash of its
 * bytes in a table of the values, and only the values in its probe sequence are compared byte for byte.
 * Dictionary codes: evaluate the predicate over the dictionary's distinct values, then map each row's code with dfgpu_like_codes.
 */
#ifndef DFGPU_STRINGS_H
#define DFGPU_STRINGS_H

#include "dfgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

enum dfgpu_string_layout {
  DFGPU_STRING_UTF8 = 1,       /* Utf8: int32 offsets[offset .. offset + length], one data buffer      */
  DFGPU_STRING_LARGE_UTF8 = 2, /* LargeUtf8: int64 offsets, one data buffer                           */
  DFGPU_STRING_UTF8_VIEW = 3   /* Utf8View: 16-byte views (16-byte aligned), any number of data buffers */
};

#define DFGPU_LIKE_NEGATED 1            /* NOT LIKE */
#define DFGPU_LIKE_CASE_INSENSITIVE 2   /* ILIKE: always DFGPU_ERR_UNSUPPORTED */
#define DFGPU_LIKE_MAX_PATTERN_BYTES 256
#define DFGPU_LIKE_MAX_SEGMENTS 16

enum dfgpu_string_cmp_op {
  DFGPU_STRING_EQ = 0, /* =  */
  DFGPU_STRING_NE = 1, /* <> */
  DFGPU_STRING_LT = 2, /* <  */
  DFGPU_STRING_LE = 3, /* <= */
  DFGPU_STRING_GT = 4, /* >  */
  DFGPU_STRING_GE = 5  /* >= */
};
#define DFGPU_STRING_MAX_LITERAL_BYTES 256   /* longest comparison literal */
#define DFGPU_STRING_IN_MAX_VALUES 64        /* most distinct non-NULL values of an IN list */
#define DFGPU_STRING_IN_MAX_BYTES 1024       /* most bytes of those values together */

/* One Arrow string array resident in HBM.  The kernels read only [data + offsets[offset], data + offsets[offset + length]) of a Utf8 /
 * LargeUtf8 array, and of a Utf8View array only the views of rows [offset, offset + length) and the bytes those views point at, so
 * unpadded buffers are fine. */
typedef struct dfgpu_string_column {
  int32_t layout;                     /* enum dfgpu_string_layout */
  int32_t n_data_buffers;             /* 1 for Utf8 / LargeUtf8; the variadic buffer count of a Utf8View (may be 0) */
  int64_t length;                     /* rows */
  int64_t offset;                     /* logical offset (elements) into offsets / views and validity */
  int64_t null_count;                 /* -1 = unknown (informational) */
  const void* offsets_or_views;       /* device: the offsets buffer, or the views buffer */
  const uint8_t* const* data_buffers; /* HOST array of n_data_buffers DEVICE pointers */
  const uint8_t* validity;            /* device LSB bitmap, or NULL = all valid */
} dfgpu_string_column;

/* LikeExpr::evaluate with a scalar Utf8 pattern (like.rs; arrow-string `like` / `nlike`).  stream: a cudaStream_t (NULL = legacy stream).
 * pattern: pattern_len bytes of UTF-8 (no terminator needed).  flags: DFGPU_LIKE_NEGATED and / or DFGPU_LIKE_CASE_INSENSITIVE.
 * Writes out_values[0 .. length) in {0, 1} (0 under NULL rows).  When col->validity is set, out_validity (at least (length + 7) / 8
 * bytes) receives the rows' validity rebased to bit 0; when it is NULL, out_validity is not written and may be NULL. */
int dfgpu_like(void* stream, const dfgpu_string_column* col, const uint8_t* pattern, int64_t pattern_len, int32_t flags,
               uint8_t* out_values, uint8_t* out_validity);

/* `col op literal` (BinaryExpr with a scalar Utf8 right operand).  op: enum dfgpu_string_cmp_op.  literal: literal_len bytes of UTF-8
 * (no terminator needed).  Outputs as in dfgpu_like. */
int dfgpu_string_compare(void* stream, const dfgpu_string_column* col, int32_t op, const uint8_t* literal, int64_t literal_len,
                         uint8_t* out_values, uint8_t* out_validity);

/* `col [NOT] IN (values)` (InListExpr with a static list).  values: a HOST array of n_values HOST pointers to the non-NULL values, each
 * value_lens[i] bytes of UTF-8 (duplicates allowed); list_has_null: the list also holds a NULL; negated: NOT IN.  Writes out_values[0 ..
 * length) in {0, 1} (0 under NULL results).  out_validity (at least (length + 7) / 8 bytes) receives each result's validity rebased to
 * bit 0; it is written when col->validity is set or list_has_null is, and may be NULL otherwise. */
int dfgpu_string_in_list(void* stream, const dfgpu_string_column* col, const uint8_t* const* values, const int64_t* value_lens,
                         int64_t n_values, int32_t list_has_null, int32_t negated, uint8_t* out_values, uint8_t* out_validity);

/* Any of these predicates over dictionary codes (an INT32 dfgpu_column of codes into one dictionary, e.g. dfgpu_dictionary_remap's
 * output): code_match[0 .. n_codes) holds the predicate's value for each distinct value (dfgpu_like, dfgpu_string_compare or
 * dfgpu_string_in_list over the dictionary values, any negation already applied).  out_values[i] = code_match[codes[i]]; a NULL code
 * gives NULL (out_validity as in dfgpu_like); a code outside [0, n_codes) gives 0.  The map carries values only: a predicate that can
 * be NULL on a non-NULL value (an IN list holding a NULL) is mapped for its non-NULL values and combined with the NULL by the caller. */
int dfgpu_like_codes(void* stream, const dfgpu_column* codes, const uint8_t* code_match, int64_t n_codes, uint8_t* out_values,
                     uint8_t* out_validity);

/* ---- the gather: arrow-select's `take` over string arrays (late materialisation of carried string columns) ----
 * sources: n_sources >= 1 string arrays of ONE layout, any slice offset, each at most 2^32 - 1 rows.  ids: a device dfgpu_column of
 *   DFGPU_UINT32 rows of sources[0] (a join's build side, concatenated into one array), or of DFGPU_INT64 ids packed as
 *   source << 32 | row (a streamed side whose output rows come from several batches), with its own offset and validity.
 * Output row i is the string sources[src(i)][row(i)]: NULL where the id is NULL (the outer side of an outer join) or the source string
 *   is NULL.  An id naming no source or a row outside its source is DFGPU_ERR_INVALID; the kernels cannot return it, so they count such
 *   ids in a device word the caller reads with the output size (below), and the output row is NULL.
 * Only the offsets / views of the rows the ids name, and those rows' bytes, are read.  Any number of sources works (64 to a launch). */

/* Utf8 / LargeUtf8, phase 1.  scratch: dfgpu_string_take_scratch_bytes(ids->length) bytes of device memory, kept for phase 2.
 * offsets: ids->length + 3 int64 of device memory.  Writes offsets[0 .. n) = the exclusive scan of the output rows' byte lengths (a
 * NULL row takes 0 bytes), offsets[n] = the total bytes, offsets[n + 1] = the number of out-of-range ids (0 = no error),
 * offsets[n + 2] = the number of NULL output rows; out_validity ((n + 7) / 8 bytes) receives the output validity rebased to bit 0. */
int64_t dfgpu_string_take_scratch_bytes(int64_t n_ids);
int dfgpu_string_take_offsets(void* stream, const dfgpu_string_column* sources, int32_t n_sources, const dfgpu_column* ids, void* scratch,
                              int64_t* offsets, uint8_t* out_validity);
/* Utf8 / LargeUtf8, phase 2, after the caller has read offsets[n .. n + 3) and refused out-of-range ids: layout: the sources' layout;
 * total_bytes: offsets[n]; scratch and offsets as phase 1 left them.  Writes out_offsets (n + 1 int32 for Utf8, int64 for LargeUtf8,
 * which may be `offsets` itself) and out_data (total_bytes bytes).  A Utf8 output beyond 2^31 - 1 bytes is DFGPU_ERR_INVALID ("offset
 * overflow", as arrow's `take` refuses it). */
int dfgpu_string_take_data(void* stream, int32_t layout, int64_t n_ids, int64_t total_bytes, const void* scratch, const int64_t* offsets,
                           void* out_offsets, uint8_t* out_data);
/* Utf8View: one phase.  Writes out_views (ids->length 16-byte views, 16-byte aligned): a view of 12 bytes or fewer as it is, a longer
 * one with its buffer index rebased by its source's first buffer in the output's buffer list, which is the concatenation of the
 * sources' data buffers in source order (no string byte is copied); a NULL row is a zero view.  out_validity: 4-byte aligned, room for
 * (n + 31) / 32 32-bit words, receives the validity rebased to bit 0.  status: 2 int64 of device memory: [0] out-of-range ids, [1] NULL
 * output rows. */
int dfgpu_string_take_views(void* stream, const dfgpu_string_column* sources, int32_t n_sources, const dfgpu_column* ids, void* out_views,
                            uint8_t* out_validity, int64_t* status);

/* the message of this thread's last failed call ("" when none) */
const char* dfgpu_strings_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* DFGPU_STRINGS_H */
