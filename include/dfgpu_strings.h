/*
 * dfgpu_strings.h — C ABI of libdfgpu_strings.so: string predicates on the H100 (sm_90a) that turn a string column into a one-byte
 * mask column, for DataFusion's `LikeExpr` (reference datafusion/physical-expr/src/expressions/like.rs, whose `evaluate` calls
 * arrow-string's `like` / `nlike` kernels, arrow-string/src/like.rs).
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

/* The same predicate over dictionary codes (an INT32 dfgpu_column of codes into one dictionary, e.g. dfgpu_dictionary_remap's output):
 * code_match[0 .. n_codes) holds the predicate's value for each distinct value (dfgpu_like over the dictionary values, NOT LIKE
 * already applied).  out_values[i] = code_match[codes[i]]; a NULL code gives NULL (out_validity as in dfgpu_like); a code outside
 * [0, n_codes) gives 0. */
int dfgpu_like_codes(void* stream, const dfgpu_column* codes, const uint8_t* code_match, int64_t n_codes, uint8_t* out_values,
                     uint8_t* out_validity);

/* the message of this thread's last failed call ("" when none) */
const char* dfgpu_strings_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* DFGPU_STRINGS_H */
