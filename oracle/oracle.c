/*
 * oracle.c — CPU RESTATEMENT of apache/datafusion 55.0.0's HashJoinExec / AggregateExec /
 * RepartitionExec algorithms for the hot path of SURVEY.md §8.
 *
 *   THIS IS TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's
 *   cpu_baseline / --impl reference legs may load it.  libdfgpu.so never links or calls it.
 *
 * The reference is Rust and cannot be compiled in this image (no cargo/rustc), so this file
 * restates its algorithms in plain C, each function citing the reference file:line it follows
 * (paths relative to /root/reference/datafusion/).  It is pinned against the reference's own
 * unit-test fixtures transcribed into tests/golden/ (see tests/golden/README.md).
 *
 * PARITY UNPINNED (hash values only): the reference hashes with foldhash 0.2 (third-party crate,
 * common/src/hash_utils.rs:27,41), which is not restated; o_hash() below is a stand-in.  Hash
 * values never reach operator output (join order = probe order x ascending build index,
 * group ids = first-seen order), so every output of this file is independent of the hash
 * function; the reference's force_hash_collisions mode (hash = 0) is reproduced to prove it.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>
#include <pthread.h>
#include <time.h>
#include "gen.h"

#define O_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------ */
/* hashing: create_hashes (common/src/hash_utils.rs:1239-1254, hash_array_primitive :306-345)   */
/*   first column: hash_one(value); later columns: re-seed with the running hash;              */
/*   NULLs leave the slot untouched (0 for column 0).  Seeds: join 12210250226015887276        */
/*   (hash_join/exec.rs:105), aggregate 15395726432021054657 (aggregates/mod.rs:236),          */
/*   repartition 0 (repartition/mod.rs:650).                                                   */
/* ------------------------------------------------------------------------------------------ */
#define SEED_JOIN 12210250226015887276ull
#define SEED_AGG 15395726432021054657ull
#define SEED_REPART 0ull

static inline uint64_t o_hash(uint64_t v, uint64_t seed) { return o_mix64(v ^ o_mix64(seed + 0x9E3779B97F4A7C15ull)); }
/* a double's bits as an unsigned key that sorts in IEEE totalOrder: all bits flipped when the sign is set, else the sign bit set */
static inline uint64_t f64_total_order(double d) { uint64_t b; memcpy(&b, &d, 8); return (b >> 63) ? ~b : (b | 0x8000000000000000ull); }

static void create_hashes(int nkeys, const int64_t* const* keys, const uint8_t* const* valid, int64_t start, int64_t n,
                          uint64_t seed, int force_collisions, uint64_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = 0;
  if (force_collisions) return; /* feature force_hash_collisions: hash_utils.rs:1185-1205 */
  for (int c = 0; c < nkeys; ++c) {
    for (int64_t i = 0; i < n; ++i) {
      if (valid && valid[c] && !valid[c][start + i]) continue;
      uint64_t v = (uint64_t)keys[c][start + i];
      out[i] = (c == 0) ? o_hash(v, seed) : o_hash(v, out[i]);
    }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* JoinHashMap: hash -> (hash, last_row+1) + next[] chain  (joins/join_hash_map.rs:143-162)    */
/* hashbrown's HashTable is restated as linear probing over (hash, idx) entries; layout is     */
/* irrelevant to results.                                                                      */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  uint64_t* hashes;
  uint64_t* idx; /* row + 1; 0 = empty */
  uint64_t mask;
  uint64_t len;   /* number of distinct hashes: map.len() */
  uint64_t* next; /* next[row] = previous head (row+1) or 0 */
  uint64_t next_len;
} JoinHashMap;

static void jhm_init(JoinHashMap* m, uint64_t cap_rows) {
  uint64_t cap = 16;
  while (cap < cap_rows * 2 + 2) cap <<= 1;
  m->hashes = (uint64_t*)calloc(cap, 8);
  m->idx = (uint64_t*)calloc(cap, 8);
  m->mask = cap - 1;
  m->len = 0;
  m->next = (uint64_t*)calloc(cap_rows ? cap_rows : 1, 8);
  m->next_len = cap_rows;
}
static void jhm_free(JoinHashMap* m) { free(m->hashes); free(m->idx); free(m->next); }

/* update_from_iter, join_hash_map.rs:307-337 */
static inline void jhm_insert(JoinHashMap* m, uint64_t row, uint64_t hash) {
  uint64_t s = o_mix64(hash) & m->mask;
  while (m->idx[s] != 0 && m->hashes[s] != hash) s = (s + 1) & m->mask;
  if (m->idx[s] != 0) {
    uint64_t prev = m->idx[s]; /* Occupied: chain the previous head behind the new row */
    m->idx[s] = row + 1;
    m->next[row] = prev;
  } else {
    m->hashes[s] = hash;
    m->idx[s] = row + 1;
    m->len++;
  }
}
static inline uint64_t jhm_find(const JoinHashMap* m, uint64_t hash) {
  uint64_t s = o_mix64(hash) & m->mask;
  while (m->idx[s] != 0) {
    if (m->hashes[s] == hash) return m->idx[s];
    s = (s + 1) & m->mask;
  }
  return 0;
}

/* growable index vectors */
typedef struct { int64_t* p; int64_t n, cap; } Vec64;
static void v_push(Vec64* v, int64_t x) {
  if (v->n == v->cap) { v->cap = v->cap ? v->cap * 2 : 1024; v->p = (int64_t*)realloc(v->p, (size_t)v->cap * 8); }
  v->p[v->n++] = x;
}

/* MapOffset = (usize, Option<u64>)  (joins/mod.rs:88) */
typedef struct { int64_t idx; int has_next; uint64_t next; } MapOffset;

/* traverse_chain, joins/chain.rs:29-70.  Returns 1 and sets *out when the limit was hit. */
static int traverse_chain(const uint64_t* next_chain, int64_t prob_idx, uint64_t start_chain_idx, int64_t* remaining,
                          Vec64* input_indices, Vec64* match_indices, int is_last_input, MapOffset* out) {
  uint64_t match_row_idx = start_chain_idx - 1;
  for (;;) {
    v_push(match_indices, (int64_t)match_row_idx);
    v_push(input_indices, prob_idx);
    *remaining -= 1;
    uint64_t next = next_chain[match_row_idx];
    if (*remaining == 0) {
      if (is_last_input && next == 0) return 0; /* finished the last input row */
      out->idx = prob_idx; out->has_next = 1; out->next = next;
      return 1;
    }
    if (next == 0) return 0;
    match_row_idx = next - 1;
  }
}

/* get_matched_indices_with_limit_offset, join_hash_map.rs:389-484.
 * hash_values: hashes of the probe batch; valid_keys[i]==0: NULL key (skipped).
 * Returns 1 if there is a next offset. */
static int jhm_lookup(const JoinHashMap* m, const uint64_t* hash_values, const uint8_t* valid_keys, int64_t len, int64_t limit,
                      MapOffset offset, Vec64* input_indices, Vec64* match_indices, MapOffset* next_offset) {
  input_indices->n = 0;
  match_indices->n = 0;
  if (m->len == m->next_len) { /* unique fast path :410-429 */
    int64_t start = offset.idx;
    int64_t end = start + limit < len ? start + limit : len;
    for (int64_t i = start; i < end; ++i) {
      if (valid_keys && !valid_keys[i]) continue;
      uint64_t idx = jhm_find(m, hash_values[i]);
      if (idx) { v_push(input_indices, i); v_push(match_indices, (int64_t)(idx - 1)); }
    }
    if (end == len) return 0;
    next_offset->idx = end; next_offset->has_next = 0; next_offset->next = 0;
    return 1;
  }
  int64_t remaining = limit;
  int64_t to_skip;
  if (!offset.has_next) to_skip = offset.idx;
  else if (offset.next == 0) to_skip = offset.idx + 1;
  else {
    int is_last = offset.idx == len - 1;
    if (traverse_chain(m->next, offset.idx, offset.next, &remaining, input_indices, match_indices, is_last, next_offset)) return 1;
    to_skip = offset.idx + 1;
  }
  for (int64_t row_idx = to_skip; row_idx < len; ++row_idx) {
    if (valid_keys && !valid_keys[row_idx]) continue;
    uint64_t idx = jhm_find(m, hash_values[row_idx]);
    if (idx) {
      int is_last = row_idx == len - 1;
      if (traverse_chain(m->next, row_idx, idx, &remaining, input_indices, match_indices, is_last, next_offset)) return 1;
    }
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* ArrayMap (joins/array_map.rs:103-372) and its selection rule (hash_join/exec.rs:111-191)     */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  uint32_t* data; uint64_t data_len; uint64_t offset;
  uint32_t* next; uint64_t next_len; /* next_len == 0: no duplicate keys */
} ArrayMap;

static void amap_fill(ArrayMap* a, const int64_t* key, const uint8_t* valid, int64_t n, uint64_t min_val, uint64_t max_val) {
  uint64_t range = max_val - min_val; /* calculate_range: wrapping_sub */
  a->data_len = range + 1;
  a->data = (uint32_t*)calloc(a->data_len, 4);
  a->offset = min_val;
  a->next = NULL;
  a->next_len = 0;
  /* fill_data :205-236: iterate in reverse so chains come out ascending */
  for (int64_t i = n - 1; i >= 0; --i) {
    if (valid && !valid[i]) continue;
    uint64_t idx = (uint64_t)key[i] - min_val;
    if (a->data[idx] != 0) {
      if (a->next_len == 0) { a->next = (uint32_t*)calloc((size_t)n, 4); a->next_len = (uint64_t)n; }
      a->next[i] = a->data[idx];
    }
    a->data[idx] = (uint32_t)i + 1;
  }
}
static inline uint32_t amap_get(const ArrayMap* a, uint64_t key) {
  uint64_t idx = key - a->offset; /* key_to_index :159-166 (wrapping) */
  if (idx >= a->data_len) return 0;
  return a->data[idx];
}
static int traverse_chain32(const uint32_t* next_chain, int64_t prob_idx, uint32_t start, int64_t* remaining, Vec64* pi, Vec64* bi,
                            int is_last, MapOffset* out) {
  uint64_t match_row_idx = (uint64_t)start - 1;
  for (;;) {
    v_push(bi, (int64_t)match_row_idx);
    v_push(pi, prob_idx);
    *remaining -= 1;
    uint32_t next = next_chain[match_row_idx];
    if (*remaining == 0) {
      if (is_last && next == 0) return 0;
      out->idx = prob_idx; out->has_next = 1; out->next = next;
      return 1;
    }
    if (next == 0) return 0;
    match_row_idx = (uint64_t)next - 1;
  }
}
/* lookup_and_get_indices, array_map.rs:276-372 */
static int amap_lookup(const ArrayMap* a, const int64_t* key, const uint8_t* valid, int64_t len, int64_t limit, MapOffset cur,
                       Vec64* pi, Vec64* bi, MapOffset* next_offset) {
  pi->n = 0; bi->n = 0;
  if (a->next_len == 0) {
    for (int64_t p = cur.idx; p < len; ++p) {
      if (bi->n == limit) { next_offset->idx = p; next_offset->has_next = 0; next_offset->next = 0; return 1; }
      if (valid && !valid[p]) continue;
      uint32_t b = amap_get(a, (uint64_t)key[p]);
      if (!b) continue;
      v_push(bi, (int64_t)b - 1);
      v_push(pi, p);
    }
    return 0;
  }
  int64_t remaining = limit;
  int64_t to_skip;
  if (!cur.has_next) to_skip = cur.idx;
  else if (cur.next == 0) to_skip = cur.idx + 1;
  else {
    int is_last = cur.idx == len - 1;
    if (traverse_chain32(a->next, cur.idx, (uint32_t)cur.next, &remaining, pi, bi, is_last, next_offset)) return 1;
    to_skip = cur.idx + 1;
  }
  for (int64_t p = to_skip; p < len; ++p) {
    if (remaining == 0) { next_offset->idx = p; next_offset->has_next = 0; next_offset->next = 0; return 1; }
    if (valid && !valid[p]) continue;
    int is_last = p == len - 1;
    uint32_t b = amap_get(a, (uint64_t)key[p]);
    if (!b) continue;
    if (traverse_chain32(a->next, p, b, &remaining, pi, bi, is_last, next_offset)) return 1;
  }
  return 0;
}

/* equal_rows_arr (joins/utils.rs:2191-2257): keep the candidate pairs whose key columns are equal; two NULLs are equal only under
 * NullEqualsNull.  Filters bi / pi in place, returns the number kept. */
static int64_t equal_rows_filter(int nkeys, const int64_t* const* bkeys, const uint8_t* const* bvalid, const int64_t* const* pk, const uint8_t* const* pv,
                                 int null_equals_null, Vec64* bi, Vec64* pi) {
  int64_t m = 0;
  for (int64_t k = 0; k < bi->n; ++k) {
    int eq = 1;
    for (int c = 0; c < nkeys && eq; ++c) {
      int ln = bvalid[c] && !bvalid[c][bi->p[k]], rn = pv[c] && !pv[c][pi->p[k]];
      if (ln || rn) eq = (ln && rn && null_equals_null);
      else eq = bkeys[c][bi->p[k]] == pk[c][pi->p[k]];
    }
    if (eq) { bi->p[m] = bi->p[k]; pi->p[m] = pi->p[k]; ++m; }
  }
  bi->n = pi->n = m;
  return m;
}
O_API int64_t oracle_equal_rows(int nkeys, const int64_t* const* lkeys, const uint8_t* const* lvalid, const int64_t* const* rkeys, const uint8_t* const* rvalid,
                                int null_equals_null, int64_t* left_idx, int64_t* right_idx, int64_t n) {
  if (nkeys == 0) return 0;   /* "empty keys returns empty" (utils.rs test_equal_rows_arr_empty_keys_returns_empty) */
  Vec64 bi = {left_idx, n, n}, pi = {right_idx, n, n};
  const uint8_t* lv[8]; const uint8_t* rv[8];
  for (int c = 0; c < nkeys; ++c) { lv[c] = lvalid ? lvalid[c] : NULL; rv[c] = rvalid ? rvalid[c] : NULL; }
  return equal_rows_filter(nkeys, lkeys, lv, rkeys, rv, null_equals_null, &bi, &pi);
}

/* ---- step-level entry points: one get_matched_indices_with_limit_offset call, so the reference's own unit tests of the
 * maps (joins/array_map.rs:428-600, joins/join_hash_map.rs:497-575) can be replayed tuple by tuple (tests/test_oracle_golden.py).
 * off / next_off = {idx, has_next, next} of MapOffset; returns 1 when a next offset exists (Some), 0 for None. ---- */
O_API int oracle_array_map_step(const int64_t* build, const uint8_t* bvalid, int64_t nb, uint64_t min_val, uint64_t max_val,
                                const int64_t* probe, const uint8_t* pvalid, int64_t np_, int64_t limit, const int64_t* off,
                                int64_t* pi_out, int64_t* bi_out, int64_t* n_out, int64_t* next_off) {
  ArrayMap a; memset(&a, 0, sizeof(a));
  amap_fill(&a, build, bvalid, nb, min_val, max_val);
  Vec64 pi = {0}, bi = {0};
  MapOffset cur = {off[0], (int)off[1], (uint64_t)off[2]}, nx = {0, 0, 0};
  int has = amap_lookup(&a, probe, pvalid, np_, limit, cur, &pi, &bi, &nx);
  for (int64_t k = 0; k < bi.n; ++k) { pi_out[k] = pi.p[k]; bi_out[k] = bi.p[k]; }
  *n_out = bi.n;
  next_off[0] = nx.idx; next_off[1] = nx.has_next; next_off[2] = (int64_t)nx.next;
  free(pi.p); free(bi.p); free(a.data); free(a.next);
  return has;
}
O_API int oracle_join_hash_map_step(const uint64_t* build_hashes, int64_t nb, const uint64_t* probe_hashes, const uint8_t* valid_keys, int64_t np_,
                                    int64_t limit, const int64_t* off, int64_t* pi_out, int64_t* bi_out, int64_t* n_out, int64_t* next_off) {
  JoinHashMap m; jhm_init(&m, (uint64_t)nb);
  for (int64_t i = 0; i < nb; ++i) jhm_insert(&m, (uint64_t)i, build_hashes[i]);   /* update_from_iter(iter.enumerate(), 0): forward order */
  Vec64 pi = {0}, bi = {0};
  MapOffset cur = {off[0], (int)off[1], (uint64_t)off[2]}, nx = {0, 0, 0};
  int has = jhm_lookup(&m, probe_hashes, valid_keys, np_, limit, cur, &pi, &bi, &nx);
  for (int64_t k = 0; k < bi.n; ++k) { pi_out[k] = pi.p[k]; bi_out[k] = bi.p[k]; }
  *n_out = bi.n;
  next_off[0] = nx.idx; next_off[1] = nx.has_next; next_off[2] = (int64_t)nx.next;
  free(pi.p); free(bi.p); jhm_free(&m);
  return has;
}

/* ------------------------------------------------------------------------------------------ */
/* join driver: collect_left_input + HashJoinStream state machine                              */
/* ------------------------------------------------------------------------------------------ */
enum { J_INNER = 0, J_LEFT, J_RIGHT, J_FULL, J_LEFT_SEMI, J_RIGHT_SEMI, J_LEFT_ANTI, J_RIGHT_ANTI, J_LEFT_MARK, J_RIGHT_MARK };

typedef struct {
  int64_t* build_idx; /* -1 = NULL */
  int64_t* probe_idx; /* -1 = NULL */
  int8_t* mark;       /* mark joins: 1/0, else NULL */
  int64_t n;
  int used_array_map;
} JoinResult;

static int row_has_null(int nkeys, const uint8_t* const* valid, int64_t row) {
  if (!valid) return 0;
  for (int c = 0; c < nkeys; ++c) if (valid[c] && !valid[c][row]) return 1;
  return 0;
}

/*
 * oracle_hash_join: keys are int64 columns (narrower integer types are widened by the caller —
 * value semantics are unchanged).  build_batch_rows / probe_batch_rows give the input batching
 * (the reference's alignment ranges and MapOffset resumption are per probe batch; the HashMap
 * path concatenates the build batches in REVERSED batch order, exec.rs:2684-2705).
 * build_order_out[i] = original build row held at concatenated position i.
 */
O_API int oracle_hash_join(int nkeys, const int64_t* const* bkeys_in, const uint8_t* const* bvalid_in, int64_t nb,
                           const int64_t* build_batch_rows, int n_build_batches,
                           const int64_t* const* pkeys, const uint8_t* const* pvalid, int64_t np_,
                           const int64_t* probe_batch_rows, int n_probe_batches,
                           int join_type, int null_equals_null, int64_t batch_size, int64_t phj_threshold, double phj_density,
                           int force_collisions, int key_is_integer, JoinResult* res, int64_t* build_order_out,
                           int (*pair_filter)(int64_t build_row, int64_t probe_row) /* JoinFilter on ORIGINAL row numbers, or NULL */,
                           int null_aware /* NOT IN semantics for LeftAnti / RightAnti on one key column (exec.rs:429-455, stream.rs:755-806) */) {
  memset(res, 0, sizeof(*res));
  Vec64 out_b = {0}, out_p = {0}, out_m = {0};
  /* ---- perfect-hash decision: try_create_array_map, exec.rs:111-191 ---- */
  int use_amap = 0;
  uint64_t minv = 0, maxv = 0;
  if (nkeys == 1 && key_is_integer && nb > 0) {
    int blocked = 0;
    if (null_equals_null && bvalid_in && bvalid_in[0]) {
      for (int64_t i = 0; i < nb; ++i) if (!bvalid_in[0][i]) { blocked = 1; break; }
    }
    if (!blocked) {
      int any = 0;
      int64_t mn = INT64_MAX, mx = INT64_MIN;
      for (int64_t i = 0; i < nb; ++i) {
        if (bvalid_in && bvalid_in[0] && !bvalid_in[0][i]) continue;
        any = 1;
        if (bkeys_in[0][i] < mn) mn = bkeys_in[0][i];
        if (bkeys_in[0][i] > mx) mx = bkeys_in[0][i];
      }
      if (any) {
        minv = (uint64_t)mn; maxv = (uint64_t)mx;
        uint64_t range = maxv - minv;
        int ok = (uint64_t)nb < 0xFFFFFFFFull && range != UINT64_MAX;
        if (ok) {
          double dense_ratio = (double)nb / ((double)range + 1.0);
          if (range >= (uint64_t)phj_threshold && dense_ratio <= phj_density) ok = 0;
        }
        use_amap = ok;
      }
    }
  }
  res->used_array_map = use_amap;
  /* ---- concatenation order of the build batches ---- */
  int64_t* order = (int64_t*)malloc((size_t)(nb ? nb : 1) * 8);
  {
    int64_t* starts = (int64_t*)malloc((size_t)(n_build_batches + 1) * 8);
    starts[0] = 0;
    for (int b = 0; b < n_build_batches; ++b) starts[b + 1] = starts[b] + build_batch_rows[b];
    int64_t pos = 0;
    if (use_amap) { for (int64_t i = 0; i < nb; ++i) order[pos++] = i; }           /* exec.rs:184 concat_batches(schema, batches) */
    else for (int b = n_build_batches - 1; b >= 0; --b) for (int64_t i = starts[b]; i < starts[b + 1]; ++i) order[pos++] = i; /* :2705 */
    free(starts);
  }
  if (build_order_out) memcpy(build_order_out, order, (size_t)nb * 8);
  /* materialise concatenated key columns */
  int64_t** bkeys = (int64_t**)malloc(sizeof(int64_t*) * (size_t)nkeys);
  uint8_t** bvalid = (uint8_t**)malloc(sizeof(uint8_t*) * (size_t)nkeys);
  for (int c = 0; c < nkeys; ++c) {
    bkeys[c] = (int64_t*)malloc((size_t)(nb ? nb : 1) * 8);
    bvalid[c] = (bvalid_in && bvalid_in[c]) ? (uint8_t*)malloc((size_t)(nb ? nb : 1)) : NULL;
    for (int64_t i = 0; i < nb; ++i) { bkeys[c][i] = bkeys_in[c][order[i]]; if (bvalid[c]) bvalid[c][i] = bvalid_in[c][order[i]]; }
  }
  /* ---- build ---- */
  JoinHashMap map; ArrayMap amap;
  memset(&map, 0, sizeof(map)); memset(&amap, 0, sizeof(amap));
  int64_t matchable_rows = 0;
  if (use_amap) {
    amap_fill(&amap, bkeys[0], bvalid[0], nb, minv, maxv);
    for (int64_t i = 0; i < nb; ++i) if (!(bvalid[0] && !bvalid[0][i])) matchable_rows++;
  } else {
    jhm_init(&map, (uint64_t)nb);
    uint64_t* h = (uint64_t*)malloc((size_t)(nb ? nb : 1) * 8);
    /* one update_hash per batch of the reversed list, rows of each batch in reverse (fifo) — the net
     * effect is a reverse pass over the concatenated rows: offset grows batch by batch (exec.rs:2684-2702) */
    int64_t offset = 0;
    for (int b = n_build_batches - 1; b >= 0; --b) {
      int64_t rows = build_batch_rows[b];
      create_hashes(nkeys, (const int64_t* const*)bkeys, (const uint8_t* const*)bvalid, offset, rows, SEED_JOIN, force_collisions, h);
      for (int64_t i = rows - 1; i >= 0; --i) {
        if (!null_equals_null && row_has_null(nkeys, (const uint8_t* const*)bvalid, offset + i)) continue; /* utils.rs:2146-2155 */
        jhm_insert(&map, (uint64_t)(offset + i), h[i]);
        matchable_rows++;
      }
      offset += rows;
    }
    free(h);
  }
  uint8_t* visited = (uint8_t*)calloc((size_t)(nb ? nb : 1), 1);
  const int need_final = join_type == J_LEFT || join_type == J_LEFT_ANTI || join_type == J_LEFT_SEMI || join_type == J_LEFT_MARK || join_type == J_FULL;
  /* ---- probe, batch by batch (stream.rs:687-1000) ---- */
  Vec64 pi = {0}, bi = {0};
  int64_t pstart = 0;
  int build_has_null = 0, probe_side_has_null = 0, probe_side_non_empty = 0;   /* JoinLeftData::build_side_has_null & the shared probe flags */
  if (bvalid[0]) for (int64_t i = 0; i < nb; ++i) if (!bvalid[0][i]) { build_has_null = 1; break; }
  for (int pb = 0; pb < n_probe_batches; ++pb) {
    const int64_t len = probe_batch_rows[pb];
    if (len == 0) continue;
    if (null_aware && join_type == J_RIGHT_ANTI && build_has_null) { pstart += len; continue; }   /* stream.rs:763-769 */
    if (null_aware && join_type == J_LEFT_ANTI) {                                                    /* stream.rs:770-805 */
      probe_side_non_empty = 1;
      if (pvalid && pvalid[0]) for (int64_t i = 0; i < len; ++i) if (!pvalid[0][pstart + i]) { probe_side_has_null = 1; break; }
      if (probe_side_has_null) { pstart += len; continue; }
    }
    /* is_empty = !has_matchable_build_rows(): build_batch_empty_build_side (utils.rs:1393-1430) */
    if (matchable_rows == 0) {
      if (join_type == J_RIGHT || join_type == J_FULL || join_type == J_RIGHT_ANTI || join_type == J_RIGHT_MARK) {
        for (int64_t i = 0; i < len; ++i) { v_push(&out_b, -1); v_push(&out_p, pstart + i); v_push(&out_m, 0); }
      }
      pstart += len;
      continue;
    }
    const int64_t* pk[8]; const uint8_t* pv[8];
    for (int c = 0; c < nkeys; ++c) { pk[c] = pkeys[c] + pstart; pv[c] = (pvalid && pvalid[c]) ? pvalid[c] + pstart : NULL; }
    uint64_t* h = (uint64_t*)malloc((size_t)len * 8);
    uint8_t* valid_keys = NULL;
    if (!use_amap) {
      create_hashes(nkeys, pk, pv, 0, len, SEED_JOIN, force_collisions, h);
      if (!null_equals_null) { /* matchable_join_keys, utils.rs:2172-2189 */
        int any_null = 0;
        valid_keys = (uint8_t*)malloc((size_t)len);
        for (int64_t i = 0; i < len; ++i) { valid_keys[i] = !row_has_null(nkeys, pv, i); any_null |= !valid_keys[i]; }
        if (!any_null) { free(valid_keys); valid_keys = NULL; }
      }
    }
    MapOffset off = {0, 0, 0};
    int64_t joined_probe_idx = -1; /* state.joined_probe_idx: None */
    for (;;) {
      MapOffset next_off = {0, 0, 0};
      int has_next;
      if (use_amap) has_next = amap_lookup(&amap, pk[0], pv[0], len, batch_size, off, &pi, &bi, &next_off);
      else has_next = jhm_lookup(&map, h, valid_keys, len, batch_size, off, &pi, &bi, &next_off);
      /* equal_rows_arr (utils.rs:2191-2257): drop hash-collision false positives */
      int64_t m = 0;
      if (!use_amap) m = equal_rows_filter(nkeys, (const int64_t* const*)bkeys, (const uint8_t* const*)bvalid, pk, pv, null_equals_null, &bi, &pi);
      else m = bi.n;
      if (pair_filter) { /* apply_join_filter_to_indices (utils.rs:1248-1320): after the key check, before visited/adjust */
        int64_t m2 = 0;
        for (int64_t k = 0; k < m; ++k) if (pair_filter(order[bi.p[k]], pstart + pi.p[k])) { bi.p[m2] = bi.p[k]; pi.p[m2] = pi.p[k]; ++m2; }
        m = bi.n = pi.n = m2;
      }
      if (need_final) for (int64_t k = 0; k < m; ++k) visited[bi.p[k]] = 1;
      int64_t last_joined = m ? pi.p[m - 1] : -1;
      int64_t range_start = joined_probe_idx < 0 ? 0 : joined_probe_idx + 1;
      int64_t range_end = !has_next ? len : (last_joined < 0 ? 0 : last_joined + 1);
      /* adjust_indices_by_join_type, utils.rs:1432-1490 */
      switch (join_type) {
        case J_INNER: case J_LEFT:
          for (int64_t k = 0; k < m; ++k) { v_push(&out_b, bi.p[k]); v_push(&out_p, pstart + pi.p[k]); v_push(&out_m, 0); }
          break;
        case J_RIGHT: case J_FULL: {
          /* append_right_indices with preserve_order_for_right=false: matched, then the unmatched of the range (get_anti_indices) */
          for (int64_t k = 0; k < m; ++k) { v_push(&out_b, bi.p[k]); v_push(&out_p, pstart + pi.p[k]); v_push(&out_m, 0); }
          int64_t nextu = range_start, k = 0;
          for (; k < m; ++k) {
            int64_t idx = pi.p[k];
            if (idx < range_start) continue;
            if (idx >= range_end) break;
            for (int64_t u = nextu; u < idx; ++u) { v_push(&out_b, -1); v_push(&out_p, pstart + u); v_push(&out_m, 0); }
            nextu = idx + 1;
          }
          for (int64_t u = nextu; u < range_end; ++u) { v_push(&out_b, -1); v_push(&out_p, pstart + u); v_push(&out_m, 0); }
          break;
        }
        case J_RIGHT_SEMI: { /* get_semi_indices */
          int64_t prev = -1;
          for (int64_t k = 0; k < m; ++k) {
            int64_t idx = pi.p[k];
            if (idx < range_start) continue;
            if (idx >= range_end) break;
            if (idx != prev) { v_push(&out_b, -1); v_push(&out_p, pstart + idx); v_push(&out_m, 0); }
            prev = idx;
          }
          break;
        }
        case J_RIGHT_ANTI: { /* get_anti_indices; a null-aware RightAnti does not emit NULL probe keys (stream.rs:937-956) */
          #define ANTI_EMIT(u) do { if (!(null_aware && pv[0] && !pv[0][(u)])) { v_push(&out_b, -1); v_push(&out_p, pstart + (u)); v_push(&out_m, 0); } } while (0)
          int64_t nextu = range_start;
          for (int64_t k = 0; k < m; ++k) {
            int64_t idx = pi.p[k];
            if (idx < range_start) continue;
            if (idx >= range_end) break;
            for (int64_t u = nextu; u < idx; ++u) ANTI_EMIT(u);
            nextu = idx + 1;
          }
          for (int64_t u = nextu; u < range_end; ++u) ANTI_EMIT(u);
          #undef ANTI_EMIT
          break;
        }
        case J_RIGHT_MARK: { /* get_mark_indices + left_indices = range */
          for (int64_t u = range_start; u < range_end; ++u) {
            int hit = 0;
            for (int64_t k = 0; k < m; ++k) if (pi.p[k] == u) { hit = 1; break; }
            v_push(&out_b, -1); v_push(&out_p, pstart + u); v_push(&out_m, hit);
          }
          break;
        }
        default: break; /* LeftSemi / LeftAnti / LeftMark: produced at the end */
      }
      if (!has_next) break;
      off = next_off;
      joined_probe_idx = last_joined >= 0 ? last_joined : joined_probe_idx; /* state.advance */
    }
    free(h);
    free(valid_keys);
    pstart += len;
  }
  /* ---- process_unmatched_build_batch (stream.rs:1002-1100) + get_final_indices_from_bit_map (utils.rs:1210-1245) ---- */
  if (need_final && !(null_aware && probe_side_has_null)) {   /* stream.rs:1016-1027: a NULL on the probe side empties a null-aware anti join */
    for (int64_t i = 0; i < nb; ++i) {
      /* stream.rs:1036-1072: NULL build keys are not output once the probe side was non-empty (NULL NOT IN (empty) is TRUE) */
      if (null_aware && join_type == J_LEFT_ANTI && probe_side_non_empty && bvalid[0] && !bvalid[0][i]) continue;
      if (join_type == J_LEFT_MARK) { v_push(&out_b, i); v_push(&out_p, -1); v_push(&out_m, visited[i]); }
      else if (join_type == J_LEFT_SEMI) { if (visited[i]) { v_push(&out_b, i); v_push(&out_p, -1); v_push(&out_m, 0); } }
      else if (!visited[i]) { v_push(&out_b, i); v_push(&out_p, -1); v_push(&out_m, 0); }
    }
  }
  /* build indices refer to the concatenated layout: map back to original build rows for the caller */
  for (int64_t k = 0; k < out_b.n; ++k) if (out_b.p[k] >= 0) out_b.p[k] = order[out_b.p[k]];
  res->n = out_b.n;
  res->build_idx = out_b.p; res->probe_idx = out_p.p;
  res->mark = (int8_t*)malloc((size_t)(out_m.n ? out_m.n : 1));
  for (int64_t k = 0; k < out_m.n; ++k) res->mark[k] = (int8_t)out_m.p[k];
  free(out_m.p);
  free(pi.p); free(bi.p); free(visited); free(order);
  for (int c = 0; c < nkeys; ++c) { free(bkeys[c]); free(bvalid[c]); }
  free(bkeys); free(bvalid);
  if (use_amap) { free(amap.data); free(amap.next); } else jhm_free(&map);
  return 0;
}

O_API void oracle_free_join_result(JoinResult* r) { free(r->build_idx); free(r->probe_idx); free(r->mark); memset(r, 0, sizeof(*r)); }

/* ------------------------------------------------------------------------------------------ */
/* aggregation: GroupValues::intern + GroupsAccumulator                                        */
/* ------------------------------------------------------------------------------------------ */
enum { A_SUM = 1, A_COUNT = 2, A_MIN = 3, A_MAX = 4, A_AVG = 5, A_COUNT_STAR = 6 };

typedef struct {
  int func;
  int is_float;        /* argument class: 0 = int64 (wrapping), 1 = float64, 2 = uint64 */
  const void* arg;     /* int64_t* or double*; state modes: the (first) state column */
  const uint8_t* arg_valid;
  const void* arg2;    /* AVG merge: sum column (double*) — arg is the count column (uint64) */
  const uint8_t* arg2_valid;
  const uint8_t* filter;       /* opt_filter values (1/0) or NULL */
  const uint8_t* filter_valid; /* filter validity or NULL */
} AggIn;

typedef struct {
  int64_t* ivals; double* fvals; /* accumulators (one of them by class) */
  uint64_t* counts;              /* COUNT / AVG */
  uint8_t* seen;                 /* NullState::seen_values; NULL while SeenValues::All */
  int64_t seen_all_num;          /* SeenValues::All { num_values } */
  int64_t cap;
} AggAcc;

typedef struct {
  int nkeys; int naggs;
  int64_t ngroups;
  int64_t** key_vals; uint8_t** key_valid; /* per key column, per group (first-seen order) */
  int64_t* out_i[8]; double* out_f[8]; uint64_t* out_c[8]; uint8_t* out_valid[8];
} GroupResult;

/* group table: hash -> group index, values compared on collision (primitive.rs:154-171; multi_group_by/mod.rs:455-512) */
typedef struct { uint64_t* hashes; int64_t* gidx; uint64_t mask; int64_t len; } GroupMap;
static void gm_init(GroupMap* g, uint64_t cap) { g->hashes = (uint64_t*)calloc(cap, 8); g->gidx = (int64_t*)malloc(cap * 8); memset(g->gidx, 0xFF, cap * 8); g->mask = cap - 1; g->len = 0; }

static inline int64_t canon_f64_bits(int64_t bits) { return ((uint64_t)bits << 1) == 0 ? 0 : bits; } /* primitive.rs:75-98 */

O_API int oracle_group_by(int nkeys, const int64_t* const* keys, const uint8_t* const* kvalid, const int* key_is_float, int64_t n,
                          int naggs, const AggIn* aggs, int merge_mode /* inputs are partial states */, int64_t batch_size,
                          int force_collisions, GroupResult* res) {
  memset(res, 0, sizeof(*res));
  res->nkeys = nkeys; res->naggs = naggs;
  GroupMap gm;
  gm_init(&gm, 1024);
  int64_t gcap = 1024, ng = 0;
  int64_t** gk = (int64_t**)malloc(sizeof(int64_t*) * (size_t)(nkeys ? nkeys : 1));
  uint8_t** gv = (uint8_t**)malloc(sizeof(uint8_t*) * (size_t)(nkeys ? nkeys : 1));
  for (int c = 0; c < nkeys; ++c) { gk[c] = (int64_t*)malloc((size_t)gcap * 8); gv[c] = (uint8_t*)malloc((size_t)gcap); }
  AggAcc acc[8];
  memset(acc, 0, sizeof(acc));
  for (int a = 0; a < naggs; ++a) {
    acc[a].cap = gcap;
    acc[a].ivals = (int64_t*)calloc((size_t)gcap, 8);
    acc[a].fvals = (double*)calloc((size_t)gcap, 8);
    acc[a].counts = (uint64_t*)calloc((size_t)gcap, 8);
  }
  int64_t* group_indices = (int64_t*)malloc((size_t)(batch_size > 0 ? batch_size : 1) * 8);
  uint64_t* h = (uint64_t*)malloc((size_t)(batch_size > 0 ? batch_size : 1) * 8);
  if (batch_size <= 0) batch_size = n > 0 ? n : 1, group_indices = (int64_t*)realloc(group_indices, (size_t)batch_size * 8), h = (uint64_t*)realloc(h, (size_t)batch_size * 8);
  for (int64_t start = 0; start < n; start += batch_size) {
    int64_t len = n - start < batch_size ? n - start : batch_size;
    /* ---- intern: hashing (aggregate seed) ---- */
    for (int64_t i = 0; i < len; ++i) h[i] = 0;
    if (!force_collisions) {
      for (int c = 0; c < nkeys; ++c) for (int64_t i = 0; i < len; ++i) {
        if (kvalid && kvalid[c] && !kvalid[c][start + i]) continue;
        int64_t kv = keys[c][start + i];
        if (key_is_float && key_is_float[c]) kv = canon_f64_bits(kv);
        h[i] = c == 0 ? o_hash((uint64_t)kv, SEED_AGG) : o_hash((uint64_t)kv, h[i]);
      }
    }
    for (int64_t i = 0; i < len; ++i) {
      const int64_t row = start + i;
      uint64_t s = o_mix64(h[i]) & gm.mask;
      int64_t g = -1;
      while (gm.gidx[s] >= 0) {
        if (gm.hashes[s] == h[i]) {
          int64_t cand = gm.gidx[s];
          int eq = 1;
          for (int c = 0; c < nkeys && eq; ++c) {
            int isnull = kvalid && kvalid[c] && !kvalid[c][row];
            if (isnull != !gv[c][cand]) eq = 0;
            else if (!isnull) {
              int64_t kv = keys[c][row];
              if (key_is_float && key_is_float[c]) kv = canon_f64_bits(kv);
              eq = gk[c][cand] == kv;
            }
          }
          if (eq) { g = cand; break; }
        }
        s = (s + 1) & gm.mask;
      }
      if (g < 0) { /* Vacant: new group id = values.len() (first-seen order, primitive.rs:166-171) */
        if (ng == gcap) {
          gcap *= 2;
          for (int c = 0; c < nkeys; ++c) { gk[c] = (int64_t*)realloc(gk[c], (size_t)gcap * 8); gv[c] = (uint8_t*)realloc(gv[c], (size_t)gcap); }
        }
        g = ng++;
        for (int c = 0; c < nkeys; ++c) {
          int isnull = kvalid && kvalid[c] && !kvalid[c][row];
          gv[c][g] = !isnull;
          int64_t kv = isnull ? 0 : keys[c][row];
          if (!isnull && key_is_float && key_is_float[c]) kv = canon_f64_bits(kv);
          gk[c][g] = kv;
        }
        gm.hashes[s] = h[i]; gm.gidx[s] = g; gm.len++;
        if ((uint64_t)gm.len * 2 > gm.mask) { /* grow + rehash */
          GroupMap ng2;
          gm_init(&ng2, (gm.mask + 1) * 4);
          for (uint64_t t = 0; t <= gm.mask; ++t) if (gm.gidx[t] >= 0) {
            uint64_t s2 = o_mix64(gm.hashes[t]) & ng2.mask;
            while (ng2.gidx[s2] >= 0) s2 = (s2 + 1) & ng2.mask;
            ng2.hashes[s2] = gm.hashes[t]; ng2.gidx[s2] = gm.gidx[t]; ng2.len++;
          }
          free(gm.hashes); free(gm.gidx);
          gm = ng2;
        }
      }
      group_indices[i] = g;
    }
    /* ---- update_batch / merge_batch per accumulator (common.rs:223-232) ---- */
    const int64_t total_num_groups = ng;
    for (int a = 0; a < naggs; ++a) {
      AggAcc* A = &acc[a];
      const AggIn* in = &aggs[a];
      if (A->cap < total_num_groups) {
        int64_t nc = A->cap;
        while (nc < total_num_groups) nc *= 2;
        A->ivals = (int64_t*)realloc(A->ivals, (size_t)nc * 8); memset(A->ivals + A->cap, 0, (size_t)(nc - A->cap) * 8);
        A->fvals = (double*)realloc(A->fvals, (size_t)nc * 8); memset(A->fvals + A->cap, 0, (size_t)(nc - A->cap) * 8);
        A->counts = (uint64_t*)realloc(A->counts, (size_t)nc * 8); memset(A->counts + A->cap, 0, (size_t)(nc - A->cap) * 8);
        if (A->seen) { A->seen = (uint8_t*)realloc(A->seen, (size_t)nc); memset(A->seen + A->cap, 0, (size_t)(nc - A->cap)); }
        A->cap = nc;
      }
      const int has_nulls = in->arg_valid != NULL; /* values.null_count() > 0 is decided per batch below */
      int batch_has_null = 0;
      if (has_nulls) for (int64_t i = 0; i < len; ++i) if (!in->arg_valid[start + i]) { batch_has_null = 1; break; }
      const int has_filter = in->filter != NULL && !merge_mode;
      const int tracks_seen = (in->func == A_SUM || in->func == A_MIN || in->func == A_MAX);
      /* NullState::accumulate (accumulate.rs:164-188): stay in SeenValues::All while no nulls / filter */
      if (tracks_seen) {
        if (!A->seen && !has_filter && !batch_has_null) A->seen_all_num = total_num_groups;
        else if (!A->seen) { /* get_builder: first num_values groups are seen (accumulate.rs:59-82) */
          A->seen = (uint8_t*)calloc((size_t)A->cap, 1);
          for (int64_t g2 = 0; g2 < A->seen_all_num; ++g2) A->seen[g2] = 1;
        }
      }
      for (int64_t i = 0; i < len; ++i) {
        const int64_t row = start + i, g = group_indices[i];
        if (has_filter) { /* only Some(true) rows pass (accumulate.rs:373-470) */
          if (in->filter_valid && !in->filter_valid[row]) continue;
          if (!in->filter[row]) continue;
        }
        if (in->func == A_COUNT_STAR && !merge_mode) { A->counts[g] += 1; continue; }
        const int isnull = in->arg_valid && !in->arg_valid[row];
        switch (in->func) {
          case A_COUNT: case A_COUNT_STAR:
            if (merge_mode) A->counts[g] += (uint64_t)((const int64_t*)in->arg)[row]; /* count.rs:675-698 */
            else if (!isnull) A->counts[g] += 1;                                       /* count.rs:648-672 */
            break;
          case A_SUM:
            if (isnull) break;
            if (in->is_float == 1) A->fvals[g] += ((const double*)in->arg)[row];
            else A->ivals[g] = (int64_t)((uint64_t)A->ivals[g] + (uint64_t)((const int64_t*)in->arg)[row]); /* add_wrapping, sum.rs:316 */
            if (A->seen) A->seen[g] = 1;
            break;
          case A_MIN: case A_MAX: {
            if (isnull) break;
            int first = A->seen ? !A->seen[g] : (A->counts[g] == 0);
            if (in->is_float == 1) {   /* IEEE totalOrder on the bits: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN */
              double v = ((const double*)in->arg)[row];
              const uint64_t kv = f64_total_order(v), kc = f64_total_order(A->fvals[g]);
              if (first || (in->func == A_MIN ? kv < kc : kv > kc)) A->fvals[g] = v;
            } else if (in->is_float == 2) {
              uint64_t v = ((const uint64_t*)in->arg)[row], cur = (uint64_t)A->ivals[g];
              if (first || (in->func == A_MIN ? v < cur : v > cur)) A->ivals[g] = (int64_t)v;
            } else {
              int64_t v = ((const int64_t*)in->arg)[row];
              if (first || (in->func == A_MIN ? v < A->ivals[g] : v > A->ivals[g])) A->ivals[g] = v;
            }
            A->counts[g] += 1; /* bookkeeping for `first` while SeenValues::All */
            if (A->seen) A->seen[g] = 1;
            break;
          }
          case A_AVG:
            if (merge_mode) { /* state = [count, sum] */
              A->counts[g] += ((const uint64_t*)in->arg)[row];
              if (!(in->arg2_valid && !in->arg2_valid[row])) A->fvals[g] += ((const double*)in->arg2)[row];
            } else if (!isnull) {
              A->fvals[g] += in->is_float == 1 ? ((const double*)in->arg)[row] : (double)((const int64_t*)in->arg)[row];
              A->counts[g] += 1;
            }
            break;
        }
      }
    }
  }
  /* ---- emit(EmitTo::All) ---- */
  res->ngroups = ng;
  res->key_vals = gk; res->key_valid = gv;
  for (int a = 0; a < naggs; ++a) {
    res->out_i[a] = acc[a].ivals; res->out_f[a] = acc[a].fvals; res->out_c[a] = acc[a].counts;
    uint8_t* ov = (uint8_t*)malloc((size_t)(ng ? ng : 1));
    for (int64_t g = 0; g < ng; ++g) {
      switch (aggs[a].func) {
        case A_SUM: case A_MIN: case A_MAX: ov[g] = acc[a].seen ? acc[a].seen[g] : 1; break; /* NullState::build, accumulate.rs:297-334 */
        case A_AVG: ov[g] = acc[a].counts[g] != 0; break;
        default: ov[g] = 1; /* COUNT is never NULL (count.rs:700-708) */
      }
    }
    res->out_valid[a] = ov;
    free(acc[a].seen);
  }
  free(group_indices); free(h); free(gm.hashes); free(gm.gidx);
  return 0;
}

O_API void oracle_free_group_result(GroupResult* r) {
  for (int c = 0; c < r->nkeys; ++c) { free(r->key_vals[c]); free(r->key_valid[c]); }
  free(r->key_vals); free(r->key_valid);
  for (int a = 0; a < r->naggs; ++a) { free(r->out_i[a]); free(r->out_f[a]); free(r->out_c[a]); free(r->out_valid[a]); }
  memset(r, 0, sizeof(*r));
}

/* ------------------------------------------------------------------------------------------ */
/* RepartitionExec hash partitioning (repartition/mod.rs:1097-1145): partition = hash % n       */
/* ------------------------------------------------------------------------------------------ */
O_API void oracle_hash_partition_ids(int nkeys, const int64_t* const* keys, const uint8_t* const* valid, int64_t n, int n_parts,
                                     uint64_t (*hashfn)(uint64_t, uint64_t), int32_t* out) {
  (void)hashfn;
  uint64_t* h = (uint64_t*)malloc((size_t)(n ? n : 1) * 8);
  create_hashes(nkeys, keys, valid, 0, n, SEED_REPART, 0, h);
  for (int64_t i = 0; i < n; ++i) out[i] = (int32_t)(h[i] % (uint64_t)n_parts);
  free(h);
}

/* ------------------------------------------------------------------------------------------ */
/* CPU baseline drivers (bench.py cpu_baseline / --impl reference): the same algorithms run the */
/* way the reference runs them — target_partitions threads, RepartitionExec(Hash) on both join  */
/* inputs (PartitionMode::Partitioned, exec.rs:1312-1325), Partial -> exchange -> FinalPartitioned */
/* aggregation (aggregates/mod.rs:28-48).  Inputs come from the shared generators (gen.h).      */
/* ------------------------------------------------------------------------------------------ */
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + ts.tv_nsec * 1e-9; }

typedef struct {
  int tid, T;
  /* generation + repartition */
  int64_t nb, np_;
  int kind_b, kind_p; uint64_t seed_b, seed_p; int64_t a_b, b_b, a_p, b_p;
  int64_t *bk, *bp, *pk, *pp;             /* generated inputs */
  int64_t *cnt_b, *cnt_p;                 /* [T][T] counts: input chunk x output partition */
  int64_t *off_b, *off_p;                 /* scatter offsets */
  int64_t *rbk, *rbp, *rpk, *rpp;         /* repartitioned columns */
  int64_t *part_b, *part_p;               /* [T+1] partition boundaries */
  int64_t* out_rows; uint64_t* checksum;  /* per thread */
  pthread_barrier_t* bar;
  int64_t batch_size; int use_amap_rule;
  double* t_start;                        /* set by thread 0 once the scratch buffers are faulted in */
} JoinBench;

static void* join_bench_thread(void* arg) {
  JoinBench* J = (JoinBench*)arg;
  const int t = J->tid, T = J->T;
  int64_t b0 = J->nb * t / T, b1 = J->nb * (t + 1) / T, p0 = J->np_ * t / T, p1 = J->np_ * (t + 1) / T;
  /* phase 0 (untimed): fault the repartition buffers in.  A long-running engine recycles its batch memory through the allocator;
   * timing the kernel's first-touch page faults of fresh multi-GB mallocs on every call would charge the CPU side for an
   * artefact of this harness (it was 2-3x of the whole join at 128 threads). */
  memset(J->rbk + b0, 0, (size_t)(b1 - b0) * 8); memset(J->rbp + b0, 0, (size_t)(b1 - b0) * 8);
  memset(J->rpk + p0, 0, (size_t)(p1 - p0) * 8); memset(J->rpp + p0, 0, (size_t)(p1 - p0) * 8);
  pthread_barrier_wait(J->bar);
  if (t == 0) *J->t_start = now_s();
  /* phase 1: this thread's input chunk: hash + count per output partition (BatchPartitioner, repartition/mod.rs:1111-1145) */
  for (int64_t i = b0; i < b1; ++i) J->cnt_b[t * T + (int)(o_hash((uint64_t)J->bk[i], SEED_REPART) % (uint64_t)T)]++;
  for (int64_t i = p0; i < p1; ++i) J->cnt_p[t * T + (int)(o_hash((uint64_t)J->pk[i], SEED_REPART) % (uint64_t)T)]++;
  pthread_barrier_wait(J->bar);
  if (t == 0) { /* offsets: partition-major, then input chunk */
    int64_t pos = 0;
    for (int p = 0; p < T; ++p) { J->part_b[p] = pos; for (int c = 0; c < T; ++c) { J->off_b[c * T + p] = pos; pos += J->cnt_b[c * T + p]; } }
    J->part_b[T] = pos; pos = 0;
    for (int p = 0; p < T; ++p) { J->part_p[p] = pos; for (int c = 0; c < T; ++c) { J->off_p[c * T + p] = pos; pos += J->cnt_p[c * T + p]; } }
    J->part_p[T] = pos;
  }
  pthread_barrier_wait(J->bar);
  /* phase 2: scatter (the `take` + channel send of pull_from_input, repartition/mod.rs:2138-2225) */
  { int64_t* o = &J->off_b[t * T];
    for (int64_t i = b0; i < b1; ++i) { int p = (int)(o_hash((uint64_t)J->bk[i], SEED_REPART) % (uint64_t)T); int64_t d = o[p]++; J->rbk[d] = J->bk[i]; J->rbp[d] = J->bp[i]; }
    o = &J->off_p[t * T];
    for (int64_t i = p0; i < p1; ++i) { int p = (int)(o_hash((uint64_t)J->pk[i], SEED_REPART) % (uint64_t)T); int64_t d = o[p]++; J->rpk[d] = J->pk[i]; J->rpp[d] = J->pp[i]; } }
  pthread_barrier_wait(J->bar);
  /* phase 3: partition t: HashJoinExec (build, probe in batch_size batches, take output columns) */
  const int64_t nb = J->part_b[t + 1] - J->part_b[t], np_ = J->part_p[t + 1] - J->part_p[t];
  const int64_t* bk = J->rbk + J->part_b[t]; const int64_t* bp = J->rbp + J->part_b[t];
  const int64_t* pk = J->rpk + J->part_p[t]; const int64_t* pp = J->rpp + J->part_p[t];
  uint64_t sum = 0; int64_t rows = 0;
  int use_amap = 0; uint64_t minv = 0, maxv = 0;
  if (J->use_amap_rule && nb > 0) {
    int64_t mn = INT64_MAX, mx = INT64_MIN;
    for (int64_t i = 0; i < nb; ++i) { if (bk[i] < mn) mn = bk[i]; if (bk[i] > mx) mx = bk[i]; }
    minv = (uint64_t)mn; maxv = (uint64_t)mx;
    uint64_t range = maxv - minv;
    use_amap = (uint64_t)nb < 0xFFFFFFFFull && range != UINT64_MAX && !(range >= 1024 && (double)nb / ((double)range + 1.0) <= 0.15);
  }
  const int64_t bs = J->batch_size;
  int64_t* ok = (int64_t*)malloc((size_t)bs * 8); int64_t* opb = (int64_t*)malloc((size_t)bs * 8); int64_t* opp = (int64_t*)malloc((size_t)bs * 8);
  Vec64 pi = {0}, bi = {0};
  if (use_amap) {
    ArrayMap am; amap_fill(&am, bk, NULL, nb, minv, maxv);
    for (int64_t s = 0; s < np_; s += bs) {
      int64_t len = np_ - s < bs ? np_ - s : bs;
      MapOffset off = {0, 0, 0}, nx;
      for (;;) {
        int more = amap_lookup(&am, pk + s, NULL, len, bs, off, &pi, &bi, &nx);
        for (int64_t k = 0; k < bi.n; ++k) { ok[k] = bk[bi.p[k]]; opb[k] = bp[bi.p[k]]; opp[k] = pp[s + pi.p[k]]; sum += (uint64_t)ok[k] + (uint64_t)opb[k] * 3 + (uint64_t)opp[k] * 5; }
        rows += bi.n;
        if (!more) break;
        off = nx;
      }
    }
    free(am.data); free(am.next);
  } else {
    JoinHashMap m; jhm_init(&m, (uint64_t)nb);
    uint64_t* h = (uint64_t*)malloc((size_t)(nb > bs ? nb : bs) * 8 + 8);
    for (int64_t i = 0; i < nb; ++i) h[i] = o_hash((uint64_t)bk[i], SEED_JOIN);
    for (int64_t i = nb - 1; i >= 0; --i) jhm_insert(&m, (uint64_t)i, h[i]);
    for (int64_t s = 0; s < np_; s += bs) {
      int64_t len = np_ - s < bs ? np_ - s : bs;
      for (int64_t i = 0; i < len; ++i) h[i] = o_hash((uint64_t)pk[s + i], SEED_JOIN);
      MapOffset off = {0, 0, 0}, nx;
      for (;;) {
        int more = jhm_lookup(&m, h, NULL, len, bs, off, &pi, &bi, &nx);
        int64_t mm = 0;
        for (int64_t k = 0; k < bi.n; ++k) if (bk[bi.p[k]] == pk[s + pi.p[k]]) { bi.p[mm] = bi.p[k]; pi.p[mm] = pi.p[k]; ++mm; } /* equal_rows_arr */
        for (int64_t k = 0; k < mm; ++k) { ok[k] = bk[bi.p[k]]; opb[k] = bp[bi.p[k]]; opp[k] = pp[s + pi.p[k]]; sum += (uint64_t)ok[k] + (uint64_t)opb[k] * 3 + (uint64_t)opp[k] * 5; }
        rows += mm;
        if (!more) break;
        off = nx;
      }
    }
    free(h); jhm_free(&m);
  }
  free(ok); free(opb); free(opp); free(pi.p); free(bi.p);
  J->out_rows[t] = rows; J->checksum[t] = sum;
  return NULL;
}

typedef struct { int64_t* dst; int kind; uint64_t seed; int64_t a, b, n; int tid, T; } GenJob;
static void* gen_thread(void* arg) {
  GenJob* g = (GenJob*)arg;
  int64_t i0 = g->n * g->tid / g->T, i1 = g->n * (g->tid + 1) / g->T;
  for (int64_t i = i0; i < i1; ++i) g->dst[i] = o_gen_value(g->kind, g->seed, g->a, g->b, (uint64_t)i);
  return NULL;
}
O_API void oracle_generate_i64(int kind, uint64_t seed, int64_t a, int64_t b, int64_t n, int threads, int64_t* dst) {
  if (threads < 1) threads = 1;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
  GenJob* jobs = (GenJob*)malloc(sizeof(GenJob) * (size_t)threads);
  for (int t = 0; t < threads; ++t) { jobs[t] = (GenJob){dst, kind, seed, a, b, n, t, threads}; pthread_create(&th[t], NULL, gen_thread, &jobs[t]); }
  for (int t = 0; t < threads; ++t) pthread_join(th[t], NULL);
  free(th); free(jobs);
}

/* returns seconds for the timed join (inputs pre-generated in RAM); out[0]=rows, out[1]=checksum */
O_API double oracle_bench_join(const int64_t* bk, const int64_t* bp, int64_t nb, const int64_t* pk, const int64_t* pp, int64_t np_,
                               int threads, int64_t batch_size, int use_amap_rule, uint64_t* out) {
  const int T = threads < 1 ? 1 : threads;
  JoinBench* J = (JoinBench*)calloc((size_t)T, sizeof(JoinBench));
  pthread_barrier_t bar; pthread_barrier_init(&bar, NULL, (unsigned)T);
  int64_t* cnt_b = (int64_t*)calloc((size_t)T * T, 8); int64_t* cnt_p = (int64_t*)calloc((size_t)T * T, 8);
  int64_t* off_b = (int64_t*)calloc((size_t)T * T, 8); int64_t* off_p = (int64_t*)calloc((size_t)T * T, 8);
  int64_t* part_b = (int64_t*)calloc((size_t)T + 1, 8); int64_t* part_p = (int64_t*)calloc((size_t)T + 1, 8);
  int64_t* rbk = (int64_t*)malloc((size_t)(nb ? nb : 1) * 8); int64_t* rbp = (int64_t*)malloc((size_t)(nb ? nb : 1) * 8);
  int64_t* rpk = (int64_t*)malloc((size_t)(np_ ? np_ : 1) * 8); int64_t* rpp = (int64_t*)malloc((size_t)(np_ ? np_ : 1) * 8);
  int64_t* out_rows = (int64_t*)calloc((size_t)T, 8); uint64_t* checksum = (uint64_t*)calloc((size_t)T, 8);
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)T);
  double t0 = now_s();
  for (int t = 0; t < T; ++t) {
    J[t].tid = t; J[t].T = T; J[t].nb = nb; J[t].np_ = np_; J[t].t_start = &t0;
    J[t].bk = (int64_t*)bk; J[t].bp = (int64_t*)bp; J[t].pk = (int64_t*)pk; J[t].pp = (int64_t*)pp;
    J[t].cnt_b = cnt_b; J[t].cnt_p = cnt_p; J[t].off_b = off_b; J[t].off_p = off_p; J[t].part_b = part_b; J[t].part_p = part_p;
    J[t].rbk = rbk; J[t].rbp = rbp; J[t].rpk = rpk; J[t].rpp = rpp; J[t].out_rows = out_rows; J[t].checksum = checksum;
    J[t].bar = &bar; J[t].batch_size = batch_size; J[t].use_amap_rule = use_amap_rule;
    pthread_create(&th[t], NULL, join_bench_thread, &J[t]);
  }
  for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
  double t1 = now_s();
  uint64_t rows = 0, sum = 0;
  for (int t = 0; t < T; ++t) { rows += (uint64_t)out_rows[t]; sum += checksum[t]; }
  out[0] = rows; out[1] = sum;
  free(J); free(cnt_b); free(cnt_p); free(off_b); free(off_p); free(part_b); free(part_p);
  free(rbk); free(rbp); free(rpk); free(rpp); free(out_rows); free(checksum); free(th);
  pthread_barrier_destroy(&bar);
  return t1 - t0;
}

/* ---- group-by baseline: Partial (per thread) -> hash exchange of states -> FinalPartitioned ---- */
typedef struct {
  int tid, T; const int64_t* g; const int64_t* v; int64_t n; int64_t batch_size;
  /* partial result of this thread */
  int64_t pn; int64_t* pk; int64_t* ps; int64_t* pc;
  struct AggBenchShared* sh;
} AggBench;
struct AggBenchShared { AggBench* all; pthread_barrier_t* bar; int64_t* out_groups; uint64_t* checksum; };

typedef struct { uint64_t* hashes; int64_t* gidx; uint64_t mask; int64_t len; int64_t* keys; int64_t* sums; int64_t* counts; int64_t cap; } SimpleAgg;
static void sa_init(SimpleAgg* a) { a->mask = (1u << 16) - 1; a->hashes = (uint64_t*)calloc(a->mask + 1, 8); a->gidx = (int64_t*)malloc((a->mask + 1) * 8); memset(a->gidx, 0xFF, (a->mask + 1) * 8);
  a->len = 0; a->cap = 1 << 15; a->keys = (int64_t*)malloc((size_t)a->cap * 8); a->sums = (int64_t*)calloc((size_t)a->cap, 8); a->counts = (int64_t*)calloc((size_t)a->cap, 8); }
static inline int64_t sa_intern(SimpleAgg* a, int64_t key) {
  uint64_t h = o_hash((uint64_t)key, SEED_AGG);
  uint64_t s = o_mix64(h) & a->mask;
  while (a->gidx[s] >= 0) { if (a->hashes[s] == h && a->keys[a->gidx[s]] == key) return a->gidx[s]; s = (s + 1) & a->mask; }
  if (a->len == a->cap) { a->cap *= 2; a->keys = (int64_t*)realloc(a->keys, (size_t)a->cap * 8);
    a->sums = (int64_t*)realloc(a->sums, (size_t)a->cap * 8); memset(a->sums + a->len, 0, (size_t)(a->cap - a->len) * 8);
    a->counts = (int64_t*)realloc(a->counts, (size_t)a->cap * 8); memset(a->counts + a->len, 0, (size_t)(a->cap - a->len) * 8); }
  int64_t g = a->len++;
  a->keys[g] = key; a->hashes[s] = h; a->gidx[s] = g;
  if ((uint64_t)a->len * 2 > a->mask) {
    uint64_t nm = (a->mask + 1) * 4 - 1;
    uint64_t* nh = (uint64_t*)calloc(nm + 1, 8); int64_t* ngx = (int64_t*)malloc((nm + 1) * 8); memset(ngx, 0xFF, (nm + 1) * 8);
    for (uint64_t t = 0; t <= a->mask; ++t) if (a->gidx[t] >= 0) { uint64_t s2 = o_mix64(a->hashes[t]) & nm; while (ngx[s2] >= 0) s2 = (s2 + 1) & nm; nh[s2] = a->hashes[t]; ngx[s2] = a->gidx[t]; }
    free(a->hashes); free(a->gidx); a->hashes = nh; a->gidx = ngx; a->mask = nm;
  }
  return g;
}
static void sa_free(SimpleAgg* a) { free(a->hashes); free(a->gidx); free(a->keys); free(a->sums); free(a->counts); }

static void* agg_bench_thread(void* arg) {
  AggBench* A = (AggBench*)arg;
  const int t = A->tid, T = A->T;
  int64_t i0 = A->n * t / T, i1 = A->n * (t + 1) / T;
  SimpleAgg part; sa_init(&part);
  const int64_t bs = A->batch_size;
  int64_t* gi = (int64_t*)malloc((size_t)bs * 8);
  for (int64_t s = i0; s < i1; s += bs) { /* PartialHashAggregateStream: intern then update_batch per accumulator */
    int64_t len = i1 - s < bs ? i1 - s : bs;
    for (int64_t i = 0; i < len; ++i) gi[i] = sa_intern(&part, A->g[s + i]);
    for (int64_t i = 0; i < len; ++i) part.sums[gi[i]] = (int64_t)((uint64_t)part.sums[gi[i]] + (uint64_t)A->v[s + i]);
    for (int64_t i = 0; i < len; ++i) part.counts[gi[i]] += 1;
  }
  free(gi);
  A->pn = part.len; A->pk = part.keys; A->ps = part.sums; A->pc = part.counts;
  pthread_barrier_wait(A->sh->bar);
  /* FinalPartitioned for partition t: merge every thread's states whose key hashes here (RepartitionExec(Hash(group keys))) */
  SimpleAgg fin; sa_init(&fin);
  for (int c = 0; c < T; ++c) {
    AggBench* P = &A->sh->all[c];
    for (int64_t i = 0; i < P->pn; ++i) {
      if ((int)(o_hash((uint64_t)P->pk[i], SEED_REPART) % (uint64_t)T) != t) continue;
      int64_t g = sa_intern(&fin, P->pk[i]);
      fin.sums[g] = (int64_t)((uint64_t)fin.sums[g] + (uint64_t)P->ps[i]);
      fin.counts[g] += P->pc[i];
    }
  }
  uint64_t sum = 0;
  for (int64_t g = 0; g < fin.len; ++g) sum += (uint64_t)fin.keys[g] * 3 + (uint64_t)fin.sums[g] * 5 + (uint64_t)fin.counts[g] * 7;
  A->sh->out_groups[t] = fin.len; A->sh->checksum[t] = sum;
  pthread_barrier_wait(A->sh->bar);
  sa_free(&fin);
  part.keys = A->pk; part.sums = A->ps; part.counts = A->pc; sa_free(&part);
  return NULL;
}
O_API double oracle_bench_groupby(const int64_t* g, const int64_t* v, int64_t n, int threads, int64_t batch_size, uint64_t* out) {
  const int T = threads < 1 ? 1 : threads;
  AggBench* A = (AggBench*)calloc((size_t)T, sizeof(AggBench));
  pthread_barrier_t bar; pthread_barrier_init(&bar, NULL, (unsigned)T);
  int64_t* og = (int64_t*)calloc((size_t)T, 8); uint64_t* cs = (uint64_t*)calloc((size_t)T, 8);
  struct AggBenchShared sh = {A, &bar, og, cs};
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)T);
  double t0 = now_s();
  for (int t = 0; t < T; ++t) { A[t].tid = t; A[t].T = T; A[t].g = g; A[t].v = v; A[t].n = n; A[t].batch_size = batch_size; A[t].sh = &sh; pthread_create(&th[t], NULL, agg_bench_thread, &A[t]); }
  for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
  double t1 = now_s();
  uint64_t groups = 0, sum = 0;
  for (int t = 0; t < T; ++t) { groups += (uint64_t)og[t]; sum += cs[t]; }
  out[0] = groups; out[1] = sum;
  free(A); free(og); free(cs); free(th); pthread_barrier_destroy(&bar);
  return t1 - t0;
}

/* ------------------------------------------------------------------------------------------ */
/* TPC-H Q3-shaped pipeline (BASELINE config C4), run the way the reference's physical plan runs */
/* it (sqllogictest/test_files/tpch/plans/q3.slt.part:60-76) with target_partitions = T threads: */
/*   FilterExec(c_mktsegment = 1)            -> RepartitionExec Hash(c_custkey)  \                */
/*   FilterExec(o_orderdate < cut)           -> RepartitionExec Hash(o_custkey)  -> HashJoinExec Partitioned RightSemi */
/*                                           -> RepartitionExec Hash(o_orderkey) \                */
/*   FilterExec(l_shipdate > cut) projection -> RepartitionExec Hash(l_orderkey) -> HashJoinExec Partitioned Inner     */
/*   -> AggregateExec SinglePartitioned gby [l_orderkey, o_orderdate, o_shippriority] SUM(l_extendedprice * (100 - l_discount)) */
/* Batches of batch_size rows; JoinHashMap + equal_rows for both joins; multi-column group table. */
/* Money is int64 fixed point as in the GPU arm (SURVEY.md §8d C4).                               */
/* ------------------------------------------------------------------------------------------ */
typedef struct { const void* src; void* dst; int width; } PCol;
typedef struct {
  int64_t n;            /* input rows */
  int64_t cap;          /* rows the repartitioned buffers can hold */
  int ncols;
  PCol col[4];          /* projected columns moved by the exchange */
  uint32_t** sel;       /* per thread: surviving row offsets within its chunk */
  uint16_t** pid;       /* per thread: output partition of each surviving row */
  int64_t* nsel;        /* per thread */
  int64_t* cnt;         /* [T][T] input chunk x output partition */
  int64_t* off;         /* [T][T] scatter offsets */
  int64_t* part;        /* [T+1] partition boundaries */
} Exchange;

static void exchange_offsets(Exchange* x, int T) { /* partition-major, then input chunk */
  int64_t pos = 0;
  for (int p = 0; p < T; ++p) { x->part[p] = pos; for (int c = 0; c < T; ++c) { x->off[c * T + p] = pos; pos += x->cnt[c * T + p]; } }
  x->part[T] = pos;
}
/* the `take` of BatchPartitioner (repartition/mod.rs:1111-1145): one pass per column over this thread's selected rows */
static void exchange_scatter(Exchange* x, int t, int T, int64_t i0) {
  int64_t* o = (int64_t*)malloc((size_t)T * 8);
  const uint32_t* sel = x->sel[t]; const uint16_t* pid = x->pid[t]; const int64_t ns = x->nsel[t];
  for (int c = 0; c < x->ncols; ++c) {
    memcpy(o, &x->off[t * T], (size_t)T * 8);
    if (x->col[c].width == 8) { const int64_t* s = (const int64_t*)x->col[c].src + i0; int64_t* d = (int64_t*)x->col[c].dst; for (int64_t j = 0; j < ns; ++j) d[o[pid[j]]++] = s[sel[j]]; }
    else { const int32_t* s = (const int32_t*)x->col[c].src + i0; int32_t* d = (int32_t*)x->col[c].dst; for (int64_t j = 0; j < ns; ++j) d[o[pid[j]]++] = s[sel[j]]; }
  }
  free(o);
}

typedef struct {
  uint64_t* hashes; int64_t* gidx; uint64_t mask; int64_t len, cap;
  int64_t* k0; int32_t* k1; int32_t* k2; int64_t* sum;
} Q3Groups; /* GroupValuesColumn restated for (int64, date32, int32) keys (multi_group_by/mod.rs:455-512) + one SUM accumulator */
static void q3g_init(Q3Groups* g) {
  g->mask = (1u << 12) - 1; g->hashes = (uint64_t*)calloc(g->mask + 1, 8); g->gidx = (int64_t*)malloc((g->mask + 1) * 8); memset(g->gidx, 0xFF, (g->mask + 1) * 8);
  g->len = 0; g->cap = 1 << 11;
  g->k0 = (int64_t*)malloc((size_t)g->cap * 8); g->k1 = (int32_t*)malloc((size_t)g->cap * 4); g->k2 = (int32_t*)malloc((size_t)g->cap * 4); g->sum = (int64_t*)calloc((size_t)g->cap, 8);
}
static inline int64_t q3g_intern(Q3Groups* g, uint64_t h, int64_t a, int32_t b, int32_t c) {
  uint64_t s = o_mix64(h) & g->mask;
  while (g->gidx[s] >= 0) { const int64_t i = g->gidx[s]; if (g->hashes[s] == h && g->k0[i] == a && g->k1[i] == b && g->k2[i] == c) return i; s = (s + 1) & g->mask; }
  if (g->len == g->cap) {
    g->cap *= 2;
    g->k0 = (int64_t*)realloc(g->k0, (size_t)g->cap * 8); g->k1 = (int32_t*)realloc(g->k1, (size_t)g->cap * 4); g->k2 = (int32_t*)realloc(g->k2, (size_t)g->cap * 4);
    g->sum = (int64_t*)realloc(g->sum, (size_t)g->cap * 8); memset(g->sum + g->len, 0, (size_t)(g->cap - g->len) * 8);
  }
  const int64_t i = g->len++;
  g->k0[i] = a; g->k1[i] = b; g->k2[i] = c; g->hashes[s] = h; g->gidx[s] = i;
  if ((uint64_t)g->len * 2 > g->mask) {
    const uint64_t nm = (g->mask + 1) * 4 - 1;
    uint64_t* nh = (uint64_t*)calloc(nm + 1, 8); int64_t* ng = (int64_t*)malloc((nm + 1) * 8); memset(ng, 0xFF, (nm + 1) * 8);
    for (uint64_t t = 0; t <= g->mask; ++t) if (g->gidx[t] >= 0) { uint64_t s2 = o_mix64(g->hashes[t]) & nm; while (ng[s2] >= 0) s2 = (s2 + 1) & nm; nh[s2] = g->hashes[t]; ng[s2] = g->gidx[t]; }
    free(g->hashes); free(g->gidx); g->hashes = nh; g->gidx = ng; g->mask = nm;
  }
  return i;
}
static void q3g_free(Q3Groups* g) { free(g->hashes); free(g->gidx); free(g->k0); free(g->k1); free(g->k2); free(g->sum); }

typedef struct Q3Shared {
  int T; int64_t bs; int32_t cut;
  int64_t nc, no, nl;
  const int64_t *c_key, *c_seg, *o_key, *o_cust, *l_key, *l_price, *l_disc; const int32_t *o_date, *o_prio, *l_ship;
  Exchange xc, xo, xl, xs;                  /* customer, orders, lineitem, semi-join output */
  /* semi-join output per partition, before its exchange */
  int64_t** so_key; int32_t** so_date; int32_t** so_prio;
  pthread_barrier_t* bar; double* t_start;
  uint64_t* out;                            /* [T][6]: groups, sum key, sum date, sum prio, sum revenue, joined rows */
  int64_t* stage;                           /* [T][3]: customers kept, orders kept by the semi join, lineitems kept */
} Q3Shared;
typedef struct { int tid; Q3Shared* sh; } Q3Thread;

static void exchange_alloc(Exchange* x, int T, int64_t n, int64_t cap, int ncols, const int* widths) {
  memset(x, 0, sizeof(*x));
  x->n = n; x->cap = cap; x->ncols = ncols;
  for (int c = 0; c < ncols; ++c) { x->col[c].width = widths[c]; x->col[c].dst = malloc((size_t)(cap ? cap : 1) * (size_t)widths[c]); }
  x->sel = (uint32_t**)calloc((size_t)T, sizeof(void*)); x->pid = (uint16_t**)calloc((size_t)T, sizeof(void*));
  x->nsel = (int64_t*)calloc((size_t)T, 8); x->cnt = (int64_t*)calloc((size_t)T * T, 8); x->off = (int64_t*)calloc((size_t)T * T, 8); x->part = (int64_t*)calloc((size_t)T + 1, 8);
}
static void exchange_free(Exchange* x, int T) {
  for (int c = 0; c < x->ncols; ++c) free(x->col[c].dst);
  for (int t = 0; t < T; ++t) { free(x->sel[t]); free(x->pid[t]); }
  free(x->sel); free(x->pid); free(x->nsel); free(x->cnt); free(x->off); free(x->part);
}
static void exchange_prefault(Exchange* x, int t, int T) { /* untimed: batch memory of a long-running engine is recycled, not freshly faulted */
  const int64_t a = x->cap * t / T, b = x->cap * (t + 1) / T;
  for (int c = 0; c < x->ncols; ++c) memset((char*)x->col[c].dst + a * x->col[c].width, 0, (size_t)(b - a) * (size_t)x->col[c].width);
  const int64_t i0 = x->n * t / T, i1 = x->n * (t + 1) / T;
  x->sel[t] = (uint32_t*)malloc((size_t)(i1 - i0 + 1) * 4); x->pid[t] = (uint16_t*)malloc((size_t)(i1 - i0 + 1) * 2);
  memset(x->sel[t], 0, (size_t)(i1 - i0 + 1) * 4); memset(x->pid[t], 0, (size_t)(i1 - i0 + 1) * 2);
}

static void* q3_bench_thread(void* arg) {
  Q3Thread* me = (Q3Thread*)arg; Q3Shared* S = me->sh;
  const int t = me->tid, T = S->T; const int64_t bs = S->bs;
  exchange_prefault(&S->xc, t, T); exchange_prefault(&S->xo, t, T); exchange_prefault(&S->xl, t, T);
  { /* the semi output of partition t cannot exceed the orders routed to it; sized after the orders exchange, prefaulted via xs.dst */
    const int64_t a = S->xs.cap * t / T, b = S->xs.cap * (t + 1) / T;
    for (int c = 0; c < S->xs.ncols; ++c) memset((char*)S->xs.col[c].dst + a * S->xs.col[c].width, 0, (size_t)(b - a) * (size_t)S->xs.col[c].width);
  }
  pthread_barrier_wait(S->bar);
  if (t == 0) *S->t_start = now_s();
  /* ---- FilterExec + BatchPartitioner::Hash, pass 1 (predicate, partition id, counts) for the three scans ---- */
  { const int64_t i0 = S->nc * t / T, i1 = S->nc * (t + 1) / T; int64_t ns = 0; Exchange* x = &S->xc;
    for (int64_t i = i0; i < i1; ++i) if (S->c_seg[i] == 1) { const int p = (int)(o_hash((uint64_t)S->c_key[i], SEED_REPART) % (uint64_t)T); x->sel[t][ns] = (uint32_t)(i - i0); x->pid[t][ns] = (uint16_t)p; x->cnt[t * T + p]++; ++ns; }
    x->nsel[t] = ns; S->stage[t * 3 + 0] = ns; }
  { const int64_t i0 = S->no * t / T, i1 = S->no * (t + 1) / T; int64_t ns = 0; Exchange* x = &S->xo;
    for (int64_t i = i0; i < i1; ++i) if (S->o_date[i] < S->cut) { const int p = (int)(o_hash((uint64_t)S->o_cust[i], SEED_REPART) % (uint64_t)T); x->sel[t][ns] = (uint32_t)(i - i0); x->pid[t][ns] = (uint16_t)p; x->cnt[t * T + p]++; ++ns; }
    x->nsel[t] = ns; }
  { const int64_t i0 = S->nl * t / T, i1 = S->nl * (t + 1) / T; int64_t ns = 0; Exchange* x = &S->xl;
    for (int64_t i = i0; i < i1; ++i) if (S->l_ship[i] > S->cut) { const int p = (int)(o_hash((uint64_t)S->l_key[i], SEED_REPART) % (uint64_t)T); x->sel[t][ns] = (uint32_t)(i - i0); x->pid[t][ns] = (uint16_t)p; x->cnt[t * T + p]++; ++ns; }
    x->nsel[t] = ns; S->stage[t * 3 + 2] = ns; }
  pthread_barrier_wait(S->bar);
  if (t == 0) exchange_offsets(&S->xc, T);
  if (t == 1 % T) exchange_offsets(&S->xo, T);
  if (t == 2 % T) exchange_offsets(&S->xl, T);
  pthread_barrier_wait(S->bar);
  exchange_scatter(&S->xc, t, T, S->nc * t / T); exchange_scatter(&S->xo, t, T, S->no * t / T); exchange_scatter(&S->xl, t, T, S->nl * t / T);
  pthread_barrier_wait(S->bar);
  /* ---- partition t: HashJoinExec RightSemi (c_custkey = o_custkey), projection [o_orderkey, o_orderdate, o_shippriority] ---- */
  Vec64 pi = {0}, bi = {0};
  uint64_t* h = NULL;
  {
    const int64_t nb = S->xc.part[t + 1] - S->xc.part[t], np_ = S->xo.part[t + 1] - S->xo.part[t];
    const int64_t* bk = (const int64_t*)S->xc.col[0].dst + S->xc.part[t];
    const int64_t* pkey = (const int64_t*)S->xo.col[0].dst + S->xo.part[t]; const int64_t* pcust = (const int64_t*)S->xo.col[1].dst + S->xo.part[t];
    const int32_t* pdate = (const int32_t*)S->xo.col[2].dst + S->xo.part[t]; const int32_t* pprio = (const int32_t*)S->xo.col[3].dst + S->xo.part[t];
    int64_t* sk = (int64_t*)malloc((size_t)(np_ + 1) * 8); int32_t* sd = (int32_t*)malloc((size_t)(np_ + 1) * 4); int32_t* sp = (int32_t*)malloc((size_t)(np_ + 1) * 4);
    S->so_key[t] = sk; S->so_date[t] = sd; S->so_prio[t] = sp;
    JoinHashMap m; jhm_init(&m, (uint64_t)nb);
    h = (uint64_t*)malloc((size_t)((nb > bs ? nb : bs) + 1) * 8);
    for (int64_t i = 0; i < nb; ++i) h[i] = o_hash((uint64_t)bk[i], SEED_JOIN);
    for (int64_t i = nb - 1; i >= 0; --i) jhm_insert(&m, (uint64_t)i, h[i]);
    int64_t ns = 0; Exchange* x = &S->xs;
    x->sel[t] = NULL; x->pid[t] = (uint16_t*)malloc((size_t)(np_ + 1) * 2);
    for (int64_t s = 0; s < np_; s += bs) {
      const int64_t len = np_ - s < bs ? np_ - s : bs;
      for (int64_t i = 0; i < len; ++i) h[i] = o_hash((uint64_t)pcust[s + i], SEED_JOIN);
      MapOffset off = {0, 0, 0}, nx;
      for (;;) {
        const int more = jhm_lookup(&m, h, NULL, len, bs, off, &pi, &bi, &nx);
        int64_t last = -1;
        for (int64_t k = 0; k < bi.n; ++k) {
          if (bk[bi.p[k]] != pcust[s + pi.p[k]]) continue;            /* equal_rows_arr */
          if (pi.p[k] == last) continue;                              /* get_semi_indices: each probe row once (utils.rs:1461-1466) */
          last = pi.p[k];
          const int64_t r = s + pi.p[k];
          sk[ns] = pkey[r]; sd[ns] = pdate[r]; sp[ns] = pprio[r];   /* take */
          const int p = (int)(o_hash((uint64_t)pkey[r], SEED_REPART) % (uint64_t)T); x->pid[t][ns] = (uint16_t)p; x->cnt[t * T + p]++; ++ns;
        }
        if (!more) break;
        off = nx;
      }
    }
    x->nsel[t] = ns; S->stage[t * 3 + 1] = ns;
    free(h); h = NULL; jhm_free(&m);
  }
  pthread_barrier_wait(S->bar);
  if (t == 0) exchange_offsets(&S->xs, T);
  pthread_barrier_wait(S->bar);
  { /* RepartitionExec Hash(o_orderkey) of the semi-join output */
    int64_t* o = (int64_t*)malloc((size_t)T * 8); const uint16_t* pid = S->xs.pid[t]; const int64_t ns = S->xs.nsel[t];
    memcpy(o, &S->xs.off[t * T], (size_t)T * 8); { int64_t* d = (int64_t*)S->xs.col[0].dst; for (int64_t j = 0; j < ns; ++j) d[o[pid[j]]++] = S->so_key[t][j]; }
    memcpy(o, &S->xs.off[t * T], (size_t)T * 8); { int32_t* d = (int32_t*)S->xs.col[1].dst; for (int64_t j = 0; j < ns; ++j) d[o[pid[j]]++] = S->so_date[t][j]; }
    memcpy(o, &S->xs.off[t * T], (size_t)T * 8); { int32_t* d = (int32_t*)S->xs.col[2].dst; for (int64_t j = 0; j < ns; ++j) d[o[pid[j]]++] = S->so_prio[t][j]; }
    free(o);
  }
  pthread_barrier_wait(S->bar);
  /* ---- partition t: HashJoinExec Inner (o_orderkey = l_orderkey) -> AggregateExec SinglePartitioned ---- */
  {
    const int64_t nb = S->xs.part[t + 1] - S->xs.part[t], np_ = S->xl.part[t + 1] - S->xl.part[t];
    const int64_t* bk = (const int64_t*)S->xs.col[0].dst + S->xs.part[t]; const int32_t* bd = (const int32_t*)S->xs.col[1].dst + S->xs.part[t]; const int32_t* bp = (const int32_t*)S->xs.col[2].dst + S->xs.part[t];
    const int64_t* pk = (const int64_t*)S->xl.col[0].dst + S->xl.part[t]; const int64_t* pprice = (const int64_t*)S->xl.col[1].dst + S->xl.part[t]; const int64_t* pdisc = (const int64_t*)S->xl.col[2].dst + S->xl.part[t];
    JoinHashMap m; jhm_init(&m, (uint64_t)nb);
    h = (uint64_t*)malloc((size_t)((nb > bs ? nb : bs) + 1) * 8);
    for (int64_t i = 0; i < nb; ++i) h[i] = o_hash((uint64_t)bk[i], SEED_JOIN);
    for (int64_t i = nb - 1; i >= 0; --i) jhm_insert(&m, (uint64_t)i, h[i]);
    /* join output batch: [o_orderdate, o_shippriority, l_orderkey, l_extendedprice, l_discount] */
    int32_t* od = (int32_t*)malloc((size_t)bs * 4); int32_t* op = (int32_t*)malloc((size_t)bs * 4);
    int64_t* ok = (int64_t*)malloc((size_t)bs * 8); int64_t* oe = (int64_t*)malloc((size_t)bs * 8); int64_t* odi = (int64_t*)malloc((size_t)bs * 8);
    int64_t* rev = (int64_t*)malloc((size_t)bs * 8); uint64_t* gh = (uint64_t*)malloc((size_t)bs * 8); int64_t* gi = (int64_t*)malloc((size_t)bs * 8);
    Q3Groups G; q3g_init(&G);
    uint64_t joined = 0;
    for (int64_t s = 0; s < np_; s += bs) {
      const int64_t len = np_ - s < bs ? np_ - s : bs;
      for (int64_t i = 0; i < len; ++i) h[i] = o_hash((uint64_t)pk[s + i], SEED_JOIN);
      MapOffset off = {0, 0, 0}, nx;
      for (;;) {
        const int more = jhm_lookup(&m, h, NULL, len, bs, off, &pi, &bi, &nx);
        int64_t mm = 0;
        for (int64_t k = 0; k < bi.n; ++k) if (bk[bi.p[k]] == pk[s + pi.p[k]]) { bi.p[mm] = bi.p[k]; pi.p[mm] = pi.p[k]; ++mm; }   /* equal_rows_arr */
        for (int64_t k = 0; k < mm; ++k) od[k] = bd[bi.p[k]];                /* build_batch_from_indices: take per column */
        for (int64_t k = 0; k < mm; ++k) op[k] = bp[bi.p[k]];
        for (int64_t k = 0; k < mm; ++k) ok[k] = pk[s + pi.p[k]];
        for (int64_t k = 0; k < mm; ++k) oe[k] = pprice[s + pi.p[k]];
        for (int64_t k = 0; k < mm; ++k) odi[k] = pdisc[s + pi.p[k]];
        /* AggregateExec: evaluate the argument, hash the three group columns, intern, update the SUM accumulator */
        for (int64_t k = 0; k < mm; ++k) rev[k] = (int64_t)((uint64_t)oe[k] * (uint64_t)(100 - odi[k]));
        for (int64_t k = 0; k < mm; ++k) gh[k] = o_hash((uint64_t)ok[k], SEED_AGG);
        for (int64_t k = 0; k < mm; ++k) gh[k] = o_hash((uint64_t)(int64_t)od[k], gh[k]);
        for (int64_t k = 0; k < mm; ++k) gh[k] = o_hash((uint64_t)(int64_t)op[k], gh[k]);
        for (int64_t k = 0; k < mm; ++k) gi[k] = q3g_intern(&G, gh[k], ok[k], od[k], op[k]);
        for (int64_t k = 0; k < mm; ++k) G.sum[gi[k]] = (int64_t)((uint64_t)G.sum[gi[k]] + (uint64_t)rev[k]);
        joined += (uint64_t)mm;
        if (!more) break;
        off = nx;
      }
    }
    uint64_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int64_t g = 0; g < G.len; ++g) { s0 += (uint64_t)G.k0[g]; s1 += (uint64_t)(int64_t)G.k1[g]; s2 += (uint64_t)(int64_t)G.k2[g]; s3 += (uint64_t)G.sum[g]; }
    uint64_t* o = &S->out[t * 6];
    o[0] = (uint64_t)G.len; o[1] = s0; o[2] = s1; o[3] = s2; o[4] = s3; o[5] = joined;
    q3g_free(&G); free(h); jhm_free(&m);
    free(od); free(op); free(ok); free(oe); free(odi); free(rev); free(gh); free(gi);
  }
  free(pi.p); free(bi.p);
  return NULL;
}

/* generate the synthetic TPC-H-shaped tables exactly as scripts/q3_device_pipeline.py gen_tables does on the device */
typedef struct { int tid, T; int64_t nc, no, nl; uint64_t seed; int64_t d0, d1;
                 int64_t *c_key, *c_seg, *o_key, *o_cust, *l_key, *l_price, *l_disc; int32_t *o_date, *o_prio, *l_ship; } Q3Gen;
static inline int64_t q3_sparse(int64_t e) { return (e / 8) * 32 + (e % 8) + 1; }
static void* q3_gen_thread(void* arg) {
  Q3Gen* g = (Q3Gen*)arg; const int t = g->tid, T = g->T; const uint64_t sd = g->seed;
  for (int64_t i = g->nc * t / T; i < g->nc * (t + 1) / T; ++i) { g->c_key[i] = 1 + i; g->c_seg[i] = (int64_t)(o_splitmix64_at(sd + 1, (uint64_t)i) % 5u); }
  const int64_t cb = g->nc * 2 / 3 > 1 ? g->nc * 2 / 3 : 1;
  for (int64_t i = g->no * t / T; i < g->no * (t + 1) / T; ++i) {
    g->o_key[i] = q3_sparse(i); g->o_cust[i] = 1 + (int64_t)(o_splitmix64_at(sd + 2, (uint64_t)i) % (uint64_t)cb);
    g->o_date[i] = (int32_t)(g->d0 + (int64_t)(o_splitmix64_at(sd + 3, (uint64_t)i) % (uint64_t)(g->d1 - g->d0 + 1))); g->o_prio[i] = 0;
  }
  for (int64_t i = g->nl * t / T; i < g->nl * (t + 1) / T; ++i) {
    g->l_key[i] = q3_sparse((int64_t)(o_splitmix64_at(sd + 4, (uint64_t)i) % (uint64_t)g->no));
    g->l_price[i] = 90000 + (int64_t)(o_splitmix64_at(sd + 5, (uint64_t)i) % 10410000u); g->l_disc[i] = (int64_t)(o_splitmix64_at(sd + 6, (uint64_t)i) % 11u);
    g->l_ship[i] = (int32_t)(g->d0 + 1 + (int64_t)(o_splitmix64_at(sd + 7, (uint64_t)i) % (uint64_t)(g->d1 - g->d0 + 121)));
  }
  return NULL;
}
O_API void oracle_q3_generate(int64_t nc, int64_t no, int64_t nl, uint64_t seed, int64_t d0, int64_t d1, int threads,
                              int64_t* c_key, int64_t* c_seg, int64_t* o_key, int64_t* o_cust, int32_t* o_date, int32_t* o_prio,
                              int64_t* l_key, int64_t* l_price, int64_t* l_disc, int32_t* l_ship) {
  const int T = threads < 1 ? 1 : threads;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)T); Q3Gen* jobs = (Q3Gen*)malloc(sizeof(Q3Gen) * (size_t)T);
  for (int t = 0; t < T; ++t) { jobs[t] = (Q3Gen){t, T, nc, no, nl, seed, d0, d1, c_key, c_seg, o_key, o_cust, l_key, l_price, l_disc, o_date, o_prio, l_ship}; pthread_create(&th[t], NULL, q3_gen_thread, &jobs[t]); }
  for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
  free(th); free(jobs);
}

/* returns seconds; out[0..5] = groups, sum l_orderkey, sum o_orderdate, sum o_shippriority, sum revenue (all mod 2^64), joined rows;
 * out[6..8] = customers kept, orders kept by the semi join, lineitems kept */
O_API double oracle_bench_q3(int64_t nc, int64_t no, int64_t nl, const int64_t* c_key, const int64_t* c_seg, const int64_t* o_key, const int64_t* o_cust,
                             const int32_t* o_date, const int32_t* o_prio, const int64_t* l_key, const int64_t* l_price, const int64_t* l_disc,
                             const int32_t* l_ship, int32_t cut, int threads, int64_t batch_size, uint64_t* out) {
  int T = threads < 1 ? 1 : threads;
  if (T > 65535) T = 65535;
  Q3Shared S; memset(&S, 0, sizeof(S));
  S.T = T; S.bs = batch_size; S.cut = cut; S.nc = nc; S.no = no; S.nl = nl;
  S.c_key = c_key; S.c_seg = c_seg; S.o_key = o_key; S.o_cust = o_cust; S.o_date = o_date; S.o_prio = o_prio; S.l_key = l_key; S.l_price = l_price; S.l_disc = l_disc; S.l_ship = l_ship;
  const int wc[1] = {8}, wo[4] = {8, 8, 4, 4}, wl[3] = {8, 8, 8}, ws[3] = {8, 4, 4};
  exchange_alloc(&S.xc, T, nc, nc, 1, wc); S.xc.col[0].src = c_key;
  exchange_alloc(&S.xo, T, no, no, 4, wo); S.xo.col[0].src = o_key; S.xo.col[1].src = o_cust; S.xo.col[2].src = o_date; S.xo.col[3].src = o_prio;
  exchange_alloc(&S.xl, T, nl, nl, 3, wl); S.xl.col[0].src = l_key; S.xl.col[1].src = l_price; S.xl.col[2].src = l_disc;
  exchange_alloc(&S.xs, T, 0, no, 3, ws);
  S.so_key = (int64_t**)calloc((size_t)T, sizeof(void*)); S.so_date = (int32_t**)calloc((size_t)T, sizeof(void*)); S.so_prio = (int32_t**)calloc((size_t)T, sizeof(void*));
  pthread_barrier_t bar; pthread_barrier_init(&bar, NULL, (unsigned)T);
  S.bar = &bar; double t0 = now_s(); S.t_start = &t0;
  S.out = (uint64_t*)calloc((size_t)T * 6, 8); S.stage = (int64_t*)calloc((size_t)T * 3, 8);
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)T); Q3Thread* args = (Q3Thread*)malloc(sizeof(Q3Thread) * (size_t)T);
  for (int t = 0; t < T; ++t) { args[t].tid = t; args[t].sh = &S; pthread_create(&th[t], NULL, q3_bench_thread, &args[t]); }
  for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
  const double t1 = now_s();
  for (int k = 0; k < 9; ++k) out[k] = 0;
  for (int t = 0; t < T; ++t) { for (int k = 0; k < 6; ++k) out[k] += S.out[t * 6 + k]; for (int k = 0; k < 3; ++k) out[6 + k] += (uint64_t)S.stage[t * 3 + k]; }
  for (int t = 0; t < T; ++t) { free(S.so_key[t]); free(S.so_date[t]); free(S.so_prio[t]); }
  free(S.so_key); free(S.so_date); free(S.so_prio);
  exchange_free(&S.xc, T); exchange_free(&S.xo, T); exchange_free(&S.xl, T); exchange_free(&S.xs, T);
  free(S.out); free(S.stage); free(th); free(args); pthread_barrier_destroy(&bar);
  return t1 - t0;
}

/* ------------------------------------------------------------------------------------------ */
/* Streaming verifier of the Q3-shaped query at ANY scale (the multi-GPU runs: SF100 x N does not fit   */
/* the partitioned port's buffers): no table is materialised — rows are regenerated from the counter-   */
/* based generators on the fly.  An independent algorithm (one shared open-addressing table built with  */
/* CAS, atomic adds), used only to fingerprint the expected result.                                     */
/* ------------------------------------------------------------------------------------------ */
typedef struct { int64_t key; int32_t date, prio; int64_t sum; int64_t rows; } Q3Slot;
typedef struct {
  int tid, T; int64_t NC, NO, NL; uint64_t seed; int64_t d0, d1; int32_t cut;
  uint64_t* cbits; Q3Slot* tab; uint64_t mask;
  pthread_barrier_t* bar; uint64_t* qualified;
} Q3Stream;
static void* q3_stream_thread(void* arg) {
  Q3Stream* g = (Q3Stream*)arg; const int t = g->tid, T = g->T; const uint64_t sd = g->seed;
  for (int64_t i = g->NC * t / T; i < g->NC * (t + 1) / T; ++i)          /* customers of the BUILDING segment: bit c_custkey */
    if (o_splitmix64_at(sd + 1, (uint64_t)i) % 5u == 1) __atomic_fetch_or(&g->cbits[(uint64_t)(1 + i) >> 6], 1ull << ((1 + i) & 63), __ATOMIC_RELAXED);
  pthread_barrier_wait(g->bar);
  const int64_t cb = g->NC * 2 / 3 > 1 ? g->NC * 2 / 3 : 1;
  uint64_t q = 0;
  for (int64_t i = g->NO * t / T; i < g->NO * (t + 1) / T; ++i) {      /* orders before the cut whose customer qualifies */
    const int32_t date = (int32_t)(g->d0 + (int64_t)(o_splitmix64_at(sd + 3, (uint64_t)i) % (uint64_t)(g->d1 - g->d0 + 1)));
    if (!(date < g->cut)) continue;
    const int64_t cust = 1 + (int64_t)(o_splitmix64_at(sd + 2, (uint64_t)i) % (uint64_t)cb);
    if (!((g->cbits[(uint64_t)cust >> 6] >> (cust & 63)) & 1)) continue;
    const int64_t key = q3_sparse(i);
    uint64_t s = o_mix64((uint64_t)key) & g->mask;
    for (;;) { int64_t expect = 0; if (__atomic_compare_exchange_n(&g->tab[s].key, &expect, key, 0, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) break; s = (s + 1) & g->mask; }
    g->tab[s].date = date; g->tab[s].prio = 0;
    ++q;
  }
  g->qualified[t] = q;
  pthread_barrier_wait(g->bar);
  for (int64_t i = g->NL * t / T; i < g->NL * (t + 1) / T; ++i) {      /* lineitems after the cut, joined and summed */
    const int32_t ship = (int32_t)(g->d0 + 1 + (int64_t)(o_splitmix64_at(sd + 7, (uint64_t)i) % (uint64_t)(g->d1 - g->d0 + 121)));
    if (!(ship > g->cut)) continue;
    const int64_t key = q3_sparse((int64_t)(o_splitmix64_at(sd + 4, (uint64_t)i) % (uint64_t)g->NO));
    uint64_t s = o_mix64((uint64_t)key) & g->mask;
    while (g->tab[s].key != 0 && g->tab[s].key != key) s = (s + 1) & g->mask;
    if (g->tab[s].key == 0) continue;
    const int64_t price = 90000 + (int64_t)(o_splitmix64_at(sd + 5, (uint64_t)i) % 10410000u), disc = (int64_t)(o_splitmix64_at(sd + 6, (uint64_t)i) % 11u);
    __atomic_fetch_add(&g->tab[s].sum, (int64_t)((uint64_t)price * (uint64_t)(100 - disc)), __ATOMIC_RELAXED);
    __atomic_fetch_add(&g->tab[s].rows, 1, __ATOMIC_RELAXED);
  }
  return NULL;
}
/* out[0..4] = groups, sum l_orderkey, sum o_orderdate, sum o_shippriority, sum revenue (mod 2^64); out[5] = joined rows; out[6] = qualified orders.
 * est_qualified: capacity hint for the table (rows); returns 0 on success, -1 if the table would overflow */
O_API int oracle_q3_stream_fingerprint(int64_t NC, int64_t NO, int64_t NL, uint64_t seed, int64_t d0, int64_t d1, int32_t cut, int threads, uint64_t* out) {
  const int T = threads < 1 ? 1 : threads;
  uint64_t cap = 1024; while (cap < (uint64_t)NO / 4) cap <<= 1;   /* ~10 % of the orders qualify: load factor <= 0.4 */
  Q3Slot* tab = (Q3Slot*)calloc(cap, sizeof(Q3Slot));
  uint64_t* cbits = (uint64_t*)calloc((size_t)(NC + 2) / 64 + 2, 8);
  uint64_t* qualified = (uint64_t*)calloc((size_t)T, 8);
  if (!tab || !cbits) { free(tab); free(cbits); free(qualified); return -1; }
  pthread_barrier_t bar; pthread_barrier_init(&bar, NULL, (unsigned)T);
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)T); Q3Stream* jobs = (Q3Stream*)malloc(sizeof(Q3Stream) * (size_t)T);
  for (int t = 0; t < T; ++t) { jobs[t] = (Q3Stream){t, T, NC, NO, NL, seed, d0, d1, cut, cbits, tab, cap - 1, &bar, qualified}; pthread_create(&th[t], NULL, q3_stream_thread, &jobs[t]); }
  for (int t = 0; t < T; ++t) pthread_join(th[t], NULL);
  for (int k = 0; k < 7; ++k) out[k] = 0;
  for (uint64_t s = 0; s < cap; ++s) if (tab[s].rows > 0) { out[0]++; out[1] += (uint64_t)tab[s].key; out[2] += (uint64_t)(int64_t)tab[s].date; out[3] += (uint64_t)(int64_t)tab[s].prio; out[4] += (uint64_t)tab[s].sum; out[5] += (uint64_t)tab[s].rows; }
  for (int t = 0; t < T; ++t) out[6] += qualified[t];
  free(tab); free(cbits); free(qualified); free(th); free(jobs); pthread_barrier_destroy(&bar);
  return 0;
}

O_API const char* oracle_version(void) { return "oracle 0.1 (restatement of apache/datafusion 55.0.0 hot path; parity unpinned for hash VALUES only)"; }
