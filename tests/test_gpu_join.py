"""Parity of the CUDA HashJoinExec path (through the C ABI) with the reference: golden KATs transcribed
from the reference's tests, the restatement oracle on seeded random inputs, and size-independent
properties at larger sizes.  Integer/index work: bit-exact."""
import itertools

import numpy as np
import pytest

from datafusion_b200 import capi as D
from oracle import oracle as O
from harness import assert_cols_equal, col_from_list, gpu_hash_join, load_golden
from test_oracle_golden import JT, KAT, MATRIX, MISC, expected_cols, kat_filter, kat_tables, out_mapping

pytestmark = pytest.mark.gpu
GJT = {"Inner": D.JOIN_INNER, "Left": D.JOIN_LEFT, "Right": D.JOIN_RIGHT, "Full": D.JOIN_FULL, "LeftSemi": D.JOIN_LEFT_SEMI,
       "RightSemi": D.JOIN_RIGHT_SEMI, "LeftAnti": D.JOIN_LEFT_ANTI, "RightAnti": D.JOIN_RIGHT_ANTI, "LeftMark": D.JOIN_LEFT_MARK,
       "RightMark": D.JOIN_RIGHT_MARK}
# join types whose emission order we reproduce exactly (probe order x ascending build row); Right/Full
# interleave unmatched probe rows per lookup chunk in the reference (utils.rs:1509-1570) -> compared sorted
ORDERED = {"Inner", "RightSemi", "RightAnti", "RightMark"}


@pytest.mark.parametrize("case", KAT, ids=[c["name"] for c in KAT])
def test_gpu_matches_reference_join_snapshots(gpu_ctx, case):
    left, right, on_b, on_p, side, idx, exp = kat_tables(case)
    for batch_size, phj in MATRIX:
        thr, dens = (819200, 0.0) if phj else (0, float("inf"))
        nl, nr = len(case["left"][0][1]), len(case["right"][0][1])
        tmap = {"date32": D.DATE32}
        bt = [tmap.get(case.get("types", {}).get(n), D.INT32) for n, _ in case["left"]]
        pt = [tmap.get(case.get("types", {}).get(n), D.INT32) for n, _ in case["right"]]
        got, h = gpu_hash_join(gpu_ctx, left, right, on_b, on_p, side, idx, GJT[case["join_type"]],
                               D.NULL_EQUALS_NULL if case["null_equality"] == "NullEqualsNull" else D.NULL_EQUALS_NOTHING,
                               batch_size=batch_size, phj=(thr, dens), probe_batch_rows=min(batch_size, nr), build_batch_rows=nl, return_handle=True,
                               filter=kat_filter(case, gpu=True), build_types=bt, probe_types=pt, null_aware=bool(case.get("null_aware")))
        ordered = (not case["sorted"]) and case["join_type"] in ORDERED
        assert_cols_equal(got, exp, ordered=ordered, what=f"{case['name']} bs={batch_size} phj={phj} ({case['ref']})")
        # assert_phj_used (exec.rs: array_map_created_count metric); "phj_expected": false = the reference asserts it is NOT used
        want = case.get("phj_expected", "config")
        if want is not None and len(on_b) == 1 and len(left[0][0]) > 0 and "types" not in case:
            assert h.metric("array_map_created_count") == (1 if (phj and want == "config") else 0), case["name"]
        h.close()


@pytest.mark.parametrize("jt", list(MISC["all_null_build_keys"]["expected_sorted"].keys()))
def test_gpu_all_null_build_keys(gpu_ctx, jt):
    m = MISC["all_null_build_keys"]
    left = [col_from_list(v) for _, v in m["left"]]; right = [col_from_list(v) for _, v in m["right"]]
    side, idx = out_mapping(jt, 2, 2)
    got = gpu_hash_join(gpu_ctx, left, right, [1], [1], side, idx, GJT[jt])
    assert_cols_equal(got, expected_cols(m["expected_sorted"][jt], side), ordered=False, what=f"{jt} ({m['ref']})")


def test_gpu_perfect_hash_edge_cases(gpu_ctx):
    m = MISC["perfect_hash_negative"]
    l = (np.array(m["left"][0][1], np.int64), None); r = (np.array(m["right"][0][1], np.int64), None)
    for phj in ((819200, 0.0), (0, float("inf"))):
        got = gpu_hash_join(gpu_ctx, [l], [r], [0], [0], [0, 1], [0, 0], phj=phj)
        exp = [(np.array([x[0] for x in m["expected_sorted"]], np.int64), None), (np.array([x[1] for x in m["expected_sorted"]], np.int64), None)]
        assert_cols_equal(got, exp, ordered=False)
    m = MISC["perfect_hash_full_range"]
    l = (np.array(m["left_i64"], np.int64), None); r = (np.array(m["right_i64"], np.int64), None)
    got, h = gpu_hash_join(gpu_ctx, [l], [r], [0], [0], [0, 1], [0, 0], phj=(819200, 0.0), return_handle=True)
    assert h.metric("array_map_created_count") == 0            # range == u64::MAX falls back to the hash table (exec.rs:165-169)
    assert got[0][0].tolist() == [m["expected_sorted"][0][0]]
    # the all-ones key (-1) lives in the dedicated slot of the open-addressing table
    l = (np.array([-1, 5, -1, 7], np.int64), None); r = (np.array([7, -1, 9], np.int64), None)
    got = gpu_hash_join(gpu_ctx, [l], [r], [0], [0], [0, 1], [0, 0], phj=(0, float("inf")))
    assert got[0][0].tolist() == [7, -1, -1] and got[1][0].tolist() == [7, -1, -1]


def random_tables(rng, nb, npr, key_space, dup, null_frac, key_dtype=np.int64, two_keys=False):
    base = rng.choice(key_space, size=max(nb // dup, 1), replace=False).astype(key_dtype)
    bk = np.resize(np.repeat(base, dup), nb); rng.shuffle(bk)
    pk = rng.integers(0, key_space, npr).astype(key_dtype)
    bv = None if null_frac == 0 else rng.random(nb) >= null_frac
    pv = None if null_frac == 0 else rng.random(npr) >= null_frac
    build = [(bk, bv), (rng.integers(-2**40, 2**40, nb).astype(np.int64), None if null_frac == 0 else rng.random(nb) >= null_frac)]
    probe = [(pk, pv), (rng.integers(0, 1000, npr).astype(np.int32), None)]
    if two_keys:
        build.append(((bk % 7).astype(np.int32), None)); probe.append(((pk % 7).astype(np.int32), None))
    return build, probe


ALL_TYPES = list(GJT.keys())


@pytest.mark.parametrize("jt", ALL_TYPES)
@pytest.mark.parametrize("dup,null_frac,phj", [(1, 0.0, True), (1, 0.0, False), (3, 0.1, False), (4, 0.05, True)])
def test_gpu_vs_oracle_random(gpu_ctx, jt, dup, null_frac, phj):
    rng = np.random.default_rng(hash((jt, dup, phj)) % 2**32)
    build, probe = random_tables(rng, 4000, 15000, 9000, dup, null_frac)
    side, idx = out_mapping(jt, 2, 2)
    kw = dict(phj_threshold=819200, phj_density=0.0) if phj else dict(phj_threshold=0, phj_density=float("inf"))
    exp = O.hash_join(build, probe, [0], [0], side, idx, join_type=JT[jt], probe_batch_rows=[5000, 5000, 5000], batch_size=8192, **kw)
    got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, GJT[jt], phj=(kw["phj_threshold"], kw["phj_density"]), probe_batch_rows=5000)
    assert_cols_equal(got, exp, ordered=jt in ORDERED, what=f"{jt} dup={dup} nulls={null_frac} phj={phj}")


@pytest.mark.parametrize("jt", ALL_TYPES)
def test_gpu_join_filter_vs_oracle(gpu_ctx, jt):
    # JoinFilter (residual predicate) on every join type: build.payload % 7 > probe.payload % 5 over duplicate-heavy keys
    rng = np.random.default_rng(hash(("filter", jt)) % 2**32)
    build, probe = random_tables(rng, 3000, 12000, 1500, 3, 0.05)
    build[1] = (build[1][0] % 7, None); probe[1] = ((probe[1][0] % 5).astype(np.int64), None)
    side, idx = out_mapping(jt, 2, 2)
    onodes = [(O.E_COLUMN, 0, None, 0, 0), (O.E_COLUMN, 1, None, 0, 0), (O.E_BINARY, O.OP_GT, None, 0, 0)]
    gnodes = [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_COLUMN, 1, 0, 0, 0, 0.0), (D.EXPR_BINARY, D.OP_GT, 0, 0, 0, 0.0)]
    exp = O.hash_join(build, probe, [0], [0], side, idx, join_type=JT[jt], filter=([0, 1], [1, 1], onodes), phj_threshold=0, phj_density=float("inf"))
    got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, GJT[jt], phj=(0, float("inf")), probe_batch_rows=5000, filter=([0, 1], [1, 1], gnodes))
    assert_cols_equal(got, exp, ordered=jt in ("Inner", "RightSemi", "RightAnti", "RightMark"), what=jt)


def test_gpu_inner_exact_order_with_chains_multibatch_and_device_path(gpu_ctx):
    rng = np.random.default_rng(11)
    build, probe = random_tables(rng, 6000, 20000, 2500, 5, 0.0)
    side, idx = out_mapping("Inner", 2, 2)
    for phj in (True, False):
        kw = dict(phj_threshold=819200, phj_density=0.0) if phj else dict(phj_threshold=0, phj_density=float("inf"))
        exp = O.hash_join(build, probe, [0], [0], side, idx, build_batch_rows=[2000, 2000, 2000], **kw)
        for device in (False, True):
            got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, phj=(kw["phj_threshold"], kw["phj_density"]), build_batch_rows=2000,
                                probe_batch_rows=7000, device=device)
            assert_cols_equal(got, exp, ordered=True, what=f"phj={phj} device={device}")


def test_gpu_null_equals_null(gpu_ctx):
    rng = np.random.default_rng(5)
    build, probe = random_tables(rng, 300, 900, 200, 2, 0.2)
    for jt in ("Inner", "Left", "RightAnti", "Full"):
        side, idx = out_mapping(jt, 2, 2)
        exp = O.hash_join(build, probe, [0], [0], side, idx, join_type=JT[jt], null_equals_null=True, phj_threshold=0, phj_density=float("inf"))
        got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, GJT[jt], D.NULL_EQUALS_NULL, phj=(0, float("inf")))
        assert_cols_equal(got, exp, ordered=jt in ORDERED, what=jt)


def test_gpu_two_column_and_narrow_keys(gpu_ctx):
    rng = np.random.default_rng(9)
    build, probe = random_tables(rng, 3000, 9000, 2000, 3, 0.05, key_dtype=np.int32, two_keys=True)
    side, idx = out_mapping("Inner", 3, 3)
    exp = O.hash_join(build, probe, [0, 2], [0, 2], side, idx)
    got = gpu_hash_join(gpu_ctx, build, probe, [0, 2], [0, 2], side, idx)
    assert_cols_equal(got, exp, ordered=True)


def test_gpu_force_hash_collisions(gpu_ctx):
    # mirror of the reference's force_hash_collisions CI job: results must not depend on hash quality
    rng = np.random.default_rng(3)
    build, probe = random_tables(rng, 500, 1500, 400, 2, 0.1)
    for jt in ("Inner", "Left", "RightSemi"):
        side, idx = out_mapping(jt, 2, 2)
        exp = O.hash_join(build, probe, [0], [0], side, idx, join_type=JT[jt], phj_threshold=0, phj_density=float("inf"))
        got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, GJT[jt], phj=(0, float("inf")), force_collisions=True)
        assert_cols_equal(got, exp, ordered=jt in ORDERED, what=jt)


def test_gpu_empty_and_ragged_inputs(gpu_ctx):
    e = (np.zeros(0, np.int64), None)
    k = (np.array([1, 2, 3], np.int64), None)
    for jt in ALL_TYPES:
        side, idx = out_mapping(jt, 1, 1)
        for b, p in ((e, k), (k, e), (e, e)):
            exp = O.hash_join([b], [p], [0], [0], side, idx, join_type=JT[jt])
            got = gpu_hash_join(gpu_ctx, [b], [p], [0], [0], side, idx, GJT[jt])
            assert_cols_equal(got, exp, ordered=False, what=f"{jt} nb={len(b[0])} np={len(p[0])}")
    # column count / type mismatches are errors, not crashes
    j = D.HashJoinHandle(gpu_ctx, [D.INT64], [D.INT64], [0], [0], [0, 1], [0, 0])
    with pytest.raises(D.DfgpuError):
        j.push_build_host([D.HostColumn(np.zeros(3, np.int32))])
    with pytest.raises(D.DfgpuError):
        j.push_probe_host([D.HostColumn(np.zeros(3, np.int64))])   # probe before finish_build
    j.close()


def test_gpu_large_join_properties(gpu_ctx):
    """BASELINE config C2 scaled (20M x 2M here; bench.py runs the full 100M x 10M): device-generated inputs,
    checked by size-independent properties: row count, probe order preserved, key equality, order-independent
    checksums against the oracle's multi-threaded run of the same generators."""
    ctx = gpu_ctx
    nb, npr = 2_000_000, 20_000_000
    bk = ctx.generate_i64(D.GEN_SPLITMIX, 42, 0, 0, 0, nb); pk = ctx.generate_i64(D.GEN_SPARSE_OF, 42, 43, nb, 0, npr)
    bp = ctx.generate_i64(D.GEN_SPLITMIX, 7, 0, 0, 0, nb); pp = ctx.generate_i64(D.GEN_SEQ, 0, 0, 0, 0, npr)
    col = lambda buf, n: D.DeviceColumn(ctx, D.INT64, n, buf)
    j = D.HashJoinHandle(ctx, [D.INT64, D.INT64], [D.INT64, D.INT64], [0], [0], [0, 0, 1, 1], [0, 1, 0, 1])
    j.push_build_device([col(bk, nb), col(bp, nb)]); j.finish_build()
    j.push_probe_device([col(pk, npr), col(pp, npr)]); j.finish_probe()
    outs = j.drain(host=True)
    k_b = np.concatenate([o.column_numpy(0)[0] for o in outs]); v_b = np.concatenate([o.column_numpy(1)[0] for o in outs])
    k_p = np.concatenate([o.column_numpy(2)[0] for o in outs]); v_p = np.concatenate([o.column_numpy(3)[0] for o in outs])
    assert len(k_b) == npr                                   # 100 % hit rate, unique build keys
    assert np.array_equal(k_b, k_p)                          # join condition
    assert np.array_equal(v_p, np.arange(npr, dtype=np.int64))  # probe order preserved (exec.rs:1338-1351)
    hbk = O.generate_i64(2, 42, 0, 0, nb, 8); hbp = O.generate_i64(2, 7, 0, 0, nb, 8); hpk = O.generate_i64(4, 42, 43, nb, npr, 8)
    assert np.array_equal(hpk, k_p)                          # device generator == oracle generator
    secs, rows, chk = O.bench_join(hbk, hbp, hpk, np.arange(npr, dtype=np.int64), threads=8)
    mine = int((k_b.view(np.uint64).sum(dtype=np.uint64) + v_b.view(np.uint64).sum(dtype=np.uint64) * np.uint64(3) + v_p.view(np.uint64).sum(dtype=np.uint64) * np.uint64(5)))
    assert rows == npr and (mine % 2**64) == chk
    j.close()


@pytest.mark.parametrize("seed", [79, 82, 85])
@pytest.mark.parametrize("with_payload", [True, False])
def test_gpu_ordered_inline_probe_keeps_reference_order(gpu_ctx, seed, with_payload):
    """The single-pass ordered probe of the inline table (join_probe_inline_kernel, hash_join.cu) must give the reference's rows in
    the reference's order: unique build keys, ~60 % hit rate, ~3 % NULL probe keys, a ragged last tile and several probe batches,
    from device and from host input."""
    rng = np.random.default_rng(seed)
    nb, npr = 30_000, 201_777
    bk = rng.permutation(100_000)[:nb].astype(np.int64) * 1_000_003 - 5
    build = [(bk, None), (rng.integers(-2**62, 2**62, nb).astype(np.int64), None)]
    pk = rng.integers(0, 100_000, npr).astype(np.int64) * 1_000_003 - 5
    probe = [(pk, rng.random(npr) > 0.03), (np.arange(npr, dtype=np.int64), None)]
    side, idx = ([0, 0, 1, 1], [0, 1, 0, 1]) if with_payload else ([0, 1, 1], [0, 0, 1])
    exp = O.hash_join(build, probe, [0], [0], side, idx, phj_threshold=0, phj_density=float("inf"))
    for device in (True, False):
        got, h = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, phj=(0, float("inf")), probe_batch_rows=70_001, device=device, return_handle=True)
        assert h.metric("array_map_created_count") == 0
        assert h.metric("radix_partitioned_probes") == 0
        h.close()
        assert_cols_equal(got, exp, ordered=True, what=f"ordered probe seed={seed} payload={with_payload} device={device}")


def test_gpu_null_aware_validation(gpu_ctx):
    """HashJoinExecBuilder validation (exec.rs:429-455; tests exec.rs:7586-7745): null_aware needs LeftAnti / RightAnti, a single
    key column, and — for RightAnti — no join filter."""
    with pytest.raises(D.DfgpuError, match="null_aware can only be true for LeftAnti joins and RightAnti joins"):
        D.HashJoinHandle(gpu_ctx, [D.INT32, D.INT32], [D.INT32, D.INT32], [0], [0], [0, 1], [0, 0], D.JOIN_INNER, null_aware=True)
    with pytest.raises(D.DfgpuError, match="null_aware anti join only supports single column join key"):
        D.HashJoinHandle(gpu_ctx, [D.INT32, D.INT32], [D.INT32, D.INT32], [0, 1], [0, 1], [0, 0], [0, 1], D.JOIN_LEFT_ANTI, null_aware=True)
    nodes = [(D.EXPR_COLUMN, 0, 0, 0, 0, 0.0), (D.EXPR_LITERAL, 0, D.INT32, 0, 8, 0.0), (D.EXPR_BINARY, D.OP_NEQ, 0, 0, 0, 0.0)]
    j = D.HashJoinHandle(gpu_ctx, [D.INT32, D.INT32], [D.INT32, D.INT32], [0], [0], [1, 1], [0, 1], D.JOIN_RIGHT_ANTI, null_aware=True)
    with pytest.raises(D.DfgpuError, match="null_aware RightAnti join does not support a join filter"):
        j.set_filter([0], [1], nodes)
    j.close()
    j = D.HashJoinHandle(gpu_ctx, [D.INT32, D.INT32], [D.INT32, D.INT32], [0], [0], [0, 0], [0, 1], D.JOIN_LEFT_ANTI, null_aware=True)
    j.set_filter([1], [1], nodes)      # allowed for LeftAnti (test_null_aware_filter_rejected_only_for_right_anti)
    j.close()


def test_gpu_null_aware_anti_large_random(gpu_ctx):
    """null-aware anti joins against the oracle on larger random inputs (NULLs on the preserved side only, several probe batches)"""
    rng = np.random.default_rng(11)
    bk = rng.integers(0, 5000, 20000).astype(np.int64); pk = rng.integers(0, 8000, 70000).astype(np.int64)
    for jt, gjt, bnull, pnull in ((O.J_LEFT_ANTI, D.JOIN_LEFT_ANTI, True, False), (O.J_RIGHT_ANTI, D.JOIN_RIGHT_ANTI, False, True)):
        build = [(bk, (rng.random(len(bk)) > 0.05) if bnull else None), (np.arange(len(bk), dtype=np.int64), None)]
        probe = [(pk, (rng.random(len(pk)) > 0.05) if pnull else None), (np.arange(len(pk), dtype=np.int64), None)]
        side, idx = ([0, 0], [0, 1]) if jt == O.J_LEFT_ANTI else ([1, 1], [0, 1])
        exp = O.hash_join(build, probe, [0], [0], side, idx, join_type=jt, null_aware=True, probe_batch_rows=[30000, 40000])
        got = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, gjt, probe_batch_rows=30000 if jt == O.J_LEFT_ANTI else 40000, null_aware=True)
        assert len(exp[0][0]) > 0
        assert_cols_equal(got, exp, ordered=False, what=f"null-aware {jt}")


@pytest.mark.parametrize("parts", [2, 8, 64])
@pytest.mark.parametrize("with_payload", [True, False])
def test_gpu_radix_partitioned_probe_gives_the_same_rows(gpu_ctx, monkeypatch, parts, with_payload):
    """The radix-partitioned probe (radix_probe.cuh: TMA-staged partition pass + per-partition probe; taken when the caller does not need
    probe order) must return the reference's rows as a multiset: unique build keys, ~60 % hit rate, odd row counts, a ragged last 2048-row
    tile, several probe batches.  DFGPU_JOIN_RADIX_PARTS forces the path on inputs far smaller than the L2."""
    rng = np.random.default_rng(91 + parts)
    nb, npr = 30_000, 201_777
    bk = rng.permutation(100_000)[:nb].astype(np.int64) * 1_000_003 - 5
    build = [(bk, None), (rng.integers(-2**62, 2**62, nb).astype(np.int64), None)]
    pk = rng.integers(0, 100_000, npr).astype(np.int64) * 1_000_003 - 5
    probe = [(pk, None), (rng.integers(-2**62, 2**62, npr).astype(np.int64), None)]
    side, idx = ([0, 0, 1, 1], [0, 1, 0, 1]) if with_payload else ([0, 1, 1], [0, 0, 1])
    exp = O.hash_join(build, probe, [0], [0], side, idx, phj_threshold=0, phj_density=float("inf"))
    monkeypatch.setenv("DFGPU_JOIN_RADIX_PARTS", str(parts))
    got, h = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, phj=(0, float("inf")), probe_batch_rows=70_001, device=True, return_handle=True, ordered_output=False)
    assert h.metric("radix_partitioned_probes") == 3 and h.metric("array_map_created_count") == 0
    h.close()
    assert_cols_equal(got, exp, ordered=False, what=f"radix probe P={parts} payload={with_payload}")
    # with ordered_output (the default) the same handle configuration keeps the exact reference order and never takes the radix path
    got, h = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, phj=(0, float("inf")), probe_batch_rows=70_001, device=True, return_handle=True)
    assert h.metric("radix_partitioned_probes") == 0
    h.close()
    assert_cols_equal(got, exp, ordered=True, what="ordered path untouched")


@pytest.mark.parametrize("hit_pct,with_payload,device", [(10, True, True), (100, True, False), (10, False, True), (0, True, True)])
def test_gpu_membership_filter_keeps_rows_and_order(gpu_ctx, hit_pct, with_payload, device):
    """dfgpu_hashjoin_options.membership_filter: a Bloom filter over the build keys tested before the table (the stand-alone join's dynamic
    filter pushdown, shared_bounds.rs) must change nothing but the number of table accesses — same rows, same (reference) order, with NULL
    probe keys, misses and several probe batches"""
    rng = np.random.default_rng(300 + hit_pct)
    nb, npr = 40_000, 150_123
    universe = rng.permutation(1_000_000)[:nb * 10].astype(np.int64) * 1_000_003 - 7
    bk = universe[:nb]
    build = [(bk, None), (rng.integers(-2**62, 2**62, nb).astype(np.int64), None)]
    hit = rng.random(npr) < hit_pct / 100.0
    pk = np.where(hit, bk[rng.integers(0, nb, npr)], universe[nb + rng.integers(0, nb * 9, npr)])
    probe = [(pk, rng.random(npr) > 0.03), (np.arange(npr, dtype=np.int64), None)]
    side, idx = ([0, 0, 1, 1], [0, 1, 0, 1]) if with_payload else ([0, 1, 1], [0, 0, 1])
    exp = O.hash_join(build, probe, [0], [0], side, idx, phj_threshold=0, phj_density=float("inf"))
    got, h = gpu_hash_join(gpu_ctx, build, probe, [0], [0], side, idx, phj=(0, float("inf")), probe_batch_rows=60_001, device=device, return_handle=True,
                           membership_filter=True)
    assert h.metric("membership_filter_bytes") >= nb * 2 and h.metric("array_map_created_count") == 0
    h.close()
    assert_cols_equal(got, exp, ordered=True, what=f"membership filter hit={hit_pct}% payload={with_payload}")
    if hit_pct in (10, 100):
        assert len(exp[0][0]) > npr * hit_pct // 100 * 0.9
