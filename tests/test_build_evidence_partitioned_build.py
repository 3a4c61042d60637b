"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so) for the fused pipeline's partitioned build: the record scatter moves
its tiles with TMA bulk copies and reads them from shared memory as 16-byte loads, the insert kernel calls nothing and prefetches its
slots, and the key / value partition kernels that the radix join and the partitioned aggregate run compile to the instructions they had
before the record kernels shared their bodies (digest of the SASS text without addresses or encodings, CUDA 12.9, sm_90a)."""
from test_build_evidence import sass
from test_build_evidence_partitioned import digest

SCATTER_RECS = "_ZN5dfgpu28radix_scatter_records_kernelEPKyliPyPNS_8RadixRecE"
HIST_RECS = "_ZN5dfgpu25radix_hist_records_kernelEPKyliPy"
INSERT_PART = "_ZN5dfgpu25lookup_insert_part_kernelENS_9LookupDevEPK10ulonglong2liPjPy"
FILTER_RECS = "_ZN5dfgpu28lookup_filter_records_kernelENS_9LookupDevEPK10ulonglong2l"
HIST = "_ZN5dfgpu17radix_hist_kernelEPKyliPy"
SCATTER = "_ZN5dfgpu24radix_scatter_tma_kernelEPKyS1_liPyPNS_8RadixRecE"


def test_record_scatter_uses_one_bulk_copy_per_tile_and_wide_shared_loads():
    code = sass(SCATTER_RECS)
    assert len(code) > 500 and len(sass(HIST_RECS)) > 50
    assert any("UBLKCP.S.G" in l for l in code) and any("UBLKCP.G.S" in l for l in code) and any("SYNCS" in l for l in code)
    # one global -> shared copy per stage (the key / value kernel issues two)
    assert sum("UBLKCP.S.G" in l for l in code) * 2 == sum("UBLKCP.S.G" in l for l in sass(SCATTER))
    assert sum("LDS.128" in l for l in code) == 8          # a thread's 8 records of a full tile


def test_partitioned_insert_calls_nothing_and_prefetches_its_slots():
    code = sass(INSERT_PART)
    assert len(code) > 200 and not any("CALL" in l for l in code)
    assert any("ATOMG.E.CAS.128" in l for l in code) and sum("CCTL" in l for l in code) == 4
    filt = sass(FILTER_RECS)
    assert len(filt) > 20 and not any("CALL" in l for l in filt) and not any("CAS" in l for l in filt)


def test_key_value_partition_kernels_are_unchanged():
    assert (len(sass(HIST)), digest(sass(HIST))) == (152, "afc25ebd1e781742")
    assert (len(sass(SCATTER)), digest(sass(SCATTER))) == (1024, "a813de9d08f56d05")
