"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so) for the fused pipeline's partitioned aggregate: its pass-1
instantiation (VAR 192 = ring + records) makes no 16-byte record lookups and calls no interpreter, the probe-aggregate kernel keeps
the lane-paired REDs, and the ring-fed aggregate and pack instantiations that run everywhere else compile to the instructions they
had before the path was added (digest of the SASS text without addresses or encodings, CUDA 12.9, sm_90a)."""
import hashlib
import re

from test_build_evidence import sass

PART_AGG = "_ZN5dfgpu11pipe_kernelILi3ELb0ELi192EEEvPKNS_10PipeParamsElPy"   # pipe_kernel<SINK_AGG, false, 192>
PROBE_AGG = "_ZN5dfgpu21pipe_probe_agg_kernelEPK10ulonglong2lNS_9LookupDevEiiPjPy"
RING_AGG = "_ZN5dfgpu11pipe_kernelILi3ELb0ELi72EEEvPKNS_10PipeParamsElPy"    # pipe_kernel<SINK_AGG, false, 72>
RING_PACK = "_ZN5dfgpu11pipe_kernelILi6ELb0ELi64EEEvPKNS_10PipeParamsElPy"   # pipe_kernel<SINK_PACK, false, 64>


def digest(code):
    return hashlib.sha256("\n".join(re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", l).split(";")[0].strip() for l in code).encode()).hexdigest()[:16]


def test_partitioned_pass_one_streams_records_without_table_lookups():
    code, ring = sass(PART_AGG), sass(RING_AGG)
    assert len(code) > 2000
    assert any("UBLKCP" in l for l in code) and not any("CALL" in l for l in code)
    assert not any("LDG.E.128.STRONG.GPU" in l for l in code) and any("LDG.E.128.STRONG.GPU" in l for l in ring)   # phase B's record lookups
    # only the fallback for rows past the record buffer reads table keys (one 8-byte load site per probe step)
    assert sum("LDG.E.64.STRONG.GPU" in l for l in code) < sum("LDG.E.64.STRONG.GPU" in l for l in ring)


def test_probe_aggregate_kernel_pairs_its_reds():
    code = sass(PROBE_AGG)
    assert sum("REDG.E.ADD.64" in l for l in code) >= 8 and sum("SHFL.BFLY" in l for l in code) >= 12
    assert not any("CALL" in l for l in code)


def test_ring_instantiations_are_unchanged():
    assert (len(sass(RING_AGG)), digest(sass(RING_AGG))) == (6736, "91e74652d2dff979")
    assert (len(sass(RING_PACK)), digest(sass(RING_PACK))) == (3752, "8110d90dd7650fb4")
