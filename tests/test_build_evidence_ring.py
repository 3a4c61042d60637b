"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so): the ring-fed instantiations of the fused pipeline kernel
(aggregate sink: VAR 72 = ring + lane-paired REDs; pack sink: VAR 64) stream their columns with TMA bulk copies completed on
mbarriers and keep the lane-paired REDs."""
from test_build_evidence import sass

RING_AGG = "_ZN5dfgpu11pipe_kernelILi3ELb0ELi72EEEvPKNS_10PipeParamsElPy"     # pipe_kernel<SINK_AGG, false, 72>
RING_PACK = "_ZN5dfgpu11pipe_kernelILi6ELb0ELi64EEEvPKNS_10PipeParamsElPy"    # pipe_kernel<SINK_PACK, false, 64>


def test_ring_pipeline_kernels_use_tma_bulk_copies():
    for fn in (RING_AGG, RING_PACK):
        code = sass(fn)
        assert len(code) > 2000, fn
        assert any("UBLKCP" in l for l in code) and any("SYNCS" in l for l in code), fn
        assert not any("CALL" in l for l in code), fn                       # no out-of-line interpreter in the ring kernels


def test_ring_aggregate_kernel_keeps_the_paired_reds_and_drops_the_argument_prefetch():
    code = sass(RING_AGG)
    assert sum("REDG.E.ADD.64" in l for l in code) >= 4
    assert not any("CCTL.E.PF2" in l for l in code)                          # the argument operands are loaded, not prefetched
