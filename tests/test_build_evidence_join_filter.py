"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so) for the fused pipeline's stage filters: every sink has its filtered
instantiations (pipe_kernel VAR bit 256 on top of the sink's default bits, integer and Decimal128 interpreter), the ordered output kernel
has its filtered twin, and the instantiations without the bit are still there.  The filtered kernels call the out-of-line interpreter."""
import pytest

from test_build_evidence import sass

# (sink, DEC, VAR): build 2, aggregate 3, unordered output 5, pack 6, dense 7, hash 8
FILT = [(2, 0, 256), (2, 1, 256), (3, 0, 267), (3, 1, 256), (5, 0, 258), (5, 1, 256),
        (6, 0, 258), (6, 1, 256), (7, 0, 256), (7, 1, 256), (8, 0, 256), (8, 1, 256)]


def pipe(sink, dec, var):
    return f"_ZN5dfgpu11pipe_kernelILi{sink}ELb{dec}ELi{var}EEEvPKNS_10PipeParamsElPy"


@pytest.mark.parametrize("sink,dec,var", FILT)
def test_filtered_pipe_kernel_instantiations_exist(sink, dec, var):
    code = sass(pipe(sink, dec, var))
    assert len(code) > 2000 and any("CALL" in l for l in code)
    assert len(sass(pipe(sink, dec, var & ~256))) > 2000          # the instantiation without stage filters


def test_ordered_output_kernel_has_a_filtered_twin():
    name = "_ZN5dfgpu18pipe_output_kernelILb{}EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_"
    plain, filt = sass(name.format(0)), sass(name.format(1))
    assert len(plain) > 2000 and len(filt) > len(plain)
