"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so) for the output sinks' bitmap and 16-byte columns: the unordered sink's
new pipe_kernel instantiations (VAR bit 512 on top of the sink's default, filtered and Decimal128-interpreter bits) and the ordered sink's
pipe_output_cols_kernel exist, write validity words with atomic ORs and 16-byte values with one 128-bit store; every instantiation that
ran before keeps its name, registers, stack and local memory (the figures of the build before these kernels were added)."""
import re
import subprocess

import pytest

from datafusion_b200 import capi


def pipe(sink, dec, var):
    return f"_ZN5dfgpu11pipe_kernelILi{sink}ELb{dec}ELi{var}EEEvPKNS_10PipeParamsElPy"


def ordered(name, filt):
    return f"_ZN5dfgpu{len(name)}{name}ILb{filt}EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_"


# (DEC, VAR) of the unordered sink (5): plain, Decimal128 interpreter, stage filters, both
NEW_UNORDERED = [(0, 514), (1, 512), (0, 770), (1, 768)]
NEW_ORDERED = [ordered("pipe_output_cols_kernel", 0), ordered("pipe_output_cols_kernel", 1)]
# REG, STACK, LOCAL of the output instantiations in the build without the new kernels
OLD = {pipe(5, 0, 2): (80, 288, 0), pipe(5, 0, 0): (80, 288, 0), pipe(5, 1, 0): (80, 592, 0), pipe(5, 0, 258): (80, 464, 0),
       pipe(5, 1, 256): (80, 752, 0), ordered("pipe_output_kernel", 0): (80, 592, 0), ordered("pipe_output_kernel", 1): (80, 800, 0)}


def res_usage():
    out = subprocess.run(["cuobjdump", "-res-usage", capi.LIB_PATH], capture_output=True, text=True).stdout
    return {m.group(1): dict(kv.split(":") for kv in m.group(2).split()) for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", out)}


def sass(fn):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", fn, capi.LIB_PATH], capture_output=True, text=True).stdout
    return [l for l in out.splitlines() if re.match(r"\s+/\*[0-9a-f]{4,5}\*/", l)]


@pytest.mark.parametrize("fn", [pipe(5, d, v) for d, v in NEW_UNORDERED] + NEW_ORDERED)
def test_new_output_instantiations_write_bitmaps_and_16_byte_values(fn):
    code = sass(fn)
    assert len(code) > 2000, fn
    assert any(re.search(r"\b(ATOMG?|REDG?)\.E\.OR\b", l) for l in code), fn        # validity words: atomic OR into the zeroed bitmap
    assert any(re.search(r"\bSTG?\.E\.128\b", l) for l in code), fn               # one 16-byte store per Decimal128 value


@pytest.mark.parametrize("fn", sorted(OLD))
def test_existing_output_instantiations_keep_their_resources(fn):
    use = res_usage()
    assert fn in use, fn
    reg, stack, local = OLD[fn]
    assert (int(use[fn]["REG"]), int(use[fn]["STACK"]), int(use[fn]["LOCAL"])) == (reg, stack, local), (fn, use[fn])


def test_new_instantiations_fit_the_registers_of_their_launch_bounds():
    use = res_usage()
    for fn in [pipe(5, d, v) for d, v in NEW_UNORDERED] + NEW_ORDERED:
        assert fn in use, fn
        assert int(use[fn]["REG"]) <= 80 and use[fn]["LOCAL"] == "0", (fn, use[fn])
