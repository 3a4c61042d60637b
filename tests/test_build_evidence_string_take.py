"""CPU-side build evidence for the string gather kernels of libdfgpu_strings.so (cuobjdump / nm): they exist, fit the registers their
launch bounds allow with no stack or local memory, use no TMA bulk copy (UBLKCP: a gather reads rows at random and stages no tile), and
libdfgpu.so exports none of the new entry points."""
import re
import subprocess

from datafusion_b200 import capi

LIB = capi.STRINGS_LIB_PATH
KERNELS = {   # kernel -> its __launch_bounds__ threads per block
    "_ZN5dfgpu4take19take_lengths_kernelIiEEvNS0_7SourcesENS0_3IdsElPlPPKhPyS8_": 256,
    "_ZN5dfgpu4take19take_lengths_kernelIlEEvNS0_7SourcesENS0_3IdsElPlPPKhPyS8_": 256,
    "_ZN5dfgpu4take22take_scan_tiles_kernelEPylS1_": 256,
    "_ZN5dfgpu4take19take_offsets_kernelElPlPKyPhPy": 256,
    "_ZN5dfgpu4take16take_copy_kernelIiEEvlPKlPKPKhPT_Ph": 256,
    "_ZN5dfgpu4take16take_copy_kernelIlEEvlPKlPKPKhPT_Ph": 256,
    "_ZN5dfgpu4take17take_views_kernelENS0_7SourcesENS0_3IdsElP5uint4PjPy": 256,
}
ENTRY_POINTS = {"dfgpu_string_take_scratch_bytes", "dfgpu_string_take_offsets", "dfgpu_string_take_data", "dfgpu_string_take_views"}


def exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if ln.split()[-2:-1] == ["T"]}


def sass_functions():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    return {f.split("\n", 1)[0].strip(): f for f in re.split(r"\n\s*Function : ", out)[1:]}


def test_entry_points_are_in_the_strings_library_only():
    assert ENTRY_POINTS <= exported(LIB)
    assert not ENTRY_POINTS & exported(capi.LIB_PATH)
    assert ENTRY_POINTS <= set(capi.STRINGS_EXPORTS)


def test_kernels_fit_their_launch_bounds_without_local_memory():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {name: {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", body)} for name, body in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out)}
    assert set(KERNELS) <= set(res), sorted(res)
    for k, threads in KERNELS.items():
        r = res[k]
        assert r["REG"] * threads <= 65536 and r["REG"] <= 255, (k, r)
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (k, r)


def test_kernels_use_no_tma_and_no_local_loads():
    funcs = sass_functions()
    for k in KERNELS:
        assert "UBLKCP" not in funcs[k], k
        assert not re.search(r"\b(LDL|STL)\b", funcs[k]), k
