"""CPU-side build evidence for libdfgpu_strings.so (cuobjdump / nm on that library only): it is built for sm_90a alone, exports exactly
the C entry points include/dfgpu_strings.h declares (and libdfgpu.so exports none of them), each kernel fits the registers its
launch bounds allow with no stack or local memory, and the Utf8 kernels stage their tiles with TMA bulk copies (UBLKCP)."""
import os
import re
import subprocess

from datafusion_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = capi.STRINGS_LIB_PATH
KERNELS = {   # kernel -> its __launch_bounds__ threads per block
    "_ZN5dfgpu4like16like_utf8_kernelIiEEvNS0_7ProgramEPKT_PKhS7_llPhS8_": 256,
    "_ZN5dfgpu4like16like_utf8_kernelIlEEvNS0_7ProgramEPKT_PKhS7_llPhS8_": 256,
    "_ZN5dfgpu4like16like_view_kernelENS0_7ProgramENS0_8ViewBufsEPK5uint4PKhllPhS8_": 256,
    "_ZN5dfgpu4like17like_codes_kernelEPKiPKhllS4_lPhS5_": 256,
}


def header_symbols():
    text = open(os.path.join(ROOT, "include", "dfgpu_strings.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dfgpu_\w+)\s*\(", text)))


def exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {ln.split()[-1] for ln in out.splitlines() if ln.split()[-2:-1] == ["T"]}


def test_library_is_sm90a_only():
    out = subprocess.run(["cuobjdump", "-lelf", LIB], capture_output=True, text=True).stdout
    assert set(re.findall(r"sm_(\d+a?)", out)) == {"90a"}, out


def test_exports_exactly_the_header():
    assert header_symbols() == sorted(capi.STRINGS_EXPORTS)
    c_symbols = {s for s in exported(LIB) if s.startswith("dfgpu_")}
    assert c_symbols == set(header_symbols())
    assert not c_symbols & exported(capi.LIB_PATH), "libdfgpu.so must not carry the string predicates"


def test_does_not_link_libdfgpu():
    out = subprocess.run(["readelf", "-d", LIB], capture_output=True, text=True, check=True).stdout
    assert "libdfgpu.so" not in out


def resources():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = {}
    for name, body in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        res[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", body)}
    return res


def test_kernels_fit_their_launch_bounds_without_local_memory():
    res = resources()
    assert set(KERNELS) <= set(res), sorted(res)
    for k, threads in KERNELS.items():
        r = res[k]
        assert r["REG"] * threads <= 65536 and r["REG"] <= 255, (k, r)
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (k, r)


def test_utf8_tiles_are_staged_with_tma():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", out)
    staged = [f.split("\n", 1)[0].strip() for f in funcs if "UBLKCP" in f]
    assert sorted(staged) == sorted(k for k in KERNELS if "utf8" in k)
