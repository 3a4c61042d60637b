"""CPU-side evidence for the hash exchange's bit-packed scatter: every single-pass scatter instantiation fits the 64 registers its
launch bounds allow without spilling; only the instantiations for bit-packed columns carry atomics (device scope locally, system
scope for peer memory); and the per-column "has a validity bitmap" flags every rank contributes to the exchange's all-gather."""
import re
import subprocess

from datafusion_b200 import capi, exchange

BITS = {"_ZN5dfgpu25partition_scatter8_kernelILb0ELb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli",
        "_ZN5dfgpu25partition_scatter8_kernelILb1ELb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli",
        "_ZN5dfgpu24partition_scatter_kernelILb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEl"}
PLAIN = {"_ZN5dfgpu25partition_scatter8_kernelILb0ELb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli",
         "_ZN5dfgpu25partition_scatter8_kernelILb1ELb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli",
         "_ZN5dfgpu24partition_scatter_kernelILb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEl"}


def res_usage():
    out = subprocess.run(["cuobjdump", "-res-usage", capi.LIB_PATH], capture_output=True, text=True).stdout
    return {m.group(1): m.group(2) for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", out)}


def atomics(fn):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", fn, capi.LIB_PATH], capture_output=True, text=True).stdout
    return re.findall(r"\b(?:ATOM|RED)[A-Z0-9.]*", out)


def test_every_scatter_instantiation_fits_its_registers_without_spills():
    use = res_usage()
    for fn in BITS | PLAIN:
        assert fn in use, fn
        f = dict(kv.split(":") for kv in use[fn].split())
        assert int(f["REG"]) <= 64 and f["STACK"] == "0" and f["LOCAL"] == "0", (fn, use[fn])


def test_only_the_bit_instantiations_carry_atomics():
    for fn in PLAIN:
        assert atomics(fn) == [], fn
    for fn in BITS:
        a = set(atomics(fn))
        assert {"ATOM.E.AND.STRONG.GPU", "ATOM.E.OR.STRONG.GPU", "ATOM.E.AND.STRONG.SYS", "ATOM.E.OR.STRONG.SYS"} <= a, (fn, a)


def test_bitmap_flags_follow_validity_and_null_count():
    cols = (capi.Column * 4)()
    for i, (validity, nulls) in enumerate([(None, 0), (0x1000, -1), (0x2000, 0), (0x3000, 7)]):
        cols[i].validity, cols[i].null_count = validity, nulls
    assert exchange.has_bitmap(cols, 4) == [0, 1, 0, 1]   # a bitmap with null_count 0 holds no NULL: the column travels without it
