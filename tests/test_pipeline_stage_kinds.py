"""The binding's probe-stage kinds against the header's dfgpu_stage_kind enum (include/dfgpu.h): every DFGPU_STAGE_* value, RIGHT included."""
import os
import re

from datafusion_b200 import capi as D

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dfgpu.h")


def test_stage_kinds_match_the_header():
    text = open(HEADER).read()
    body = re.search(r"enum dfgpu_stage_kind \{(.*?)\};", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    kinds = {m.group(1): int(m.group(2)) for m in re.finditer(r"DFGPU_STAGE_(\w+)\s*=\s*(\d+)", body)}
    assert kinds == {k: getattr(D, "STAGE_" + k) for k in kinds}
    assert kinds["RIGHT"] == D.STAGE_RIGHT == 6 and len(kinds) == 7
