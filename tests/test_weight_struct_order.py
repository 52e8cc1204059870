"""CPU: the ctypes mirrors of the packed-weight structs list their members in the header's order.  The C ABI grows by
appending members (B200LatteWeights' and B200T2VWeights' e4m3 copies); a field inserted, dropped or swapped on one side only
would hand the library a pointer in the wrong slot without any error."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _members(struct):
    with open(os.path.join(ROOT, "include", "latte_b200.h")) as f:
        src = f.read()
    m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), src, re.S)
    assert m, f"{struct} not found in include/latte_b200.h"
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    return tuple(re.findall(r"^\s*const\s+\w+\s*\*\s*(\w+)\s*;", body, re.M))


@pytest.mark.parametrize("struct,fields", [("B200LatteWeights", "WEIGHT_FIELDS"), ("B200T2VWeights", "T2V_WEIGHT_FIELDS")])
def test_weight_struct_member_order(struct, fields):
    from latte_b200 import _lib
    members = _members(struct)
    assert len(members) > 20
    assert members == getattr(_lib, fields)


def test_t2v_fp8_fields_are_appended():
    from latte_b200 import _lib
    assert _lib.T2V_WEIGHT_FIELDS[-8:] == ("s_qkv_w8", "s_qkv_ws", "s_fc1_w8", "s_fc1_ws",
                                           "t_qkv_w8", "t_qkv_ws", "t_fc1_w8", "t_fc1_ws")
