"""tests/ingest.py's mirror of the conversion kernel choice, on the CPU: its truth table, and the source it
mirrors still states the same rule (a change there must change the mirror, or the GPU ingest tests would count
coverage they no longer have)."""
import os
import re

import pytest

from ingest import Q15, SCALAR, VEC, conv_kind, device_offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_conv_kind_truth_table(fmt):
    pair = 8 if fmt == "cs16" else 4
    assert conv_kind(fmt, False, 2048, 0) == VEC
    assert conv_kind(fmt, False, 2048, 0, ptr=4096) == VEC
    assert conv_kind(fmt, False, 2048, 0, ptr=4096 + pair) == VEC
    assert conv_kind(fmt, False, 2047, 0) == SCALAR  # odd n
    assert conv_kind(fmt, False, 2048, 1) == SCALAR  # odd stream position
    assert conv_kind(fmt, False, 1, 0) == SCALAR
    for off in range(1, pair):
        assert conv_kind(fmt, False, 2048, 0, ptr=4096 + off) == SCALAR
    for n, S, ptr in ((2048, 0, None), (7, 3, 4098), (0, 5, None)):
        assert conv_kind(fmt, True, n, S, ptr) == Q15


def test_device_offsets():
    assert device_offsets("cu8") == [0, 2, 4, 8]
    assert device_offsets("cs8") == [0, 2, 4, 8]
    assert device_offsets("cs16") == [0, 4, 8]


def test_mirror_matches_launch_convert():
    with open(os.path.join(ROOT, "sdr-server_b200", "csrc", "xlating_group.cu")) as f:
        src = f.read()
    body = src[src.index("static void launch_convert("):]
    body = body[:body.index("\n}\n")]
    assert "const size_t pair_bytes = FMT == 2 ? 8 : 4;" in body
    cond = re.search(r"if \(q15\) \{\s*convert_q15_kernel<FMT>.*?\} else if \((.*?)\) \{\s*(?:const int per_cta[^\n]*\s*)?"
                     r"convert_cf32_vec_kernel", body, re.S)
    assert cond, body
    assert cond.group(1) == "(n & 1) == 0 && (S & 1) == 0 && ((uintptr_t)raw % pair_bytes) == 0"
    # and device inputs reach it only when aligned to one complex sample
    submit = src[src.index('extern "C" int64_t xlg_submit('):]
    assert "(uintptr_t)input % sample_bytes != 0" in submit[:submit.index("const bool q15")]
