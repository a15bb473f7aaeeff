"""Device scratch has one owner (Scratch in vb_common.cuh): no library source may bring back numbered workspace
slots, whose sharing rested on comments about which calls never nest, or a function-static pointer that keeps a
scratch range alive from one call to the next.  Handles and images own their memory with cudaMalloc, which stays
allowed."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pgvector_b200", "csrc")

BANNED = [
    (re.compile(r"\bworkspace\s*\("), "workspace(): take ranges from a Scratch instead"),
    (re.compile(r"\benum\s*\{\s*WS\w*\s*="), "a WS*_ slot enum"),
    (re.compile(r"\bws_slot\b|\bws_bytes\b|\bws\s*\["), "a workspace slot"),
    (re.compile(r"\(\s*int\s+\w*slot\s*,\s*size_t\s+\w+\s*,\s*void\s*\*\*"), "an allocator keyed by a slot number"),
    (re.compile(r"^\s+static\s+[^(;=]*\*\s*\w+\s*(=|;)", re.M), "a function-static pointer (scratch does not outlive its call)"),
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))


@pytest.mark.parametrize("name", sources())
def test_no_slot_numbers_or_static_scratch(name):
    with open(os.path.join(CSRC, name)) as f:
        text = f.read()
    found = []
    for rx, what in BANNED:
        for m in rx.finditer(text):
            found.append(f"{name}:{text.count(chr(10), 0, m.start()) + 1}: {what}: {m.group(0).strip()}")
    assert not found, "\n".join(found)


def test_the_rules_catch_what_they_ban():
    samples = ["VB_TRY(workspace(WS_OUT, 64, &p));", "enum { WSX_A = 3 };", "int ws_slot",
               "int scratch_slot(int slot, size_t bytes, void** out);", "    static void* qn_buf = nullptr;"]
    for s in samples:
        assert any(rx.search(s) for rx, _ in BANNED), s
