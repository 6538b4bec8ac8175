"""Host-side resources of the native library: device and pinned memory are allocated and freed only by the owning
arrays of csrc/rl_cuda_host.h, and every error message is formatted by csrc/rl_error.h, which cuts a long message
without splitting a UTF-8 sequence."""
import os
import re
import shutil
import subprocess

import pytest

from limitador_b200 import matcher as MT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "limitador_b200", "csrc")


def _calls(pattern):
    """{file: [line, ...]} of the sources under csrc/ whose code (comments stripped) calls `pattern`."""
    out = {}
    for f in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, f), encoding="utf-8") as fh:
            for no, line in enumerate(fh, 1):
                if re.search(pattern, line.split("//")[0]):
                    out.setdefault(f, []).append(no)
    return out


def test_cuda_memory_is_allocated_and_freed_only_by_the_owning_arrays():
    calls = _calls(r"\bcuda(Malloc|Free)\w*\s*\(")
    assert "rl_cuda_host.h" in calls
    assert {f: v for f, v in calls.items() if f != "rl_cuda_host.h"} == {}


def test_messages_are_formatted_only_by_rl_error_h():
    calls = _calls(r"\bvsnprintf\s*\(")
    assert "rl_error.h" in calls
    assert {f: v for f, v in calls.items() if f != "rl_error.h"} == {}


_DRIVER = r"""
#include <iostream>
#include <string>
#include "rl_error.h"
int main() {
    std::string line;
    while (std::getline(std::cin, line)) std::cout << rl_format("%s", line.c_str()) << '\n';
    return 0;
}
"""

_CUT = 511  # rl_format's buffer holds 511 bytes and the terminator


def _longest_whole_prefix(b: bytes, limit: int) -> bytes:
    """The longest prefix of b within `limit` bytes that does not end inside a UTF-8 sequence."""
    k = min(len(b), limit)
    while 0 < k < len(b) and (b[k] & 0xC0) == 0x80:  # b[k], the first byte cut off, continues a sequence
        k -= 1
    return b[:k]


def test_formatter_cuts_long_messages_on_a_character_boundary(tmp_path):
    cc = shutil.which("g++")
    if cc is None:
        pytest.skip("g++ not found")
    src, exe = tmp_path / "fmt.cpp", tmp_path / "fmt"
    src.write_text(_DRIVER)
    subprocess.run([cc, "-std=c++17", "-Wall", "-Werror", f"-I{CSRC}", str(src), "-o", str(exe)], check=True)
    msgs = []
    for ch in ("é", "€", "😀"):  # 2-, 3- and 4-byte sequences
        w = len(ch.encode())
        for start in range(_CUT - w - 1, _CUT + 2):  # the character ends before, across or after the cut
            msgs.append(("a" * start + ch + "z" * 40).encode())
    r = subprocess.run([str(exe)], input=b"\n".join(msgs) + b"\n", capture_output=True, check=True)
    got = r.stdout.split(b"\n")[:-1]
    assert len(got) == len(msgs)
    for full, out in zip(msgs, got):
        out.decode("utf-8")  # valid UTF-8
        assert full.startswith(out)
        assert out == _longest_whole_prefix(full, _CUT)


def test_matcher_error_of_a_cut_condition_decodes():
    cond = "descriptors[0]['k'].size() == " + "ü€😀" * 80  # unsupported, and far longer than a message holds
    with pytest.raises(MT.MatcherError) as ei:
        MT.Matcher().add_limit("ns", 5, 60, [cond])
    msg = str(ei.value)
    assert msg.startswith("unsupported condition expression: descriptors[0]")
    assert ("unsupported condition expression: " + cond).startswith(msg)
    assert len(msg.encode()) > _CUT - 4
