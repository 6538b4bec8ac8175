"""Register and spill budgets of the batch kernels, read from ptxas without a GPU.

rl_engine.cu is compiled for sm_90a with `-Xptxas -v` into a temporary directory.  How many CTAs of k_main and
k_front an SM holds at once is set by their registers per thread (DESIGN.md §3.2), and a spill turns register
traffic into local-memory round trips on the replay's critical path, so both are pinned here:
  * C2's replay, k_main<7, 4, RecordSrc, 0, 128, false> (record batches of 4-cell row groups in 128-access chunks),
    fits 80 registers without spilling: 6 CTAs per SM, 792 slots on 132 SMs for a 65536-request batch's ~800 chunks;
  * k_front's record instantiations (the front of every record batch, C2's included) fit 64 registers without
    spilling, so that four of its 256-thread CTAs fit the register file beside the replay;
  * no instantiation of k_main, k_front or k_hot uses more registers or spills more bytes than CEILINGS says.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "limitador_b200", "csrc")

# mangled entry name -> (registers, spill store bytes, spill load bytes) of the sm_90a build
CEILINGS = {
    "_Z6k_mainILi7ELi7E9RecordSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (128, 128, 108),
    "_Z6k_mainILi7ELi7E9RecordSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (128, 128, 108),
    "_Z5k_hotILi7ELi7E9RecordSrcLi0ELb0EEv5RlDev7RlBatchT1_": (120, 0, 0),
    "_Z6k_mainILi7ELi7E9RecordSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (128, 192, 172),
    "_Z6k_mainILi7ELi7E9RecordSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (128, 232, 216),
    "_Z5k_hotILi7ELi7E9RecordSrcLi0ELb1EEv5RlDev7RlBatchT1_": (128, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (113, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (80, 0, 0),
    "_Z5k_hotILi7ELi4E9RecordSrcLi0ELb0EEv5RlDev7RlBatchT1_": (100, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (120, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 24, 16),
    "_Z5k_hotILi7ELi4E9RecordSrcLi0ELb1EEv5RlDev7RlBatchT1_": (118, 0, 0),
    "_Z6k_mainILi3ELi3E9RecordSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (109, 0, 0),
    "_Z6k_mainILi3ELi3E9RecordSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (90, 0, 0),
    "_Z5k_hotILi3ELi3E9RecordSrcLi0ELb0EEv5RlDev7RlBatchT1_": (96, 0, 0),
    "_Z6k_mainILi3ELi3E9RecordSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (116, 0, 0),
    "_Z6k_mainILi3ELi3E9RecordSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 0, 0),
    "_Z5k_hotILi3ELi3E9RecordSrcLi0ELb1EEv5RlDev7RlBatchT1_": (112, 0, 0),
    "_Z6k_mainILi1ELi1E9RecordSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (64, 0, 0),
    "_Z6k_mainILi1ELi1E9RecordSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (62, 0, 0),
    "_Z5k_hotILi1ELi1E9RecordSrcLi0ELb0EEv5RlDev7RlBatchT1_": (64, 12, 28),
    "_Z6k_mainILi1ELi1E9RecordSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (64, 180, 176),
    "_Z6k_mainILi1ELi1E9RecordSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (64, 180, 176),
    "_Z5k_hotILi1ELi1E9RecordSrcLi0ELb1EEv5RlDev7RlBatchT1_": (102, 0, 0),
    "_Z6k_mainILi7ELi7E9RecordSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (126, 0, 0),
    "_Z6k_mainILi7ELi7E9RecordSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (126, 0, 0),
    "_Z5k_hotILi7ELi7E9RecordSrcLi2ELb0EEv5RlDev7RlBatchT1_": (96, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (99, 0, 0),
    "_Z6k_mainILi7ELi4E9RecordSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (88, 0, 0),
    "_Z5k_hotILi7ELi4E9RecordSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 112, 188),
    "_Z6k_mainILi3ELi3E9RecordSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (90, 0, 0),
    "_Z6k_mainILi3ELi3E9RecordSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (86, 0, 0),
    "_Z5k_hotILi3ELi3E9RecordSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 44, 68),
    "_Z6k_mainILi1ELi1E9RecordSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (64, 0, 0),
    "_Z6k_mainILi1ELi1E9RecordSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (61, 0, 0),
    "_Z5k_hotILi1ELi1E9RecordSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 0, 0),
    "_Z6k_mainILi7ELi7E6AccSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (128, 348, 320),
    "_Z6k_mainILi7ELi7E6AccSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (128, 372, 344),
    "_Z5k_hotILi7ELi7E6AccSrcLi0ELb0EEv5RlDev7RlBatchT1_": (122, 0, 0),
    "_Z6k_mainILi7ELi7E6AccSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (128, 284, 256),
    "_Z6k_mainILi7ELi7E6AccSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (128, 284, 256),
    "_Z5k_hotILi7ELi7E6AccSrcLi0ELb1EEv5RlDev7RlBatchT1_": (128, 0, 0),
    "_Z6k_mainILi7ELi4E6AccSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (127, 0, 0),
    "_Z6k_mainILi7ELi4E6AccSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (96, 172, 144),
    "_Z5k_hotILi7ELi4E6AccSrcLi0ELb0EEv5RlDev7RlBatchT1_": (108, 0, 0),
    "_Z6k_mainILi7ELi4E6AccSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (124, 0, 0),
    "_Z6k_mainILi7ELi4E6AccSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 108, 92),
    "_Z5k_hotILi7ELi4E6AccSrcLi0ELb1EEv5RlDev7RlBatchT1_": (119, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (112, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (96, 0, 0),
    "_Z5k_hotILi3ELi3E6AccSrcLi0ELb0EEv5RlDev7RlBatchT1_": (100, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (116, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 0, 0),
    "_Z5k_hotILi3ELi3E6AccSrcLi0ELb1EEv5RlDev7RlBatchT1_": (114, 0, 0),
    "_Z6k_mainILi1ELi1E6AccSrcLi0ELi256ELb0EEv5RlDev7RlBatchT1_j": (64, 132, 120),
    "_Z6k_mainILi1ELi1E6AccSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (64, 132, 120),
    "_Z5k_hotILi1ELi1E6AccSrcLi0ELb0EEv5RlDev7RlBatchT1_": (64, 48, 80),
    "_Z6k_mainILi1ELi1E6AccSrcLi0ELi256ELb1EEv5RlDev7RlBatchT1_j": (64, 196, 188),
    "_Z6k_mainILi1ELi1E6AccSrcLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (64, 196, 188),
    "_Z5k_hotILi1ELi1E6AccSrcLi0ELb1EEv5RlDev7RlBatchT1_": (102, 0, 0),
    "_Z6k_mainILi7ELi7E10AccSrcWideLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (128, 372, 344),
    "_Z6k_mainILi7ELi7E10AccSrcWideLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (128, 208, 184),
    "_Z6k_mainILi7ELi4E10AccSrcWideLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (96, 164, 136),
    "_Z6k_mainILi7ELi4E10AccSrcWideLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 160, 132),
    "_Z6k_mainILi3ELi3E10AccSrcWideLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (96, 0, 0),
    "_Z6k_mainILi3ELi3E10AccSrcWideLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (96, 0, 0),
    "_Z6k_mainILi1ELi1E10AccSrcWideLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": (64, 132, 120),
    "_Z6k_mainILi1ELi1E10AccSrcWideLi0ELi128ELb1EEv5RlDev7RlBatchT1_j": (64, 192, 184),
    "_Z6k_mainILi7ELi7E6AccSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (128, 0, 0),
    "_Z6k_mainILi7ELi7E6AccSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (128, 0, 0),
    "_Z5k_hotILi7ELi7E6AccSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 104, 112),
    "_Z6k_mainILi7ELi4E6AccSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (101, 0, 0),
    "_Z6k_mainILi7ELi4E6AccSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (90, 0, 0),
    "_Z5k_hotILi7ELi4E6AccSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (91, 0, 0),
    "_Z6k_mainILi3ELi3E6AccSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (84, 0, 0),
    "_Z5k_hotILi3ELi3E6AccSrcLi2ELb0EEv5RlDev7RlBatchT1_": (64, 0, 0),
    "_Z6k_mainILi1ELi1E6AccSrcLi2ELi256ELb0EEv5RlDev7RlBatchT1_j": (62, 0, 0),
    "_Z6k_mainILi1ELi1E6AccSrcLi2ELi128ELb0EEv5RlDev7RlBatchT1_j": (61, 0, 0),
    "_Z5k_hotILi1ELi1E6AccSrcLi2ELb0EEv5RlDev7RlBatchT1_": (60, 0, 0),
    "_Z7k_frontILi7E6AccSrcEv5RlDev7RlBatchT0_": (80, 0, 0),
    "_Z7k_frontILi3E6AccSrcEv5RlDev7RlBatchT0_": (80, 0, 0),
    "_Z7k_frontILi1E6AccSrcEv5RlDev7RlBatchT0_": (80, 0, 0),
    "_Z7k_frontILi7E9RecordSrcEv5RlDev7RlBatchT0_": (64, 0, 0),
    "_Z7k_frontILi3E9RecordSrcEv5RlDev7RlBatchT0_": (64, 0, 0),
    "_Z7k_frontILi1E9RecordSrcEv5RlDev7RlBatchT0_": (64, 0, 0),
}

# kernel -> register budget, with no spill: C2's replay (6 CTAs of 128 threads per SM) and the record fronts
# (4 CTAs of 256 threads)
BUDGETS = {"_Z6k_mainILi7ELi4E9RecordSrcLi0ELi128ELb0EEv5RlDev7RlBatchT1_j": 80,
           **{k: 64 for k in CEILINGS if k.startswith("_Z7k_frontI") and "9RecordSrc" in k}}


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _readable(mangled: str) -> str:
    m = re.match(r"_Z\d+(k_[a-z]+)I(.*?)Ev\d", mangled)
    if not m:
        return mangled
    args = re.findall(r"Li(\d+)E|Lb([01])E|\d+(RecordSrc|AccSrcWide|AccSrc)", m.group(2) + "E")
    return f"{m.group(1)}<{', '.join(a or ('true' if b == '1' else 'false' if b else c) for a, b, c in args)}>"


@pytest.fixture(scope="module")
def ptxas():
    """mangled entry -> (registers, spill store bytes, spill load bytes) of every kernel of rl_engine.cu."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
               "-diag-suppress", "128,177", "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v",
               "-c", "-o", os.path.join(tmp, "rl_engine.o"), os.path.join(CSRC, "rl_engine.cu")]
        p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    res, cur, spill = {}, None, None
    for line in p.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur, spill = m.group(1), None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spill = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur is not None and spill is not None:
            res[cur] = (int(m.group(1)), *spill)
            cur = None
    return res


def test_every_budgeted_kernel_is_compiled(ptxas):
    missing = [_readable(k) for k in CEILINGS if k not in ptxas]
    assert not missing, f"not found in the ptxas output: {missing}"


@pytest.mark.parametrize("name", list(BUDGETS), ids=_readable)
def test_fits_its_register_budget_without_spilling(ptxas, name):
    regs, st, ld = ptxas[name]
    assert regs <= BUDGETS[name] and st == 0 and ld == 0, \
        f"{_readable(name)}: {regs} registers (budget {BUDGETS[name]}), {st} B spill stores, {ld} B spill loads"


def test_no_kernel_uses_more_registers_or_spills_more_than_recorded(ptxas):
    worse = []
    for name, (regs, st, ld) in CEILINGS.items():
        got = ptxas.get(name)
        if got is not None and (got[0] > regs or got[1] > st or got[2] > ld):
            worse.append(f"{_readable(name)}: {got} > {(regs, st, ld)}")
    assert not worse, "\n".join(worse)
