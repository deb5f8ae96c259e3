"""Register budget of the fused four-step kernel (fused.h run_fused), checked from the ptxas report the build writes.

The consumer warpgroups raise their budget with setmaxnreg; the default instantiations must then keep every value in
registers, because spilled values leave the SM's small L1 (the kernel claims nearly all of it as shared memory) and
cost an L2 round trip on every tile.  No GPU needed: a regression shows up at build time."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTXAS_LOG = os.path.join(ROOT, "rustfft_b200", "csrc", "ptxas.log")

# (N1, N2) the planner picks for f32 FourStep sizes, by log2 N
TWO_STAGE_PLANS = {15: (128, 256), 16: (256, 256), 17: (256, 512), 18: (512, 512), 19: (512, 1024), 20: (1024, 1024)}
# three-stage 2048- / 4096-point tiles: spill stores (bytes) before the consumers had their own register budget
THREE_STAGE_SPILL_STORES_BEFORE = {21: ((1024, 2048), 84), 22: ((2048, 2048), 132), 23: ((2048, 4096), 136), 24: ((4096, 4096), 108)}
LAUNCH_REGS = 96  # __launch_bounds__(640, 1): what every thread holds before setmaxnreg

_ENTRY = re.compile(
    r"Compiling entry function '(_ZN2b29run_fused[^']*)' for 'sm_90a'\n"
    r"(?:ptxas info\s*: Function properties for \S+\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n)?"
    r"ptxas info\s*: Used (\d+) registers")
# TmaTileKernel<Geo<float, L, ...>, M0, M1, ROLE, SW, TILED, DOUT>
_KERNEL = re.compile(r"TmaTileKernel<b2::Geo<float, (\d+), [^<>]*<[^<>]*>, \d+>, \(b2::Map\)\d, \(b2::Map\)\d, (\d), (true|false), (\d+), (true|false)>")


def _default_fused_entries():
    """{(N1, N2, inverse): (spill stores, spill loads, registers)} of the default run_fused instantiations: contiguous
    ring (TILED = 0), pass-B output through the TMA store (DOUT = false)."""
    if not os.path.exists(PTXAS_LOG):
        pytest.fail(f"{PTXAS_LOG} missing: build() writes it")
    if shutil.which("c++filt") is None:
        pytest.fail("c++filt (binutils) is needed to read the kernel names")
    entries = _ENTRY.findall(open(PTXAS_LOG).read())
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in entries), capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(names) == len(entries)
    out = {}
    for (_, _, st, ld, regs), name in zip(entries, names):
        ka, kb = _KERNEL.findall(name.split("(b2::FusedKernel")[0])
        (l1, _, sw, tiled, _), (l2, _, _, _, dout) = ka, kb
        if tiled == "0" and dout == "false":
            out[(int(l1), int(l2), sw == "true")] = (int(st or 0), int(ld or 0), int(regs))
    return out


def test_two_stage_fused_plans_do_not_spill():
    got = _default_fused_entries()
    for lg, (n1, n2) in TWO_STAGE_PLANS.items():
        for inverse in (False, True):
            assert (n1, n2, inverse) in got, f"2^{lg}: run_fused {n1}x{n2} not in the ptxas report"
            st, ld, regs = got[(n1, n2, inverse)]
            assert (st, ld) == (0, 0), f"2^{lg} {n1}x{n2} inverse={inverse}: {st} bytes spill stores, {ld} bytes spill loads"
            assert regs <= LAUNCH_REGS, f"2^{lg} {n1}x{n2}: {regs} registers at entry"


def test_three_stage_fused_plans_spill_less_than_before():
    got = _default_fused_entries()
    for lg, ((n1, n2), before) in THREE_STAGE_SPILL_STORES_BEFORE.items():
        for inverse in (False, True):
            assert (n1, n2, inverse) in got, f"2^{lg}: run_fused {n1}x{n2} not in the ptxas report"
            st, _, regs = got[(n1, n2, inverse)]
            assert st < before, f"2^{lg} {n1}x{n2} inverse={inverse}: {st} bytes spill stores (was {before})"
            assert regs <= LAUNCH_REGS, f"2^{lg} {n1}x{n2}: {regs} registers at entry"
