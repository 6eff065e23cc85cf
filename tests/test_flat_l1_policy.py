"""CPU: the cache policy of the x gathers in csr_flat_kernel, read from the built library's SASS.

The kernel has two instantiations per value type: HOT = true for a matrix with a hot plan (the packed hot columns xh are
gathered through L1 with a plain read-only load, every other column with ldg_cold, whose policy B200_FLAT_COLD picks), and
HOT = false for a matrix without one (every gather through L1, as with no hot plan at all).  What each spells in SASS:
plain __ldg -> LDG.E[.64].CONSTANT, L1::evict_first -> LDG.E.EF[.64].CONSTANT, .cg -> LDG.E[.64].STRONG.GPU."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMON = os.path.join(ROOT, "cudalibrarysamples_b200", "csrc", "spmv_common.cuh")
MIN_CTAS = 10                          # __launch_bounds__(128, B200_FLAT_MIN_CTAS) of csr_flat_kernel
REGS_PER_SM = 65536


def cold_policy():
    return int(re.search(r"#define B200_FLAT_COLD (\d)", open(COMMON).read()).group(1))


def cold_sass(t, policy):
    """the SASS of ldg_cold for value type t ('d' / 'f') under policy 1 or 2"""
    w = r"\.64" if t == "d" else ""
    return {1: r"LDG\.E\.EF" + w + r"\.CONSTANT", 2: r"LDG\.E" + w + r"\.STRONG\.GPU"}[policy]


def flat_bodies(built_lib):
    sass = subprocess.check_output(["cuobjdump", "-sass", built_lib], text=True)
    bodies = {}
    for m in re.finditer(r"Function : _ZN4b20015csr_flat_kernelI([df])Lb([01])E\S*(.*?)(?=Function :|\Z)", sass, re.S):
        bodies[(m.group(1), m.group(2) == "1")] = m.group(3)
    assert sorted(bodies) == [("d", False), ("d", True), ("f", False), ("f", True)], sorted(bodies)
    return bodies


def test_cold_gathers_follow_the_policy_with_a_hot_plan(built_lib):
    """With a hot plan: 8 cold gathers (one per 32-non-zero step) spelled as B200_FLAT_COLD says, and the hot gathers stay
    plain read-only loads -- 8 of them in the fp64 kernel; in the fp32 kernel as many plain 32-bit loads as without a hot
    plan, where those 8 are the plain gathers."""
    p = cold_policy()
    assert p in (1, 2), "the cold gathers of a hot plan take a policy of their own"
    b = flat_bodies(built_lib)
    for t in ("d", "f"):
        assert len(re.findall(cold_sass(t, p), b[(t, True)])) == 8
    assert len(re.findall(r"LDG\.E\.64\.CONSTANT", b[("d", True)])) == 8
    assert len(re.findall(r"LDG\.E\.CONSTANT", b[("f", True)])) == len(re.findall(r"LDG\.E\.CONSTANT", b[("f", False)]))


def test_without_a_hot_plan_every_gather_goes_through_l1(built_lib):
    """No hot plan: no L2-only or evict-first gather, and the 8 gathers of the fp64 kernel are plain read-only loads."""
    b = flat_bodies(built_lib)
    for t in ("d", "f"):
        assert not re.search(r"STRONG\.GPU|\.EF\b|\.EF\.", b[(t, False)])
    assert len(re.findall(r"LDG\.E\.64\.CONSTANT", b[("d", False)])) == 8


def test_streams_and_gathers_keep_their_spelling(built_lib):
    """The val[] / col_ind[] streams stay L1-no-allocate (8 + 8 per warp chunk) in every instantiation; none of the gathers
    takes that spelling."""
    for (t, hot), body in flat_bodies(built_lib).items():
        assert len(re.findall(r"LDG\.E\.NA\.64", body)) == (8 if t == "d" else 0)
        assert len(re.findall(r"LDG\.E\.NA\.CONSTANT", body)) == (8 if t == "d" else 16)


def test_no_local_memory_and_ten_ctas_fit(built_lib):
    """No spills, and the register count lets B200_FLAT_MIN_CTAS CTAs of 128 threads share an SM."""
    out = subprocess.check_output(["cuobjdump", "-res-usage", built_lib], text=True)
    found = re.findall(r"Function _ZN4b20015csr_flat_kernelI[df]Lb[01]E\S*:\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert len(found) == 4
    for reg, stack, local in found:
        assert int(stack) == 0 and int(local) == 0
        assert int(reg) * 128 * MIN_CTAS <= REGS_PER_SM
