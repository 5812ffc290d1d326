"""The trace grid's reserve for list kernels (pb2_trace_blocks_with_reserve), on the CPU.

With several wavefront pipelines the persistent trace grid leaves room on every SM for one block of the frame's largest
list kernel.  The arithmetic is checked by hand on its limits, and on the benchmark's class-0 kernels as ptxas built them
(cuobjdump's resource usage of lib/libpb2.so): the two-child trace kernel at 56 registers and the class-0 shade step at
128 registers leave room for 6 trace blocks of 128 threads per SM (6 x 7168 + 16 384 = 59 392 of 65 536 registers;
a seventh would need 66 560).
"""
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT


def cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


def reserve(pb, trace_regs, trace_smem, list_regs, list_smem, max_blocks=8):
    return pb.lib().pb2_trace_blocks_with_reserve(trace_regs, trace_smem, list_regs, list_smem, max_blocks)


def test_reserve_arithmetic(pb):
    # registers: per warp, in units of 256
    assert reserve(pb, 56, 0, 128, 0) == 6                 # 6 x 7168 + 16 384 <= 65 536 < 7 x 7168 + 16 384
    assert reserve(pb, 48, 0, 128, 0) == 8                 # 8 x 6144 + 16 384 = 65 536 exactly
    assert reserve(pb, 49, 0, 128, 0) == 6                 # 49 x 32 rounds up to 1792 registers per warp, as 56 does
    assert reserve(pb, 32, 0, 32, 0, max_blocks=32) == 15  # threads: 16 blocks of 128 fill the SM's 2048
    assert reserve(pb, 56, 0, 128, 0, max_blocks=4) == 4   # never more than the kernel's own limit
    # shared memory: 228 KB per SM, 1 KB of it per block
    assert reserve(pb, 32, 17 * 1024, 32, 34 * 1024) == 8
    assert reserve(pb, 32, 40 * 1024, 32, 34 * 1024) == 4  # 4 x 41 KB + 35 KB = 199 KB; a fifth block would need 240 KB
    assert reserve(pb, 32, 0, 32, 228 * 1024) == 0         # a list block that fills the SM leaves nothing
    assert reserve(pb, 255, 0, 255, 0) == 1                # 255 x 32 rounds up to 8192 a warp: two blocks fill the SM
    assert reserve(pb, 255, 0, 255, 0, max_blocks=0) == 0


def resource_usage():
    """{demangled kernel name: (registers, static shared memory bytes)} of lib/libpb2.so."""
    tool = cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not installed")
    lib = os.path.join(ROOT, "pbrt_v3_b200", "lib", "libpb2.so")
    out = subprocess.run([tool, "-res-usage", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):", out)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), stdout=subprocess.PIPE, text=True, check=True).stdout.split("\n")
    usage = {}
    for name, m in zip(demangled, re.finditer(r"Function \S+:\s*REG:(\d+)\s+STACK:\d+\s+SHARED:(\d+)", out)):
        usage[name.split("(")[0].replace("void ", "")] = (int(m.group(1)), int(m.group(2)))
    return usage


def test_reserve_of_the_bench_kernels(pb):
    usage = resource_usage()
    trace = usage["k_wf_trace_w<2, 0>"]
    lists = [usage[k] for k in ("k_wf_gen<0>", "k_wf_advance<false, 7, 0>", "k_wf_advance<true, 4, 0>")]
    list_regs, list_smem = max(r for r, _ in lists), max(s for _, s in lists)
    assert trace[0] == 56 and list_regs == 128, (trace, lists)
    assert reserve(pb, trace[0], trace[1], list_regs, list_smem) == 6
