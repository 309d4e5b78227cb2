"""The Bedrock (group 0) and OpenAI passthrough (group 1) walk kernels keep the walker in registers.  The walk runs one thread per
body; when the walker object's address escaped to an out-of-line planner, every plan push and token access went through local
memory.  So the planner chain is inlined, and the only local array is one 48-entry stack of token indices that validate_tokens
and emit_any take turns on.  ptxas reports that as the kernel's stack frame: this test compiles both units for sm_90a and checks
the frame, the spills and that nothing is left out of line.  Cross-compiles: no GPU needed."""
import concurrent.futures
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "aigw_b200", "csrc")
MAX_FRAME = 96   # bytes: Walker::stk, 48 uint16 token indices


def _nvcc():
    from aigw_b200 import build
    c = build.nvcc()
    return c if (os.path.isabs(c) and os.path.exists(c)) or shutil.which(c) else None


def _ptxas_report(nvcc, src, out):
    cmd = [nvcc] + ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o", out, os.path.join(CSRC, src)]
    r = subprocess.run(cmd, capture_output=True, text=True, check=True)
    return r.stderr


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_bedrock_and_passthrough_walk_frames(tmp_path):
    nvcc = _nvcc()
    units = {0: "chat_walk_g0.cu", 1: "chat_walk_g1.cu"}
    with concurrent.futures.ThreadPoolExecutor(len(units)) as ex:
        logs = dict(zip(units, ex.map(lambda g: _ptxas_report(nvcc, units[g], str(tmp_path / f"g{g}.cubin")), units)))
    for g, log in logs.items():
        kernel = f"chat_walk_kernel_g{g}"
        # every function in the unit: the kernel and anything ptxas kept out of line
        props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
        assert any(kernel in name for name, *_ in props), log
        for name, frame, st, ld in props:
            assert int(st) == 0 and int(ld) == 0, (g, name, st, ld)
            if kernel in name:
                assert int(frame) <= MAX_FRAME, (g, name, frame)
            else:
                pytest.fail(f"group {g}: {name} is compiled out of line")
