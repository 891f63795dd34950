"""Resource usage of the stereo frame wavefront (k_chain_direct4), read from the sm_90a build (no GPU needed).

The recurrence is latency-bound, so a spill sits on its critical path: every instantiation must keep its stack frame
(k_chain_direct4<8, fast> has carried a 96-byte one since before the write-back was aligned; no other may have one). Eight
one-warp CTAs per SM need the tiles plus at most 1 KB of static shared memory (static_assert in chain_direct4.cuh; the
register file is never the limit, __launch_bounds__(32) caps a thread at 255 registers = 8 warps per SM). The fill must
also keep its L2 prefetch hint: the spectrum rows are read 16 bytes per lane per chunk."""
import os
import re
import shutil
import subprocess

import pytest

# pre-existing frames, not to grow; every other instantiation must have none
STACK_ALLOWED = {(8, True): 96}


def _tool(name):
    nvcc = shutil.which("nvcc")
    tool = os.path.join(os.path.dirname(nvcc), name) if nvcc else shutil.which(name)
    if not tool or not os.path.exists(tool):
        pytest.fail("%s not found next to nvcc" % name)
    return tool


def _res_usage(lib):
    text = subprocess.run([_tool("cuobjdump"), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {}
    for name, fields in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", text):
        usage[name] = dict((k, int(v)) for k, v in re.findall(r"(\w+):(\d+)", fields))
    return usage


def _name(lt, fast):
    return "_ZN5b200s15k_chain_direct4ILi%dELb%dEEEvNS_3CtxE" % (lt, int(fast))


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("lt", range(1, 9))  # every L the kernel is instantiated for: 3 / 4 are presetCheaper / presetDefault at 48 kHz
def test_stereo_chain_keeps_its_stack_frame_and_fits_eight_ctas(cuda_lib, lt, fast):
    u = _res_usage(cuda_lib).get(_name(lt, fast))
    assert u is not None, _name(lt, fast)
    assert u["STACK"] <= STACK_ALLOWED.get((lt, fast), 0), u
    assert u["LOCAL"] == 0, u
    assert u["SHARED"] <= 1024, u  # the static part the static_assert on Chain4Tiles budgets for


def test_stereo_chain_fill_prefetches_into_l2(cuda_lib):
    sass = subprocess.run([_tool("cuobjdump"), "-sass", cuda_lib], capture_output=True, text=True, check=True).stdout
    body = sass[sass.index("Function : " + _name(4, True)):]
    body = body[:body.find("Function : ", 1)] if body.find("Function : ", 1) > 0 else body
    copies = re.findall(r"LDGSTS\S*", body)
    assert copies, "no cp.async in k_chain_direct4"
    assert any("LTC256B" in c for c in copies), sorted(set(copies))
