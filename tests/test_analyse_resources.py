"""Resource usage and store path of the paired analysis kernel (k_analyse2), read from the sm_90a build (no GPU needed).

Two 256-thread CTAs per SM cap the kernel at 128 registers, and it must fit them without spilling (a stack frame of
0 bytes). The spectrum leaves the SM as whole rows: the last FFT pass puts the bins back into shared memory in bin order
and one thread bulk-copies the rows to global memory, so the kernel has no per-thread global store."""
import os
import re
import shutil
import subprocess

import pytest


def _tool(name):
    nvcc = shutil.which("nvcc")
    tool = os.path.join(os.path.dirname(nvcc), name) if nvcc else shutil.which(name)
    if not tool or not os.path.exists(tool):
        pytest.fail("%s not found next to nvcc" % name)
    return tool


def _name(kt):
    return "_ZN5b200s10k_analyse2ILi%dELi0EEEvNS_3CtxE" % kt


def _sass(lib, name):
    sass = subprocess.run([_tool("cuobjdump"), "-sass", lib], capture_output=True, text=True, check=True).stdout
    start = sass.index("Function : " + name)
    end = sass.find("Function : ", start + 1)
    return sass[start:end if end > 0 else len(sass)]


@pytest.mark.parametrize("kt", [3072, 2560])
def test_paired_analysis_kernel_does_not_spill(cuda_lib, kt):
    text = subprocess.run([_tool("cuobjdump"), "-res-usage", cuda_lib], capture_output=True, text=True, check=True).stdout
    usage = {n: dict((k, int(v)) for k, v in re.findall(r"(\w+):(\d+)", f))
             for n, f in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", text)}
    u = usage.get(_name(kt))
    assert u is not None, sorted(n for n in usage if "analyse2" in n)
    assert u["STACK"] == 0, u
    assert u["LOCAL"] == 0, u
    assert u["REG"] <= 128, u  # two 256-thread CTAs per SM


@pytest.mark.parametrize("kt", [3072, 2560])
def test_paired_analysis_stores_rows_by_bulk_copy(cuda_lib, kt):
    body = _sass(cuda_lib, _name(kt))
    ops = re.findall(r"\b(UBLKCP\.\w+\.\w+|STG\S*)", body)
    assert "UBLKCP.G.S" in ops, sorted(set(ops))  # cp.async.bulk shared -> global
    assert not [o for o in ops if o.startswith("STG")], sorted(set(ops))
