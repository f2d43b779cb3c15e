"""The wgmma kernels compile to an asynchronous MMA pipeline: no serialized wgmma, no spills, chains not drained per MMA.

Any function call in a kernel that issues wgmma (a device-side printf, assert, or an out-of-line helper) makes ptxas
serialize every wgmma in it, which roughly halves tensor throughput without changing a single result.  This compiles
gemm.cu and attention.cu with the build's flags (nvcc cross-compiles for sm_90a without a GPU) and reads ptxas' report and
the SASS.
"""
import os
import re
import subprocess

import pytest

import __graft_entry__ as ge

KERNELS = ("gemm_bf16_kernel", "flash_attn_fwd_kernel")


@pytest.fixture(scope="module", params=["gemm.cu", "attention.cu"])
def compiled(request, tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("sass") / request.param.replace(".cu", ".o"))
    res = subprocess.run([ge._nvcc(), *ge.NVCC_FLAGS, "-c", os.path.join(ge.CSRC, request.param), "-o", obj],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    return request.param, res.stdout + res.stderr, sass


def test_no_serialized_wgmma(compiled):
    src, ptxas, _ = compiled
    lines = [l for l in ptxas.splitlines() if "wgmma.mma_async instructions are serialized" in l]
    assert not lines, f"{src}: " + "\n".join(lines)


def test_no_spills(compiled):
    src, ptxas, _ = compiled
    entries = re.findall(r"Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", ptxas)
    checked = [e for e in entries if any(k in e[0] for k in KERNELS)]
    assert checked, f"{src}: no wgmma kernel in the ptxas report"
    for name, _, stores, loads in checked:
        assert stores == "0" and loads == "0", f"{src}: {name} spills {stores} B / loads {loads} B"


def test_wgmma_chains_are_not_drained_per_mma(compiled):
    """In a serialized chain every HGMMA is followed by its own WARPGROUP.DEPBAR; in a pipelined one most are followed by
    the next HGMMA of the chain."""
    src, _, sass = compiled
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    checked = 0
    for f in funcs:
        name = f.split("\n", 1)[0].strip()
        if not any(k in name for k in KERNELS):
            continue
        ops = re.findall(r"\b(HGMMA|WARPGROUP\.DEPBAR)\b", f)
        n_mma = ops.count("HGMMA")
        back_to_back = sum(1 for a, b in zip(ops, ops[1:]) if a == b == "HGMMA")
        assert n_mma > 0, f"{src}: {name} has no HGMMA"
        assert 2 * back_to_back >= n_mma, f"{src}: {name}: only {back_to_back} of {n_mma} HGMMAs issue back to back"
        checked += 1
    assert checked, f"{src}: no wgmma kernel in the SASS"
