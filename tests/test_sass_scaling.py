"""CPU: static evidence from the built library's SASS for the cone-scaling kernels (kernels_scaling.cuh): no
local-memory traffic (STL / LDL: a spill or a dynamically indexed register array) and no WARPSYNC.COLLECTIVE (a
shuffle or warp barrier the compiler cannot prove warp-uniform) in any instantiation."""
import os
import re
import shutil
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "clarabel.jl_b200", "libclarabel_b200.so")
KERNELS = ("k_scale_nn", "k_scale_socILi32", "k_scale_socILi256", "k_scale_psdILb1", "k_scale_psdILb0")


@pytest.fixture(scope="module")
def sass():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=300).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); funcs[cur] = []
        elif cur is not None:
            mm = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", line)
            if mm:
                funcs[cur].append(mm.group(1))
    return funcs


@pytest.mark.parametrize("name", KERNELS)
def test_scaling_kernel_has_no_local_memory_or_collective(sass, name):
    hits = [k for k in sass if name in k]
    assert len(hits) == 1, f"{name}: {hits}"
    ops = sass[hits[0]]
    assert len(ops) > 20
    assert not [o for o in ops if o.startswith(("STL", "LDL"))], name
    assert "WARPSYNC.COLLECTIVE" not in ops, name
