"""CPU: static evidence from the built library's SASS (cuobjdump ships with the toolkit).

  * the dense-front GEMM is TMA-fed (UTMALDG = cp.async.bulk.tensor) through an mbarrier ring
    (SYNCS.*) and computes on the FP64 tensor-core path (DMMA);
  * the latency-critical kernels contain no `WARPSYNC.COLLECTIVE` beyond the slow-path landing pads of
    __syncwarp(): a __shfl_sync inside a loop / branch the compiler cannot prove warp-uniform is
    wrapped in WARPSYNC.COLLECTIVE ... ENDCOLLECTIVE and costs tens of cycles per shuffle."""
import os
import re
import shutil
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "clarabel.jl_b200", "libclarabel_b200.so")


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


def _kernel(funcs, name):
    hits = [k for k in funcs if name in k]
    assert hits, f"{name} not in the library"
    return [op for k in hits for op in funcs[k]]


def _dmma_units(ops):
    """FP64 tensor-core work in units of one m8n8k4 MMA: sm_90a issues mma.m16n8k16.f64 as a single
    DMMA.16x8x16 (8 units), other targets as several DMMA.8x8x4."""
    units = 0
    for o in ops:
        m = re.match(r"DMMA\.(\d+)x(\d+)x(\d+)", o)
        if m:
            units += int(m.group(1)) * int(m.group(2)) * int(m.group(3)) // 256
        elif o.startswith("DMMA"):
            units += 1
    return units


def test_dense_front_gemm_is_tma_fed_dmma(sass):
    ops = _kernel(sass, "k_ldl_update_tma")
    assert any(o.startswith("UTMALDG") for o in ops)                 # cp.async.bulk.tensor.3d
    assert any(o.startswith("SYNCS.ARRIVE.TRANS64") for o in ops)    # mbarrier expect_tx / arrive
    assert any("TRYWAIT" in o for o in ops)                          # mbarrier try_wait
    assert _dmma_units(ops) >= 64                                    # FP64 tensor-core MMAs
    assert not any(o.startswith("LDG") and False for o in ops)


def test_default_gemm_tile_keeps_its_fragments_in_registers(sass):
    """k_ldl_update_tma<64> (the default tile, 3 CTAs per SM, 128 registers) moves no 64-bit value through
    local memory: a fragment or accumulator spill would cost local-memory traffic on every k-step."""
    ops = _kernel(sass, "k_ldl_update_tmaILi64")
    assert not any(o.startswith(("STL.64", "LDL.64", "LDL.LU.64", "STL.128", "LDL.128", "LDL.LU.128")) for o in ops)


def test_pivot_kernels_use_dmma_or_registers_only(sass):
    assert _dmma_units(_kernel(sass, "k_piv_rows")) >= 8
    assert not any(o.startswith("SHFL") for o in _kernel(sass, "k_piv_diag"))


@pytest.mark.parametrize("name,limit", [
    ("k_piv_diag", 0), ("k_piv_rows", 0), ("k_fwd_warp", 0), ("k_bwd_warp", 6), ("k_fwd_cta", 0),
    ("k_bwd_cta", 8), ("k_big_tri_fwd", 0), ("k_big_tri_bwd", 8), ("k_big_gemvT_bwd", 4),
    ("k_factor_panel", 8), ("k_factor_small", 0), ("k_ldl_update_tma", 0)])
def test_no_collective_shuffles_in_hot_kernels(sass, name, limit):
    """per instantiation: the limit is the number of __syncwarp() landing pads the kernel may have"""
    hits = [k for k in sass if name in k]
    assert hits, f"{name} not in the library"
    for k in hits:
        n = sum(o == "WARPSYNC.COLLECTIVE" for o in sass[k])
        assert n <= limit, f"{k}: {n} WARPSYNC.COLLECTIVE"


def test_tma_gemm_releases_a_stage_only_after_the_next_wait(sass):
    """The consumer warps' mbarrier arrive on the `empty` barrier (SYNCS.ARRIVE...A1T0, lane 0 only) must sit
    directly behind the try-wait of the NEXT stage, before any shared-memory load or DMMA of that stage: every
    DMMA of the released stage has then been issued (they cannot sink below the spin loop), i.e. every LDS of it
    has completed.  With the arrive at the end of the stage's own iteration ptxas put it behind the last LDS
    issue and ahead of the DMMAs, and now and then a tile was computed from a refilled stage
    (DESIGN.md section 4)."""
    hits = [k for k in sass if "k_ldl_update_tma" in k]
    assert len(hits) >= 2
    for k in hits:
        ops = sass[k]
        idx = [i for i, o in enumerate(ops) if o.startswith("SYNCS.ARRIVE") and o.endswith("A1T0")]
        assert idx, f"{k}: consumer arrive not found"
        for i in idx:
            j = i - 1
            while j >= 0 and "TRYWAIT" not in ops[j]:
                assert not ops[j].startswith(("LDS", "DMMA")), f"{k}: {ops[j]} between the wait and the release"
                j -= 1
            assert j >= 0
