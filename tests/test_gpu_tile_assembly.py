"""Assembly of large fronts from per-tile child rectangles (symbolic.h, build_tile_lists).

One design reaches the cases of the rectangle walk: a Schur tile fed by three children whose rows
interleave, a child whose columns reach a tile whose rows it does not, Schur tiles no child reaches
(they must come out as exactly -L21 D L21'), a root panel tile with 64 children, and a front with
more than MANY_CHILDREN children (assembled atomically and updated in place) in the same batch as a
gather front.  test_tile_lists.py asserts on the CPU that the lists have these shapes; here D and the
panel storage are compared with the extended-precision reference at 1e-12 under the default plan,
the 128 tile and the LDG GEMM."""
import numpy as np
import pytest
import front_zoo as fz
import test_gpu_kernels as tgk
import test_gpu_schur_assembly as tsa


def part_tiles():
    d = tsa.RowDesign("tiles", 23)
    R = d.node(300)                                            # large root, nr = 0: every tile is a panel tile
    P = d.node(70, R, 250)                                     # gather front, U rows 70..319
    for k in range(3):                                         # rows interleaved: 70 + k, 73 + k, ... < 250
        d.node(4, P, sel=np.r_[0, np.arange(70 + k, 250, 3)])
    d.node(5, P, sel=np.r_[0, np.arange(70, 128)])             # reaches column strip 1 but no row below 128
    Q = d.node(64, R, 100)                                     # same level as P, atomic assembly
    d.children(Q, fz.MANY_CHILDREN + 1, 1, [60 + k % 50 for k in range(fz.MANY_CHILDREN + 1)])
    for k in range(64):                                        # 64 children meet in R's first tile
        d.node(2, R, sel=np.r_[0, np.arange(1 + k % 5, 300, 7 + k % 4)])
    return d


PARTS = {d.name: d for d in (part_tiles(),)}


@pytest.mark.gpu
@pytest.mark.parametrize("part", list(PARTS))
@pytest.mark.parametrize("variant", list(tsa.VARIANTS))
def test_factor_parity(monkeypatch, variant, part):
    env = tsa.VARIANTS[variant]
    tgk._set_env(monkeypatch, env)
    R = tgk.reference(PARTS[part], env)
    h = tgk._handle(R["K"], R["sg"])
    assert h.refactor()
    tgk.check_factor(h, R)
    assert h.download(5, 1)[0] == 0
    tgk.check_solves(h, R, PARTS[part])
    st = h.stats()
    assert st["use_tma"] == (0 if env.get("CB200_NO_TMA") == "1" else 1)
    assert st["schur_tiles"] > 0 and st["schur_rects"] > 0 and st["asm_tiles"] > 0 and st["asm_rects"] >= 64
