"""CPU check of orderings on a late-iteration SDP KKT matrix: AMD vs ND vs ND with cone blocks kept
whole, through the numpy multifrontal emulation and the QDLDL oracle (same permutation)."""
import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys; sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import clarabel_jl_b200 as cb
from clarabel_jl_b200 import lib
from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
from oracle import qdldl as oq
cb.register_kktsolver("qdldl", OracleDirectLDLKKTSolver)
from common import small_instances
from mf_numpy import MFNumpy
name = sys.argv[1] if len(sys.argv) > 1 else "C4m"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 10
P,q,A,b,K = small_instances(cb)[name]()
s = cb.Solver(P,q,A,b,K,cb.Settings(direct_solve_method="qdldl")); s.solve(max_iter=iters)
ks = s.kktsystem.kktsolver
s.cones.update_scaling(s.variables.s, s.variables.z, s.info.mu)
ks.update(s.cones)
Kd = ks.KKT.copy()
eps = ks.diagonal_regularizer
Kd.data[ks.map.diag_full] += np.where(ks.Dsigns==1, eps, -eps)
N = Kd.shape[0]
bid = lib.cone_block_ids(s.cones, s.data.n, N)
print("eps", eps, "qdldl(AMD 1.5) nreg", ks.ldl.regularize_count, "blocks", None if bid is None else int(bid.max())+1)
for label, kw in (("AMD", dict(ordering=0)), ("ND plain", dict(ordering=1, nd_leaf=96)), ("ND + blocks", dict(ordering=1, nd_leaf=96, block_id=bid))):
    S = lib.Symbolic(Kd, **kw); a = S.arrays()
    mf = MFNumpy(a)
    with np.errstate(all="ignore"):
        D = mf.factor(Kd.data, ks.Dsigns)
    F = oq.QDLDLFactorisation(Kd, ks.Dsigns, perm=a["perm"]); F.refactor()
    print(f"{label:12s} levels={S.stats['nlevels']:4d} nnzL={S.stats['nnzL']:.3e} flops={S.stats['flops']:.3e} max_front={S.stats['max_front']} | MF nreg={mf.nreg} min|D|={np.nanmin(np.abs(D)):.3e} | qdldl same perm nreg={F.regularize_count}")
