import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys, time; sys.path.insert(0, ROOT)
import numpy as np
import clarabel_jl_b200 as cb
from clarabel_jl_b200 import lib, problems as pr, kkt_assembly as ka
name = sys.argv[1]
gen = {"C5": pr.c5_block_angular, "C3": pr.c3_socp, "C2": pr.c2_portfolio, "C5q": lambda: pr.c5_block_angular(nblocks=16)}[name]
P,q,A,b,K = gen()
data = cb.problemdata.ProblemData(P,q,A,b,K,cb.Settings()); cones = cb.CompositeCone(data.cones)
KKT, mp = ka.assemble_kkt_matrix(data.P, data.A, cones)
S = lib.Symbolic(KKT, ordering=1, nd_leaf=96); a = S.arrays(); st = S.stats
ns=np.diff(a["sn_first"]); nr=np.diff(a["rows_ptr"]); nf=ns+nr; lev=a["sn_level"]
print(st)
sz = ns.astype(np.int64)*nf
tot = sz.sum()
for lo,hi in ((0,32),(32,160),(160,256),(256,1024),(1024,2048),(2048,10**9)):
    sel=(nf>lo)&(nf<=hi)
    print(f"nf in ({lo},{hi}]: count={sel.sum()} panel share={sz[sel].sum()/tot:.3f} flops share={(ns[sel].astype(float)*nf[sel].astype(float)**2).sum()/ (ns.astype(float)*nf.astype(float)**2).sum():.3f} levels {np.unique(lev[sel])[:3]}..{np.unique(lev[sel])[-3:] if sel.any() else []}")
top = np.argsort(-sz)[:25]
for s in top: print(f"  sn {s}: level {lev[s]} ns={ns[s]} nr={nr[s]} nf={nf[s]} nchildren={len(a['children'][s])}")
print("levels:", np.bincount(lev).tolist())
