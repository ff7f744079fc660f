import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys, time; sys.path.insert(0, ROOT)
import numpy as np
import clarabel_jl_b200 as cb
from clarabel_jl_b200 import lib, problems as pr, kkt_assembly as ka
def stats(name, gen, orderings=((0,0),(1,96))):
    t=time.time(); P,q,A,b,K = gen(); tg=time.time()-t
    data = cb.problemdata.ProblemData(P,q,A,b,K,cb.Settings()); cones = cb.CompositeCone(data.cones)
    KKT, mp = ka.assemble_kkt_matrix(data.P, data.A, cones)
    for ordn, leaf in orderings:
        t=time.time(); S = lib.Symbolic(KKT, ordering=ordn, nd_leaf=leaf); ts=time.time()-t
        st = S.stats
        a = S.arrays()
        ns=np.diff(a["sn_first"]); nr=np.diff(a["rows_ptr"]); nf=ns+nr
        lv=np.bincount(a["sn_level"])
        big = nf>160
        print(f"{name} ord={ordn} leaf={leaf}: N={st['N']} nnzK={st['nnzK']} nsuper={st['nsuper']} nnzL={st['nnzL']:.3e} flops={st['flops']:.3e} levels={st['nlevels']} max_front={st['max_front']} max_width={st['max_width']} upd={st['upd_total']*8/1e9:.2f}GB panel={st['panel_total']*8/1e9:.2f}GB large_fronts={big.sum()} flops_in_large={float(((ns[big].astype(float))*(nf[big].astype(float))**2).sum()):.3e} gen={tg:.1f}s sym={ts:.1f}s")
        print("    nf hist", np.histogram(nf,bins=[0,8,16,32,64,96,128,160,256,512,1024,1e9])[0].tolist(), "level sizes", lv[:8].tolist(), "...", lv[-6:].tolist())
w = sys.argv[1:]
if "C1" in w: stats("C1", pr.c1_random_qp)
if "C2" in w: stats("C2", pr.c2_portfolio, orderings=((1,96),))
if "C3" in w: stats("C3", pr.c3_socp)
if "C5" in w: stats("C5", pr.c5_block_angular, orderings=((0,0),))
if "C4" in w: stats("C4", pr.c4_sdp, orderings=((0,0),))
