"""Dev tool: run whole IP solves through the b200 backend and print per-phase device times."""
import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys, time; sys.path.insert(0, ROOT)
import numpy as np
import clarabel_jl_b200 as cb
from clarabel_jl_b200 import problems as pr
GEN = {"C1": pr.c1_random_qp, "C2": pr.c2_portfolio, "C2s": lambda: pr.c2_portfolio(n=20000),
       "C3": pr.c3_socp, "C3s": lambda: pr.c3_socp(n=100000, ncones=2000),
       "C4s": lambda: pr.c4_sdp(ncones=20, side=30, n=3000, vars_per_cone=200),
       "C4": pr.c4_sdp,
       "C5": pr.c5_block_angular, "C5h": lambda: pr.c5_block_angular(nblocks=32),
       "C5s": lambda: pr.c5_block_angular(nblocks=8, grid=60, nlink=100, link_nnz=32)}
def run(name, cpu=False):
    t=time.time(); P,q,A,b,K = GEN[name](); tg=time.time()-t
    t=time.time(); s = cb.Solver(P,q,A,b,K,cb.Settings(direct_solve_method="b200")); ts=time.time()-t
    ks = s.kktsystem.kktsolver
    info = ks.ldl.info()
    ks.ldl.reset_timers()
    t=time.time(); sol = s.solve(); tv=time.time()-t
    tm = ks.ldl.timers(); T = s.timers
    nf, nsv = max(1,tm["nfactor"]), max(1,tm["nsolve"])
    print(f"{name}: n={A.shape[1]} m={A.shape[0]} N={ks.KKT.shape[0]} nnzK={ks.KKT.nnz} nnzL={info.nnzL} gen={tg:.1f}s setup={ts:.1f}s(kkt init {T['kkt init']:.1f}) "
          f"solve={tv:.2f}s status={sol.status_name} it={sol.iterations} obj={sol.obj_val:.8g}")
    print(f"    host sections: kkt_update={T['kkt update']:.3f}s kkt_solve={T['kkt solve']:.3f}s scale={T['scale cones']:.3f}s | device: cone={tm['cone_ms']/nf:.3f}ms/f factor={tm['factor_ms']/nf:.3f}ms/f "
          f"trisolve={tm['solve_ms']/nsv:.3f}ms/solve spmv={tm['spmv_ms']/nsv:.3f}ms nfactor={tm['nfactor']} nsolve={tm['nsolve']} IR={ks.ir_rounds}/{ks.n_solves} launches={tm['nlaunch']}")
    it = max(1, sol.iterations)
    print(f"    IP-iterations/sec (kkt update + kkt solve sections) = {it/(T['kkt update']+T['kkt solve']):.2f}")
    if cpu:
        from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
        cb.register_kktsolver("qdldl", OracleDirectLDLKKTSolver)
        s2 = cb.Solver(P,q,A,b,K,cb.Settings(direct_solve_method="qdldl")); so = s2.solve(); T2=s2.timers
        print(f"    CPU oracle: status={so.status_name} it={so.iterations} obj={so.obj_val:.8g} kkt_update={T2['kkt update']:.3f}s kkt_solve={T2['kkt solve']:.3f}s -> {so.iterations/(T2['kkt update']+T2['kkt solve']):.2f} it/s")
for a in sys.argv[1:]:
    cpu = a.endswith("+cpu"); run(a.replace("+cpu",""), cpu)
