import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys; sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import clarabel_jl_b200 as cb
from oracle.kktsolver_oracle import OracleDirectLDLKKTSolver
cb.register_kktsolver("qdldl", OracleDirectLDLKKTSolver)
from common import small_instances
P,q,A,b,K = small_instances(cb)["C4m"]()
so_s = cb.Solver(P,q,A,b,K,cb.Settings(direct_solve_method="qdldl")); so=so_s.solve()
sg_s = cb.Solver(P,q,A,b,K,cb.Settings(direct_solve_method="b200")); sg=sg_s.solve()
print(so.status_name, so.iterations, sg.status_name, sg.iterations)
for a,b_ in zip(so_s.iter_log, sg_s.iter_log):
    print("it %d  cpu pc %.10e dc %.10e rp %.3e rd %.3e mu %.3e a %.4f | gpu pc %.10e dc %.10e rp %.3e rd %.3e mu %.3e a %.4f" % (a[0],a[1],a[2],a[3],a[4],a[5],a[6], b_[1],b_[2],b_[3],b_[4],b_[5],b_[6]))
print("cpu IR", so_s.kktsystem.kktsolver.ir_rounds, so_s.kktsystem.kktsolver.n_solves, "reg", so_s.kktsystem.kktsolver.ldl.regularize_count)
g = sg_s.kktsystem.kktsolver
print("gpu IR", g.ir_rounds, g.n_solves, "nreg", g.ldl.download(5,1), g.ldl.timers(), g.ldl.info().nnzL)
