"""Dev tool (GPU): per-kernel-class device time of one KKT step (factor + 3 solves with refinement).

    python tools/fine_breakdown.py C5 [C3 C4r ...]     # workloads of bench.WORKLOADS

Uses cb200_set_detail(h, 2): CUDA events around every launch group, graph replay off, so the sum is
a little above the bench's ms_per_step; the SHARES are what to read.  One table per workload, also
written as JSON to $FINE_OUT/fine_<workload>.json when FINE_OUT names a directory."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import bench  # noqa: E402
import clarabel_jl_b200 as cb  # noqa: E402
from clarabel_jl_b200 import problems  # noqa: E402


def run(name, nsteps=3):
    P, q, A, b, K = bench.make_problem(name)
    solver = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    ks = solver.kktsystem.kktsolver
    rec = bench.Recorder(ks)
    solver.solve(max_iter=int(os.environ.get("CB200_FINE_ITERS", "3")))
    rec.detach()
    replay = [s for s in rec.steps[1:] if len(s["rhs"]) == 3] or rec.steps[-1:]
    lx, lz = np.zeros(solver.data.n), np.zeros(solver.data.m)

    def step(i):
        s = replay[i % len(replay)]
        ks.update(bench.FakeCones(s["state"]))
        for rx, rz in s["rhs"]:
            ks.setrhs(rx, rz); ks.solve(lx, lz)

    ks.ldl.set_resident(True)
    ks.ldl.set_detail(2)
    step(0)
    ks.ldl.reset_timers()
    for i in range(nsteps):
        step(i)
    fine = ks.ldl.fine_timers(); tm = ks.ldl.timers()
    ks.ldl.set_detail(0); ks.ldl.set_resident(False)
    per = {k: v / nsteps for k, v in fine.items() if v > 0}
    tot = sum(per.values())
    st = ks.ldl.stats()
    print(f"   [stats] tma={int(st.get('use_tma', -1))} kmajor={int(st.get('tma_kmajor', -1))} ordering={int(st.get('ordering_used', -1))}")
    print(f"== {name}: N={ks.KKT.shape[0]} nnzL={int(st['nnzL'])} levels={int(st['nlevels'])} supernodes={int(st['nsuper'])} "
          f"| per step: factor {tm['factor_ms'] / nsteps:.2f} ms, solves {tm['solve_ms'] / nsteps:.2f} ms "
          f"({tm['nsolve'] / nsteps:.1f} sweeps), spmv {tm['spmv_ms'] / nsteps:.2f} ms, launches {tm['nlaunch'] / nsteps:.0f}")
    for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
        print(f"   {k:24s} {v:9.3f} ms  {100 * v / tot:5.1f} %")
    out = os.environ.get("FINE_OUT")
    if out and os.path.isdir(out):
        json.dump({"workload": name, "ms_per_step": per, "coarse": {k: float(v) / nsteps for k, v in tm.items()},
                   "stats": st}, open(os.path.join(out, f"fine_{name}.json"), "w"), indent=1)


if __name__ == "__main__":
    for w in sys.argv[1:] or ["C5"]:
        run(w)
