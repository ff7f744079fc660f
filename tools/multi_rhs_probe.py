"""Dev tool (GPU): what the multi-right-hand-side entry points save on one recorded KKT step.

    python tools/multi_rhs_probe.py C5 [C3 C4r ...]     # workloads of bench.WORKLOADS

Records a GPU solve with bench.Recorder, takes the last step with three right-hand sides and reports, with
the card name and power limit read in the same run:
  1. device time of the triangular sweeps (timer 2) of one k-column cb200_solve_multi against k calls of
     cb200_solve, k = 1, 2, 4 (alternating repetitions, medians);
  2. the batched step - update, solve_ir_multi on [constant, affine], solve_ir on the combined system -
     against the bench-style step of update + 3 x solve_ir, resident mode, CUDA events (medians).  This is
     the per-iteration gain a loop that batches the two independent solves (SURVEY.md H4) would get;
  3. whether the batched step's solutions and refinement rounds are bitwise equal to the three single solves.
JSON goes to $PROBE_OUT/multi_rhs_<workload>.json when PROBE_OUT names a directory."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import bench  # noqa: E402
import clarabel_jl_b200 as cb  # noqa: E402

REPS = int(os.environ.get("PROBE_REPS", "7"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run(name):
    P, q, A, b, K = bench.make_problem(name)
    solver = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    ks = solver.kktsystem.kktsolver
    rec = bench.Recorder(ks)
    solver.solve(max_iter=int(os.environ.get("PROBE_ITERS", "4")))
    rec.detach()
    step = [s for s in rec.steps if len(s["rhs"]) == 3][-1]
    ldl, N, n, m = ks.ldl, ks.KKT.shape[0], solver.data.n, solver.data.m
    ks.update(bench.FakeCones(step["state"]))
    out = {"workload": name, "card": card(), "N": N, "nnzL": int(ldl.stats()["nnzL"])}

    # 1. sweep device time, k columns batched vs k single solves
    rng = np.random.default_rng(0)
    sweeps = {}
    for k in (1, 2, 4):
        B = np.asfortranarray(rng.standard_normal((N, k)))
        X = np.zeros_like(B); x = np.zeros(N)
        ldl.solve_multi(X, B); ldl.solve(x, np.ascontiguousarray(B[:, 0]))       # warm-up (graph capture)
        tm, ts = [], []
        for _ in range(REPS):
            ldl.reset_timers(); ldl.solve_multi(X, B); tm.append(ldl.timers()["solve_ms"])
            ldl.reset_timers()
            for j in range(k):
                ldl.solve(x, np.ascontiguousarray(B[:, j]))
            ts.append(ldl.timers()["solve_ms"])
        sweeps[k] = {"multi_ms": float(np.median(tm)), "singles_ms": float(np.median(ts))}
    out["sweeps"] = sweeps
    out["sweep_ratio_2_vs_1"] = sweeps[2]["multi_ms"] / sweeps[1]["multi_ms"]
    out["sweep_ratio_4_vs_1"] = sweeps[4]["multi_ms"] / sweeps[1]["multi_ms"]

    # 2. + 3. batched step vs bench-style step, resident mode
    (cx, cz), (ax, az), (mx, mz) = step["rhs"]
    dev = lambda v: torch.tensor(np.ascontiguousarray(v), device="cuda")
    t_cx, t_cz, t_ax, t_az, t_mx, t_mz = map(dev, (cx, cz, ax, az, mx, mz))
    t_px = torch.stack([t_cx, t_ax]); t_pz = torch.stack([t_cz, t_az])     # C-order 2 x n == column-major n x 2
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(ldl.stream_ptr())
    cones = bench.FakeCones(step["state"])
    ldl.set_resident(True)

    def single_solves():
        sols, rounds = [], []
        for px, pz in ((t_cx, t_cz), (t_ax, t_az), (t_mx, t_mz)):
            r0 = ks.ir_rounds
            ks.setrhs_staged(px.data_ptr(), pz.data_ptr()); ks.solve(None, None)
            rounds.append(ks.ir_rounds - r0); sols.append(ldl.download(6, N))
        return sols, rounds

    def batched_solves():
        _, r2 = ks.solve_multi_staged(t_px.data_ptr(), t_pz.data_ptr(), 2)
        two = ldl.download(8, 2 * N).reshape(2, N)
        r0 = ks.ir_rounds
        ks.setrhs_staged(t_mx.data_ptr(), t_mz.data_ptr()); ks.solve(None, None)
        return [two[0], two[1], ldl.download(6, N)], [int(r2[0]), int(r2[1]), ks.ir_rounds - r0]

    def single_step():
        ks.update(cones); single_solves()

    def batched_step():
        ks.update(cones); batched_solves()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); fn(); e1.record(stream); e1.synchronize()
        return e0.elapsed_time(e1)

    single_step(); batched_step()
    ts, tb = [], []
    for _ in range(REPS):
        ts.append(timed(single_step)); tb.append(timed(batched_step))
    ks.update(cones)                          # one factorisation for both, so only the solves are compared
    s_sol, s_r = single_solves(); b_sol, b_r = batched_solves()
    ks.update(cones)                          # does a second factorisation of the same values repeat the first?
    out["refactor_bitwise_repeatable"] = bool(all(np.array_equal(u, v) for u, v in zip(single_solves()[0], s_sol)))
    ldl.set_resident(False)
    out["step_single_ms"] = float(np.median(ts)); out["step_batched_ms"] = float(np.median(tb))
    out["bitwise_equal_per_solution"] = [bool(np.array_equal(u, v)) for u, v in zip(s_sol, b_sol)]
    out["bitwise_equal"] = bool(all(out["bitwise_equal_per_solution"]) and s_r == b_r)
    out["ir_rounds"] = s_r
    print(f"== {name} on {out['card']}: N={N} nnzL={out['nnzL']}")
    for k, v in sweeps.items():
        print(f"   sweeps k={k}: multi {v['multi_ms']:.3f} ms   {k} x single {v['singles_ms']:.3f} ms")
    print(f"   2-column / 1-column sweep: {out['sweep_ratio_2_vs_1']:.3f}   4 / 1: {out['sweep_ratio_4_vs_1']:.3f}")
    print(f"   step: update + 3 x solve_ir {out['step_single_ms']:.3f} ms, batched {out['step_batched_ms']:.3f} ms"
          f"   bitwise equal: {out['bitwise_equal_per_solution']}  rounds {s_r} / {b_r}"
          f"   (refactor repeatable: {out['refactor_bitwise_repeatable']})")
    d = os.environ.get("PROBE_OUT")
    if d and os.path.isdir(d):
        json.dump(out, open(os.path.join(d, f"multi_rhs_{name}.json"), "w"), indent=1)
    return out


if __name__ == "__main__":
    for w in sys.argv[1:] or ["C5"]:
        run(w)
