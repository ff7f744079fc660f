"""Dev tool (GPU): host against device NT scaling (update_scaling!) on a real iterate.

    python tools/scaling_probe.py C3 C4r C4 C5      # workloads of bench.WORKLOADS (default: all four)

Runs PROBE_ITERS (default 8) IP iterations of a b200 solve with host scaling to reach a realistic (s, z), then
reports per-call medians over PROBE_REPS (default 7) alternating repetitions, with the card name and power limit
read in the same run:
  host_ms            cones.update_scaling (numpy), wall clock;
  device_ms          cb200_update_scaling kernels alone (CUDA events, timer slot 11);
  device_call_ms     B200KKTSolver.update_scaling: upload of s and z, the kernels, the download of the state into
                     the CompositeCone fields (wall clock; every piece ends in a stream synchronise);
  update_upload_ms   kkt update from the host state (export_state, upload, refactor), wall clock;
  update_device_ms   kkt update from the device state (NULL pointers, refactor), wall clock.
host_ms + update_upload_ms is what an iteration pays today, device_call_ms + update_device_ms what it pays with
Settings.b200_device_cone_scaling.  JSON goes to $PROBE_OUT/scaling_<workload>.json when PROBE_OUT names a
directory."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import bench  # noqa: E402
import clarabel_jl_b200 as cb  # noqa: E402

REPS = int(os.environ.get("PROBE_REPS", "7"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def wall(fn):
    t = time.perf_counter(); r = fn(); return (time.perf_counter() - t) * 1e3, r


def run(name):
    P, q, A, b, K = bench.make_problem(name)
    solver = cb.Solver(P, q, A, b, K, cb.Settings(direct_solve_method="b200"))
    solver.solve(max_iter=int(os.environ.get("PROBE_ITERS", "8")))
    ks, cones, v = solver.kktsystem.kktsolver, solver.cones, solver.variables
    s, z, mu = v.s.copy(), v.z.copy(), solver.info.mu
    dev_cones = cb.CompositeCone(solver.data.cones)
    assert cones.update_scaling(s, z, mu) and ks.update_scaling(s, z, dev_cones)      # warm-up of both paths
    ks.update(dev_cones)
    rows = {k: [] for k in ("host_ms", "device_ms", "device_call_ms", "update_upload_ms", "update_device_ms")}
    for _ in range(REPS):
        t, ok = wall(lambda: cones.update_scaling(s, z, mu)); assert ok
        rows["host_ms"].append(t)
        t, ok = wall(lambda: ks.update(cones)); assert ok
        rows["update_upload_ms"].append(t)
        d0 = ks.ldl.timers()["scale_ms"]
        t, ok = wall(lambda: ks.update_scaling(s, z, dev_cones)); assert ok
        rows["device_call_ms"].append(t)
        rows["device_ms"].append(ks.ldl.timers()["scale_ms"] - d0)
        t, ok = wall(lambda: ks.update(dev_cones)); assert ok
        rows["update_device_ms"].append(t)
    st = ks.ldl.stats()
    out = {"workload": name, "card": card(), "m": int(solver.data.m), "nsoc": int(cones.nsoc),
           "npsd": int(sum(len(g["cones"]) for g in cones.psd_groups)), "iterations_before": int(solver.info.iterations),
           "psd_scale_smem": int(st["psd_scale_smem"]), "psd_scale_global": int(st["psd_scale_global"]),
           "jacobi_sweeps": int(st["jacobi_sweeps"])}
    out.update({k: float(np.median(x)) for k, x in rows.items()})
    out["today_ms"] = out["host_ms"] + out["update_upload_ms"]
    out["device_path_ms"] = out["device_call_ms"] + out["update_device_ms"]
    print(f"== {name} on {out['card']}: m={out['m']} SOC={out['nsoc']} PSD={out['npsd']} "
          f"(Jacobi sweeps {out['jacobi_sweeps']})")
    print(f"   host scaling {out['host_ms']:.3f} ms | device kernels {out['device_ms']:.3f} ms, "
          f"device call + download {out['device_call_ms']:.3f} ms")
    print(f"   kkt update with upload {out['update_upload_ms']:.3f} ms, from device state {out['update_device_ms']:.3f} ms")
    print(f"   scaling + update: host path {out['today_ms']:.3f} ms, device path {out['device_path_ms']:.3f} ms")
    d = os.environ.get("PROBE_OUT")
    if d and os.path.isdir(d):
        json.dump(out, open(os.path.join(d, f"scaling_{name}.json"), "w"), indent=1)
    return out


if __name__ == "__main__":
    for w in sys.argv[1:] or ["C3", "C4r", "C4", "C5"]:
        run(w)
