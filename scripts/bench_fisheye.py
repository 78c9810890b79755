"""Cost of the fisheye projection (optimize_for_fisheye) in the device-resident solver (bsfm_sba_motstr_levmar_model[_fe],
vmask / p / x on the GPU), on the config-2 workload: 50 cameras, 20k points, 100k observations, cnp = 9.  Two legs, which
alternate in this process:
  ordinary  synth.ba_scene(50, 20000, 5) solved with the ordinary projection (bsfm_sba_motstr_levmar_model)
  fisheye   synth.ba_scene_fisheye(50, 20000, 5) with every camera fisheye, solved with optimize_for_fisheye = 1
Each forward-difference Jacobian evaluates the projection 13 times per observation, and the fisheye mapping adds a
square root, an fp64 atan and divisions to each.  Printed per leg: LM iterations/s (untimed phases), the time per
linear system, and the device time of the residual / Jacobian / U, V, W phase per LM iteration (bsfm_ba_last_timing
ms[1], from a separate solve with the phase timers on), with the GPU name and power limit.
    python scripts/bench_fisheye.py [--reps 5] [--itmax 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bundler_sfm_b200 import bundle, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--itmax", type=int, default=20)
    args = ap.parse_args()
    import torch
    legs = {}
    for name, scene in (("ordinary", synth.ba_scene(50, 20000, 5, seed=1234)),
                        ("fisheye", synth.ba_scene_fisheye(50, 20000, 5, seed=1234, ordinary_fraction=0.0))):
        n, m = scene["vmask"].shape
        p0, cnp = bundle.pack_params(scene)
        cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], **synth.fe_kwargs(scene))
        legs[name] = dict(scene=scene, n=n, m=m, cnp=cnp, cams=cams,
                          d_vmask=torch.from_numpy(np.ascontiguousarray(scene["vmask"], np.int8)).cuda(),
                          d_x=torch.from_numpy(np.ascontiguousarray(scene["projections"]).reshape(-1)).cuda(),
                          src=torch.from_numpy(p0).cuda(), d_p=torch.empty(p0.shape[0], dtype=torch.float64, device="cuda"))

    def solve(name):
        L = legs[name]
        L["d_p"].copy_(L["src"])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fe = {"init_params": L["cams"], "optimize_for_fisheye": 1} if name == "fisheye" else {}
        its, info = bundle.levmar_model(L["n"], L["m"], L["d_vmask"].data_ptr(), L["d_p"].data_ptr(), L["d_x"].data_ptr(), L["cnp"],
                                        L["scene"]["R"], L["scene"]["f"], itmax=args.itmax, eps5=0.0, **fe)
        torch.cuda.synchronize()
        return its / (time.perf_counter() - t0), info

    for name in legs:               # warm-up: module load, pools, the shapes of both legs
        solve(name)
    rates = {name: [] for name in legs}
    work, jac_ms = {}, {name: [] for name in legs}
    for _ in range(args.reps):
        for name in legs:
            r, info = solve(name)
            rates[name].append(r)
            work[name] = (int(info[5]), int(info[7]), int(info[9]))
    os.environ["BSFM_BA_TIMING"] = "1"      # phase timers on: separate solves, not in the rates above
    for _ in range(args.reps):
        for name in legs:
            solve(name)
            t = bundle.last_timing()
            jac_ms[name].append(t["jacobian_uvw_ms"] / max(t["iterations"], 1))
    del os.environ["BSFM_BA_TIMING"]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    L = legs["ordinary"]
    print(f"GPU: {gpu}; scene {L['m']} cameras, {L['n']} points, {L['scene']['projections'].shape[0]} observations, cnp {L['cnp']}, "
          f"{args.itmax} LM iterations per solve")
    for name in legs:
        v = np.array(rates[name])
        print(f"{name:9s}: median {np.median(v):8.1f} LM it/s  (min {v.min():.1f}, max {v.max():.1f}, {len(v)} solves; "
              f"iterations, function evaluations, linear systems {work[name]}; "
              f"{1e3 * work[name][0] / np.median(v) / work[name][2]:.3f} ms per linear system; "
              f"residual/Jacobian/UVW phase {np.median(jac_ms[name]):.3f} ms per iteration)")
    print(f"fisheye / ordinary LM it/s: {np.median(rates['fisheye']) / np.median(rates['ordinary']):.4f}; "
          f"Jacobian phase: {np.median(jac_ms['fisheye']) / np.median(jac_ms['ordinary']):.3f}x")


if __name__ == "__main__":
    main()
