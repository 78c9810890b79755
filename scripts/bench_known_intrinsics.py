"""LM iterations/s of the device-resident solver (bsfm_sba_motstr_levmar_model[_ki], vmask / p / x on the GPU) on the
50-camera / 20k-point / 100k-observation scene of synth.ba_scene, solved once as ordinary focal-only cameras and once
with every camera marked calibrated (known_intrinsics, K_known = diag(f, f, 1), k_known = 0: the same projection, run
by the KI kernels).  Both legs estimate the focal length without the radial step (cnp = 7): with the radial step a
calibrated camera's (f, k1, k2) has an exact null direction, and the two legs would no longer solve the same problem.
The calibrated branch still rounds differently (x_n * f instead of -b * f / z), so the script prints iterations,
function evaluations and linear systems of each leg, and the time per linear system, next to LM iterations/s.  The
legs alternate, and the GPU name and power limit are printed beside the numbers.
    python scripts/bench_known_intrinsics.py [--reps 5] [--itmax 20]"""
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
    scene = synth.ba_scene(50, 20000, 5, seed=1234)
    n, m = scene["vmask"].shape
    p0, cnp = bundle.pack_params(scene, est_focal_length=1, undistort=0)
    K = np.zeros((m, 9)); K[:, 0] = scene["f"]; K[:, 4] = scene["f"]; K[:, 8] = 1.0
    cams = bundle.make_cameras(scene["R"], scene["c"], scene["f"], scene["k"], known=np.ones(m), K_known=K, k_known=np.zeros((m, 5)))
    d_vmask = torch.from_numpy(np.ascontiguousarray(scene["vmask"], np.int8)).cuda()
    d_x = torch.from_numpy(np.ascontiguousarray(scene["projections"]).reshape(-1)).cuda()
    d_p = torch.empty(p0.shape[0], dtype=torch.float64, device="cuda")
    src = torch.from_numpy(p0).cuda()

    def solve(ki):
        d_p.copy_(src)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        its, info = bundle.levmar_model(n, m, d_vmask.data_ptr(), d_p.data_ptr(), d_x.data_ptr(), cnp, scene["R"], scene["f"],
                                        undistort=0, itmax=args.itmax, eps5=0.0, init_params=cams if ki else None)
        torch.cuda.synchronize()
        return its / (time.perf_counter() - t0), info

    for ki in (False, True):        # warm-up: module load, pools, the shapes of both legs
        solve(ki)
    rates = {False: [], True: []}
    work = {}
    for _ in range(args.reps):
        for ki in (False, True):
            r, info = solve(ki)
            rates[ki].append(r)
            work[ki] = (int(info[5]), int(info[7]), int(info[9]))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {gpu}; scene {m} cameras, {n} points, {scene['projections'].shape[0]} observations, {args.itmax} LM iterations per solve")
    for ki, name in ((False, "ordinary cameras  "), (True, "calibrated cameras")):
        v = np.array(rates[ki])
        print(f"{name}: median {np.median(v):8.1f} LM it/s  (min {v.min():.1f}, max {v.max():.1f}, {len(v)} solves; "
              f"iterations, function evaluations, linear systems {work[ki]}; "
              f"{1e3 * work[ki][0] / np.median(v) / work[ki][2]:.3f} ms per linear system)")
    print(f"calibrated / ordinary: {np.median(rates[True]) / np.median(rates[False]):.4f}")


if __name__ == "__main__":
    main()
