"""Wall time of the solve / outlier-removal loop of RunSFM_SBA, three ways, alternated in one process:
  loop   bsfm_run_sfm_outlier_loop (the scene stays on the GPU between rounds)
  crs    a host loop over bsfm_run_sfm_crs_fe + bsfm_reprojection_outliers_crs_fe + numpy compaction
  dense  the same host loop over the dense entries, building the n x m mask every round as RunSFM_SBA does
Scenes: config 2 (50 cameras / 20k points) and config 3 (1000 / 500k / 3M observations) with injected outliers.
2 warm-ups, then median and range of 5 runs; host-to-device bytes per round from the library's count (loop) and from
shapes (host loops).  Prints one JSON line per scene with the card's name and power limit.  Needs a GPU.

    python scripts/bench_outlier_loop.py [--config 2|3|both] [--runs 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bundler_sfm_b200 import bundle, synth  # noqa: E402
from tests import outlier_loop_restatement as rs  # noqa: E402

CONFIGS = {2: (50, 20000, 5, 400), 3: (1000, 500000, 6, 4000)}      # cameras, points, views per point, injected outliers
KW = {"min_outliers": 40}


def host_loop(scene, dense):
    def solve(s, pc):
        return bundle.run_sfm(rs.dense_scene(s) if dense else s, optimize_for_fisheye=0)

    def outlier_pass(s, prot):
        return bundle.reprojection_outliers(rs.dense_scene(s) if dense else s, optimize_for_fisheye=0)

    return rs.run_loop(scene, solve, outlier_pass, **KW)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="both")
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    os.environ.setdefault("BSFM_BA_VERBOSE", "0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for cfg in ([2, 3] if a.config == "both" else [int(a.config)]):
        m, n, L, bad = CONFIGS[cfg]
        scene, _ = synth.inject_outliers(synth.crs_scene(synth.ba_scene(m, n, L, seed=1234)), bad, seed=99)
        legs = {"loop": lambda: bundle.run_sfm_outlier_loop(scene, **KW), "crs": lambda: host_loop(scene, False),
                "dense": lambda: host_loop(scene, True)}
        times = {k: [] for k in legs}
        last = {}
        devnull = os.open(os.devnull, os.O_WRONLY)
        saved = os.dup(1)
        sys.stdout.flush()
        os.dup2(devnull, 1)              # the per-iteration prints of the reference's run_sfm
        try:
            for rep in range(2 + a.runs):
                for name, leg in legs.items():
                    t0 = time.perf_counter()
                    last[name] = leg()       # every entry ends in a device synchronisation
                    if rep >= 2:
                        times[name].append(time.perf_counter() - t0)
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
        rounds = last["loop"]["rounds"]
        assert last["loop"]["count"] == last["crs"]["count"] == last["dense"]["count"]
        assert last["loop"]["pts"].tobytes() == last["crs"]["pts"].tobytes() == last["dense"]["pts"].tobytes()
        cam = 8 * m * 9
        h2d = {"loop": [r["h2d_bytes"] for r in rounds],
               # per round: solve (CRS or mask, projections, parameters) + pass (the same visibility and projections, points)
               "crs": [2 * (4 * (r["num_pts"] + 1) + 4 * r["nvis"] + 16 * r["nvis"]) + 2 * 24 * r["num_pts"] + cam for r in rounds],
               "dense": [2 * (r["num_pts"] * m + 16 * r["nvis"]) + 2 * 24 * r["num_pts"] + cam for r in rounds]}
        print(json.dumps({"config": cfg, "card": card, "rounds": len(rounds), "outliers": [r["num_outliers"] for r in rounds],
                          "seconds": {k: {"median": float(np.median(v)), "min": min(v), "max": max(v)} for k, v in times.items()},
                          "h2d_bytes_per_round": h2d}), flush=True)


if __name__ == "__main__":
    main()
