"""Where the time of the large dense Cholesky goes with and without the camera order (ba_order.cu), on config 3 of bench.py
(synth.ba_scene(1000, 500000, 6), seed 1234).  Each order runs in its own child process (BSFM_BA_CAMERA_ORDER is read once
per process): `warmup` untimed solves, then `rounds` solves with the per-phase events (BSFM_BA_TIMING) and the per-kernel-class
events of the large Cholesky (bsfm_ba_chol_profile: diagonal blocks, look-ahead side stream included; panel solves; trailing
updates; back substitution).  Reports per solve: phases, kernel classes, launches, executed trailing-update FLOPs, LM
iterations, stop reason and nlss, and the host time of the order itself (bsfm_ba_camera_order on the scene's Schur blocks).
With the order, config 3's system is banded and takes the one-launch band factorisation (ba_chol_dataflow.cu: its launch
counts as "diag_block", its back substitution as "back_substitution", no panel solve or update runs; "path" says which);
without it the envelope is too wide and the panel path runs, so the two children show the two paths side by side.
Needs the GPU; prints the GPU name and power limit of the run (nvidia-smi, read-only).

usage: python scripts/bench_camera_order.py [--rounds 3] [--warmup 1]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BA3 = dict(num_cameras=1000, num_points=500000, views_per_point=6)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def schur_keys(vmask, views):
    """block keys j * m + k (j <= k) of a visibility mask whose points all have `views` observations"""
    n, m = vmask.shape
    cams = np.nonzero(vmask)[1].reshape(n, views).astype(np.int64)
    a, b = np.triu_indices(views)
    return np.unique(cams[:, a] * m + cams[:, b]).astype(np.uint32)


def order_host_ms(lib, keys, m, cnp, reps=20):
    fn = lib.bsfm_ba_camera_order
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    pos, scores = np.zeros(m, np.int32), np.zeros(2, np.int64)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        rc = fn(m, 0, cnp, keys.ctypes.data, len(keys), pos.ctypes.data, scores.ctypes.data)
        times.append(1e3 * (time.perf_counter() - t0))
    return {"rcm_taken": rc, "kept_tiles_natural": int(scores[0]), "kept_tiles_rcm": int(scores[1]),
            "host_ms_median": float(np.median(times)), "host_ms_min": float(min(times))}


def child(rounds, warmup):
    os.environ["BSFM_BA_TIMING"] = "1"
    os.environ.setdefault("BSFM_BA_VERBOSE", "0")
    from bundler_sfm_b200 import bundle, synth
    lib = bundle.load_library()
    lib.bsfm_ba_chol_profile.argtypes = [ctypes.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    scene = synth.ba_scene(seed=1234, **BA3)
    saved = os.dup(1)
    devnull = os.open(os.devnull, os.O_WRONLY)
    os.dup2(devnull, 1)        # the solver's reference-compatible prints
    try:
        for _ in range(warmup):
            bundle.run_sfm(scene)
        phases, classes, launches, flops, infos = [], [], [], [], []
        for _ in range(rounds):
            lib.bsfm_ba_chol_profile(1)
            out = bundle.run_sfm(scene)
            ms, ln, fl = (ctypes.c_float * 4)(), (ctypes.c_int * 4)(), ctypes.c_double()
            lib.bsfm_ba_chol_profile_read(ms, ln, ctypes.byref(fl))
            lib.bsfm_ba_chol_profile(0)
            phases.append(bundle.last_timing())
            classes.append(list(ms)); launches.append(list(ln)); flops.append(fl.value); infos.append(out["info"])
    finally:
        sys.stdout.flush()
        os.dup2(saved, 1)
        os.close(saved); os.close(devnull)
    names = ["diag_block", "panel_solve", "trailing_update", "back_substitution"]
    med = np.median(np.asarray(classes), axis=0)
    res = {
        "camera_order": os.environ.get("BSFM_BA_CAMERA_ORDER", "1"),
        "path": "band" if launches[-1][1] == 0 and launches[-1][2] == 0 else "panels",
        "iterations": int(infos[-1][5]), "stop": int(infos[-1][6]), "nlss": int(infos[-1][9]),
        "phase_ms_median": {k: float(np.median([p[k] for p in phases])) for k in phases[0] if k.endswith("_ms")},
        "cholesky_class_ms_median": dict(zip(names, map(float, med))),
        "cholesky_class_ms_all": [dict(zip(names, (round(x, 2) for x in c))) for c in classes],
        "launches": dict(zip(names, launches[-1])),
        "trailing_update_gflop": flops[-1] / 1e9,
        "order": order_host_ms(lib, schur_keys(scene["vmask"], BA3["views_per_point"]), BA3["num_cameras"], 9),
    }
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        return child(args.rounds, args.warmup)
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for flag in ("1", "0"):
        subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--rounds", str(args.rounds), "--warmup", str(args.warmup)],
                       check=True, env=dict(os.environ, BSFM_BA_CAMERA_ORDER=flag))


if __name__ == "__main__":
    main()
