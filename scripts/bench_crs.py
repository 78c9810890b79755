"""Dense mask vs CRS visibility, end to end: bsfm_run_sfm against bsfm_run_sfm_crs on the BA configurations of bench.py
(config 2: synth.ba_scene(50, 20000, 5), config 3: synth.ba_scene(1000, 500000, 6), seed 1234), with every bulk input in
pinned host memory for both legs.  The legs alternate in one process; for each the script reports the wall time of the
C call, the setup phase of bsfm_ba_last_timing (ms[0]: H2D copies, visibility, Schur structure) and the H2D bytes
computed from shapes, and it asserts that both legs return the same bits.  Needs the GPU; prints the GPU name and power
limit of the run (nvidia-smi, read-only).

usage: python scripts/bench_crs.py [--configs ba2,ba3] [--rounds 5] [--warmup 2]"""
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

CONFIGS = {"ba2": dict(num_cameras=50, num_points=20000, views_per_point=5),
           "ba3": dict(num_cameras=1000, num_points=500000, views_per_point=6)}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


class Leg:
    """one run_sfm-shaped call with its arguments bound once; cameras and points are restored before every call"""

    def __init__(self, torch, bundle, scene, cnp=9):
        def pinned(a):
            t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
            self.keep.append(t)
            return t.numpy()
        self.keep = []
        self.crs = "vis_ptr" in scene
        vis = {k: pinned(scene[k]) for k in (("vis_ptr", "vis_cam") if self.crs else ("vmask",))}
        sc = dict(scene, projections=pinned(scene["projections"]), **vis)
        self.name = "bsfm_run_sfm_crs" if self.crs else "bsfm_run_sfm"
        n, m, vis_args, keep = bundle._visibility_args(sc)
        self.keep += keep
        self.cams = bundle.make_cameras(sc["R"], sc["c"], sc["f"], sc["k"])
        self.cams0 = bytes(self.cams)
        self.pts = pinned(sc["pts"])
        self.pts0 = self.pts.copy()
        self.info = np.zeros(10)
        nvis = sc["projections"].shape[0]
        self.args = [n, m, 0, *vis_args, sc["projections"].ctypes.data, 1, 0, 1, 1, ctypes.addressof(self.cams),
                     self.pts.ctypes.data, 0, 0, None, 0.0, 0, 0, 1e-12, None, None, None, None, self.info.ctypes.data]
        params = 8 * (m * cnp + 3 * n) + 8 * 9 * m + 8 * m          # p, R_init, f_fixed
        self.vis_bytes = (4 * (n + 1) + 4 * nvis) if self.crs else n * m
        self.h2d = self.vis_bytes + 16 * nvis + params

    def __call__(self, fn, lib):
        ctypes.memmove(ctypes.addressof(self.cams), self.cams0, len(self.cams0))
        self.pts[:] = self.pts0
        t0 = time.perf_counter()
        rc = fn(*self.args)
        wall = time.perf_counter() - t0
        assert rc == 0, (self.name, rc, lib.bsfm_last_error())
        ms = (ctypes.c_float * 6)()
        it, ln = ctypes.c_int(), ctypes.c_int()
        lib.bsfm_ba_last_timing(ms, ctypes.byref(it), ctypes.byref(ln))
        out = (self.info.copy(), bytes(self.cams), self.pts.copy())
        return wall, float(ms[0]), float(ms[5]), it.value, ln.value, out


def stats(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}


def run_config(key, rounds, warmup, torch, bundle, synth):
    scene = synth.ba_scene(seed=1234, **CONFIGS[key])
    crs = synth.crs_scene(scene)
    legs = {"dense": Leg(torch, bundle, scene), "crs": Leg(torch, bundle, crs)}
    del scene, crs
    lib = bundle.load_library()
    fns = {}
    for k, leg in legs.items():        # the prototypes bundle.run_sfm binds
        fn = getattr(lib, leg.name)
        bundle._bind_run_sfm(fn)
        if leg.crs:
            fn.argtypes = fn.argtypes[:3] + [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + fn.argtypes[4:]
        fn.argtypes = fn.argtypes + [ctypes.c_void_p]
        fn.restype = ctypes.c_int
        fns[k] = fn
    res = {k: {"wall_ms": [], "setup_ms": [], "device_ms": [], "iterations": [], "launches": []} for k in legs}
    ref = None
    for r in range(warmup + rounds):
        for k in (("dense", "crs") if r % 2 == 0 else ("crs", "dense")):
            wall, setup, total, its, launches, out = legs[k](fns[k], lib)
            if ref is None:
                ref = out
            assert np.array_equal(out[0], ref[0]) and out[1] == ref[1] and np.array_equal(out[2], ref[2]), (key, k, "outputs differ")
            if r >= warmup:
                res[k]["wall_ms"].append(1e3 * wall); res[k]["setup_ms"].append(setup); res[k]["device_ms"].append(total)
                res[k]["iterations"].append(its); res[k]["launches"].append(launches)
    summary = {"config": key, **CONFIGS[key], "rounds": rounds, "outputs_bitwise_equal": True}
    for k, leg in legs.items():
        d = res[k]
        summary[k] = {"wall_ms": stats(d["wall_ms"]), "setup_ms": stats(d["setup_ms"]), "device_ms": stats(d["device_ms"]),
                      "iterations": sorted(set(d["iterations"])), "launches": sorted(set(d["launches"])),
                      "h2d_bytes": leg.h2d, "visibility_bytes": leg.vis_bytes,
                      "wall_ms_all": [round(x, 2) for x in d["wall_ms"]], "setup_ms_all": [round(x, 2) for x in d["setup_ms"]]}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="ba2,ba3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    os.environ["BSFM_BA_TIMING"] = "1"        # per-phase CUDA events, for ms[0] of bsfm_ba_last_timing
    os.environ.setdefault("BSFM_BA_VERBOSE", "0")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_crs.py needs a CUDA device")
    from bundler_sfm_b200 import bundle, synth
    print(json.dumps({"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    for key in args.configs.split(","):
        sys.stdout.flush()
        saved = os.dup(1)
        devnull = os.open(os.devnull, os.O_WRONLY)
        os.dup2(devnull, 1)            # the solver's reference-compatible prints ("[run_sfm] Number of iterations", ...)
        try:
            summary = run_config(key, args.rounds, args.warmup, torch, bundle, synth)
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved); os.close(devnull)
        print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
