"""dev: time and check bsfm_sba_Axb_Chol on random SPD systems (run on the GPU box).
usage: python scripts/dev_chol.py [sizes...]"""
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bundler_sfm_b200 import _lib


def spd(n, seed, spread=3.0):
    rng = np.random.default_rng(seed)
    k = max(8, n // 4)
    G = rng.standard_normal((n, k))
    S = G @ G.T / k
    S += np.eye(n) * 1e-3 * np.trace(S) / n
    d = 10.0 ** rng.uniform(-spread, spread, n)        # row/column scales spanning 10^(2 spread)
    S = S * d[:, None] * d[None, :]
    return (S + S.T) * 0.5


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [450, 1547, 2048, 4500, 9000]
    lib = _lib.load_library()
    fn = lib.bsfm_sba_Axb_Chol_timed
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    fn.restype = ctypes.c_int
    for n in sizes:
        A = spd(n, seed=n)
        rng = np.random.default_rng(1)
        xt = rng.standard_normal(n)
        b = A @ xt
        x = np.zeros(n)
        ms = ctypes.c_float(0)
        rc = fn(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, 1, ctypes.byref(ms))          # warm-up (allocations, attributes)
        reps = 5 if n >= 4000 else 20
        rc = fn(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, reps, ctypes.byref(ms))
        if n > 1536:
            lib.bsfm_ba_chol_profile(1)
            m2 = ctypes.c_float(0)
            fn(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, 3, ctypes.byref(m2))
            pms = (ctypes.c_float * 4)(); pl = (ctypes.c_int * 4)(); fl = ctypes.c_double()
            lib.bsfm_ba_chol_profile_read(pms, pl, ctypes.byref(fl))
            lib.bsfm_ba_chol_profile(0)
            print(f"    per solve: diag {pms[0]/3:.3f} ms ({pl[0]//3} launches)  trsm {pms[1]/3:.3f} ms  trailing {pms[2]/3:.3f} ms "
                  f"({fl.value/3/(pms[2]/3*1e-3)/1e12:.1f} TF/s fp64)  backsolve {pms[3]/3:.3f} ms", flush=True)
        dp = (ctypes.c_uint64 * 8)()
        if lib.bsfm_debug_df_prof(dp) == 0 and dp[7]:
            v = list(dp); st = max(v[6], 1)
            print(f"    dataflow CTA0: kernel {v[0]/v[7]/1e3:.1f} us/launch; cycles/step: potf2 {v[1]/st:.0f}  barrier {v[2]/st:.0f}  strips+wait-for-inputs {v[3]/st:.0f}  "
                  f"update {v[4]/st:.0f}  end-barrier {v[5]/st:.0f}  ({v[6]} steps, {v[7]} launches)", flush=True)
        if rc != 1:
            print(f"n={n}: rc={rc} err={lib.bsfm_last_error()}")
            continue
        t0 = time.perf_counter()
        xr = np.linalg.solve(A, b)
        tcpu = time.perf_counter() - t0
        res = np.linalg.norm(A @ x - b) / (np.linalg.norm(A, 2 if n <= 2048 else 'fro') * np.linalg.norm(x))
        res_ref = np.linalg.norm(A @ xr - b) / (np.linalg.norm(A, 2 if n <= 2048 else 'fro') * np.linalg.norm(xr))
        err = np.linalg.norm(x - xr) / np.linalg.norm(xr)
        errt = np.linalg.norm(x - xt) / np.linalg.norm(xt)
        errt_ref = np.linalg.norm(xr - xt) / np.linalg.norm(xt)
        tf = (n ** 3 / 3.0 + 2.0 * n * n) / (ms.value * 1e-3) / 1e12
        print(f"n={n}: {ms.value:8.3f} ms  {tf:6.2f} TF/s(fp64-equiv)  resid={res:.2e} (lapack {res_ref:.2e})  |x-x_lapack|/|x|={err:.2e}  "
              f"err_vs_truth={errt:.2e} (lapack {errt_ref:.2e})  cpu={tcpu*1e3:.0f} ms", flush=True)


if __name__ == "__main__":
    main()
