"""Writes tests/golden/chol_sparse_golden.npz: the solutions x of bsfm_sba_Axb_Chol on the seeded block-sparse SPD
systems of tests/chol_sparse_systems.py (one array per case).  It was run on an H100 with the build from before the
large Cholesky skipped all-zero panel blocks, so test_chol_sparse_gpu.py checks that the skip changes no bit.
usage (from the repository root, after build()): python tests/golden/make_chol_sparse_golden.py"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bundler_sfm_b200 import _lib  # noqa: E402
from tests.chol_sparse_systems import CASES, case_system  # noqa: E402


def main():
    lib = _lib.load_library()
    fn = lib.bsfm_sba_Axb_Chol
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    fn.restype = ctypes.c_int
    out = {}
    for name, _, n in CASES:
        A, b = case_system(name)
        x = np.zeros(n)
        rc = fn(A.ctypes.data, b.ctypes.data, x.ctypes.data, n, 0)
        assert rc == 1, (name, rc)
        out[name] = x
        print(f"{name}: n={n} |x|={np.linalg.norm(x):.6e}", flush=True)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "chol_sparse_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
