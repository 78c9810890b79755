"""Band plan of large reduced camera systems (ba_order.cu: bsfm_ba_chol_band_plan), CPU only: the library's envelope, tile
count, largest live set and verdict equal the restatement of tests/chol_band_restatement.py."""
import ctypes

import numpy as np
import pytest

from bundler_sfm_b200._lib import load_library
from tests import camera_order_restatement as R
from tests import chol_band_restatement as B

C3_OFFSETS = [166 * t for t in range(1, 6)]      # synth.ba_scene(1000, 500000, 6), as in tests/test_ba_camera_order.py
H100_WORKERS = 131                               # 132 SMs, one of them the diagonal chain


def lib_plan(first, workers):
    lib = load_library()
    fn = lib.bsfm_ba_chol_band_plan
    fn.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    first = np.ascontiguousarray(first, np.int32)
    n = len(first)
    env = np.full(-(-n // 32) + 1, -1, np.int32)
    out = np.zeros(3, np.int64)
    rc = fn(n, first.ctypes.data, workers, env.ctypes.data, out.ctypes.data)
    assert rc >= 0, lib.bsfm_last_error()
    return bool(rc), list(env), int(out[0]), int(out[1]), int(out[2])


def config3_first():
    keys = R.circulant_block_keys(1000, C3_OFFSETS)
    chosen, pos, _, _ = R.camera_order(keys, 1000, 0, 9)
    assert chosen == 1
    return B.camera_first_cols(keys, 1000, 0, 9, pos)


def ring_first(m, offsets, cnp=9):
    keys = R.circulant_block_keys(m, offsets)
    return B.camera_first_cols(keys, m, 0, cnp, list(range(m)))


def arrow_first(n, cam=9):
    """every camera coupled to camera 0: every row reaches back to column 0"""
    return np.zeros(n, np.int32)


def blockdiag_first(n, size):
    i = np.arange(n)
    return ((i // size) * size).astype(np.int32)


CASES = {
    "config3_rcm": lambda: config3_first(),
    "ring_natural": lambda: ring_first(300, [1, 2, 3]),               # a ring numbered around: the wrap-around rows reach column 0
    "band_w5": lambda: B.tile_band_first(4100, 5),
    "band_w1": lambda: B.tile_band_first(2000, 1),
    "arrowhead": lambda: arrow_first(3000),
    "blockdiag": lambda: blockdiag_first(4000, 90),
    "jagged": lambda: B.camera_band_first(5003, 12, seed=4),
    "n_not_mult_32": lambda: B.camera_band_first(1537, 3, seed=2),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("workers", [H100_WORKERS, 4])
def test_plan_equals_restatement(case, workers):
    first = CASES[case]()
    got = lib_plan(first, workers)
    want = B.band_plan(first, len(first), workers)
    assert got[0] == want[0] and got[1] == want[1], case
    assert got[2:] == want[2:], case


def test_config3_envelope():
    """config 3 under RCM: 282 block rows reaching at most 5 tiles left of the diagonal (3.2 on average), 1468 envelope tiles
    with the right-hand-side row; fits"""
    first = config3_first()
    fits, env, ntile, max_live, workers = lib_plan(first, H100_WORKERS)
    width = np.arange(282) - np.array(env[:282])
    assert len(env) == 283 and width.max() <= 5 and 3.0 <= width.mean() <= 3.4
    assert ntile == 1468
    assert fits and max_live <= 2 * workers and workers <= H100_WORKERS


def test_wide_envelopes_do_not_fit():
    """an arrowhead's last rows reach column 0: its envelope is the dense triangle, far more tiles than the workspace holds"""
    assert not lib_plan(arrow_first(3000), H100_WORKERS)[0]
    assert not lib_plan(B.tile_band_first(9000, 40), H100_WORKERS)[0]      # 40 tiles wide: more live tiles than 2 x 131
    assert lib_plan(B.tile_band_first(4100, 5), H100_WORKERS)[0]


def test_bad_first_column_is_refused():
    lib = load_library()
    fn = lib.bsfm_ba_chol_band_plan
    fn.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    first = np.arange(100, dtype=np.int32) + 1
    out = np.zeros(3, np.int64)
    assert fn(100, first.ctypes.data, 8, None, out.ctypes.data) < 0
