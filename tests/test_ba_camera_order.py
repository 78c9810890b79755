"""Camera order of large reduced camera systems (ba_order.cu: bsfm_ba_camera_order; applied by schur_final_kernel and
backsub_kernel).

CPU: the library's order and scores equal the restatement of tests/camera_order_restatement.py; what it chooses on the
config-3 camera graph, on graphs that are already banded and on block-diagonal ones; the permutation, determinism and fixed
cameras.  GPU: the trailing update's executed FLOPs equal the symbolic prediction for the chosen order; solves with the
order equal solves without it (BSFM_BA_CAMERA_ORDER=0) up to rounding, bit for bit where the natural order is kept, and the
exported S is the caller's order either way."""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from bundler_sfm_b200 import bundle, synth
from bundler_sfm_b200._lib import load_library
from tests import camera_order_restatement as R
from tests.chol_exact_systems import executed_flops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C3_OFFSETS = [166 * t for t in range(1, 6)]      # synth.ba_scene(1000, 500000, 6): step 166, every ring start is used


def lib_order(keys, m, mcon, cnp):
    lib = load_library()
    fn = lib.bsfm_ba_camera_order
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    keys = np.ascontiguousarray(keys, np.uint32)
    pos = np.full(m - mcon, -1, np.int32)
    scores = np.zeros(2, np.int64)
    rc = fn(m, mcon, cnp, keys.ctypes.data, len(keys), pos.ctypes.data, scores.ctypes.data)
    assert rc >= 0, lib.bsfm_last_error()
    return rc, pos, int(scores[0]), int(scores[1])


def band_keys(m, width, mcon=0):
    keys = {j * m + k for j in range(mcon, m) for k in range(j, min(m, j + width + 1))}
    return np.array(sorted(keys), np.uint32)


def block_diagonal_keys(m, size):
    keys = {j * m + k for j in range(m) for k in range(j, min(m, (j // size + 1) * size))}
    return np.array(sorted(keys), np.uint32)


def random_keys(m, edges, seed, mcon=0):
    rng = np.random.default_rng(seed)
    a, b = rng.integers(mcon, m, edges), rng.integers(mcon, m, edges)
    keys = {int(min(x, y)) * m + int(max(x, y)) for x, y in zip(a, b)} | {j * m + j for j in range(mcon, m)}
    return np.array(sorted(keys), np.uint32)


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["config3", "ring250_cnp9", "ring250_cnp7", "ring250_mcon3", "random300", "two_rings"])
def test_library_order_equals_restatement(case):
    m, mcon, cnp = {"config3": (1000, 0, 9), "ring250_cnp9": (250, 0, 9), "ring250_cnp7": (250, 0, 7),
                    "ring250_mcon3": (250, 3, 9), "random300": (300, 0, 9), "two_rings": (400, 0, 8)}[case]
    if case == "config3":
        keys = R.circulant_block_keys(m, C3_OFFSETS)
    elif case == "random300":
        keys = random_keys(m, 900, seed=3)
    elif case == "two_rings":      # two components
        a = R.circulant_block_keys(200, [33, 66, 99])
        keys = np.array(sorted(set(int(k // 200) * m + int(k % 200) for k in a) |
                               set((int(k // 200) + 200) * m + int(k % 200) + 200 for k in a)), np.uint32)
    else:
        keys = R.circulant_block_keys(m, [41 * t for t in range(1, 6)])
        keys = keys[(keys // m) >= mcon]
    rc, pos, s_nat, s_rcm = lib_order(keys, m, mcon, cnp)
    chosen, pos_ref, s_nat_ref, s_rcm_ref = R.camera_order(keys, m, mcon, cnp)
    assert (rc, s_nat, s_rcm) == (chosen, s_nat_ref, s_rcm_ref)
    assert np.array_equal(pos, pos_ref)


def test_config3_scores():
    """config 3 (1000 cameras, cnp 9, 9000 unknowns): the natural order keeps 46 % of the dense update's tiles, RCM a few per
    panel (the right-hand-side row's among them)"""
    keys = R.circulant_block_keys(1000, C3_OFFSETS)
    rc, pos, s_nat, s_rcm = lib_order(keys, 1000, 0, 9)
    dense = R.dense_tiles(9000)
    assert rc == 1
    assert s_nat == 13415 and 0.45 < s_nat / dense < 0.47
    assert 33 <= s_rcm <= 300


def test_circulant_keys_are_the_strided_ring_scene():
    """circulant_block_keys restates the Schur blocks of synth.ba_scene when every ring start is used"""
    m, L = 60, 6
    scene = synth.ba_scene(m, 3000, L, seed=2)
    pi, cj = np.nonzero(scene["vmask"])
    assert np.array_equal(R.scene_block_keys(pi, cj, m), R.circulant_block_keys(m, [(m // L) * t for t in range(1, L)]))


@pytest.mark.parametrize("keys_fn", [lambda m: band_keys(m, 4), lambda m: block_diagonal_keys(m, 20)], ids=["banded", "block_diagonal"])
def test_natural_order_kept_where_it_is_already_good(keys_fn):
    m = 300
    keys = keys_fn(m)
    rc, pos, s_nat, s_rcm = lib_order(keys, m, 0, 9)
    assert rc == 0 and np.array_equal(pos, np.arange(m))
    assert s_nat > 0 and 4 * s_rcm > 3 * s_nat


def test_small_systems_keep_the_natural_order_unscored():
    m = 170      # 170 x 9 = 1530 <= 1536: the small paths
    rc, pos, s_nat, s_rcm = lib_order(R.circulant_block_keys(m, [28 * t for t in range(1, 6)]), m, 0, 9)
    assert (rc, s_nat, s_rcm) == (0, 0, 0) and np.array_equal(pos, np.arange(m))


def test_order_is_a_deterministic_permutation_of_the_free_cameras():
    m, mcon = 400, 5
    keys = random_keys(m, 1500, seed=11, mcon=mcon)
    first = lib_order(keys, m, mcon, 9)
    assert first[0] == 1
    assert np.array_equal(np.sort(first[1]), np.arange(m - mcon))
    for _ in range(3):
        again = lib_order(keys, m, mcon, 9)
        assert again[0] == first[0] and again[2:] == first[2:] and np.array_equal(again[1], first[1])
    # blocks of fixed cameras (j < mcon) are not part of the graph: adding them changes nothing
    extra = np.array(sorted(set(keys.tolist()) | {j * m + k for j in range(mcon) for k in range(j, m, 7)}), np.uint32)
    other = lib_order(extra, m, mcon, 9)
    assert other[0] == first[0] and other[2:] == first[2:] and np.array_equal(other[1], first[1])


def test_bad_arguments_are_refused():
    lib = load_library()
    pos = np.zeros(10, np.int32)
    scores = np.zeros(2, np.int64)
    bad = np.array([5 * 10 + 3], np.uint32)      # j > k
    fn = lib.bsfm_ba_camera_order
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    assert fn(10, 0, 9, bad.ctypes.data, 1, pos.ctypes.data, scores.ctypes.data) < 0
    assert fn(10, 10, 9, bad.ctypes.data, 0, pos.ctypes.data, scores.ctypes.data) < 0


# ---- GPU ------------------------------------------------------------------------------------------------------------
def relabel_cameras(scene, pos):
    """the same scene with camera j renumbered pos[j] (visibility, projections in point-major / ascending-camera order, and
    the per-camera arrays)"""
    pos = np.asarray(pos)
    inv = np.argsort(pos)
    pi, cj = np.nonzero(scene["vmask"])
    nj = pos[cj]
    order = np.lexsort((nj, pi))
    out = dict(scene)
    vm = np.zeros_like(scene["vmask"])
    vm[pi, nj] = 1
    out["vmask"] = vm
    out["projections"] = np.ascontiguousarray(scene["projections"][order])
    for key in ("R", "c", "f", "k"):
        out[key] = scene[key][inv].copy()
    return out


def _scene(case):
    """(scene, run_sfm keywords) of a large-path case"""
    if case == "ring200_cnp9":      # the 200-camera scene test_ba_gpu.py solves against the oracle
        return synth.ba_scene(200, 6000, 6, seed=5), {}
    if case.startswith("ring250"):
        scene = synth.ba_scene(250, 6000, 6, seed=250)
        kw = {"undistort": 0} if case == "ring250_cnp7" else {}
        if case == "ring250_constrained":
            m = 250
            rng = np.random.default_rng(5)
            constrained = np.zeros((m, 9), np.int8)
            constrained[::4, :3] = 1
            constraints = np.zeros((m, 9))
            constraints[:, :3] = scene["c"] + 0.01 * rng.standard_normal((m, 3))
            weights = np.zeros((m, 9))
            weights[:, :3] = 2.0
            kw = {"ncons": 3, "use_constraints": 1, "constrained": constrained, "constraints": constraints, "weights": weights}
        if case == "ring250_rcm_labelled":      # cameras already numbered in RCM order: the natural order is kept
            pi, cj = np.nonzero(scene["vmask"])
            adj = R.free_graph(R.scene_block_keys(pi, cj, 250), 250, 0)
            order = R.rcm(adj)
            pos = np.empty(250, np.int64)
            pos[order] = np.arange(250)
            scene = relabel_cameras(scene, pos)
        return scene, kw
    if case == "known240":
        scene = synth.ba_scene_known_intrinsics(240, 4000, 5, seed=241, ordinary_fraction=0.25)
        return scene, dict(undistort=0, **synth.ki_kwargs(scene))
    scene = synth.ba_scene_fisheye(180, 4000, 5, seed=183, ordinary_fraction=0.25, known_fraction=0.2)
    return scene, dict(optimize_for_fisheye=1, **synth.fe_kwargs(scene))


def _cnp(kw):
    return 6 + (0 if kw.get("est_focal_length", 1) == 0 else 1) + (0 if kw.get("undistort", 1) == 0 else 2)


_CHILD = ("import sys, numpy as np; sys.path.insert(0, %r); from tests.test_ba_camera_order import _scene; "
          "from bundler_sfm_b200 import bundle; scene, kw = _scene(sys.argv[2]); "
          "out = bundle.run_sfm(scene, export='S' if sys.argv[3] == '1' else False, **kw); "
          "np.savez(sys.argv[1], **{k: np.asarray(out[k]) for k in ('R', 'c', 'f', 'k', 'pts', 'info') + (('S',) if sys.argv[3] == '1' else ())})") % ROOT


def _on_and_off(case, export=False):
    outs = []
    with tempfile.TemporaryDirectory() as td:
        for flag in ("1", "0"):
            f = os.path.join(td, f"{case}_{flag}.npz")
            subprocess.run([sys.executable, "-c", _CHILD, f, case, "1" if export else "0"], check=True, stdout=subprocess.DEVNULL,
                           env=dict(os.environ, BSFM_BA_CAMERA_ORDER=flag))
            outs.append(dict(np.load(f)))
    return outs


def _chosen(case):
    scene, kw = _scene(case)
    m = len(scene["f"])
    mcon = kw.get("ncons", 0)
    pi, cj = np.nonzero(scene["vmask"])
    return R.camera_order(R.scene_block_keys(pi, cj, m, mcon), m, mcon, _cnp(kw))


@pytest.mark.gpu
def test_trailing_update_flops_equal_the_symbolic_prediction():
    """the device's zero flags of every panel, as the trailing update executed them, are those of the symbolic block structure
    of L in the chosen order (the host model of the order and the kernel's keep rule agree)"""
    scene, kw = _scene("ring250_cnp9")
    chosen, pos, s_nat, s_rcm = _chosen("ring250_cnp9")
    assert chosen == 1
    lib = load_library()
    lib.bsfm_ba_chol_profile.argtypes = [ctypes.c_int]
    lib.bsfm_ba_chol_profile_read.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    lib.bsfm_ba_chol_profile(1)
    try:
        out = bundle.run_sfm(scene, **kw)
        ms, launches, fl = (ctypes.c_float * 4)(), (ctypes.c_int * 4)(), ctypes.c_double()
        lib.bsfm_ba_chol_profile_read(ms, launches, ctypes.byref(fl))
    finally:
        lib.bsfm_ba_chol_profile(0)
    adj = R.free_graph(R.scene_block_keys(*np.nonzero(scene["vmask"]), 250), 250, 0)
    n = 250 * 9
    flags = R.slab_flags(R.l_structure(adj, pos), 9)
    per_solve = executed_flops(n, flags)
    panels = len({k1 for k1, _, _ in R.update_launches(n)})
    nfact = launches[1] // panels
    assert nfact >= int(out["info"][9]) >= 1 and launches[1] == nfact * panels
    assert fl.value == nfact * per_solve
    assert per_solve < 0.5 * executed_flops(n, R.slab_flags(R.l_structure(adj, list(range(250))), 9))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ring200_cnp9", "ring250_cnp7", "ring250_constrained", "known240", "fisheye180"])
def test_order_equals_natural_order_up_to_rounding(case):
    """Same LM path: iterations, stop reason and linear systems solved, final error and parameters.  ring250_cnp9 is left out on
    purpose: near its end the damping term falls to ~1e-11 of U's largest diagonal, the gain ratio of one step is +-0.005
    (the step changes the error in its ninth digit), and whether that step is taken is decided by rounding: the ordered
    factorisation takes 26 iterations where the natural one takes 25, and the ordered one with the tail hand-over switched
    off (BSFM_BA_CHOL_TAIL=0, another rounding of the same order) takes 25 again."""
    on, off = _on_and_off(case)
    for q in (5, 6, 9):      # iterations, stop reason, linear systems solved
        assert on["info"][q] == off["info"][q], (case, q, on["info"][q], off["info"][q])
    # the reordered elimination rounds differently; how far that carries to the solution depends on the conditioning of the
    # scene.  Measured: ~1e-15 (RMSE) and ~1e-9 (parameters) on the cnp-7, constrained, calibrated and fisheye scenes, but
    # 6e-9 and 1.7e-5 on the cnp-9 ring, whose focal lengths and distortion are nearly degenerate with depth: there the
    # parameters are held to the project's 1e-4 (PARAM_TOL of test_ba_gpu.py), with the same LM path
    rmse_tol, par_tol = (1e-7, 1e-4) if case == "ring200_cnp9" else (1e-9, 1e-6)
    assert abs(np.sqrt(on["info"][1]) - np.sqrt(off["info"][1])) <= rmse_tol * np.sqrt(off["info"][1])
    for key in ("R", "c", "f", "pts"):
        assert np.max(np.abs(on[key] - off[key])) <= par_tol * np.max(np.abs(off[key])), (case, key)
    assert np.max(np.abs(on["k"] - off["k"])) * 5.0 <= par_tol * max(1.0, 5.0 * np.max(np.abs(off["k"])))


@pytest.mark.gpu
def test_natural_order_kept_is_bit_identical():
    chosen = _chosen("ring250_rcm_labelled")[0]
    assert chosen == 0
    on, off = _on_and_off("ring250_rcm_labelled")
    for key in on:
        assert np.array_equal(on[key], off[key]), key


def export_S_at_start(case):
    """bsfm_sba_motstr_levmar_model with itmax = 0 and Sout: the undamped S at the initial parameters, which do not depend on
    the order the solves would factor S in"""
    scene, kw = _scene(case)
    m, n = len(scene["f"]), scene["pts"].shape[0]
    p, cnp = bundle.pack_params(scene)
    vmask = np.ascontiguousarray(scene["vmask"], np.int8)
    x = np.ascontiguousarray(scene["projections"], np.float64)
    R_init = np.ascontiguousarray(scene["R"], np.float64)
    f_fixed = np.ascontiguousarray(scene["f"], np.float64)
    lib = load_library()
    fn = lib.bsfm_sba_motstr_levmar_model
    c = ctypes
    fn.argtypes = [c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int,
                   c.c_void_p, c.c_int, c.c_int, c.c_int, c.c_void_p, c.c_void_p, c.c_int, c.c_void_p, c.c_int, c.c_void_p,
                   c.c_void_p, c.c_void_p, c.c_void_p, c.c_void_p]
    fn.restype = c.c_int
    model = bundle.SfmModel(1, 1, 1, 0.001, 5.0, R_init.ctypes.data, f_fixed.ctypes.data)
    opts = np.array([1.0e-3, 1.0e-10, 1e-12, 1.0e-12, 0.0, 4.0e-2])
    info = np.zeros(10)
    S = np.zeros((m * cnp, m * cnp))
    rc = fn(n, m, 0, vmask.ctypes.data, p.ctypes.data, cnp, 3, x.ctypes.data, None, 2, ctypes.addressof(model), 0, 0, 0,
            opts.ctypes.data, info.ctypes.data, 0, None, 0, None, None, S.ctypes.data, None, None)
    assert rc >= 0, lib.bsfm_last_error()
    return S


@pytest.mark.gpu
def test_exported_S_is_in_the_callers_camera_order():
    """S goes out in the caller's camera order: byte for byte what the natural order exports at the same parameters, and
    within rounding of it at the end of the two solves (whose parameters agree to ~1e-6)"""
    assert _chosen("ring200_cnp9")[0] == 1
    code = ("import sys, numpy as np; sys.path.insert(0, %r); from tests.test_ba_camera_order import export_S_at_start; "
            "np.save(sys.argv[1], export_S_at_start('ring200_cnp9'))") % ROOT
    with tempfile.TemporaryDirectory() as td:
        start = []
        for flag in ("1", "0"):
            f = os.path.join(td, f"S{flag}.npy")
            subprocess.run([sys.executable, "-c", code, f], check=True, stdout=subprocess.DEVNULL, env=dict(os.environ, BSFM_BA_CAMERA_ORDER=flag))
            start.append(np.load(f))
    assert np.any(start[0] != 0) and start[0].tobytes() == start[1].tobytes()
    on, off = _on_and_off("ring200_cnp9", export=True)
    assert np.max(np.abs(on["S"] - off["S"])) <= 1e-5 * np.max(np.abs(off["S"]))
