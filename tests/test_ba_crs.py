"""Sparse (CRS) visibility: bsfm_run_sfm_crs and bsfm_reprojection_outliers_crs (include/bsfm_b200_ba.h).

CPU: synth.crs_scene against np.nonzero, and the acceptance rule (tests/crs_restatement.py) on hand-made arrays.
GPU: the _crs entries on synth.crs_scene of a scene against the dense entries on the scene itself, bit for bit (one
visibility builder serves both, ba_setup.cu); host, pinned and device CRS pointers; malformed arrays refused with the
point the restatement names."""
import re

import numpy as np
import pytest

from bundler_sfm_b200 import _lib, bundle, synth
from tests import crs_restatement as rs

SOLVE_KEYS = ("rc", "info", "R", "c", "f", "k", "pts")


def ragged_mask(n, m, density, seed, empty_rows=(), empty_cols=()):
    rng = np.random.default_rng(seed)
    vmask = (rng.random((n, m)) < density).astype(np.int8)
    vmask[list(empty_rows), :] = 0
    vmask[:, list(empty_cols)] = 0
    return vmask


# ------------------------------------------------------------------------------------------------
# CPU: crs_scene and the restatement
# ------------------------------------------------------------------------------------------------
def check_crs_of(scene):
    crs = synth.crs_scene(scene)
    vmask = scene["vmask"]
    n = vmask.shape[0]
    pi, cj = np.nonzero(vmask)
    assert "vmask" not in crs and "vmask" in scene
    assert crs["vis_ptr"].dtype == np.int32 and crs["vis_cam"].dtype == np.int32
    assert np.array_equal(crs["vis_ptr"], np.concatenate([[0], np.cumsum(np.count_nonzero(vmask, axis=1))]))
    assert np.array_equal(crs["vis_cam"], cj)
    assert np.array_equal(np.repeat(np.arange(n), np.diff(crs["vis_ptr"])), pi)
    for k in scene:
        if k != "vmask":
            assert crs[k] is scene[k], k
    assert rs.check_crs(crs["vis_ptr"], crs["vis_cam"], len(crs["vis_cam"]), n, vmask.shape[1]) is None
    pb, cb = bundle.observations(crs)
    assert np.array_equal(pb, pi) and np.array_equal(cb, cj)
    return crs


@pytest.mark.parametrize("make", [
    lambda: synth.ba_scene(10, 500, 4, seed=3),
    lambda: synth.ba_scene(7, 300, 7, seed=5),
    lambda: synth.ba_scene_known_intrinsics(9, 400, 3, seed=8, ordinary_fraction=0.3),
])
def test_crs_scene_of_synthetic_scenes(make):
    check_crs_of(make())


@pytest.mark.parametrize("n,m,density,empty_rows,empty_cols", [
    (50, 1, 0.6, (0, 7, 49), ()),               # one camera, points without observations
    (200, 37, 0.1, (0, 1, 199), (0, 5, 36)),    # m not a power of two, unobserved first / middle / last cameras
    (64, 64, 0.02, (), (63,)),
    (30, 129, 0.5, tuple(range(0, 30, 3)), (64, 128)),
    (5, 3, 0.0, (), ()),                        # no observation at all
    (40, 8, 1.0, (39,), ()),
])
def test_crs_scene_of_ragged_masks(n, m, density, empty_rows, empty_cols):
    vmask = ragged_mask(n, m, density, n * 31 + m, empty_rows, empty_cols)
    vmask[vmask != 0] = np.random.default_rng(1).integers(1, 127, size=int(np.count_nonzero(vmask)))   # any non-zero byte
    crs = check_crs_of({"vmask": vmask, "projections": np.zeros((int(np.count_nonzero(vmask)), 2))})
    assert np.array_equal(np.diff(crs["vis_ptr"])[list(empty_rows)], np.zeros(len(empty_rows)))


# a well-formed CRS of 6 points and 5 cameras, and malformed variants of it: (name, vis_ptr, vis_cam, nvis, expected)
BASE_PTR = [0, 2, 4, 4, 7, 9, 11]
BASE_CAM = [0, 3, 1, 2, 0, 1, 4, 2, 3, 0, 4]
N, M = 6, 5


def variant(ptr=None, cam=None, nvis=None):
    p, c = list(BASE_PTR), list(BASE_CAM)
    for i, v in (ptr or {}).items():
        p[i] = v
    for i, v in (cam or {}).items():
        c[i] = v
    return np.array(p, np.int64), np.array(c, np.int64), len(c) if nvis is None else nvis


MALFORMED = [
    ("nvis_negative", variant(nvis=-1), (-1, "nvis")),
    ("nvis_doubled_overflows_int", variant(nvis=2 ** 30), (-1, "nvis")),
    ("first_ptr_not_zero", variant(ptr={0: 1}), (0, 1)),
    ("last_ptr_not_nvis", variant(ptr={6: 10}), (5, 2)),
    ("ptr_beyond_nvis", variant(ptr={2: 50}), (1, 3)),
    ("ptr_int_max", variant(ptr={1: 2 ** 31 - 1}), (0, 3)),
    ("ptr_decreases", variant(ptr={3: 1}), (2, 4)),
    ("ptr_negative", variant(ptr={2: -3}), (1, 4)),
    ("ptr_int_min", variant(ptr={4: -2 ** 31}), (3, 4)),
    ("camera_negative", variant(cam={5: -1}), (3, 5)),
    ("camera_equals_m", variant(cam={10: 5}), (5, 5)),
    ("camera_huge", variant(cam={0: 2 ** 31 - 1}), (0, 5)),
    ("duplicate_camera", variant(cam={3: 1}), (1, 6)),
    ("descending_cameras", variant(cam={0: 3, 1: 0}), (0, 6)),
    ("range_fault_before_order_fault", variant(cam={4: 4, 5: 1, 6: 9}), (3, 5)),
    ("lowest_point_wins", variant(cam={7: 3, 8: 2, 10: 9}), (4, 6)),
    ("empty_ptr_but_nvis", (np.zeros(N + 1, np.int64), np.zeros(3, np.int64), 3), (5, 2)),
]


def test_restatement_accepts_well_formed_crs():
    assert rs.check_crs(*variant(), N, M) is None
    assert rs.check_crs(np.zeros(N + 1), np.zeros(0), 0, N, M) is None                        # no observation
    assert rs.check_crs([0, 0, 3, 3], [0, 1, 2], 3, 3, 3) is None                              # empty first / last point
    assert rs.check_crs([0, 1], [0], 1, 1, 1) is None                                          # one point, one camera


@pytest.mark.parametrize("name,arrays,want", MALFORMED, ids=[c[0] for c in MALFORMED])
def test_restatement_rejects_malformed_crs(name, arrays, want):
    assert rs.check_crs(*arrays, N, M) == want


def test_restatement_edge_points():
    # n == 1: the first-pointer fault is reported before the last-pointer fault of the same point
    assert rs.check_crs([1, 2], [0, 0], 2, 1, 1) == (0, 1)
    assert rs.check_crs([0, 1], [0, 0], 2, 1, 1) == (0, 2)
    # the largest accepted nvis
    assert rs.check_crs([0, 0], [], 2 ** 30 - 1, 1, 1) == (0, 2)


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_crs_entries_fail_loudly_without_gpu():
    crs = synth.crs_scene(synth.ba_scene(4, 40, 3, seed=2))
    for call in (lambda: bundle.run_sfm(crs), lambda: bundle.reprojection_outliers(crs)):
        with pytest.raises(_lib.BsfmError) as e:
            call()
        assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


# ------------------------------------------------------------------------------------------------
# GPU: dense vs CRS, bit for bit
# ------------------------------------------------------------------------------------------------
def same_solve(a, b, what, export=""):
    for k in SOLVE_KEYS + tuple(export):
        assert np.array_equal(a[k], b[k]), (what, k)


def dense_vs_crs(scene, **kw):
    dense = bundle.run_sfm(scene, **kw)
    crs = bundle.run_sfm(synth.crs_scene(scene), **kw)
    same_solve(dense, crs, kw, kw.get("export", ""))
    return dense


def with_holes(scene, empty_points, empty_cams):
    """the scene with some points and cameras left without observations (their projections dropped)"""
    vmask = scene["vmask"].copy()
    pi, cj = np.nonzero(vmask)
    vmask[list(empty_points), :] = 0
    vmask[:, list(empty_cams)] = 0
    keep = vmask[pi, cj] != 0
    return dict(scene, vmask=vmask, projections=np.ascontiguousarray(scene["projections"][keep]))


@pytest.mark.gpu
@pytest.mark.parametrize("est_focal_length,undistort", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("explicit_camera_centers", [0, 1])
def test_run_sfm_crs_equals_dense_every_camera_model(est_focal_length, undistort, explicit_camera_centers):
    scene = synth.ba_scene(9, 600, 4, seed=21)
    out = dense_vs_crs(scene, est_focal_length=est_focal_length, undistort=undistort,
                       explicit_camera_centers=explicit_camera_centers)
    assert out["rc"] == 0 and out["info"][5] > 0


@pytest.mark.gpu
def test_run_sfm_crs_equals_dense_with_constraints():
    scene = synth.ba_scene(8, 300, 4, seed=9)
    m = len(scene["f"])
    rng = np.random.default_rng(4)
    constrained = (rng.random((m, 9)) < 0.3).astype(np.int8)
    constraints = np.zeros((m, 9))
    constraints[:, 0:3] = scene["gt_c"]
    constraints[:, 6] = scene["gt_f"]
    weights = rng.uniform(0.5, 2.0, (m, 9))
    pc = np.zeros_like(scene["pts"])
    pc[::7] = scene["gt_pts"][::7]
    dense_vs_crs(scene, use_constraints=1, constrained=constrained, constraints=constraints, weights=weights)
    dense_vs_crs(scene, use_point_constraints=1, points_constraints=pc, point_constraint_weight=0.5)
    dense_vs_crs(scene, use_constraints=1, constrained=constrained, constraints=constraints, weights=weights,
                 use_point_constraints=1, points_constraints=pc, point_constraint_weight=0.5)


@pytest.mark.gpu
def test_run_sfm_crs_equals_dense_fixed_cameras_motion_only_export():
    scene = synth.ba_scene(9, 400, 4, seed=12)
    out = dense_vs_crs(scene, ncons=2)
    assert np.array_equal(out["c"][:2], scene["c"][:2])
    out = dense_vs_crs(scene, fix_points=1)
    assert np.array_equal(out["pts"], scene["pts"])
    dense_vs_crs(scene, fix_points=1, est_focal_length=0)
    dense_vs_crs(synth.ba_scene(6, 120, 3, seed=46), export="SUVW")
    dense_vs_crs(synth.ba_scene(3, 80, 3, seed=43), export="S")


@pytest.mark.gpu
def test_run_sfm_crs_equals_dense_calibrated_cameras():
    scene = synth.ba_scene_known_intrinsics(12, 900, 4, seed=17, ordinary_fraction=0.25)
    ki = synth.ki_kwargs(scene)
    dense_vs_crs(scene, **ki)
    dense_vs_crs(scene, fix_points=1, **ki)
    dense = bundle.reprojection_outliers(scene, 1, 2.0, 16.0, **ki)
    crs = bundle.reprojection_outliers(synth.crs_scene(scene), 1, 2.0, 16.0, **ki)
    same_outliers(dense, crs, "calibrated")


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", [("syn10", {}), ("syn6nf", {"est_focal_length": 0, "undistort": 0}),
                                     ("syn8nd", {"est_focal_length": 1, "undistort": 0}), ("kermit", {}), ("kermitc", None)])
def test_run_sfm_crs_equals_dense_golden_cases(name, kw):
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ba_golden.npz"))
    scene = {k: g[f"{name}_{k}"] for k in ("vmask", "projections", "R", "c", "f", "k", "pts")}
    if kw is None:
        kw = dict(use_constraints=1, constrained=g["kermitc_constrained"], constraints=g["kermitc_constraints"],
                  weights=g["kermitc_weights"])
    dense_vs_crs(scene, **kw)


@pytest.mark.gpu
def test_run_sfm_crs_equals_dense_empty_points_and_unobserved_cameras():
    scene = with_holes(synth.ba_scene(12, 800, 5, seed=33), empty_points=(0, 5, 400, 799), empty_cams=(0, 7, 11))
    crs = synth.crs_scene(scene)
    assert np.count_nonzero(np.diff(crs["vis_ptr"]) == 0) == 4
    assert set(range(12)) - set(crs["vis_cam"].tolist()) == {0, 7, 11}
    dense_vs_crs(scene)
    dense_vs_crs(scene, ncons=1)


@pytest.mark.gpu
def test_run_sfm_crs_equals_dense_on_the_large_cholesky_path():
    """240 cameras with cnp = 7: a 1680-unknown reduced camera system, above the 1536 of the small paths"""
    scene = synth.ba_scene(240, 6000, 5, seed=240)
    dense_vs_crs(scene, est_focal_length=1, undistort=0)


@pytest.mark.gpu
def test_empty_visibility_behaves_like_an_empty_mask():
    scene = synth.ba_scene(5, 60, 3, seed=6)
    empty = dict(scene, vmask=np.zeros_like(scene["vmask"]), projections=np.zeros((0, 2)))
    dense = bundle.run_sfm(empty)
    assert "fewer measurements" in _lib.last_error()
    crs = bundle.run_sfm(synth.crs_scene(empty))
    assert "fewer measurements" in _lib.last_error()
    same_solve(dense, crs, "empty")
    assert dense["info"][5] == 0
    for sc in (empty, synth.crs_scene(empty)):
        with pytest.raises(_lib.BsfmError, match="empty visibility"):
            bundle.reprojection_outliers(sc)


# ------------------------------------------------------------------------------------------------
# GPU: the outlier pass
# ------------------------------------------------------------------------------------------------
def same_outliers(a, b, what):
    for k in ("count", "dist", "stats", "outliers", "errors", "global_mean"):
        assert np.array_equal(a[k], b[k], equal_nan=k == "stats"), (what, k)   # an empty camera's mean is NaN


@pytest.mark.gpu
@pytest.mark.parametrize("name", ("kermit_default", "kermit_tight", "syn"))
def test_outliers_crs_equals_dense_golden_cases(name):
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "outlier_golden.npz"))
    scene = {k: g[f"{name}_{k}"] for k in ("vmask", "projections", "R", "c", "f", "k", "pts")}
    lo, hi = g[f"{name}_thresholds"]
    prot = g[f"{name}_protected"] if f"{name}_protected" in g.files else None
    dense = bundle.reprojection_outliers(scene, 1, float(lo), float(hi), prot)
    crs = bundle.reprojection_outliers(synth.crs_scene(scene), 1, float(lo), float(hi), prot)
    same_outliers(dense, crs, name)
    assert np.array_equal(dense["outliers"], g[f"{name}_ref_outliers"])


# ------------------------------------------------------------------------------------------------
# GPU: pointer kinds
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_crs_pointer_kinds_give_the_same_bits():
    import torch
    scene = synth.ba_scene(10, 700, 4, seed=55)
    crs = synth.crs_scene(scene)
    kinds = {"pageable": crs}
    for kind, move in (("pinned", lambda t: t.pin_memory()), ("device", lambda t: t.cuda())):
        kinds[kind] = dict(crs, vis_ptr=move(torch.from_numpy(crs["vis_ptr"])), vis_cam=move(torch.from_numpy(crs["vis_cam"])))
    torch.cuda.synchronize()
    dense = bundle.run_sfm(scene)
    dense_ol = bundle.reprojection_outliers(dict(scene, **{k: dense[k] for k in ("R", "c", "f", "k", "pts")}), 1, 2.0, 16.0)
    for kind, sc in kinds.items():
        same_solve(dense, bundle.run_sfm(sc), kind)
        ol = bundle.reprojection_outliers(dict(sc, **{k: dense[k] for k in ("R", "c", "f", "k", "pts")}), 1, 2.0, 16.0)
        same_outliers(dense_ol, ol, kind)


# ------------------------------------------------------------------------------------------------
# GPU: malformed CRS is refused, naming the point the restatement names
# ------------------------------------------------------------------------------------------------
def malformed_scene(vis_ptr, vis_cam, nvis):
    scene = synth.ba_scene(M, N, 3, seed=70)
    crs = synth.crs_scene(scene)
    crs.update(vis_ptr=np.asarray(vis_ptr, np.int32), vis_cam=np.asarray(vis_cam, np.int32), nvis=nvis,
               projections=np.zeros((max(len(vis_cam), 1), 2)))
    return crs


def check_refusal(err, want):
    msg = str(err)
    assert "failed (-3)" in msg, msg          # BSFM_ERR_ARG
    point, fault = want
    if point < 0:
        assert "nvis = " in msg, msg
    else:
        m = re.search(r"at point (\d+): (.*)$", msg)
        assert m and int(m.group(1)) == point and m.group(2) == rs.FAULTS[fault], (msg, want)


@pytest.mark.gpu
def test_malformed_crs_is_refused_by_both_entries():
    for name, arrays, want in MALFORMED:
        assert rs.check_crs(*arrays, N, M) == want, name
        for entry in (bundle.run_sfm, bundle.reprojection_outliers):
            with pytest.raises(_lib.BsfmError) as e:
                entry(malformed_scene(*arrays))
            check_refusal(e.value, want)
    # the process goes on: a well-formed solve and outlier pass afterwards give the dense results
    scene = synth.ba_scene(8, 500, 4, seed=71)
    dense_vs_crs(scene)
    same_outliers(bundle.reprojection_outliers(scene), bundle.reprojection_outliers(synth.crs_scene(scene)), "after")
