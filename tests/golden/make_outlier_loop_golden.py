"""Writes tests/golden/outlier_loop_golden.npz: the loop of BundlerApp::RunSFM_SBA (tests/outlier_loop_restatement.py)
over the UNMODIFIED reference -- run_sfm of oracle/_ref/libref_sba.so for the solve, oracle/outlier_oracle.py (the
reference's sfm_project_rd and kth_element_copy) for the outlier pass -- on the scenes of tests/outlier_loop_scenes.py.
Needs oracle/_ref (built by __graft_entry__.build() where the reference sources are present).

    python tests/golden/make_outlier_loop_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import loader, outlier_oracle  # noqa: E402
from tests import outlier_loop_restatement as rs  # noqa: E402
from tests import outlier_loop_scenes as scenes  # noqa: E402

# rounds every scene is built to take (None: no round count is part of the scene's purpose)
EXPECT_ROUNDS = {"three_rounds": 3, "stops_small": 1, "too_few": 1, "protected_quirk": 2, "empty_on_entry": 2, "fix_points": 2, "kermit": 1}


def reference_loop(scene, kw):
    """the restatement's loop with the reference behind both callables"""
    loop_kw, solve_kw, outl_kw = scenes.split_kw(kw)

    def solve(round_scene, pc):
        return loader.run_sfm_ref(rs.dense_scene(round_scene), points_constraints=pc, **solve_kw)

    def outlier_pass(round_scene, prot):
        return outlier_oracle.reprojection_outliers(rs.dense_scene(round_scene), pt_protected=prot, **outl_kw)

    return rs.run_loop(scene, solve, outlier_pass, **loop_kw)


def flatten(name, ref):
    out = {f"{name}_{k}": ref[k] for k in ("R", "c", "f", "k", "pts", "pt_round", "pt_error", "cam_stats")}
    out[f"{name}_count"] = np.int64(ref["count"])
    out[f"{name}_mean_error"] = np.float64(ref["mean_error"])
    out[f"{name}_info"] = np.array([r["info"] for r in ref["rounds"]]).reshape(-1, 10)
    out[f"{name}_sizes"] = np.array([[r["num_pts"], r["nvis"], r["num_outliers"]] for r in ref["rounds"]], np.int64).reshape(-1, 3)
    out[f"{name}_global_mean"] = np.array([r["global_mean"] for r in ref["rounds"]])
    return out


if __name__ == "__main__":
    assert loader.ref_sba() is not None, "oracle/_ref/libref_sba.so is not built"
    gold = {}
    for name, make in scenes.GOLDEN.items():
        scene, kw = make()
        ref = reference_loop(scene, kw)
        print(name, "rounds", ref["count"], "outliers per round", [r["num_outliers"] for r in ref["rounds"]],
              "iterations", [int(r["info"][5]) for r in ref["rounds"]], "stop", [int(r["info"][6]) for r in ref["rounds"]], flush=True)
        assert EXPECT_ROUNDS[name] == ref["count"], (name, ref["count"])
        gold.update(flatten(name, ref))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "outlier_loop_golden.npz"), **gold)
