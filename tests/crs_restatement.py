"""The rule by which bsfm_run_sfm_crs / bsfm_reprojection_outliers_crs accept or refuse a caller's CRS visibility
(include/bsfm_b200_ba.h; crs_check_kernel in bundler_sfm_b200/csrc/ba_setup.cu), restated in plain Python.

check_crs returns None for a well-formed CRS, else (point, fault): the lowest offending point and, for that point, the
first fault in FAULTS order.  Faults about nvis itself are not tied to a point and come back as (-1, "nvis")."""
import numpy as np

INT_MAX = 2 ** 31 - 1

# fault codes of crs_check_kernel, in the order one point reports them, and the words of the library's message
FAULTS = {
    1: "vis_ptr[0] != 0",
    2: "vis_ptr[num_pts] != nvis",
    3: "vis_ptr outside [0, nvis]",
    4: "vis_ptr decreases",
    5: "camera index outside [0, num_cameras)",
    6: "cameras not strictly ascending",
}


def point_fault(i, vis_ptr, vis_cam, n, m, nvis):
    """the fault code of point i (0 when it is sound)"""
    p0, p1 = int(vis_ptr[i]), int(vis_ptr[i + 1])
    if i == 0 and p0 != 0:
        return 1
    if i == n - 1 and p1 != nvis:
        return 2
    if p0 < 0 or p1 > nvis:
        return 3
    if p1 < p0:
        return 4
    cams = [int(c) for c in vis_cam[p0:p1]]
    if any(c < 0 or c >= m for c in cams):
        return 5
    if any(b <= a for a, b in zip(cams, cams[1:])):
        return 6
    return 0


def check_crs(vis_ptr, vis_cam, nvis, n, m):
    """None when (vis_ptr, vis_cam, nvis) is a well-formed CRS of n points and m cameras, else (point, fault code)"""
    if nvis < 0 or nvis > INT_MAX // 2:       # the solver counts 2 * nvis measurements in an int
        return (-1, "nvis")
    vis_ptr = np.asarray(vis_ptr, dtype=np.int64)
    vis_cam = np.asarray(vis_cam, dtype=np.int64)
    assert len(vis_ptr) == n + 1
    for i in range(n):
        f = point_fault(i, vis_ptr, vis_cam, n, m, nvis)
        if f:
            return (i, f)
    return None
