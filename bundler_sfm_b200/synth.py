"""Synthetic workloads of SURVEY.md section 8(d): SIFT-like uint8 descriptors (MATCH, config 4) and
ring-camera bundle-adjustment scenes (BA, configs 2/3).  Deterministic given the seed."""
import numpy as np


def sift_like_descriptors(num_images, keys_per_image, seed=7, copy_frac=0.3, noise=0.08):
    """List of [K,128] uint8 arrays.  gamma(0.6) magnitudes -> L2 normalise -> clip 0.2 -> renormalise
    -> x512 -> floor -> clamp 255.  `copy_frac` of every image's keys are noisy copies of keys of the
    previous image so that true matches exist."""
    rng = np.random.default_rng(seed)
    if np.isscalar(keys_per_image):
        keys_per_image = [int(keys_per_image)] * num_images

    def quantise(f):
        f = f / np.maximum(np.linalg.norm(f, axis=1, keepdims=True), 1e-12)
        f = np.minimum(f, 0.2)
        f = f / np.maximum(np.linalg.norm(f, axis=1, keepdims=True), 1e-12)
        return np.clip(np.floor(f * 512.0), 0, 255).astype(np.uint8)

    out, prev_f = [], None
    for i in range(num_images):
        K = keys_per_image[i]
        f = rng.gamma(0.6, 1.0, size=(K, 128)).astype(np.float32)
        f = f / np.maximum(np.linalg.norm(f, axis=1, keepdims=True), 1e-12)
        if prev_f is not None and K > 0 and prev_f.shape[0] > 0:
            nc = min(int(copy_frac * K), prev_f.shape[0])
            src = rng.choice(prev_f.shape[0], size=nc, replace=False)
            dst = rng.choice(K, size=nc, replace=False)
            f[dst] = np.abs(prev_f[src] + noise * rng.standard_normal((nc, 128)).astype(np.float32) * np.linalg.norm(prev_f[src], axis=1, keepdims=True) / np.sqrt(128.0))
        prev_f = f
        out.append(quantise(f))
    return out


def random_descriptors(n, seed, lo=0, hi=256):
    """uniform uint8 descriptors (adversarial/edge-case tests)"""
    rng = np.random.default_rng(seed)
    return rng.integers(lo, hi, size=(n, 128), dtype=np.int64).astype(np.uint8)


# ------------------------------------------------------------------------------------------------
# BA scenes (SURVEY.md 8d): cameras on a ring of radius 6 looking at the origin (Bundler convention:
# the camera looks down -z, P = R (X - c)), f = 800, k = 0; points uniform in [-1,1]^3; each point is
# seen by L cameras; pixel noise N(0, 0.5^2); perturbed initial estimate.
# ------------------------------------------------------------------------------------------------
def ba_scene(num_cameras=50, num_points=20000, views_per_point=5, seed=1234, pixel_noise=0.5,
             pt_noise=0.02, cam_noise=0.01, f_noise=0.01, focal=800.0):
    """Returns a dict with the arguments of run_sfm (numpy arrays):
    vmask [n,m] int8, projections [nvis,2], R [m,9], c [m,3] (camera centres), f [m], k [m,2], pts [n,3]
    (the perturbed initial estimate) and the ground truth (gt_*)."""
    rng = np.random.default_rng(seed)
    m, n, L = num_cameras, num_points, views_per_point
    ang = 2.0 * np.pi * np.arange(m) / m
    c = np.stack([6.0 * np.cos(ang), 0.3 * np.sin(3 * ang), 6.0 * np.sin(ang)], 1)
    R = np.zeros((m, 3, 3))
    for j in range(m):
        z = c[j] / np.linalg.norm(c[j])          # camera looks down -z => z axis points away from the scene
        up = np.array([0.0, 1.0, 0.0])
        xax = np.cross(up, z); xax /= np.linalg.norm(xax)
        yax = np.cross(z, xax)
        R[j] = np.stack([xax, yax, z], 0)
    pts = rng.uniform(-1.0, 1.0, size=(n, 3))
    vmask = np.zeros((n, m), np.int8)
    step = max(m // L, 1)
    starts = (np.arange(n) * 7) % m
    for k in range(L):
        vmask[np.arange(n), (starts + k * step) % m] = 1
    pi, cj = np.nonzero(vmask)                    # row-major: point-major, ascending camera
    Pc = np.einsum("oij,oj->oi", R[cj], pts[pi] - c[cj])
    proj = -Pc[:, :2] * focal / Pc[:, 2:3]
    proj = proj + pixel_noise * rng.standard_normal(proj.shape)
    scene = {
        "vmask": vmask, "projections": np.ascontiguousarray(proj),
        "gt_pts": pts, "gt_c": c, "gt_R": R.reshape(m, 9).copy(), "gt_f": np.full(m, focal),
        "R": R.reshape(m, 9).copy(),
        "c": c + cam_noise * rng.standard_normal(c.shape),
        "f": focal * (1.0 + f_noise * rng.standard_normal(m)),
        "k": np.zeros((m, 2)),
        "pts": pts + pt_noise * rng.standard_normal(pts.shape),
    }
    return scene


def ba_scene_known_intrinsics(num_cameras=20, num_points=2000, views_per_point=5, seed=4321, ordinary_fraction=0.0,
                              pixel_noise=0.5, pt_noise=0.02, cam_noise=0.01, f_noise=0.01, focal=800.0):
    """A ba_scene whose cameras are calibrated (camera_params_t::known_intrinsics, lib/sfm-driver/sfm.c:339-357).
    Every calibrated camera has its own K_known (focal lengths near `focal`, skew, an off-centre principal point) and
    k_known (radial k0, k1, k4 and tangential k2, k3 all nonzero); its measurements come from that model plus
    N(0, pixel_noise^2).  A seeded `ordinary_fraction` of the cameras stay focal-only pinhole cameras (measured as in
    ba_scene).  Adds known [m] int8, K_known [m,9], k_known [m,5] to the ba_scene dict; "f" is the initial focal
    parameter of every camera (what the radial step and est_focal_length act on).  Use ki_kwargs(scene) to pass the
    calibration to run_sfm and friends."""
    rng = np.random.default_rng(seed)
    m, n, L = num_cameras, num_points, views_per_point
    ang = 2.0 * np.pi * np.arange(m) / m
    c = np.stack([6.0 * np.cos(ang), 0.3 * np.sin(3 * ang), 6.0 * np.sin(ang)], 1)
    R = np.zeros((m, 3, 3))
    for j in range(m):
        z = c[j] / np.linalg.norm(c[j])
        xax = np.cross(np.array([0.0, 1.0, 0.0]), z); xax /= np.linalg.norm(xax)
        R[j] = np.stack([xax, np.cross(z, xax), z], 0)
    known = np.ones(m, np.int8)
    n_ord = int(round(ordinary_fraction * m))
    if n_ord:
        known[rng.choice(m, size=n_ord, replace=False)] = 0
    K_known = np.zeros((m, 3, 3))
    K_known[:, 0, 0] = focal * (1.0 + 0.05 * rng.standard_normal(m))
    K_known[:, 0, 1] = rng.uniform(-3.0, 3.0, m)                 # skew
    K_known[:, 0, 2] = rng.uniform(-25.0, 25.0, m)               # principal point (Bundler's centred pixel frame)
    K_known[:, 1, 1] = K_known[:, 0, 0] * (1.0 + 0.01 * rng.standard_normal(m))
    K_known[:, 1, 2] = rng.uniform(-25.0, 25.0, m)
    K_known[:, 2, 2] = 1.0
    k_known = np.stack([rng.uniform(-0.12, -0.04, m), rng.uniform(0.01, 0.04, m), rng.uniform(-2e-3, 2e-3, m),
                        rng.uniform(-2e-3, 2e-3, m), rng.uniform(-4e-3, 4e-3, m)], 1)
    pts = rng.uniform(-1.0, 1.0, size=(n, 3))
    vmask = np.zeros((n, m), np.int8)
    step = max(m // L, 1)
    starts = (np.arange(n) * 7) % m
    for k in range(L):
        vmask[np.arange(n), (starts + k * step) % m] = 1
    pi, cj = np.nonzero(vmask)
    Pc = np.einsum("oij,oj->oi", R[cj], pts[pi] - c[cj])
    proj = -Pc[:, :2] * focal / Pc[:, 2:3]
    kn = known[cj] != 0
    x_n, y_n = -Pc[kn, 0] / Pc[kn, 2], -Pc[kn, 1] / Pc[kn, 2]
    kk, KK = k_known[cj[kn]], K_known[cj[kn]]
    rsq = x_n * x_n + y_n * y_n
    factor = 1.0 + kk[:, 0] * rsq + kk[:, 1] * rsq ** 2 + kk[:, 4] * rsq ** 3
    x_d = x_n * factor + 2 * kk[:, 2] * x_n * y_n + kk[:, 3] * (rsq + 2 * x_n * x_n)
    y_d = y_n * factor + kk[:, 2] * (rsq + 2 * y_n * y_n) + 2 * kk[:, 3] * x_n * y_n
    proj[kn, 0] = KK[:, 0, 0] * x_d + KK[:, 0, 1] * y_d + KK[:, 0, 2]
    proj[kn, 1] = KK[:, 1, 1] * y_d + KK[:, 1, 2]
    proj = proj + pixel_noise * rng.standard_normal(proj.shape)
    f0 = np.where(known != 0, K_known[:, 0, 0], focal)
    return {
        "vmask": vmask, "projections": np.ascontiguousarray(proj),
        "gt_pts": pts, "gt_c": c, "gt_R": R.reshape(m, 9).copy(), "gt_f": f0.copy(),
        "R": R.reshape(m, 9).copy(),
        "c": c + cam_noise * rng.standard_normal(c.shape),
        "f": f0 * (1.0 + f_noise * rng.standard_normal(m)),
        "k": np.zeros((m, 2)),
        "pts": pts + pt_noise * rng.standard_normal(pts.shape),
        "known": known, "K_known": K_known.reshape(m, 9).copy(), "k_known": k_known,
    }


def fisheye_map(u, params):
    """sfm_fisheye_distort (lib/sfm-driver/sfm.c:426-446) of pinhole points u (N x 2) with per-point fisheye_params
    (N x 5: f_cx, f_cy, f_rad, f_angle, f_focal), in the reference's operation order -> pixels (N x 2)"""
    cx, cy, rad, fang, F = (params[:, q] for q in range(5))
    r = np.sqrt(u[:, 0] * u[:, 0] + u[:, 1] * u[:, 1])
    angle = 180.0 * np.arctan(r / F) / np.pi
    rnew = rad * angle / (0.5 * fang)
    return np.stack([u[:, 0] * (rnew / r) + cx, u[:, 1] * (rnew / r) + cy], 1)


def ba_scene_fisheye(num_cameras=20, num_points=2000, views_per_point=5, seed=2468, ordinary_fraction=0.25, known_fraction=0.0,
                     pixel_noise=0.5, pt_noise=0.02, cam_noise=0.01, f_noise=0.01, focal=800.0, min_radius=5.0):
    """A ba_scene measured through the reference's fisheye projection (sfm_project_point2_fisheye, lib/sfm-driver/
    sfm.c:448-492): the pinhole without the radial step, then, for the fisheye cameras, sfm_fisheye_distort with the
    camera's f_cx, f_cy, f_rad, f_angle, f_focal, plus N(0, pixel_noise^2).  A seeded `ordinary_fraction` of the cameras are
    not fisheye; a seeded `known_fraction` are calibrated (known_intrinsics, K_known / k_known as in
    ba_scene_known_intrinsics) and may be fisheye too.  Points are redrawn until every pinhole projection lies at least
    `min_radius` px from the principal point (the mapping is 0/0 there).  Adds fisheye [m] int8 and fisheye_params [m,5]
    (and known / K_known / k_known with known_fraction) to the ba_scene dict; fe_kwargs(scene) passes them on."""
    rng = np.random.default_rng(seed)
    m, n, L = num_cameras, num_points, views_per_point
    ang = 2.0 * np.pi * np.arange(m) / m
    c = np.stack([6.0 * np.cos(ang), 0.3 * np.sin(3 * ang), 6.0 * np.sin(ang)], 1)
    R = np.zeros((m, 3, 3))
    for j in range(m):
        z = c[j] / np.linalg.norm(c[j])
        xax = np.cross(np.array([0.0, 1.0, 0.0]), z); xax /= np.linalg.norm(xax)
        R[j] = np.stack([xax, np.cross(z, xax), z], 0)
    fisheye = np.ones(m, np.int8)
    n_ord = int(round(ordinary_fraction * m))
    if n_ord:
        fisheye[rng.choice(m, size=n_ord, replace=False)] = 0
    F = focal * (1.0 + 0.05 * rng.standard_normal(m))
    fang = rng.uniform(160.0, 200.0, m)
    rad = F * (0.5 * fang) * (np.pi / 180.0) * rng.uniform(0.9, 1.1, m)     # near-unit scale at the image centre
    params = np.stack([rng.uniform(-20.0, 20.0, m), rng.uniform(-20.0, 20.0, m), rad, fang, F], 1)
    known = np.zeros(m, np.int8)
    n_kn = int(round(known_fraction * m))
    if n_kn:
        known[rng.choice(m, size=n_kn, replace=False)] = 1
    K_known = np.zeros((m, 3, 3))
    K_known[:, 0, 0] = focal * (1.0 + 0.05 * rng.standard_normal(m))
    K_known[:, 0, 1] = rng.uniform(-3.0, 3.0, m)
    K_known[:, 0, 2] = rng.uniform(-25.0, 25.0, m)
    K_known[:, 1, 1] = K_known[:, 0, 0] * (1.0 + 0.01 * rng.standard_normal(m))
    K_known[:, 1, 2] = rng.uniform(-25.0, 25.0, m)
    K_known[:, 2, 2] = 1.0
    k_known = np.stack([rng.uniform(-0.12, -0.04, m), rng.uniform(0.01, 0.04, m), rng.uniform(-2e-3, 2e-3, m),
                        rng.uniform(-2e-3, 2e-3, m), rng.uniform(-4e-3, 4e-3, m)], 1)
    vmask = np.zeros((n, m), np.int8)
    step = max(m // L, 1)
    starts = (np.arange(n) * 7) % m
    for k in range(L):
        vmask[np.arange(n), (starts + k * step) % m] = 1
    pi, cj = np.nonzero(vmask)
    pts = rng.uniform(-1.0, 1.0, size=(n, 3))
    while True:
        Pc = np.einsum("oij,oj->oi", R[cj], pts[pi] - c[cj])
        u = -Pc[:, :2] * focal / Pc[:, 2:3]
        kn = known[cj] != 0
        if kn.any():
            from .bundle import project_known
            u[kn] = project_known(Pc[kn], K_known[cj[kn]].reshape(-1, 9), k_known[cj[kn]])
        near = np.unique(pi[np.hypot(u[:, 0], u[:, 1]) < min_radius])
        if not len(near):
            break
        pts[near] = rng.uniform(-1.0, 1.0, size=(len(near), 3))
    fe = fisheye[cj] != 0
    proj = u.copy()
    proj[fe] = fisheye_map(u[fe], params[cj[fe]])
    proj = proj + pixel_noise * rng.standard_normal(proj.shape)
    f0 = np.where(known != 0, K_known[:, 0, 0], focal)
    scene = {
        "vmask": vmask, "projections": np.ascontiguousarray(proj),
        "gt_pts": pts, "gt_c": c, "gt_R": R.reshape(m, 9).copy(), "gt_f": f0.copy(),
        "R": R.reshape(m, 9).copy(),
        "c": c + cam_noise * rng.standard_normal(c.shape),
        "f": f0 * (1.0 + f_noise * rng.standard_normal(m)),
        "k": np.zeros((m, 2)),
        "pts": pts + pt_noise * rng.standard_normal(pts.shape),
        "fisheye": fisheye, "fisheye_params": params,
    }
    if n_kn:
        scene.update(known=known, K_known=K_known.reshape(m, 9).copy(), k_known=k_known)
    return scene


def fe_kwargs(scene):
    """the camera keywords of a fisheye scene (fisheye, fisheye_params, and the calibration when it has one) for run_sfm /
    call_run_sfm / reprojection_outliers; empty for a scene without them"""
    return {k: scene[k] for k in ("fisheye", "fisheye_params", "known", "K_known", "k_known") if k in scene}


def crs_scene(scene):
    """a copy of a scene dict whose visibility is CRS instead of the dense vmask: vis_ptr [n+1] int32 (point i's
    observations are vis_ptr[i]..vis_ptr[i+1]) and vis_cam [nvis] int32 (ascending camera within a point), i.e.
    np.nonzero(vmask) in row-major order, the order of `projections`"""
    vmask = np.asarray(scene["vmask"])
    pi, cj = np.nonzero(vmask)
    out = {k: v for k, v in scene.items() if k != "vmask"}
    out["vis_ptr"] = np.concatenate([[0], np.cumsum(np.bincount(pi, minlength=vmask.shape[0]))]).astype(np.int32)
    out["vis_cam"] = cj.astype(np.int32)
    return out


def inject_outliers(scene, count, seed, displacement=50.0, all_views=False, candidates=None, camera=None):
    """a copy of a (dense or CRS) scene in which `count` seeded points are gross outliers: the measurement of one of
    their views (seeded), or of all of them, is moved by `displacement` to 2 * `displacement` pixels in a seeded
    direction.  The default 50 px is far above the largest threshold the outlier pass can use (16 px with Bundler's
    settings).  candidates: the points to choose from (default: every point with a view).  camera: choose among the
    points this camera sees and move their view in it (a camera with more than a fifth of its views displaced raises its
    own threshold, which is how a scene is made to take several rounds).  Returns (scene, chosen points, ascending)."""
    rng = np.random.default_rng(seed)
    if "vis_ptr" in scene:
        ptr = np.asarray(scene["vis_ptr"], dtype=np.int64)
    else:
        ptr = np.concatenate([[0], np.cumsum(np.count_nonzero(scene["vmask"], axis=1))])
    views = np.diff(ptr)
    pool = np.nonzero(views > 0)[0] if candidates is None else np.asarray(candidates)
    if camera is not None:
        from .bundle import observations
        obs_pt, obs_cam = observations(scene)
        in_cam = np.nonzero(obs_cam == camera)[0]
        cam_view = dict(zip(obs_pt[in_cam].tolist(), in_cam.tolist()))
        pool = np.array([i for i in pool if i in cam_view], dtype=np.int64)
    chosen = np.sort(rng.choice(pool, size=count, replace=False))
    proj = np.array(scene["projections"], dtype=np.float64)
    for i in chosen:
        obs = np.arange(ptr[i], ptr[i + 1]) if all_views else [cam_view[int(i)] if camera is not None else ptr[i] + rng.integers(views[i])]
        for o in obs:
            ang = rng.uniform(0.0, 2.0 * np.pi)
            proj[o] += rng.uniform(displacement, 2.0 * displacement) * np.array([np.cos(ang), np.sin(ang)])
    out = dict(scene)
    out["projections"] = proj
    return out, chosen


def ki_kwargs(scene):
    """the calibration keywords (known, K_known, k_known) of a scene for run_sfm / call_run_sfm / reprojection_rmse /
    reprojection_outliers; empty for a scene without calibrated cameras"""
    return {k: scene[k] for k in ("known", "K_known", "k_known") if k in scene}


def write_key_file(path, desc, seed=0):
    """Lowe text .key file (src/keys2a.cpp:183-253): "<num> 128", then per key "<y> <x> <scale> <ori>" and the
    128 descriptor values in 7 lines of 20,20,20,20,20,20,8 integers."""
    rng = np.random.default_rng(seed)
    n = desc.shape[0]
    with open(path, "w") as f:
        f.write(f"{n} 128\n")
        loc = rng.uniform(0, 1000, size=(n, 2)); sc = rng.uniform(1, 8, size=n); ori = rng.uniform(-3.14, 3.14, size=n)
        for i in range(n):
            f.write(f"{loc[i, 0]:.2f} {loc[i, 1]:.2f} {sc[i]:.2f} {ori[i]:.3f}\n")
            d = desc[i]
            for a in range(0, 128, 20):
                f.write(" " + " ".join(str(int(v)) for v in d[a:a + 20]) + "\n")
