"""Synthetic inputs for the two hot paths (SURVEY.md §8d).

PatchMatch: an analytic textured height field rendered into 1 + N pinhole views (ground-truth depth
and normal are exact), cameras on an arc with 5-15 degree triangulation angles.

Bundle adjustment: the semantics of colmap::SynthesizeDataset / SynthesizeNoise
(src/colmap/scene/synthetic.cc:341-672, benchmark/runtime/bundle_adjustment.cc:62-83) with tracks
sampled directly (points on the unit sphere, cameras at radius 5 looking at the origin).
"""
import numpy as np

from .patch_match import Image, Problem


# --------------------------------------------------------------------------------------------------
# PatchMatch scene
# --------------------------------------------------------------------------------------------------
class _HeightField:
    """z = h(x, y) in world coordinates, cameras look along +z from z ~ 0."""

    def __init__(self, rng, z0=5.0):
        self.z0 = z0
        self.amp = 0.18
        self.kx, self.ky = 1.1, 0.9
        self.sx, self.sy = 0.12, -0.07  # global slant
        self.px, self.py = rng.uniform(0, 2 * np.pi, 2)

    def h(self, x, y):
        return (self.z0 + self.sx * x + self.sy * y
                + self.amp * np.sin(self.kx * x + self.px) * np.cos(self.ky * y + self.py))

    def grad(self, x, y):
        hx = self.sx + self.amp * self.kx * np.cos(self.kx * x + self.px) * np.cos(self.ky * y + self.py)
        hy = self.sy - self.amp * self.ky * np.sin(self.kx * x + self.px) * np.sin(self.ky * y + self.py)
        return hx, hy


class _Texture:
    """Band-limited procedural texture on the (x, y) surface parameterisation."""

    def __init__(self, rng, min_wavelength, num_waves=28):
        lam = min_wavelength * np.exp(rng.uniform(0.0, np.log(24.0), num_waves))
        ang = rng.uniform(0, np.pi, num_waves)
        self.fx = (2 * np.pi / lam * np.cos(ang)).astype(np.float32)
        self.fy = (2 * np.pi / lam * np.sin(ang)).astype(np.float32)
        self.ph = rng.uniform(0, 2 * np.pi, num_waves).astype(np.float32)
        self.amp = (lam / lam.max()) ** 0.35
        self.amp = (self.amp / np.sqrt(0.5 * np.sum(self.amp ** 2))).astype(np.float32)

    def __call__(self, x, y):
        acc = np.zeros_like(x, dtype=np.float32)
        for fx, fy, ph, a in zip(self.fx, self.fy, self.ph, self.amp):
            acc += a * np.sin(fx * x + fy * y + ph)
        return acc  # unit variance


def _look_at_R(center, target):
    """World->camera rotation for a camera at `center` looking at `target`, x right, y down."""
    z = target - center
    z = z / np.linalg.norm(z)
    up = np.array([0.0, -1.0, 0.0])
    x = np.cross(-up, z)
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    return np.stack([x, y, z])  # rows


def _render(hf, tex, K, R, T, width, height, contrast=45.0):
    """Exact per-pixel ray / height-field intersection.  Returns (uint8 image, depth, normal_cam)."""
    C = -R.T @ T
    u, v = np.meshgrid(np.arange(width, dtype=np.float64), np.arange(height, dtype=np.float64))
    dcx = (u - K[0, 2]) / K[0, 0]
    dcy = (v - K[1, 2]) / K[1, 1]
    # d_world = R^T (dcx, dcy, 1)
    dx = R[0, 0] * dcx + R[1, 0] * dcy + R[2, 0]
    dy = R[0, 1] * dcx + R[1, 1] * dcy + R[2, 1]
    dz = R[0, 2] * dcx + R[1, 2] * dcy + R[2, 2]
    t = (hf.z0 - C[2]) / dz
    for _ in range(12):
        t = (hf.h(C[0] + t * dx, C[1] + t * dy) - C[2]) / dz
    x = C[0] + t * dx
    y = C[1] + t * dy
    img = 128.0 + contrast * tex(x.astype(np.float32), y.astype(np.float32))
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    hx, hy = hf.grad(x, y)
    nw = np.stack([hx, hy, -np.ones_like(hx)])
    nw /= np.linalg.norm(nw, axis=0, keepdims=True)
    nc = np.einsum("ij,jhw->ihw", R, nw)
    return img, t.astype(np.float32), nc.astype(np.float32)


def make_patch_match_scene(width=1920, height=1080, num_src=8, seed=0, with_gt_maps=False):
    """Returns dict(images=[Image] (index 0 = reference), problem=Problem, depth_gt, normal_gt,
    depth_min, depth_max[, depth_maps, normal_maps for every view])."""
    rng = np.random.default_rng(seed)
    hf = _HeightField(rng)
    f = 0.9 * width
    K = np.array([[f, 0, (width - 1) / 2.0], [0, f, (height - 1) / 2.0], [0, 0, 1]], np.float64)
    pixel = hf.z0 / f
    tex = _Texture(rng, min_wavelength=5.0 * pixel)
    target = np.array([0.0, 0.0, hf.z0])
    # world frame deliberately not aligned with the reference camera
    centers = [np.array([0.05, -0.03, 0.0])]
    for k in range(num_src):
        ang = 2 * np.pi * (k + 0.37) / max(num_src, 1)
        tri = np.deg2rad(rng.uniform(5.0, 15.0))
        rad = hf.z0 * np.tan(tri)
        centers.append(centers[0] + np.array([rad * np.cos(ang), rad * np.sin(ang), rng.uniform(-0.15, 0.15)]))
    images, depths, normals = [], [], []
    for k, c in enumerate(centers):
        tgt = target + (0 if k == 0 else rng.uniform(-0.15, 0.15, 3) * np.array([1, 1, 0]))
        R = _look_at_R(c, tgt)
        T = -R @ c
        if k == 0 or with_gt_maps:
            img, d, n = _render(hf, tex, K, R, T, width, height)
        else:
            img, d, n = _render(hf, tex, K, R, T, width, height)
        images.append(Image(bitmap=img, K=K.astype(np.float32), R=R.astype(np.float32), T=T.astype(np.float32)))
        depths.append(d)
        normals.append(n)
    problem = Problem(ref_image_idx=0, src_image_idxs=list(range(1, num_src + 1)), images=images)
    dmin, dmax = float(depths[0].min()), float(depths[0].max())
    out = dict(images=images, problem=problem, depth_gt=depths[0], normal_gt=normals[0],
               depth_min=0.75 * dmin, depth_max=1.25 * dmax)
    if with_gt_maps:
        out["depth_maps"] = depths
        out["normal_maps"] = normals
    return out


def make_workspace_scene(width, height, num_images, seed=0, device=None):
    """A workspace-shaped scene (BASELINE config C4): `num_images` views of one textured height field, cameras on a ring
    (mutual triangulation angles of a few degrees), every view a reference image.  Rendered with torch on `device` when
    given (4K frames take seconds per view in numpy).  Returns dict(images=[Image], depth_gt=[...], depth_min, depth_max,
    centers)."""
    rng = np.random.default_rng(seed)
    hf = _HeightField(rng)
    f = 0.9 * width
    K = np.array([[f, 0, (width - 1) / 2.0], [0, f, (height - 1) / 2.0], [0, 0, 1]], np.float64)
    tex = _Texture(rng, min_wavelength=5.0 * hf.z0 / f)
    target = np.array([0.0, 0.0, hf.z0])
    centers = []
    for k in range(num_images):
        ang = 2 * np.pi * k / num_images
        rad = hf.z0 * np.tan(np.deg2rad(rng.uniform(4.0, 9.0)))
        centers.append(np.array([rad * np.cos(ang), rad * np.sin(ang), rng.uniform(-0.15, 0.15)]))
    images, depths = [], []
    for c in centers:
        R = _look_at_R(c, target + rng.uniform(-0.1, 0.1, 3) * np.array([1, 1, 0]))
        T = -R @ c
        if device is None:
            img, d, _ = _render(hf, tex, K, R, T, width, height)
        else:
            img, d = _render_torch(hf, tex, K, R, T, width, height, device)
        images.append(Image(bitmap=img, K=K.astype(np.float32), R=R.astype(np.float32), T=T.astype(np.float32)))
        depths.append(d)
    dmin, dmax = min(float(d.min()) for d in depths), max(float(d.max()) for d in depths)
    return dict(images=images, depth_gt=depths, depth_min=0.75 * dmin, depth_max=1.25 * dmax, centers=np.stack(centers))


def _render_torch(hf, tex, K, R, T, width, height, device, contrast=45.0):
    """_render on a torch device (same ray / height-field intersection and texture; bench inputs, not bit-pinned)."""
    import torch
    C = -R.T @ T
    dd = torch.float64
    u = torch.arange(width, dtype=dd, device=device)[None, :].expand(height, width)
    v = torch.arange(height, dtype=dd, device=device)[:, None].expand(height, width)
    dcx = (u - K[0, 2]) / K[0, 0]
    dcy = (v - K[1, 2]) / K[1, 1]
    dx = R[0, 0] * dcx + R[1, 0] * dcy + R[2, 0]
    dy = R[0, 1] * dcx + R[1, 1] * dcy + R[2, 1]
    dz = R[0, 2] * dcx + R[1, 2] * dcy + R[2, 2]

    def h(x, y):
        return hf.z0 + hf.sx * x + hf.sy * y + hf.amp * torch.sin(hf.kx * x + hf.px) * torch.cos(hf.ky * y + hf.py)
    t = (hf.z0 - C[2]) / dz
    for _ in range(12):
        t = (h(C[0] + t * dx, C[1] + t * dy) - C[2]) / dz
    x = (C[0] + t * dx).to(torch.float32)
    y = (C[1] + t * dy).to(torch.float32)
    acc = torch.zeros_like(x)
    for fx, fy, ph, a in zip(tex.fx, tex.fy, tex.ph, tex.amp):
        acc += float(a) * torch.sin(float(fx) * x + float(fy) * y + float(ph))
    img = torch.clamp(torch.round(128.0 + contrast * acc), 0, 255).to(torch.uint8)
    return img.cpu().numpy(), t.to(torch.float32).cpu().numpy()


# --------------------------------------------------------------------------------------------------
# Bundle adjustment scenes (colmap::SynthesizeDataset / SynthesizeNoise semantics, tracks sampled directly)
# --------------------------------------------------------------------------------------------------
def _quat_from_two_vectors(a, b):
    """Eigen::Quaterniond::FromTwoVectors(a, b) for unit vectors, (x, y, z, w); vectorised over rows of a."""
    a = a / np.linalg.norm(a, axis=-1, keepdims=True)
    b = np.broadcast_to(b / np.linalg.norm(b), a.shape)
    c = np.sum(a * b, axis=-1, keepdims=True)
    axis = np.cross(a, b)
    s = np.sqrt((1.0 + c) * 2.0)
    q = np.concatenate([axis / s, s * 0.5], axis=-1)
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _quat_mul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def _quat_rotate(q, p):
    v = q[..., :3]
    w = q[..., 3:4]
    t = 2.0 * np.cross(v, p)
    return p + w * t + np.cross(v, t)


_MODEL_DEFAULTS = {0: [1280.0, 512.0, 384.0], 1: [1280.0, 1280.0, 512.0, 384.0], 2: [1280.0, 512.0, 384.0, 0.05],
                   3: [1280.0, 512.0, 384.0, 0.05, 0.01], 8: [1280.0, 512.0, 384.0, 0.05], 9: [1280.0, 512.0, 384.0, 0.05, 0.01],
                   # the twelve models beyond the radial pinhole family (sensor/models.h:533-800): mild distortion
                   4: [1280.0, 1270.0, 512.0, 384.0, 0.04, -0.01, 1e-3, -8e-4],                               # OPENCV
                   5: [1280.0, 1270.0, 512.0, 384.0, 0.03, -0.01, 2e-3, -1e-3],                               # OPENCV_FISHEYE
                   6: [1280.0, 1270.0, 512.0, 384.0, 0.04, -0.01, 1e-3, -8e-4, 2e-3, 0.01, -3e-3, 1e-3],      # FULL_OPENCV
                   7: [1280.0, 1270.0, 512.0, 384.0, 0.3],                                                    # FOV
                   10: [1280.0, 1270.0, 512.0, 384.0, 0.03, -0.01, 1e-3, -8e-4, 2e-3, -1e-3, 5e-4, -4e-4],    # THIN_PRISM_FISHEYE
                   11: [1280.0, 1270.0, 512.0, 384.0, 0.03, -0.01, 2e-3, -1e-3, 5e-4, -2e-4, 1e-3, -8e-4, 5e-4, -4e-4, 3e-4, -2e-4],
                   12: [1280.0, 512.0, 384.0, -0.02], 13: [1280.0, 1270.0, 512.0, 384.0, -0.02],              # (SIMPLE_)DIVISION
                   14: [1280.0, 512.0, 384.0], 15: [1280.0, 1270.0, 512.0, 384.0],                            # (SIMPLE_)FISHEYE
                   16: [1280.0, 1270.0, 512.0, 384.0, 0.5, 1.1],                                              # EUCM
                   17: [2048.0, 1024.0]}                                                                      # EQUIRECTANGULAR


def _project(model, params, pc):
    if model not in (0, 1, 2, 3, 8, 9):   # wide models: the product's own host formulas (b200ba_test_project_wide), point by point
        import ctypes
        from ._lib import load_library
        lib = load_library()
        f64p = ctypes.POINTER(ctypes.c_double)
        lib.b200ba_test_project_wide.argtypes = [ctypes.c_int, f64p, f64p, f64p, f64p, f64p]
        out = np.empty((len(pc), 2))
        P = params.shape[-1]
        xy = np.zeros(2); Ju = np.zeros(6); Jp = np.zeros(2 * P)
        pcc = np.ascontiguousarray(pc, np.float64); prm = np.ascontiguousarray(params, np.float64)
        for k in range(len(pc)):
            ok = lib.b200ba_test_project_wide(int(model), prm[k].ctypes.data_as(f64p), pcc[k].ctypes.data_as(f64p), xy.ctypes.data_as(f64p),
                                              Ju.ctypes.data_as(f64p), Jp.ctypes.data_as(f64p))
            assert ok == 1, (model, pcc[k])
            out[k] = xy
        return out
    uu = pc[..., 0] / pc[..., 2]
    vv = pc[..., 1] / pc[..., 2]
    if model == 0:
        return np.stack([params[..., 0] * uu + params[..., 1], params[..., 0] * vv + params[..., 2]], -1)
    if model == 1:
        return np.stack([params[..., 0] * uu + params[..., 2], params[..., 1] * vv + params[..., 3]], -1)
    if model in (8, 9):   # equidistant fisheye: (uu, vv) <- (atan r / r)(uu, vv), then the radial polynomial
        r = np.sqrt(uu * uu + vv * vv)
        s = np.where(r > 1e-12, np.arctan(r) / np.maximum(r, 1e-300), 1.0)
        uu, vv = s * uu, s * vv
    r2 = uu * uu + vv * vv
    rad = params[..., 3] * r2 if model in (2, 8) else params[..., 3] * r2 + params[..., 4] * r2 * r2
    return np.stack([params[..., 0] * uu * (1 + rad) + params[..., 1], params[..., 0] * vv * (1 + rad) + params[..., 2]], -1)


def synthesize_ba_problem(num_images, num_points, track_length, models=(2,), shared_camera=False, seed=42,
                          point2D_stddev=1.0, point3D_stddev=0.05, translation_stddev=0.01, rotation_stddev_deg=1.0,
                          num_obs=None, track_lengths=None):
    """Ground truth + noisy flat BA problems.  `models`: camera model ids cycled over the images (one camera per
    image) or a single shared camera.  `num_obs` (optional) = exact observation count (tracks of length
    floor/ceil(num_obs/num_points)).  Noise defaults = benchmark/runtime/bundle_adjustment.cc:76-80."""
    from .bundle_adjustment import MODEL_NUM_PARAMS, FlatProblem
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1, 1, (num_points, 3))
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    view = -rng.uniform(-1, 1, (num_images, 3))
    view /= np.linalg.norm(view, axis=1, keepdims=True)
    q = _quat_from_two_vectors(view, np.array([0.0, 0.0, 1.0]))
    t = _quat_rotate(q, 5.0 * view)
    poses = np.concatenate([q, t], axis=1)
    if shared_camera:
        cam_model = [models[0]]
        img_cam = np.zeros(num_images, np.int32)
    else:
        cam_model = [models[i % len(models)] for i in range(num_images)]
        img_cam = np.arange(num_images, dtype=np.int32)
    cam_off, off = [], 0
    for m in cam_model:
        cam_off.append(off); off += MODEL_NUM_PARAMS[m]
    cam_params = np.concatenate([np.asarray(_MODEL_DEFAULTS[m]) for m in cam_model])
    # tracks
    if track_lengths is not None:
        lens = np.asarray(track_lengths, np.int64)
    elif num_obs is None:
        lens = np.full(num_points, track_length, np.int64)
    else:
        base = num_obs // num_points
        lens = np.full(num_points, base, np.int64)
        lens[: num_obs - base * num_points] += 1
    obs_point = np.repeat(np.arange(num_points, dtype=np.int32), lens)
    # distinct random images per point: random keys, take the `len` smallest per point (vectorised for equal lens)
    maxlen = int(lens.max())
    keys = rng.random((num_points, num_images)) if num_points * num_images <= 5e7 else None
    if keys is not None:
        order = np.argsort(keys, axis=1)[:, :maxlen]
        sel = order[np.arange(maxlen)[None, :] < lens[:, None]]
    else:
        # large problems: sample with replacement then de-duplicate by re-drawing collisions a few times
        cand = rng.integers(0, num_images, (num_points, maxlen))
        for _ in range(8):
            cs = np.sort(cand, axis=1)
            dup = np.zeros_like(cand, bool)
            dup[:, 1:] = cs[:, 1:] == cs[:, :-1]
            if not dup.any():
                break
            cand = cs
            cand[dup] = rng.integers(0, num_images, int(dup.sum()))
        sel = cand[np.arange(maxlen)[None, :] < lens[:, None]]
    obs_pose = sel.astype(np.int32)
    obs_cam = img_cam[obs_pose]
    # exact projections
    pc = _quat_rotate(poses[obs_pose, :4], pts[obs_point]) + poses[obs_pose, 4:]
    xy = np.empty((len(obs_pose), 2))
    cm = np.asarray(cam_model)[obs_cam]
    for m in set(cam_model):
        msk = cm == m
        offs = np.asarray(cam_off)[obs_cam[msk]]
        prm = cam_params[offs[:, None] + np.arange(MODEL_NUM_PARAMS[m])[None, :]]
        xy[msk] = _project(m, prm, pc[msk])
    n_img, n_cam = num_images, len(cam_model)
    gt = FlatProblem(poses, np.zeros(n_img, np.uint8), -np.ones(n_img, np.int8), cam_model, cam_off, cam_params,
                     np.zeros(n_cam, np.uint8), pts, np.zeros(num_points, np.uint8), obs_pose, obs_cam, obs_point, xy)
    noisy = gt.copy()
    # SynthesizeNoise (synthetic.cc:675-733)
    if rotation_stddev_deg > 0:
        ang = np.deg2rad(np.clip(rng.normal(0, rotation_stddev_deg, num_images), -180, 180))
        qz = np.stack([np.zeros(num_images), np.zeros(num_images), np.sin(ang / 2), np.cos(ang / 2)], 1)
        noisy.poses[:, :4] = _quat_mul(noisy.poses[:, :4], qz)
    if translation_stddev > 0:
        noisy.poses[:, 4:] += rng.normal(0, translation_stddev, (num_images, 3))
    if point2D_stddev > 0:
        noisy.obs_xy = noisy.obs_xy + rng.normal(0, point2D_stddev, noisy.obs_xy.shape)
    if point3D_stddev > 0:
        noisy.points += rng.normal(0, point3D_stddev, noisy.points.shape)
    return gt, noisy


def flat_to_reconstruction(flat):
    """FlatProblem -> minimal Reconstruction (ids are 1-based like COLMAP's)."""
    from .bundle_adjustment import MODEL_NUM_PARAMS, Camera, Image, Point2D, Point3D, Reconstruction
    rec = Reconstruction()
    for c in range(len(flat.cam_model)):
        n = MODEL_NUM_PARAMS[int(flat.cam_model[c])]
        rec.cameras[c + 1] = Camera(c + 1, int(flat.cam_model[c]), flat.cam_params[flat.cam_off[c]:flat.cam_off[c] + n].copy())
    img_cam = {}
    for o in range(len(flat.obs_pose)):
        img_cam[int(flat.obs_pose[o])] = int(flat.obs_cam[o])
    for i in range(len(flat.poses)):
        rec.images[i + 1] = Image(i + 1, img_cam.get(i, 0) + 1, flat.poses[i].copy())
    for p in range(len(flat.points)):
        rec.points3D[p + 1] = Point3D(flat.points[p].copy())
    for o in range(len(flat.obs_pose)):
        im = rec.images[int(flat.obs_pose[o]) + 1]
        pid = int(flat.obs_point[o]) + 1
        im.points2D.append(Point2D(flat.obs_xy[o].copy(), pid))
        rec.points3D[pid].track.append((im.image_id, len(im.points2D) - 1))
    return rec


def synthesize_rig_problem(num_frames, num_sensors, num_points, track_length, models=(2,), seed=42, point2D_stddev=1.0,
                           point3D_stddev=0.05, translation_stddev=0.01, rotation_stddev_deg=1.0, sensor_translation_stddev=0.005,
                           sensor_rotation_stddev_deg=0.3):
    """Rig scene (SynthesizeDataset with num_cameras_per_rig > 1, scene/synthetic.cc:341-672): ONE rig of `num_sensors`
    cameras (sensor 0 = reference sensor, the others carry a sensor_from_rig pose), `num_frames` frames (one
    rig_from_world pose each), every point seen from `track_length` random (frame, sensor) pairs.  In the flat problem
    obs_pose_idx is the FRAME and obs_camera_idx the sensor's camera.  Returns (ground truth, noisy) FlatProblems."""
    from .bundle_adjustment import MODEL_NUM_PARAMS, FlatProblem
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1, 1, (num_points, 3))
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    view = -rng.uniform(-1, 1, (num_frames, 3))
    view /= np.linalg.norm(view, axis=1, keepdims=True)
    q = _quat_from_two_vectors(view, np.array([0.0, 0.0, 1.0]))
    poses = np.concatenate([q, _quat_rotate(q, 5.0 * view)], axis=1)                 # rig_from_world per frame
    # sensor_from_rig of the non-reference sensors: a few degrees of rotation, a 0.1-0.3 baseline
    ns = num_sensors - 1
    ax = rng.normal(size=(ns, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.deg2rad(rng.uniform(2.0, 6.0, ns))
    sq = np.concatenate([ax * np.sin(ang / 2)[:, None], np.cos(ang / 2)[:, None]], axis=1)
    st = rng.uniform(-0.3, 0.3, (ns, 3))
    sensors = np.concatenate([sq, st], axis=1)
    cam_model = [models[i % len(models)] for i in range(num_sensors)]
    cam_off, off = [], 0
    for m in cam_model:
        cam_off.append(off); off += MODEL_NUM_PARAMS[m]
    cam_params = np.concatenate([np.asarray(_MODEL_DEFAULTS[m]) for m in cam_model])
    cam_sensor = np.array([-1] + list(range(ns)), np.int32)
    # tracks over (frame, sensor) slots
    slots = num_frames * num_sensors
    obs_point = np.repeat(np.arange(num_points, dtype=np.int32), track_length)
    keys = rng.random((num_points, slots))
    sel = np.argsort(keys, axis=1)[:, :track_length].reshape(-1)
    obs_pose = (sel // num_sensors).astype(np.int32)
    obs_cam = (sel % num_sensors).astype(np.int32)
    pr = _quat_rotate(poses[obs_pose, :4], pts[obs_point]) + poses[obs_pose, 4:]
    pc = pr.copy()
    nr = obs_cam > 0
    pc[nr] = _quat_rotate(sensors[obs_cam[nr] - 1, :4], pr[nr]) + sensors[obs_cam[nr] - 1, 4:]
    xy = np.empty((len(obs_pose), 2))
    for c in range(num_sensors):
        msk = obs_cam == c
        m = cam_model[c]
        prm = np.broadcast_to(cam_params[cam_off[c]:cam_off[c] + MODEL_NUM_PARAMS[m]], (int(msk.sum()), MODEL_NUM_PARAMS[m]))
        xy[msk] = _project(m, prm, pc[msk])
    gt = FlatProblem(poses, np.zeros(num_frames, np.uint8), -np.ones(num_frames, np.int8), cam_model, cam_off, cam_params,
                     np.zeros(num_sensors, np.uint8), pts, np.zeros(num_points, np.uint8), obs_pose, obs_cam, obs_point, xy)
    gt.set_sensors(sensors, np.zeros(ns, np.uint8), cam_sensor)
    noisy = gt.copy()
    if rotation_stddev_deg > 0:
        a = np.deg2rad(rng.normal(0, rotation_stddev_deg, num_frames))
        noisy.poses[:, :4] = _quat_mul(noisy.poses[:, :4], np.stack([0 * a, 0 * a, np.sin(a / 2), np.cos(a / 2)], 1))
    if translation_stddev > 0:
        noisy.poses[:, 4:] += rng.normal(0, translation_stddev, (num_frames, 3))
    if ns and sensor_rotation_stddev_deg > 0:
        a = np.deg2rad(rng.normal(0, sensor_rotation_stddev_deg, ns))
        noisy.sensors[:, :4] = _quat_mul(noisy.sensors[:, :4], np.stack([0 * a, 0 * a, np.sin(a / 2), np.cos(a / 2)], 1))
    if ns and sensor_translation_stddev > 0:
        noisy.sensors[:, 4:] += rng.normal(0, sensor_translation_stddev, (ns, 3))
    if point2D_stddev > 0:
        noisy.obs_xy = noisy.obs_xy + rng.normal(0, point2D_stddev, noisy.obs_xy.shape)
    if point3D_stddev > 0:
        noisy.points += rng.normal(0, point3D_stddev, noisy.points.shape)
    return gt, noisy


def synthesize_rig_reconstruction(num_rigs, num_cameras_per_rig, num_frames_per_rig, num_points3D, model=2, seed=0,
                                  point2D_stddev=0.0, prior_position=False):
    """SynthesizeDataset with rigs (scene/synthetic.cc:341-672) as a Reconstruction of the Python mirror: `num_rigs` rigs of
    `num_cameras_per_rig` cameras each (own intrinsics; the first camera of a rig is its reference sensor), every rig
    with `num_frames_per_rig` frames, one image per (frame, sensor), image / camera / frame / rig ids ascending from 1 in
    that order, every point observed by every image (as in the reference's small test scenes).  prior_position=True
    returns (rec, pose_priors) with one PosePrior per image at its projection centre and no covariance
    (scene/synthetic.cc:497-523); synthesize_noise perturbs them."""
    from .bundle_adjustment import Camera, Frame, Image, MODEL_NUM_PARAMS, Point2D, Point3D, Reconstruction, Rig, _rigid_compose
    rng = np.random.default_rng(seed)
    rec = Reconstruction()
    pts = rng.uniform(-1, 1, (num_points3D, 3))
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)
    for k in range(num_points3D):
        rec.points3D[k + 1] = Point3D(xyz=pts[k].copy())
    cam_id = img_id = frame_id = 0
    for r in range(1, num_rigs + 1):
        cams = []
        for _ in range(num_cameras_per_rig):
            cam_id += 1
            rec.cameras[cam_id] = Camera(cam_id, model, np.asarray(_MODEL_DEFAULTS[model], np.float64).copy())
            cams.append(cam_id)
        rig = Rig(r, cams[0])
        for c in cams[1:]:
            ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
            ang = np.deg2rad(rng.uniform(2.0, 6.0))
            rig.sensors[c] = np.concatenate([ax * np.sin(ang / 2), [np.cos(ang / 2)], rng.uniform(-0.3, 0.3, 3)])
        rec.rigs[r] = rig
        for _ in range(num_frames_per_rig):
            frame_id += 1
            view = -rng.uniform(-1, 1, 3); view /= np.linalg.norm(view)
            q = _quat_from_two_vectors(view[None], np.array([0.0, 0.0, 1.0]))[0]
            rfw = np.concatenate([q, _quat_rotate(q[None], 5.0 * view[None])[0]])
            rec.frames[frame_id] = Frame(frame_id, r, rfw)
            for c in cams:
                img_id += 1
                cfw = rfw if c == rig.ref_sensor else _rigid_compose(rig.sensors[c], rfw)
                pc = _quat_rotate(np.broadcast_to(cfw[:4], (num_points3D, 4)), pts) + cfw[4:]
                prm = rec.cameras[c].params
                xy = _project(model, np.broadcast_to(prm, (num_points3D, MODEL_NUM_PARAMS[model])), pc)
                if point2D_stddev > 0:
                    xy = xy + rng.normal(0, point2D_stddev, xy.shape)
                im = Image(img_id, c, cfw.copy(), frame_id=frame_id)
                for k in range(num_points3D):
                    im.points2D.append(Point2D(xy[k].copy(), k + 1))
                    rec.points3D[k + 1].track.append((img_id, k))
                rec.images[img_id] = im
    if prior_position:
        from .bundle_adjustment import PosePrior, projection_center
        return rec, [PosePrior(i, projection_center(rec, i)) for i in sorted(rec.images)]
    return rec


def synthesize_noise(rec, pose_priors=None, point2D_stddev=0.0, point3D_stddev=0.0, rig_from_world_rotation_stddev=0.0,
                     rig_from_world_translation_stddev=0.0, prior_position_stddev=0.0, seed=1):
    """SynthesizeNoise (scene/synthetic.cc:675-768) on a reconstruction with frames, in place: Gaussian pixel and point
    noise, rig_from_world rotation noise (degrees, about a random axis) and translation noise, and Gaussian noise on the
    prior positions with covariance prior_position_stddev^2 I (the covariance is set even for a zero stddev only when
    pose_priors are given and the stddev is positive)."""
    from .bundle_adjustment import _rigid_compose
    rng = np.random.default_rng(seed)
    for f in sorted(rec.frames):
        fr = rec.frames[f]
        if rig_from_world_rotation_stddev > 0:
            ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
            a = np.deg2rad(rng.normal(0, rig_from_world_rotation_stddev))
            dq = np.concatenate([ax * np.sin(a / 2), [np.cos(a / 2)]])
            fr.rig_from_world[:4] = _quat_mul(dq[None], fr.rig_from_world[None, :4])[0]
        if rig_from_world_translation_stddev > 0:
            fr.rig_from_world[4:] += rng.normal(0, rig_from_world_translation_stddev, 3)
    for im in rec.images.values():   # keep the derived image poses in step with the frames
        fr = rec.frames[im.frame_id]
        rig = rec.rigs[fr.rig_id]
        im.cam_from_world[:] = fr.rig_from_world if rig.ref_sensor == im.camera_id else _rigid_compose(rig.sensors[im.camera_id], fr.rig_from_world)
        if point2D_stddev > 0:
            for p2 in im.points2D:
                p2.xy = p2.xy + rng.normal(0, point2D_stddev, 2)
    if point3D_stddev > 0:
        for k in sorted(rec.points3D):
            rec.points3D[k].xyz += rng.normal(0, point3D_stddev, 3)
    if pose_priors is not None and prior_position_stddev > 0:
        for pp in pose_priors:
            pp.position = pp.position + rng.normal(0, prior_position_stddev, 3)
            pp.position_covariance = prior_position_stddev ** 2 * np.eye(3)
    return rec



def synthesize_global_positioning(num_frames, num_points, num_observations, seed=0, ray_stddev=5e-3):
    """A flat global-positioning problem (FlatGlobalPositioning): frame centres on a sphere of radius 5 around points in
    the unit cube, num_observations // num_points observations per point in distinct frames, unit rays with Gaussian
    noise of ray_stddev, the reference's random initial centres and points (100 * U(-1, 1)), unit scales and the 0.5
    loss weight of cameras without a prior focal length."""
    from .global_positioning import FlatGlobalPositioning
    rng = np.random.default_rng(seed)
    C = rng.normal(size=(num_frames, 3))
    C *= 5 / np.linalg.norm(C, axis=1, keepdims=True)
    X = rng.uniform(-1, 1, (num_points, 3))
    k = num_observations // num_points
    obs_point = np.repeat(np.arange(num_points), k)
    obs_frame = (rng.integers(0, num_frames, num_points)[:, None] + np.arange(k)[None, :] * max(1, num_frames // k)).reshape(-1) % num_frames
    d = X[obs_point] - C[obs_frame]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d += rng.normal(0, ray_stddev, d.shape)
    return FlatGlobalPositioning(frame_centers=100 * rng.uniform(-1, 1, (num_frames, 3)),
                                 points=100 * rng.uniform(-1, 1, (num_points, 3)), obs_frame=obs_frame, obs_point=obs_point,
                                 obs_ray=d, obs_scale=np.ones(len(obs_point)), obs_loss_weight=np.full(len(obs_point), 0.5))


def _random_rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    x, y, z, w = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


def _exp_so3(w):
    w = np.asarray(w, np.float64).reshape(-1, 3)
    th = np.linalg.norm(w, axis=1)
    a = w / np.where(th > 0, th, 1.0)[:, None]
    K = np.zeros((len(w), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -a[:, 2], a[:, 1], -a[:, 0]
    K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = a[:, 2], -a[:, 1], a[:, 0]
    s, c = np.sin(th)[:, None, None], np.cos(th)[:, None, None]
    return c * np.eye(3) + (1 - c) * a[:, :, None] * a[:, None, :] + s * K


def _log_so3(R):
    R = np.asarray(R).reshape(-1, 3, 3)
    c = np.clip((np.trace(R, axis1=1, axis2=2) - 1) / 2, -1, 1)
    th = np.arccos(c)
    v = np.stack([R[:, 2, 1] - R[:, 1, 2], R[:, 0, 2] - R[:, 2, 0], R[:, 1, 0] - R[:, 0, 1]], 1)
    s = np.sin(th)
    f = np.where(s > 1e-12, th / np.where(s > 1e-12, 2 * s, 1.0), 0.5)
    return f[:, None] * v


def synthesize_rotation_averaging(num_frames, edges_per_frame=20, noise_deg=1.0, outlier_ratio=0.1, seed=0,
                                  init_noise_deg=5.0, gravity_fraction=0.0, num_cameras=0, reweighting=False,
                                  banded=False, gravity_frames=None):
    """A flat rotation-averaging problem (FlatRotationAveraging) and its ground-truth rotations.

    A frame is gravity-aligned (1-DOF) with probability gravity_fraction, or, when gravity_frames (a boolean mask over
    the frames) is given, exactly where the mask is set; the random stream is the same either way, so everything else
    stays as gravity_fraction would draw it.  Frames get uniformly random rotations (a gravity-aligned 1-DOF frame a
    rotation about y); about
    num_frames * edges_per_frame / 2 pairs join them: a chain through all frames plus random pairs, or, with banded,
    each frame with its next edges_per_frame / 2 frames.  Relative rotations carry Gaussian angle-axis noise of
    noise_deg, and a fraction outlier_ratio of them is replaced by a random rotation.  Pairs between two 1-DOF frames
    are 1-DOF (angle and xz_error).  With num_cameras > 0, one image of some 3-DOF pairs sits in an estimated camera c
    with a random cam_from_rig.  The initial estimate is the ground truth perturbed by init_noise_deg (y only for 1-DOF
    frames; cameras as after the reference's rig initialisation); the gauge is the first 1-DOF frame if there is one, else frame 0, fixed at its
    initial rotation.  Returns (flat, gt) with gt the ground-truth parameter vector."""
    from .rotation_averaging import FlatRotationAveraging
    rng = np.random.default_rng(seed)
    F, C = num_frames, num_cameras
    dof = np.where(rng.uniform(size=F) < gravity_fraction, 1, 3).astype(np.uint8)
    if gravity_frames is not None:
        mask = np.asarray(gravity_frames, bool)
        if mask.shape != (F,):
            raise ValueError(f"gravity_frames must be a boolean mask of {F} frames, not of shape {mask.shape}")
        dof = np.where(mask, 1, 3).astype(np.uint8)
    Rg = _random_rotations(rng, F)
    ang = rng.uniform(-np.pi, np.pi, F)
    one = dof == 1
    if one.any():
        Rg[one] = _exp_so3(np.stack([np.zeros(one.sum()), ang[one], np.zeros(one.sum())], 1))
    Rc = _random_rotations(rng, C) if C else np.zeros((0, 3, 3))
    k = max(1, edges_per_frame // 2)
    if banded:
        pairs = [(i, j) for i in range(F) for j in range(i + 1, min(F, i + 1 + k))]
    else:
        pairs = {(i, i + 1) for i in range(F - 1)}
        target = max(len(pairs), F * k)
        while len(pairs) < target:
            a, b = rng.integers(0, F, 2)
            if a != b:
                pairs.add((min(a, b), max(a, b)))
        pairs = sorted(pairs)
    P = len(pairs)
    f1 = np.array([p[0] for p in pairs], np.int32).reshape(-1)
    f2 = np.array([p[1] for p in pairs], np.int32).reshape(-1)
    pdof = np.where(one[f1] & one[f2], 1, 3).astype(np.uint8)
    c1 = np.full(P, -1, np.int32)
    c2 = np.full(P, -1, np.int32)
    if C:
        sel = (pdof == 3) & (rng.uniform(size=P) < 0.5)
        which = rng.integers(0, 2, P)
        cam = rng.integers(0, C, P)
        c1[sel & (which == 0)] = cam[sel & (which == 0)]
        c2[sel & (which == 1)] = cam[sel & (which == 1)]
    R1 = Rg[f1].copy()
    R2 = Rg[f2].copy()
    m1, m2 = c1 >= 0, c2 >= 0
    R1[m1] = Rc[c1[m1]] @ R1[m1]
    R2[m2] = Rc[c2[m2]] @ R2[m2]
    R12 = R2 @ np.transpose(R1, (0, 2, 1))
    R12 = _exp_so3(rng.normal(0, np.radians(noise_deg), (P, 3))) @ R12
    out = rng.uniform(size=P) < outlier_ratio
    if out.any():
        R12[out] = _random_rotations(rng, int(out.sum()))
    pangle = np.zeros(P)
    pxz = np.zeros(P)
    if (pdof == 1).any():
        s = pdof == 1
        pangle[s] = ang[f2[s]] - ang[f1[s]] + rng.normal(0, np.radians(noise_deg), s.sum())
        pangle[s & out] = rng.uniform(-np.pi, np.pi, (s & out).sum())
        pxz[s] = rng.normal(0, np.radians(noise_deg), s.sum()) ** 2
    # parameters: ground truth and initial estimate
    gt, x0 = [], []
    for f in range(F):
        if dof[f] == 1:
            gt.append([ang[f]])
            x0.append([ang[f] + rng.normal(0, np.radians(init_noise_deg))])
        else:
            w = _log_so3(Rg[f])[0]
            gt.append(w)
            x0.append(_log_so3(_exp_so3(rng.normal(0, np.radians(init_noise_deg), 3)) @ Rg[f])[0])
    for c in range(C):
        gt.append(_log_so3(Rc[c])[0])
        x0.append(_log_so3(_exp_so3(rng.normal(0, np.radians(init_noise_deg), 3)) @ Rc[c])[0])
    gt = np.concatenate([np.asarray(g, np.float64).reshape(-1) for g in gt])
    x0 = np.concatenate([np.asarray(g, np.float64).reshape(-1) for g in x0])
    gauge = int(np.argmax(one)) if one.any() else 0
    off = np.concatenate([[0], np.cumsum(dof.astype(np.int64))[:-1]])
    g0 = np.zeros(3)
    if dof[gauge] == 1:
        g0[1] = x0[off[gauge]]
    else:
        g0[:] = x0[off[gauge]:off[gauge] + 3]
    cs, cf = None, None
    if C:
        lists = [sorted(set(f1[c1 == c].tolist()) | set(f2[c2 == c].tolist())) or [0] for c in range(C)]
        cs = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
        cf = np.concatenate([np.asarray(x, np.int32) for x in lists])
    flat = FlatRotationAveraging(frame_dof=dof, rotations=x0, pair_frame1=f1, pair_frame2=f2, pair_dof=pdof, pair_R=R12,
                                 gauge_frame=gauge, gauge_rotation=g0, num_cameras=C,
                                 pair_cam1=c1 if C else None, pair_cam2=c2 if C else None,
                                 pair_angle=pangle if (pdof == 1).any() else None,
                                 pair_xz_error=pxz if (pdof == 1).any() else None,
                                 pair_reweighting=rng.uniform(0.05, 1.0, P) if reweighting else None,
                                 cam_frame_start=cs, cam_frames=cf)
    return flat, gt


def synthesize_pose_graph(rec, noise_deg=0.0, outlier_ratio=0.0, seed=0, gravity=False, max_num_matches=500):
    """A PoseGraph over every image pair of ``rec`` (a reconstruction with frames, e.g. from
    synthesize_rig_reconstruction) and its pose priors.  Each edge holds the true cam2_from_cam1 rotation (translation
    left at zero) with Gaussian angle-axis noise of noise_deg, a fraction outlier_ratio of them replaced by a random
    rotation, and a random inlier match count in [max_num_matches / 10, max_num_matches].  With gravity, every image
    gets a PosePrior whose gravity is the world's +y axis in the camera frame.  Returns (pose_graph, pose_priors)."""
    from .bundle_adjustment import PosePrior, _quat_to_R
    from .global_positioning import PoseGraph, PoseGraphEdge
    from .rotation_averaging import _R_to_quat
    rng = np.random.default_rng(seed)
    ids = sorted(rec.images)
    R = {i: _quat_to_R(rec.images[i].cam_from_world[:4]) for i in ids}
    pg = PoseGraph()
    for a in range(len(ids)):
        for b in range(a + 1, len(ids)):
            i1, i2 = ids[a], ids[b]
            R12 = _exp_so3(rng.normal(0, np.radians(noise_deg), 3))[0] @ R[i2] @ R[i1].T
            if rng.uniform() < outlier_ratio:
                R12 = _random_rotations(rng, 1)[0]
            n = int(rng.integers(max_num_matches // 10, max_num_matches + 1))
            pg.AddEdge(i1, i2, PoseGraphEdge(np.concatenate([_R_to_quat(R12), np.zeros(3)]), n))
    priors = [PosePrior(i, gravity=R[i] @ np.array([0.0, 1.0, 0.0])) for i in ids] if gravity else []
    return pg, priors


# --------------------------------------------------------------------------------------------------
# SIFT descriptors
# --------------------------------------------------------------------------------------------------
def FeatureDescriptorsToUnsignedByte(x):
    """FeatureDescriptorsToUnsignedByte (feature/utils.cc:57-69): round(512 x) (half away from zero), clamped to
    [0, 255], in float32."""
    s = np.float32(512.0) * np.asarray(x, np.float32)
    r = np.sign(s) * np.floor(np.abs(s) + np.float32(0.5))
    return np.clip(r, 0, 255).astype(np.uint8)


def CreateRandomFeatureDescriptors(num_features, seed=0):
    """The descriptors of the reference's matcher tests (feature/sift_test.cc:211-227): 10 random dimensions set to 1,
    L2-normalised, to uint8.  Every row is 162 on 10 dimensions and 0 elsewhere, so dot products between rows take
    few distinct values and tie often."""
    rng = np.random.default_rng(seed)
    x = np.zeros((num_features, 128), np.float32)
    if num_features:
        dims = np.argsort(rng.random((num_features, 128)), axis=1)[:, :10]
        np.put_along_axis(x, dims, np.float32(1.0), axis=1)
        x /= np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)
    return FeatureDescriptorsToUnsignedByte(x)


def _sift_like(rng, n):
    """Non-negative, sparse-ish unit rows, clipped at 0.2 and renormalised as SIFT does, in float32."""
    x = rng.gamma(0.6, 1.0, (n, 128)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x = np.minimum(x, np.float32(0.2))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def make_sift_view_pair(n1, n2, overlap=0.5, noise=(0.0, 3.0), seed=0):
    """Descriptors of two overlapping views, (n1, 128) and (n2, 128) uint8.  Image 2 holds noisy copies of a random
    subset of image 1's rows (min(n1, n2) * overlap of them, each with its own noise level drawn from `noise`, relative
    to the row's norm), the rest are unrelated distractors, in a random order.  The spread of noise levels puts many
    rows on both sides of the ratio and distance thresholds.  Returns (desc1, desc2, truth), truth[k] = (i1, i2) of
    each planted copy."""
    rng = np.random.default_rng(seed)
    a = _sift_like(rng, n1)
    k = int(min(n1, n2) * overlap)
    src = rng.choice(n1, size=k, replace=False) if k else np.zeros(0, np.int64)
    sigma = rng.uniform(noise[0], noise[1], (k, 1)).astype(np.float32)
    copies = a[src] + sigma * np.abs(rng.normal(0, 1, (k, 128))).astype(np.float32) / np.sqrt(np.float32(128))
    copies = np.maximum(copies, 0)
    copies /= np.maximum(np.linalg.norm(copies, axis=1, keepdims=True), np.float32(1e-12))
    b = np.concatenate([copies, _sift_like(rng, n2 - k)], axis=0)
    perm = rng.permutation(n2)
    b = b[perm]
    inv = np.empty(n2, np.int64); inv[perm] = np.arange(n2)
    truth = np.stack([src, inv[np.arange(k)]], axis=1) if k else np.zeros((0, 2), np.int64)
    return FeatureDescriptorsToUnsignedByte(a), FeatureDescriptorsToUnsignedByte(b), truth


def _project_two_view(model_id, params, X):
    """ImgFromCam of the models make_guided_view_pair uses (sensor/models.h): SIMPLE_PINHOLE, SIMPLE_RADIAL,
    SIMPLE_RADIAL_FISHEYE and EQUIRECTANGULAR; X is (n, 3) in the camera frame."""
    p = np.asarray(params, np.float64)
    if model_id == 17:
        theta = np.arctan2(X[:, 0], X[:, 2])
        phi = np.arcsin(np.clip(-X[:, 1] / np.linalg.norm(X, axis=1), -1, 1))
        return np.stack([p[0] * (theta / (2 * np.pi) + 0.5), p[1] * (0.5 - phi / np.pi)], axis=1)
    u, v = X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    if model_id == 8:
        r = np.hypot(u, v)
        s = np.where(r > 1e-12, np.arctan(r) / np.maximum(r, 1e-12), 1.0)
        u, v = u * s, v * s
    if model_id in (2, 8):
        rad = p[3] * (u * u + v * v)
        u, v = u + u * rad, v + v * rad
    return np.stack([p[0] * u + p[1], p[0] * v + p[2]], axis=1)


def make_guided_view_pair(n1, n2, model_id=0, plane=False, overlap=0.5, pixel_noise=0.5, seed=0):
    """Two views of planted 3D points for guided matching.  Descriptors come from make_sift_view_pair (noisy copies of
    a subset plus distractors); each planted copy (i1, i2) is a 3D point seen by both cameras, and its keypoints are
    its projections with Gaussian pixel noise; every other keypoint is uniform over the image.  Both cameras share
    `model_id`: 0 SIMPLE_PINHOLE, 2 SIMPLE_RADIAL, 8 SIMPLE_RADIAL_FISHEYE or 17 EQUIRECTANGULAR.  With `plane` the
    points lie on one plane.  Returns a dict with desc1, desc2, xy1, xy2 ((n, 2) float32), camera1, camera2
    (bundle_adjustment.Camera), truth, E (cam2_from_cam1: ray2^T E ray1 = 0), F (the pinhole F of E, for model 0),
    H (the pixel homography of the plane, with `plane` and model 0)."""
    from .bundle_adjustment import Camera
    rng = np.random.default_rng(seed)
    d1, d2, truth = make_sift_view_pair(n1, n2, overlap=overlap, seed=seed)
    W, Hh = (1024, 512) if model_id == 17 else (640, 480)
    params = {0: [500.0, 320.0, 240.0], 2: [500.0, 320.0, 240.0, -0.08], 8: [300.0, 320.0, 240.0, 0.03],
              17: [float(W), float(Hh)]}[model_id]
    cam = Camera(1, model_id, np.array(params, np.float64))
    ang = rng.normal(0, 0.05, 3)
    th = np.linalg.norm(ang)
    k = ang / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = np.array([1.0, 0.1, 0.05]) + rng.normal(0, 0.05, 3)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = tx @ R
    m = len(truth)
    # points in front of both cameras, inside the pinhole field of view of camera 1
    x = rng.uniform(-0.5, 0.5, (m, 2))
    depth = np.full(m, 6.0) if plane else rng.uniform(4.0, 12.0, m)
    X1 = np.concatenate([x * depth[:, None], depth[:, None]], axis=1)
    if plane:   # the plane z = 6 tilted: n . X = d
        nrm = np.array([0.1, -0.2, 1.0]); nrm /= np.linalg.norm(nrm)
        dpl = 6.0
        X1 = X1 * (dpl / (X1 @ nrm))[:, None]
    X2 = X1 @ R.T + t
    xy1 = rng.uniform([0, 0], [W, Hh], (n1, 2))
    xy2 = rng.uniform([0, 0], [W, Hh], (n2, 2))
    if m:
        xy1[truth[:, 0]] = _project_two_view(model_id, params, X1) + rng.normal(0, pixel_noise, (m, 2))
        xy2[truth[:, 1]] = _project_two_view(model_id, params, X2) + rng.normal(0, pixel_noise, (m, 2))
    out = {"desc1": d1, "desc2": d2, "xy1": xy1.astype(np.float32), "xy2": xy2.astype(np.float32), "camera1": cam,
           "camera2": Camera(2, model_id, np.array(params, np.float64)), "truth": truth, "E": E, "F": None, "H": None}
    if model_id == 0:
        K = np.array([[params[0], 0, params[1]], [0, params[0], params[2]], [0, 0, 1.0]])
        Ki = np.linalg.inv(K)
        out["F"] = Ki.T @ E @ Ki
        if plane:
            out["H"] = K @ (R + np.outer(t, nrm) / dpl) @ Ki
    return out
