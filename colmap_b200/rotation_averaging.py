"""Host-side mirror of COLMAP's rotation averaging solve over the C-ABI (include/b200_rotation_averaging.h).

Mirrors ``RotationEstimatorOptions`` and the flat form of ``RotationAveragingProblem`` after construction
(src/colmap/estimators/rotation_averaging{,_impl}.{h,cc}); ``RotationAveragingSolver::Solve`` (the L1 ADMM phase, then
IRLS) runs in libcolmap_b200.so on the GPU.  No CPU fallback.  ``RotationEstimator``, ``RunRotationAveraging`` and
``InitializeRigRotationsFromImages`` restate estimators/rotation_averaging.cc on the mirror's Reconstruction.
"""
import copy
import ctypes
import dataclasses
import enum
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from ._lib import load_library

MAX_AXIS_DIM = 32768
ERR_INPUT, ERR_TOO_LARGE, ERR_CUDA = -1, -2, -3
SUCCESS, FACTORIZATION_FAILED, NAN_STEP, NAN_WEIGHT, UNDERDETERMINED = 0, 1, 2, 3, 4
GEMAN_MCCLURE, HALF_NORM = 0, 1

_f64p = ctypes.POINTER(ctypes.c_double)
_u8p = ctypes.POINTER(ctypes.c_uint8)
_i32p = ctypes.POINTER(ctypes.c_int32)


class _COptions(ctypes.Structure):
    _fields_ = [("max_num_l1_iterations", ctypes.c_int), ("l1_step_convergence_threshold", ctypes.c_double),
                ("max_num_irls_iterations", ctypes.c_int), ("irls_step_convergence_threshold", ctypes.c_double),
                ("irls_loss_parameter_sigma", ctypes.c_double), ("ridge_regularization", ctypes.c_double),
                ("weight_type", ctypes.c_int), ("gpu_index", ctypes.c_int)]


class _CProblem(ctypes.Structure):
    _fields_ = [("num_frames", ctypes.c_int), ("frame_dof", _u8p), ("num_cameras", ctypes.c_int), ("rotations", _f64p),
                ("num_pairs", ctypes.c_int), ("pair_frame1", _i32p), ("pair_frame2", _i32p), ("pair_cam1", _i32p),
                ("pair_cam2", _i32p), ("pair_dof", _u8p), ("pair_R", _f64p), ("pair_angle", _f64p),
                ("pair_xz_error", _f64p), ("pair_reweighting", _f64p), ("gauge_frame", ctypes.c_int),
                ("gauge_rotation", ctypes.c_double * 3), ("cam_frame_start", _i32p), ("cam_frames", _i32p)]


class _CSummary(ctypes.Structure):
    _fields_ = [("status", ctypes.c_int), ("num_l1_iterations", ctypes.c_int), ("num_irls_iterations", ctypes.c_int),
                ("admm_iterations", _i32p), ("step_history", _f64p), ("n_xz", ctypes.c_int), ("n_y", ctypes.c_int),
                ("num_residuals", ctypes.c_int), ("l1_ms", ctypes.c_double), ("irls_ms", ctypes.c_double),
                ("build_ms", ctypes.c_double), ("factor_ms", ctypes.c_double), ("solve_ms", ctypes.c_double)]


def _bind(lib):
    if getattr(lib, "_ra_bound", False):
        return lib
    lib.b200ra_options_init.argtypes = [ctypes.POINTER(_COptions)]
    lib.b200ra_solve.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.POINTER(_CSummary)]
    lib.b200ra_solve.restype = ctypes.c_int
    lib.b200ra_last_error.restype = ctypes.c_char_p
    lib._ra_bound = True
    return lib


class RotationAveragingError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


class RotationAveragingReweighting(enum.IntEnum):
    """RotationAveragingReweighting: UNIFORM, or the pair's inlier match count over the largest one."""
    UNIFORM = 0
    INLIER_MATCH_COUNT = 1


@dataclass
class RotationEstimatorOptions:
    """RotationEstimatorOptions (estimators/rotation_averaging.h:25-96)."""
    random_seed: int = -1
    max_num_l1_iterations: int = 5
    l1_step_convergence_threshold: float = 0.001
    max_num_irls_iterations: int = 100
    irls_step_convergence_threshold: float = 0.001
    gravity_dir: np.ndarray = field(default_factory=lambda: np.array([0.0, 1.0, 0.0]))
    irls_loss_parameter_sigma: float = 5.0
    ridge_regularization: float = 1e-9
    weight_type: int = GEMAN_MCCLURE
    skip_initialization: bool = False
    use_gravity: bool = False
    use_stratified: bool = True
    filter_unregistered: bool = False
    max_rotation_error_deg: float = 10.0
    refine_sensor_from_rig: bool = True
    reweighting: RotationAveragingReweighting = RotationAveragingReweighting.UNIFORM
    gpu_index: int = -1

    def to_c(self) -> _COptions:
        o = _COptions()
        _bind(load_library()).b200ra_options_init(ctypes.byref(o))
        o.max_num_l1_iterations, o.l1_step_convergence_threshold = self.max_num_l1_iterations, self.l1_step_convergence_threshold
        o.max_num_irls_iterations, o.irls_step_convergence_threshold = self.max_num_irls_iterations, self.irls_step_convergence_threshold
        o.irls_loss_parameter_sigma, o.ridge_regularization = self.irls_loss_parameter_sigma, self.ridge_regularization
        o.weight_type, o.gpu_index = int(self.weight_type), self.gpu_index
        return o


@dataclass
class RotationAveragingSummary:
    status: int = SUCCESS
    num_l1_iterations: int = 0
    num_irls_iterations: int = 0
    admm_iterations: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int32))
    step_history: np.ndarray = field(default_factory=lambda: np.zeros(0))
    n_xz: int = 0
    n_y: int = 0
    num_residuals: int = 0
    l1_ms: float = 0.0
    irls_ms: float = 0.0
    build_ms: float = 0.0
    factor_ms: float = 0.0
    solve_ms: float = 0.0

    def success(self) -> bool:
        return self.status == SUCCESS


@dataclass
class FlatRotationAveraging:
    """The flat problem of the C-ABI (b200ra_problem); ``rotations`` is updated in place by solve_flat on success.

    Parameters: frame blocks (3 components, or 1 for a gravity-aligned frame), then estimated camera blocks (3).
    Pair i links frame blocks pair_frame1/2[i] and optional camera blocks pair_cam1/2[i] (-1: none)."""
    frame_dof: np.ndarray                          # [F] uint8, 1 or 3
    rotations: np.ndarray                          # [num_params]
    pair_frame1: np.ndarray                        # [P] int32
    pair_frame2: np.ndarray                        # [P] int32
    pair_dof: np.ndarray                           # [P] uint8, 1 or 3
    pair_R: np.ndarray                             # [P, 3, 3] R_cam2_from_cam1 (3-DOF pairs)
    gauge_frame: int = 0
    gauge_rotation: np.ndarray = field(default_factory=lambda: np.zeros(3))
    num_cameras: int = 0
    pair_cam1: Optional[np.ndarray] = None         # [P] int32
    pair_cam2: Optional[np.ndarray] = None         # [P] int32
    pair_angle: Optional[np.ndarray] = None        # [P] (1-DOF pairs)
    pair_xz_error: Optional[np.ndarray] = None     # [P] (1-DOF pairs)
    pair_reweighting: Optional[np.ndarray] = None  # [P] or None (UNIFORM)
    cam_frame_start: Optional[np.ndarray] = None   # [C + 1] int32
    cam_frames: Optional[np.ndarray] = None        # int32

    def __post_init__(self):
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64)
        i32 = lambda a: None if a is None else np.ascontiguousarray(a, np.int32)
        self.frame_dof = np.ascontiguousarray(self.frame_dof, np.uint8)
        self.pair_dof = np.ascontiguousarray(self.pair_dof, np.uint8)
        self.rotations, self.pair_angle, self.pair_xz_error = f64(self.rotations), f64(self.pair_angle), f64(self.pair_xz_error)
        self.pair_R = f64(self.pair_R).reshape(-1, 3, 3)
        self.pair_reweighting, self.gauge_rotation = f64(self.pair_reweighting), f64(self.gauge_rotation)
        self.pair_frame1, self.pair_frame2 = i32(self.pair_frame1), i32(self.pair_frame2)
        self.pair_cam1, self.pair_cam2 = i32(self.pair_cam1), i32(self.pair_cam2)
        self.cam_frame_start, self.cam_frames = i32(self.cam_frame_start), i32(self.cam_frames)
        self.gauge_frame, self.num_cameras = int(self.gauge_frame), int(self.num_cameras)

    @property
    def num_params(self) -> int:
        return int(self.frame_dof.astype(np.int64).sum()) + 3 * self.num_cameras

    def param_offsets(self) -> np.ndarray:
        """First parameter component of every block (frames, then cameras)."""
        d = np.concatenate([self.frame_dof.astype(np.int64), np.full(self.num_cameras, 3, np.int64)])
        return np.concatenate([[0], np.cumsum(d)[:-1]]).astype(np.int64)

    def copy(self) -> "FlatRotationAveraging":
        return FlatRotationAveraging(**{k: (np.array(v, copy=True) if isinstance(v, np.ndarray) else v)
                                        for k, v in self.__dict__.items()})

    def to_c(self) -> _CProblem:
        p = lambda a, t: None if a is None else a.ctypes.data_as(t)
        c = _CProblem()
        c.num_frames, c.frame_dof, c.num_cameras = len(self.frame_dof), p(self.frame_dof, _u8p), self.num_cameras
        c.rotations, c.num_pairs = p(self.rotations, _f64p), len(self.pair_frame1)
        c.pair_frame1, c.pair_frame2 = p(self.pair_frame1, _i32p), p(self.pair_frame2, _i32p)
        c.pair_cam1, c.pair_cam2, c.pair_dof = p(self.pair_cam1, _i32p), p(self.pair_cam2, _i32p), p(self.pair_dof, _u8p)
        c.pair_R, c.pair_angle, c.pair_xz_error = p(self.pair_R, _f64p), p(self.pair_angle, _f64p), p(self.pair_xz_error, _f64p)
        c.pair_reweighting, c.gauge_frame = p(self.pair_reweighting, _f64p), self.gauge_frame
        for k in range(3):
            c.gauge_rotation[k] = float(self.gauge_rotation[k])
        c.cam_frame_start, c.cam_frames = p(self.cam_frame_start, _i32p), p(self.cam_frames, _i32p)
        return c


def solve_flat(options: RotationEstimatorOptions, flat: FlatRotationAveraging) -> RotationAveragingSummary:
    """b200ra_solve on the flat problem, in place.  Raises RotationAveragingError on a refused input."""
    lib = _bind(load_library())
    admm = np.zeros(max(options.max_num_l1_iterations, 1), np.int32)
    hist = np.zeros(max(options.max_num_l1_iterations, 0) + max(options.max_num_irls_iterations, 0) + 1)
    s = _CSummary()
    s.admm_iterations, s.step_history = admm.ctypes.data_as(_i32p), hist.ctypes.data_as(_f64p)
    c = flat.to_c()
    rc = lib.b200ra_solve(ctypes.byref(options.to_c()), ctypes.byref(c), ctypes.byref(s))
    if rc != 0:
        raise RotationAveragingError(rc, lib.b200ra_last_error().decode())
    return RotationAveragingSummary(s.status, s.num_l1_iterations, s.num_irls_iterations, admm[:s.num_l1_iterations].copy(),
                                    hist[:s.num_l1_iterations + s.num_irls_iterations].copy(), s.n_xz, s.n_y,
                                    s.num_residuals, s.l1_ms, s.irls_ms, s.build_ms, s.factor_ms, s.solve_ms)


# ------------------------------------------------------------------------------------------------ RotationEstimator
# Restates estimators/rotation_averaging.cc and the set-up of RotationAveragingProblem (rotation_averaging_impl.cc:79-482)
# on the Python mirror's Reconstruction (every image in a frame).  Departures, stated: frames, cameras and pairs are
# visited in id order (the reference uses hash order), so the gauge is the smallest active frame id (or the first
# gravity-aligned one) and the global rotation of the result can differ from the reference's; the spanning tree breaks
# weight ties by pair order and is rooted at the smallest active image id.
_NAN3 = np.full(3, np.nan)


def _aa_to_R(w):
    """AngleAxisToRotationMatrix (geometry/pose.cc:137-156)."""
    w = np.asarray(w, np.float64)
    a = float(np.linalg.norm(w))
    if a <= 1e-12:
        return np.array([[1.0, -w[2], w[1]], [w[2], 1.0, -w[0]], [-w[1], w[0], 1.0]])
    k = w / a
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    return np.cos(a) * np.eye(3) + (1 - np.cos(a)) * np.outer(k, k) + np.sin(a) * K


def _R_to_quat(M):
    """Eigen's Quaternion(Matrix3d) as (x, y, z, w)."""
    q = np.zeros(4)
    t = M[0, 0] + M[1, 1] + M[2, 2]
    if t > 0:
        s = np.sqrt(t + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[:3] = [(M[2, 1] - M[1, 2]) * s, (M[0, 2] - M[2, 0]) * s, (M[1, 0] - M[0, 1]) * s]
    else:
        i = 0 if M[1, 1] <= M[0, 0] else 1
        i = 2 if M[2, 2] > M[i, i] else i
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(M[i, i] - M[j, j] - M[k, k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3], q[j], q[k] = (M[k, j] - M[j, k]) * s, (M[j, i] + M[i, j]) * s, (M[k, i] + M[i, k]) * s
    return q


def _R_to_aa(M):
    """RotationMatrixToAngleAxis through Eigen's quaternion."""
    q = _R_to_quat(M)
    n = float(np.linalg.norm(q[:3]))
    if n == 0.0:
        return np.zeros(3)
    ang = 2 * np.arctan2(n, abs(q[3]))
    return (-ang if q[3] < 0 else ang) / n * q[:3]


def _quat_R(q):
    from .bundle_adjustment import _quat_to_R
    q = np.asarray(q, np.float64)
    return _quat_to_R(q / np.linalg.norm(q))


def _average_rotations(Rs):
    """AverageQuaternions with unit weights (geometry/pose.cc:40-75, 182-199): the principal eigenvector of the mean
    of q q^T; the sign of the average does not change the rotation."""
    Q = np.stack([_R_to_quat(R) for R in Rs])
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    if len(Q) == 1:
        return _quat_R(Q[0])
    _, V = np.linalg.eigh(Q.T @ Q / len(Q))
    return _quat_R(V[:, -1])


def _gravity_aligned_rotation(g):
    """GravityAlignedRotation (geometry/pose.cc:278-297): columns (n0, g, n1) from a Householder basis of g's null space,
    right-handed."""
    g = np.asarray(g, np.float64)
    Q, _ = np.linalg.qr(g.reshape(3, 1), mode="complete")
    R = np.stack([Q[:, 1], g, Q[:, 2]], 1)
    if np.linalg.det(R) < 0:
        R[:, 2] = -R[:, 2]
    return R


def _frame_has_pose(rec, frame_id):
    T = rec.frames[frame_id].rig_from_world
    return T is not None and bool(np.all(np.isfinite(T[:4])))


def _sensor(rec, rig_id, camera_id):
    """(known, cam_from_rig) of a non-reference camera: known is False where the rig has no calibration for it."""
    T = rec.rigs[rig_id].sensors.get(camera_id)
    return T is not None and bool(np.all(np.isfinite(T[:4]))), T


def _image_R(rec, image_id):
    """R(cam_from_world) of an image from its frame, or None without a pose."""
    im = rec.images[image_id]
    if not _frame_has_pose(rec, im.frame_id):
        return None
    fr = rec.frames[im.frame_id]
    Rf = _quat_R(fr.rig_from_world[:4])
    if rec.IsRefInFrame(image_id):
        return Rf
    known, T = _sensor(rec, fr.rig_id, im.camera_id)
    return _quat_R(T[:4]) @ Rf if known else None


def _sync_images(rec, frame_ids):
    for im in rec.images.values():
        if im.frame_id not in frame_ids or rec.frames[im.frame_id].rig_from_world is None:
            continue
        R = _image_R(rec, im.image_id)
        if R is not None:
            im.cam_from_world = np.concatenate([_R_to_quat(R), _NAN3])


def _largest_component_image_ids(pose_graph, rec, filter_unregistered):
    frames = pose_graph.ComputeLargestConnectedFrameComponent(rec, filter_unregistered)
    return {i for i, im in rec.images.items() if im.frame_id in frames}


def _has_unknown_cams_from_rig(rec):
    return any(not (T is not None and np.all(np.isfinite(T[:4]))) for rig in rec.rigs.values() for T in rig.sensors.values())


def _gravity_by_image(pose_priors):
    return {p.image_id: p.gravity for p in pose_priors if getattr(p, "sensor_type", "CAMERA") == "CAMERA" and p.HasGravity()}


def InitializeRigRotationsFromImages(cams_from_world, reconstruction, refine_sensor_from_rig=True) -> bool:
    """InitializeRigRotationsFromImages (rotation_averaging.cc): cams_from_world maps image id -> R(cam_from_world).
    Unknown cam_from_rig rotations are averaged from the frames that observe both sensors, then every frame's
    rig_from_world rotation is averaged from its images (translations become unknown)."""
    rec = reconstruction
    images_of = {}
    for i in sorted(rec.images):
        images_of.setdefault(rec.images[i].frame_id, []).append(i)
    samples = {}
    for fid in sorted(rec.frames):
        ids = images_of.get(fid, [])
        ref = [i for i in ids if rec.IsRefInFrame(i)]
        if not ref or ref[0] not in cams_from_world:
            continue
        Rref = cams_from_world[ref[0]]
        for i in ids:
            if i == ref[0] or i not in cams_from_world:
                continue
            cam = rec.images[i].camera_id
            samples.setdefault(cam, (rec.frames[fid].rig_id, []))[1].append(cams_from_world[i] @ Rref.T)
    if refine_sensor_from_rig:
        for cam in sorted(samples):
            rig_id, Rs = samples[cam]
            T = rec.rigs[rig_id].sensors.get(cam)
            if T is not None and np.all(np.isfinite(T)):
                continue
            rec.rigs[rig_id].sensors[cam] = np.concatenate([_R_to_quat(_average_rotations(Rs)), _NAN3])
    else:
        for rig_id, rig in rec.rigs.items():
            for cam, T in rig.sensors.items():
                if T is None or not np.all(np.isfinite(T[:4])):
                    raise ValueError(f"sensor_from_rig has NaN rotation but refine_sensor_from_rig=false "
                                     f"(rig_id={rig_id}, sensor_id={cam})")
    for fid in sorted(rec.frames):
        Rs = []
        for i in images_of.get(fid, []):
            if i not in cams_from_world:
                continue
            if rec.IsRefInFrame(i):
                Rs.append(cams_from_world[i])
            else:
                known, T = _sensor(rec, rec.frames[fid].rig_id, rec.images[i].camera_id)
                if known:
                    Rs.append(_quat_R(T[:4]).T @ cams_from_world[i])
        if Rs:
            rec.frames[fid].rig_from_world = np.concatenate([_R_to_quat(_average_rotations(Rs)), _NAN3])
    _sync_images(rec, set(rec.frames))
    return True


class _ProblemMap:
    """RotationAveragingProblem's construction on the mirror: the flat problem plus what ApplyResultsToReconstruction
    needs to write it back."""

    def __init__(self, options, pose_graph, pose_priors, active_image_ids, rec):
        o = options
        gravity_img = _gravity_by_image(pose_priors)
        self.frames = sorted({rec.images[i].frame_id for i in active_image_ids})
        # frame gravity: the prior of the frame's reference image
        self.gravity = {}
        for i, g in gravity_img.items():
            if i in rec.images and rec.IsRefInFrame(i):
                self.gravity[rec.images[i].frame_id] = g
        self.has_g = lambda f: o.use_gravity and f in self.gravity
        cam_rig = {rec.images[i].camera_id: rec.frames[rec.images[i].frame_id].rig_id for i in active_image_ids}
        self.cams = []
        init_cam = {}
        if o.refine_sensor_from_rig:
            for cam in sorted(cam_rig):
                rig = rec.rigs[cam_rig[cam]]
                if rig.ref_sensor == cam:
                    continue
                T = rig.sensors.get(cam)
                if T is None or not np.all(np.isfinite(T)):
                    self.cams.append(cam)
                    init_cam[cam] = _R_to_aa(_quat_R(T[:4])) if T is not None and np.all(np.isfinite(T[:4])) else np.zeros(3)
        self.cam_rig = cam_rig
        cam_idx = {c: k for k, c in enumerate(self.cams)}
        fidx = {f: k for k, f in enumerate(self.frames)}
        dof, x = [], []
        gauge, g0 = -1, np.zeros(3)
        for f in self.frames:
            Rf = _quat_R(rec.frames[f].rig_from_world[:4]) if _frame_has_pose(rec, f) else np.eye(3)
            if self.has_g(f):
                a = _R_to_aa(_gravity_aligned_rotation(self.gravity[f]).T @ Rf)[1]
                dof.append(1); x.append([a])
                if gauge < 0:
                    gauge, g0 = fidx[f], np.array([0.0, a, 0.0])
            else:
                dof.append(3); x.append(_R_to_aa(Rf))
        for c in self.cams:
            x.append(init_cam[c])
        if gauge < 0 and self.frames:
            f = self.frames[0]
            gauge = 0
            g0 = _R_to_aa(_quat_R(rec.frames[f].rig_from_world[:4])) if _frame_has_pose(rec, f) else np.zeros(3)
        images_of = {}
        for i in sorted(rec.images):
            images_of.setdefault(rec.images[i].frame_id, []).append(i)
        cam_frames = [[fidx[f] for f in self.frames for i in images_of.get(f, []) if rec.images[i].camera_id == c]
                      for c in self.cams]
        f1, f2, c1, c2, pdof, pR, pang, pxz, nm = [], [], [], [], [], [], [], [], []
        for (i1, i2), e in pose_graph.Edges().items():
            if not e.valid or i1 not in rec.images or i2 not in rec.images:
                continue
            im1, im2 = rec.images[i1], rec.images[i2]
            if im1.frame_id not in fidx or im2.frame_id not in fidx:
                continue
            k1 = None if rec.IsRefInFrame(i1) or im1.camera_id in cam_idx else _sensor(rec, rec.frames[im1.frame_id].rig_id, im1.camera_id)[1]
            k2 = None if rec.IsRefInFrame(i2) or im2.camera_id in cam_idx else _sensor(rec, rec.frames[im2.frame_id].rig_id, im2.camera_id)[1]
            if k1 is not None and k2 is not None and im1.frame_id == im2.frame_id:
                continue
            R = _quat_R(e.cam2_from_cam1[:4])
            R = (_quat_R(k2[:4]).T if k2 is not None else np.eye(3)) @ R @ (_quat_R(k1[:4]) if k1 is not None else np.eye(3))
            g1, g2 = self.has_g(im1.frame_id), self.has_g(im2.frame_id)
            if g1:
                R = R @ _gravity_aligned_rotation(self.gravity[im1.frame_id])
            if g2:
                R = _gravity_aligned_rotation(self.gravity[im2.frame_id]).T @ R
            f1.append(fidx[im1.frame_id]); f2.append(fidx[im2.frame_id])
            c1.append(cam_idx.get(im1.camera_id, -1)); c2.append(cam_idx.get(im2.camera_id, -1))
            if g1 and g2:
                aa = _R_to_aa(R)
                pdof.append(1); pang.append(aa[1]); pxz.append(aa[0] ** 2 + aa[2] ** 2); pR.append(np.eye(3))
            else:
                pdof.append(3); pang.append(0.0); pxz.append(0.0); pR.append(R)
            nm.append(float(e.num_matches))
        rw = None
        if o.reweighting == RotationAveragingReweighting.INLIER_MATCH_COUNT and nm:
            mx = max(nm)
            rw = np.asarray(nm) / mx if mx > 0 else np.ones(len(nm))
        one = any(d == 1 for d in pdof)
        self.flat = FlatRotationAveraging(
            frame_dof=np.asarray(dof, np.uint8), rotations=np.concatenate([np.ravel(v) for v in x]) if x else np.zeros(0),
            pair_frame1=np.asarray(f1, np.int32), pair_frame2=np.asarray(f2, np.int32), pair_dof=np.asarray(pdof, np.uint8),
            pair_R=np.asarray(pR, np.float64).reshape(-1, 3, 3), gauge_frame=max(gauge, 0), gauge_rotation=g0,
            num_cameras=len(self.cams), pair_cam1=np.asarray(c1, np.int32) if self.cams else None,
            pair_cam2=np.asarray(c2, np.int32) if self.cams else None,
            pair_angle=np.asarray(pang) if one else None, pair_xz_error=np.asarray(pxz) if one else None,
            pair_reweighting=rw,
            cam_frame_start=np.concatenate([[0], np.cumsum([len(v) for v in cam_frames])]).astype(np.int32) if self.cams else None,
            cam_frames=np.concatenate([np.asarray(v, np.int32) for v in cam_frames]) if self.cams else None)

    def apply(self, rec, options):
        """ApplyResultsToReconstruction (rotation_averaging_impl.cc:644-684)."""
        off = self.flat.param_offsets()
        x = self.flat.rotations
        for k, f in enumerate(self.frames):
            if self.flat.frame_dof[k] == 1:
                R = _gravity_aligned_rotation(self.gravity[f]) @ _aa_to_R([0.0, x[off[k]], 0.0])
            else:
                R = _aa_to_R(x[off[k]:off[k] + 3])
            rec.frames[f].rig_from_world = np.concatenate([_R_to_quat(R), _NAN3])
        if options.refine_sensor_from_rig:
            for j, c in enumerate(self.cams):
                o = off[len(self.frames) + j]
                rec.rigs[self.cam_rig[c]].sensors[c] = np.concatenate([_R_to_quat(_aa_to_R(x[o:o + 3])), _NAN3])
        _sync_images(rec, set(self.frames))


class RotationEstimator:
    """RotationEstimator (estimators/rotation_averaging.{h,cc}); the flat solve runs on the GPU (b200ra_solve)."""

    def __init__(self, options: RotationEstimatorOptions):
        self.options_ = options
        self.summaries = []

    def _solve_flat(self, flat):
        """The solve of one assembled problem, in place; returns a summary with .status (a test substitutes the CPU
        oracle here)."""
        return solve_flat(self.options_, flat)

    def EstimateRotations(self, pose_graph, pose_priors, active_image_ids, reconstruction) -> bool:
        o = self.options_
        use_gravity = o.use_gravity and any(p.HasGravity() for p in pose_priors)
        if use_gravity and _has_unknown_cams_from_rig(reconstruction):
            return False   # gravity-aligned rotation needs every rig's calibration
        if use_gravity and o.use_stratified:
            if not self._maybe_solve_gravity_aligned_subset(pose_graph, pose_priors, active_image_ids, reconstruction):
                return False
        if not self._solve(pose_graph, pose_priors, active_image_ids, reconstruction):
            return False
        for i in sorted(active_image_ids):
            fid = reconstruction.images[i].frame_id
            assert _frame_has_pose(reconstruction, fid)
            reconstruction.RegisterFrame(fid)
        return True

    def _maybe_solve_gravity_aligned_subset(self, pose_graph, pose_priors, active_image_ids, rec):
        from .global_positioning import PoseGraph, PoseGraphEdge
        grav = _gravity_by_image(pose_priors)
        gpg = PoseGraph()
        total = 0
        for i1, i2 in pose_graph.ValidEdges():
            if i1 not in rec.images or i2 not in rec.images or i1 not in active_image_ids or i2 not in active_image_ids:
                continue
            total += 1
            if i1 in grav and i2 in grav:
                gpg.AddEdge(i1, i2, PoseGraphEdge(pose_graph.EdgeData(i1, i2).cam2_from_cam1.copy()))
        n = gpg.NumEdges()
        if not (n > 0 and n <= total * 0.95):
            return True
        grec = copy.deepcopy(rec)
        gids = _largest_component_image_ids(gpg, grec, False)
        gpg.InvalidatePairsOutsideActiveImageIds(gids)
        if not self._solve(gpg, pose_priors, gids, grec):
            return False
        for fid, fr in grec.frames.items():
            if _frame_has_pose(grec, fid):
                rec.frames[fid].rig_from_world = fr.rig_from_world.copy()
        if self.options_.refine_sensor_from_rig:
            for rid, rig in grec.rigs.items():
                for cam, T in rig.sensors.items():
                    if T is not None:
                        rec.rigs[rid].sensors[cam] = T.copy()
        return True

    def _solve(self, pose_graph, pose_priors, active_image_ids, rec):
        """SolveRotationAveraging: spanning-tree initialisation, the problem, the solve, the write-back."""
        if not self.options_.skip_initialization:
            self._initialize_from_maximum_spanning_tree(pose_graph, active_image_ids, rec)
        pm = _ProblemMap(self.options_, pose_graph, pose_priors, active_image_ids, rec)
        if not pm.frames:
            return False
        s = self._solve_flat(pm.flat)
        self.summaries.append(s)
        if s.status != SUCCESS:
            return False   # also an underdetermined problem, where the reference throws
        pm.apply(rec, self.options_)
        return True

    def _initialize_from_maximum_spanning_tree(self, pose_graph, active_image_ids, rec):
        ids = sorted(active_image_ids)
        if not ids:
            return
        edges = [(i1, i2, pose_graph.EdgeData(i1, i2).num_matches) for i1, i2 in sorted(pose_graph._key(*e) for e in pose_graph.ValidEdges())
                 if i1 in active_image_ids and i2 in active_image_ids]
        # Kruskal on decreasing match counts, ties in pair order
        parent = {i: i for i in ids}

        def find(a):
            while parent[a] != a:
                parent[a] = parent[parent[a]]
                a = parent[a]
            return a
        adj = {i: [] for i in ids}
        for i1, i2, _ in sorted(edges, key=lambda e: -e[2]):
            a, b = find(i1), find(i2)
            if a != b:
                parent[a] = b
                adj[i1].append(i2)
                adj[i2].append(i1)
        root = ids[0]
        cams = {}
        seen, queue = {root}, [root]
        while queue:
            cur = queue.pop(0)
            for ch in adj[cur]:
                if ch in seen:
                    continue
                seen.add(ch)
                queue.append(ch)
                Rp = cams.setdefault(cur, np.eye(3))
                cams[ch] = _quat_R(pose_graph.GetEdge(cur, ch).cam2_from_cam1[:4]) @ Rp
        InitializeRigRotationsFromImages(cams, rec, self.options_.refine_sensor_from_rig)


def _create_expanded_reconstruction(rec):
    """CreateExpandedReconstruction: every camera with an unknown cam_from_rig becomes the reference sensor of a rig of
    its own, and each of its images a frame of its own with an unknown pose."""
    from .bundle_adjustment import Frame, Reconstruction, Rig
    out = Reconstruction(cameras=rec.cameras, images={}, points3D={}, rigs={}, frames={})
    next_rig = max(rec.rigs, default=0) + 1
    single = {}
    for rid in sorted(rec.rigs):
        rig = rec.rigs[rid]
        r = Rig(rid, rig.ref_sensor)
        for cam in sorted(rig.sensors):
            T = rig.sensors[cam]
            if T is not None and np.all(np.isfinite(T[:4])):
                r.sensors[cam] = T.copy()
            else:
                single[cam] = next_rig
                out.rigs[next_rig] = Rig(next_rig, cam)
                next_rig += 1
        out.rigs[rid] = r
    next_frame = max(rec.frames, default=0) + 1
    for fid in sorted(rec.frames):
        fr = rec.frames[fid]
        T = fr.rig_from_world.copy() if _frame_has_pose(rec, fid) else None
        out.frames[fid] = Frame(fid, fr.rig_id, T)
    for iid in sorted(rec.images):
        im = rec.images[iid]
        new = copy.copy(im)
        new.points2D = []
        if im.camera_id in single and im.camera_id != rec.rigs[rec.frames[im.frame_id].rig_id].ref_sensor:
            out.frames[next_frame] = Frame(next_frame, single[im.camera_id], None)
            new.frame_id = next_frame
            next_frame += 1
        out.images[iid] = new
    return out


def _filter_edges_by_relative_rotation(pose_graph, rec, max_angle_deg):
    max_rad = np.radians(max_angle_deg)
    for i1, i2 in pose_graph.ValidEdges():
        R1, R2 = _image_R(rec, i1), _image_R(rec, i2)
        if R1 is None or R2 is None:
            continue
        D = (R2 @ R1.T).T @ _quat_R(pose_graph.EdgeData(i1, i2).cam2_from_cam1[:4])
        if np.linalg.norm(_R_to_aa(D)) > max_rad:
            pose_graph.SetInvalidEdge(i1, i2)


def RunRotationAveraging(options: RotationEstimatorOptions, pose_graph, reconstruction, pose_priors=(),
                         estimator=RotationEstimator) -> bool:
    """RunRotationAveraging (rotation_averaging.cc): the largest connected component, the estimate (through an expanded
    reconstruction and rig initialisation when some cam_from_rig is unknown), then the relative-rotation filter and the
    de-registration of frames that leave the component.  ``estimator`` is the RotationEstimator class used."""
    rec, pose_priors = reconstruction, list(pose_priors)
    if not _has_unknown_cams_from_rig(rec):
        active = _largest_component_image_ids(pose_graph, rec, options.filter_unregistered)
        if not active:
            return False
        pose_graph.InvalidatePairsOutsideActiveImageIds(active)
        if not estimator(options).EstimateRotations(pose_graph, pose_priors, active, rec):
            return False
    else:
        exp = _create_expanded_reconstruction(rec)
        active = _largest_component_image_ids(pose_graph, exp, options.filter_unregistered)
        if not active:
            return False
        pose_graph.InvalidatePairsOutsideActiveImageIds(active)
        if not estimator(options).EstimateRotations(pose_graph, pose_priors, active, exp):
            return False
        cams = {i: R for i in exp.images if (R := _image_R(exp, i)) is not None}
        InitializeRigRotationsFromImages(cams, rec, options.refine_sensor_from_rig)
        active = _largest_component_image_ids(pose_graph, rec, options.filter_unregistered)
        if not active:
            return False
        pose_graph.InvalidatePairsOutsideActiveImageIds(active)
        opts = dataclasses.replace(options, skip_initialization=True, use_stratified=False)
        if not estimator(opts).EstimateRotations(pose_graph, pose_priors, active, rec):
            return False
    if options.max_rotation_error_deg > 0:
        _filter_edges_by_relative_rotation(pose_graph, rec, options.max_rotation_error_deg)
        active = _largest_component_image_ids(pose_graph, rec, True)
        if not active:
            return False
        pose_graph.InvalidatePairsOutsideActiveImageIds(active)
        frames = {rec.images[i].frame_id for i in active}
        for fid in rec.RegFrameIds():
            if fid not in frames:
                rec.DeRegisterFrame(fid)
    return True
