"""Host-side mirror of COLMAP's bundle-adjustment interface over the C-ABI (include/b200_bundle_adjustment.h).

Mirrors (same names / meaning):
  * ``BundleAdjustmentOptions``  src/colmap/estimators/bundle_adjustment.h:175-208 (+ the Ceres solver options
    COLMAP sets, bundle_adjustment_ceres.cc:102-116)
  * ``BundleAdjustmentConfig``   bundle_adjustment.h:77-151
  * ``BundleAdjuster`` / ``CreateDefaultBundleAdjuster``  bundle_adjustment.h:212-234, bundle_adjustment.cc:314-336
  * a minimal ``Reconstruction`` (cameras, images with cam_from_world, points3D with tracks) — just what
    DefaultBundleAdjuster touches (bundle_adjustment_ceres.cc:606-898), trivial frames only.

The flattening below is a harness-level restatement of DefaultBundleAdjuster's problem assembly
(AddImageToProblem / AddPointToProblem / Parameterize*, bundle_adjustment_ceres.cc:688-888,419-565); the solve
itself happens in libcolmap_b200.so on the GPU.  No CPU fallback.
"""
import ctypes
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from ._lib import load_library

# CameraModelId (sensor/models.h:90-109)
SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL, OPENCV, OPENCV_FISHEYE, FULL_OPENCV, FOV = 0, 1, 2, 3, 4, 5, 6, 7
SIMPLE_RADIAL_FISHEYE, RADIAL_FISHEYE, THIN_PRISM_FISHEYE, RAD_TAN_THIN_PRISM_FISHEYE = 8, 9, 10, 11
SIMPLE_DIVISION, DIVISION, SIMPLE_FISHEYE, FISHEYE, EUCM, EQUIRECTANGULAR = 12, 13, 14, 15, 16, 17
MODEL_NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12, 11: 16, 12: 4, 13: 5, 14: 3, 15: 4, 16: 6, 17: 2}
AUTO, DENSE_SCHUR, SPARSE_SCHUR, ITERATIVE_SCHUR = 0, 1, 2, 3
TRIVIAL, SOFT_L1, CAUCHY, HUBER = 0, 1, 2, 3
CONVERGENCE, NO_CONVERGENCE, FAILURE = 0, 1, 2
UNSPECIFIED_GAUGE, TWO_CAMS_FROM_WORLD, THREE_POINTS = 0, 1, 2


class _COptions(ctypes.Structure):
    _fields_ = [("refine_focal_length", ctypes.c_int), ("refine_principal_point", ctypes.c_int),
                ("refine_extra_params", ctypes.c_int), ("refine_rig_from_world", ctypes.c_int),
                ("refine_points3D", ctypes.c_int), ("constant_rig_from_world_rotation", ctypes.c_int),
                ("loss_function_type", ctypes.c_int), ("loss_function_scale", ctypes.c_double),
                ("linear_solver_type", ctypes.c_int), ("max_num_iterations", ctypes.c_int),
                ("max_linear_solver_iterations", ctypes.c_int), ("function_tolerance", ctypes.c_double),
                ("gradient_tolerance", ctypes.c_double), ("parameter_tolerance", ctypes.c_double),
                ("initial_trust_region_radius", ctypes.c_double), ("max_trust_region_radius", ctypes.c_double),
                ("min_trust_region_radius", ctypes.c_double), ("min_relative_decrease", ctypes.c_double),
                ("min_lm_diagonal", ctypes.c_double), ("max_lm_diagonal", ctypes.c_double), ("eta", ctypes.c_double),
                ("jacobi_scaling", ctypes.c_int), ("gpu_index", ctypes.c_int), ("refine_sensor_from_rig", ctypes.c_int)]


_f64p = ctypes.POINTER(ctypes.c_double)
_u8p = ctypes.POINTER(ctypes.c_uint8)
_i8p = ctypes.POINTER(ctypes.c_int8)
_i32p = ctypes.POINTER(ctypes.c_int32)


class _CProblem(ctypes.Structure):
    _fields_ = [("num_poses", ctypes.c_int), ("poses", _f64p), ("pose_constant", _u8p),
                ("pose_fixed_translation_dim", _i8p), ("num_cameras", ctypes.c_int), ("camera_model_id", _i32p),
                ("camera_param_offset", _i32p), ("camera_params", _f64p), ("camera_constant", _u8p),
                ("num_points", ctypes.c_int64), ("points", _f64p), ("point_constant", _u8p),
                ("num_observations", ctypes.c_int64), ("obs_pose_idx", _i32p), ("obs_camera_idx", _i32p),
                ("obs_point_idx", _i32p), ("obs_xy", _f64p), ("num_config_images", ctypes.c_int32),
                ("num_sensors", ctypes.c_int32), ("sensor_from_rig", _f64p), ("sensor_constant", _u8p),
                ("camera_sensor_idx", _i32p)]


class _CSummary(ctypes.Structure):
    _fields_ = [("termination_type", ctypes.c_int), ("num_residuals", ctypes.c_int),
                ("num_effective_parameters", ctypes.c_int), ("num_successful_steps", ctypes.c_int),
                ("num_unsuccessful_steps", ctypes.c_int), ("num_linear_solver_iterations", ctypes.c_int),
                ("linear_solver_type_used", ctypes.c_int), ("initial_cost", ctypes.c_double),
                ("final_cost", ctypes.c_double), ("solve_ms", ctypes.c_double), ("setup_ms", ctypes.c_double),
                ("spmv_ms_total", ctypes.c_double), ("spmv_launches", ctypes.c_int), ("kernel_launches", ctypes.c_int)]


@dataclass
class BundleAdjustmentOptions:
    """BundleAdjustmentOptions (bundle_adjustment.h:175-208) + Ceres solver options set by COLMAP."""
    refine_focal_length: bool = True
    refine_principal_point: bool = False
    refine_extra_params: bool = True
    refine_sensor_from_rig: bool = True
    refine_rig_from_world: bool = True
    refine_points3D: bool = True
    min_track_length: int = 0
    constant_rig_from_world_rotation: bool = False
    print_summary: bool = False
    backend: str = "B200"
    loss_function_type: int = TRIVIAL
    loss_function_scale: float = 1.0
    linear_solver_type: int = AUTO          # auto_select_solver_type (bundle_adjustment_ceres.cc:202-212)
    max_num_iterations: int = 100
    max_linear_solver_iterations: int = 200
    function_tolerance: float = 0.0
    gradient_tolerance: float = 1e-4
    parameter_tolerance: float = 0.0
    gpu_index: int = -1

    def Check(self) -> bool:
        return self.min_track_length >= 0 and self.loss_function_scale >= 0 and self.max_num_iterations >= 0

    def to_c(self) -> _COptions:
        return _COptions(int(self.refine_focal_length), int(self.refine_principal_point), int(self.refine_extra_params),
                         int(self.refine_rig_from_world), int(self.refine_points3D),
                         int(self.constant_rig_from_world_rotation), self.loss_function_type, self.loss_function_scale,
                         self.linear_solver_type, self.max_num_iterations, self.max_linear_solver_iterations,
                         self.function_tolerance, self.gradient_tolerance, self.parameter_tolerance,
                         1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 0.1, 1, self.gpu_index, int(self.refine_sensor_from_rig))


@dataclass
class BundleAdjustmentSummary:
    termination_type: int = FAILURE
    num_residuals: int = 0
    num_effective_parameters: int = 0
    num_successful_steps: int = 0
    num_unsuccessful_steps: int = 0
    num_linear_solver_iterations: int = 0
    linear_solver_type_used: int = 0
    initial_cost: float = 0.0
    final_cost: float = 0.0
    solve_ms: float = 0.0
    setup_ms: float = 0.0
    spmv_ms_total: float = 0.0
    spmv_launches: int = 0
    kernel_launches: int = 0

    def IsSolutionUsable(self) -> bool:
        return self.termination_type in (CONVERGENCE, NO_CONVERGENCE)

    @staticmethod
    def from_c(c) -> "BundleAdjustmentSummary":
        return BundleAdjustmentSummary(**{f[0]: getattr(c, f[0]) for f in _CSummary._fields_})


# ------------------------------------------------------------------------------------------------ scene types
@dataclass
class Camera:
    camera_id: int
    model_id: int
    params: np.ndarray           # float64
    has_prior_focal_length: bool = False


@dataclass
class Point2D:
    xy: np.ndarray
    point3D_id: int = -1


@dataclass
class Image:
    image_id: int
    camera_id: int
    cam_from_world: np.ndarray   # 7: qx qy qz qw tx ty tz (Rigid3d::params); with rigs: derived, the frame holds the pose
    points2D: List[Point2D] = field(default_factory=list)
    frame_id: Optional[int] = None   # None = trivial frame (frame id == image id, the image is its rig's reference sensor)


@dataclass
class Rig:
    """scene/rig.h: the reference sensor defines the rig frame, the other sensors carry sensor_from_rig.  A sensor is a
    camera (sensor_t{CAMERA, camera_id}); a camera belongs to exactly one rig."""
    rig_id: int
    ref_sensor: int                                          # camera id of the reference sensor
    sensors: Dict[int, np.ndarray] = field(default_factory=dict)   # non-reference sensors: camera id -> sensor_from_rig (7)


@dataclass
class Frame:
    frame_id: int
    rig_id: int
    rig_from_world: np.ndarray   # 7


@dataclass
class Point3D:
    xyz: np.ndarray
    track: List[tuple] = field(default_factory=list)   # (image_id, point2D_idx)


@dataclass
class Reconstruction:
    cameras: Dict[int, Camera] = field(default_factory=dict)
    images: Dict[int, Image] = field(default_factory=dict)
    points3D: Dict[int, Point3D] = field(default_factory=dict)
    rigs: Dict[int, Rig] = field(default_factory=dict)       # empty = trivial frames throughout
    frames: Dict[int, Frame] = field(default_factory=dict)
    reg_frame_ids: List[int] = field(default_factory=list)   # registered frames, in registration order

    def RegisterFrame(self, frame_id):
        """Reconstruction::RegisterFrame: a frame with a pose joins the registered set (once)."""
        if frame_id not in self.reg_frame_ids:
            self.reg_frame_ids.append(frame_id)

    def DeRegisterFrame(self, frame_id):
        """Reconstruction::DeRegisterFrame: leaves the registered set, its images' observations are deleted and its pose
        is reset.  A frame that is not registered is ignored."""
        if frame_id not in self.reg_frame_ids:
            return
        self.reg_frame_ids.remove(frame_id)
        for image_id, im in self.images.items():
            if im.frame_id != frame_id:
                continue
            for k, p2 in enumerate(im.points2D):
                if p2.point3D_id in self.points3D:
                    pt = self.points3D[p2.point3D_id]
                    pt.track = [t for t in pt.track if t != (image_id, k)]
                p2.point3D_id = -1
        self.frames[frame_id].rig_from_world = None

    def RegFrameIds(self) -> List[int]:
        return list(self.reg_frame_ids)

    def IsRefInFrame(self, image_id) -> bool:
        """Image::IsRefInFrame: the image's camera is the reference sensor of its frame's rig."""
        im = self.images[image_id]
        return im.frame_id is None or self.rigs[self.frames[im.frame_id].rig_id].ref_sensor == im.camera_id


class BundleAdjustmentConfig:
    """BundleAdjustmentConfig (bundle_adjustment.h:77-151); with trivial frames the frame id is the image id."""

    def __init__(self):
        self.fixed_gauge_ = UNSPECIFIED_GAUGE
        self.image_ids_ = set()
        self.constant_cam_intrinsics_ = set()
        self.constant_rig_from_world_poses_ = set()
        self.constant_sensor_from_rig_poses_ = set()
        self.variable_point3D_ids_ = set()
        self.constant_point3D_ids_ = set()
        self.ignored_point3D_ids_ = set()

    def FixGauge(self, gauge): self.fixed_gauge_ = gauge
    def FixedGauge(self): return self.fixed_gauge_
    def NumImages(self): return len(self.image_ids_)
    def AddImage(self, image_id): self.image_ids_.add(image_id)
    def HasImage(self, image_id): return image_id in self.image_ids_
    def RemoveImage(self, image_id): self.image_ids_.discard(image_id)
    def SetConstantCamIntrinsics(self, camera_id): self.constant_cam_intrinsics_.add(camera_id)
    def SetVariableCamIntrinsics(self, camera_id): self.constant_cam_intrinsics_.discard(camera_id)
    def HasConstantCamIntrinsics(self, camera_id): return camera_id in self.constant_cam_intrinsics_
    def SetConstantRigFromWorldPose(self, frame_id): self.constant_rig_from_world_poses_.add(frame_id)
    def SetVariableRigFromWorldPose(self, frame_id): self.constant_rig_from_world_poses_.discard(frame_id)
    def HasConstantRigFromWorldPose(self, frame_id): return frame_id in self.constant_rig_from_world_poses_
    def SetConstantSensorFromRigPose(self, sensor_id): self.constant_sensor_from_rig_poses_.add(sensor_id)       # sensor id = camera id
    def SetVariableSensorFromRigPose(self, sensor_id): self.constant_sensor_from_rig_poses_.discard(sensor_id)
    def HasConstantSensorFromRigPose(self, sensor_id): return sensor_id in self.constant_sensor_from_rig_poses_
    def AddVariablePoint(self, pid): self.variable_point3D_ids_.add(pid)
    def AddConstantPoint(self, pid): self.constant_point3D_ids_.add(pid)
    def IgnorePoint(self, pid): self.ignored_point3D_ids_.add(pid)
    def HasPoint(self, pid): return pid in self.variable_point3D_ids_ or pid in self.constant_point3D_ids_
    def IsIgnoredPoint(self, pid): return pid in self.ignored_point3D_ids_
    def Images(self): return self.image_ids_
    def VariablePoints(self): return self.variable_point3D_ids_
    def ConstantPoints(self): return self.constant_point3D_ids_


class FlatProblem:
    """Arrays behind a b200ba_problem (kept alive here)."""

    def __init__(self, poses, pose_constant, pose_fixed_dim, cam_model, cam_off, cam_params, cam_constant, points,
                 point_constant, obs_pose, obs_cam, obs_point, obs_xy):
        c = np.ascontiguousarray
        self.poses = c(poses, np.float64).reshape(-1, 7)
        self.pose_constant = c(pose_constant, np.uint8)
        self.pose_fixed_dim = c(pose_fixed_dim, np.int8)
        self.cam_model = c(cam_model, np.int32)
        self.cam_off = c(cam_off, np.int32)
        self.cam_params = c(cam_params, np.float64)
        self.cam_constant = c(cam_constant, np.uint8)
        self.points = c(points, np.float64).reshape(-1, 3)
        self.point_constant = c(point_constant, np.uint8)
        self.obs_pose = c(obs_pose, np.int32)
        self.obs_cam = c(obs_cam, np.int32)
        self.obs_point = c(obs_point, np.int32)
        self.obs_xy = c(obs_xy, np.float64).reshape(-1, 2)
        self.num_config_images = 0      # config.NumImages(); 0 = poses that appear in observations
        # rigs: non-reference sensors (cam_from_world = sensor_from_rig * rig_from_world); empty for trivial frames
        self.sensors = np.zeros((0, 7), np.float64)
        self.sensor_constant = np.zeros(0, np.uint8)
        self.cam_sensor = -np.ones(len(self.cam_model), np.int32)

    def set_sensors(self, sensors, sensor_constant, cam_sensor):
        c = np.ascontiguousarray
        self.sensors = c(sensors, np.float64).reshape(-1, 7)
        self.sensor_constant = c(sensor_constant, np.uint8)
        self.cam_sensor = c(cam_sensor, np.int32)
        return self

    def copy(self):
        f = self._copy()
        f.num_config_images = self.num_config_images
        f.sensors, f.sensor_constant, f.cam_sensor = self.sensors.copy(), self.sensor_constant, self.cam_sensor
        return f

    def _copy(self):
        return FlatProblem(self.poses.copy(), self.pose_constant, self.pose_fixed_dim, self.cam_model, self.cam_off,
                           self.cam_params.copy(), self.cam_constant, self.points.copy(), self.point_constant,
                           self.obs_pose, self.obs_cam, self.obs_point, self.obs_xy)

    def to_c(self) -> _CProblem:
        p = _CProblem()
        p.num_poses = len(self.poses); p.poses = self.poses.ctypes.data_as(_f64p)
        p.pose_constant = self.pose_constant.ctypes.data_as(_u8p)
        p.pose_fixed_translation_dim = self.pose_fixed_dim.ctypes.data_as(_i8p)
        p.num_cameras = len(self.cam_model); p.camera_model_id = self.cam_model.ctypes.data_as(_i32p)
        p.camera_param_offset = self.cam_off.ctypes.data_as(_i32p)
        p.camera_params = self.cam_params.ctypes.data_as(_f64p)
        p.camera_constant = self.cam_constant.ctypes.data_as(_u8p)
        p.num_points = len(self.points); p.points = self.points.ctypes.data_as(_f64p)
        p.point_constant = self.point_constant.ctypes.data_as(_u8p)
        p.num_observations = len(self.obs_pose)
        p.obs_pose_idx = self.obs_pose.ctypes.data_as(_i32p); p.obs_camera_idx = self.obs_cam.ctypes.data_as(_i32p)
        p.obs_point_idx = self.obs_point.ctypes.data_as(_i32p); p.obs_xy = self.obs_xy.ctypes.data_as(_f64p)
        p.num_config_images = int(self.num_config_images)
        p.num_sensors = len(self.sensors)
        if len(self.sensors):
            p.sensor_from_rig = self.sensors.ctypes.data_as(_f64p)
            p.sensor_constant = self.sensor_constant.ctypes.data_as(_u8p)
        p.camera_sensor_idx = self.cam_sensor.ctypes.data_as(_i32p)
        return p


def _bind(lib):
    if getattr(lib, "_ba_bound", False):
        return lib
    lib.b200ba_comm_unique_id.argtypes = [ctypes.c_void_p]
    lib.b200ba_comm_init.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    lib.b200ba_comm_destroy.argtypes = [ctypes.c_void_p]
    lib.b200ba_comm_destroy.restype = None
    lib.b200ba_comm_peer_memory.argtypes = [ctypes.c_void_p]
    lib.b200ba_comm_peer_memory.restype = ctypes.c_int
    lib.b200ba_solve_sharded.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.c_void_p,
                                         ctypes.POINTER(_CSummary)]
    lib.b200ba_options_init.argtypes = [ctypes.POINTER(_COptions)]
    lib.b200ba_options_init.restype = None
    lib.b200ba_solve.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.POINTER(_CSummary)]
    lib.b200ba_fix_gauge_two_cams_from_world.argtypes = [ctypes.POINTER(_CProblem), ctypes.POINTER(_COptions), _u8p, _i8p]
    lib.b200ba_last_error.restype = ctypes.c_char_p
    lib._ba_bound = True
    return lib


class BundleAdjustmentError(RuntimeError):
    pass


def solve_flat(options: BundleAdjustmentOptions, flat: FlatProblem) -> BundleAdjustmentSummary:
    """b200ba_solve on a flat problem; flat.poses / cam_params / points are updated in place."""
    lib = _bind(load_library())
    co, cp, cs = options.to_c(), flat.to_c(), _CSummary()
    rc = lib.b200ba_solve(ctypes.byref(co), ctypes.byref(cp), ctypes.byref(cs))
    if rc != 0:
        raise BundleAdjustmentError(f"b200ba_solve failed ({rc}): {lib.b200ba_last_error().decode()}")
    return BundleAdjustmentSummary.from_c(cs)


# ------------------------------------------------------------------------------------------------ multi-GPU
def shard_flat_problem(flat: FlatProblem, rank: int, world: int) -> "FlatProblem":
    """Point sharding (SURVEY.md §8e): contiguous point ranges balanced by observation count; a rank receives its
    points and ALL their observations, poses and cameras are replicated.  Returns the local FlatProblem; its
    `point_ids` attribute maps local points back to the global problem."""
    npts = len(flat.points)
    counts = np.bincount(flat.obs_point, minlength=npts).astype(np.int64)
    csum = np.concatenate([[0], np.cumsum(counts)])
    total = csum[-1]
    bounds = [int(np.searchsorted(csum, total * r / world, side="left")) for r in range(world)] + [npts]
    bounds[0] = 0
    lo, hi = bounds[rank], bounds[rank + 1]
    sel = (flat.obs_point >= lo) & (flat.obs_point < hi)
    local = FlatProblem(flat.poses.copy(), flat.pose_constant, flat.pose_fixed_dim, flat.cam_model, flat.cam_off,
                        flat.cam_params.copy(), flat.cam_constant, flat.points[lo:hi].copy(), flat.point_constant[lo:hi],
                        flat.obs_pose[sel], flat.obs_cam[sel], flat.obs_point[sel] - lo, flat.obs_xy[sel])
    local.point_ids = np.arange(lo, hi)
    local.num_config_images = flat.num_config_images or int(len(np.unique(flat.obs_pose)))
    local.sensors, local.sensor_constant, local.cam_sensor = flat.sensors.copy(), flat.sensor_constant, flat.cam_sensor
    return local


class BAComm:
    """NCCL communicator of the sharded solve.  `id_bytes` comes from rank 0 (unique_id()) and is distributed by the
    launcher (torch.distributed broadcast, a multiprocessing queue, ...).  Call on the rank's CUDA device."""

    def __init__(self, id_bytes: bytes, rank: int, world: int):
        self._lib = _bind(load_library())
        self._h = ctypes.c_void_p()
        buf = ctypes.create_string_buffer(id_bytes, 128)
        rc = self._lib.b200ba_comm_init(buf, rank, world, ctypes.byref(self._h))
        if rc != 0:
            raise BundleAdjustmentError(f"b200ba_comm_init failed ({rc}): {self._lib.b200ba_last_error().decode()}")
        self.rank, self.world = rank, world

    @staticmethod
    def unique_id() -> bytes:
        lib = _bind(load_library())
        buf = ctypes.create_string_buffer(128)
        rc = lib.b200ba_comm_unique_id(buf)
        if rc != 0:
            raise BundleAdjustmentError(f"b200ba_comm_unique_id failed ({rc}): {lib.b200ba_last_error().decode()}")
        return buf.raw

    def peer_memory(self) -> bool:
        """True once the small collectives run as the library's own one-shot all-reduce over NVLink peer memory."""
        return bool(self._h) and bool(self._lib.b200ba_comm_peer_memory(self._h))

    def close(self):
        if self._h:
            self._lib.b200ba_comm_destroy(self._h)
            self._h = ctypes.c_void_p()


def solve_flat_sharded(options: "BundleAdjustmentOptions", local: FlatProblem, comm: BAComm) -> "BundleAdjustmentSummary":
    """b200ba_solve_sharded on this rank's shard; poses / cam_params come back identical on every rank."""
    lib = _bind(load_library())
    co, cp, cs = options.to_c(), local.to_c(), _CSummary()
    rc = lib.b200ba_solve_sharded(ctypes.byref(co), ctypes.byref(cp), comm._h, ctypes.byref(cs))
    if rc != 0:
        raise BundleAdjustmentError(f"b200ba_solve_sharded failed ({rc}): {lib.b200ba_last_error().decode()}")
    return BundleAdjustmentSummary.from_c(cs)


def flatten_reconstruction(options: BundleAdjustmentOptions, config: BundleAdjustmentConfig, rec: Reconstruction):
    """DefaultBundleAdjuster's problem assembly (bundle_adjustment_ceres.cc:606-664,688-888) -> FlatProblem.
    Returns (flat, image_ids, camera_ids, point_ids) with the id lists giving the flat order."""
    if rec.frames:
        return _flatten_reconstruction_rigs(options, config, rec)
    image_ids = sorted(rec.images.keys())            # poses of images outside the config are constant
    camera_ids = sorted(rec.cameras.keys())
    point_ids = sorted(rec.points3D.keys())
    pose_idx = {i: k for k, i in enumerate(image_ids)}
    cam_idx = {c: k for k, c in enumerate(camera_ids)}
    pt_idx = {p: k for k, p in enumerate(point_ids)}
    cfg_images = sorted(config.Images())
    obs_pose, obs_cam, obs_point, obs_xy = [], [], [], []
    point_num_obs = {}
    # AddImageToProblem (:688-751)
    parameterized_images = set()                     # images that contributed >= 1 observation (:745-748)
    for image_id in cfg_images:
        im = rec.images[image_id]
        for p2 in im.points2D:
            pid = p2.point3D_id
            if pid < 0 or pid not in rec.points3D or config.IsIgnoredPoint(pid):
                continue
            if len(rec.points3D[pid].track) < options.min_track_length:
                continue
            point_num_obs[pid] = point_num_obs.get(pid, 0) + 1
            parameterized_images.add(image_id)
            obs_pose.append(pose_idx[image_id]); obs_cam.append(cam_idx[im.camera_id]); obs_point.append(pt_idx[pid])
            obs_xy.append(p2.xy)
    # AddPointToProblem (:829-888): explicit config points get the observations from images outside the config
    extra_const_pose = set()
    for pid in sorted(config.VariablePoints() | config.ConstantPoints()):
        pt = rec.points3D[pid]
        if options.min_track_length > 0 and len(pt.track) < options.min_track_length:   # :835-838
            continue
        if point_num_obs.get(pid, 0) == len(pt.track):
            continue
        for image_id, p2_idx in pt.track:
            if config.HasImage(image_id):
                continue
            im = rec.images[image_id]
            point_num_obs[pid] = point_num_obs.get(pid, 0) + 1
            extra_const_pose.add(image_id)
            obs_pose.append(pose_idx[image_id]); obs_cam.append(cam_idx[im.camera_id]); obs_point.append(pt_idx[pid])
            obs_xy.append(im.points2D[p2_idx].xy)
    pose_constant = np.ones(len(image_ids), np.uint8)
    for image_id in cfg_images:
        if not config.HasConstantRigFromWorldPose(image_id):
            pose_constant[pose_idx[image_id]] = 0
    # cameras that only appear through constant-pose factors of outside images stay constant (:863-878)
    cam_in_cfg = {rec.images[i].camera_id for i in cfg_images if i in parameterized_images}
    cam_constant = np.array([1 if (c not in cam_in_cfg or config.HasConstantCamIntrinsics(c)) else 0 for c in camera_ids], np.uint8)
    # ParameterizePoints (:540-565)
    point_constant = np.ones(len(point_ids), np.uint8)
    for pid, n in point_num_obs.items():
        if options.refine_points3D and len(rec.points3D[pid].track) <= n:
            point_constant[pt_idx[pid]] = 0
    for pid in config.ConstantPoints():
        point_constant[pt_idx[pid]] = 1
    cam_off, off = [], 0
    for c in camera_ids:
        cam_off.append(off); off += MODEL_NUM_PARAMS[rec.cameras[c].model_id]
    flat = FlatProblem(
        np.stack([rec.images[i].cam_from_world for i in image_ids]) if image_ids else np.zeros((0, 7)),
        pose_constant, -np.ones(len(image_ids), np.int8),
        [rec.cameras[c].model_id for c in camera_ids], cam_off,
        np.concatenate([rec.cameras[c].params for c in camera_ids]) if camera_ids else np.zeros(0), cam_constant,
        np.stack([rec.points3D[p].xyz for p in point_ids]) if point_ids else np.zeros((0, 3)), point_constant,
        obs_pose, obs_cam, obs_point, np.asarray(obs_xy, np.float64).reshape(-1, 2))
    flat.num_config_images = config.NumImages()
    flat.parameterized_image_ids = parameterized_images
    return flat, image_ids, camera_ids, point_ids


def _rigid_compose(a, b):
    """(a * b): x -> a(b(x)) for 7-vectors qx qy qz qw tx ty tz."""
    from .synthetic import _quat_mul, _quat_rotate
    q = _quat_mul(a[None, :4], b[None, :4])[0]
    t = _quat_rotate(a[None, :4], b[None, 4:])[0] + a[4:]
    return np.concatenate([q, t])


def _rigid_inverse(a):
    from .synthetic import _quat_rotate
    qi = np.array([-a[0], -a[1], -a[2], a[3]])
    return np.concatenate([qi, -_quat_rotate(qi[None], a[None, 4:])[0]])


def _flatten_reconstruction_rigs(options, config, rec):
    """flatten_reconstruction for reconstructions with rigs and frames (AddImageWithNonTrivialFrame, ParameterizeRigsAndFrames,
    the rig-aware FixGaugeWithTwoCamsFromWorld: bundle_adjustment_ceres.cc:308-417,470-538,752-827).  Flat layout: pose k =
    frame k (ascending frame id) holding rig_from_world, followed by one CONSTANT pose per image outside the config that
    a config point brings in (a copy of its frame's rig_from_world: the reference bakes those observations with a constant
    pose, :846-878); sensor s = the s-th non-reference camera in ascending camera id.  The gauge is applied here.
    Returns (flat, frame_ids, camera_ids, point_ids); flat.sensor_camera_ids lists the sensors' camera ids.
    One deliberate difference: for an outside image on a NON-reference sensor whose sensor_from_rig is being refined the
    reference freezes the product sensor_from_rig * rig_from_world; here the frozen rig_from_world is composed with the
    current sensor_from_rig (the flat problem ties the sensor to the camera, not to the observation)."""
    frame_ids, camera_ids, point_ids = sorted(rec.frames), sorted(rec.cameras), sorted(rec.points3D)
    for im in rec.images.values():
        if im.frame_id not in rec.frames:
            raise BundleAdjustmentError(f"image {im.image_id}: a reconstruction with frames needs a frame for every image")
    frame_idx = {f: k for k, f in enumerate(frame_ids)}
    cam_idx = {c: k for k, c in enumerate(camera_ids)}
    pt_idx = {p: k for k, p in enumerate(point_ids)}
    cam_rig = {}
    for r in rec.rigs.values():
        cam_rig[r.ref_sensor] = r.rig_id
        for c in r.sensors:
            cam_rig[c] = r.rig_id
    sensor_cams = [c for c in camera_ids if c in cam_rig and rec.rigs[cam_rig[c]].ref_sensor != c]
    sensor_idx = {c: k for k, c in enumerate(sensor_cams)}
    cfg_images = sorted(config.Images())
    obs_pose, obs_cam, obs_point, obs_xy = [], [], [], []
    point_num_obs, parameterized_images = {}, []
    for image_id in cfg_images:                       # AddImageToProblem (:688-827)
        im = rec.images[image_id]
        n0 = len(obs_pose)
        for p2 in im.points2D:
            pid = p2.point3D_id
            if pid < 0 or pid not in rec.points3D or config.IsIgnoredPoint(pid):
                continue
            if len(rec.points3D[pid].track) < options.min_track_length:
                continue
            point_num_obs[pid] = point_num_obs.get(pid, 0) + 1
            obs_pose.append(frame_idx[im.frame_id]); obs_cam.append(cam_idx[im.camera_id]); obs_point.append(pt_idx[pid])
            obs_xy.append(p2.xy)
        if len(obs_pose) > n0:
            parameterized_images.append(image_id)
    poses = [rec.frames[f].rig_from_world for f in frame_ids]
    extra_pose_of_image = {}
    for pid in sorted(config.VariablePoints() | config.ConstantPoints()):        # AddPointToProblem (:829-888)
        pt = rec.points3D[pid]
        if options.min_track_length > 0 and len(pt.track) < options.min_track_length:
            continue
        if point_num_obs.get(pid, 0) == len(pt.track):
            continue
        for image_id, p2_idx in pt.track:
            if config.HasImage(image_id):
                continue
            im = rec.images[image_id]
            if image_id not in extra_pose_of_image:
                extra_pose_of_image[image_id] = len(poses)
                poses.append(rec.frames[im.frame_id].rig_from_world.copy())
            point_num_obs[pid] = point_num_obs.get(pid, 0) + 1
            obs_pose.append(extra_pose_of_image[image_id]); obs_cam.append(cam_idx[im.camera_id]); obs_point.append(pt_idx[pid])
            obs_xy.append(im.points2D[p2_idx].xy)
    num_poses = len(poses)
    pose_constant = np.ones(num_poses, np.uint8)
    for image_id in cfg_images:
        f = rec.images[image_id].frame_id
        if not config.HasConstantRigFromWorldPose(f):
            pose_constant[frame_idx[f]] = 0
    cam_in_cfg = {rec.images[i].camera_id for i in parameterized_images}
    cam_constant = np.array([1 if (c not in cam_in_cfg or config.HasConstantCamIntrinsics(c)) else 0 for c in camera_ids], np.uint8)
    point_constant = np.ones(len(point_ids), np.uint8)
    for pid, n in point_num_obs.items():
        if options.refine_points3D and len(rec.points3D[pid].track) <= n:
            point_constant[pt_idx[pid]] = 0
    for pid in config.ConstantPoints():
        point_constant[pt_idx[pid]] = 1
    # ParameterizeRigsAndFrames (:470-538): sensor_from_rig constant when not refined, constant in the config, or when the
    # rig's reference sensor is not part of the problem
    # (a sensor_from_rig is a parameter block only through a parameterized image of the config on that camera, :752-827;
    # images outside the config contribute constant-pose observations)
    sensor_constant = np.array([1 if (not options.refine_sensor_from_rig or config.HasConstantSensorFromRigPose(c)
                                      or c not in cam_in_cfg) else 0 for c in sensor_cams], np.uint8)
    param_rigs = {rec.frames[rec.images[i].frame_id].rig_id for i in parameterized_images}
    for rig_id in param_rigs:
        rig = rec.rigs[rig_id]
        if rig.ref_sensor not in cam_in_cfg:
            for c in rig.sensors:
                sensor_constant[sensor_idx[c]] = 1
    cam_sensor = np.array([sensor_idx.get(c, -1) for c in camera_ids], np.int32)
    cam_off, off = [], 0
    for c in camera_ids:
        cam_off.append(off); off += MODEL_NUM_PARAMS[rec.cameras[c].model_id]
    flat = FlatProblem(np.stack(poses) if poses else np.zeros((0, 7)), pose_constant, -np.ones(num_poses, np.int8),
                       [rec.cameras[c].model_id for c in camera_ids], cam_off,
                       np.concatenate([rec.cameras[c].params for c in camera_ids]) if camera_ids else np.zeros(0), cam_constant,
                       np.stack([rec.points3D[p].xyz for p in point_ids]) if point_ids else np.zeros((0, 3)), point_constant,
                       obs_pose, obs_cam, obs_point, np.asarray(obs_xy, np.float64).reshape(-1, 2))
    flat.set_sensors(np.stack([rec.rigs[cam_rig[c]].sensors[c] for c in sensor_cams]) if sensor_cams else np.zeros((0, 7)),
                     sensor_constant, cam_sensor)
    flat.num_config_images = config.NumImages()
    flat.parameterized_image_ids = set(parameterized_images)
    flat.sensor_camera_ids = sensor_cams
    flat.num_frames = len(frame_ids)
    # ---- gauge
    three_points = config.FixedGauge() == THREE_POINTS
    if config.FixedGauge() == TWO_CAMS_FROM_WORLD and options.refine_rig_from_world:
        def const_sensor(image_id):       # IsParameterizedConstSensor (:324-343)
            s = sensor_idx.get(rec.images[image_id].camera_id, -1)
            return s < 0 or bool(flat.sensor_constant[s])
        image1 = image2 = None
        dim2, done = 0, False
        for i in parameterized_images:
            if config.HasConstantRigFromWorldPose(rec.images[i].frame_id) and const_sensor(i):
                if image1 is None:
                    image1 = i
                elif rec.images[image1].frame_id != rec.images[i].frame_id:
                    done = True             # two frames are already fixed
                    break
        if not done:
            for i in parameterized_images:
                f = rec.images[i].frame_id
                if image1 is None and const_sensor(i):
                    image1 = i
                elif (image1 is not None and rec.images[image1].frame_id != f and const_sensor(i)
                      and not config.HasConstantRigFromWorldPose(f)):       # its rig_from_world is a parameter block
                    base = _rigid_compose(rec.frames[rec.images[image1].frame_id].rig_from_world,
                                          _rigid_inverse(rec.frames[f].rig_from_world))[4:]
                    mi = int(np.argmax(np.abs(base)))
                    if abs(base[mi]) > 1e-9:
                        image2, dim2 = i, mi
                        break
            if image1 is None or image2 is None:
                three_points = True         # "Falling back to fixing Gauge with three points" (:390-394)
            else:
                f1, f2 = rec.images[image1].frame_id, rec.images[image2].frame_id
                flat.pose_constant[frame_idx[f1]] = 1
                if not config.HasConstantRigFromWorldPose(f2):
                    flat.pose_fixed_dim[frame_idx[f2]] = dim2
    if three_points:
        fix_gauge_three_points(flat)
    return flat, frame_ids, camera_ids, point_ids


class _CScene(ctypes.Structure):
    _fields_ = [("num_images", ctypes.c_int), ("image_id", ctypes.POINTER(ctypes.c_uint32)), ("image_camera", _i32p),
                ("cam_from_world", _f64p), ("point2D_offset", ctypes.POINTER(ctypes.c_int64)), ("point2D_xy", _f64p),
                ("point2D_point3D", ctypes.POINTER(ctypes.c_int64)), ("num_cameras", ctypes.c_int), ("camera_model_id", _i32p),
                ("camera_param_offset", _i32p), ("camera_params", _f64p), ("num_points3D", ctypes.c_int64), ("xyz", _f64p),
                ("track_offset", ctypes.POINTER(ctypes.c_int64)), ("track_image", _i32p), ("track_point2D", _i32p),
                ("num_frames", ctypes.c_int), ("image_frame", _i32p), ("rig_from_world", _f64p), ("frame_rig", _i32p),
                ("num_rigs", ctypes.c_int), ("rig_ref_camera", _i32p), ("camera_rig", _i32p), ("camera_sensor_from_rig", _f64p)]


class _CConfig(ctypes.Structure):
    _fields_ = [("image_in_config", _u8p), ("image_constant_pose", _u8p), ("camera_constant", _u8p), ("point_variable", _u8p),
                ("point_constant", _u8p), ("point_ignored", _u8p), ("fixed_gauge", ctypes.c_int), ("min_track_length", ctypes.c_int),
                ("frame_constant_pose", _u8p), ("camera_constant_sensor_from_rig", _u8p)]


def assemble_reconstruction(options: BundleAdjustmentOptions, config: BundleAdjustmentConfig, rec: Reconstruction):
    """b200ba_assemble: the C++ problem assembly (DefaultBundleAdjuster's constructor incl. the two-cams gauge) on flat
    views of the reconstruction.  Returns (flat, image_ids, camera_ids, point_ids) like flatten_reconstruction."""
    lib = _bind(load_library())
    i64p, u32p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_uint32)
    lib.b200ba_assemble.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CScene), ctypes.POINTER(_CConfig), ctypes.POINTER(ctypes.c_void_p)]
    lib.b200ba_assembly_problem.argtypes = [ctypes.c_void_p]; lib.b200ba_assembly_problem.restype = ctypes.POINTER(_CProblem)
    lib.b200ba_assembly_free.argtypes = [ctypes.c_void_p]
    image_ids, camera_ids, point_ids = sorted(rec.images), sorted(rec.cameras), sorted(rec.points3D)
    img_idx = {i: k for k, i in enumerate(image_ids)}; cam_idx = {c: k for k, c in enumerate(camera_ids)}; pt_idx = {p: k for k, p in enumerate(point_ids)}
    c = np.ascontiguousarray
    ids = c(image_ids, np.uint32); icam = c([cam_idx[rec.images[i].camera_id] for i in image_ids], np.int32)
    poses = c(np.stack([rec.images[i].cam_from_world for i in image_ids]) if image_ids else np.zeros((0, 7)), np.float64)
    p2off = np.zeros(len(image_ids) + 1, np.int64)
    p2off[1:] = np.cumsum([len(rec.images[i].points2D) for i in image_ids])
    p2xy = c([p.xy for i in image_ids for p in rec.images[i].points2D], np.float64).reshape(-1, 2)
    p2pt = c([pt_idx.get(p.point3D_id, -1) if p.point3D_id >= 0 else -1 for i in image_ids for p in rec.images[i].points2D], np.int64)
    cmodel = c([rec.cameras[k].model_id for k in camera_ids], np.int32)
    coff = np.zeros(len(camera_ids), np.int32); off = 0
    for k, cid in enumerate(camera_ids):
        coff[k] = off; off += MODEL_NUM_PARAMS[rec.cameras[cid].model_id]
    cparams = c(np.concatenate([rec.cameras[k].params for k in camera_ids]) if camera_ids else np.zeros(0), np.float64)
    xyz = c(np.stack([rec.points3D[p].xyz for p in point_ids]) if point_ids else np.zeros((0, 3)), np.float64)
    toff = np.zeros(len(point_ids) + 1, np.int64)
    toff[1:] = np.cumsum([len(rec.points3D[p].track) for p in point_ids])
    timg = c([img_idx[i] for p in point_ids for i, _ in rec.points3D[p].track], np.int32)
    tp2 = c([k for p in point_ids for _, k in rec.points3D[p].track], np.int32)
    flags = lambda keys, pred: c([1 if pred(k) else 0 for k in keys], np.uint8)
    f_in = flags(image_ids, config.HasImage); f_cp = flags(image_ids, config.HasConstantRigFromWorldPose)
    f_cc = flags(camera_ids, config.HasConstantCamIntrinsics)
    f_pv = flags(point_ids, lambda p: p in config.VariablePoints()); f_pc = flags(point_ids, lambda p: p in config.ConstantPoints())
    f_pi = flags(point_ids, config.IsIgnoredPoint)
    P = lambda a, t: a.ctypes.data_as(t)
    sc = _CScene(len(image_ids), P(ids, u32p), P(icam, _i32p), P(poses, _f64p), P(p2off, i64p), P(p2xy, _f64p), P(p2pt, i64p),
                 len(camera_ids), P(cmodel, _i32p), P(coff, _i32p), P(cparams, _f64p), len(point_ids), P(xyz, _f64p), P(toff, i64p),
                 P(timg, _i32p), P(tp2, _i32p))
    cf = _CConfig(P(f_in, _u8p), P(f_cp, _u8p), P(f_cc, _u8p), P(f_pv, _u8p), P(f_pc, _u8p), P(f_pi, _u8p), int(config.FixedGauge()),
                  int(options.min_track_length))
    frame_ids = sorted(rec.frames)
    if frame_ids:       # rigs and frames
        rig_ids = sorted(rec.rigs)
        fr_idx = {f: k for k, f in enumerate(frame_ids)}; rig_idx = {r: k for k, r in enumerate(rig_ids)}
        cam_rig_id = {}
        for r in rec.rigs.values():
            cam_rig_id[r.ref_sensor] = r.rig_id
            for cc in r.sensors:
                cam_rig_id[cc] = r.rig_id
        img_frame = c([fr_idx[rec.images[i].frame_id] for i in image_ids], np.int32)
        rfw = c(np.stack([rec.frames[f].rig_from_world for f in frame_ids]), np.float64)
        frame_rig = c([rig_idx[rec.frames[f].rig_id] for f in frame_ids], np.int32)
        rig_ref = c([cam_idx[rec.rigs[r].ref_sensor] for r in rig_ids], np.int32)
        cam_rig = c([rig_idx[cam_rig_id[k]] for k in camera_ids], np.int32)
        ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
        cam_sfr = c(np.stack([rec.rigs[cam_rig_id[k]].sensors.get(k, ident) for k in camera_ids]), np.float64)
        f_fc = flags(frame_ids, config.HasConstantRigFromWorldPose); f_sc = flags(camera_ids, config.HasConstantSensorFromRigPose)
        sc.num_frames = len(frame_ids); sc.image_frame = P(img_frame, _i32p); sc.rig_from_world = P(rfw, _f64p)
        sc.frame_rig = P(frame_rig, _i32p); sc.num_rigs = len(rig_ids); sc.rig_ref_camera = P(rig_ref, _i32p)
        sc.camera_rig = P(cam_rig, _i32p); sc.camera_sensor_from_rig = P(cam_sfr, _f64p)
        cf.frame_constant_pose = P(f_fc, _u8p); cf.camera_constant_sensor_from_rig = P(f_sc, _u8p)
    co, h = options.to_c(), ctypes.c_void_p()
    rc = lib.b200ba_assemble(ctypes.byref(co), ctypes.byref(sc), ctypes.byref(cf), ctypes.byref(h))
    if rc != 0:
        raise BundleAdjustmentError(f"b200ba_assemble failed ({rc}): {lib.b200ba_last_error().decode()}")
    try:
        pr = lib.b200ba_assembly_problem(h).contents
        n_obs, n_cam, n_pt, n_img = pr.num_observations, pr.num_cameras, pr.num_points, pr.num_poses
        arr = lambda ptr, n, dt: np.ctypeslib.as_array(ptr, shape=(max(n, 1),))[:n].astype(dt, copy=True) if n else np.zeros(0, dt)
        flat = FlatProblem(arr(pr.poses, 7 * n_img, np.float64), arr(pr.pose_constant, n_img, np.uint8),
                           arr(pr.pose_fixed_translation_dim, n_img, np.int8), arr(pr.camera_model_id, n_cam, np.int32),
                           arr(pr.camera_param_offset, n_cam, np.int32), arr(pr.camera_params, len(cparams), np.float64),
                           arr(pr.camera_constant, n_cam, np.uint8), arr(pr.points, 3 * n_pt, np.float64),
                           arr(pr.point_constant, n_pt, np.uint8), arr(pr.obs_pose_idx, n_obs, np.int32),
                           arr(pr.obs_camera_idx, n_obs, np.int32), arr(pr.obs_point_idx, n_obs, np.int32),
                           arr(pr.obs_xy, 2 * n_obs, np.float64))
        flat.num_config_images = int(pr.num_config_images)
        if pr.num_sensors > 0 or frame_ids:
            ns = int(pr.num_sensors)
            flat.set_sensors(arr(pr.sensor_from_rig, 7 * ns, np.float64), arr(pr.sensor_constant, ns, np.uint8),
                             arr(pr.camera_sensor_idx, n_cam, np.int32))
            flat.sensor_camera_ids = [camera_ids[k] for k in range(n_cam) if flat.cam_sensor[k] >= 0]
            flat.num_frames = len(frame_ids)
    finally:
        lib.b200ba_assembly_free(h)
    return flat, (frame_ids if frame_ids else image_ids), camera_ids, point_ids


def fix_gauge_three_points(flat: FlatProblem) -> int:
    """FixGaugeWithThreePoints (bundle_adjustment_ceres.cc:270-306) on a flat problem: already-constant observed points
    count first, then variable ones are fixed, until three linearly independent coordinate vectors are held (ascending
    point index; the reference walks a hash map).  Returns the number of points holding the gauge."""
    observed = np.zeros(len(flat.points), bool)
    observed[flat.obs_point] = True
    basis, max_pivot = [], 0.0
    flat.point_constant = flat.point_constant.copy()

    def maybe_add(X):
        nonlocal max_pivot
        if len(basis) >= 3:
            return False
        r = np.array(X, np.float64)
        for q in basis:
            r = r - (r @ q) * q
        nr, nx = float(np.sqrt(r @ r)), float(np.sqrt(X @ X))
        if not nr > 3.0 * 2.220446049250313e-16 * max(max_pivot, nx):
            return False
        basis.append(r / nr); max_pivot = max(max_pivot, nx)
        return True

    for k in np.nonzero(observed & (flat.point_constant != 0))[0]:
        if len(basis) < 3:
            maybe_add(flat.points[k])
    for k in np.nonzero(observed & (flat.point_constant == 0))[0]:
        if len(basis) >= 3:
            break
        if maybe_add(flat.points[k]):
            flat.point_constant[k] = 1
    return len(basis)


class BundleAdjuster:
    """BundleAdjuster (bundle_adjustment.h:212-226), B200 backend: Solve() updates the reconstruction in place."""

    def __init__(self, options, config, reconstruction):
        self.options_, self.config_, self.reconstruction_ = options, config, reconstruction

    def Options(self): return self.options_
    def Config(self): return self.config_

    def flat_problem(self):
        """The flat problem Solve() hands to the GPU: the flattening of the reconstruction with the gauge applied.
        Returns (flat, pose_ids, camera_ids, point_ids); pose_ids are image ids, or frame ids for reconstructions with
        frames.  EstimateBACovariance reads the same problem."""
        rec = self.reconstruction_
        flat, image_ids, camera_ids, point_ids = flatten_reconstruction(self.options_, self.config_, rec)
        if rec.frames:      # rigs: the flattening applied the gauge
            return flat, image_ids, camera_ids, point_ids
        lib = _bind(load_library())
        if self.config_.FixedGauge() == TWO_CAMS_FROM_WORLD and self.options_.refine_rig_from_world:
            # gauge search runs over the images of the config in ascending id (std::set<image_t>), :346-385
            co, cp = self.options_.to_c(), flat.to_c()
            pc = flat.pose_constant.copy()
            # images outside the config are not candidates: mark them "not in problem" for the search
            in_cfg = np.array([1 if (i in self.config_.Images() and i in flat.parameterized_image_ids) else 0 for i in image_ids], np.uint8)
            sub = FlatProblem(flat.poses[in_cfg == 1], flat.pose_constant[in_cfg == 1], flat.pose_fixed_dim[in_cfg == 1],
                              flat.cam_model, flat.cam_off, flat.cam_params, flat.cam_constant, flat.points,
                              flat.point_constant, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32),
                              np.zeros((0, 2)))
            out_c = np.zeros(len(sub.poses), np.uint8); out_d = -np.ones(len(sub.poses), np.int8)
            csub = sub.to_c()
            rc = lib.b200ba_fix_gauge_two_cams_from_world(ctypes.byref(csub), ctypes.byref(co), out_c.ctypes.data_as(_u8p),
                                                          out_d.ctypes.data_as(_i8p))
            if rc == 1:     # no valid pair: the reference falls back to three fixed points (bundle_adjustment_ceres.cc:390-394)
                fix_gauge_three_points(flat)
            else:
                idx = np.nonzero(in_cfg)[0]
                flat.pose_constant[idx] = out_c
                flat.pose_fixed_dim[idx] = out_d
        elif self.config_.FixedGauge() == THREE_POINTS:
            fix_gauge_three_points(flat)
        return flat, image_ids, camera_ids, point_ids

    def _solve_flat(self, flat, pose_ids):
        return solve_flat(self.options_, flat)

    def Solve(self) -> BundleAdjustmentSummary:
        rec = self.reconstruction_
        flat, image_ids, camera_ids, point_ids = self.flat_problem()
        if rec.frames:      # poses are frames, sensors the non-reference cameras
            summary = self._solve_flat(flat, image_ids)
            for k, f in enumerate(image_ids):
                rec.frames[f].rig_from_world[:] = flat.poses[k]
            for k, c in enumerate(flat.sensor_camera_ids):
                for rig in rec.rigs.values():
                    if c in rig.sensors:
                        rig.sensors[c][:] = flat.sensors[k]
            for k, c in enumerate(camera_ids):
                n = MODEL_NUM_PARAMS[rec.cameras[c].model_id]
                rec.cameras[c].params[:] = flat.cam_params[flat.cam_off[k]:flat.cam_off[k] + n]
            for k, p in enumerate(point_ids):
                rec.points3D[p].xyz[:] = flat.points[k]
            return summary
        summary = self._solve_flat(flat, image_ids)
        # write back in place (variable blocks only changed)
        for k, i in enumerate(image_ids):
            rec.images[i].cam_from_world[:] = flat.poses[k]
        for k, c in enumerate(camera_ids):
            n = MODEL_NUM_PARAMS[rec.cameras[c].model_id]
            rec.cameras[c].params[:] = flat.cam_params[flat.cam_off[k]:flat.cam_off[k] + n]
        for k, p in enumerate(point_ids):
            rec.points3D[p].xyz[:] = flat.points[k]
        return summary


def CreateDefaultBundleAdjuster(options, config, reconstruction) -> BundleAdjuster:
    """Factory (bundle_adjustment.cc:314-336); this build has exactly one backend."""
    return BundleAdjuster(options, config, reconstruction)


# ------------------------------------------------------------------------------------------------ covariance
class BACovarianceOptions:
    """BACovarianceOptions (covariance.h): for which parameters, and the damping of the point (and, in the POSES modes,
    the intrinsics / sensor) diagonal blocks."""
    POSES, POINTS, POSES_AND_POINTS, ALL = 0, 1, 2, 3

    def __init__(self, params=3, damping=1e-8):
        self.params, self.damping = params, damping


class _CCovOptions(ctypes.Structure):
    _fields_ = [("params", ctypes.c_int), ("damping", ctypes.c_double)]


def _bind_cov(lib):
    if getattr(lib, "_cov_bound", False):
        return lib
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    lib.b200ba_estimate_covariance.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CCovOptions), ctypes.POINTER(_CProblem),
                                               ctypes.POINTER(vp)]
    lib.b200ba_estimate_covariance_with_position_priors.argtypes = [
        ctypes.POINTER(_COptions), ctypes.POINTER(_CCovOptions), ctypes.POINTER(_CProblem), ctypes.POINTER(_CPositionPriors),
        ctypes.POINTER(vp)]
    lib.b200ba_covariance_point.argtypes = [vp, i64, _f64p]
    lib.b200ba_covariance_pose.argtypes = [vp, ctypes.c_int, _f64p]
    lib.b200ba_covariance_pose_cross.argtypes = [vp, ctypes.c_int, ctypes.c_int, _f64p, _i32p, _i32p]
    lib.b200ba_covariance_camera.argtypes = [vp, ctypes.c_int, _f64p]
    lib.b200ba_covariance_sensor.argtypes = [vp, ctypes.c_int, _f64p]
    lib.b200ba_covariance_poses_all.argtypes = [vp, _f64p, _i8p]
    lib.b200ba_covariance_points_all.argtypes = [vp, _f64p, _u8p]
    lib.b200ba_covariance_info.argtypes = [vp, _f64p]
    lib.b200ba_covariance_free.argtypes = [vp]
    lib.b200ba_covariance_free.restype = None
    lib._cov_bound = True
    return lib


class FlatCovariance:
    """b200ba_covariance over flat indices (pose, camera, sensor, point index of the FlatProblem).  Every getter returns
    None where the reference returns nullopt.  close() (or garbage collection) frees the device memory."""

    def __init__(self, lib, handle, num_poses, num_points):
        self._lib, self._h, self.num_poses, self.num_points = lib, handle, num_poses, num_points

    def __del__(self):
        self.close()

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200ba_covariance_free(self._h)
            self._h = None

    def _square(self, fn, idx, cap):
        buf = np.zeros(cap)
        n = fn(self._h, idx, buf.ctypes.data_as(_f64p))
        return buf[:n * n].reshape(n, n).copy() if n else None

    def point(self, k):
        return self._square(self._lib.b200ba_covariance_point, int(k), 9)

    def pose(self, i):
        return self._square(self._lib.b200ba_covariance_pose, int(i), 36)

    def camera(self, c):
        return self._square(self._lib.b200ba_covariance_camera, int(c), 256)

    def sensor(self, s):
        return self._square(self._lib.b200ba_covariance_sensor, int(s), 36)

    def pose_cross(self, i, j):
        buf, r, c = np.zeros(36), ctypes.c_int32(), ctypes.c_int32()
        n = self._lib.b200ba_covariance_pose_cross(self._h, int(i), int(j), buf.ctypes.data_as(_f64p), ctypes.byref(r), ctypes.byref(c))
        return buf[:n].reshape(r.value, c.value).copy() if n else None

    def poses_all(self):
        """(out[num_poses, 6, 6], size[num_poses]): block i is out[i, :size[i], :size[i]]."""
        out, size = np.zeros((self.num_poses, 36)), np.zeros(self.num_poses, np.int8)
        rc = self._lib.b200ba_covariance_poses_all(self._h, out.ctypes.data_as(_f64p), size.ctypes.data_as(_i8p))
        if rc:
            raise BundleAdjustmentError(f"b200ba_covariance_poses_all failed ({rc}): {self._lib.b200ba_last_error().decode()}")
        blocks = np.zeros((self.num_poses, 6, 6))
        for i in np.nonzero(size)[0]:
            n = int(size[i])
            blocks[i, :n, :n] = out[i, :n * n].reshape(n, n)
        return blocks, size

    def points_all(self):
        """(out[num_points, 3, 3], valid[num_points])."""
        out, valid = np.zeros((self.num_points, 9)), np.zeros(self.num_points, np.uint8)
        rc = self._lib.b200ba_covariance_points_all(self._h, out.ctypes.data_as(_f64p), valid.ctypes.data_as(_u8p))
        if rc:
            raise BundleAdjustmentError(f"b200ba_covariance_points_all failed ({rc}): {self._lib.b200ba_last_error().decode()}")
        return out.reshape(-1, 3, 3), valid

    def info(self):
        """(dimension of the factorised matrix, {phase: device ms}) of the estimate."""
        ms = np.zeros(4)
        n = self._lib.b200ba_covariance_info(self._h, ms.ctypes.data_as(_f64p))
        return n, dict(zip(("setup", "build", "factorize", "inverse"), ms.tolist()))


class CovarianceNotEstimable(BundleAdjustmentError):
    pass


def estimate_covariance_flat(options: BundleAdjustmentOptions, cov_options: BACovarianceOptions, flat: FlatProblem,
                             raise_not_estimable=False, priors: Optional["FlatPositionPriors"] = None):
    """b200ba_estimate_covariance on a flat problem (rigs included), or, with `priors` (FlatPositionPriors in the frame
    of `flat`), b200ba_estimate_covariance_with_position_priors.  Returns a FlatCovariance, or None when the reduced
    matrix is rank deficient (raise_not_estimable: raise CovarianceNotEstimable with the library's message instead)."""
    lib = _bind_cov(_bind(load_library()))
    co, cc, cp, h = options.to_c(), _CCovOptions(int(cov_options.params), float(cov_options.damping)), flat.to_c(), ctypes.c_void_p()
    if priors is None:
        name = "b200ba_estimate_covariance"
        rc = lib.b200ba_estimate_covariance(ctypes.byref(co), ctypes.byref(cc), ctypes.byref(cp), ctypes.byref(h))
    else:
        name, cpr = "b200ba_estimate_covariance_with_position_priors", priors.to_c()
        rc = lib.b200ba_estimate_covariance_with_position_priors(ctypes.byref(co), ctypes.byref(cc), ctypes.byref(cp),
                                                                  ctypes.byref(cpr), ctypes.byref(h))
    if rc == 1:
        if raise_not_estimable:
            raise CovarianceNotEstimable(lib.b200ba_last_error().decode())
        return None
    if rc != 0:
        raise BundleAdjustmentError(f"{name} failed ({rc}): {lib.b200ba_last_error().decode()}")
    return FlatCovariance(lib, h.value, len(flat.poses), len(flat.points))


# Rigid3d (geometry/rigid3.h) uncertainty propagation; a pose is the 7-vector qx qy qz qw tx ty tz, covariances are in the
# left-perturbation tangent order [rotation, translation]
def _quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _cross_matrix(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def rigid3d_adjoint(T):
    """Rigid3d::Adjoint: [[R, 0], [[t]x R, R]]."""
    T = np.asarray(T, np.float64)
    R = _quat_to_R(T[:4])
    A = np.zeros((6, 6))
    A[:3, :3] = R; A[3:, 3:] = R; A[3:, :3] = _cross_matrix(T[4:]) @ R
    return A


def rigid3d_adjoint_inverse(T):
    """Rigid3d::AdjointInverse: [[R^T, 0], [-R^T [t]x, R^T]]."""
    T = np.asarray(T, np.float64)
    Rt = _quat_to_R(T[:4]).T
    A = np.zeros((6, 6))
    A[:3, :3] = Rt; A[3:, 3:] = Rt; A[3:, :3] = -Rt @ _cross_matrix(T[4:])
    return A


def rigid3d_inverse(T):
    return _rigid_inverse(np.asarray(T, np.float64))


def GetCovarianceForRigid3dInverse(rigid3, covar):
    """Covariance (6 x 6) of rigid3.inverse()."""
    Ai = rigid3d_adjoint_inverse(rigid3)
    return Ai @ covar @ Ai.T


def GetCovarianceForComposedRigid3d(a_from_b, covar):
    """Covariance (6 x 6) of a_from_c = a_from_b * b_from_c from the 12 x 12 covariance of (a_from_b, b_from_c)."""
    J = np.hstack([np.eye(6), rigid3d_adjoint(a_from_b)])
    return J @ covar @ J.T


def GetCovarianceForRelativeRigid3d(a_from_c, b_from_c, covar):
    """Covariance (6 x 6) of b_from_a = b_from_c * a_from_c^-1 from the 12 x 12 covariance of (a_from_c, b_from_c)."""
    J = np.hstack([-rigid3d_adjoint(b_from_c) @ rigid3d_adjoint_inverse(a_from_c), np.eye(6)])
    return J @ covar @ J.T


class BACovariance:
    """BACovariance (covariance.h) over the ids of the reconstruction."""

    def __init__(self, flat_cov: FlatCovariance, pose_index, point_index, other_index):
        self.flat_cov = flat_cov
        self._pose, self._point, self._other = pose_index, point_index, other_index

    def GetPointCov(self, point3D_id):
        k = self._point.get(point3D_id)
        return None if k is None else self.flat_cov.point(k)

    def GetCamCovFromWorld(self, image_id):
        k = self._pose.get(image_id)
        return None if k is None else self.flat_cov.pose(k)

    def GetCamCrossCovFromWorld(self, image_id1, image_id2):
        k1, k2 = self._pose.get(image_id1), self._pose.get(image_id2)
        return None if k1 is None or k2 is None else self.flat_cov.pose_cross(k1, k2)

    def GetCam2CovFromCam1(self, image_id1, cam1_from_world, image_id2, cam2_from_world):
        """Covariance of cam2_from_cam1; None unless both poses are fully variable (6 dimensions)."""
        cov_11, cov_22 = self.GetCamCovFromWorld(image_id1), self.GetCamCovFromWorld(image_id2)
        if cov_11 is None or cov_22 is None or cov_11.shape[0] != 6 or cov_22.shape[0] != 6:
            return None
        cov_12 = self.GetCamCrossCovFromWorld(image_id1, image_id2)
        cov = np.zeros((12, 12))
        cov[:6, :6], cov[6:, 6:], cov[:6, 6:], cov[6:, :6] = cov_11, cov_22, cov_12, cov_12.T
        return GetCovarianceForRelativeRigid3d(cam1_from_world, cam2_from_world, cov)

    def GetOtherParamsCov(self, params):
        """params: the array the reconstruction holds (camera.params, or rig.sensors[camera_id] for a sensor_from_rig)."""
        for arr, kind, k in self._other:
            if arr is params:
                return self.flat_cov.camera(k) if kind == "camera" else self.flat_cov.sensor(k)
        return None


def EstimateBACovariance(options: BACovarianceOptions, reconstruction: Reconstruction, bundle_adjuster: BundleAdjuster):
    """EstimateBACovariance (covariance.cc): the covariance of the problem `bundle_adjuster` solves, at the parameters
    the reconstruction holds now (call it after Solve()).  None when the problem is not estimable (unfixed gauge).
    A PosePriorBundleAdjuster's prior residuals are part of the problem, taken in the frame the reconstruction is in
    (normalized after the constructor, metric after Solve())."""
    rec = reconstruction
    for image_id in rec.images:
        if not rec.IsRefInFrame(image_id):
            raise BundleAdjustmentError(f"image {image_id} is not the reference sensor of its frame: pose covariances of "
                                        "non-trivial frames are not supported")
    flat, pose_ids, camera_ids, point_ids = bundle_adjuster.flat_problem()
    priors = None
    if isinstance(bundle_adjuster, PosePriorBundleAdjuster):
        priors = bundle_adjuster.flat_priors(flat, pose_ids, normalized=bundle_adjuster.in_normalized_frame_)
    cov = estimate_covariance_flat(bundle_adjuster.Options(), options, flat, priors=priors)
    if cov is None:
        return None
    if rec.frames:      # pose k = frame k; every image is its frame's reference sensor
        frame_index = {f: k for k, f in enumerate(pose_ids)}
        pose_index = {i: frame_index[im.frame_id] for i, im in rec.images.items() if im.frame_id in frame_index}
    else:
        pose_index = {i: k for k, i in enumerate(pose_ids)}
    others = [(rec.cameras[c].params, "camera", k) for k, c in enumerate(camera_ids)]
    for s, c in enumerate(getattr(flat, "sensor_camera_ids", [])):
        for rig in rec.rigs.values():
            if c in rig.sensors:
                others.append((rig.sensors[c], "sensor", s))
    return BACovariance(cov, pose_index, {p: k for k, p in enumerate(point_ids)}, others)


# ------------------------------------------------------------------------------------------------ pose priors
# PosePriorBundleAdjuster (bundle_adjustment_ceres.cc:900-1080) over include/b200_ba_pose_prior.h.  The alignment to the
# priors and the normalisation happen here on the host, as the reference does them before it builds the problem; the GPU
# solve receives the priors already in the normalized frame.
CHI_SQUARE_95_THREE_DOF = 7.814727903251179


class _CPositionPriors(ctypes.Structure):
    _fields_ = [("num_priors", ctypes.c_int), ("pose_idx", _i32p), ("sensor_idx", _i32p), ("position", _f64p),
                ("covariance", _f64p), ("loss_function_type", ctypes.c_int), ("loss_function_scale", ctypes.c_double)]


class FlatPositionPriors:
    """Arrays behind a b200ba_position_priors (kept alive here).  pose_idx / sensor_idx index the FlatProblem."""

    def __init__(self, pose_idx, sensor_idx, position, covariance, loss_function_type=TRIVIAL,
                 loss_function_scale=float(np.sqrt(CHI_SQUARE_95_THREE_DOF))):
        c = np.ascontiguousarray
        self.pose_idx = c(pose_idx, np.int32).reshape(-1)
        self.sensor_idx = c(sensor_idx, np.int32).reshape(-1)
        self.position = c(position, np.float64).reshape(-1, 3)
        self.covariance = c(covariance, np.float64).reshape(-1, 3, 3)
        self.loss_function_type, self.loss_function_scale = int(loss_function_type), float(loss_function_scale)

    def __len__(self):
        return len(self.pose_idx)

    def to_c(self) -> _CPositionPriors:
        n = len(self.pose_idx)
        if not (len(self.sensor_idx) == len(self.position) == len(self.covariance) == n):
            raise ValueError("prior arrays differ in length")
        return _CPositionPriors(n, self.pose_idx.ctypes.data_as(_i32p), self.sensor_idx.ctypes.data_as(_i32p),
                                self.position.ctypes.data_as(_f64p), self.covariance.ctypes.data_as(_f64p),
                                self.loss_function_type, self.loss_function_scale)


def _bind_prior(lib):
    if getattr(lib, "_prior_bound", False):
        return lib
    _bind(lib)
    lib.b200ba_solve_with_position_priors.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem),
                                                      ctypes.POINTER(_CPositionPriors), ctypes.POINTER(_CSummary)]
    lib.b200ba_position_priors_init.argtypes = [ctypes.POINTER(_CPositionPriors)]
    lib.b200ba_position_priors_init.restype = None
    lib.b200ba_test_prior_position.argtypes = [_f64p, _f64p, _f64p, _f64p, _f64p, _f64p]
    lib.b200ba_test_prior_position.restype = None
    lib.b200ba_test_prior_weight.argtypes = [_f64p, _f64p]
    lib._prior_bound = True
    return lib


def solve_flat_with_position_priors(options: BundleAdjustmentOptions, flat: FlatProblem,
                                    priors: FlatPositionPriors) -> BundleAdjustmentSummary:
    """b200ba_solve_with_position_priors; flat is updated in place like solve_flat."""
    lib = _bind_prior(load_library())
    co, cp, cpr, cs = options.to_c(), flat.to_c(), priors.to_c(), _CSummary()
    rc = lib.b200ba_solve_with_position_priors(ctypes.byref(co), ctypes.byref(cp), ctypes.byref(cpr), ctypes.byref(cs))
    if rc != 0:
        raise BundleAdjustmentError(f"b200ba_solve_with_position_priors failed ({rc}): {lib.b200ba_last_error().decode()}")
    return BundleAdjustmentSummary.from_c(cs)


@dataclass
class PosePrior:
    """PosePrior (geometry/pose_prior.h) for a CAMERA sensor: a Cartesian position of the image's projection centre; a NaN
    covariance means none was given."""
    image_id: int
    position: np.ndarray = field(default_factory=lambda: np.full(3, np.nan))
    position_covariance: np.ndarray = field(default_factory=lambda: np.full((3, 3), np.nan))
    sensor_type: str = "CAMERA"
    gravity: np.ndarray = field(default_factory=lambda: np.full(3, np.nan))   # unit gravity direction in the camera frame

    def HasPosition(self) -> bool:
        return bool(np.all(np.isfinite(self.position)))

    def HasPositionCov(self) -> bool:
        return bool(np.all(np.isfinite(self.position_covariance)))

    def HasGravity(self) -> bool:
        return bool(np.all(np.isfinite(self.gravity)))


@dataclass
class RANSACOptions:
    """RANSACOptions (optim/ransac.h:50-90); max_error <= 0 lets AlignReconstructionToPosePriors choose it."""
    max_error: float = 0.0
    min_inlier_ratio: float = 0.1
    confidence: float = 0.99
    dyn_num_trials_multiplier: float = 3.0
    min_num_trials: int = 0
    max_num_trials: int = 100000
    random_seed: int = -1


@dataclass
class PosePriorBundleAdjustmentOptions:
    """PosePriorBundleAdjustmentOptions (bundle_adjustment.h:236-270) with the Ceres prior-loss options
    (bundle_adjustment_ceres.h:102-112)."""
    prior_position_fallback_stddev: float = 1.0
    alignment_ransac_options: RANSACOptions = field(default_factory=RANSACOptions)
    prior_position_loss_function_type: int = TRIVIAL
    prior_position_loss_scale: float = float(np.sqrt(CHI_SQUARE_95_THREE_DOF))

    def Check(self) -> bool:
        return self.prior_position_fallback_stddev > 0 and self.prior_position_loss_scale > 0


class Sim3d:
    """Sim3d (geometry/sim3.h): x_new = scale * R(q) x + t, q = (x, y, z, w)."""

    def __init__(self, scale=1.0, rotation=(0.0, 0.0, 0.0, 1.0), translation=(0.0, 0.0, 0.0)):
        self.scale = float(scale)
        self.rotation = np.asarray(rotation, np.float64)
        self.translation = np.asarray(translation, np.float64)

    def R(self):
        return _quat_to_R(self.rotation)

    def __mul__(self, x):
        return self.scale * (np.asarray(x, np.float64) @ self.R().T) + self.translation

    def inverse(self) -> "Sim3d":
        qi = np.array([-self.rotation[0], -self.rotation[1], -self.rotation[2], self.rotation[3]])
        return Sim3d(1.0 / self.scale, qi, -(_quat_to_R(qi) @ self.translation) / self.scale)


def _R_to_quat(R):
    """Eigen::Quaterniond(Matrix3d), (x, y, z, w)"""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = np.zeros(4)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    return q / np.linalg.norm(q)


def estimate_sim3_umeyama(src, tgt) -> Optional[Sim3d]:
    """Umeyama's least-squares similarity tgt ~ s R src + t (Eigen::umeyama, as SimilarityTransformEstimator uses it)."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    n = len(src)
    if n < 3:
        return None
    ms, mt = src.mean(0), tgt.mean(0)
    xs, xt = src - ms, tgt - mt
    C = xt.T @ xs / n
    U, d, Vt = np.linalg.svd(C)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1
    R = U @ np.diag(S) @ Vt
    var_s = (xs ** 2).sum() / n
    if not var_s > 0:
        return None
    scale = float((d * S).sum() / var_s)
    if not (np.isfinite(scale) and scale > 0):
        return None
    return Sim3d(scale, _R_to_quat(R), mt - scale * (R @ ms))


def estimate_sim3_robust(src, tgt, ransac: RANSACOptions):
    """EstimateSim3dRobust: LO-RANSAC over Umeyama's minimal (3-point) fits with a local refit on the inliers; the inlier
    test is the squared error against max_error^2.  Seeded by ransac.random_seed (-1: a fixed default seed, so the result
    is reproducible).  Returns (Sim3d or None, inlier mask)."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    n = len(src)
    if n < 3 or not ransac.max_error > 0:
        return None, np.zeros(n, bool)
    rng = np.random.default_rng(ransac.random_seed if ransac.random_seed >= 0 else 0)
    thr2 = ransac.max_error ** 2

    def inliers_of(T):
        return ((tgt - T * src) ** 2).sum(1) <= thr2

    best, best_mask, best_n = None, np.zeros(n, bool), 0
    max_trials, trial = ransac.max_num_trials, 0
    while trial < max_trials:
        trial += 1
        idx = rng.choice(n, 3, replace=False)
        T = estimate_sim3_umeyama(src[idx], tgt[idx])
        if T is None:
            continue
        mask = inliers_of(T)
        if mask.sum() > best_n:
            for _ in range(10):      # local optimisation: refit on the inliers while their number grows
                T2 = estimate_sim3_umeyama(src[mask], tgt[mask])
                if T2 is None:
                    break
                m2 = inliers_of(T2)
                if m2.sum() < mask.sum():
                    break
                T, grew, mask = T2, m2.sum() > mask.sum(), m2
                if not grew:
                    break
            best, best_mask, best_n = T, mask, int(mask.sum())
            ratio = best_n / n
            # dynamic trial count (RANSAC::ComputeNumTrials)
            nom = 1.0 - ransac.confidence
            denom = 1.0 - ratio ** 3
            needed = 0 if denom <= 0 else int(np.ceil(np.log(nom) / np.log(denom) * ransac.dyn_num_trials_multiplier)) if nom > 0 else max_trials
            max_trials = min(ransac.max_num_trials, max(ransac.min_num_trials, needed))
    if best is None or best_n < 3 or best_n / n < ransac.min_inlier_ratio:
        return None, best_mask
    return best, best_mask


def align_reconstruction_to_pose_priors(rec: Reconstruction, pose_priors, ransac: RANSACOptions,
                                        fallback_stddev: float) -> Optional[Sim3d]:
    """AlignReconstructionToPosePriors (alignment.cc:240-299): robust Sim3 from projection centres to prior positions.
    None when fewer than three priors apply or the fit fails."""
    if not fallback_stddev > 0:
        raise ValueError("prior_position_fallback_stddev must be positive")
    by_image = {}
    for pp in pose_priors:
        if pp.sensor_type == "CAMERA" and pp.HasPosition():
            if pp.image_id in by_image:
                raise ValueError(f"duplicate pose prior for image {pp.image_id}")
            by_image[pp.image_id] = pp
    src, tgt, rms_vars = [], [], []
    for image_id in sorted(rec.images):
        pp = by_image.get(image_id)
        if pp is None:
            continue
        src.append(projection_center(rec, image_id))
        tgt.append(pp.position)
        tr = float(np.trace(pp.position_covariance))
        if tr > 0.0:
            rms_vars.append(tr / 3.0)
    if len(src) < 3:
        return None
    ransac = RANSACOptions(**vars(ransac))
    if ransac.max_error <= 0:
        ransac.max_error = automatic_alignment_max_error(rms_vars, fallback_stddev)
    T, _ = estimate_sim3_robust(np.array(src), np.array(tgt), ransac)
    return T


def automatic_alignment_max_error(rms_vars, fallback_stddev):
    """sqrt(chi2_95(3) * median(trace(cov) / 3)); the fallback variance when no prior has a covariance.  The median of an
    even count is the mean of the two middle values (colmap Median)."""
    v = list(rms_vars) if len(rms_vars) else [fallback_stddev * fallback_stddev]
    return float(np.sqrt(CHI_SQUARE_95_THREE_DOF * np.median(v)))


def _image_cam_from_world(rec: Reconstruction, image_id):
    im = rec.images[image_id]
    if im.frame_id is None:
        return im.cam_from_world
    fr = rec.frames[im.frame_id]
    rig = rec.rigs[fr.rig_id]
    if rig.ref_sensor == im.camera_id:
        return fr.rig_from_world
    return _rigid_compose(rig.sensors[im.camera_id], fr.rig_from_world)


def projection_center(rec: Reconstruction, image_id):
    """Image::ProjectionCenter: -R^T t of cam_from_world."""
    T = _image_cam_from_world(rec, image_id)
    return -_quat_to_R(T[:4]).T @ T[4:]


def _transform_camera_world(sim: Sim3d, cam_from_world):
    """TransformCameraWorld (geometry/sim3.cc): the same camera in the new world, its translation scaled."""
    R = _quat_to_R(cam_from_world[:4]) @ sim.R().T
    t = sim.scale * cam_from_world[4:] - R @ sim.translation
    return np.concatenate([_R_to_quat(R), t])


def transform_reconstruction(rec: Reconstruction, new_from_old: Sim3d):
    """Reconstruction::Transform (reconstruction.cc:788-805): sensor_from_rig translations scaled, rig_from_world (or the
    image pose of a trivial frame) and the points moved to the new world."""
    for rig in rec.rigs.values():
        for T in rig.sensors.values():
            T[4:] *= new_from_old.scale
    if rec.frames:
        for fr in rec.frames.values():
            fr.rig_from_world[:] = _transform_camera_world(new_from_old, fr.rig_from_world)
    else:
        for im in rec.images.values():
            im.cam_from_world[:] = _transform_camera_world(new_from_old, im.cam_from_world)
    for pt in rec.points3D.values():
        pt.xyz[:] = new_from_old * pt.xyz


def normalization_centroid(centers, min_percentile=0.1, max_percentile=0.9):
    """ComputeBoundingBoxAndCentroid (geometry/normalization.cc:39-90): per axis, the mean of the order statistics
    floor(min_p * (n - 1)) .. ceil(max_p * (n - 1))."""
    c = np.sort(np.asarray(centers, np.float64), axis=0)
    end = len(c) - 1
    lo, hi = min(end, int(np.floor(min_percentile * end))), min(end, int(np.ceil(max_percentile * end)))
    return c[lo:hi + 1].mean(0)


def normalize_reconstruction(rec: Reconstruction, fixed_scale=True, extent=10.0, min_percentile=0.1, max_percentile=0.9) -> Sim3d:
    """Reconstruction::Normalize(fixed_scale, extent, percentiles, use_images=true) (reconstruction.cc:698-728)."""
    centers = [projection_center(rec, i) for i in sorted(rec.images)]
    nreg = len(rec.frames) if rec.frames else len(rec.images)
    if nreg < 2:
        return Sim3d()
    centroid = normalization_centroid(centers, min_percentile, max_percentile)
    scale = 1.0
    if not fixed_scale:
        c = np.sort(np.asarray(centers), axis=0)
        end = len(c) - 1
        lo, hi = min(end, int(np.floor(min_percentile * end))), min(end, int(np.ceil(max_percentile * end)))
        old_extent = float(np.linalg.norm(c[hi] - c[lo]))
        if old_extent >= np.finfo(float).eps:
            scale = extent / old_extent
    tform = Sim3d(scale, (0.0, 0.0, 0.0, 1.0), -scale * centroid)
    transform_reconstruction(rec, tform)
    return tform


def filter_pose_priors(pose_priors, config: BundleAdjustmentConfig):
    """The constructor's filter (bundle_adjustment_ceres.cc:915-925): a position, a CAMERA sensor, an image in the config."""
    return [pp for pp in pose_priors if pp.HasPosition() and pp.sensor_type == "CAMERA" and config.HasImage(pp.image_id)]


class PosePriorBundleAdjuster(BundleAdjuster):
    """PosePriorBundleAdjuster (bundle_adjustment_ceres.cc:900-1080), B200 backend.  The constructor filters the priors,
    aligns the reconstruction to them and normalises it (or, with fewer than three priors or a failed alignment, fixes
    the TWO_CAMS_FROM_WORLD gauge), so Config().FixedGauge() is final before Solve()."""

    def __init__(self, options, prior_options: PosePriorBundleAdjustmentOptions, config, pose_priors, reconstruction):
        if not prior_options.Check():
            raise ValueError("invalid PosePriorBundleAdjustmentOptions")
        super().__init__(options, config, reconstruction)
        self.prior_options_ = prior_options
        self.pose_priors_ = filter_pose_priors(pose_priors, config)
        self.normalized_from_metric_ = Sim3d()
        self.use_prior_position_ = False
        if len(self.pose_priors_) >= 3:
            metric_from_orig = align_reconstruction_to_pose_priors(
                reconstruction, self.pose_priors_, prior_options.alignment_ransac_options,
                prior_options.prior_position_fallback_stddev)
            if metric_from_orig is not None:
                transform_reconstruction(reconstruction, metric_from_orig)
                self.use_prior_position_ = True
        if self.use_prior_position_:
            self.normalized_from_metric_ = normalize_reconstruction(reconstruction, fixed_scale=True)
        else:
            config.FixGauge(TWO_CAMS_FROM_WORLD)
        # the frame the reconstruction is in: normalized until Solve() transforms it back to the metric frame
        self.in_normalized_frame_ = self.use_prior_position_

    def flat_priors(self, flat: FlatProblem, pose_ids, normalized=True) -> FlatPositionPriors:
        """The priors of the parameterized images, indexed into `flat` (AddImagePosePriorToProblem,
        bundle_adjustment_ceres.cc:987-1039; the library skips those whose blocks are all constant).  normalized: in the
        normalized frame the solve runs in; else in the metric frame of the priors as given.  Empty when the adjuster
        fell back to the TWO_CAMS_FROM_WORLD gauge."""
        rec, po = self.reconstruction_, self.prior_options_
        pose_index = {p: k for k, p in enumerate(pose_ids)}
        sensor_of_cam = {c: k for k, c in enumerate(getattr(flat, "sensor_camera_ids", []))}
        to_frame = self.normalized_from_metric_ if normalized else Sim3d()
        sR = to_frame.scale * to_frame.R()
        pose_idx, sensor_idx, pos, cov = [], [], [], []
        if self.use_prior_position_:
            for pp in self.pose_priors_:
                if pp.image_id not in flat.parameterized_image_ids:
                    continue
                im = rec.images[pp.image_id]
                pose_idx.append(pose_index[im.frame_id if rec.frames else pp.image_id])
                sensor_idx.append(-1 if rec.IsRefInFrame(pp.image_id) else sensor_of_cam[im.camera_id])
                pos.append(to_frame * pp.position)
                C = pp.position_covariance if pp.HasPositionCov() else po.prior_position_fallback_stddev ** 2 * np.eye(3)
                cov.append(sR @ C @ sR.T)
        return FlatPositionPriors(pose_idx, sensor_idx, np.reshape(pos, (-1, 3)), np.reshape(cov, (-1, 3, 3)),
                                  po.prior_position_loss_function_type, po.prior_position_loss_scale)

    def _solve_flat(self, flat, pose_ids):
        return solve_flat_with_position_priors(self.options_, flat, self.flat_priors(flat, pose_ids))

    def Solve(self) -> BundleAdjustmentSummary:
        summary = super().Solve()
        transform_reconstruction(self.reconstruction_, self.normalized_from_metric_.inverse())
        self.in_normalized_frame_ = False
        return summary


def CreatePosePriorBundleAdjuster(options, prior_options, config, pose_priors, reconstruction) -> PosePriorBundleAdjuster:
    """Factory (bundle_adjustment.cc:373-390); this build has exactly one backend."""
    return PosePriorBundleAdjuster(options, prior_options, config, pose_priors, reconstruction)
