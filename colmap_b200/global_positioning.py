"""Host-side mirror of COLMAP's global positioner over the C-ABI (include/b200_global_positioning.h).

Mirrors ``GlobalPositionerOptions``, ``GlobalPositioner`` and ``RunGlobalPositioning``
(src/colmap/estimators/global_positioning.{h,cc}): the set-up of the BATA point-to-camera problem (constrained frames,
random initialisation, rays, scales, rig residuals, loss weights) is restated here; the LM solve runs in
libcolmap_b200.so on the GPU.  No CPU fallback.

The random initialisation draws ``100 * U(-1, 1)`` per coordinate in the reference's order (frame centres, then points,
then camera-in-rig positions) from numpy's ``default_rng(random_seed)``.  That stream differs from the reference's
``std::mt19937``, so a seeded run starts from other positions than the reference's run with the same seed.
"""
import ctypes
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from ._lib import load_library
from .bundle_adjustment import CONVERGENCE, FAILURE, NO_CONVERGENCE, Reconstruction, _quat_to_R, _rigid_inverse

SCALE_LOWER_BOUND = 1e-5
MAX_REDUCED_DIM = 32768
ERR_INPUT, ERR_TOO_LARGE, ERR_CUDA = -1, -2, -3

_f64p = ctypes.POINTER(ctypes.c_double)
_u8p = ctypes.POINTER(ctypes.c_uint8)
_i32p = ctypes.POINTER(ctypes.c_int32)


class _COptions(ctypes.Structure):
    _fields_ = [("optimize_positions", ctypes.c_int), ("optimize_points", ctypes.c_int),
                ("optimize_scales", ctypes.c_int), ("refine_sensor_from_rig", ctypes.c_int),
                ("loss_function_scale", ctypes.c_double), ("max_num_iterations", ctypes.c_int),
                ("function_tolerance", ctypes.c_double), ("gradient_tolerance", ctypes.c_double),
                ("parameter_tolerance", ctypes.c_double), ("initial_trust_region_radius", ctypes.c_double),
                ("max_trust_region_radius", ctypes.c_double), ("min_trust_region_radius", ctypes.c_double),
                ("min_relative_decrease", ctypes.c_double), ("min_lm_diagonal", ctypes.c_double),
                ("max_lm_diagonal", ctypes.c_double), ("gpu_index", ctypes.c_int)]


class _CProblem(ctypes.Structure):
    _fields_ = [("num_frames", ctypes.c_int), ("frame_centers", _f64p), ("frame_constant", _u8p),
                ("world_from_rig", _f64p), ("num_points", ctypes.c_int64), ("points", _f64p),
                ("num_sensors", ctypes.c_int), ("cams_in_rig", _f64p), ("num_observations", ctypes.c_int64),
                ("obs_frame", _i32p), ("obs_point", _i32p), ("obs_sensor", _i32p), ("obs_ray", _f64p),
                ("obs_rig_offset", _f64p), ("obs_scale", _f64p), ("obs_loss_weight", _f64p)]


class _CSummary(ctypes.Structure):
    _fields_ = [("termination_type", ctypes.c_int), ("num_successful_steps", ctypes.c_int),
                ("num_unsuccessful_steps", ctypes.c_int), ("num_residuals", ctypes.c_int),
                ("reduced_dim", ctypes.c_int), ("initial_cost", ctypes.c_double), ("final_cost", ctypes.c_double),
                ("solve_ms", ctypes.c_double), ("cost_history", _f64p), ("num_iterations", ctypes.c_int)]


def _bind(lib):
    if getattr(lib, "_gp_bound", False):
        return lib
    lib.b200gp_options_init.argtypes = [ctypes.POINTER(_COptions)]
    lib.b200gp_solve.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.POINTER(_CSummary)]
    lib.b200gp_solve.restype = ctypes.c_int
    lib.b200gp_cam_ray_from_img.argtypes = [ctypes.c_int, _f64p, _f64p, _f64p]
    lib.b200gp_cam_ray_from_img.restype = ctypes.c_int
    lib.b200gp_last_error.restype = ctypes.c_char_p
    lib._gp_bound = True
    return lib


class GlobalPositioningError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


@dataclass
class GlobalPositionerOptions:
    """GlobalPositionerOptions (global_positioning.h:13-60) and the Ceres solver options it keeps or sets."""
    generate_random_positions: bool = True
    generate_random_points: bool = True
    generate_scales: bool = True
    optimize_positions: bool = True
    optimize_points: bool = True
    optimize_scales: bool = True
    refine_sensor_from_rig: bool = True
    use_gpu: bool = True
    gpu_index: int = -1
    min_num_view_per_track: int = 3
    random_seed: int = -1
    loss_function_scale: float = 0.1
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5
    gradient_tolerance: float = 1e-10
    parameter_tolerance: float = 1e-8

    def to_c(self) -> _COptions:
        o = _COptions()
        _bind(load_library()).b200gp_options_init(ctypes.byref(o))
        o.optimize_positions, o.optimize_points = int(self.optimize_positions), int(self.optimize_points)
        o.optimize_scales, o.refine_sensor_from_rig = int(self.optimize_scales), int(self.refine_sensor_from_rig)
        o.loss_function_scale, o.max_num_iterations = self.loss_function_scale, self.max_num_iterations
        o.function_tolerance, o.gradient_tolerance = self.function_tolerance, self.gradient_tolerance
        o.parameter_tolerance, o.gpu_index = self.parameter_tolerance, self.gpu_index
        return o


@dataclass
class GlobalPositioningSummary:
    termination_type: int = FAILURE
    num_successful_steps: int = 0
    num_unsuccessful_steps: int = 0
    num_residuals: int = 0
    reduced_dim: int = 0
    initial_cost: float = 0.0
    final_cost: float = 0.0
    solve_ms: float = 0.0
    cost_history: np.ndarray = field(default_factory=lambda: np.zeros(0))

    def IsSolutionUsable(self) -> bool:
        return self.termination_type in (CONVERGENCE, NO_CONVERGENCE)


@dataclass
class FlatGlobalPositioning:
    """The flat problem of the C-ABI (b200gp_problem); arrays are updated in place by solve_flat."""
    frame_centers: np.ndarray                      # [F, 3]
    points: np.ndarray                             # [P, 3]
    obs_frame: np.ndarray                          # [N] int32
    obs_point: np.ndarray                          # [N] int32
    obs_ray: np.ndarray                            # [N, 3]
    obs_scale: np.ndarray                          # [N]
    obs_sensor: Optional[np.ndarray] = None        # [N] int32, -1 = none
    obs_rig_offset: Optional[np.ndarray] = None    # [N, 3]
    obs_loss_weight: Optional[np.ndarray] = None   # [N]
    frame_constant: Optional[np.ndarray] = None    # [F] uint8
    world_from_rig: Optional[np.ndarray] = None    # [F, 3, 3]
    cams_in_rig: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))

    def __post_init__(self):
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64)
        self.frame_centers, self.points, self.obs_ray = f64(self.frame_centers), f64(self.points), f64(self.obs_ray)
        self.obs_scale, self.cams_in_rig = f64(self.obs_scale), f64(self.cams_in_rig).reshape(-1, 3)
        self.obs_rig_offset, self.obs_loss_weight, self.world_from_rig = f64(self.obs_rig_offset), f64(self.obs_loss_weight), f64(self.world_from_rig)
        self.obs_frame = np.ascontiguousarray(self.obs_frame, np.int32)
        self.obs_point = np.ascontiguousarray(self.obs_point, np.int32)
        if self.obs_sensor is not None:
            self.obs_sensor = np.ascontiguousarray(self.obs_sensor, np.int32)
        if self.frame_constant is not None:
            self.frame_constant = np.ascontiguousarray(self.frame_constant, np.uint8)

    def copy(self) -> "FlatGlobalPositioning":
        return FlatGlobalPositioning(**{k: (None if v is None else np.array(v, copy=True)) for k, v in self.__dict__.items()})

    def to_c(self) -> _CProblem:
        p = lambda a, t: None if a is None else a.ctypes.data_as(t)
        return _CProblem(len(self.frame_centers), p(self.frame_centers, _f64p), p(self.frame_constant, _u8p),
                         p(self.world_from_rig, _f64p), len(self.points), p(self.points, _f64p), len(self.cams_in_rig),
                         p(self.cams_in_rig, _f64p), len(self.obs_frame), p(self.obs_frame, _i32p),
                         p(self.obs_point, _i32p), p(self.obs_sensor, _i32p), p(self.obs_ray, _f64p),
                         p(self.obs_rig_offset, _f64p), p(self.obs_scale, _f64p), p(self.obs_loss_weight, _f64p))


def solve_flat(options: GlobalPositionerOptions, flat: FlatGlobalPositioning) -> GlobalPositioningSummary:
    """b200gp_solve on the flat problem, in place.  Raises GlobalPositioningError on a refused input."""
    lib = _bind(load_library())
    hist = np.zeros(max(options.max_num_iterations, 0) + 1)
    s = _CSummary()
    s.cost_history = hist.ctypes.data_as(_f64p)
    c = flat.to_c()
    rc = lib.b200gp_solve(ctypes.byref(options.to_c()), ctypes.byref(c), ctypes.byref(s))
    if rc != 0:
        raise GlobalPositioningError(rc, lib.b200gp_last_error().decode())
    return GlobalPositioningSummary(s.termination_type, s.num_successful_steps, s.num_unsuccessful_steps, s.num_residuals,
                                    s.reduced_dim, s.initial_cost, s.final_cost, s.solve_ms,
                                    hist[:s.num_iterations + 1].copy())


def cam_ray_from_img(model_id: int, params, xy) -> Optional[np.ndarray]:
    """CameraModelCamRayFromImg: the unit ray of pixel xy, or None where the reference returns nullopt."""
    lib = _bind(load_library())
    prm = np.ascontiguousarray(params, np.float64)
    pt = np.ascontiguousarray(xy, np.float64)
    ray = np.zeros(3)
    if lib.b200gp_cam_ray_from_img(int(model_id), prm.ctypes.data_as(_f64p), pt.ctypes.data_as(_f64p), ray.ctypes.data_as(_f64p)) != 0:
        return None
    return ray


@dataclass
class PoseGraphEdge:
    """PoseGraph::Edge: the relative pose cam2_from_cam1 (7: qx qy qz qw tx ty tz), the inlier match count and the
    valid flag."""
    cam2_from_cam1: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]))
    num_matches: int = 0
    valid: bool = True


@dataclass
class PoseGraph:
    """PoseGraph (scene/pose_graph.h): edges between images keyed by pair (image_id1 < image_id2).  ``edges`` lists the
    pairs; ``edge_data`` holds an edge's relative pose, match count and valid flag (an edge without data is valid, with
    the identity pose and no matches), so PoseGraph(edges=[...]) still builds the graph the global positioner reads."""
    edges: List[Tuple[int, int]] = field(default_factory=list)
    edge_data: Dict[Tuple[int, int], PoseGraphEdge] = field(default_factory=dict)

    @staticmethod
    def _key(i1, i2):
        return (i1, i2) if i1 < i2 else (i2, i1)

    def AddEdge(self, image_id1, image_id2, edge: PoseGraphEdge):
        """Stores the edge under its pair; given as (larger, smaller) id, cam2_from_cam1 is inverted."""
        if image_id1 > image_id2:
            edge = PoseGraphEdge(_rigid_inverse(edge.cam2_from_cam1), edge.num_matches, edge.valid)
            image_id1, image_id2 = image_id2, image_id1
        if (image_id1, image_id2) not in self.edge_data and (image_id1, image_id2) not in self.edges:
            self.edges.append((image_id1, image_id2))
        self.edge_data[(image_id1, image_id2)] = edge

    def DeleteEdge(self, image_id1, image_id2):
        k = self._key(image_id1, image_id2)
        self.edges = [e for e in self.edges if self._key(*e) != k]
        self.edge_data.pop(k, None)

    def Edges(self) -> Dict[Tuple[int, int], PoseGraphEdge]:
        """Every edge by pair, in pair order."""
        return {k: self.EdgeData(*k) for k in sorted(self._key(*e) for e in self.edges)}

    def EdgeData(self, image_id1, image_id2) -> PoseGraphEdge:
        k = self._key(image_id1, image_id2)
        if k not in self.edge_data:
            self.edge_data[k] = PoseGraphEdge()
        return self.edge_data[k]

    def GetEdge(self, image_id1, image_id2) -> PoseGraphEdge:
        """The edge from image_id1 to image_id2 (inverted when stored the other way)."""
        e = self.EdgeData(image_id1, image_id2)
        return e if image_id1 < image_id2 else PoseGraphEdge(_rigid_inverse(e.cam2_from_cam1), e.num_matches, e.valid)

    def NumEdges(self):
        return len(self.edges)

    def ValidEdges(self):
        """The valid edges as (image_id1, image_id2) pairs, in insertion order."""
        return [e for e in self.edges if self.EdgeData(*e).valid]

    def SetInvalidEdge(self, image_id1, image_id2):
        self.EdgeData(image_id1, image_id2).valid = False

    def InvalidatePairsOutsideActiveImageIds(self, active_image_ids):
        for e in self.edges:
            if e[0] not in active_image_ids or e[1] not in active_image_ids:
                self.SetInvalidEdge(*e)

    def ComputeLargestConnectedFrameComponent(self, rec, filter_unregistered=False):
        """The frames of the largest connected component of the valid edges (images must have frames); ties go to the
        component with the smallest frame id."""
        parent = {}

        def find(a):
            while parent[a] != a:
                parent[a] = parent[parent[a]]
                a = parent[a]
            return a
        for i1, i2 in self.ValidEdges():
            f1, f2 = rec.images[i1].frame_id, rec.images[i2].frame_id
            if filter_unregistered and (rec.frames[f1].rig_from_world is None or rec.frames[f2].rig_from_world is None):
                continue
            parent.setdefault(f1, f1)
            parent.setdefault(f2, f2)
            a, b = find(f1), find(f2)
            if a != b:
                parent[max(a, b)] = min(a, b)
        comps = {}
        for f in parent:
            comps.setdefault(find(f), set()).add(f)
        if not comps:
            return set()
        return max(comps.values(), key=lambda c: (len(c), -min(c)))


class GlobalPositioner:
    def __init__(self, options: GlobalPositionerOptions):
        self.options_ = options
        self.summary = None
        self.rng_ = np.random.default_rng(options.random_seed if options.random_seed >= 0 else None)

    def GetOptions(self):
        return self.options_

    # frames: an image with frame_id None is its own trivial frame, keyed ("image", image_id)
    @staticmethod
    def _frame_key(rec, image_id):
        im = rec.images[image_id]
        return ("image", image_id) if im.frame_id is None else im.frame_id

    @staticmethod
    def _frame_pose(rec, key):
        return rec.images[key[1]].cam_from_world if isinstance(key, tuple) else rec.frames[key].rig_from_world

    @staticmethod
    def _has_pose(rec, image_id):
        im = rec.images[image_id]
        if im.cam_from_world is None:
            return False
        return im.frame_id is None or rec.frames[im.frame_id].rig_from_world is not None

    def _rand3(self):
        return self.rng_.uniform(-1.0, 1.0, 3)

    def Solve(self, pose_graph: PoseGraph, rec: Reconstruction) -> bool:
        o = self.options_
        if len(rec.images) == 0 or len(rec.points3D) == 0:
            return False
        # InitializeRandomPositions (global_positioning.cc:99-136)
        constrained = set()
        for i1, i2 in pose_graph.ValidEdges():
            constrained.add(self._frame_key(rec, i1)); constrained.add(self._frame_key(rec, i2))
        for pid in sorted(rec.points3D):
            pt = rec.points3D[pid]
            if len(pt.track) < o.min_num_view_per_track:
                continue
            for image_id, _ in pt.track:
                if image_id not in rec.images:
                    raise KeyError(f"image {image_id} of point {pid} does not exist")
                if self._has_pose(rec, image_id):
                    constrained.add(self._frame_key(rec, image_id))
        frame_keys = sorted((k for k in constrained), key=lambda k: (isinstance(k, tuple), k if not isinstance(k, tuple) else k[1]))
        frame_idx = {k: i for i, k in enumerate(frame_keys)}
        centers = np.zeros((len(frame_keys), 3))
        for i, k in enumerate(frame_keys):
            if o.generate_random_positions and o.optimize_positions:
                centers[i] = 100.0 * self._rand3()
            else:
                T = self._frame_pose(rec, k)
                centers[i] = -_quat_to_R(T[:4]).T @ T[4:]
        # AddPointToCameraConstraints / AddPoint3DToProblem (:138-273)
        random_init = o.optimize_points and o.generate_random_points
        point_ids, pts = [], []
        ob_f, ob_p, ob_s, ob_d, ob_off, ob_sc, ob_w = [], [], [], [], [], [], []
        sensors = {}                      # camera id -> sensor index, in first-use order (cams_in_rig_)
        wfr = np.tile(np.eye(3), (len(frame_keys), 1, 1))
        for pid in sorted(rec.points3D):
            pt = rec.points3D[pid]
            if len(pt.track) < o.min_num_view_per_track:
                continue
            if random_init:
                pt.xyz = 100.0 * self._rand3()
            pidx = len(point_ids)
            point_ids.append(pid); pts.append(pt.xyz)
            for image_id, p2d in pt.track:
                if image_id not in rec.images or not self._has_pose(rec, image_id):
                    continue
                im = rec.images[image_id]
                cam = rec.cameras[im.camera_id]
                ray = cam_ray_from_img(cam.model_id, cam.params, im.points2D[p2d].xy)
                if ray is None:
                    continue
                R_cw = _quat_to_R(im.cam_from_world[:4])
                d = R_cw.T @ ray
                fk = self._frame_key(rec, image_id)
                fi = frame_idx[fk]
                scale = 1.0
                if not o.generate_scales and random_init:
                    t = pt.xyz - centers[fi]
                    scale = max(SCALE_LOWER_BOUND, float(d @ t) / float(t @ t))
                sensor, off = -1, np.zeros(3)
                if not rec.IsRefInFrame(image_id):
                    rig = rec.rigs[rec.frames[im.frame_id].rig_id]
                    cam_from_rig = rig.sensors[im.camera_id]
                    if not np.isnan(cam_from_rig[4:]).any():
                        off = R_cw.T @ cam_from_rig[4:]
                    else:
                        if not o.refine_sensor_from_rig:
                            raise ValueError(f"sensor_from_rig has NaN translation but refine_sensor_from_rig=false "
                                             f"(image_id={image_id})")
                        sensor = sensors.setdefault(im.camera_id, len(sensors))
                        wfr[fi] = _quat_to_R(rec.frames[im.frame_id].rig_from_world[:4]).T
                ob_f.append(fi); ob_p.append(pidx); ob_s.append(sensor); ob_d.append(d); ob_off.append(off)
                ob_sc.append(scale); ob_w.append(1.0 if getattr(cam, "has_prior_focal_length", False) else 0.5)
        # ParameterizeVariables (:313-359): random camera-in-rig positions when optimising positions
        cams_in_rig = np.zeros((len(sensors), 3))
        if o.optimize_positions:
            for s in range(len(sensors)):
                cams_in_rig[s] = self._rand3()
        flat = FlatGlobalPositioning(
            frame_centers=centers, points=np.asarray(pts, np.float64).reshape(-1, 3), obs_frame=np.asarray(ob_f, np.int32),
            obs_point=np.asarray(ob_p, np.int32), obs_ray=np.asarray(ob_d, np.float64).reshape(-1, 3),
            obs_scale=np.asarray(ob_sc, np.float64), obs_sensor=np.asarray(ob_s, np.int32),
            obs_rig_offset=np.asarray(ob_off, np.float64).reshape(-1, 3), obs_loss_weight=np.asarray(ob_w, np.float64),
            world_from_rig=wfr, cams_in_rig=cams_in_rig)
        self.flat_problem = flat.copy()
        self.summary = self._solve_flat(flat)
        # ConvertBackResults (:422-441): every constrained frame, with or without residuals
        for i, k in enumerate(frame_keys):
            T = self._frame_pose(rec, k)
            T[4:] = _quat_to_R(T[:4]) @ -flat.frame_centers[i]
        for cam_id, s in sensors.items():
            for rig in rec.rigs.values():
                if cam_id in rig.sensors:
                    rig.sensors[cam_id][4:] = _quat_to_R(rig.sensors[cam_id][:4]) @ -flat.cams_in_rig[s]
                    break
        for i, pid in enumerate(point_ids):
            rec.points3D[pid].xyz = flat.points[i].copy()
        self._sync_image_poses(rec)
        return self.summary.IsSolutionUsable()

    def _solve_flat(self, flat):
        """The LM solve of the assembled problem, in place (a test substitutes the CPU oracle here)."""
        return solve_flat(self.options_, flat)

    @staticmethod
    def _sync_image_poses(rec):
        from .bundle_adjustment import _rigid_compose
        for im in rec.images.values():
            if im.frame_id is None:
                continue
            fr = rec.frames[im.frame_id]
            rig = rec.rigs[fr.rig_id]
            im.cam_from_world[:] = fr.rig_from_world if rig.ref_sensor == im.camera_id else _rigid_compose(rig.sensors[im.camera_id], fr.rig_from_world)


def RunGlobalPositioning(options: GlobalPositionerOptions, pose_graph: PoseGraph, reconstruction: Reconstruction) -> bool:
    return GlobalPositioner(options).Solve(pose_graph, reconstruction)
