"""Host-side mirror of COLMAP's PatchMatch interface over the C-ABI (include/b200_patch_match.h).

Mirrors, with the same names and argument meaning:
  * ``mvs::PatchMatchOptions``        src/colmap/mvs/patch_match_options.h:37-126
  * ``mvs::Image``                    src/colmap/mvs/image.h:39-104 (K, R, T + grey bitmap)
  * ``mvs::PatchMatch::Problem``      src/colmap/mvs/patch_match.h:57-75
  * ``mvs::PatchMatch``               src/colmap/mvs/patch_match.h:55-96, patch_match.cc:50-154
    (Check / Run / GetDepthMap / GetNormalMap / GetSelProbMap / GetConsistencyGraph)

All computation happens in libcolmap_b200.so (CUDA, sm_90a).  There is no CPU path here.
"""
import ctypes
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from ._lib import load_library

MAX_PATCH_MATCH_WINDOW_RADIUS = 20  # kMaxPatchMatchWindowRadius (patch_match_options.h)


class _COptions(ctypes.Structure):
    _fields_ = [
        ("depth_min", ctypes.c_double), ("depth_max", ctypes.c_double),
        ("sigma_spatial", ctypes.c_double), ("sigma_color", ctypes.c_double),
        ("ncc_sigma", ctypes.c_double), ("min_triangulation_angle", ctypes.c_double),
        ("incident_angle_sigma", ctypes.c_double),
        ("geom_consistency_regularizer", ctypes.c_double),
        ("geom_consistency_max_cost", ctypes.c_double),
        ("filter_min_ncc", ctypes.c_double),
        ("filter_min_triangulation_angle", ctypes.c_double),
        ("filter_geom_consistency_max_cost", ctypes.c_double),
        ("window_radius", ctypes.c_int), ("window_step", ctypes.c_int),
        ("num_samples", ctypes.c_int), ("num_iterations", ctypes.c_int),
        ("filter_min_num_consistent", ctypes.c_int),
        ("geom_consistency", ctypes.c_int), ("filter", ctypes.c_int),
        ("gpu_index", ctypes.c_int),
    ]


_u8p = ctypes.POINTER(ctypes.c_uint8)
_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int)


class _CProblem(ctypes.Structure):
    _fields_ = [
        ("ref_width", ctypes.c_int), ("ref_height", ctypes.c_int),
        ("ref_gray", _u8p),
        ("ref_K", ctypes.c_float * 9), ("ref_R", ctypes.c_float * 9), ("ref_T", ctypes.c_float * 3),
        ("num_src", ctypes.c_int),
        ("src_width", _i32p), ("src_height", _i32p),
        ("src_gray", ctypes.POINTER(_u8p)),
        ("src_K", _f32p), ("src_R", _f32p), ("src_T", _f32p),
        ("src_depth", ctypes.POINTER(_f32p)),
        ("ref_depth_init", _f32p), ("ref_normal_init", _f32p),
        ("src_image_idxs", _i32p),
        ("maps_on_device", ctypes.c_int),
    ]


@dataclass
class PatchMatchOptions:
    """mvs::PatchMatchOptions — same field names and defaults (patch_match_options.h:37-126)."""
    depth_min: float = -1.0
    depth_max: float = -1.0
    sigma_spatial: float = -1.0
    sigma_color: float = 0.2
    ncc_sigma: float = 0.6
    min_triangulation_angle: float = 1.0
    incident_angle_sigma: float = 0.9
    geom_consistency_regularizer: float = 0.3
    geom_consistency_max_cost: float = 3.0
    filter_min_ncc: float = 0.1
    filter_min_triangulation_angle: float = 3.0
    filter_geom_consistency_max_cost: float = 1.0
    cache_size: float = 32.0
    gpu_index: str = "-1"
    max_image_size: int = -1
    window_radius: int = 5
    window_step: int = 1
    num_samples: int = 15
    num_iterations: int = 5
    filter_min_num_consistent: int = 2
    num_threads: int = -1
    geom_consistency: bool = True
    filter: bool = True
    allow_missing_files: bool = False
    write_consistency_graph: bool = False

    def Check(self) -> bool:
        """PatchMatchOptions::Check (patch_match_options.cc:72-99)."""
        ok = True
        if self.depth_min != -1.0 or self.depth_max != -1.0:
            ok &= self.depth_min <= self.depth_max and self.depth_min >= 0.0
        ok &= 0 < self.window_radius <= MAX_PATCH_MATCH_WINDOW_RADIUS
        ok &= self.sigma_color > 0.0
        ok &= 0 < self.window_step <= 2
        ok &= self.num_samples > 0 and self.ncc_sigma > 0.0
        ok &= 0.0 <= self.min_triangulation_angle < 180.0
        ok &= self.incident_angle_sigma > 0.0 and self.num_iterations > 0
        ok &= self.geom_consistency_regularizer >= 0.0 and self.geom_consistency_max_cost >= 0.0
        ok &= -1.0 <= self.filter_min_ncc <= 1.0
        ok &= 0.0 <= self.filter_min_triangulation_angle <= 180.0
        ok &= self.filter_min_num_consistent >= 0 and self.filter_geom_consistency_max_cost >= 0.0
        ok &= self.cache_size > 0 and self.num_threads >= -1
        return bool(ok)

    def to_c(self) -> _COptions:
        gpu = self.gpu_index if isinstance(self.gpu_index, int) else int(str(self.gpu_index).split(",")[0])
        return _COptions(
            self.depth_min, self.depth_max, self.sigma_spatial, self.sigma_color, self.ncc_sigma,
            self.min_triangulation_angle, self.incident_angle_sigma, self.geom_consistency_regularizer,
            self.geom_consistency_max_cost, self.filter_min_ncc, self.filter_min_triangulation_angle,
            self.filter_geom_consistency_max_cost, self.window_radius, self.window_step, self.num_samples,
            self.num_iterations, self.filter_min_num_consistent, int(self.geom_consistency), int(self.filter), gpu)


@dataclass
class Image:
    """mvs::Image: grey bitmap + float K (3x3), R (3x3), T (3) (image.h:39-104)."""
    bitmap: np.ndarray  # (H, W) uint8
    K: np.ndarray
    R: np.ndarray
    T: np.ndarray

    def GetWidth(self) -> int:
        return int(self.bitmap.shape[1])

    def GetHeight(self) -> int:
        return int(self.bitmap.shape[0])


@dataclass
class Problem:
    """mvs::PatchMatch::Problem (patch_match.h:57-75)."""
    ref_image_idx: int = -1
    src_image_idxs: List[int] = field(default_factory=list)
    images: Optional[List[Image]] = None
    depth_maps: Optional[List[np.ndarray]] = None    # (H, W) float32 each - numpy arrays, or CUDA torch tensors
    normal_maps: Optional[List[np.ndarray]] = None   # (3, H, W) float32 each   (device-resident maps, see workspace.py)


def marshal(options: PatchMatchOptions, problem: Problem):
    """Flatten (options, problem) into the C structs.  Returns (c_options, c_problem, keepalive)."""
    keep = []
    images = problem.images
    ref = images[problem.ref_image_idx]
    n = len(problem.src_image_idxs)

    def c_arr(a, dtype):
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a

    cp = _CProblem()
    cp.ref_width, cp.ref_height = ref.GetWidth(), ref.GetHeight()
    cp.ref_gray = c_arr(ref.bitmap, np.uint8).ctypes.data_as(_u8p)
    cp.ref_K = (ctypes.c_float * 9)(*np.asarray(ref.K, np.float32).reshape(9))
    cp.ref_R = (ctypes.c_float * 9)(*np.asarray(ref.R, np.float32).reshape(9))
    cp.ref_T = (ctypes.c_float * 3)(*np.asarray(ref.T, np.float32).reshape(3))
    cp.num_src = n
    srcs = [images[i] for i in problem.src_image_idxs]
    cp.src_width = c_arr([s.GetWidth() for s in srcs], np.int32).ctypes.data_as(_i32p)
    cp.src_height = c_arr([s.GetHeight() for s in srcs], np.int32).ctypes.data_as(_i32p)
    gray_ptrs = (_u8p * max(n, 1))()
    for k, s in enumerate(srcs):
        gray_ptrs[k] = c_arr(s.bitmap, np.uint8).ctypes.data_as(_u8p)
    keep.append(gray_ptrs)
    cp.src_gray = ctypes.cast(gray_ptrs, ctypes.POINTER(_u8p))
    cp.src_K = c_arr(np.stack([np.asarray(s.K, np.float32).reshape(9) for s in srcs]) if n else np.zeros(0), np.float32).ctypes.data_as(_f32p)
    cp.src_R = c_arr(np.stack([np.asarray(s.R, np.float32).reshape(9) for s in srcs]) if n else np.zeros(0), np.float32).ctypes.data_as(_f32p)
    cp.src_T = c_arr(np.stack([np.asarray(s.T, np.float32).reshape(3) for s in srcs]) if n else np.zeros(0), np.float32).ctypes.data_as(_f32p)
    if options.geom_consistency and problem.depth_maps is not None and problem.normal_maps is not None:
        on_device = hasattr(problem.depth_maps[problem.ref_image_idx], "data_ptr")   # CUDA torch tensors: stay in HBM

        def map_ptr(a):
            if on_device:
                assert a.is_cuda and a.is_contiguous() and str(a.dtype) == "torch.float32"
                keep.append(a)
                return ctypes.cast(ctypes.c_void_p(a.data_ptr()), _f32p)
            return c_arr(a, np.float32).ctypes.data_as(_f32p)
        dptrs = (_f32p * max(n, 1))()
        for k, i in enumerate(problem.src_image_idxs):
            dptrs[k] = map_ptr(problem.depth_maps[i])
        keep.append(dptrs)
        cp.src_depth = ctypes.cast(dptrs, ctypes.POINTER(_f32p))
        cp.ref_depth_init = map_ptr(problem.depth_maps[problem.ref_image_idx])
        cp.ref_normal_init = map_ptr(problem.normal_maps[problem.ref_image_idx])
        cp.maps_on_device = 1 if on_device else 0
    cp.src_image_idxs = c_arr(problem.src_image_idxs, np.int32).ctypes.data_as(_i32p)
    co = options.to_c()
    if co.sigma_spatial <= 0:
        co.sigma_spatial = float(options.window_radius)  # patch_match.cc:436-438
    return co, cp, keep


def _bind(lib):
    if getattr(lib, "_pm_bound", False):
        return lib
    H = ctypes.c_void_p
    lib.b200pm_options_init.argtypes = [ctypes.POINTER(_COptions)]
    lib.b200pm_options_init.restype = None
    lib.b200pm_check.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem)]
    lib.b200pm_create.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.POINTER(H)]
    lib.b200pm_run.argtypes = [H]
    lib.b200pm_last_run_ms.argtypes = [H]
    lib.b200pm_last_run_ms.restype = ctypes.c_float
    lib.b200pm_last_sweep_ms.argtypes = [H]
    lib.b200pm_last_sweep_ms.restype = ctypes.c_float
    lib.b200pm_last_num_launches.argtypes = [H]
    lib.b200pm_last_pass_ms.argtypes = [H, ctypes.c_int]
    lib.b200pm_last_pass_ms.restype = ctypes.c_float
    lib.b200pm_last_sweep_pass_ms.argtypes = [H, ctypes.c_int, ctypes.c_int]
    lib.b200pm_last_sweep_pass_ms.restype = ctypes.c_float
    lib.b200pm_patch_store_bytes.argtypes = [H]
    lib.b200pm_patch_store_bytes.restype = ctypes.c_size_t
    lib.b200pm_get_depth.argtypes = [H, _f32p]
    lib.b200pm_get_normal.argtypes = [H, _f32p]
    lib.b200pm_get_sel_prob.argtypes = [H, _f32p]
    lib.b200pm_get_depth_device.argtypes = [H, ctypes.c_void_p]
    lib.b200pm_get_normal_device.argtypes = [H, ctypes.c_void_p]
    lib.b200pm_get_consistency.argtypes = [H, ctypes.POINTER(_i32p), ctypes.POINTER(ctypes.c_size_t)]
    lib.b200pm_get_consistency_mask.argtypes = [H, _u8p]
    lib.b200pm_free.argtypes = [ctypes.c_void_p]
    lib.b200pm_free.restype = None
    lib.b200pm_destroy.argtypes = [H]
    lib.b200pm_destroy.restype = None
    lib.b200pm_last_error.restype = ctypes.c_char_p
    lib._pm_bound = True
    return lib


class PatchMatchError(RuntimeError):
    pass


class PatchMatch:
    """mvs::PatchMatch (patch_match.h:55-96).  ``Run()`` executes on the GPU selected by
    ``options.gpu_index``; results are fetched with the Get* methods, as in the reference."""

    def __init__(self, options: PatchMatchOptions, problem: Problem):
        self.options_ = options
        self.problem_ = problem
        self._lib = _bind(load_library())
        self._h = ctypes.c_void_p()
        self._created = False
        self._dims = None

    def _err(self, what, code):
        raise PatchMatchError(f"{what} failed ({code}): {self._lib.b200pm_last_error().decode()}")

    def Check(self):
        """PatchMatch::Check (patch_match.cc:67-126): raises on an invalid problem."""
        if not self.options_.Check():
            raise PatchMatchError("PatchMatchOptions::Check failed")
        co, cp, keep = marshal(self.options_, self.problem_)
        rc = self._lib.b200pm_check(ctypes.byref(co), ctypes.byref(cp))
        if rc != 0:
            self._err("PatchMatch::Check", rc)

    def Create(self):
        """PatchMatchCuda constructor: upload + prefilter + init (host -> device)."""
        if self._created:
            return
        co, cp, keep = marshal(self.options_, self.problem_)
        rc = self._lib.b200pm_create(ctypes.byref(co), ctypes.byref(cp), ctypes.byref(self._h))
        if rc != 0:
            self._err("b200pm_create", rc)
        self._created = True
        self._dims = (cp.ref_height, cp.ref_width, cp.num_src)

    def Run(self):
        """PatchMatch::Run (patch_match.cc:128-135)."""
        self.Check()
        self.Create()
        rc = self._lib.b200pm_run(self._h)
        if rc != 0:
            self._err("b200pm_run", rc)

    def RunOnly(self):
        """Device-resident re-run used by bench.py (inputs already in HBM)."""
        rc = self._lib.b200pm_run(self._h)
        if rc != 0:
            self._err("b200pm_run", rc)

    def last_run_ms(self):
        return float(self._lib.b200pm_last_run_ms(self._h))

    def last_sweep_ms(self):
        return float(self._lib.b200pm_last_sweep_ms(self._h))

    def last_pass_ms(self, which):
        return float(self._lib.b200pm_last_pass_ms(self._h, which))

    def last_sweep_pass_ms(self, sweep, which):
        """Device time of one pass (0 = rand + msg side by side, 1 = pixel, 2 = serial, 3 = rand alone, 4 = msg alone)
        in one sweep of the last run."""
        return float(self._lib.b200pm_last_sweep_pass_ms(self._h, sweep, which))

    def patch_store_bytes(self):
        """Device bytes of the reference-patch store; 0 when every pass builds the patch inline."""
        return int(self._lib.b200pm_patch_store_bytes(self._h))

    def last_num_launches(self):
        return int(self._lib.b200pm_last_num_launches(self._h))

    def GetDepthMap(self) -> np.ndarray:
        h, w, _ = self._dims
        out = np.empty((h, w), np.float32)
        rc = self._lib.b200pm_get_depth(self._h, out.ctypes.data_as(_f32p))
        if rc != 0:
            self._err("b200pm_get_depth", rc)
        return out

    def GetNormalMap(self) -> np.ndarray:
        h, w, _ = self._dims
        out = np.empty((3, h, w), np.float32)
        rc = self._lib.b200pm_get_normal(self._h, out.ctypes.data_as(_f32p))
        if rc != 0:
            self._err("b200pm_get_normal", rc)
        return out

    def GetDepthMapDevice(self, out):
        """Depth map into a CUDA torch tensor (H, W) float32 on the handle's GPU: no host copy."""
        h, w, _ = self._dims
        assert out.is_cuda and out.is_contiguous() and tuple(out.shape) == (h, w)
        rc = self._lib.b200pm_get_depth_device(self._h, ctypes.c_void_p(out.data_ptr()))
        if rc != 0:
            self._err("b200pm_get_depth_device", rc)
        return out

    def GetNormalMapDevice(self, out):
        h, w, _ = self._dims
        assert out.is_cuda and out.is_contiguous() and tuple(out.shape) == (3, h, w)
        rc = self._lib.b200pm_get_normal_device(self._h, ctypes.c_void_p(out.data_ptr()))
        if rc != 0:
            self._err("b200pm_get_normal_device", rc)
        return out

    def GetSelProbMap(self) -> np.ndarray:
        h, w, n = self._dims
        out = np.empty((n, h, w), np.float32)
        rc = self._lib.b200pm_get_sel_prob(self._h, out.ctypes.data_as(_f32p))
        if rc != 0:
            self._err("b200pm_get_sel_prob", rc)
        return out

    def GetConsistencyMask(self) -> np.ndarray:
        h, w, n = self._dims
        out = np.empty((n, h, w), np.uint8)
        rc = self._lib.b200pm_get_consistency_mask(self._h, out.ctypes.data_as(_u8p))
        if rc != 0:
            self._err("b200pm_get_consistency_mask", rc)
        return out

    def GetConsistentImageIdxs(self) -> np.ndarray:
        """PatchMatchCuda::GetConsistentImageIdxs: flat [col,row,n,idx...] list."""
        data = _i32p()
        count = ctypes.c_size_t()
        rc = self._lib.b200pm_get_consistency(self._h, ctypes.byref(data), ctypes.byref(count))
        if rc != 0:
            self._err("b200pm_get_consistency", rc)
        out = np.ctypeslib.as_array(data, shape=(count.value,)).copy() if count.value else np.zeros(0, np.int32)
        self._lib.b200pm_free(data)
        return out

    def close(self):
        if self._created:
            self._lib.b200pm_destroy(self._h)
            self._created = False

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def consistency_list_from_mask(mask: np.ndarray, src_image_idxs) -> np.ndarray:
    """Host restatement of GetConsistentImageIdxs (patch_match_cuda.cu:1367-1391) for tests."""
    n, h, w = mask.shape
    out = []
    idxs = np.asarray(src_image_idxs)
    any_px = mask.any(axis=0)
    rows, cols = np.nonzero(any_px)
    for r, c in zip(rows, cols):
        sel = idxs[mask[:, r, c] != 0]
        out.extend([int(c), int(r), int(len(sel))])
        out.extend(int(v) for v in sel)
    return np.asarray(out, np.int32)
