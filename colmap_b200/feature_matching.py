"""Mirror of the reference's SIFT feature matcher (src/colmap/feature/sift.{h,cc}, feature/matcher.h) over
include/b200_sift_matching.h: brute-force matching of uint8 SIFT descriptors on the GPU with the decisions of
FindBestMatchesBruteForce, bit for bit.  Names follow the reference: SiftMatchingOptions, FeatureMatchingOptions,
FeatureMatcher::Image (here FeatureMatcherImage), CreateSiftFeatureMatcher(options).Match(image1, image2).

Like SiftGPUFeatureMatcher::Match, a matcher keeps each image's descriptors on the device and uploads again only when
the image_id in that position changes; MatchPairs matches a whole block of pairs in one call.

MatchGuided (FeatureMatcher::MatchGuided) and MatchGuidedPairs follow the reference's CPU guided matcher
(SiftCPUFeatureMatcher::MatchGuided): L2 descriptor distances, a geometric filter from the pair's E, F or H, and
FindBestMatchesIndex, bit for bit."""
import ctypes
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from ._lib import load_library
from .bundle_adjustment import Camera

kInvalidImageId = 2 ** 32 - 1

_u8p = ctypes.POINTER(ctypes.c_uint8)
_u32p = ctypes.POINTER(ctypes.c_uint32)
_u64p = ctypes.POINTER(ctypes.c_uint64)
_i32p = ctypes.POINTER(ctypes.c_int)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)

GUIDED_NONE, GUIDED_E, GUIDED_F, GUIDED_H = 0, 1, 2, 3
EQUIRECTANGULAR = 17          # the one spherical camera model (CameraModelIsSpherical)


class FeatureMatchingError(RuntimeError):
    pass


class _COptions(ctypes.Structure):
    _fields_ = [("max_ratio", ctypes.c_double), ("max_distance", ctypes.c_double), ("cross_check", ctypes.c_int),
                ("max_num_matches", ctypes.c_int), ("gpu_index", ctypes.c_int)]


class _CGuided(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("max_error", ctypes.c_double), ("M", ctypes.c_double * 9)]


_BOUND = None


def _lib():
    global _BOUND
    if _BOUND is None:
        L = load_library()
        L.b200sm_last_error.restype = ctypes.c_char_p
        L.b200sm_options_init.argtypes = [ctypes.POINTER(_COptions)]
        L.b200sm_options_init.restype = None
        L.b200sm_create.argtypes = [ctypes.POINTER(_COptions), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
        L.b200sm_set_descriptors.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, _u8p]
        L.b200sm_match_capacity.argtypes = [ctypes.c_void_p, ctypes.c_int, _i32p, _i32p]
        L.b200sm_match_capacity.restype = ctypes.c_int64
        L.b200sm_match_pairs.argtypes = [ctypes.c_void_p, ctypes.c_int, _i32p, _i32p, _u64p, _u32p, ctypes.c_size_t]
        L.b200sm_last_timing.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]
        L.b200sm_set_keypoints.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, _f32p]
        L.b200sm_set_camera.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, _f64p]
        L.b200sm_cam_ray_from_img_with_jac.argtypes = [ctypes.c_int, _f64p, _f64p, _f64p]
        L.b200sm_match_guided_pairs.argtypes = [ctypes.c_void_p, ctypes.c_int, _i32p, _i32p, ctypes.POINTER(_CGuided),
                                                _u64p, _u32p, ctypes.c_size_t]
        L.b200sm_destroy.argtypes = [ctypes.c_void_p]
        L.b200sm_destroy.restype = None
        _BOUND = L
    return _BOUND


def _check(rc, what):
    if rc < 0:
        raise FeatureMatchingError(f"{what} failed ({rc}): {_lib().b200sm_last_error().decode()}")
    return rc


@dataclass
class SiftMatchingOptions:
    """SiftMatchingOptions (feature/sift.h:114-123), the fields the brute-force matcher reads."""
    max_ratio: float = 0.8
    max_distance: float = 0.7
    cross_check: bool = True

    def Check(self) -> bool:
        return self.max_ratio > 0 and self.max_distance > 0


@dataclass
class FeatureMatchingOptions:
    """FeatureMatchingOptions (feature/matcher.h:58-110), the fields the SIFT matcher reads.  gpu_index names one
    device ("-1": the current one)."""
    gpu_index: str = "-1"
    max_num_matches: int = 32768
    sift: SiftMatchingOptions = field(default_factory=SiftMatchingOptions)

    def Check(self) -> bool:
        return self.max_num_matches > 0 and self.sift.Check()

    def to_c(self) -> _COptions:
        c = _COptions()
        _lib().b200sm_options_init(ctypes.byref(c))
        c.max_ratio, c.max_distance = float(self.sift.max_ratio), float(self.sift.max_distance)
        c.cross_check = 1 if self.sift.cross_check else 0
        c.max_num_matches = int(self.max_num_matches)
        gi = str(self.gpu_index).strip()
        if "," in gi:
            raise FeatureMatchingError("gpu_index names one device; lists of devices are not supported")
        c.gpu_index = int(gi)
        return c


def _as_descriptors(d) -> np.ndarray:
    a = np.asarray(d)
    if a.dtype != np.uint8:
        raise FeatureMatchingError(f"SIFT descriptors must be uint8, got {a.dtype}")
    if a.ndim != 2 or a.shape[1] != 128:
        raise FeatureMatchingError(f"SIFT descriptors must be (n, 128), got shape {a.shape}")
    return np.ascontiguousarray(a)


def _as_keypoints(k) -> np.ndarray:
    a = np.asarray(k)
    if a.ndim != 2 or a.shape[1] != 2 or not np.issubdtype(a.dtype, np.floating):
        raise FeatureMatchingError(f"keypoints must be (n, 2) floating point, got {a.dtype} {a.shape}")
    return np.ascontiguousarray(a, np.float32)


@dataclass
class FeatureMatcherImage:
    """FeatureMatcher::Image (feature/matcher.h:114-122): the part the descriptor matcher reads.  camera and keypoints
    (x, y per descriptor row) are read by guided matching only."""
    image_id: int
    descriptors: np.ndarray   # (n, 128) uint8
    camera: Optional[Camera] = None
    keypoints: Optional[np.ndarray] = None   # (n, 2) float32

    def __post_init__(self):
        self.descriptors = _as_descriptors(self.descriptors)
        if self.keypoints is not None:
            self.keypoints = _as_keypoints(self.keypoints)


@dataclass
class TwoViewGeometry:
    """TwoViewGeometry (scene/two_view_geometry.h:41-110), the fields guided matching reads and writes.  E, F and H are
    3 x 3 and map image 1 to image 2; camera1 / camera2 are the intrinsics the two-view solver estimated, if any."""
    UNDEFINED, DEGENERATE, CALIBRATED, UNCALIBRATED, PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC, WATERMARK, MULTIPLE, \
        CALIBRATED_RIG = range(10)
    config: int = 0
    E: Optional[np.ndarray] = None
    F: Optional[np.ndarray] = None
    H: Optional[np.ndarray] = None
    camera1: Optional[Camera] = None
    camera2: Optional[Camera] = None
    inlier_matches: np.ndarray = field(default_factory=lambda: np.zeros((0, 2), np.uint32))


def UseEssentialMatrixForGuidedMatching(g: TwoViewGeometry) -> bool:
    """sift.cc:1053-1065: E when the intrinsics are known, from priors or from the two-view solver."""
    if g.E is None:
        return False
    if g.config in (TwoViewGeometry.CALIBRATED, TwoViewGeometry.CALIBRATED_RIG):
        return True
    if g.config == TwoViewGeometry.UNCALIBRATED:
        return g.camera1 is not None or g.camera2 is not None
    return False


def SelectGuidedModel(g: TwoViewGeometry, image1: FeatureMatcherImage, image2: FeatureMatcherImage):
    """The model MatchGuided filters with (sift.cc:1171-1196): (GUIDED_E/F/H/NONE, 3 x 3 float64 matrix or None, the
    effective camera of each image).  Refuses a homography with a spherical effective camera."""
    cam1 = g.camera1 if g.camera1 is not None else image1.camera
    cam2 = g.camera2 if g.camera2 is not None else image2.camera
    use_e = UseEssentialMatrixForGuidedMatching(g)
    use_f = not use_e and g.config == TwoViewGeometry.UNCALIBRATED and g.F is not None
    use_h = g.config in (TwoViewGeometry.PLANAR, TwoViewGeometry.PANORAMIC,
                         TwoViewGeometry.PLANAR_OR_PANORAMIC) and g.H is not None
    if (use_e or use_h) and (cam1 is None or cam2 is None):
        raise FeatureMatchingError("guided matching with E or H needs a camera for each image")
    if use_h and (cam1.model_id == EQUIRECTANGULAR or cam2.model_id == EQUIRECTANGULAR):
        raise FeatureMatchingError("a homography is not a valid model for a spherical camera")
    if use_e:
        return GUIDED_E, np.asarray(g.E, np.float64).reshape(3, 3), cam1, cam2
    if use_f:
        return GUIDED_F, np.asarray(g.F, np.float64).reshape(3, 3), cam1, cam2
    if use_h:
        return GUIDED_H, np.asarray(g.H, np.float64).reshape(3, 3), cam1, cam2
    return GUIDED_NONE, None, cam1, cam2


def _camera_key(cam: Camera):
    return (int(cam.model_id), tuple(np.asarray(cam.params, np.float64).ravel().tolist()))


def _check_guided_image(image: FeatureMatcherImage):
    """ThrowCheckFeatureTypesMatch with check_keypoints (sift.cc:100-116)."""
    if not isinstance(image, FeatureMatcherImage) or image.camera is None or image.keypoints is None:
        raise FeatureMatchingError("guided matching needs each image's camera and keypoints")
    if len(image.keypoints) != len(image.descriptors):
        raise FeatureMatchingError(f"image {image.image_id}: {len(image.keypoints)} keypoints but "
                                   f"{len(image.descriptors)} descriptors")


def CamRayFromImgWithJac(camera: Camera, xy) -> Optional[Tuple[np.ndarray, np.ndarray]]:
    """Camera::CamRayFromImgWithJac (scene/camera.h:355-371) as the guided matcher computes it: (unit ray (3,),
    d(ray)/d(pixel) (3, 2)), or None where the reference returns nullopt."""
    prm = np.ascontiguousarray(camera.params, np.float64)
    pt = np.ascontiguousarray(xy, np.float64).reshape(2)
    out = np.zeros(9, np.float64)
    rc = _check(_lib().b200sm_cam_ray_from_img_with_jac(int(camera.model_id), prm.ctypes.data_as(_f64p),
                                                        pt.ctypes.data_as(_f64p), out.ctypes.data_as(_f64p)),
                "b200sm_cam_ray_from_img_with_jac")
    return (out[:3].copy(), out[3:].reshape(3, 2).copy()) if rc == 1 else None


class SiftFeatureMatcher:
    """Brute-force SIFT matching on one GPU.  Used by one thread at a time; close() frees the device memory."""

    def __init__(self, options: FeatureMatchingOptions):
        if not options.Check():
            raise FeatureMatchingError("FeatureMatchingOptions::Check failed")
        self.options = options
        self._copts = options.to_c()
        self._h = ctypes.c_void_p()
        self._num_slots = 0
        self._slot_ids: List[int] = []
        self._reserve(2)

    def _reserve(self, num_slots):
        if num_slots <= self._num_slots:
            return
        self.close()
        h = ctypes.c_void_p()
        _check(_lib().b200sm_create(ctypes.byref(self._copts), num_slots, ctypes.byref(h)), "b200sm_create")
        self._h, self._num_slots, self._slot_ids = h, num_slots, [kInvalidImageId] * num_slots
        self._slot_geo = [(False, None)] * num_slots

    def _upload(self, slot, image: FeatureMatcherImage):
        if not isinstance(image, FeatureMatcherImage):
            image = FeatureMatcherImage(kInvalidImageId, image)
        if image.image_id != kInvalidImageId and self._slot_ids[slot] == image.image_id:
            return
        d = image.descriptors
        self._slot_ids[slot] = kInvalidImageId
        self._slot_geo[slot] = (False, None)     # uploading descriptors clears the slot's keypoints and camera
        _check(_lib().b200sm_set_descriptors(self._h, slot, len(d), d.ctypes.data_as(_u8p)), "b200sm_set_descriptors")
        self._slot_ids[slot] = image.image_id

    def _upload_guided(self, slot, image: FeatureMatcherImage, camera: Optional[Camera]):
        """Descriptors and keypoints of `image`, and with `camera` its rays, into `slot`.  The cache key is the image id,
        whether keypoints are on the device, and the camera's model and parameters (the reference's
        SameNormalizationCamera, sift.cc:1523-1580)."""
        self._upload(slot, image)
        fresh = image.image_id == kInvalidImageId
        has_kp, cam_key = self._slot_geo[slot]
        if fresh or not has_kp:
            k = image.keypoints
            self._slot_geo[slot] = (False, None)
            _check(_lib().b200sm_set_keypoints(self._h, slot, len(k), k.ctypes.data_as(_f32p)), "b200sm_set_keypoints")
            self._slot_geo[slot] = (True, None)
            cam_key = None
        if camera is not None and (fresh or cam_key != _camera_key(camera)):
            prm = np.zeros(16, np.float64)
            p = np.asarray(camera.params, np.float64).ravel()
            prm[:len(p)] = p
            self._slot_geo[slot] = (True, None)
            _check(_lib().b200sm_set_camera(self._h, slot, int(camera.model_id), prm.ctypes.data_as(_f64p)),
                   "b200sm_set_camera")
            self._slot_geo[slot] = (True, _camera_key(camera))

    def _run(self, slot1: np.ndarray, slot2: np.ndarray, guided=None) -> List[np.ndarray]:
        L = _lib()
        P = len(slot1)
        s1 = np.ascontiguousarray(slot1, np.int32); s2 = np.ascontiguousarray(slot2, np.int32)
        p1, p2 = s1.ctypes.data_as(_i32p), s2.ctypes.data_as(_i32p)
        cap = _check(L.b200sm_match_capacity(self._h, P, p1, p2), "b200sm_match_capacity")
        offsets = np.zeros(P + 1, np.uint64)
        matches = np.zeros((max(cap, 1), 2), np.uint32)
        po, pm = offsets.ctypes.data_as(_u64p), matches.ctypes.data_as(_u32p)
        if guided is None:
            _check(L.b200sm_match_pairs(self._h, P, p1, p2, po, pm, cap), "b200sm_match_pairs")
        else:
            _check(L.b200sm_match_guided_pairs(self._h, P, p1, p2, guided, po, pm, cap), "b200sm_match_guided_pairs")
        return [matches[int(offsets[p]):int(offsets[p + 1])].copy() for p in range(P)]

    def Match(self, image1: FeatureMatcherImage, image2: FeatureMatcherImage) -> np.ndarray:
        """Matches of image1 against image2: (k, 2) uint32 (point2D_idx1, point2D_idx2), ascending point2D_idx1."""
        self._check_open()
        self._upload(0, image1)
        self._upload(1, image2)
        return self._run(np.array([0], np.int32), np.array([1], np.int32))[0]

    def MatchPairs(self, images: Sequence[FeatureMatcherImage], pairs: Sequence[Tuple[int, int]]) -> List[np.ndarray]:
        """Matches of every (i, j) in `pairs` (indices into `images`) in one device call: a list of (k, 2) uint32."""
        self._check_open()
        pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
        if len(pairs) and (pairs.min() < 0 or pairs.max() >= len(images)):
            raise FeatureMatchingError("pair index outside the image list")
        self._reserve(len(images))
        for k, im in enumerate(images):
            self._upload(k, im)
        return self._run(pairs[:, 0].astype(np.int32), pairs[:, 1].astype(np.int32))

    def MatchGuided(self, max_error: float, image1: FeatureMatcherImage, image2: FeatureMatcherImage,
                    two_view_geometry: TwoViewGeometry) -> None:
        """FeatureMatcher::MatchGuided (feature/matcher.h:129): sets two_view_geometry.inlier_matches to the guided
        matches, (k, 2) uint32 in ascending point2D_idx1 (none when the geometry gives no model)."""
        self.MatchGuidedPairs([image1, image2], [(0, 1)], [two_view_geometry], max_error)

    def MatchGuidedPairs(self, images: Sequence[FeatureMatcherImage], pairs: Sequence[Tuple[int, int]],
                         geometries: Sequence[TwoViewGeometry], max_error: float) -> List[np.ndarray]:
        """MatchGuided of every (i, j) in `pairs` under geometries[p], in one device call.  Sets each geometry's
        inlier_matches and returns them.  An E pair runs on the rays of its effective cameras, so an image seen through
        different effective cameras takes one slot per camera."""
        self._check_open()
        pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
        if len(pairs) != len(geometries):
            raise FeatureMatchingError("one two-view geometry per pair")
        if len(pairs) and (pairs.min() < 0 or pairs.max() >= len(images)):
            raise FeatureMatchingError("pair index outside the image list")
        if not np.isfinite(max_error) or max_error < 0:
            raise FeatureMatchingError("max_error must be finite and >= 0")
        for g in geometries:
            g.inlier_matches = np.zeros((0, 2), np.uint32)
        slot_of, uploads = {}, []          # (image index, camera key or None) -> slot

        def slot(k, cam):
            key = (k, None if cam is None else _camera_key(cam))
            if key not in slot_of:
                slot_of[key] = len(uploads)
                uploads.append((images[k], cam))
            return slot_of[key]

        c = (_CGuided * max(len(pairs), 1))()
        s1, s2 = np.zeros(len(pairs), np.int32), np.zeros(len(pairs), np.int32)
        for p, ((i, j), g) in enumerate(zip(pairs, geometries)):
            _check_guided_image(images[i]); _check_guided_image(images[j])
            typ, M, cam1, cam2 = SelectGuidedModel(g, images[i], images[j])
            e = typ == GUIDED_E
            s1[p], s2[p] = slot(i, cam1 if e else None), slot(j, cam2 if e else None)
            c[p].type, c[p].max_error = typ, float(max_error)
            if M is not None:
                c[p].M[:] = M.ravel().tolist()
        self._reserve(max(len(uploads), 2))
        for k, (im, cam) in enumerate(uploads):
            self._upload_guided(k, im, cam)
        out = self._run(s1, s2, c)
        for g, m in zip(geometries, out):
            g.inlier_matches = m
        return out

    def LastTiming(self) -> Tuple[float, float]:
        """Device time (ms) of the last call: the product and top-2 scan, and all of the call's device work."""
        a, b = ctypes.c_double(), ctypes.c_double()
        _check(_lib().b200sm_last_timing(self._h, ctypes.byref(a), ctypes.byref(b)), "b200sm_last_timing")
        return a.value, b.value

    def _check_open(self):
        if not self._h:
            raise FeatureMatchingError("matcher is closed")

    def close(self):
        if self._h:
            _lib().b200sm_destroy(self._h)
        self._h, self._num_slots, self._slot_ids, self._slot_geo = ctypes.c_void_p(), 0, [], []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def CreateSiftFeatureMatcher(options: Optional[FeatureMatchingOptions] = None) -> SiftFeatureMatcher:
    """CreateSiftFeatureMatcher (feature/sift.h:140) with use_gpu: the brute-force matcher on one GPU."""
    return SiftFeatureMatcher(options if options is not None else FeatureMatchingOptions())
