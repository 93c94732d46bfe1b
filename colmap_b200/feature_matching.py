"""Mirror of the reference's SIFT feature matcher (src/colmap/feature/sift.{h,cc}, feature/matcher.h) over
include/b200_sift_matching.h: brute-force matching of uint8 SIFT descriptors on the GPU with the decisions of
FindBestMatchesBruteForce, bit for bit.  Names follow the reference: SiftMatchingOptions, FeatureMatchingOptions,
FeatureMatcher::Image (here FeatureMatcherImage), CreateSiftFeatureMatcher(options).Match(image1, image2).

Like SiftGPUFeatureMatcher::Match, a matcher keeps each image's descriptors on the device and uploads again only when
the image_id in that position changes; MatchPairs matches a whole block of pairs in one call."""
import ctypes
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from ._lib import load_library

kInvalidImageId = 2 ** 32 - 1

_u8p = ctypes.POINTER(ctypes.c_uint8)
_u32p = ctypes.POINTER(ctypes.c_uint32)
_u64p = ctypes.POINTER(ctypes.c_uint64)
_i32p = ctypes.POINTER(ctypes.c_int)


class FeatureMatchingError(RuntimeError):
    pass


class _COptions(ctypes.Structure):
    _fields_ = [("max_ratio", ctypes.c_double), ("max_distance", ctypes.c_double), ("cross_check", ctypes.c_int),
                ("max_num_matches", ctypes.c_int), ("gpu_index", ctypes.c_int)]


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


@dataclass
class FeatureMatcherImage:
    """FeatureMatcher::Image (feature/matcher.h:114-122): the part the descriptor matcher reads."""
    image_id: int
    descriptors: np.ndarray   # (n, 128) uint8

    def __post_init__(self):
        self.descriptors = _as_descriptors(self.descriptors)


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

    def _upload(self, slot, image: FeatureMatcherImage):
        if not isinstance(image, FeatureMatcherImage):
            image = FeatureMatcherImage(kInvalidImageId, image)
        if image.image_id != kInvalidImageId and self._slot_ids[slot] == image.image_id:
            return
        d = image.descriptors
        self._slot_ids[slot] = kInvalidImageId
        _check(_lib().b200sm_set_descriptors(self._h, slot, len(d), d.ctypes.data_as(_u8p)), "b200sm_set_descriptors")
        self._slot_ids[slot] = image.image_id

    def _run(self, slot1: np.ndarray, slot2: np.ndarray) -> List[np.ndarray]:
        L = _lib()
        P = len(slot1)
        s1 = np.ascontiguousarray(slot1, np.int32); s2 = np.ascontiguousarray(slot2, np.int32)
        p1, p2 = s1.ctypes.data_as(_i32p), s2.ctypes.data_as(_i32p)
        cap = _check(L.b200sm_match_capacity(self._h, P, p1, p2), "b200sm_match_capacity")
        offsets = np.zeros(P + 1, np.uint64)
        matches = np.zeros((max(cap, 1), 2), np.uint32)
        _check(L.b200sm_match_pairs(self._h, P, p1, p2, offsets.ctypes.data_as(_u64p), matches.ctypes.data_as(_u32p), cap),
               "b200sm_match_pairs")
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
        self._h, self._num_slots, self._slot_ids = ctypes.c_void_p(), 0, []

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
