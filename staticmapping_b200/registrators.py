"""Host-side mirror of the reference's plugin surface, registrator::Interface
(registrators/interface.h:67-119 of the reference), over the C ABI of libsm_b200.so.

Same member names, argument meaning and error behaviour as the reference:

* ``CreateMatcher(options)``            interface.cc:139-173
* ``Interface.InitWithXml(node)``       interface.cc:62-90  (unknown <param> -> CheckFailure,
                                         the reference glog-CHECK-aborts)
* ``SetInputSource / SetInputTarget``   icp_fast.cc:421-431 (deep copy; target needs normals)
* ``Align(guess) -> (ok, result)``      icp_fast.cc:455-529 (C++: bool Align(guess, result&))
* ``GetFitnessScore / GetType / PrintOptions / Enable/DisableInnerCompensation``

Clouds are passed as the data the reference's ``InnerPointCloudData`` holds for each
matcher: an ``EigenCloud`` (double points [+ normals]) for IcpFast.
"""
from __future__ import annotations

import ctypes as C
import enum
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import _lib


class Type(enum.IntEnum):
    """registrator::Type (interface.h:41-50)."""
    kNoType = 0
    kIcpPM = 1
    kLibicp = 2
    kNdtWithGicp = 3
    kLegoLoam = 4
    kNdt = 5
    kFastIcp = 6


class CheckFailure(RuntimeError):
    """Raised where the reference would glog CHECK-fail (abort)."""


class NeighborSearchMethod(enum.IntEnum):
    """pclomp::NeighborSearchMethod (registrators/pclomp/ndt_omp.h:52-57), for Ndt.SetNeighborhoodSearchMethod."""
    KDTREE = 0
    DIRECT26 = 1
    DIRECT7 = 2
    DIRECT1 = 3


class ErrorMinimizer(enum.IntEnum):
    """The ICP iteration's error minimizer, for IcpFast / IcpUsingPointMatcher.SetErrorMinimizer.
    POINT_TO_PLANE (the default) is what the reference runs; POINT_TO_POINT is its ComputePointToPoint
    (icp_fast.cc:326-375), libpointmatcher's PointToPointErrorMinimizer."""
    POINT_TO_PLANE = 0
    POINT_TO_POINT = 1


class SurfaceNormals(enum.IntEnum):
    """The reference filter of IcpUsingPointMatcher (libpointmatcher's SamplingSurfaceNormalDataPointsFilter, knn 7),
    for IcpUsingPointMatcher.SetSurfaceNormals.  LEAST_SQUARES (the default) is CalculateNormals' plane fit
    (cloud_types.cc:73-103), the reference author's port of the filter; EIGENVECTOR is the filter's own leaf: the
    float box mean and the smallest eigenvector of the box covariance.  See sm_set_pm_surface_normals."""
    LEAST_SQUARES = 0
    EIGENVECTOR = 1


class ReadingSampler(enum.IntEnum):
    """The reading filter of IcpUsingPointMatcher (libpointmatcher's RandomSamplingDataPointsFilter, prob 0.9), for
    IcpUsingPointMatcher.SetReadingSampler.  HASH (the default) keeps point i by a counter hash of (i, sample_seed);
    GLIBC_RAND by (float)rand() / (float)RAND_MAX < prob with glibc's rand() stream after srand(sample_seed), from
    the matcher's stream position (GetRandPosition / SetRandPosition).  See sm_set_pm_reading_sampler."""
    HASH = 0
    GLIBC_RAND = 1


@dataclass
class EigenCloud:
    """data::EigenPointCloud (cloud_types.h:121-147): (N,3) float64 points, optional normals.
    C-contiguous (N,3) == Eigen's 3xN column-major storage."""
    points: np.ndarray
    normals: Optional[np.ndarray] = None

    def __post_init__(self):
        self.points = np.ascontiguousarray(np.asarray(self.points, dtype=np.float64))
        if self.points.ndim != 2 or self.points.shape[1] != 3:
            raise ValueError("points must be (N,3)")
        if self.normals is not None:
            self.normals = np.ascontiguousarray(np.asarray(self.normals, dtype=np.float64))
            if self.normals.shape != self.points.shape:
                raise ValueError("normals must match points")

    def HasNormals(self):
        return self.normals is not None and self.normals.shape[0] > 0

    @staticmethod
    def FromPointCloud(xyz_f32):
        """EigenPointCloud::FromPointCloud (cloud_types.cc:328-345): float AoS -> double."""
        return EigenCloud(np.asarray(xyz_f32, dtype=np.float32).astype(np.float64))


@dataclass
class InnerCloud:
    """data::InnerCloudType (cloud_types.h:59-77): the float cloud `Ndt` / `NdtWithGicp` keep
    (x, y, z of InnerPointType; intensity / factor are not used by the matchers).
    points: (N,3) float32, or (N,5) float32 rows laid out like InnerPointType (20-byte stride)."""
    points: np.ndarray

    def __post_init__(self):
        self.points = np.ascontiguousarray(np.asarray(self.points, dtype=np.float32))
        if self.points.ndim != 2 or self.points.shape[1] not in (3, 5):
            raise ValueError("points must be (N,3) or (N,5) float32")

    def Empty(self):
        return self.points.shape[0] == 0

    @property
    def stride_bytes(self):
        return 4 * self.points.shape[1]


@dataclass
class MatcherOptions:
    """registrator::MatcherOptions (interface.h:59-65)."""
    type: Type = Type.kIcpPM
    accepted_min_score: float = 0.7
    registrator_options_node: Optional[object] = None   # xml string / Element / dict
    inner_filters_node: Optional[object] = None


def _params_from_node(node):
    if node is None:
        return []
    if isinstance(node, dict):
        return [(k, str(v)) for k, v in node.items()]
    if isinstance(node, (str, bytes)):
        node = ET.fromstring(node)
    return [(p.attrib.get("name", ""), (p.text or "").strip()) for p in node.findall("param")]


class Interface:
    """registrator::Interface.  One instance is used by one thread at a time; distinct
    instances may run concurrently (each owns a CUDA stream + workspace)."""

    _type = Type.kNoType

    def __init__(self, device: int = 0):
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        rc = self._lib.sm_create(int(self._type), device, C.byref(self._h))
        if rc == -20:
            raise RuntimeError("staticmapping_b200: no CUDA device visible and there is no CPU "
                               "fallback (SM_ERR_NO_DEVICE)")
        if rc != 0:
            raise RuntimeError(f"sm_create failed with {rc}")
        self._inner_compensation = False
        self._source = None
        self._target = None

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self._lib.sm_destroy(h)
            self._h = C.c_void_p()

    def _check(self, rc, what):
        if rc < 0:
            msg = self._lib.sm_last_error(self._h)
            raise CheckFailure(f"{what}: {msg.decode() if msg else rc} (code {rc})")
        return rc

    # --- options -------------------------------------------------------------------------
    def InitWithXml(self, node):
        for name, text in _params_from_node(node):
            self._check(self._lib.sm_set_option(self._h, name.encode(), text.encode()),
                        "InitWithXml")

    def InitInnerFiltersWithXml(self, node):
        return None  # interface.cc:92-113: a TODO in the reference, no effect

    def InitWithOptions(self):
        return None

    def PrintOptions(self):
        buf = C.create_string_buffer(4096)
        self._lib.sm_print_options(self._h, buf, 4096)
        text = buf.value.decode()
        print(text, end="")
        return text

    # interface.cc:34-36; takes effect from the next Align.  IcpFast de-skews the source in every
    # iteration (icp_fast.cc:487-491); the other types keep the flag without effect, as in the reference.
    def EnableInnerCompensation(self):
        self._inner_compensation = True
        self._check(self._lib.sm_set_inner_compensation(self._h, 1), "EnableInnerCompensation")

    def DisableInnerCompensation(self):
        self._inner_compensation = False
        self._check(self._lib.sm_set_inner_compensation(self._h, 0), "DisableInnerCompensation")

    # --- data ----------------------------------------------------------------------------
    def SetInputSource(self, cloud: EigenCloud):
        raise NotImplementedError

    def SetInputTarget(self, cloud: EigenCloud):
        raise NotImplementedError

    def Align(self, guess):
        """Returns (ok, result 4x4).  C++: bool Align(const Matrix4d& guess, Matrix4d& result)."""
        g = np.ascontiguousarray(np.asarray(guess, dtype=np.float64).T).ravel()
        res = np.zeros(16, dtype=np.float64)
        rc = self._check(self._lib.sm_align(self._h, g.ctypes.data_as(_lib._DP),
                                            res.ctypes.data_as(_lib._DP)), "Align")
        return bool(rc), res.reshape(4, 4).T.copy()

    def AlignAsync(self, guess):
        """First half of Align: enqueue and return (engine extension, see sm_align_async)."""
        g = np.ascontiguousarray(np.asarray(guess, dtype=np.float64).T).ravel()
        self._check(self._lib.sm_align_async(self._h, g.ctypes.data_as(_lib._DP)), "AlignAsync")

    def AlignWait(self):
        """Second half of Align: returns (ok, result 4x4)."""
        res = np.zeros(16, dtype=np.float64)
        rc = self._check(self._lib.sm_align_wait(self._h, res.ctypes.data_as(_lib._DP)), "AlignWait")
        return bool(rc), res.reshape(4, 4).T.copy()

    def GetFitnessScore(self):
        return float(self._lib.sm_get_fitness_score(self._h))

    def GetType(self):
        return Type(self._lib.sm_get_type(self._h))

    def SetStream(self, cuda_stream: int = 0):
        """Run on the caller's CUDA stream (0 / None -> the handle's own stream)."""
        self._check(self._lib.sm_set_stream(self._h, cuda_stream or None), "SetStream")

    def GetAlignInfo(self):
        info = _lib.AlignInfo()
        self._lib.sm_get_align_info(self._h, C.byref(info))
        out = {k: getattr(info, k) for k, _ in _lib.AlignInfo._fields_ if k not in ("reserved", "aux")}
        out["aux"] = [float(v) for v in info.aux]
        return out


class IcpFast(Interface):
    """registrator::IcpFast (icp_fast.h:37-62)."""
    _type = Type.kFastIcp

    def SetInputSource(self, cloud: EigenCloud):
        if cloud is None or cloud.points.shape[0] == 0:
            raise CheckFailure("SetInputSource: CHECK(cloud) failed (icp_fast.cc:422-423)")
        self._check(self._lib.sm_set_input_source(self._h, cloud.points.ctypes.data,
                                                  cloud.points.shape[0]), "SetInputSource")

    def SetInputTarget(self, cloud: EigenCloud):
        if cloud is None or cloud.points.shape[0] == 0:
            raise CheckFailure("SetInputTarget: CHECK(cloud) failed (icp_fast.cc:428-429)")
        if not cloud.HasNormals():
            raise CheckFailure("SetInputTarget: CHECK(HasNormals()) failed (icp_fast.cc:430)")
        self._check(self._lib.sm_set_input_target(self._h, cloud.points.ctypes.data,
                                                  cloud.normals.ctypes.data,
                                                  cloud.points.shape[0]), "SetInputTarget")

    def SetErrorMinimizer(self, minimizer):
        """An ErrorMinimizer; applies from the next Align on.  Target normals are still required (icp_fast.cc:430)
        but point-to-point does not read them.  See sm_set_icp_error_minimizer in include/sm_b200.h."""
        self._check(self._lib.sm_set_icp_error_minimizer(self._h, int(minimizer)), "SetErrorMinimizer")

    # device-resident variants (pointers to 3xN column-major doubles in this GPU's memory)
    def SetInputSourceDevice(self, dev_ptr: int, n: int):
        self._check(self._lib.sm_set_input_source_device(self._h, dev_ptr, n), "SetInputSource")

    def SetInputTargetDevice(self, dev_points: int, dev_normals: int, n: int):
        self._check(self._lib.sm_set_input_target_device(self._h, dev_points, dev_normals, n),
                    "SetInputTarget")


class Ndt(Interface):
    """registrator::Ndt (ndt.h / ndt.cc:28-64): pclomp NDT, resolution 1.0, KDTREE neighbour
    search.  GetFitnessScore() is PCL's mean squared NN distance (LOWER is better), unlike the
    ICP matchers' exp(-distance) (SURVEY 3.4)."""
    _type = Type.kNdt

    def InitWithXml(self, node):
        # Ndt registers no option (ndt.cc:28-34): any <param> hits the CHECK in interface.cc:66
        for name, _ in _params_from_node(node):
            raise CheckFailure(f"Init an unknown option of this matcher! ({name})")

    def SetEngineOptions(self, **kw):
        """pclomp setters the reference hard-codes (resolution, step_size, outlier_ratio,
        transformation_epsilon, max_iterations); not reachable from the reference's XML."""
        for k, v in kw.items():
            self._check(self._lib.sm_set_option(self._h, k.encode(), str(v).encode()), "option")

    def SetNeighborhoodSearchMethod(self, method):
        """pclomp setNeighborhoodSearchMethod (ndt_omp.h:184): a NeighborSearchMethod; applies from the next
        Align on.  KDTREE (the reference's choice, ndt.cc:33) is the default; see sm_set_ndt_search_method in
        include/sm_b200.h for what the direct searches visit.  NdtWithGicp raises CheckFailure: its NDT stage is
        stock PCL's, which has no such setter."""
        self._check(self._lib.sm_set_ndt_search_method(self._h, int(method)), "SetNeighborhoodSearchMethod")

    def SetInputSource(self, cloud: InnerCloud):
        # Interface::SetInputSource (interface.cc:38-48): null resets, empty only warns
        self._source = None
        if cloud is None:
            return
        if cloud.Empty():
            print("cloud is empty.")
            return
        self._check(self._lib.sm_set_input_source_f32(self._h, cloud.points.ctypes.data,
                                                      cloud.points.shape[0], cloud.stride_bytes),
                    "SetInputSource")
        self._source = cloud

    def SetInputTarget(self, cloud: InnerCloud):
        self._target = None
        if cloud is None:
            return
        if cloud.Empty():
            print("cloud is empty.")
            return
        self._check(self._lib.sm_set_input_target_f32(self._h, cloud.points.ctypes.data,
                                                      cloud.points.shape[0], cloud.stride_bytes),
                    "SetInputTarget")
        self._target = cloud

    def Align(self, guess):
        if self._source is None or self._target is None:   # ndt.cc:40-42
            return False, np.asarray(guess, dtype=np.float64).copy()
        return super().Align(guess)


class NdtWithGicp(Ndt):
    """registrator::NdtWithGicp (ndt_gicp.h / ndt_gicp.cc:28-112): ApproximateVoxelGrid(0.2 m) on
    both clouds -> stock PCL NDT (resolution 1.0, step 0.1, eps 0.01, 35 it) -> stock PCL GICP
    (rotation eps 1e-3, 35 it), gated on NDT fitness <= 1.  GetFitnessScore() = exp(-GICP fitness).
    Registered options (ndt_gicp.cc:31-36): use_ndt, using_voxel_filter, voxel_resolution."""
    _type = Type.kNdtWithGicp

    def InitWithXml(self, node):
        Interface.InitWithXml(self, node)

    def Align(self, guess):
        if self._source is None or self._target is None:
            raise CheckFailure("NdtWithGicp::Align: input cloud not set (null dereference in the reference)")
        return Interface.Align(self, guess)


class IcpUsingPointMatcher(Ndt):
    """Stand-in for registrator::IcpUsingPointMatcher (icp_pointmatcher.h / .cc:125-247), the
    libpointmatcher-driven ICP that loop_detector.cc:304-308 constructs directly.  Same module
    chain as the reference's default config (:166-247): reading filter RandomSampling 0.9,
    reference filter SamplingSurfaceNormal knn 7 (== CalculateNormals), k-d tree matcher eps 3.16,
    TrimmedDist 0.7, point-to-plane minimiser, 150-iteration counter + 4-sample differential
    checker; GetFitnessScore() = exp(-mean kept distance) of the UNFILTERED clouds re-matched after
    the result (:131-148), Align() is False below 0.6 (:145).
    libpointmatcher itself (1.3.1, float, std::rand) is external to the reference tree, so this is
    a deterministic double-precision equivalent built from the IcpFast kernels, not a bit-level
    restatement.  It registers no XML option (the reference takes a YAML file name instead)."""
    _type = Type.kIcpPM

    def __init__(self, device: int = 0, ymal_file: str = ""):
        if ymal_file:
            raise CheckFailure("IcpUsingPointMatcher: YAML configs are not supported, only loadDefaultConfig()")
        super().__init__(device)

    def SetErrorMinimizer(self, minimizer):
        """An ErrorMinimizer for the ICP chain of the stand-in (the reference's loadDefaultConfig builds
        PointToPointErrorMinimizer, icp_pointmatcher.cc:202-204, before it installs point-to-plane, :239);
        applies from the next Align on."""
        self._check(self._lib.sm_set_icp_error_minimizer(self._h, int(minimizer)), "SetErrorMinimizer")

    def SetSurfaceNormals(self, mode):
        """A SurfaceNormals mode for the reference filter; applies from the next Align on, which filters the
        reference cloud anew when the mode changed.  See sm_set_pm_surface_normals in include/sm_b200.h."""
        self._check(self._lib.sm_set_pm_surface_normals(self._h, int(mode)), "SetSurfaceNormals")

    def SetReadingSampler(self, mode):
        """A ReadingSampler mode for the reading filter; applies from the next Align on.  In GLIBC_RAND mode every
        Align filters the reading cloud anew and advances the stream position by its size.  See
        sm_set_pm_reading_sampler in include/sm_b200.h."""
        self._check(self._lib.sm_set_pm_reading_sampler(self._h, int(mode)), "SetReadingSampler")

    def GetRandPosition(self):
        """The number of rand() draws taken since srand(sample_seed) (sm_get_pm_rand_position)."""
        pos = C.c_int64()
        self._check(self._lib.sm_get_pm_rand_position(self._h, C.byref(pos)), "GetRandPosition")
        return pos.value

    def SetRandPosition(self, position):
        """Where the next GLIBC_RAND Align starts drawing: the draws taken since srand(sample_seed), >= 0
        (sm_set_pm_rand_position).  Setting sample_seed resets it to 0."""
        self._check(self._lib.sm_set_pm_rand_position(self._h, int(position)), "SetRandPosition")

    def Align(self, guess):
        if self._source is None or self._target is None:
            raise CheckFailure("IcpUsingPointMatcher::Align: input cloud not set")
        return Interface.Align(self, guess)


def CreateMatcher(options: MatcherOptions, verbose: bool = False, device: int = 0) -> Interface:
    """registrator::CreateMatcher (interface.cc:139-173)."""
    t = Type(options.type)
    if t == Type.kFastIcp:
        matcher = IcpFast(device)
    elif t in (Type.kLibicp, Type.kLegoLoam):
        raise CheckFailure("The registrator using libicp & lego-loam is deprecated. "
                           "please choose another type")   # LOG(FATAL), interface.cc:154-157
    elif t == Type.kNdt:
        matcher = Ndt(device)
    elif t == Type.kNdtWithGicp:
        matcher = NdtWithGicp(device)
    elif t == Type.kIcpPM:
        matcher = IcpUsingPointMatcher(device)
    else:
        print("Wrong type")   # PRINT_ERROR + nullptr, interface.cc:158-160
        return None
    if options.registrator_options_node is not None:
        matcher.InitWithXml(options.registrator_options_node)
    if verbose:
        matcher.PrintOptions()
    matcher.InitWithOptions()
    return matcher


def AlignBatch(matchers, guesses):
    """Batched Align over matcher instances whose inputs are set (sm_align_batch): what
    loop_detector.cc:216-228 / map_builder.cc:706-708 do with a thread pool, from one host thread.
    Returns (oks, results) with results of shape (n, 4, 4)."""
    n = len(matchers)
    lib = _lib.lib()
    hs = (C.c_void_p * n)(*[m._h for m in matchers])
    g = np.ascontiguousarray(np.stack([np.asarray(x, dtype=np.float64).T for x in guesses]).reshape(n, 16))
    res = np.zeros((n, 16), dtype=np.float64)
    rcs = np.zeros(n, dtype=np.int32)
    lib.sm_align_batch(hs, n, g.ctypes.data, res.ctypes.data, rcs.ctypes.data)
    for m, rc in zip(matchers, rcs):
        m._check(int(rc), "AlignBatch")
    return [bool(r) for r in rcs], res.reshape(n, 4, 4).transpose(0, 2, 1).copy()


def AlignPairs(matchers, pairs):
    """n_pairs independent IcpFast alignments pipelined over the given instances (sm_align_pairs).
    `pairs`: sequence of dicts {source, target, normals, guess (optional), on_device (optional)} where
    the clouds are (N, 3) float64 C-contiguous arrays (host; pinned memory overlaps best) or, with
    on_device, integer device pointers plus n_source / n_target.
    Returns (rcs, results (n, 4, 4), scores (n,))."""
    n = len(pairs)
    lib = _lib.lib()
    hs = (C.c_void_p * len(matchers))(*[m._h for m in matchers])
    arr = (_lib.Pair * n)()
    keep = []
    for k, pr in enumerate(pairs):
        dev = bool(pr.get("on_device", False))
        if dev:
            arr[k].source, arr[k].target, arr[k].target_normals = pr["source"], pr["target"], pr["normals"]
            arr[k].n_source, arr[k].n_target = int(pr["n_source"]), int(pr["n_target"])
        else:
            src, tgt, nrm = pr["source"], pr["target"], pr["normals"]
            arr[k].source, arr[k].target, arr[k].target_normals = _ptr(src), _ptr(tgt), _ptr(nrm)
            arr[k].n_source = int(pr["n_source"]) if "n_source" in pr else len(src)
            arr[k].n_target = int(pr["n_target"]) if "n_target" in pr else len(tgt)
        g = pr.get("guess")
        if g is not None:
            g = np.ascontiguousarray(np.asarray(g, dtype=np.float64).T).ravel()
            keep.append(g)
            arr[k].guess = g.ctypes.data
        arr[k].on_device = 1 if dev else 0
    res = np.zeros((n, 16), dtype=np.float64)
    scores = np.zeros(n, dtype=np.float64)
    rcs = np.zeros(n, dtype=np.int32)
    rc = lib.sm_align_pairs(hs, len(matchers), arr, n, res.ctypes.data, scores.ctypes.data, rcs.ctypes.data)
    if rc == -11:
        raise CheckFailure("AlignPairs: IcpFast instances only")
    for k, r in enumerate(rcs):
        matchers[k % len(matchers)]._check(int(r), "AlignPairs")
    return rcs, res.reshape(n, 4, 4).transpose(0, 2, 1).copy(), scores


def _ptr(a):
    """address of a float64 (N, 3) C-contiguous numpy array or torch tensor (data_ptr), or an int"""
    if isinstance(a, int):
        return a
    if hasattr(a, "data_ptr"):
        return int(a.data_ptr())
    a = np.asarray(a)
    if a.dtype != np.float64 or not a.flags["C_CONTIGUOUS"]:
        raise ValueError("AlignPairs needs C-contiguous float64 clouds (no hidden copies: the engine reads them asynchronously)")
    return a.ctypes.data


def knn1(target, query, epsilon=3.16, bucket_size=8, device=0, queries_per_cta=0):
    """libnabo-compatible 1-NN on the GPU (NNS::create + knn, icp_fast.cc:466-467,177-178).
    queries_per_cta > 0: the test hook sm_debug_knn1_batched (the launch shape of batched alignments)."""
    lib = _lib.lib()
    t = np.ascontiguousarray(np.asarray(target, dtype=np.float64))
    q = np.ascontiguousarray(np.asarray(query, dtype=np.float64))
    ids = np.empty(q.shape[0], dtype=np.int32)
    d2 = np.empty(q.shape[0], dtype=np.float64)
    if queries_per_cta:
        rc = lib.sm_debug_knn1_batched(device, t.ctypes.data, t.shape[0], q.ctypes.data, q.shape[0], float(epsilon),
                                       int(bucket_size), int(queries_per_cta), ids.ctypes.data, d2.ctypes.data)
    else:
        rc = lib.sm_knn1(device, t.ctypes.data, t.shape[0], q.ctypes.data, q.shape[0], float(epsilon),
                         int(bucket_size), ids.ctypes.data, d2.ctypes.data)
    if rc == -20:
        raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
    if rc != 0:
        raise RuntimeError(f"sm_knn1 failed with {rc}")
    return ids, d2


def knn(target, query, k, epsilon=0.0, max_radius=float("inf"), allow_self_match=True, bucket_size=8, device=0):
    """libnabo's k-nearest-neighbour search on the GPU: NNS::create(target, 3, KDTREE_LINEAR_HEAP) + knn(query, k,
    epsilon, flags, max_radius), k = 1..64.  target / query: (n, 3) float64.  Returns (ids int32, d2 float64), each of
    shape (n_query, k): row i holds query i's neighbours in ascending squared distance, (-1, +inf) where fewer than k
    points lie within max_radius (or the target is smaller than k).  allow_self_match=False drops points at squared
    distance <= DBL_EPSILON (libnabo's ALLOW_SELF_MATCH flag unset)."""
    lib = _lib.lib()
    t = np.ascontiguousarray(np.asarray(target, dtype=np.float64))
    q = np.ascontiguousarray(np.asarray(query, dtype=np.float64))
    if t.ndim != 2 or t.shape[1] != 3 or q.ndim != 2 or q.shape[1] != 3:
        raise ValueError("knn needs (n, 3) target and query clouds")
    kk = int(k)
    ids = np.empty((q.shape[0], max(kk, 1)), dtype=np.int32)
    d2 = np.empty((q.shape[0], max(kk, 1)), dtype=np.float64)
    flags = 1 if allow_self_match else 0
    rc = lib.sm_knn(device, t.ctypes.data, t.shape[0], q.ctypes.data, q.shape[0], kk, float(epsilon),
                    float(max_radius), flags, int(bucket_size), ids.ctypes.data, d2.ctypes.data)
    if rc == -20:
        raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
    if rc == -1:
        raise ValueError(f"sm_knn rejected its arguments (k={k}, epsilon={epsilon}, max_radius={max_radius}, "
                         f"bucket_size={bucket_size}, n_target={t.shape[0]})")
    if rc != 0:
        raise RuntimeError(f"sm_knn failed with {rc}")
    return ids, d2


def CalculateNormals(points, device=0) -> EigenCloud:
    """EigenPointCloud::CalculateNormals on the GPU (cloud_types.cc:347-368): returns the
    decimated cloud (one mean point + unit normal per valid <=7-point leaf)."""
    lib = _lib.lib()
    p = np.ascontiguousarray(np.asarray(points, dtype=np.float64))
    out_p = np.empty_like(p)
    out_n = np.empty_like(p)
    m = C.c_int64(0)
    rc = lib.sm_calculate_normals(device, p.ctypes.data, p.shape[0], out_p.ctypes.data,
                                  out_n.ctypes.data, C.byref(m))
    if rc == -20:
        raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
    if rc != 0:
        raise RuntimeError(f"sm_calculate_normals failed with {rc}")
    return EigenCloud(out_p[:m.value].copy(), out_n[:m.value].copy())


def MotionCompensation(raw_cloud, delta_transform, device=0):
    """MotionCompensation (builder/map_builder.cc:232-257) on the GPU.  `raw_cloud` is an (N,5)
    float32 array of InnerPointType rows (x, y, z, intensity, factor); every point is moved by
    common::InterpolateTransform(Identity, delta, factor) (common/math.h:198-211).  Raises
    CheckFailure where the reference CHECK-fails (a factor outside [0, 1])."""
    lib = _lib.lib()
    pts = np.ascontiguousarray(np.asarray(raw_cloud, dtype=np.float32))
    if pts.ndim != 2 or pts.shape[1] != 5:
        raise ValueError("raw_cloud must be (N,5): x, y, z, intensity, factor")
    d = np.asfortranarray(np.asarray(delta_transform, dtype=np.float64))
    if d.shape != (4, 4):
        raise ValueError("delta_transform must be 4x4")
    out = np.empty_like(pts)
    rc = lib.sm_motion_compensation(device, pts.ctypes.data, pts.shape[0], 20, d.ctypes.data_as(_lib._DP),
                                    out.ctypes.data)
    if rc == -20:
        raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
    if rc == -1:
        raise CheckFailure("Check failed: factor >= 0. && factor <= 1. (common/math.h:201)")
    if rc != 0:
        raise RuntimeError(f"sm_motion_compensation failed with {rc}")
    return out


def RotationMatrixToEulerAngles(R):
    """common/math.h:107-127 (host-side 3x3 math; the reference runs it once per frame)."""
    R = np.asarray(R, dtype=np.float64)
    sy = np.sqrt(R[0, 0] * R[0, 0] + R[1, 0] * R[1, 0])
    if not sy < 1e-6:
        return np.array([np.arctan2(R[2, 1], R[2, 2]), np.arctan2(-R[2, 0], sy), np.arctan2(R[1, 0], R[0, 0])])
    return np.array([np.arctan2(-R[1, 2], R[1, 1]), np.arctan2(-R[2, 0], sy), 0.0])


def AverageTransforms(transforms):
    """common::AverageTransforms (common/math.cc:177-195): mean translation, mean Euler angles
    (yaw * pitch * roll composition).  Used by the front end between Align and the second
    MotionCompensation when motion_compensation_options.use_average is set
    (map_builder.cc:333-341)."""
    ts = [np.asarray(t, dtype=np.float64) for t in transforms]
    if not ts:
        raise CheckFailure("Check failed: !transforms.empty() (common/math.cc:180)")
    tr = sum(t[:3, 3] for t in ts) / float(len(ts))
    ang = sum(RotationMatrixToEulerAngles(t[:3, :3]) for t in ts) / float(len(ts))

    def quat(angle, axis):
        q = np.zeros(4)
        q[0] = np.cos(0.5 * angle)
        q[1 + axis] = np.sin(0.5 * angle)
        return q

    def mul(a, b):
        return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                         a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                         a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                         a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])

    w, x, y, z = mul(mul(quat(ang[2], 2), quat(ang[1], 1)), quat(ang[0], 0))
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    out = np.eye(4)
    out[:3, :3] = [[1.0 - (tyy + tzz), txy - twz, txz + twy],
                   [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                   [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]
    out[:3, 3] = tr
    return out


def VoxelGridFilter(cloud, voxel_size, device=0):
    """pre_processers::filter::VoxelGrid::Filter (pre_processors/filter_voxel_grid.cc:37-78) on
    the GPU.  `cloud`: (N,5) float32 InnerPointType rows; returns the (M,5) voxel means in
    ascending (ix, iy, iz) order (the reference's order is std::unordered_map iteration order)."""
    lib = _lib.lib()
    pts = np.ascontiguousarray(np.asarray(cloud, dtype=np.float32))
    if pts.ndim != 2 or pts.shape[1] != 5:
        raise ValueError("cloud must be (N,5): x, y, z, intensity, factor")
    out = np.empty_like(pts)
    m = C.c_int64(0)
    rc = lib.sm_voxel_grid_filter(device, pts.ctypes.data, pts.shape[0], 20, float(voxel_size), out.ctypes.data,
                                  C.byref(m))
    if rc == -20:
        raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
    if rc == -1:
        raise CheckFailure("VoxelGrid: invalid voxel_size (ConfigsValid) or a coordinate outside the voxel index range")
    if rc != 0:
        raise RuntimeError(f"sm_voxel_grid_filter failed with {rc}")
    return out[:m.value].copy()


class M2dp:
    """descriptor::M2dp (descriptor/m2dp.h:45-84) on the GPU: setInputCloud / getFinalDescriptor."""

    def __init__(self, r=0.1, max_distance=100.0, t=16, p=4, q=16, device=0):
        self.r, self.max_distance, self.t, self.p, self.q, self.device = float(r), float(max_distance), int(t), int(p), int(q), device
        self._descriptor = None
        self.signature_matrix = None

    def setInputCloud(self, cloud):
        """cloud: InnerCloud or (N,3)/(N,5) float32 array.  Returns False for an empty cloud (m2dp.cc:130-133)."""
        pts = cloud.points if isinstance(cloud, InnerCloud) else np.ascontiguousarray(np.asarray(cloud, dtype=np.float32))
        lib = _lib.lib()
        n = lib.sm_m2dp_descriptor_length(self.r, self.max_distance, self.t, self.p, self.q)
        if n < 0:
            raise CheckFailure("M2dp: r is too small (m2dp.cc:64-67) or bad parameters")
        desc = np.zeros(n, np.float32)
        A = np.zeros((self.p * self.q, (n - self.p * self.q)), np.int32)
        rc = lib.sm_m2dp(self.device, pts.ctypes.data, pts.shape[0], 4 * pts.shape[1], self.r, self.max_distance,
                         self.t, self.p, self.q, desc.ctypes.data, n, A.ctypes.data)
        if rc == -20:
            raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
        if rc < 0:
            raise CheckFailure(f"sm_m2dp failed with {rc}")
        if rc == 0:
            return False
        self._descriptor, self.signature_matrix = desc, A
        return True

    def getFinalDescriptor(self):
        return self._descriptor


def matchTwoM2dpDescriptors(P, Q):
    """descriptor::matchTwoM2dpDescriptors (m2dp.cc:155-170): |Pearson correlation| in (0, 1), -1 on mismatch."""
    P = np.ascontiguousarray(P, np.float32); Q = np.ascontiguousarray(Q, np.float32)
    if P.shape != Q.shape:
        return -1.0
    return float(_lib.lib().sm_m2dp_match(P.ctypes.data, Q.ctypes.data, P.shape[0]))
