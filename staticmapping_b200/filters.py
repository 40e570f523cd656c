"""pre_processers::filter::Factory (pre_processors/filter_factory.h, filter_factory.cc:54-106) over the GPU filter
chain of libsm_b200.so (sm_filter_chain_*, include/sm_b200.h): Range, AxisRange, BoundingBoxRemoval, RandomSampler (a
deterministic stand-in by default, or std::mt19937 at a given seed, see the header), RangeImage and GroundRemoval2, and
RangeImage::DepthCluster; with
Factory.SetAllFilters(True) also StatisticRemoval, GroundRemoval and VoxelGrid.  StatisticRemoval, PCL's statistical
outlier removal, GroundRemoval, the voxel height-range ground filter, and the submap sampler
RandomSamplerWithPlaneDetect also run on their own handles (sm_statistic_removal_*, sm_ground_removal_*,
sm_plane_sampler_*).  There is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import xml.etree.ElementTree as ET
from typing import NamedTuple

import numpy as np

from . import _lib
from .registrators import CheckFailure, InnerCloud


class DepthClusters(NamedTuple):
    """RangeImage::DepthCluster's labelled cloud: clusters in ascending label, each in the reference's visiting order."""
    xyz: np.ndarray            # (m, 3) float32, the input points
    label: np.ndarray          # (m,) uint32
    index: np.ndarray          # (m,) int32, the points' indices in the input cloud
    point_label: np.ndarray    # (n,) uint32, the label of every pixel owner of the input (small clusters too), else 0


def _records(cloud):
    pts = cloud.points if isinstance(cloud, InnerCloud) else np.ascontiguousarray(np.asarray(cloud, dtype=np.float32))
    if pts.ndim != 2 or pts.shape[1] != 5:
        raise ValueError("cloud must be (N,5): x, y, z, intensity, factor")
    return pts


def _param_type(text):
    """a <param>'s type attribute, -1 when it is missing or not an integer (the ABI refuses it)"""
    try:
        return int(text)
    except (TypeError, ValueError):
        return -1


class _RecordFilter:
    """A GPU filter over (N,5) records behind a C handle, whose functions are named `_abi`_create, _run and so on.
    SetInputCloud + Filter run it; `Filter` returns the kept InnerCloud, Inliers() / Outliers() are indices into the
    input."""
    _abi = ""

    def __init__(self, device: int = 0):
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        if self._fn("create")(device, C.byref(self._h)) != 0:
            raise RuntimeError(f"{self._abi}_create failed")
        self._cloud = None
        self._inliers = np.zeros(0, np.int32)
        self._outliers = np.zeros(0, np.int32)

    def __del__(self):
        if getattr(self, "_h", None):
            self._fn("destroy")(self._h)
            self._h = None

    def _fn(self, name):
        return getattr(self._lib, f"{self._abi}_{name}")

    def _error(self):
        return (self._fn("last_error")(self._h) or b"").decode()

    def _check(self, rc, name):
        """the exception for return code `rc` of the entry point `name`"""
        if rc == -20:
            raise RuntimeError("staticmapping_b200: no CUDA device (no CPU fallback)")
        if rc == -5:
            raise CheckFailure(self._error())
        if rc == -1:       # e.g. a RangeImage size of 0, where the reference keeps its previous cloud without a CHECK
            raise ValueError(self._error())
        if rc != 0:
            raise RuntimeError(f"{self._abi}_{name} failed with {rc}: {self._error()}")

    def InitFromXmlText(self, text):
        self.InitFromXmlNode(ET.fromstring(text))

    def SetInputCloud(self, cloud):
        self._cloud = _records(cloud)

    def Filter(self):
        if self._cloud is None:
            return None
        pts = self._cloud
        n = pts.shape[0]
        out = np.empty_like(pts)
        index = np.empty(n, np.int32)
        m = C.c_int64(0)
        self._check(self._fn("run")(self._h, pts.ctypes.data, n, 20, out.ctypes.data, C.byref(m), index.ctypes.data),
                    "run")
        self._inliers = index[:m.value].copy()
        mask = np.ones(n, bool)
        mask[self._inliers] = False
        self._outliers = np.nonzero(mask)[0].astype(np.int32)
        return InnerCloud(out[:m.value].copy())

    def Inliers(self):
        return self._inliers

    def Outliers(self):
        return self._outliers


class Factory(_RecordFilter):
    """filter::Factory.  InitFromXmlText / InitFromXmlNode take the <filters> node; SetInputCloud + Filter run the
    chain on the GPU.  `Filter` returns the InnerCloud of the last filter's records; Inliers() are their indices into
    the input in emission order (ascending unless the chain holds GroundRemoval or VoxelGrid, whose records are a
    voxel's and carry its first member's index) and Outliers() the other input indices, ascending."""
    _abi = "sm_filter_chain"

    def __init__(self, device: int = 0):
        super().__init__(device)
        self.filter_names = []
        self.messages = []

    def InitFromXmlNode(self, filters_node):
        """filter_factory.cc:63-81.  A name the reference does not register is skipped with a message; a <param> with
        an unknown name or without a type of 0 / 1 raises CheckFailure (filter_interface.cc:57), and so does
        GroundRemoval, StatisticRemoval or VoxelGrid unless SetAllFilters(True) was called before."""
        if isinstance(filters_node, (str, bytes)):
            filters_node = ET.fromstring(filters_node)
        for node in filters_node.findall("filter"):
            name = node.attrib.get("name", "")
            index = self._lib.sm_filter_chain_add(self._h, name.encode())
            if index == -10:
                self.messages.append(f"{name} not supported yet.")
                continue
            if index < 0:
                raise CheckFailure(self._error())
            self.filter_names.append(name)
            for param in node.findall("param"):
                rc = self._lib.sm_filter_chain_set_param(self._h, index, param.attrib.get("name", "").encode(),
                                                         _param_type(param.attrib.get("type")),
                                                         (param.text or "").strip().encode())
                if rc != 0:
                    raise CheckFailure(self._error())

    def ConfigsValid(self, index):
        return self._lib.sm_filter_chain_validate(self._h, index) == 1

    def SetSampleSeed(self, seed):
        self._lib.sm_filter_chain_set_option(self._h, b"sample_seed", str(int(seed)).encode())

    def SetRandomSampler(self, filter_index, mode, seed=0):
        """The generator of the chain's RandomSampler `filter_index`, a RandomSamplerMode.  MT19937 draws from
        std::mt19937(seed) anew on every Filter, as the reference does when its random_device returns `seed` (an
        unsigned 32-bit value); HASH ignores `seed`.  A filter that is not a RandomSampler or an unknown mode raises
        ValueError and leaves the chain unchanged.  See sm_filter_chain_set_random_sampler."""
        self._check(self._lib.sm_filter_chain_set_random_sampler(self._h, int(filter_index), int(mode),
                                                                 int(seed) & 0xFFFFFFFF), "set_random_sampler")

    def SetVoxelOrder(self, filter_index, order):
        """The emission order of the chain's VoxelGrid `filter_index`, a VoxelOrder (ASCENDING by default;
        UNORDERED_MAP is the reference's std::unordered_map order).  Each record keeps the scan index of its voxel's
        first member.  A filter that is not a VoxelGrid or an unknown order raises ValueError and leaves the chain
        unchanged.  See sm_filter_chain_set_voxel_order."""
        self._check(self._lib.sm_filter_chain_set_voxel_order(self._h, int(filter_index), int(order)),
                    "set_voxel_order")

    def SetAllFilters(self, flag):
        """True: the filters added from now on may also be GroundRemoval, StatisticRemoval and VoxelGrid, whose chain
        stages are the GPU filters of GroundRemoval, StatisticRemoval and VoxelGridFilter (include/sm_b200.h, the
        all_filters option); False restores the refusal.  Filters already added stay."""
        self._lib.sm_filter_chain_set_option(self._h, b"all_filters", b"1" if flag else b"0")

    def DepthCluster(self, filter_index, cloud):
        """RangeImage::DepthCluster (filter_range_image.cc:143-173) after SetInputCloud(cloud) + Filter on the chain's
        filter `filter_index`, which must be a RangeImage; `cloud` is that filter's own input, (N,5) records.  An empty
        cloud raises CheckFailure (CHECK(inner_cloud_ != nullptr)); a filter that is not a RangeImage or a grid with
        horizontal_line_num < 2 raises ValueError."""
        pts = _records(cloud)
        n = pts.shape[0]
        xyz = np.empty((max(n, 1), 3), np.float32)
        label = np.empty(max(n, 1), np.uint32)
        index = np.empty(max(n, 1), np.int32)
        point_label = np.zeros(max(n, 1), np.uint32)
        m = C.c_int64(0)
        self._check(self._lib.sm_filter_chain_depth_cluster(self._h, int(filter_index), pts.ctypes.data, n, 20,
                                                            xyz.ctypes.data, label.ctypes.data, index.ctypes.data,
                                                            C.byref(m), point_label.ctypes.data), "depth_cluster")
        k = m.value
        return DepthClusters(xyz[:k].copy(), label[:k].copy(), index[:k].copy(), point_label[:n].copy())


class _OwnHandleFilter(_RecordFilter):
    """A filter the chain does not build, on its own handle: configured from its one <filter name=`_name`> node."""
    _name = ""

    def InitFromXmlNode(self, filter_node):
        """A <param> with an unknown name or without a type of 0 / 1 raises CheckFailure (filter_interface.cc:57);
        a node that is not <filter name=`_name`> raises ValueError."""
        if isinstance(filter_node, (str, bytes)):
            filter_node = ET.fromstring(filter_node)
        if filter_node.tag != "filter" or filter_node.attrib.get("name", "") != self._name:
            raise ValueError(f'expected a <filter name="{self._name}"> node')
        for param in filter_node.findall("param"):
            self.SetParam(param.attrib.get("name", ""), param.attrib.get("type"), (param.text or "").strip())

    def SetParam(self, name, ptype, text):
        rc = self._fn("set_param")(self._h, str(name).encode(), _param_type(ptype), str(text).encode())
        if rc != 0:
            raise CheckFailure(self._error())


class StatisticRemoval(_OwnHandleFilter):
    """pre_processers::filter::StatisticRemoval as PCL's StatisticalOutlierRemoval (setMeanK(point_num_meank),
    setStddevMulThresh(std_mul)), the call the reference leaves as a TODO, on the GPU (sm_statistic_removal_*,
    include/sm_b200.h).  InitFromXmlText / InitFromXmlNode take one <filter name="StatisticRemoval"> node and parse its
    <param>s as Factory does; SetInputCloud + Filter run it.  `Filter` returns the kept InnerCloud and raises
    CheckFailure for 1..point_num_meank finite points, ValueError for a point_num_meank outside 1..63; Inliers() /
    Outliers() are indices into the input and Stats() is (mean, stddev, threshold, valid) of the last run."""
    _abi = "sm_statistic_removal"
    _name = "StatisticRemoval"

    def Stats(self):
        """(mean, stddev, threshold, valid) of the last run"""
        s = (C.c_double * 4)()
        self._lib.sm_statistic_removal_stats(self._h, s)
        return tuple(s)


class GroundRemoval(_OwnHandleFilter):
    """pre_processers::filter::GroundRemoval (v1, pre_processors/filter_ground_removal.{h,cc}) on the GPU
    (sm_ground_removal_*, include/sm_b200.h): voxels of leaf_size in the reference's std::map order; a voxel of fewer
    than min_point_num_in_voxel points is skipped, one with z index <= 0 and a z range in [0, height_threshold] is
    ground, every other one is emitted.  InitFromXmlText / InitFromXmlNode take one <filter name="GroundRemoval"> node
    and parse its <param>s as Factory does; SetInputCloud + Filter run it.  `Filter` returns the emitted InnerCloud in
    voxel order; Inliers() / Outliers() are the points of the emitted and of the ground voxels, ascending indices into
    the input (a skipped voxel's points are in neither).  A span of voxel indices past the 63-bit key raises
    ValueError."""
    _abi = "sm_ground_removal"
    _name = "GroundRemoval"

    def Filter(self):
        if self._cloud is None:
            return None
        pts = self._cloud
        n = pts.shape[0]
        out = np.empty_like(pts)
        m = C.c_int64(0)
        self._check(self._fn("run")(self._h, pts.ctypes.data, n, 20, out.ctypes.data, C.byref(m), None), "run")
        inliers, outliers = np.empty(n, np.int32), np.empty(n, np.int32)
        ni, no = C.c_int64(0), C.c_int64(0)
        self._check(self._fn("indices")(self._h, inliers.ctypes.data, C.byref(ni), outliers.ctypes.data, C.byref(no)),
                    "indices")
        self._inliers = inliers[:ni.value].copy()
        self._outliers = outliers[:no.value].copy()
        return InnerCloud(out[:m.value].copy())


class RandomSamplerWithPlaneDetect(_RecordFilter):
    """The submap sampler RandomSamplerWithPlaneDetect (pre_processors/random_sample_with_plane_detect.h) with its
    PlaneDetector on the GPU (sm_plane_sampler_*, include/sm_b200.h): the points of flat low voxels and of voxels whose
    RANSAC plane holds more than 85 % of their points are kept, and the other points are sampled at SetSamplingRate's
    rate in input order.  Configured by its setters (no XML node); SetInputCloud + Filter run it.  `Filter` returns the
    kept InnerCloud in input order; Inliers() / Outliers() are the kept and the dropped input indices and
    PlaneIndices() the plane points, all ascending.  More than 2^24 points, or a span of voxel indices past the 63-bit
    key, raise ValueError."""
    _abi = "sm_plane_sampler"

    def __init__(self, device: int = 0):
        super().__init__(device)
        self._plane = np.zeros(0, np.int32)
        self.messages = []

    def _setter(self, name, value):
        self._check(self._fn(name)(self._h, value), name)
        message = self._error()
        if message:
            self.messages.append(message)

    def SetSamplingRate(self, rate):
        """above 1 -> 1, below 1e-6 -> 1e-6, with the reference's warning in `messages`"""
        self._setter("set_sampling_rate", float(rate))

    def SetLeafSize(self, size):
        self._setter("set_leaf_size", float(size))

    def SetMinPointNumInVoxel(self, num):
        """a size_t: below 5 -> 5, with the reference's warning in `messages`"""
        self._setter("set_min_point_num_in_voxel", int(num) % (1 << 64))

    def Filter(self):
        if self._cloud is None:
            return None
        pts = self._cloud
        n = pts.shape[0]
        out = np.empty_like(pts)
        m = C.c_int64(0)
        self._check(self._fn("run")(self._h, pts.ctypes.data, n, 20, out.ctypes.data, C.byref(m), None), "run")
        inliers, outliers = np.empty(n, np.int32), np.empty(n, np.int32)
        ni, no, npl = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self._fn("indices")(self._h, inliers.ctypes.data, C.byref(ni), outliers.ctypes.data, C.byref(no)),
                    "indices")
        plane = np.empty(n, np.int32)
        self._check(self._fn("plane_indices")(self._h, plane.ctypes.data, C.byref(npl)), "plane_indices")
        self._inliers = inliers[:ni.value].copy()
        self._outliers = outliers[:no.value].copy()
        self._plane = plane[:npl.value].copy()
        return InnerCloud(out[:m.value].copy())

    def PlaneIndices(self):
        return self._plane
