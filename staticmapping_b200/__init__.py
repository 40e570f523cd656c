"""staticmapping_b200 — H100-native scan matching behind StaticMapping's
registrator::Interface.  The compute lives in libsm_b200.so (hand-written sm_90a CUDA,
C ABI in include/sm_b200.h); this package is the thin host-side mirror used by the tests
and the bench.  There is no CPU fallback."""
from .registrators import (AlignBatch, AlignPairs, CalculateNormals, CheckFailure, CreateMatcher, EigenCloud, ErrorMinimizer, IcpFast, IcpUsingPointMatcher, InnerCloud,  # noqa: F401
                           Interface, M2dp, MatcherOptions, matchTwoM2dpDescriptors, MotionCompensation, AverageTransforms, Ndt, NdtWithGicp, NeighborSearchMethod, ReadingSampler, SurfaceNormals, Type, VoxelGridFilter, knn, knn1)
from .filters import Factory, GroundRemoval, RandomSamplerWithPlaneDetect, StatisticRemoval  # noqa: F401

__all__ = ["AlignBatch", "AlignPairs", "CalculateNormals", "CheckFailure", "CreateMatcher", "EigenCloud", "ErrorMinimizer", "Factory", "GroundRemoval", "IcpFast", "IcpUsingPointMatcher", "InnerCloud", "Interface", "M2dp", "matchTwoM2dpDescriptors", "Ndt", "NdtWithGicp", "NeighborSearchMethod", "RandomSamplerWithPlaneDetect", "StatisticRemoval",
           "MatcherOptions", "MotionCompensation", "AverageTransforms", "ReadingSampler", "SurfaceNormals", "Type", "VoxelGridFilter", "knn", "knn1"]
