"""quatro_b200 -- H100-native global-registration hot path (drop-in for url-kaist/Quatro's
voxel-FPFH -> match -> TIM graph -> max clique -> GNC-TLS yaw + COTE path).

The product is the C-ABI shared library (include/quatro_b200.h, built from quatro_b200/csrc/*.cu
for sm_90a).  This package only carries the ctypes binding used by tests/bench, the build helper
and the synthetic-scan generator.  There is no CPU fallback anywhere in this package.
"""
from .capi import (  # noqa: F401
    Params, Config, Result, Pair, Handle, QuatroB200Error, default_params, default_config, load_library,
    PMC_EXACT, PMC_HEU, KCORE_HEU, INLIER_NONE, COTE_MEDIAN, COTE_WEIGHTED_MEAN, MEM_HOST, MEM_DEVICE,
    PairLists, ListBuffers, FLAG_LISTS_TRUNCATED, FeaturePair, DescriptorPair, FeatureOut, POINT_ARRAYS, VOXEL_ARRAYS, MATCH_LISTS,
)

__all__ = ["Params", "Config", "Result", "Pair", "Handle", "QuatroB200Error", "default_params",
           "default_config", "load_library", "PairLists", "ListBuffers", "FeaturePair", "DescriptorPair", "FeatureOut",
           "POINT_ARRAYS", "VOXEL_ARRAYS", "MATCH_LISTS"]
