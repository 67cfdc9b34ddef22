"""fast_slic_b200 -- H100-native (sm_90a) SLIC superpixels behind the fast_slic Python surface.

Mirrors fast-slic/fast_slic/__init__.py:1-4 (``from .base_slic import *``, ``supported_archs``).
"""
from .base_slic import (ARCH_NAME, LSC, BaseSlic, NodeConnectivity, Slic, SlicCuda, SlicModel, SlicRealDist, SlicRealDistL2,
                        SlicRealDistNoQ, clear_engine_cache, enforce_connectivity,
                        get_cca_engine, get_engine, get_supported_archs, is_supported_arch)
from .crf import SimpleCRF, SimpleCRFFrame
from .engine import CLUSTER_DTYPE, Engine
from .stream import SlicStream

supported_archs = tuple(get_supported_archs())
__all__ = ["ARCH_NAME", "BaseSlic", "Slic", "SlicCuda", "SlicModel", "Engine", "CLUSTER_DTYPE",
           "enforce_connectivity", "get_supported_archs", "is_supported_arch", "supported_archs", "get_engine",
           "clear_engine_cache", "SlicStream", "get_cca_engine", "NodeConnectivity", "SlicRealDist", "SlicRealDistL2", "SlicRealDistNoQ", "LSC",
           "SimpleCRF", "SimpleCRFFrame"]
