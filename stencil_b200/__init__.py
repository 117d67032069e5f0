"""stencil_b200 -- H100-native halo exchange + jacobi hot path behind the cwpearson/stencil API.

The compute lives in hand-written sm_90a CUDA (stencil_b200/csrc) behind a C ABI
(include/stencil_b200.h); this package is the Python host mirror of the reference's domain API.
"""
from ._lib import LIB_PATH, StencilError, lib  # noqa: F401
from .domain import (  # noqa: F401
    ALL_DIRS,
    CopyPlan,
    DataHandle,
    DistributedDomain,
    LocalDomain,
    Method,
    Partition,
    PlacementStrategy,
    Radius,
    box_copy,
    fill,
    get_neighbor,
    halo_extent,
    halo_pos,
    jacobi3d,
    prime_factors,
    raw_size,
)

__all__ = [n for n in dir() if not n.startswith("_")]
