"""stencil_b200 -- H100-native halo exchange + jacobi hot path behind the cwpearson/stencil API.

The compute lives in hand-written sm_90a CUDA (stencil_b200/csrc) behind a C ABI
(include/stencil_b200.h); this package is the Python host mirror of the reference's domain API.
"""
from ._lib import LIB_PATH, StencilError, lib  # noqa: F401
from .domain import (  # noqa: F401
    ALL_DIRS,
    BC,
    BCKind,
    BCPlan,
    Boundary,
    CopyPlan,
    FACES,
    Topology,
    bc_regions,
    DataHandle,
    DistributedDomain,
    ExactReducePlan,
    KrylovPlan,
    LocalDomain,
    Method,
    Partition,
    PlacementStrategy,
    Radius,
    Reduction,
    ReducePlan,
    TransferPlan,
    box_copy,
    fill,
    get_neighbor,
    halo_extent,
    halo_pos,
    jacobi3d,
    prime_factors,
    raw_size,
    reduce_combine,
    reduce_exact_combine,
    reduce_exact_round,
    transfer_check,
)
from .stencil_op import StencilOp, StencilPlan, StencilSystem, SystemPlan  # noqa: F401
from .multigrid import Multigrid  # noqa: F401
from .krylov import PCG  # noqa: F401
from .bicgstab import BiCGStab  # noqa: F401

__all__ = [n for n in dir() if not n.startswith("_")]
