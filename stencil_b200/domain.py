"""Host-side mirror of the reference's domain API for the halo-exchange path, over the C ABI.

Names and argument meaning follow cwpearson/stencil (include/stencil/stencil.hpp:33-225,
local_domain.cuh:34-276, radius.hpp, method.hpp) so that tests read like the reference's own:

    dd = DistributedDomain(512, 512, 512)
    dd.set_radius(Radius.face_edge_corner(1, 0, 0))
    h = dd.add_data(np.float64, "d")
    dd.realize()
    dd.exchange(); dd.swap()

Two deployment modes, one code path:
  * one process driving several GPUs (the reference's 1 rank x N GPUs, src/stencil.cu:74-85):
    peer access is enabled all-pairs and each source GPU runs ONE fused kernel that writes every
    outgoing halo straight into the neighbours' ghost cells;
  * one process per GPU under torch.distributed (torchrun): allocations and completion flags are
    shared through CUDA IPC handles exchanged with all_gather_object; the same fused kernel writes
    through the IPC mappings over NVLink, ordered by device-side ready/done flags (no host barrier
    in the exchange).

All arithmetic on coordinates is delegated to the C ABI (sb_halo_pos, sb_node_partition,
sb_exchange_messages, sb_staging_layout, ...); this module only sequences calls.  No CPU fallback exists.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum
import math
import itertools
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import BoxCopy, I27, Pitched, check, i3, lib, o3, stream_ptr, t3

Vec = Tuple[int, int, int]

ALL_DIRS: List[Vec] = [
    (x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)
]


class Method(enum.IntFlag):
    """include/stencil/method.hpp:5-16.  On one NVSwitch node every message takes the fused
    direct-write path; the flags are kept so reference call sites (set_methods) keep working and
    so exchange_bytes_for_method can attribute bytes the way the reference does."""

    NONE = 0
    CudaMpi = 1
    ColoPackMemcpyUnpack = 2
    ColoQuantityKernel = 4
    ColoRegionKernel = 8
    ColoMemcpy3d = 16
    ColoDomainKernel = 32
    CudaMemcpyPeer = 64
    CudaKernel = 128
    Default = 1 + 2 + 64 + 128


class PlacementStrategy(enum.Enum):
    NodeAware = 0
    Trivial = 1
    IntraNodeRandom = 2


class Radius:
    """include/stencil/radius.hpp -- 27 radii; x(d)/y(d)/z(d) read the face entries."""

    def __init__(self):
        self._r: Dict[Vec, int] = {(x, y, z): 0 for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)}

    @staticmethod
    def constant(r: int) -> "Radius":
        out = Radius()
        for k in out._r:
            out._r[k] = int(r)
        return out

    @staticmethod
    def face_edge_corner(face: int, edge: int, corner: int) -> "Radius":
        out = Radius()
        for d in out._r:
            out._r[d] = (0, face, edge, corner)[sum(1 for c in d if c)]
        return out

    def dir(self, x, y=None, z=None) -> int:
        d = tuple(x) if y is None else (x, y, z)
        return self._r[d]

    def set_dir(self, d: Vec, v: int) -> None:
        self._r[tuple(d)] = int(v)

    def x(self, d: int) -> int:
        return self._r[(d, 0, 0)]

    def y(self, d: int) -> int:
        return self._r[(0, d, 0)]

    def z(self, d: int) -> int:
        return self._r[(0, 0, d)]

    def set_face(self, r: int) -> None:
        for d in self._r:
            if sum(1 for c in d if c) == 1:
                self._r[d] = int(r)

    def set_edge(self, r: int) -> None:
        for d in self._r:
            if sum(1 for c in d if c) == 2:
                self._r[d] = int(r)

    def set_corner(self, r: int) -> None:
        for d in self._r:
            if sum(1 for c in d if c) == 3:
                self._r[d] = int(r)

    def c27(self) -> I27:
        return I27(*[self._r[(x, y, z)] for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)])

    def __eq__(self, o) -> bool:
        return isinstance(o, Radius) and self._r == o._r


class DataHandle:
    """DataHandle<T>, local_domain.cuh:18-26"""

    def __init__(self, idx: int, dtype, name: str = ""):
        self.id = idx
        self.dtype = np.dtype(dtype)
        self.name = name


# ------------------------------------------------------------------------------------------ geometry (C ABI)
def halo_pos(d: Vec, sz: Vec, radius: Radius, halo: bool) -> Vec:
    out = o3()
    check(lib().sb_halo_pos(i3(d), i3(sz), radius.c27(), int(bool(halo)), out))
    return t3(out)


def halo_extent(d: Vec, sz: Vec, radius: Radius) -> Vec:
    out = o3()
    check(lib().sb_halo_extent(i3(d), i3(sz), radius.c27(), out))
    return t3(out)


def raw_size(sz: Vec, radius: Radius) -> Vec:
    out = o3()
    check(lib().sb_raw_size(i3(sz), radius.c27(), out))
    return t3(out)


def prime_factors(n: int) -> List[int]:
    buf = (C.c_int64 * 64)()
    k = check(lib().sb_prime_factors(int(n), buf, 64))
    return [int(buf[i]) for i in range(k)]


class Partition:
    """NodePartition (default) or RankPartition ("trivial") through the C ABI."""

    def __init__(self, size: Vec, radius: Radius, n_nodes: int, gpus_per_node: int, trivial: bool = False):
        dim, base, rem = o3(), o3(), o3()
        if trivial:
            check(lib().sb_rank_partition(i3(size), n_nodes * gpus_per_node, dim, base, rem))
            self.sys_dim, self.node_dim = (1, 1, 1), t3(dim)
        else:
            sysd, noded = o3(), o3()
            check(lib().sb_node_partition(i3(size), radius.c27(), n_nodes, gpus_per_node, sysd, noded, base, rem))
            self.sys_dim, self.node_dim = t3(sysd), t3(noded)
        self.dim = tuple(self.sys_dim[a] * self.node_dim[a] for a in range(3))
        self._base, self._rem = base, rem

    def subdomain_size(self, idx: Vec) -> Vec:
        out = o3()
        check(lib().sb_subdomain_size(self._base, self._rem, i3(idx), out))
        return t3(out)

    def subdomain_origin(self, idx: Vec) -> Vec:
        out = o3()
        check(lib().sb_subdomain_origin(self._base, self._rem, i3(idx), out))
        return t3(out)

    def indices(self) -> List[Vec]:
        d = self.dim
        return [(x, y, z) for z in range(d[2]) for y in range(d[1]) for x in range(d[0])]


def get_neighbor(idx: Vec, d: Vec, dim: Vec) -> Vec:
    """Topology::get_neighbor with periodic boundaries (src/topology.cpp:5-18)."""
    return tuple((idx[a] + d[a]) % dim[a] for a in range(3))


# ------------------------------------------------------------------------------------------ topology and boundaries
class Boundary(enum.Enum):
    """How the grid closes along one axis (include/stencil/topology.hpp): PERIODIC wraps around, FIXED ends at a wall."""

    PERIODIC = 1
    FIXED = 2


class Topology:
    """The grid of subdomains with one Boundary per axis (include/stencil/topology.hpp)."""

    def __init__(self, dim: Vec, boundaries: Sequence[Boundary] = (Boundary.PERIODIC,) * 3):
        self.dim = tuple(int(v) for v in dim)
        self.boundaries = tuple(boundaries)

    def get_neighbor(self, idx: Vec, d: Vec) -> Optional[Vec]:
        """The subdomain one step in direction d from idx; None when the step leaves the grid along a FIXED axis."""
        out = []
        for a in range(3):
            v = idx[a] + d[a]
            if self.boundaries[a] == Boundary.PERIODIC:
                v %= self.dim[a]
            elif not 0 <= v < self.dim[a]:
                return None
            out.append(v)
        return tuple(out)

    def is_wall(self, idx: Vec, face: int) -> bool:
        """Is face `face` (0..5 = -x, +x, -y, +y, -z, +z) of subdomain idx a wall face (its step has no neighbour)?"""
        d = [0, 0, 0]
        d[face // 2] = 1 if face % 2 else -1
        return self.get_neighbor(idx, tuple(d)) is None


def grid_args(part: Partition, topology: Topology, radius: Radius) -> tuple:
    """The (dim, base, rem, boundary, radius27) arguments of sb_exchange_messages and sb_staging_layout."""
    return i3(part.dim), part._base, part._rem, (C.c_int32 * 3)(*[b.value for b in topology.boundaries]), radius.c27()


def exchange_messages(part: Partition, topology: Topology, radius: Radius, src_idx: Vec) -> List[dict]:
    """sb_exchange_messages: every message subdomain src_idx sends, in direction order z, y, x ascending.
    dict(src_idx, dst_idx, dir, src_pos, dst_pos, ext)."""
    out = (_lib.Message * 26)()
    n = check(lib().sb_exchange_messages(*grid_args(part, topology, radius), i3(src_idx), out, 26))
    return [
        dict(src_idx=tuple(src_idx), dst_idx=t3(m.dst_idx), dir=t3(m.dir), src_pos=t3(m.src_pos), dst_pos=t3(m.dst_pos), ext=t3(m.extent))
        for m in out[:n]
    ]


def quantity_mask(qs) -> int:
    """The quantity set of sb_staging_layout_subset: bit q for each quantity q of qs (a sorted tuple), every bit for None
    (all quantities)."""
    return (1 << 64) - 1 if qs is None else sum(1 << q for q in qs)


def op_moved_coefs(op, coef_qs: Sequence[int]) -> List[int]:
    """The coefficient quantities (coef_qs[k] is field k) that a term of op reads at a non-zero coefficient offset: with
    the src, what exchange="reads" moves."""
    return [coef_qs[k] for k in sorted({t[3] for t in op.terms if len(t) == 5 and any(t[4])})]


class BCKind(enum.IntEnum):
    """sb_bc_kind"""

    NONE = 0
    VALUE = 1
    EVEN = 2
    ODD = 3


FACES: List[Vec] = [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]  # face numbering 0..5


def face_index(face: Vec) -> int:
    face = tuple(int(v) for v in face)
    if face not in FACES:
        raise _lib.StencilError(f"{face} is not a face direction (one component +-1, the others 0)")
    return FACES.index(face)


class BC:
    """A boundary condition of one quantity on one wall face (include/stencil/boundary_condition.hpp):
    BC.NONE() (ghost cells untouched), BC.VALUE(c) (ghost = c), BC.EVEN() (mirror image), BC.ODD(c=0) (2c - mirror
    image; c is the value at the face).  The mirror and the order in which walls compose are those of sb_bc_regions."""

    def __init__(self, kind: BCKind = BCKind.NONE, value: float = 0.0):
        self.kind = BCKind(kind)
        self.value = float(value)

    @staticmethod
    def NONE() -> "BC":
        return BC(BCKind.NONE)

    @staticmethod
    def VALUE(c: float) -> "BC":
        return BC(BCKind.VALUE, c)

    @staticmethod
    def EVEN() -> "BC":
        return BC(BCKind.EVEN)

    @staticmethod
    def ODD(c: float = 0.0) -> "BC":
        return BC(BCKind.ODD, c)

    def __eq__(self, o) -> bool:
        return isinstance(o, BC) and (self.kind, self.value) == (o.kind, o.value)

    def __repr__(self) -> str:
        return f"BC({self.kind.name}, {self.value})"


def bc_dtype(dtype) -> int:
    """sb_dtype of a numpy dtype: float32 / float64 carry arithmetic, anything else is copied as raw bytes."""
    dt = np.dtype(dtype)
    if dt == np.float32:
        return 1
    if dt == np.float64:
        return 2
    return 0


def bc_regions(size: Vec, radius: Radius, kinds: Sequence[int]) -> List[dict]:
    """sb_bc_regions: the ghost boxes a subdomain's boundary conditions write (pure geometry, host only).
    dict(dir, pos, ext, mirror, faces): source coordinate = mirror[a] - p[a] on wall axes (mirror[a] >= 0), else p[a]."""
    buf = (_lib.BcRegion * 26)()
    n = check(lib().sb_bc_regions(i3(size), radius.c27(), _lib.I6(*[int(k) for k in kinds]), buf, 26))
    return [
        dict(dir=t3(r.dir), pos=t3(r.pos), ext=t3(r.extent), mirror=t3(r.mirror), faces=int(r.faces)) for r in buf[:n]
    ]


class BCPlan:
    """sb_bc_plan: every boundary-condition region of every quantity of one subdomain, one launch."""

    def __init__(self, device: int, quantities: Sequence[_lib.BcQuantity], size: Vec, radius: Radius):
        arr = (_lib.BcQuantity * max(1, len(quantities)))(*quantities)
        h = C.c_void_p()
        check(lib().sb_bc_plan_create(C.byref(h), device, arr, len(quantities), i3(size), radius.c27()))
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_bc_plan_bytes(h))

    def launch(self, stream=None) -> None:
        check(lib().sb_bc_plan_launch(self._h, stream_ptr(stream)))

    def destroy(self) -> None:
        if self._h:
            lib().sb_bc_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------ multigrid transfers
def transfer_check(fine_dim: Vec, coarse_dim: Vec, fine_origins: Sequence[Vec], fine_sizes: Sequence[Vec], coarse_origins: Sequence[Vec],
                   coarse_sizes: Sequence[Vec], coarse_radius: Optional[Radius] = None) -> None:
    """sb_transfer_check: whether a fine and a coarse partition pair for transfers (pure geometry, host only).  Per
    subdomain index in partition order (x fastest): origins and sizes.  coarse_radius=None checks restriction only;
    with a radius, prolongation's one ghost layer in all 26 directions as well.  Raises StencilError."""

    def arr(vs):
        return (C.c_int64 * (3 * max(1, len(vs))))(*[int(v) for t in vs for v in t])

    r = coarse_radius.c27() if coarse_radius is not None else None
    check(lib().sb_transfer_check(i3(fine_dim), i3(coarse_dim), arr(fine_origins), arr(fine_sizes), arr(coarse_origins), arr(coarse_sizes), r))


class TransferPlan:
    """sb_transfer_plan: one restriction (kind 0; dst coarse, src fine) or prolongation (kind 1; dst fine, src coarse,
    optional aux with dst's layout) over the box [lo, hi) of dst (global coordinates); one launch."""

    def __init__(self, device: int, dtype, kind: int, dst: Pitched, dst_origin: Vec, dst_zsize: int, src: Pitched, src_origin: Vec,
                 src_zsize: int, aux: Optional[Pitched], lo: Vec, hi: Vec):
        h = C.c_void_p()
        check(lib().sb_transfer_plan_create(C.byref(h), device, bc_dtype(dtype), int(kind), dst, i3(dst_origin), int(dst_zsize), src,
                                            i3(src_origin), int(src_zsize), aux if aux is not None else Pitched(None, 0, 0), i3(lo), i3(hi)))
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_transfer_plan_bytes(h))

    @classmethod
    def fused(cls, device: int, op, dst: Pitched, dst_origin: Vec, dst_zsize: int, src: Pitched, src_origin: Vec, src_zsize: int,
              aux: Optional[Pitched], boxes: Sequence[Tuple[Vec, Vec]], coefs: Optional[Sequence[Pitched]] = None) -> "TransferPlan":
        """sb_transfer_oplan_create: the fused residual-restriction, dst (coarse) = the restriction of op(src, aux) (fine;
        aux shares src's layout) over the coarse boxes [lo, hi) (global coordinates); op is a StencilOp of reach <= 1.
        An op with coefficient terms takes coefs, its fine coefficient allocations (sb_transfer_voplan_create)."""
        nb = len(boxes)
        lo = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[0]])
        hi = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[1]])
        h = C.c_void_p()
        a = aux if aux is not None else Pitched(None, 0, 0)
        if op.has_coef:
            cs = list(coefs or [])
            carr = (Pitched * max(1, len(cs)))(*cs)
            check(lib().sb_transfer_voplan_create(C.byref(h), device, op.dtype_code, op.c_vterms(), len(op.terms), dst, i3(dst_origin),
                                                  int(dst_zsize), src, i3(src_origin), int(src_zsize), a, carr, len(cs), nb, lo, hi))
        else:
            check(lib().sb_transfer_oplan_create(C.byref(h), device, op.dtype_code, op.c_terms(), len(op.terms), dst, i3(dst_origin),
                                                 int(dst_zsize), src, i3(src_origin), int(src_zsize), a, nb, lo, hi))
        return cls._wrap(h, device)

    @classmethod
    def face(cls, device: int, dtype, axis: int, dst: Pitched, dst_origin: Vec, dst_zsize: int, src: Pitched, src_origin: Vec, src_zsize: int,
             lo: Vec, hi: Vec) -> "TransferPlan":
        """sb_transfer_fplan_create: dst (coarse) = the face-coefficient restriction of src (fine), faces normal to axis,
        over the coarse box [lo, hi)."""
        h = C.c_void_p()
        check(lib().sb_transfer_fplan_create(C.byref(h), device, bc_dtype(dtype), int(axis), dst, i3(dst_origin), int(dst_zsize), src,
                                             i3(src_origin), int(src_zsize), i3(lo), i3(hi)))
        return cls._wrap(h, device)

    @classmethod
    def _wrap(cls, h, device: int) -> "TransferPlan":
        self = cls.__new__(cls)
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_transfer_plan_bytes(h))
        return self

    def launch(self, stream=None) -> None:
        check(lib().sb_transfer_plan_launch(self._h, stream_ptr(stream)))

    def destroy(self) -> None:
        if self._h:
            lib().sb_transfer_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------ reductions
@dataclasses.dataclass(frozen=True)
class Reduction:
    """sb_reduce_result: min and max of the per-cell value v, sum of v, sum of its squared term q, number of cells."""

    min: float
    max: float
    sum: float
    sumsq: float
    count: int

    def mean(self) -> float:
        return self.sum / self.count if self.count else math.nan

    def rms(self) -> float:
        """sqrt(sumsq / count): the RMS of a scalar, or of |u| for a NORM3 item."""
        return math.sqrt(self.sumsq / self.count) if self.count else math.nan

    def l2(self) -> float:
        """sqrt(sumsq): the 2-norm (of a - b for a DIFF item)."""
        return math.sqrt(self.sumsq)

    @staticmethod
    def of(r: _lib.ReduceResult) -> "Reduction":
        return Reduction(r.min, r.max, r.sum, r.sumsq, int(r.count))

    def to_c(self) -> _lib.ReduceResult:
        return _lib.ReduceResult(self.min, self.max, self.sum, self.sumsq, self.count)


def reduce_combine(parts: Sequence[Reduction]) -> Reduction:
    """sb_reduce_combine: per-subdomain results merged by the library's fixed pairwise tree, in the order given."""
    arr = (_lib.ReduceResult * max(1, len(parts)))(*[p.to_c() for p in parts])
    out = _lib.ReduceResult()
    check(lib().sb_reduce_combine(arr, len(parts), C.byref(out)))
    return Reduction.of(out)


class ReducePlan:
    """sb_reduce_plan: several reductions of one subdomain, one launch sequence, results into a device buffer the plan
    owns.  One launch in flight at a time."""

    def __init__(self, device: int, items: Sequence[_lib.ReduceItem]):
        arr = (_lib.ReduceItem * len(items))(*items)
        h = C.c_void_p()
        check(lib().sb_reduce_plan_create(C.byref(h), device, arr, len(items)))
        self._h = h
        self.device = device
        self.n = len(items)
        self.bytes = int(lib().sb_reduce_plan_bytes(h))
        out = C.c_void_p()
        nbytes = self.n * C.sizeof(_lib.ReduceResult)
        if lib().sb_malloc(C.byref(out), nbytes, device) != 0:
            self.destroy()
            raise _lib.StencilError(f"reduction output buffer: {lib().sb_last_error().decode()}")
        self.out_dev = out.value

    def launch(self, stream=None) -> None:
        check(lib().sb_reduce_plan_launch(self._h, C.c_void_p(self.out_dev), stream_ptr(stream)))

    def results(self, stream=None) -> List[Reduction]:
        """Copy the last launch's results (ordered after it on `stream`) to the host."""
        host = (_lib.ReduceResult * self.n)()
        check(lib().sb_memcpy(C.addressof(host), C.c_void_p(self.out_dev), C.sizeof(host), self.device, stream_ptr(stream)))
        check(lib().sb_stream_sync(self.device, stream_ptr(stream)))
        return [Reduction.of(r) for r in host]

    def destroy(self) -> None:
        if getattr(self, "out_dev", None):
            lib().sb_free(C.c_void_p(self.out_dev), self.device)
            self.out_dev = None
        if self._h:
            lib().sb_reduce_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def reduce_exact_combine(parts: Sequence[_lib.ReduceExactPart]) -> _lib.ReduceExactPart:
    """sb_reduce_exact_combine: parts (e.g. one per subdomain) merged; the result does not depend on their order."""
    arr = (_lib.ReduceExactPart * max(1, len(parts)))(*parts)
    out = _lib.ReduceExactPart()
    check(lib().sb_reduce_exact_combine(arr, len(parts), C.byref(out)))
    return out


def reduce_exact_round(part: _lib.ReduceExactPart) -> Reduction:
    """sb_reduce_exact_round: min, max and count as they are, sum and sumsq correctly rounded."""
    out = _lib.ReduceResult()
    check(lib().sb_reduce_exact_round(C.byref(part), C.byref(out)))
    return Reduction.of(out)


class ExactReducePlan:
    """sb_reduce_exact_plan: the items of a ReducePlan with exact sums; results are sb_reduce_exact_parts, to be
    combined across subdomains and then rounded.  One launch in flight at a time."""

    def __init__(self, device: int, items: Sequence[_lib.ReduceItem]):
        arr = (_lib.ReduceItem * len(items))(*items)
        h = C.c_void_p()
        check(lib().sb_reduce_exact_plan_create(C.byref(h), device, arr, len(items)))
        self._h = h
        self.device = device
        self.n = len(items)
        self.bytes = int(lib().sb_reduce_exact_plan_bytes(h))
        out = C.c_void_p()
        nbytes = self.n * C.sizeof(_lib.ReduceExactPart)
        if lib().sb_malloc(C.byref(out), nbytes, device) != 0:
            self.destroy()
            raise _lib.StencilError(f"reduction output buffer: {lib().sb_last_error().decode()}")
        self.out_dev = out.value

    def launch(self, stream=None) -> None:
        check(lib().sb_reduce_exact_plan_launch(self._h, C.c_void_p(self.out_dev), stream_ptr(stream)))

    def parts(self, stream=None) -> List[_lib.ReduceExactPart]:
        """Copy the last launch's parts (ordered after it on `stream`) to the host."""
        host = (_lib.ReduceExactPart * self.n)()
        check(lib().sb_memcpy(C.addressof(host), C.c_void_p(self.out_dev), C.sizeof(host), self.device, stream_ptr(stream)))
        check(lib().sb_stream_sync(self.device, stream_ptr(stream)))
        return list(host)

    def results(self, stream=None) -> List[Reduction]:
        """The last launch's parts, each rounded: the whole result when the plan covers the whole region."""
        return [reduce_exact_round(p) for p in self.parts(stream)]

    def destroy(self) -> None:
        if getattr(self, "out_dev", None):
            lib().sb_free(C.c_void_p(self.out_dev), self.device)
            self.out_dev = None
        if self._h:
            lib().sb_reduce_exact_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class KrylovPlan:
    """sb_krylov_plan: one Krylov vector pass (KRYLOV_DOT, KRYLOV_XPBY, KRYLOV_UPDATE or KRYLOV_BICG_P) over one box,
    with its parts (sb_reduce_exact_part, one per dot) written to a device buffer the plan owns.  One launch in flight at
    a time."""

    def __init__(self, device: int, mode: int, dtype, bufs: Sequence[Pitched], acc_origin: Vec, lo: Vec, hi: Vec):
        arr = (Pitched * max(1, len(bufs)))(*bufs)
        h = C.c_void_p()
        check(lib().sb_krylov_plan_create(C.byref(h), device, int(mode), bc_dtype(dtype), arr, len(bufs), i3(acc_origin), i3(lo), i3(hi)))
        self._h = h
        self.device = device
        self.n = len(bufs) - 1 if mode == _lib.KRYLOV_DOT else len(bufs) - 3 if mode == _lib.KRYLOV_UPDATE else 0
        self.bytes = int(lib().sb_krylov_plan_bytes(h))
        self.out_dev = None
        if self.n:
            out = C.c_void_p()
            if lib().sb_malloc(C.byref(out), self.n * C.sizeof(_lib.ReduceExactPart), device) != 0:
                self.destroy()
                raise _lib.StencilError(f"krylov parts buffer: {lib().sb_last_error().decode()}")
            self.out_dev = out.value
        self.s = 0.0  # the scalar of the next launch
        self.t = 0.0  # the second scalar of the next launch (KRYLOV_BICG_P's omega; the other modes ignore it)

    def launch(self, stream=None, s: Optional[float] = None, t: Optional[float] = None) -> None:
        """Queue the pass on `stream` with the scalars s and t (default: the attributes s and t, so a plan runs where a
        schedule calls launch(stream) alone)."""
        s = self.s if s is None else s
        t = self.t if t is None else t
        check(lib().sb_krylov_plan_launch2(self._h, C.c_double(float(s)), C.c_double(float(t)), C.c_void_p(self.out_dev or 0), stream_ptr(stream)))

    def parts(self, stream=None) -> List[_lib.ReduceExactPart]:
        """Copy the last launch's parts (ordered after it on `stream`) to the host."""
        host = (_lib.ReduceExactPart * max(1, self.n))()
        if self.n:
            check(lib().sb_memcpy(C.addressof(host), C.c_void_p(self.out_dev), C.sizeof(host), self.device, stream_ptr(stream)))
        check(lib().sb_stream_sync(self.device, stream_ptr(stream)))
        return list(host)[: self.n]

    def destroy(self) -> None:
        if getattr(self, "out_dev", None):
            lib().sb_free(C.c_void_p(self.out_dev), self.device)
            self.out_dev = None
        if getattr(self, "_h", None):
            lib().sb_krylov_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class _Clear:
    """A one-launch plan that sets a quantity's whole curr allocation to +0 (ghost cells included; an exchange refills
    them before any read)."""

    def __init__(self, d, q: int):
        raw = d.raw_size()
        self.gpu, self.ptr, self.nbytes = d.gpu(), d.curr_[q], raw[0] * raw[1] * raw[2] * d.elem_size(q)

    def launch(self, stream=None) -> None:
        check(lib().sb_memset(C.c_void_p(self.ptr), 0, self.nbytes, self.gpu, stream_ptr(stream)))


# ------------------------------------------------------------------------------------------ LocalDomain
class LocalDomain:
    """One subdomain on one GPU: curr/next allocation per quantity (local_domain.cuh:34-276,
    src/local_domain.cu).  Rows are unpitched (pitch == raw_x * elem_size) exactly like the
    reference, because astaroth-style kernels index i + j*mx + k*mx*my."""

    def __init__(self, sz: Vec, origin: Vec, dev: int):
        self.sz_ = tuple(int(v) for v in sz)
        self.origin_ = tuple(int(v) for v in origin)
        self.dev_ = int(dev)
        self.radius_ = Radius.constant(0)
        self.elem_sizes_: List[int] = []
        self.dtypes_: List[np.dtype] = []
        self.names_: List[str] = []
        self.curr_: List[int] = []  # device addresses
        self.next_: List[int] = []
        self._owned = False

    # -- configuration
    def set_radius(self, r) -> None:
        self.radius_ = r if isinstance(r, Radius) else Radius.constant(int(r))

    def add_data(self, dtype, name: str = "") -> DataHandle:
        dt = np.dtype(dtype)
        self.dtypes_.append(dt)
        self.elem_sizes_.append(dt.itemsize)
        self.names_.append(name)
        return DataHandle(len(self.dtypes_) - 1, dt, name)

    def lead_bytes(self, es: int) -> int:
        """HBM layout rule (DESIGN.md section 1): when every row has the same 16-byte phase (pitch % 16 == 0) the
        allocation starts `lead` bytes into its cudaMalloc block so that the first COMPUTE cell of every row is 16-byte
        aligned -- 512 FP64 cells are then exactly 256 aligned vectors (8 warp strips) and the halo rows of the y / z
        faces are 128-bit copyable.  The reference starts at the block (src/local_domain.cu:187-203); the layout inside
        the allocation (x fastest, unpitched) is unchanged.  SB_ALLOC_ALIGN=0 restores the reference placement."""
        import os

        if os.environ.get("SB_ALLOC_ALIGN", "1") == "0":
            return 0
        raw = self.raw_size()
        if (raw[0] * es) % 16 != 0:
            return 0
        return (16 - (self.radius_.x(-1) * es) % 16) % 16

    def realize(self) -> None:
        raw = self.raw_size()
        self._base_of = {}  # pointer handed out -> cudaMalloc block (for free and CUDA IPC)
        for es in self.elem_sizes_:
            nbytes = raw[0] * raw[1] * raw[2] * es
            lead = self.lead_bytes(es)
            for store in (self.curr_, self.next_):
                p = C.c_void_p()
                check(lib().sb_malloc(C.byref(p), nbytes + 32, self.dev_))
                check(lib().sb_memset(p, 0, nbytes + 32, self.dev_, None))
                store.append(int(p.value) + lead)
                self._base_of[int(p.value) + lead] = int(p.value)
        check(lib().sb_device_sync(self.dev_))
        self._owned = True

    def free(self) -> None:
        if self._owned:
            for p in self.curr_ + self.next_:
                lib().sb_free(C.c_void_p(self._base_of.get(p, p)), self.dev_)
            self.curr_, self.next_, self._owned = [], [], False

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    # -- queries
    def gpu(self) -> int:
        return self.dev_

    def size(self) -> Vec:
        return self.sz_

    def origin(self) -> Vec:
        return self.origin_

    def radius(self) -> Radius:
        return self.radius_

    def num_data(self) -> int:
        return len(self.elem_sizes_)

    def elem_size(self, q: int) -> int:
        return self.elem_sizes_[q]

    def raw_size(self) -> Vec:
        return raw_size(self.sz_, self.radius_)

    def halo_pos(self, d: Vec, halo: bool) -> Vec:
        return halo_pos(d, self.sz_, self.radius_, halo)

    def halo_extent(self, d: Vec) -> Vec:
        return halo_extent(d, self.sz_, self.radius_)

    def halo_bytes(self, d: Vec, q: int) -> int:
        e = self.halo_extent(d)
        return self.elem_sizes_[q] * e[0] * e[1] * e[2]

    def get_compute_region(self) -> Tuple[Vec, Vec]:
        return self.origin_, tuple(self.origin_[a] + self.sz_[a] for a in range(3))

    def accessor_origin(self) -> Vec:
        """Accessor origin: subdomain origin minus the negative-side radius (local_domain.cuh:153-173)."""
        r = self.radius_
        return (self.origin_[0] - r.x(-1), self.origin_[1] - r.y(-1), self.origin_[2] - r.z(-1))

    def pitched(self, q: int, which: str = "curr") -> Pitched:
        raw = self.raw_size()
        ptr = (self.curr_ if which == "curr" else self.next_)[q]
        return Pitched(ptr, raw[0] * self.elem_sizes_[q], raw[1])

    def curr_data(self, q: int) -> Pitched:
        return self.pitched(q, "curr")

    def next_data(self, q: int) -> Pitched:
        return self.pitched(q, "next")

    def swap(self) -> None:
        """LocalDomain::swap, src/local_domain.cu:67-84"""
        self.curr_, self.next_ = self.next_, self.curr_

    # -- host transfers (test / IO helpers; reference region_to_host etc., src/local_domain.cu:131-157)
    def quantity_to_host(self, q: int, which: str = "curr") -> np.ndarray:
        raw = self.raw_size()
        out = np.empty(raw[::-1], dtype=self.dtypes_[q])
        p = (self.curr_ if which == "curr" else self.next_)[q]
        check(lib().sb_memcpy(out.ctypes.data, C.c_void_p(p), out.nbytes, self.dev_, None))
        check(lib().sb_stream_sync(self.dev_, None))
        return out

    def interior_to_host(self, q: int) -> np.ndarray:
        full = self.quantity_to_host(q)
        p = self.halo_pos((0, 0, 0), True)
        e = self.sz_
        return np.ascontiguousarray(full[p[2] : p[2] + e[2], p[1] : p[1] + e[1], p[0] : p[0] + e[0]])

    def quantity_from_host(self, q: int, arr: np.ndarray, which: str = "curr") -> None:
        raw = self.raw_size()
        arr = np.ascontiguousarray(arr, dtype=self.dtypes_[q])
        assert arr.shape == raw[::-1], (arr.shape, raw)
        p = (self.curr_ if which == "curr" else self.next_)[q]
        check(lib().sb_memcpy(C.c_void_p(p), arr.ctypes.data, arr.nbytes, self.dev_, None))
        check(lib().sb_stream_sync(self.dev_, None))


# ------------------------------------------------------------------------------------------ copy plans
class CopyPlan:
    """sb_copy_plan: many box copies, one launch."""

    def __init__(self, device: int, copies: Sequence[BoxCopy]):
        arr = (BoxCopy * max(1, len(copies)))(*copies)
        h = C.c_void_p()
        check(lib().sb_copy_plan_create(C.byref(h), device, arr, len(copies)))
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_copy_plan_bytes(h))
        self.num_tiles = int(lib().sb_copy_plan_num_tiles(h))

    def launch(self, stream=None) -> None:
        check(lib().sb_copy_plan_launch(self._h, stream_ptr(stream)))

    def destroy(self) -> None:
        if self._h:
            lib().sb_copy_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def box_copy(dst: Pitched, dst_pos: Vec, src: Pitched, src_pos: Vec, ext: Vec, es: int) -> BoxCopy:
    return BoxCopy(dst, i3(dst_pos), src, i3(src_pos), i3(ext), es)


# ------------------------------------------------------------------------------------------ DistributedDomain
_SERIALS = itertools.count()


class DistributedDomain:
    """include/stencil/stencil.hpp:33-225 / src/stencil.cu for one NVSwitch node."""

    def __init__(self, x: int, y: int, z: int):
        self.size_ = (int(x), int(y), int(z))
        self._serial = next(_SERIALS)  # names this domain in its handles (picklable, unlike a reference)
        self.radius_ = Radius.constant(0)
        self.dtypes_: List[np.dtype] = []
        self.names_: List[str] = []
        self.gpus_: Optional[List[int]] = None
        self.flags_ = Method.Default
        self.strategy_ = PlacementStrategy.NodeAware
        self.domains_: List[LocalDomain] = []
        self.domain_idx_: List[Vec] = []
        self.partition_: Optional[Partition] = None
        self._plans: List[List[CopyPlan]] = []  # [parity][local domain]
        self._parity = 0
        self._streams = []
        self._bytes_kernel = 0
        self._bytes_peer = 0
        self._remote = None  # CUDA-IPC mappings of the other ranks (dist.RemoteDomains)
        self._nccl = None  # NCCL fallback (dist.NcclExchange)
        self._use_nccl = False
        self._epoch = 0
        self.boundary_: Tuple[Boundary, Boundary, Boundary] = (Boundary.PERIODIC,) * 3
        self.bcs_: Dict[Tuple[int, int], BC] = {}  # (quantity, face 0..5) -> BC
        self.topology_: Optional[Topology] = None
        self._bc_plans: List[List[Optional[BCPlan]]] = []  # [parity][local domain]
        self._subset_plans: Dict[tuple, tuple] = {}  # (parity, quantities) -> exchange(only=) plans (_exchange_plans)
        self._agreed: set = set()  # the subsets every rank has been checked to pass alike
        self._reduce_plans: Dict[tuple, List[ReducePlan]] = {}  # (item keys, parity) -> one plan per local domain
        self._krylov_plans: Dict[tuple, List[KrylovPlan]] = {}  # (mode, quantities, parity) -> one plan per local domain
        self._stencil_plans: Dict[tuple, list] = {}  # (op, buffers, exchange, parity) -> per local domain: plans
        self._apply_streams: list = []  # per local domain: (interior stream, exterior stream)
        self._transfer_plans: Dict[tuple, list] = {}  # (coarse domain, kind, buffers, both parities) -> per local domain
        self._paired: set = set()  # (coarse domain, with ghosts) that passed the pairing check

    # -- configuration (call before realize)
    def set_radius(self, r) -> None:
        self.radius_ = r if isinstance(r, Radius) else Radius.constant(int(r))

    def set_boundary(self, x: Boundary, y: Optional[Boundary] = None, z: Optional[Boundary] = None) -> None:
        """How the grid closes: one Boundary for all three axes, or one per axis (x, y, z).  On a FIXED axis no message
        crosses the grid's outer faces; their ghost cells are filled by the boundary conditions set for them."""
        if (y is None) != (z is None):
            raise _lib.StencilError("set_boundary takes one Boundary (all axes) or three (x, y, z)")
        b = (x, x, x) if y is None else (x, y, z)
        for v in b:
            if not isinstance(v, Boundary):
                raise _lib.StencilError(f"{v!r} is not a Boundary")
        self.boundary_ = tuple(b)

    def set_boundary_condition(self, h: DataHandle, face: Vec, bc: BC) -> None:
        """The boundary condition of quantity h on the wall face `face` ((+-1,0,0), (0,+-1,0) or (0,0,+-1)) of the whole
        grid; call before realize().  exchange() fills the ghost cells behind that face."""
        if not isinstance(bc, BC):
            raise _lib.StencilError(f"{bc!r} is not a BC")
        self.bcs_[(h.id, face_index(face))] = bc

    def get_topology(self) -> Optional[Topology]:
        return self.topology_

    def has_boundary_conditions(self) -> bool:
        return any(bc.kind != BCKind.NONE for bc in self.bcs_.values())

    def wall_kinds(self, idx: Vec, q: int) -> Tuple[List[int], List[float]]:
        """Per face of subdomain idx: (sb_bc_kind, value) of quantity q, NONE on faces that are not walls of idx."""
        kinds, values = [0] * 6, [0.0] * 6
        for (qq, f), bc in self.bcs_.items():
            if qq == q and self.topology_.is_wall(idx, f):
                kinds[f], values[f] = int(bc.kind), bc.value
        return kinds, values

    def _check_boundaries(self) -> None:
        """The errors realize() reports before it allocates anything (host only)."""
        for (q, f), bc in sorted(self.bcs_.items()):
            if bc.kind == BCKind.NONE:
                continue
            if self.boundary_[f // 2] == Boundary.PERIODIC:
                raise _lib.StencilError(f"quantity {q}: a boundary condition on face {FACES[f]} of a periodic axis (set_boundary FIXED first)")
            if bc.kind in (BCKind.VALUE, BCKind.ODD) and bc_dtype(self.dtypes_[q]) == 0:
                raise _lib.StencilError(f"quantity {q} ({self.dtypes_[q]}): {bc.kind.name} needs float32 or float64 (EVEN copies any type)")
        if self.has_boundary_conditions():
            for idx in self.partition_.indices():
                for q in range(len(self.dtypes_)):
                    bc_regions(self.partition_.subdomain_size(idx), self.radius_, self.wall_kinds(idx, q)[0])  # raises on g > n

    def add_data(self, dtype, name: str = "") -> DataHandle:
        self.dtypes_.append(np.dtype(dtype))
        self.names_.append(name)
        h = DataHandle(len(self.dtypes_) - 1, dtype, name)
        h._domain = self._serial  # exchange(only=) refuses the handles of another domain
        return h

    def set_methods(self, flags: Method) -> None:
        if (flags & Method.ColoQuantityKernel) and (flags & Method.ColoPackMemcpyUnpack):
            raise _lib.StencilError("can't use Direct Access and Pack-Memcpy-Unpack for colocated ranks")  # stencil.cu:192-197
        self.flags_ = flags

    def set_placement(self, strategy: PlacementStrategy) -> None:
        self.strategy_ = strategy

    def set_gpus(self, cuda_ids: Sequence[int]) -> None:
        self.gpus_ = [int(g) for g in cuda_ids]

    # -- queries
    def size(self) -> Vec:
        return self.size_

    def domains(self) -> List[LocalDomain]:
        return self.domains_

    def get_compute_region(self) -> Tuple[Vec, Vec]:
        return (0, 0, 0), self.size_

    def get_origin(self, i: int) -> Vec:
        return self.domains_[i].origin()

    def get_interior(self, r27=None) -> List[Tuple[Vec, Vec]]:
        """r27: the 27 radii to cut by (default: the domain's)."""
        out = []
        for d in self.domains_:
            lo, hi = d.get_compute_region()
            ilo, ihi = o3(), o3()
            check(lib().sb_interior(i3(lo), i3(hi), self.radius_.c27() if r27 is None else r27, ilo, ihi))
            out.append((t3(ilo), t3(ihi)))
        return out

    def get_exterior(self, r27=None) -> List[List[Tuple[Vec, Vec]]]:
        """r27: the 27 radii to cut by (default: the domain's)."""
        out = []
        for d in self.domains_:
            lo, hi = d.get_compute_region()
            elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
            n = check(lib().sb_exterior(i3(lo), i3(hi), self.radius_.c27() if r27 is None else r27, elo, ehi))
            out.append([(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(n)])
        return out

    def exchange_bytes_for_method(self, method: Method) -> int:
        """src/stencil.cu:139-161: same-GPU messages count as CudaKernel, cross-GPU as CudaMemcpyPeer
        (the transport that carries them here is the fused direct write in both cases)."""
        total = 0
        if method & Method.CudaKernel:
            total += self._bytes_kernel
        if method & Method.CudaMemcpyPeer:
            total += self._bytes_peer
        return total

    # -- realize
    def do_placement(self) -> None:
        from . import dist as _dist

        world = _dist.world()
        if self.gpus_ is None:
            n = C.c_int(0)
            check(lib().sb_device_count(C.byref(n)))
            if world.size > 1:
                self.gpus_ = [world.local_device]
            else:
                self.gpus_ = list(range(n.value))
        n_sub = len(self.gpus_) * world.size
        trivial = self.strategy_ == PlacementStrategy.Trivial
        # one node: NodePartition(size, radius, 1 node, n_sub gpus)  (partition.hpp:157-211)
        self.partition_ = Partition(self.size_, self.radius_, 1, n_sub, trivial=trivial)
        self.topology_ = Topology(self.partition_.dim, self.boundary_)
        self._world = world
        self._assign_owners()

    def realize(self) -> None:
        from . import dist as _dist

        self.do_placement()
        self._check_boundaries()
        world = self._world
        part = self.partition_
        all_idx = part.indices()
        my = [idx for idx in all_idx if self._owner[idx][0] == world.rank]
        for slot, idx in enumerate(my):
            d = LocalDomain(part.subdomain_size(idx), part.subdomain_origin(idx), self.gpus_[slot])
            d.set_radius(self.radius_)
            for dt, nm in zip(self.dtypes_, self.names_):
                d.add_data(dt, nm)
            d.realize()
            self.domains_.append(d)
            self.domain_idx_.append(idx)
        # peer access between all local GPUs (src/stencil.cu:123-127)
        for a in set(self.gpus_):
            for b in set(self.gpus_):
                ok = C.c_int(0)
                check(lib().sb_enable_peer(a, b, C.byref(ok)))
                if not ok.value:
                    raise _lib.StencilError(f"GPU {a} cannot map GPU {b}: P2P unavailable (NCCL fallback not selected)")
        self._remote, self._nccl = None, None
        self._alloc_staging()
        if world.size > 1:
            force_nccl = os.environ.get("SB_FORCE_NCCL", "0") == "1"
            if not force_nccl:
                try:
                    self._remote = _dist.share_domains(self, world)
                except _lib.StencilError as e:  # no IPC / peer mapping between these GPUs
                    import warnings

                    warnings.warn(f"CUDA IPC mapping unavailable ({e}); falling back to NCCL send/recv")
                    force_nccl = True
            self._use_nccl = force_nccl
            if force_nccl:
                self._drop_remote_staging()
        else:
            self._use_nccl = False
        self._build_plans()
        if self._use_nccl:
            self._nccl = _dist.NcclExchange(self, world)
        import torch

        self._streams = [torch.cuda.Stream(device=d.gpu(), priority=-1) for d in self.domains_]

    def _pitched_of(self, idx: Vec, q: int, parity: int) -> Tuple[Pitched, int]:
        """(pitched ptr, device) of the CURR buffer of quantity q of subdomain idx when the local swap
        parity is `parity` (every rank swaps in lock step)."""
        rank, slot = self._owner[idx]
        if rank == self._world.rank:
            d = self.domains_[slot]
            which = "curr" if parity == 0 else "next"
            # parity 1 means swap() was called an odd number of times: what is now curr was next at realize
            base = (d._curr0 if which == "curr" else d._next0)[q]
            raw = d.raw_size()
            return Pitched(base, raw[0] * d.elem_size(q), raw[1]), d.gpu()
        return self._remote.pitched(idx, q, parity)

    def _elem_sizes(self) -> List[int]:
        return [dt.itemsize for dt in self.dtypes_]

    def _gpu_key(self, idx: Vec):
        """Identity of the GPU holding subdomain idx (for 'same GPU?' decisions)."""
        rank, slot = self._owner[tuple(idx)]
        if rank == self._world.rank:
            return (rank, self.gpus_[slot])
        return (rank, -1 - slot)

    def _drop_remote_staging(self) -> None:
        """NCCL mode: messages from other ranks arrive packed through NCCL, not through staging buffers."""
        for key in [k for k in self._recv_local if self._owner[k[0]][0] != self._world.rank]:
            lib().sb_free(C.c_void_p(self._recv_local.pop(key)), self.domains_[0].gpu())

    def _layout(self, src_idx: Vec, dst_idx: Vec, qs=None) -> Tuple[int, List[dict]]:
        """dist.staging_layout of the (src -> dst) pair for the quantities qs (None: all), computed once per realize()."""
        from . import dist as _dist

        key = (tuple(src_idx), tuple(dst_idx), qs)
        if key not in self._layouts:
            self._layouts[key] = _dist.staging_layout(self, *key)
        return self._layouts[key]

    def _alloc_staging(self) -> None:
        """Receive buffers (on MY GPUs) for the thin messages other GPUs send to my subdomains (dist.staging_layout)."""
        self._recv_local: Dict[tuple, int] = {}
        self._layouts: Dict[tuple, Tuple[int, List[dict]]] = {}
        for di, dst_idx in enumerate(self.domain_idx_):
            srcs = {self.topology_.get_neighbor(dst_idx, d) for d in ALL_DIRS} - {None}
            for src_idx in sorted(srcs):
                if self._gpu_key(src_idx) == self._gpu_key(dst_idx):
                    continue
                total, _ = self._layout(src_idx, dst_idx)
                if total == 0:
                    continue
                p = C.c_void_p()
                check(lib().sb_malloc(C.byref(p), total, self.domains_[di].gpu()))
                self._recv_local[(tuple(src_idx), tuple(dst_idx))] = int(p.value)

    def _staging_target(self, src_idx: Vec, dst_idx: Vec):
        """Address of the staging buffer for (src -> dst), wherever dst lives; None if this pair is not staged."""
        key = (tuple(src_idx), tuple(dst_idx))
        if key in self._recv_local:
            return self._recv_local[key]
        if self._remote is not None and key in self._remote.recv:
            return self._remote.recv[key]
        return None

    def plan_messages(self, rank: Optional[int] = None) -> List[dict]:
        """The send plan of `rank` (default: this rank).  Pure geometry, no GPU: every rank can compute every other
        rank's plan.  exchange_messages of each subdomain the rank owns, in partition order, with the owners added:
        dict(src_slot, src_idx, dst_idx, dst_rank, dst_slot, dir, src_pos, dst_pos, ext)."""
        rank = self._world.rank if rank is None else rank
        out = []
        for idx in self.partition_.indices():
            owner, slot = self._owner[idx]
            if owner != rank:
                continue
            for m in exchange_messages(self.partition_, self.topology_, self.radius_, idx):
                dst_rank, dst_slot = self._owner[m["dst_idx"]]
                out.append(dict(m, src_slot=slot, dst_rank=dst_rank, dst_slot=dst_slot))
        return out

    def _assign_owners(self) -> None:
        # subdomain k of the node (linear order of the partition) lives on (rank, local gpu slot),
        # rank-major: the reference's global id = node*gpusPerNode + id with an identity placement
        # (NVSwitch is uniform, so the QAP of partition.hpp:706-716 is permutation-invariant -- DESIGN.md)
        per_rank = len(self.gpus_)
        self._owner = {idx: (k // per_rank, k % per_rank) for k, idx in enumerate(self.partition_.indices())}

    def _build_plans(self) -> None:
        """The exchange plans of every quantity, for both swap parities (_copy_plans), their byte counts and the stream
        dependencies of phase 2 and of the BC launches."""
        for d in self.domains_:
            d._curr0, d._next0 = list(d.curr_), list(d.next_)
        self._plans, self._unpack_plans = [], []
        self._subset_plans, self._agreed = {}, set()
        msgs = self.plan_messages()
        for parity in (0, 1):
            plans, unplans, count = self._copy_plans(msgs, parity, None)
            self._plans.append(plans)
            self._unpack_plans.append(unplans)
            if parity == 0:
                self._bytes_kernel, self._bytes_peer, self._staged_bytes = count
        # in-process senders of each local receiver (for the phase-1 -> phase-2 stream dependency)
        self._stage_senders: List[List[int]] = []
        for di, dst_idx in enumerate(self.domain_idx_):
            snd = set()
            for (src_idx, d_idx) in self._recv_local:
                if d_idx == tuple(dst_idx) and self._owner[src_idx][0] == self._world.rank:
                    snd.add(self._owner[src_idx][1])
            self._stage_senders.append(sorted(snd))
        self._bc_senders = []
        if self.has_boundary_conditions():
            self._bc_plans = [self._bc_plans_of(parity, None) for parity in (0, 1)]
            for idx in self.domain_idx_:
                srcs = {self.topology_.get_neighbor(idx, dv) for dv in ALL_DIRS} - {None}
                self._bc_senders.append(sorted({self._owner[s][1] for s in srcs if self._owner[s][0] == self._world.rank}))
        else:
            self._bc_plans = []

    def _copy_plans(self, msgs: List[dict], parity: int, qs):
        """The two copy phases of an exchange of the quantities qs (a sorted tuple; None: every quantity) for one swap
        parity.  Phase 1 (one launch per local subdomain): every outgoing halo region is stored either straight into
        the neighbour's ghost cells (same GPU, or wide rows over NVLink) or, for thin rows bound for another GPU, into
        the neighbour's dense staging buffer.  Phase 2 (one launch per local subdomain that has staged senders):
        scatter the staging buffers into the ghost cells.  A subset stages at the full layout's offsets
        (dist.staging_layout), so it uses the buffers realize() allocated.  Returns (phase 1 plans, phase 2 plans or
        None, (same-GPU bytes, cross-GPU bytes, staged bytes))."""
        plans, unplans = [], []
        kernel = peer = staged_bytes = 0
        for di, d in enumerate(self.domains_):
            mine = range(d.num_data()) if qs is None else qs
            copies: List[BoxCopy] = []
            for m in msgs:
                if m["src_slot"] != di:
                    continue
                remote = m["dst_rank"] != self._world.rank
                if self._use_nccl and remote:
                    peer += sum(d.elem_size(q) for q in mine) * m["ext"][0] * m["ext"][1] * m["ext"][2]
                    continue  # carried by the NCCL fallback, not by the fused kernel
                stage_base = None if self._gpu_key(m["src_idx"]) == self._gpu_key(m["dst_idx"]) else self._staging_target(m["src_idx"], m["dst_idx"])
                staged = {}
                if stage_base is not None:
                    staged = {e["q"]: e for e in self._layout(m["src_idx"], m["dst_idx"], qs)[1] if e["dir"] == m["dir"]}
                for q in mine:
                    es = d.elem_size(q)
                    src_p, _ = self._pitched_of(m["src_idx"], q, parity)
                    nbytes = es * m["ext"][0] * m["ext"][1] * m["ext"][2]
                    if q in staged:
                        dense = Pitched(stage_base + staged[q]["offset"], m["ext"][0] * es, m["ext"][1])
                        copies.append(box_copy(dense, (0, 0, 0), src_p, m["src_pos"], m["ext"], es))
                        staged_bytes += nbytes
                    else:
                        dst_p, _ = self._pitched_of(m["dst_idx"], q, parity)
                        copies.append(box_copy(dst_p, m["dst_pos"], src_p, m["src_pos"], m["ext"], es))
                    if self._gpu_key(m["src_idx"]) == self._gpu_key(m["dst_idx"]):
                        kernel += nbytes
                    else:
                        peer += nbytes
            plans.append(CopyPlan(d.gpu(), copies))
            # phase 2 of this subdomain as a receiver
            ucopies: List[BoxCopy] = []
            for (src_idx, dst_idx), base in self._recv_local.items():
                if dst_idx != tuple(self.domain_idx_[di]):
                    continue
                for e in self._layout(src_idx, dst_idx, qs)[1]:
                    dst_p, _ = self._pitched_of(dst_idx, e["q"], parity)
                    dense = Pitched(base + e["offset"], e["ext"][0] * e["es"], e["ext"][1])
                    ucopies.append(box_copy(dst_p, e["dst_pos"], dense, (0, 0, 0), e["ext"], e["es"]))
            unplans.append(CopyPlan(d.gpu(), ucopies) if ucopies else None)
        return plans, unplans, (kernel, peer, staged_bytes)

    def _bc_plans_of(self, parity: int, qs) -> List[Optional[BCPlan]]:
        """One boundary-condition plan per local subdomain over the quantities qs (None: all), for one swap parity (None
        where the subdomain has no wall face with a BC of those quantities)."""
        plans = []
        for di, d in enumerate(self.domains_):
            idx = self.domain_idx_[di]
            bq = []
            for q in range(d.num_data()) if qs is None else qs:
                kinds, values = self.wall_kinds(idx, q)
                p, _ = self._pitched_of(idx, q, parity)
                bq.append(_lib.BcQuantity(p, d.elem_size(q), (C.c_double * 6)(*values), bc_dtype(self.dtypes_[q]), _lib.I6(*kinds)))
            plan = BCPlan(d.gpu(), bq, d.size(), self.radius_)
            plans.append(plan if plan.bytes else None)
        return plans

    # -- the hot path
    def exchange_key(self, only) -> Optional[Tuple[int, ...]]:
        """The quantities exchange(only=only) moves, as a sorted tuple of quantity indices; None for every quantity (only
        is None, or names every quantity of the domain).  Refuses (StencilError) an empty subset, a quantity named twice
        and anything that is not a DataHandle of this domain.  Host only."""
        if only is None:
            return None
        if isinstance(only, DataHandle):
            raise _lib.StencilError("exchange: only must be a sequence of DataHandles (or None), not one DataHandle")
        qs = []
        for h in only:
            owner = getattr(h, "_domain", None)
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(self.dtypes_) or (owner is not None and owner != self._serial):
                raise _lib.StencilError(f"exchange: {h!r} is not a DataHandle of this domain")
            if h.id in qs:
                raise _lib.StencilError(f"exchange: quantity {h.id} ({self.names_[h.id] or 'unnamed'}) is named twice")
            qs.append(h.id)
        if not qs:
            raise _lib.StencilError("exchange: only names no quantity (None exchanges every quantity)")
        if len(qs) == len(self.dtypes_):
            return None
        if max(qs) >= 64:
            raise _lib.StencilError(f"exchange: quantity {max(qs)}: a subset names quantities 0..63 only")
        return tuple(sorted(qs))

    def _agree_on_subset(self, qs: Tuple[int, ...]) -> None:
        """exchange() is collective, so every rank must exchange the same quantities: checked once per subset, when its
        plans are first built (one all_gather_object), never on later calls."""
        if qs in self._agreed:
            return
        if self._world.size > 1:
            from . import dist as _dist

            everyone = _dist.all_gather_object(qs)
            for r, theirs in enumerate(everyone):
                if tuple(theirs) != qs:
                    raise _lib.StencilError(f"exchange: rank {r} exchanges quantities {list(theirs)}, rank {self._world.rank} "
                                            f"{list(qs)}: every rank must pass the same subset")
        self._agreed.add(qs)

    def _exchange_plans(self, qs):
        """(phase 1, phase 2, BC plans or None) of an exchange of qs (None: every quantity) for the current swap parity;
        a subset's are built on first use and kept per (swap parity, subset) until close()."""
        parity = self._parity
        if qs is None:
            return self._plans[parity], self._unpack_plans[parity], self._bc_plans[parity] if self._bc_plans else None
        key = (parity, qs)
        if key not in self._subset_plans:
            self._agree_on_subset(qs)
            plans, unplans, _ = self._copy_plans(self.plan_messages(), parity, qs)
            bcs = self._bc_plans_of(parity, qs) if self._bc_plans else None
            if bcs is not None and all(b is None for b in bcs):
                bcs = None
            self._subset_plans[key] = (plans, unplans, bcs)
        return self._subset_plans[key]

    def exchange_bytes(self, only=None) -> int:
        """Bytes the first copy phase of one exchange(only=only) moves on this rank (the box copies of every local
        subdomain, staged rows included); the messages the NCCL fallback carries and the ghost bytes of the BC fill are
        not counted.  For a subset not used yet it builds the subset's plans, which is collective under torchrun like
        exchange() itself: every rank calls it with the same subset."""
        plans, _, _ = self._exchange_plans(self.exchange_key(only))
        return sum(p.bytes for p in plans)

    def exchange_async(self, only=None) -> None:
        """Enqueue the halo exchange on the library's high-priority streams (one per local subdomain).  only: the
        quantities to exchange, a sequence of DataHandles of this domain (see exchange()); None: every quantity."""
        if self.partition_ is None or not self._plans:
            raise _lib.StencilError("exchange: call realize() first")
        self._exchange_async(self.exchange_key(only))

    def _exchange_async(self, qs) -> None:
        import torch

        plans, unplans, bcs = self._exchange_plans(qs)
        if self._remote is not None:
            self._epoch += 1
            self._remote.begin(self._epoch, self._streams)
        phase1 = []
        for plan, s in zip(plans, self._streams):
            plan.launch(s)
            if bcs is not None:  # the BC launch of every receiver waits for its local senders' phase 1
                ev = torch.cuda.Event()
                ev.record(s)
                phase1.append(ev)
        if self._remote is not None:
            self._remote.finish(self._epoch, self._streams)  # every remote sender's phase 1 has landed
            if len(self._streams) > 1:
                ev0 = torch.cuda.Event()
                ev0.record(self._streams[0])
                for o in self._streams[1:]:
                    o.wait_event(ev0)
        if self._nccl is not None:
            self._nccl.exchange(self._parity, self._streams[0], qs)
        # phase 2: scatter what other GPUs staged for my subdomains
        if any(u is not None for u in unplans):
            events = {}
            for di, snd in enumerate(self._stage_senders):
                for sj in snd:
                    if sj not in events and sj != di:
                        ev = torch.cuda.Event()
                        ev.record(self._streams[sj])
                        events[sj] = ev
            for di, u in enumerate(unplans):
                if u is None:
                    continue
                for sj in self._stage_senders[di]:
                    if sj != di:
                        self._streams[di].wait_event(events[sj])
                u.launch(self._streams[di])
        # boundary conditions: after this subdomain's phase 2 (stream order), its local senders' phase 1 (events), the
        # remote senders' phase 1 (RemoteDomains.finish above) and the NCCL unpack (stream 0)
        if bcs is not None:
            nccl_done = None
            if self._nccl is not None and len(self._streams) > 1:
                nccl_done = torch.cuda.Event()
                nccl_done.record(self._streams[0])
            for di, b in enumerate(bcs):
                if b is None:
                    continue
                s = self._streams[di]
                for sj in self._bc_senders[di]:
                    if sj != di:
                        s.wait_event(phase1[sj])
                if nccl_done is not None and di != 0:
                    s.wait_event(nccl_done)
                b.launch(s)

    def exchange(self, only=None) -> None:
        """DistributedDomain::exchange (src/stencil.cu:1002-1186): returns when every ghost cell of
        every local subdomain holds its neighbour's current value.

        only: a sequence of DataHandles of this domain (DESIGN.md section 2.15).  Only those quantities' boxes are
        copied and only their walls' boundary conditions filled, with the same kernels, staging buffers and ordering as
        the full exchange; every byte of the other quantities, ghost cells included, is left as it was.  None, or every
        quantity, is the full exchange.  An empty subset, a quantity named twice or a handle of another domain is a
        StencilError.  The plans of a subset are built on its first use and kept per (swap parity, subset) until close().
        Under torchrun the exchange is collective and every rank passes the same subset: the first use of each subset
        checks that with one all_gather_object (later calls do not).
            dd.exchange(only=[u])          # before a sweep that reads u at an offset and f at offset 0"""
        self.exchange_async(only)
        for d, s in zip(self.domains_, self._streams):
            check(lib().sb_stream_sync(d.gpu(), stream_ptr(s)))

    def _exchange_sel(self, name: str, exchange, reads) -> object:
        """What an operator call exchanges: False (nothing), True (every quantity) or a sorted tuple of quantities.
        exchange: a bool, "reads" (the quantities of `reads`, those the call reads at a non-zero offset; none of them
        means no exchange, all of them the full exchange), or a tuple of DataHandles of this domain (the solvers: the
        vector the call reads at an offset, its coefficient fields exchanged when they change)."""
        if isinstance(exchange, str) and exchange == "reads":
            qs = set(reads)
        elif isinstance(exchange, tuple):
            qs = {h.id for h in exchange}
        elif isinstance(exchange, str):
            raise _lib.StencilError(f"{name}: exchange must be True, False or 'reads', not {exchange!r}")
        else:
            return bool(exchange)  # any other value by its truth, as before "reads" existed
        if not qs:
            return False
        return True if len(qs) == len(self.dtypes_) else tuple(sorted(qs))

    def exchange_streams(self):
        return self._streams

    def swap(self) -> None:
        """DistributedDomain::swap (src/stencil.cu:852-872).  The exchange plans exist for both
        parities, so -- unlike the reference's captured pack graphs (SURVEY.md 4, latent bug) -- the
        next exchange reads the new curr buffers."""
        for d in self.domains_:
            d.swap()
        self._parity ^= 1

    # -- reductions
    _REDUCE_KINDS = {"scalar": (_lib.REDUCE_SCALAR, 1), "diff": (_lib.REDUCE_DIFF, 1), "norm": (_lib.REDUCE_NORM3, 3)}

    def reduce(self, h: DataHandle, which: str = "curr", exact: bool = False) -> Reduction:
        """min, max, sum and sum of squares of quantity h (its curr or next buffer) over the whole compute region.
        exact=True: sum and sumsq correctly rounded, the same bits for every partition (sb_reduce_exact_*)."""
        return self.reduce_many([("scalar", h, which)], exact=exact)[0]

    def reduce_diff(self, h: DataHandle, exact: bool = False) -> Reduction:
        """The same statistics of curr - next of quantity h; .l2() is the 2-norm of the last update after a swap."""
        return self.reduce_many([("diff", h)], exact=exact)[0]

    def reduce_norm(self, hx: DataHandle, hy: DataHandle, hz: DataHandle, exact: bool = False) -> Reduction:
        """Statistics of |u| = sqrt(hx^2 + hy^2 + hz^2) (curr buffers); .rms() is sqrt(sum |u|^2 / N)."""
        return self.reduce_many([("norm", hx, hy, hz)], exact=exact)[0]

    def reduce_plans(self, items: Sequence[tuple], exact: bool = False) -> list:
        """The plans reduce_many(items, exact) launches, one per local subdomain, for the current swap parity
        (ReducePlan, or ExactReducePlan with exact=True).  They are built on first use and kept, per item list,
        exactness and parity, until close(): a program should reduce a fixed set of item lists rather than build a new
        list every iteration, or each new list holds device memory until close()."""
        keys = [self._reduce_key(it) for it in items]
        if not keys:
            raise _lib.StencilError("reduce_plans: no items")
        ck = (tuple(keys), self._parity, bool(exact))
        plans = self._reduce_plans.get(ck)
        if plans is None:
            cls = ExactReducePlan if exact else ReducePlan
            plans = [cls(d.gpu(), [self._reduce_item(di, k) for k in keys]) for di, d in enumerate(self.domains_)]
            self._reduce_plans[ck] = plans
        return plans

    def reduce_many(self, items: Sequence[tuple], exact: bool = False) -> List[Reduction]:
        """Several reductions, one launch sequence per local subdomain.  Items: ("scalar", h[, "curr" | "next"]),
        ("diff", h) (curr - next), ("norm", hx, hy, hz).  Waits for all work queued on the local devices, reduces on
        the exchange streams, gathers every rank's per-subdomain results and merges them with sb_reduce_combine in
        global subdomain-index order (x fastest), so every rank returns the same bits.  exact=True: the per-subdomain
        exact parts are gathered, combined by sb_reduce_exact_combine and rounded once, so sum and sumsq are correctly
        rounded and the same bits for every partition and rank count.  Collective under torchrun.  The plans are cached
        as reduce_plans() describes."""
        from . import dist as _dist

        if not items:
            return []
        n = len(items)
        plans = self.reduce_plans(items, exact)
        for dev in sorted({d.gpu() for d in self.domains_}):
            check(lib().sb_device_sync(dev))
        for plan, s in zip(plans, self._streams):
            plan.launch(s)
        if exact:
            return self._exact_gather([(idx, plan.parts(s)) for idx, plan, s in zip(self.domain_idx_, plans, self._streams)], n)
        dim = self.partition_.dim
        mine = [(idx, [(r.min, r.max, r.sum, r.sumsq, r.count) for r in plan.results(s)])
                for idx, plan, s in zip(self.domain_idx_, plans, self._streams)]  # fmt: skip
        everyone = _dist.all_gather_object(mine) if self._world.size > 1 else [mine]
        parts = sorted((p for rank_parts in everyone for p in rank_parts), key=lambda p: p[0][0] + dim[0] * (p[0][1] + dim[1] * p[0][2]))
        return [reduce_combine([Reduction(*p[1][i]) for p in parts]) for i in range(n)]

    def _reduce_key(self, it: tuple) -> tuple:
        if not it or it[0] not in self._REDUCE_KINDS:
            raise _lib.StencilError(f"reduction item {it!r}: the first element must be 'scalar', 'diff' or 'norm'")
        kind, nsrc = self._REDUCE_KINDS[it[0]]
        hs = it[1 : 1 + nsrc]
        rest = it[1 + nsrc :]
        if len(hs) != nsrc or not all(isinstance(h, DataHandle) for h in hs):
            raise _lib.StencilError(f"reduction item {it!r}: '{it[0]}' takes {nsrc} DataHandle(s)")
        which = "curr"
        if kind == _lib.REDUCE_SCALAR and rest:
            which = rest[0]
            rest = rest[1:]
        if rest or which not in ("curr", "next"):
            raise _lib.StencilError(f"reduction item {it!r}: unexpected {rest or which!r}")
        dts = {self.dtypes_[h.id] for h in hs}
        if len(dts) != 1 or bc_dtype(dts.pop()) == 0:
            raise _lib.StencilError(f"reduction item {it!r}: the sources must all be float32 or all float64")
        return (kind, tuple(h.id for h in hs), which)

    def _reduce_item(self, di: int, key: tuple) -> _lib.ReduceItem:
        kind, qs, which = key
        d, idx = self.domains_[di], self.domain_idx_[di]
        parity = self._parity if which == "curr" else self._parity ^ 1
        srcs = [self._pitched_of(idx, q, parity)[0] for q in qs]
        srcs += [srcs[0]] * (3 - len(srcs))
        if kind == _lib.REDUCE_DIFF:
            srcs[1] = self._pitched_of(idx, qs[0], self._parity ^ 1)[0]
        lo, hi = d.get_compute_region()
        return _lib.ReduceItem(kind, bc_dtype(self.dtypes_[qs[0]]), (Pitched * 3)(*srcs), i3(d.accessor_origin()), i3(lo), i3(hi))

    def _exact_gather(self, mine: Sequence[tuple], n: int) -> List[Reduction]:
        """mine: (subdomain index, [n exact parts]) per local subdomain.  Every rank's parts gathered, combined by
        sb_reduce_exact_combine and rounded once: the same bits on every rank and for every partition.  The one exact
        combine of reduce_many(exact=True), dot() and the PCG solver."""
        from . import dist as _dist

        mine = [(idx, [bytes(p) for p in parts]) for idx, parts in mine]
        everyone = _dist.all_gather_object(mine) if self._world.size > 1 else [mine]
        dim = self.partition_.dim
        parts = sorted((p for rank_parts in everyone for p in rank_parts), key=lambda p: p[0][0] + dim[0] * (p[0][1] + dim[1] * p[0][2]))
        return [reduce_exact_round(reduce_exact_combine([_lib.ReduceExactPart.from_buffer_copy(p[1][i]) for p in parts])) for i in range(n)]

    def krylov_plans(self, mode: int, handles: Sequence[DataHandle]) -> List[KrylovPlan]:
        """The KrylovPlans of one pass over the compute region of every local subdomain, on the curr buffers of handles
        (in sb_krylov_plan_create's order: DOT a, b[, c]; XPBY p, z; UPDATE x, p, r, q[, c]; BICG_P p, r, v), for the
        current swap parity.
        Built on first use and kept until close(), like reduce_plans()."""
        if self.partition_ is None or not self._plans:
            raise _lib.StencilError("krylov_plans: call realize() first")
        qs = []
        for h in handles:
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(self.dtypes_):
                raise _lib.StencilError(f"krylov_plans: {h!r} is not a DataHandle of this domain")
            qs.append(h.id)
        dts = {self.dtypes_[q] for q in qs}
        if len(dts) != 1 or bc_dtype(next(iter(dts))) == 0:
            raise _lib.StencilError("krylov_plans: the quantities must all be float32 or all float64")
        key = (int(mode), tuple(qs), self._parity)
        plans = self._krylov_plans.get(key)
        if plans is None:
            plans = []
            try:
                for d in self.domains_:
                    lo, hi = d.get_compute_region()
                    plans.append(KrylovPlan(d.gpu(), mode, self.dtypes_[qs[0]], [d.pitched(q, "curr") for q in qs], d.accessor_origin(), lo, hi))
            except Exception:
                for p in plans:
                    p.destroy()
                raise
            self._krylov_plans[key] = plans
        return plans

    def dot(self, a: DataHandle, b: DataHandle) -> float:
        """The exact inner product <a, b> of the curr buffers of two float32 or float64 quantities over the whole compute
        region (DESIGN.md section 2.13): the exact sum over the cells of fl64(double(a) * double(b)), rounded once to
        double, so every partition, rank count and layout gives the same bits (a may be b: <a, a> = ||a||^2).  Waits for
        all work queued on the local devices, computes on the exchange streams and gathers every rank's parts: collective
        under torchrun.  The plans are cached as krylov_plans() describes."""
        plans = self.krylov_plans(_lib.KRYLOV_DOT, (a, b))
        for dev in sorted({d.gpu() for d in self.domains_}):
            check(lib().sb_device_sync(dev))
        for plan, s in zip(plans, self._streams):
            plan.launch(s)
        return self._exact_gather([(idx, plan.parts(s)) for idx, plan, s in zip(self.domain_idx_, plans, self._streams)], 1)[0].sum

    # -- linear stencil operators
    def apply(self, op, dst, src, aux=None, exchange=True, coefs=None, colour=None) -> None:
        """dst = op(src, aux, coefs) over the whole compute region of every local subdomain (DESIGN.md section 2.7).

        Buffers are (DataHandle, "curr" | "next"); a bare handle means "next" for dst and "curr" for src and aux.  src is
        always a curr buffer (the one exchange() fills); dst may be aux, never src; all share op's element type.
        coefs: one DataHandle per coefficient field the op names (op.ncoef of them, field k = coefs[k]), read from their
        curr buffers, which exchange() fills like src's (with the quantity's own BC on a wall); a coefficient must not be
        dst.  swap() turns every quantity's buffers, coefficients included, so a static coefficient must hold the same
        compute cells in curr and next.
        exchange=True: the interior runs on its own stream while exchange() fills the ghost cells, then the exterior slabs
        of each subdomain run as one launch; exchange=False: one launch over the whole region, and the caller guarantees
        the ghost cells are current; exchange="reads": the schedule of True, with an exchange of only the quantities the
        call reads at a non-zero offset (exchange(only=...), DESIGN.md section 2.15): src, and each coefficient field
        that a term reads at a non-zero coefficient offset.  The launches and the exchange are ordered after the work
        queued on the caller's current stream, and the call returns when the update is complete.  The plans are built
        on first use and kept, per (op, buffers, exchange, swap parity, colour), until close().  Under torchrun every
        rank calls it (exchange() is collective).
        colour=(m, c), m in 1, 2, 8 (DESIGN.md section 2.9): only the cells of colour c of the colouring m (taken from global
        coordinates) are written, each from the buffers as they were before the call, and with m > 1 dst may be src, so
        a Gauss-Seidel / SOR sweep is one call per colour:
            sor = op.relax(omega)                         # op: A of A u = f
            for c in range(2):
                dd.apply(sor, (u, "curr"), u, f, colour=(2, c))
        Every src term with a non-zero offset must read another colour (op.check(radius, colours=m)).  In place the
        schedule is the same, with the interior cut by the larger radius of both sides of each axis, so that it writes
        no cell exchange() sends (a slab as wide as the opposite side's radius); the exterior runs after exchange()."""
        self._run_plans(*self._apply_plans(op, dst, src, aux, exchange, coefs, colour))

    def relax(self, A, dst, u, f, coefs=None, colour=None, omega: float = 1.0, exchange=True) -> None:
        """One relaxation pass of A u = f that divides by A's own diagonal (DESIGN.md section 2.12): dst[p] = u(p) +
        omega ((f(p) - (A u)(p)) / d(p)), d(p) the sum of the factors (weight, times the coefficient for a coefficient
        term) of A's terms at offset 0, for the cells of colour c of colour=(m, c) (None: every cell, weighted Jacobi,
        dst must not be u).  A has src terms only (plain or coefficient terms) and at least one term at offset 0; for
        div(kappa grad u) the diagonal differs from cell to cell, which A.relax(omega) cannot express.  Buffers, coefs,
        the colour condition, the schedule (exchange="reads" included: u and the coefficients read at an offset, f is
        read at offset 0), the in-place interior cut and the plan cache are apply()'s, with u as src and f as aux; omega
        joins the plan key.  A red-black Gauss-Seidel sweep of -div(kappa grad u) = f:
            A = StencilOp.div_grad((h, h, h), np.float64).scaled(-1.0)
            for c in range(2):
                dd.relax(A, (u, "curr"), u, f, coefs=[kx, ky, kz], colour=(2, c))
        A zero or non-finite diagonal gives whatever IEEE arithmetic gives."""
        if not np.isfinite(float(omega)):
            raise _lib.StencilError(f"relax: omega = {omega} must be finite")
        self._run_plans(*self._apply_plans(A, dst, u, f, exchange, coefs, colour, omega=float(omega)))

    def _apply_plans(self, op, dst, src, aux=None, exchange=True, coefs=None, colour=None, omega=None):
        """apply()'s checks and cached plans, returned with its schedule as the arguments of _run_plans.  omega: relax()'s
        plans (aux is f)."""
        from .stencil_op import StencilOp, StencilPlan

        name = "apply" if omega is None else "relax"
        if not isinstance(op, StencilOp):
            raise _lib.StencilError(f"{op!r} is not a StencilOp")
        if self.partition_ is None or not self._plans:
            raise _lib.StencilError(f"{name}: call realize() first")

        def buf(arg, default, role):
            h, which = (arg, default) if isinstance(arg, DataHandle) else tuple(arg)
            if not isinstance(h, DataHandle) or which not in ("curr", "next"):
                raise _lib.StencilError(f"{name}: {role} must be a DataHandle or (DataHandle, 'curr' | 'next'), not {arg!r}")
            if self.dtypes_[h.id] != op.dtype:
                raise _lib.StencilError(f"{name}: {role} is {self.dtypes_[h.id]}, the op computes in {op.dtype}")
            return h.id, which

        d_q, d_w = buf(dst, "next", "dst")
        s_q, s_w = buf(src, "curr", "src")
        if s_w != "curr":
            raise _lib.StencilError(f"{name}: src must be a curr buffer (the one exchange() fills)")
        ncol, col = (1, 0) if colour is None else (int(colour[0]), int(colour[1]))
        if ncol not in (1, 2, 8) or not 0 <= col < ncol:
            raise _lib.StencilError(f"{name}: colour {colour!r} must be (m, c) with m in 1, 2, 8 and 0 <= c < m")
        if (d_q, d_w) == (s_q, s_w) and ncol == 1:
            raise _lib.StencilError(f"{name}: dst must not be src")
        a = buf(aux, "curr", "aux" if omega is None else "f") if aux is not None else None
        if op.has_aux and a is None:
            raise _lib.StencilError(f"{name}: the op has a term on aux, but no aux buffer was given")
        if omega is not None:
            if op.has_aux:
                raise _lib.StencilError("relax: A has a term on aux; A reads u only (f is the right-hand side)")
            if not any(t[0] == 0 and t[1] == (0, 0, 0) for t in op.terms):
                raise _lib.StencilError("relax: A has no term at offset (0, 0, 0), so no diagonal")
            if a is None:
                raise _lib.StencilError("relax: f is needed")
        cs = list(coefs) if coefs is not None else []
        if len(cs) != op.ncoef:
            raise _lib.StencilError(f"{name}: the op reads {op.ncoef} coefficient fields, but {len(cs)} were given")
        c_q = []
        for k, c in enumerate(cs):
            q, w = buf(c, "curr", f"coefficient {k}")
            if w != "curr":
                raise _lib.StencilError(f"{name}: coefficient {k} must be a curr buffer (the one exchange() fills)")
            if (q, w) == (d_q, d_w):
                raise _lib.StencilError(f"{name}: coefficient {k} must not be dst")
            c_q.append(q)
        op.check(self.radius_, colours=ncol)
        reads_aux = op.has_aux or omega is not None
        exchange = self._exchange_sel(name, exchange, [s_q] + op_moved_coefs(op, c_q))
        key = (op.key(), (d_q, d_w), s_q, a if reads_aux else None, tuple(c_q), bool(exchange), self._parity, (ncol, col))
        if omega is not None:
            key += ("diag", omega)

        def make(di, d, boxes):
            P = (d.pitched(d_q, d_w), d.pitched(s_q, "curr"), d.pitched(a[0], a[1]) if a is not None and reads_aux else Pitched(None, 0, 0))
            K = [d.pitched(q, "curr") for q in c_q] if op.has_coef else None
            return StencilPlan(d.gpu(), op, *P, d.accessor_origin(), d.raw_size()[2], boxes, K, (ncol, col) if ncol > 1 else None, omega)

        return self._plans_for(key, exchange, make, writes_src=(d_q, d_w) == (s_q, s_w)), exchange

    def apply_system(self, system, outputs, inputs, exchange=True) -> None:
        """outputs = system(inputs) over the whole compute region of every local subdomain (DESIGN.md section 2.8).

        outputs: system.nout buffers, inputs: system.nin buffers, each (DataHandle, "curr" | "next"); a bare handle means
        "next" for an output and "curr" for an input; an input no term reads may be None.  All share the system's element
        type.  An input read at a non-zero offset (as a source or a coefficient) must be a curr buffer, the one
        exchange() fills.  Outputs are pairwise distinct; an output may be an input only if every read of that input is
        at offset 0 (an in-place update such as E = E + dt curl H).
        The schedule, the plan cache (per system, buffers, exchange and swap parity) and the torchrun rule are apply()'s;
        exchange="reads" exchanges the inputs of system.moved_inputs() only."""
        from .stencil_op import StencilSystem, SystemPlan

        if not isinstance(system, StencilSystem):
            raise _lib.StencilError(f"{system!r} is not a StencilSystem")
        if self.partition_ is None or not self._plans:
            raise _lib.StencilError("apply_system: call realize() first")
        outputs, inputs = list(outputs), list(inputs)
        if len(outputs) != system.nout or len(inputs) != system.nin:
            raise _lib.StencilError(f"apply_system: the system has {system.nin} inputs and {system.nout} outputs, "
                                    f"but {len(inputs)} inputs and {len(outputs)} outputs were given")

        def buf(arg, default, role):
            h, which = (arg, default) if isinstance(arg, DataHandle) else tuple(arg)
            if not isinstance(h, DataHandle) or which not in ("curr", "next"):
                raise _lib.StencilError(f"apply_system: {role} must be a DataHandle or (DataHandle, 'curr' | 'next'), not {arg!r}")
            if self.dtypes_[h.id] != system.dtype:
                raise _lib.StencilError(f"apply_system: {role} is {self.dtypes_[h.id]}, the system computes in {system.dtype}")
            return h.id, which

        outs = [buf(o, "next", f"output {j}") for j, o in enumerate(outputs)]
        reads, moved = system.read_inputs(), system.moved_inputs()
        ins = []
        for i, a in enumerate(inputs):
            if a is None:
                if i in reads:
                    raise _lib.StencilError(f"apply_system: input {i} is read by a term, but it is None")
                ins.append(None)
                continue
            q = buf(a, "curr", f"input {i}")
            if i in moved and q[1] != "curr":
                raise _lib.StencilError(f"apply_system: input {i} is read at a non-zero offset, so it must be a curr buffer (the one exchange() fills)")
            ins.append(q if i in reads else None)
        if len(set(outs)) != len(outs):
            raise _lib.StencilError("apply_system: the outputs must be distinct buffers")
        for j, o in enumerate(outs):
            for i in moved:
                if ins[i] == o:
                    raise _lib.StencilError(f"apply_system: output {j} is input {i}, which is read at a non-zero offset")
        system.check(self.radius_)
        exchange = self._exchange_sel("apply_system", exchange, [ins[i][0] for i in moved])
        key = ("system", system.key(), tuple(outs), tuple(ins), bool(exchange), self._parity)

        def make(di, d, boxes):
            O = [d.pitched(q, w) for q, w in outs]
            I = [d.pitched(q[0], q[1]) if q is not None else Pitched(None, 0, 0) for q in ins]
            return SystemPlan(d.gpu(), system, O, I, d.accessor_origin(), d.raw_size()[2], boxes)

        self._run_plans(self._plans_for(key, exchange, make), exchange)

    def _plans_for(self, key, exchange: bool, make, writes_src: bool = False):
        """The cached per-domain plans of key: (interior, exterior) pairs with exchange, else one plan over the whole
        compute region; make(di, d, boxes) builds one plan.  writes_src: the plans write src (a coloured apply in place).
        exchange() sends from side s of a subdomain a slab as wide as the radius on side -s, so such an interior also
        keeps clear of that: it is cut by max(radius(d), radius(-d)) in every direction d."""
        plans = self._stencil_plans.get(key)
        if plans is None:
            plans = []
            r = list(self.radius_.c27())
            r27 = I27(*[max(r[i], r[26 - i]) for i in range(27)]) if writes_src else None
            interiors, exteriors = (self.get_interior(r27), self.get_exterior(r27)) if exchange else (None, None)
            for di, d in enumerate(self.domains_):
                if exchange:
                    plans.append((make(di, d, [interiors[di]]), make(di, d, exteriors[di])))
                else:
                    plans.append((make(di, d, [d.get_compute_region()]),))
            self._stencil_plans[key] = plans
        return plans

    def _run_plans(self, plans, exchange: bool, queued: bool = False) -> None:
        """The schedule of every operator call, ordered by CUDA events only.  Each interior (or the one plan without
        exchange) waits for the previous exterior on its subdomain's apply streams; with exchange, the exchange waits for
        every apply stream as they were before this interior (_queue_exchange), and each exterior waits for the exchange.
        A public call first orders the apply streams after the caller's stream and returns when its work is complete
        (wait_queued); queued=True (a solver that owns the schedule) returns at once."""
        self._ensure_apply_streams()
        if not queued:
            self._follow_caller()
        multi = len({d.gpu() for d in self.domains_}) > 1
        apply_ev, _ = self._queue_events()
        for (si, se), pair in zip(self._apply_streams, apply_ev):
            pair[1].record(se)
            si.wait_event(pair[1])
        if exchange:
            self._queue_exchange(exchange)
        for d, p, (si, _) in zip(self.domains_, plans, self._apply_streams):
            if multi:
                _set_current_device(d.gpu())
            p[0].launch(si)
        if exchange:
            self._wait_exchange(self, interior=False)
            for d, p, (_, se) in zip(self.domains_, plans, self._apply_streams):
                if multi:
                    _set_current_device(d.gpu())
                p[1].launch(se)
        if not queued:
            wait_queued([self])

    # -- the queued schedule: nothing waits on the host, CUDA events order the launches
    def _ensure_apply_streams(self) -> None:
        """Two apply streams per local domain (interior, exterior), made on first use."""
        if not self._apply_streams:
            import torch

            self._apply_streams = [(torch.cuda.Stream(device=d.gpu()), torch.cuda.Stream(device=d.gpu())) for d in self.domains_]

    def _follow_caller(self) -> None:
        """Every apply stream waits for the work queued so far on the caller's current stream of its device."""
        import torch

        self._ensure_apply_streams()
        for d, (si, se) in zip(self.domains_, self._apply_streams):
            ev = torch.cuda.current_stream(d.gpu()).record_event()
            si.wait_event(ev)
            se.wait_event(ev)

    def _queue_clear(self, h: DataHandle) -> None:
        """h's whole curr allocation set to +0, queued on the interior apply streams after the previous exterior."""
        self._run_plans([(_Clear(d, h.id),) for d in self.domains_], False, queued=True)

    def _queue_events(self):
        """The events of the queued schedule, created once and recorded again on each use (a wait takes the record made
        before it): per local domain a pair for its apply streams, and one per exchange stream."""
        import torch

        ev = getattr(self, "_queue_ev", None)
        if ev is None or len(ev[0]) != len(self._apply_streams):
            ev = ([(torch.cuda.Event(), torch.cuda.Event()) for _ in self._apply_streams], [torch.cuda.Event() for _ in self._streams])
            self._queue_ev = ev
        return ev

    def _queue_exchange(self, exchange=True) -> None:
        """exchange() without a host wait.  Every exchange stream first waits for every local apply stream, on every GPU
        of the process: the exchange then neither sends a value still being written nor overwrites a ghost cell an
        earlier launch still reads, and across ranks the exchange signals its neighbours only after those waits.
        exchange: what _exchange_sel returned (True: every quantity, or a tuple of quantities)."""
        apply_ev, _ = self._queue_events()
        for pair, evs in zip(self._apply_streams, apply_ev):
            for st, ev in zip(pair, evs):
                ev.record(st)
        for x in self._streams:
            for evs in apply_ev:
                for ev in evs:
                    x.wait_event(ev)
        self._exchange_async(None if exchange is True else exchange)

    def _wait_exchange(self, other: "DistributedDomain", interior: bool = True) -> None:
        """Every exterior apply stream of this domain (and every interior one with interior=True) waits for the
        exchange queued last on other's exchange streams."""
        self._ensure_apply_streams()
        _, evs = other._queue_events()
        for x, ev in zip(other._streams, evs):
            ev.record(x)
        for si, se in self._apply_streams:
            for ev in evs:
                se.wait_event(ev)
                if interior:
                    si.wait_event(ev)

    # -- multigrid transfers
    def restrict_to(self, coarse: "DistributedDomain", dst, src, op=None, aux=None, exchange=True, coefs=None, face=None) -> None:
        """dst (a quantity of coarse) = the 8-cell average of src (a quantity of this domain) over every coarse compute
        cell (DESIGN.md section 2.10).  Buffers follow apply(): a bare handle means "next" for dst and "curr" for src;
        src may be curr or next, as restriction reads no ghost cells.  coarse must pair with this domain: the same
        partition dim, every subdomain exactly twice as coarse, on the same rank and GPU (sb_transfer_check; checked
        once per coarse domain).  One launch per local subdomain on the apply streams, after the work queued on the
        caller's current stream (with an op and exchange, the exchange too); returns when it is complete.  Plans are
        cached as prolong_from() describes.
            fine.restrict_to(coarse, (f2, "curr"), (r, "curr"))
        op: a StencilOp (plain terms, reach <= 1): dst = the 8-cell average of op(src, aux), the fine values never
        stored (DESIGN.md section 2.11), the same bits as apply() into a scratch quantity followed by restrict_to().
        src must then be a curr buffer, as op reads its ghost cells; aux (a bare handle means "curr") is needed when a
        term reads it.  exchange=True follows apply(): the coarse interior (the coarse compute region cut by 1, which
        reads no fine ghost cell) runs while exchange() fills the ghost cells, then the exterior slabs; exchange=False:
        one launch over the whole region, the caller guarantees the ghost cells; exchange="reads": only src and the
        coefficient fields the op reads at a non-zero offset are exchanged.  The op is part of the plan key.
            fine.restrict_to(coarse, (f2, "curr"), u, op=residual, aux=(f, "curr"))   # f2 = R (f - A u)
        An op with coefficient terms takes coefs, as apply() does (op.ncoef DataHandles of this domain, curr buffers,
        exchanged like src); the result is the bits of apply() into a scratch quantity followed by restrict_to()
        (sb_transfer_voplan_create; DESIGN.md section 2.12).
        face=a (0, 1 or 2): src holds values on the faces normal to axis a (C_a(p) on the face between p - e_a and p, as
        div_grad's coefficient field a), and dst = the average of the four fine faces that make up each coarse face
        (sb_transfer_fplan_create); no op.
            fine.restrict_to(coarse, (kx2, "curr"), (kx, "curr"), face=0)"""
        if face is not None:
            if op is not None or aux is not None or coefs is not None:
                raise _lib.StencilError("restrict_to: a face restriction takes no op, aux or coefs")
            if int(face) not in (0, 1, 2):
                raise _lib.StencilError(f"restrict_to: face {face!r} must be the axis 0, 1 or 2")
            self._transfer(coarse, _lib.TRANSFER_RESTRICT, dst, src, None, False, face=int(face))
        elif op is None:
            if aux is not None or coefs is not None:
                raise _lib.StencilError("restrict_to: aux and coefs are read only by an op")
            self._transfer(coarse, _lib.TRANSFER_RESTRICT, dst, src, None, False)
        else:
            self._transfer(coarse, _lib.TRANSFER_RESTRICT, dst, src, aux, exchange, op, coefs=coefs)

    def prolong_from(self, coarse: "DistributedDomain", dst, src, aux=None, exchange=True) -> None:
        """dst = aux + P src (or P src without aux) over every fine compute cell, P the trilinear interpolation from the
        coarse grid (DESIGN.md section 2.10).  dst and aux are quantities of this domain (bare handles: "next" and
        "curr"); aux may be dst, which gives the in-place correction u <- u + P e.  src is a quantity of coarse and must
        be a curr buffer: its ghost cells are read.  exchange=True runs coarse.exchange() first (collective: every rank
        calls it), with exchange=False the caller guarantees the coarse ghost cells, exchange="reads" exchanges the coarse
        src only (coarse.exchange(only=[src])).  The exchange and the launches are ordered after the work queued on the
        caller's current stream, and the call returns when they are complete.  The coarse radius must be >= 1 in
        all 26 directions.  Plans are built on first use and kept, per (coarse domain, kind, buffers, the swap parity
        of both domains), until close().
            fine.prolong_from(coarse, (u, "curr"), (e, "curr"), aux=(u, "curr"))"""
        self._transfer(coarse, _lib.TRANSFER_PROLONG, dst, src, aux, exchange)

    def _transfer(self, coarse, kind: int, dst, src, aux, exchange, op=None, queued: bool = False, coefs=None, face=None) -> None:
        """restrict_to / prolong_from, through _run_plans; queued: no host wait, for a solver that owns the cycle; coefs:
        the fine coefficient quantities of a coefficient op; face: the axis of a face restriction."""
        from .stencil_op import StencilOp

        name = "restrict_to" if kind == _lib.TRANSFER_RESTRICT else "prolong_from"
        if not isinstance(coarse, DistributedDomain) or coarse is self:
            raise _lib.StencilError(f"{name}: coarse must be another DistributedDomain, not {coarse!r}")
        if self.partition_ is None or not self._plans or coarse.partition_ is None or not coarse._plans:
            raise _lib.StencilError(f"{name}: call realize() on both domains first")
        restrict = kind == _lib.TRANSFER_RESTRICT
        dst_dom, src_dom = (coarse, self) if restrict else (self, coarse)

        def buf(dom, arg, default, role):
            h, which = (arg, default) if isinstance(arg, DataHandle) else tuple(arg)
            if not isinstance(h, DataHandle) or which not in ("curr", "next") or not 0 <= h.id < len(dom.dtypes_):
                raise _lib.StencilError(f"{name}: {role} must be a DataHandle of the {'coarse' if dom is coarse else 'fine'} domain "
                                        f"or (DataHandle, 'curr' | 'next'), not {arg!r}")
            return h.id, which

        d = buf(dst_dom, dst, "next", "dst")
        s = buf(src_dom, src, "curr", "src")
        a = buf(self, aux, "curr", "aux") if aux is not None else None
        dtype = dst_dom.dtypes_[d[0]]
        if src_dom.dtypes_[s[0]] != dtype or (a is not None and self.dtypes_[a[0]] != dtype) or bc_dtype(dtype) == 0:
            raise _lib.StencilError(f"{name}: dst, src and aux must all be float32 or all float64")
        if not restrict and s[1] != "curr":
            raise _lib.StencilError(f"{name}: src must be a curr buffer (the one coarse.exchange() fills)")
        c_q = []
        if op is not None:
            if not isinstance(op, StencilOp):
                raise _lib.StencilError(f"{name}: op must be a StencilOp, not {op!r}")
            cs = list(coefs) if coefs is not None else []
            if len(cs) != op.ncoef:
                raise _lib.StencilError(f"{name}: the op reads {op.ncoef} coefficient fields, but {len(cs)} were given")
            for k, c in enumerate(cs):
                q = buf(self, c, "curr", f"coefficient {k}")
                if q[1] != "curr" or self.dtypes_[q[0]] != dtype:
                    raise _lib.StencilError(f"{name}: coefficient {k} must be a curr buffer (the one exchange() fills) of the quantities' type")
                c_q.append(q[0])
            if op.dtype != dtype:
                raise _lib.StencilError(f"{name}: the op computes in {op.dtype}, the quantities are {dtype}")
            if s[1] != "curr":
                raise _lib.StencilError(f"{name}: with an op, src must be a curr buffer (the one exchange() fills)")
            if op.has_aux and a is None:
                raise _lib.StencilError(f"{name}: the op has a term on aux, but no aux buffer was given")
            op.check(self.radius_)
            a = a if op.has_aux else None
        self._check_pairing(coarse, not restrict)
        if restrict:
            exchange = self._exchange_sel(name, exchange, [s[0]] + op_moved_coefs(op, c_q)) if op is not None else False
        else:
            exchange = coarse._exchange_sel(name, exchange, [s[0]])
        fused_exchange = op is not None and bool(exchange)
        key = (coarse, kind, d, s, a, self._parity, coarse._parity) + ((op.key(), fused_exchange, tuple(c_q)) if op is not None else ())
        if face is not None:
            key += (("face", face),)
        plans = self._transfer_plans.get(key)
        if plans is None:
            plans = []
            if op is not None:
                one = Radius.constant(1).c27()
                boxes = list(zip(coarse.get_interior(one), coarse.get_exterior(one))) if fused_exchange else None
            for di, (fd, cd) in enumerate(zip(self.domains_, coarse.domains_)):
                dd, sd = (cd, fd) if restrict else (fd, cd)
                if op is not None:
                    args = (fd.gpu(), op, cd.pitched(*d), cd.accessor_origin(), cd.raw_size()[2], fd.pitched(*s), fd.accessor_origin(),
                            fd.raw_size()[2], fd.pitched(*a) if a is not None else None)
                    K = [fd.pitched(q, "curr") for q in c_q]
                    if fused_exchange:
                        plans.append((TransferPlan.fused(*args, [boxes[di][0]], K), TransferPlan.fused(*args, boxes[di][1], K)))
                    else:
                        plans.append((TransferPlan.fused(*args, [cd.get_compute_region()], K),))
                    continue
                lo, hi = dd.get_compute_region()
                if face is not None:
                    plans.append((TransferPlan.face(fd.gpu(), dtype, face, dd.pitched(*d), dd.accessor_origin(), dd.raw_size()[2], sd.pitched(*s),
                                                    sd.accessor_origin(), sd.raw_size()[2], lo, hi),))
                    continue
                plans.append((TransferPlan(fd.gpu(), dtype, kind, dd.pitched(*d), dd.accessor_origin(), dd.raw_size()[2], sd.pitched(*s),
                                           sd.accessor_origin(), sd.raw_size()[2], fd.pitched(*a) if a is not None else None, lo, hi),))
            self._transfer_plans[key] = plans
        if not restrict and exchange:
            if not queued:  # the coarse exchange waits for coarse's apply streams, which are this domain's only in a solver
                coarse._follow_caller()
            coarse._queue_exchange(exchange)
            self._wait_exchange(coarse)
        self._run_plans(plans, exchange if fused_exchange else False, queued)

    def _check_pairing(self, coarse, ghosts: bool) -> None:
        """The pairing of sb_transfer_check over every subdomain index (global information, so every rank reaches the same
        verdict), plus the same owner rank and GPU for every index; ghosts: prolongation's coarse radius as well."""
        if (coarse, ghosts) in self._paired:
            return
        fp, cp = self.partition_, coarse.partition_
        if fp.dim != cp.dim:
            raise _lib.StencilError(f"transfer: the fine partition is {fp.dim} subdomains, the coarse one {cp.dim}: they must be the same")
        idx = fp.indices()
        transfer_check(fp.dim, cp.dim, [fp.subdomain_origin(i) for i in idx], [fp.subdomain_size(i) for i in idx],
                       [cp.subdomain_origin(i) for i in idx], [cp.subdomain_size(i) for i in idx], coarse.radius_ if ghosts else None)
        for i in idx:
            if self._owner[i] != coarse._owner[i]:
                raise _lib.StencilError(f"transfer: subdomain {i} belongs to rank / slot {self._owner[i]} on the fine level and "
                                        f"{coarse._owner[i]} on the coarse one")
        for i, fd, cd in zip(self.domain_idx_, self.domains_, coarse.domains_):
            if fd.gpu() != cd.gpu():
                raise _lib.StencilError(f"transfer: subdomain {i} is on GPU {fd.gpu()} on the fine level and GPU {cd.gpu()} on the coarse one")
        self._paired.add((coarse, ghosts))

    def close(self) -> None:
        for plans in self._transfer_plans.values():
            for per_dom in plans:
                for p in per_dom:
                    p.destroy()
        self._transfer_plans = {}
        self._paired = set()
        for plans in self._stencil_plans.values():
            for per_dom in plans:
                for p in per_dom:
                    p.destroy()
        self._stencil_plans = {}
        self._apply_streams = []
        for plans in self._reduce_plans.values():
            for p in plans:
                p.destroy()
        self._reduce_plans = {}
        for plans in self._krylov_plans.values():
            for p in plans:
                p.destroy()
        self._krylov_plans = {}
        subset = [plans for per_key in self._subset_plans.values() for plans in per_key if plans is not None]
        for plans in self._plans + getattr(self, "_unpack_plans", []) + self._bc_plans + subset:
            for p in plans:
                if p is not None:
                    p.destroy()
        self._plans, self._unpack_plans, self._bc_plans, self._subset_plans = [], [], [], {}

        if self._remote is not None:
            self._remote.close()
            self._remote = None
        if getattr(self, "_nccl", None) is not None:
            self._nccl.close()
            self._nccl = None
        # staging buffers: only after every peer has unmapped them (barrier inside RemoteDomains.close)
        for ptr in getattr(self, "_recv_local", {}).values():
            lib().sb_free(C.c_void_p(ptr), self.domains_[0].gpu() if self.domains_ else 0)
        self._recv_local = {}
        for d in self.domains_:
            d.free()
        self.domains_ = []


def wait_queued(doms: Sequence[DistributedDomain]) -> None:
    """Return when the work queued on the apply and exchange streams of every domain in doms is complete: the one host
    wait that ends a public operator call and a Multigrid cycle.  Apply streams that several domains share (a solver's
    levels) are waited for once."""
    for s in dict.fromkeys(s for dd in doms for pair in dd._apply_streams for s in pair):
        s.synchronize()
    for dd in doms:
        for x in dd._streams:
            x.synchronize()


# ------------------------------------------------------------------------------------------ jacobi helpers
def _set_current_device(dev: int) -> None:
    """LocalDomain::set_device: kernels launched on a stream need that stream's device to be current."""
    import torch

    if torch.cuda.current_device() != dev:
        torch.cuda.set_device(dev)


def jacobi3d(d: LocalDomain, h: DataHandle, region: Tuple[Vec, Vec], compute_region: Tuple[Vec, Vec], stream=None) -> None:
    """One application of the reference's stencil_kernel (bin/jacobi3d.cu:40-85) to `region` of
    subdomain d: reads curr, writes next."""
    _set_current_device(d.gpu())
    check(
        lib().sb_jacobi3d(
            d.next_data(h.id),
            d.curr_data(h.id),
            d.elem_size(h.id),
            i3(d.accessor_origin()),
            i3(region[0]),
            i3(region[1]),
            i3(compute_region[0]),
            i3(compute_region[1]),
            stream_ptr(stream),
        )
    )


def fill(d: LocalDomain, h: DataHandle, region: Tuple[Vec, Vec], value: float, which: str = "curr", stream=None) -> None:
    """init_kernel (bin/jacobi3d.cu:18-29)."""
    _set_current_device(d.gpu())
    check(
        lib().sb_fill(d.pitched(h.id, which), d.elem_size(h.id), i3(d.accessor_origin()), i3(region[0]), i3(region[1]), float(value), stream_ptr(stream))
    )
