"""Integer geometry, partition and message planning of cwpearson/stencil -- CPU oracle.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Pure Python ints; every function
cites the reference file:line (relative to the reference checkout) that it restates.
Coordinates are (x, y, z) tuples everywhere, x fastest in memory.
"""
from __future__ import annotations

import functools
import itertools
from typing import Dict, Iterable, List, Sequence, Tuple

Vec = Tuple[int, int, int]

ALL_DIRS: List[Vec] = [
    (x, y, z)
    for z in (-1, 0, 1)
    for y in (-1, 0, 1)
    for x in (-1, 0, 1)
    if (x, y, z) != (0, 0, 0)
]  # iteration order of the planner loops, src/stencil.cu:330-332 (z outer, x inner)


def neg(d: Vec) -> Vec:
    return (-d[0], -d[1], -d[2])


def flatten(v: Vec) -> int:
    """Dim3::flatten, include/stencil/dim3.hpp:68."""
    return v[0] * v[1] * v[2]


# --------------------------------------------------------------------------- Radius
class Radius:
    """27 independently settable radii, include/stencil/radius.hpp:14-103.

    Stored as ``r[(dx,dy,dz)]``.  ``x(d)``/``y(d)``/``z(d)`` read the *face*
    entries (radius.hpp:25-40).
    """

    def __init__(self, table: Dict[Vec, int] | None = None):
        self.r: Dict[Vec, int] = {(x, y, z): 0 for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)}
        if table:
            self.r.update(table)

    @staticmethod
    def constant(r: int) -> "Radius":
        # radius.hpp:79-90 -- sets all 27 entries, the centre included
        out = Radius()
        for k in out.r:
            out.r[k] = r
        return out

    @staticmethod
    def face_edge_corner(face: int, edge: int, corner: int) -> "Radius":
        # radius.hpp:94-102 -- centre forced to 0
        out = Radius()
        for d in out.r:
            nz = sum(1 for c in d if c != 0)
            out.r[d] = {0: 0, 1: face, 2: edge, 3: corner}[nz]
        return out

    def dir(self, d: Vec) -> int:
        return self.r[tuple(d)]

    def set_dir(self, d: Vec, v: int) -> None:
        self.r[tuple(d)] = v

    def x(self, d: int) -> int:
        return self.r[(d, 0, 0)]

    def y(self, d: int) -> int:
        return self.r[(0, d, 0)]

    def z(self, d: int) -> int:
        return self.r[(0, 0, d)]

    def axis(self, ax: int, d: int) -> int:
        v = [0, 0, 0]
        v[ax] = d
        return self.r[tuple(v)]

    def as_list27(self) -> List[int]:
        """Flat [z+1][y+1][x+1] order = DirectionMap storage, direction_map.hpp:15,44-50."""
        return [self.r[(x, y, z)] for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


# --------------------------------------------------------------------------- halo geometry
def halo_pos(d: Vec, sz: Vec, radius: Radius, halo: bool) -> Vec:
    """LocalDomain::halo_pos, src/local_domain.cu:86-125 (allocation-relative elements)."""
    out = []
    for ax in range(3):
        rm = radius.axis(ax, -1)
        if d[ax] == 1:
            out.append(sz[ax] + (rm if halo else 0))
        elif d[ax] == -1:
            out.append(0 if halo else rm)
        elif d[ax] == 0:
            out.append(rm)
        else:
            raise ValueError("direction component out of range")
    return tuple(out)


def halo_extent(d: Vec, sz: Vec, radius: Radius) -> Vec:
    """LocalDomain::halo_extent, include/stencil/local_domain.cuh:212-222."""
    return tuple(sz[ax] if d[ax] == 0 else radius.axis(ax, d[ax]) for ax in range(3))


def raw_size(sz: Vec, radius: Radius) -> Vec:
    """LocalDomain::raw_size, local_domain.cuh:236-239."""
    return tuple(sz[ax] + radius.axis(ax, -1) + radius.axis(ax, 1) for ax in range(3))


def halo_bytes(d: Vec, sz: Vec, radius: Radius, elem_size: int) -> int:
    """LocalDomain::halo_bytes, local_domain.cuh:228-230."""
    return elem_size * flatten(halo_extent(d, sz, radius))


def halo_coords(d: Vec, sz: Vec, origin: Vec, radius: Radius, halo: bool) -> Tuple[Vec, Vec]:
    """LocalDomain::halo_coords, src/local_domain.cu:40-59 -> (lo, hi) in global coordinates."""
    pos = halo_pos(d, sz, radius, halo)
    ext = halo_extent(d, sz, radius)
    lo = tuple(pos[ax] - radius.axis(ax, -1) + origin[ax] for ax in range(3))
    return lo, tuple(lo[ax] + ext[ax] for ax in range(3))


def accessor_origin(origin: Vec, radius: Radius) -> Vec:
    """Origin an Accessor uses: subdomain origin minus the negative-side radius, local_domain.cuh:153-173."""
    return tuple(origin[ax] - radius.axis(ax, -1) for ax in range(3))


# --------------------------------------------------------------------------- numeric
def prime_factors(n: int) -> List[int]:
    """src/numeric.cpp:6-26 -- sorted DESCENDING."""
    out: List[int] = []
    if n == 0:
        return out
    while n % 2 == 0:
        out.append(2)
        n //= 2
    i = 3
    while i * i <= n:  # reference: i <= sqrt(n)
        while n % i == 0:
            out.append(i)
            n //= i
        i += 2
    if n > 2:
        out.append(n)
    out.sort(reverse=True)
    return out


def div_ceil(n: int, d: int) -> int:
    return (n + d - 1) // d


def next_power_of_two(x: int) -> int:
    """numeric.hpp:9-19 (for x >= 1)."""
    p = 1
    while p < x:
        p <<= 1
    return p


def next_align_of(x: int, a: int) -> int:
    """include/stencil/align.cuh:7-9."""
    return (x + a - 1) & ~(a - 1)


# --------------------------------------------------------------------------- partition
class _PartitionBase:
    size_: Vec  # base (ceil) subdomain size
    rem_: Vec

    def dim(self) -> Vec:
        raise NotImplementedError

    def subdomain_size(self, idx: Vec) -> Vec:
        # partition.hpp:55-70 / :225-240
        out = list(self.size_)
        for ax in range(3):
            if self.rem_[ax] != 0 and idx[ax] >= self.rem_[ax]:
                out[ax] -= 1
        return tuple(out)

    def subdomain_origin(self, idx: Vec) -> Vec:
        # partition.hpp:72-86 / :242-256
        out = [self.size_[ax] * idx[ax] for ax in range(3)]
        for ax in range(3):
            if self.rem_[ax] != 0 and idx[ax] >= self.rem_[ax]:
                out[ax] -= idx[ax] - self.rem_[ax]
        return tuple(out)

    def linearize(self, idx: Vec) -> int:
        d = self.dim()
        return idx[0] + idx[1] * d[0] + idx[2] * d[1] * d[0]

    def dimensionize(self, i: int) -> Vec:
        d = self.dim()
        x = i % d[0]
        i //= d[0]
        y = i % d[1]
        i //= d[1]
        return (x, y, i)

    def all_indices(self) -> List[Vec]:
        d = self.dim()
        return [(x, y, z) for z in range(d[2]) for y in range(d[1]) for x in range(d[0])]


class RankPartition(_PartitionBase):
    """partition.hpp:20-116 -- split the longest axis by each prime factor (descending)."""

    def __init__(self, size: Vec, n: int):
        dim = [1, 1, 1]
        sz = list(size)
        for amt in prime_factors(n):
            if amt < 2:
                continue
            if sz[0] >= sz[1] and sz[0] >= sz[2]:
                ax = 0
            elif sz[1] >= sz[2]:
                ax = 1
            else:
                ax = 2
            sz[ax] = div_ceil(sz[ax], amt)
            dim[ax] *= amt
        self.dim_ = tuple(dim)
        self.size_ = tuple(sz)
        self.rem_ = tuple(size[ax] % dim[ax] for ax in range(3))

    def dim(self) -> Vec:
        return self.dim_


class NodePartition(_PartitionBase):
    """partition.hpp:120-256 -- two-level (nodes, then gpus) split along the smallest radius-weighted interface."""

    def __init__(self, size: Vec, radius: Radius, nodes: int, gpus: int):
        sz = list(size)

        def split(count: int) -> Vec:
            dim = [1, 1, 1]
            for amt in prime_factors(count):
                if amt < 2:
                    continue
                x_if = sz[1] * sz[2] * (radius.dir((1, 0, 0)) + radius.dir((-1, 0, 0)))
                y_if = sz[0] * sz[2] * (radius.dir((0, 1, 0)) + radius.dir((0, -1, 0)))
                z_if = sz[0] * sz[1] * (radius.dir((0, 0, 1)) + radius.dir((0, 0, -1)))
                if x_if <= y_if and x_if <= z_if:
                    ax = 0
                elif y_if <= z_if:
                    ax = 1
                else:
                    ax = 2
                sz[ax] = div_ceil(sz[ax], amt)
                dim[ax] *= amt
            return tuple(dim)

        self.sys_dim_ = split(nodes)
        self.node_dim_ = split(gpus)
        self.size_ = tuple(sz)
        d = self.dim()
        self.rem_ = tuple(size[ax] % d[ax] for ax in range(3))

    def sys_dim(self) -> Vec:
        return self.sys_dim_

    def node_dim(self) -> Vec:
        return self.node_dim_

    def dim(self) -> Vec:
        return tuple(self.sys_dim_[ax] * self.node_dim_[ax] for ax in range(3))


# --------------------------------------------------------------------------- topology
def wrap(v: Vec, lims: Vec) -> Vec:
    """Dim3::wrap, dim3.hpp:208-229."""
    return tuple(v[ax] % lims[ax] for ax in range(3))


def get_neighbor(index: Vec, d: Vec, extent: Vec) -> Vec:
    """Topology::get_neighbor with PERIODIC boundary, src/topology.cpp:5-18."""
    return wrap(tuple(index[ax] + d[ax] for ax in range(3)), extent)


# --------------------------------------------------------------------------- messages / packer layout
def dir_less(a: Vec, b: Vec) -> bool:
    """Dim3::operator< -- lexicographic x, y, z; dim3.hpp:70-86."""
    return a < b  # python tuple order is the same lexicographic order


def sort_messages_by_size(msgs: Iterable[Tuple[Vec, Vec]]) -> List[Tuple[Vec, Vec]]:
    """Message::by_size, tx_common.hpp:25-36.  msgs = [(dir, ext)]; larger ext.flatten() first, ties by dir."""

    def cmp(l, r):
        fl, fr = flatten(l[1]), flatten(r[1])
        if fl > fr:
            return -1
        if fl < fr:
            return 1
        if l[0] < r[0]:
            return -1
        if r[0] < l[0]:
            return 1
        return 0

    return sorted(msgs, key=functools.cmp_to_key(cmp))


def packer_layout(sz: Vec, radius: Radius, elem_sizes: Sequence[int], msgs: Sequence[Tuple[Vec, Vec]]):
    """DevicePacker::prepare + launch_pack_kernels, src/packer.cu:66-148.

    msgs: [(dir, sort_ext)] -- ``sort_ext`` is the Message's ext_ (only used for ordering;
    tests pass (0,0,0), the planner passes the receiver's halo extent).
    Returns (total_bytes, entries) with entries = [dict(dir, q, offset, pos, ext, nbytes)] in wire
    order.  ``pos`` is the *pack source* position (interior side of ``dir``), ``ext`` the halo
    extent in ``-dir``.

    Wire format = the HOST-side offset walk (packer.cu:72-81, :137-141), which is what defines
    size(): before each quantity ``offset = next_align_of(offset, elem_size)``, then
    ``offset += elem_size * ext.flatten()``.  The device kernel (dev_packer_pack_domain,
    packer.cu:10-26) restarts its own walk at 0 relative to the unaligned message start; the two
    agree whenever every message ends on a boundary aligned for the first quantity (always true
    for same-typed quantities -- every case the reference tests or benchmarks).  Where they
    differ the reference kernel would issue misaligned accesses, so the host walk is the
    intended semantics and the one pinned by the golden size 264 (test_cuda_packer.cu:96-97).
    """
    ordered = sort_messages_by_size(msgs)
    entries = []
    size = 0
    for d, _ in ordered:
        pos = halo_pos(d, sz, radius, False)
        ext = halo_extent(neg(d), sz, radius)
        for q, es in enumerate(elem_sizes):
            size = next_align_of(size, es)
            nbytes = es * flatten(ext)
            entries.append(dict(dir=d, q=q, offset=size, pos=pos, ext=ext, nbytes=nbytes))
            size += nbytes
    return size, entries


def unpacker_layout(sz: Vec, radius: Radius, elem_sizes: Sequence[int], msgs: Sequence[Tuple[Vec, Vec]]):
    """DeviceUnpacker::prepare + launch_unpack_kernels, src/packer.cu:178-253.  Same wire order;
    ``pos`` is the halo position on the ``-dir`` side of the receiving domain."""
    total, entries = packer_layout(sz, radius, elem_sizes, msgs)
    for e in entries:
        nd = neg(e["dir"])
        e["pos"] = halo_pos(nd, sz, radius, True)
        e["ext"] = halo_extent(nd, sz, radius)
    return total, entries


# --------------------------------------------------------------------------- planner
def plan_sends(dim: Vec, sizes: Dict[Vec, Vec], radius: Radius):
    """The message plan of DistributedDomain::realize, src/stencil.cu:327-412, for ALL subdomains.

    Returns a list of dicts(src_idx, dst_idx, dir, src_pos, dst_pos, ext):  the source region is the
    interior side of ``dir`` in src; the destination is the halo on the ``-dir`` side of dst; the
    extent is the receiver's halo extent in ``-dir`` (stencil.cu:361-363).  A direction is skipped
    when radius.dir(-dir) == 0 (stencil.cu:344).
    """
    plan = []
    for idx in [(x, y, z) for z in range(dim[2]) for y in range(dim[1]) for x in range(dim[0])]:
        for d in ALL_DIRS:
            if radius.dir(neg(d)) == 0:
                continue
            dst = get_neighbor(idx, d, dim)
            ext = halo_extent(neg(d), sizes[dst], radius)
            if flatten(ext) == 0:
                # packer.cu:122-124 makes a zero-sized message fatal; the planner never creates one
                # when the face radii are consistent with the edge/corner radii.
                continue
            plan.append(
                dict(
                    src_idx=idx,
                    dst_idx=dst,
                    dir=d,
                    src_pos=halo_pos(d, sizes[idx], radius, False),
                    dst_pos=halo_pos(neg(d), sizes[dst], radius, True),
                    ext=ext,
                )
            )
    return plan


# --------------------------------------------------------------------------- interior / exterior
def get_interior(lo: Vec, hi: Vec, radius: Radius) -> Tuple[Vec, Vec]:
    """DistributedDomain::get_interior for one subdomain, src/stencil.cu:878-921.
    (lo, hi) = the subdomain's compute region in global coordinates."""
    ilo, ihi = list(lo), list(hi)
    for d in ALL_DIRS:
        r = radius.dir(d)
        for ax in range(3):
            if d[ax] < 0:
                ilo[ax] = max(lo[ax] + r, ilo[ax])
            elif d[ax] > 0:
                ihi[ax] = min(hi[ax] - r, ihi[ax])
    return tuple(ilo), tuple(ihi)


def get_exterior(lo: Vec, hi: Vec, radius: Radius) -> List[Tuple[Vec, Vec]]:
    """DistributedDomain::get_exterior for one subdomain, src/stencil.cu:927-977:
    slabs peeled in the order +x, +y, +z, -x, -y, -z, each against the already-shrunk box."""
    ilo, ihi = get_interior(lo, hi, radius)
    clo, chi = list(lo), list(hi)
    out = []
    for ax in range(3):  # +x, +y, +z
        if ihi[ax] != chi[ax]:
            slo = list(clo)
            slo[ax] = ihi[ax]
            out.append((tuple(slo), tuple(chi)))
            chi[ax] = ihi[ax]
    for ax in range(3):  # -x, -y, -z
        if ilo[ax] != clo[ax]:
            shi = list(chi)
            shi[ax] = ilo[ax]
            out.append((tuple(clo), tuple(shi)))
            clo[ax] = ilo[ax]
    return out


def make_block_dim(extent: Vec, threads: int) -> Vec:
    """Dim3::make_block_dim, dim3.hpp:233-254."""
    threads = min(threads, 1024)
    x = min(threads, next_power_of_two(extent[0]))
    threads //= x
    y = min(threads, next_power_of_two(extent[1]))
    threads //= y
    z = min(threads, next_power_of_two(extent[2]))
    return (min(x, 1024), min(y, 1024), min(z, 64))


def jacobi_scaled_size(x: int, y: int, z: int, num_subdoms: int) -> Vec:
    """Weak-scaling size rule of bin/jacobi3d.cu:189-199 (single node): multiply the prime factors of
    the subdomain count into the currently smallest dimension."""
    for pf in prime_factors(num_subdoms):
        if x <= y and x <= z:
            x *= pf
        elif y <= z:
            y *= pf
        else:
            z *= pf
    return (x, y, z)
