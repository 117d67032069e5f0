"""CPU oracle of non-periodic grids and their boundary conditions (BCs), on top of oracle/geometry.py and
oracle/np_oracle.py: the message plan with per-axis periodicity, the exchange it performs, and the per-cell BC rule of
include/stencil_b200.h applied literally in numpy, in the quantity's dtype.

Faces are numbered 0..5 = -x, +x, -y, +y, -z, +z; kinds are 0 NONE, 1 VALUE, 2 EVEN, 3 ODD (sb_bc_kind)."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

from oracle import geometry as g
from oracle import np_oracle as no

Vec = Tuple[int, int, int]
NONE, VALUE, EVEN, ODD = 0, 1, 2, 3
PERIODIC = (True, True, True)


def get_neighbor(idx: Vec, d: Vec, dim: Vec, periodic: Sequence[bool] = PERIODIC):
    """Topology::get_neighbor with one boundary per axis: None when the step leaves the grid along a walled axis."""
    out = []
    for a in range(3):
        v = idx[a] + d[a]
        if periodic[a]:
            v %= dim[a]
        elif not 0 <= v < dim[a]:
            return None
        out.append(v)
    return tuple(out)


def plan_sends(dim: Vec, sizes: Dict[Vec, Vec], radius: g.Radius, periodic: Sequence[bool] = PERIODIC):
    """oracle.geometry.plan_sends with per-axis periodicity: no message crosses a wall."""
    plan = []
    for idx in [(x, y, z) for z in range(dim[2]) for y in range(dim[1]) for x in range(dim[0])]:
        for d in g.ALL_DIRS:
            if radius.dir(g.neg(d)) == 0:
                continue
            dst = get_neighbor(idx, d, dim, periodic)
            if dst is None:
                continue
            ext = g.halo_extent(g.neg(d), sizes[dst], radius)
            if g.flatten(ext) == 0:
                continue
            plan.append(dict(src_idx=idx, dst_idx=dst, dir=d, src_pos=g.halo_pos(d, sizes[idx], radius, False),
                             dst_pos=g.halo_pos(g.neg(d), sizes[dst], radius, True), ext=ext))
    return plan


class Domains(no.Domains):
    """np_oracle.Domains with a periodic flag per axis (default: periodic everywhere)."""

    def __init__(self, size, radius, dtypes, n_subdomains=1, partition="node", periodic: Sequence[bool] = PERIODIC):
        super().__init__(size, radius, dtypes, n_subdomains, partition)
        self.periodic = tuple(bool(p) for p in periodic)

    def exchange(self) -> int:
        moved = 0
        for m in plan_sends(self.dim, self.sizes, self.radius, self.periodic):
            for q in range(len(self.dtypes)):
                no.translate(self.arrays[m["dst_idx"]][q], m["dst_pos"], self.arrays[m["src_idx"]][q], m["src_pos"], m["ext"])
                moved += self.dtypes[q].itemsize * g.flatten(m["ext"])
        return moved

    def expected_after_exchange(self, fn, idx: Vec, q: int) -> np.ndarray:
        """As on a periodic grid, except that ghost cells beyond a wall (global coordinate outside the grid along a
        walled axis) keep the poison: no message reaches them."""
        out = super().expected_after_exchange(fn, idx, q)
        sz, org = self.sizes[idx], self.origins[idx]
        raw = g.raw_size(sz, self.radius)
        ao = g.accessor_origin(org, self.radius)
        outside = np.zeros(raw[::-1], dtype=bool)
        for a in range(3):
            if self.periodic[a]:
                continue
            c = np.arange(ao[a], ao[a] + raw[a])
            bad = (c < 0) | (c >= self.size[a])
            shape = [1, 1, 1]
            shape[2 - a] = raw[a]
            outside |= bad.reshape(shape)
        out[outside] = no.poison(self.dtypes[q])
        return out

    def wall_kinds(self, idx: Vec, q: int, bcs) -> Tuple[List[int], List[float]]:
        """(kinds, values) per face of subdomain idx for quantity q; NONE where the face is not a wall of idx."""
        kinds, values = [NONE] * 6, [0.0] * 6
        for (qq, f), (kind, c) in bcs.items():
            a, s = f // 2, (1 if f % 2 else -1)
            d = [0, 0, 0]
            d[a] = s
            if qq == q and get_neighbor(idx, tuple(d), self.dim, self.periodic) is None:
                kinds[f], values[f] = kind, c
        return kinds, values


def face_of(a: int, s: int) -> int:
    return 2 * a + (1 if s > 0 else 0)


def bc_regions(size: Vec, radius: g.Radius, kinds: Sequence[int]) -> List[dict]:
    """The regions a subdomain's BCs write, in direction order z, y, x ascending: dict(dir, pos, ext, mirror, faces)."""
    out = []
    for d in g.ALL_DIRS:
        if radius.dir(d) == 0:
            continue
        faces = 0
        for a in range(3):
            if d[a] and kinds[face_of(a, d[a])] != NONE:
                faces |= 1 << face_of(a, d[a])
        if not faces:
            continue
        pos, ext = g.halo_pos(d, size, radius, True), g.halo_extent(d, size, radius)
        if g.flatten(ext) == 0:
            continue
        mirror = []
        for a in range(3):
            if d[a] and faces & (1 << face_of(a, d[a])):
                gm = radius.axis(a, -1)
                mirror.append(2 * gm - 1 if d[a] < 0 else 2 * (gm + size[a]) - 1)
            else:
                mirror.append(-1)
        out.append(dict(dir=d, pos=pos, ext=ext, mirror=tuple(mirror), faces=faces))
    return out


def check_widths(size: Vec, radius: g.Radius, kinds: Sequence[int]) -> None:
    """EVEN and ODD need a ghost width no larger than the subdomain on that axis."""
    for f, k in enumerate(kinds):
        a, s = f // 2, (1 if f % 2 else -1)
        if k in (EVEN, ODD) and radius.axis(a, s) > size[a]:
            raise ValueError(f"face {f}: ghost width {radius.axis(a, s)} > {size[a]}")


def apply_regions(arr: np.ndarray, size: Vec, radius: g.Radius, kinds: Sequence[int], values: Sequence[float]) -> None:
    """The per-cell rule on one allocation: v = arr at the mirrored source (as the exchange left it), then the wall
    faces in order x, y, z -- VALUE v = T(c), EVEN v, ODD v = 2 T(c) - v -- in the array's dtype."""
    T = arr.dtype.type
    src_arr = arr.copy()
    raw = arr.shape[::-1]
    for reg in bc_regions(size, radius, kinds):
        pos, ext, mir = reg["pos"], reg["ext"], reg["mirror"]
        coords = []
        for a in range(3):
            p = np.arange(pos[a], pos[a] + ext[a])
            s = mir[a] - p if mir[a] >= 0 else p
            coords.append(np.clip(s, 0, raw[a] - 1))  # only a VALUE face can mirror out of the allocation; it discards v
        v = src_arr[np.ix_(coords[2], coords[1], coords[0])]
        for a in range(3):
            if mir[a] < 0:
                continue
            f = face_of(a, reg["dir"][a])
            if kinds[f] == VALUE:
                v = np.full_like(v, T(values[f]))
            elif kinds[f] == ODD:
                v = (T(2) * T(values[f]) - v).astype(arr.dtype)
        no.box(arr, pos, ext)[...] = v


def apply_boundary(domains: Domains, bcs: Dict[Tuple[int, int], Tuple[int, float]]) -> None:
    """Every subdomain's wall ghost cells after an exchange.  bcs: (quantity, face) -> (kind, value)."""
    for idx in domains.indices:
        for q, arr in enumerate(domains.arrays[idx]):
            kinds, values = domains.wall_kinds(idx, q, bcs)
            check_widths(domains.sizes[idx], domains.radius, kinds)
            apply_regions(arr, domains.sizes[idx], domains.radius, kinds, values)
