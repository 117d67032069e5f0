"""Host-side restatement of the launch decisions of the jacobi kernels, and the case lists of tests/test_gpu_jacobi_layouts.py.

The functions below restate, in allocation coordinates (lo / hi / raw along x as capi.cu's to_alloc_box makes them), what the
launchers decide before a kernel marches:
  * pick_vectors                 stencil_b200/csrc/jacobi.cu pick_vectors (vector width, strip origin, the overhang fallback)
  * has_tail_lane                jacobi.cu march_body: tail_lane / xin (unshifted rows)
  * sweep_branches               jacobi.cu launch_jacobi (thin regions take the cell kernel)
  * fused_plan                   capi.cu sb_jacobi3d_fused_sync (self-neighbour wrap requests) + jacobi.cu launch_jacobi_fused
                                 (x-wrap layout rule, dense-x precondition) + launch_fused (face-group limit, tail-column tiles)
The host test (tests/test_jacobi_layout_host.py) asserts that the GPU case lists reach every branch, so the sweep stays honest
when its shapes are edited; the GPU tests use fused_plan to know which ghost faces a launch must write and which it must not.
Pointers are given by their lead: bytes after a 256-byte aligned block start, so the 16-byte phase is lead % 16.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

MAX_GROUPS = 4096  # SB_FUSED_MAX_GROUPS
THIN_X = 16  # launch_jacobi: regions narrower than this take jacobi_cell_kernel (kThinX)
FACES = ("-x", "+x", "-y", "+y", "-z", "+z")


def pick_vectors(s_lead: int, d_lead: int, pitch: int, slice_: int, es: int, lo0: int, hi0: int, raw0: int):
    """jacobi.cu pick_vectors -> (vx, x0a, kind).  kind: "phase0" / "phase" (full 16-byte vectors, rows of one phase, equal
    src and dst phase 0 / not 0), "shift" (full vectors on rows alternating between two phases), "pairs" (FP32 8-byte pairs),
    "scalar", "overhang" (unshifted vectors where the last one holding compute cells would hang over the end of its row:
    march_body would give that lane a stand-in load, so the launch takes the scalar path) or "tail_lane0" (the vector after
    the last compute cell hangs over the row and the lane before it is lane 0 of a strip, which cannot be march_body's
    tail_lane: scalar path as well)."""
    s, d = s_lead & 15, d_lead & 15
    full = 16 // es

    def origin(vx, phase):
        xal = ((16 - phase) & 15) // es % vx  # x (mod vx) of the aligned cells
        return lo0 - (lo0 - xal) % vx

    if pitch % 16 == 0 and slice_ % 16 == 0 and s == d and s % es == 0:
        vx, x0a, kind = full, origin(full, s), ("phase0" if s == 0 else "phase")
    elif s == 0 and d == 0 and slice_ % 16 == 0 and pitch % 16 == 8:
        return full, origin(full, 0), "shift"
    elif es == 4 and (s_lead | d_lead | pitch | slice_) % 8 == 0:
        vx, x0a, kind = 2, origin(2, 0), "pairs"
    else:
        return 1, lo0, "scalar"
    last = x0a + ((hi0 - 1 - x0a) // vx) * vx  # first cell of the last vector holding compute cells
    if last + vx > raw0:
        return 1, lo0, "overhang"
    if last + vx == hi0 and last + 2 * vx > raw0 and (last - x0a) // vx % 32 == 0:
        return 1, lo0, "tail_lane0"  # the tail lane would be lane 0, whose one edge scalar is its left neighbour
    return vx, x0a, kind


def has_tail_lane(vx: int, x0a: int, hi0: int, raw0: int, shift: bool) -> bool:
    """march_body tail_lane: on unshifted rows, a lane other than 31 whose vector ends at the last compute cell while the next
    lane's vector hangs over the end of the row (that lane loads a stand-in, so this one takes the ghost cell as its edge
    scalar)."""
    if shift or vx == 1 or (hi0 - x0a) % vx:
        return False
    lane = ((hi0 - x0a) // vx - 1) % 32
    return lane != 31 and hi0 + vx > raw0


def sweep_branches(es: int, s_lead: int, d_lead: int, raw: Tuple[int, int, int], lo0: int, hi0: int) -> set:
    """The branches one sb_jacobi3d launch over x range [lo0, hi0) of an allocation of raw (x, y, z) elements takes."""
    if hi0 - lo0 < THIN_X:
        return {"cell"}
    pitch = raw[0] * es
    vx, x0a, kind = pick_vectors(s_lead, d_lead, pitch, pitch * raw[1], es, lo0, hi0, raw[0])
    out = {kind}
    if has_tail_lane(vx, x0a, hi0, raw[0], kind == "shift"):
        out.add("tail_lane")
    return out


@dataclass
class FusedPlan:
    """What sb_jacobi3d_fused does with one subdomain of compute size `size`, ghost width 1 on every face."""

    error: Optional[str] = None  # "thin", "dense", "too_tall": the call returns SB_ERR_INVALID
    vx: int = 0
    x0a: int = 0
    kind: str = ""
    tail_lane: bool = False
    wrap: Tuple[bool, bool, bool] = (False, False, False)  # periodic self-neighbour read in place, per axis
    push: Tuple[bool, ...] = (False,) * 6  # the launch stores its face cells into that neighbour's ghost cells
    dense: Tuple[bool, bool] = (False, False)  # x faces travel through dense [y][z] arrays instead
    column: bool = False  # the last vector of phase-shifted rows runs as tail-column tiles (march_column)
    column_geometry: bool = False  # ... would, but the +x face is pushed, so the launcher keeps the fifth strip
    branches: set = field(default_factory=set)


def fused_plan(es: int, s_lead: int, d_lead: int, size: Tuple[int, int, int], nbr: Tuple[str, ...], x_dense: Tuple[bool, bool] = (False, False)) -> FusedPlan:
    """nbr[f] for the faces -x, +x, -y, +y, -z, +z: "self" (this subdomain's own dst), "other" (another allocation) or
    "null".  x_dense[s]: side s pushes into a dense array and reads its x ghosts from a received one (x_recv)."""
    nx, ny, nz = size
    lo = (1, 1, 1)
    hi = (nx + 1, ny + 1, nz + 1)
    raw = (nx + 2, ny + 2, nz + 2)
    pl = FusedPlan()
    if nx < 16:  # capi.cu sb_jacobi3d_fused_sync
        pl.error = "thin"
        return pl
    pitch = raw[0] * es
    pl.vx, pl.x0a, pl.kind = pick_vectors(s_lead, d_lead, pitch, pitch * raw[1], es, lo[0], hi[0], raw[0])
    vx, shift = pl.vx, pl.kind == "shift"
    pl.tail_lane = has_tail_lane(vx, pl.x0a, hi[0], raw[0], shift)
    whole_strips = pl.x0a == lo[0] and nx % (32 * vx) == 0
    # capi.cu: wrap requests for a self-neighbour on both sides of an axis; launch_jacobi_fused drops the x request when the
    # first compute cell does not open lane 0 or the last one does not close lane 31 (unshifted rows)
    xwrap = nbr[0] == "self" and nbr[1] == "self" and (shift or whole_strips)
    ywrap = nbr[2] == "self" and nbr[3] == "self" and (pitch % 16 == 0 or ny % 2 == 0)
    zwrap = nbr[4] == "self" and nbr[5] == "self"
    pl.wrap = (xwrap, ywrap, zwrap)
    pl.dense = tuple(bool(x_dense[s]) and nbr[s] != "null" for s in (0, 1))
    if any(x_dense) and not (not shift and whole_strips):  # launch_jacobi_fused: dense x arrays need the wrap's layout
        pl.error = "dense"
        return pl
    pl.push = tuple(nbr[f] != "null" and not pl.wrap[f // 2] and not (f < 2 and pl.dense[f]) for f in range(6))
    # launch_fused: face groups, then the tail-column tiles
    tiles_x = (hi[0] - pl.x0a + (vx // 2 if shift else 0) + 32 * vx - 1) // (32 * vx)
    tiles_y = (ny + 7) // 8
    across = max(tiles_x, tiles_y)
    zchunk = 8 if ((nz + 7) // 8) * across <= MAX_GROUPS else (16 if ((nz + 15) // 16) * across <= MAX_GROUPS else 32)
    zchunk = min(zchunk, nz)
    tiles_z = (nz + zchunk - 1) // zchunk
    if tiles_z * tiles_y > MAX_GROUPS or tiles_z * tiles_x > MAX_GROUPS or tiles_y * tiles_x > MAX_GROUPS:
        pl.error = "too_tall"
        return pl
    if shift and tiles_x >= 2:
        xcol = pl.x0a + (tiles_x - 1) * 32 * vx
        geometry = hi[0] - (xcol - vx // 2) <= vx and xcol - vx // 2 >= lo[0]
        pl.column = geometry and not (pl.push[1] or pl.dense[1])
        pl.column_geometry = geometry
    b = {pl.kind}
    if pl.tail_lane:
        b.add("tail_lane")
    for a, name in enumerate("xyz"):
        if pl.wrap[a]:
            b.add(f"{name}_wrap")
        elif any(nbr[2 * a + s] == "self" and pl.push[2 * a + s] for s in (0, 1)):
            b.add(f"{name}_self_push")
    if any(pl.dense):
        b.add("x_dense")
    if all(n == "null" for n in nbr):
        b.add("all_null")
    if pl.column:
        b.add("column")
    if pl.column_geometry and not pl.column:
        b.add("column_with_x_push")
    pl.branches = b
    return pl


# ------------------------------------------------------------------------------------------------ the GPU case lists
LEADS = {4: (0, 4, 8, 12), 8: (0, 8)}
# different src / dst leads: rows of one phase but two phases between the buffers
MIXED_LEADS = {4: ((0, 8), (4, 12), (12, 0)), 8: ((0, 8),)}
GHOSTS = (1, 2, 3)
# x widths: tiny (cell kernel), one strip, the 30..33 remainders, and around every FP64 (64) / FP32 (128) strip multiple
SWEEP_NX = (1, 2, 3, 5, 16, 30, 31, 32, 33, 62, 63, 64, 65, 66, 126, 127, 128, 129, 130, 131, 190, 256)


@dataclass(frozen=True)
class SweepCase:
    es: int
    s_lead: int
    d_lead: int
    nx: int
    ny: int
    nz: int
    ghost: int

    @property
    def raw(self):
        g = self.ghost
        return (self.nx + 2 * g, self.ny + 2 * g, self.nz + 2 * g)

    def x_ranges(self):
        """[lo, hi) along x of the sb_jacobi3d boxes: the compute region and boxes starting 1..3 cells later."""
        g = self.ghost
        return [(g + k, g + self.nx) for k in range(4) if k < self.nx]


def sweep_cases() -> List[SweepCase]:
    """Every (lead pair, x width, ghost width) for each dtype; ny alternates between odd and even (rows alternating between
    two 16-byte phases keep full vectors only when the slice is a multiple of 16 bytes), nz between 9 and 12."""
    out = []
    for es in (4, 8):
        pairs = [(lead, lead) for lead in LEADS[es]] + list(MIXED_LEADS[es])
        for s_lead, d_lead in pairs:
            for i, nx in enumerate(SWEEP_NX):
                for g in GHOSTS:
                    ny = 9 + (i + g) % 2  # 9 or 10 rows (+ 2g): both slice phases
                    out.append(SweepCase(es, s_lead, d_lead, nx, ny, 9 + 3 * ((i + g) % 2), g))
    return out


def sweep_case_branches(c: SweepCase) -> set:
    out = set()
    for lo0, hi0 in c.x_ranges():
        out |= sweep_branches(c.es, c.s_lead, c.d_lead, c.raw, lo0, hi0)
    return out


FUSED_NX = (16, 17, 30, 31, 32, 33, 62, 64, 66, 126, 128, 130, 192, 256)
FUSED_NY = (1, 7, 8, 9, 17)
FUSED_NZ = (1, 2, 9, 33)


@dataclass(frozen=True)
class FusedCase:
    """Subdomains of one periodic global grid, cut along `axis` (None: one subdomain).  sizes[i], leads[i] = (curr, next)."""

    es: int
    config: str  # "self", "null", "cut_x", "cut_y", "cut_z", "dense_x"
    sizes: Tuple[Tuple[int, int, int], ...]
    leads: Tuple[Tuple[int, int], ...]

    @property
    def axis(self):
        return {"cut_x": 0, "dense_x": 0, "cut_y": 1, "cut_z": 2}.get(self.config)

    @property
    def global_size(self):
        a = self.axis
        out = list(self.sizes[0])
        if a is not None:
            out[a] = sum(s[a] for s in self.sizes)
        return tuple(out)

    def origins(self):
        a, o, out = self.axis, 0, []
        for s in self.sizes:
            org = [0, 0, 0]
            if a is not None:
                org[a] = o
                o += s[a]
            out.append(tuple(org))
        return out

    def nbrs(self, i: int) -> Tuple[str, ...]:
        if self.config == "null":
            return ("null",) * 6
        a = self.axis
        return tuple("other" if (a is not None and f // 2 == a) else "self" for f in range(6))

    def plans(self, parity: int) -> List[FusedPlan]:
        """The plan of each subdomain at iteration parity 0 (src = curr) or 1 (src = next)."""
        dense = (True, True) if self.config == "dense_x" else (False, False)
        out = []
        for i, (s, (lc, ln)) in enumerate(zip(self.sizes, self.leads)):
            sl, dl = (lc, ln) if parity == 0 else (ln, lc)
            out.append(fused_plan(self.es, sl, dl, s, self.nbrs(i), dense))
        return out

    def id(self):
        sz = "+".join("x".join(str(v) for v in s) for s in self.sizes)
        ld = "+".join(f"{a}.{b}" for a, b in self.leads)
        return f"f{8 * self.es}-{self.config}-{sz}-lead{ld}"


def _dense_ok(es: int, nx: int, lead: int) -> bool:
    return fused_plan(es, lead, lead, (nx, 8, 8), ("other", "other", "self", "self", "self", "self"), (True, True)).error is None


def fused_cases() -> List[FusedCase]:
    """A fixed-seed sample of nx x ny x nz per dtype and configuration, plus the layouts that reach the rare branches."""
    rng = random.Random(20261015)
    out: List[FusedCase] = []
    for es in (4, 8):
        leads = LEADS[es]
        for config in ("self", "null", "cut_x", "cut_y", "cut_z"):
            for _ in range(7):
                nx, ny, nz = rng.choice(FUSED_NX), rng.choice(FUSED_NY), rng.choice(FUSED_NZ)
                la, lb = rng.choice(leads), rng.choice(leads)
                if config == "self" or config == "null":
                    out.append(FusedCase(es, config, ((nx, ny, nz),), ((la, la),)))
                    continue
                a = {"cut_x": 0, "cut_y": 1, "cut_z": 2}[config]
                pool = {0: FUSED_NX, 1: FUSED_NY, 2: FUSED_NZ}[a]
                s0 = [nx, ny, nz]
                s1 = list(s0)
                s1[a] = rng.choice([v for v in pool if v != s0[a]])  # unequal sizes along the cut
                out.append(FusedCase(es, config, (tuple(s0), tuple(s1)), ((la, la), (lb, lb))))
        # an x cut with dense x arrays wherever the layout allows it (FP64: lead 8; FP32: the scalar layouts, leads 4 / 12)
        dense_nx = [nx for nx in FUSED_NX if any(_dense_ok(es, nx, lead) for lead in leads)]
        for _ in range(3):
            n0, n1 = rng.sample(dense_nx, 2)
            ny, nz = rng.choice(FUSED_NY), rng.choice(FUSED_NZ)
            lead = [lead for lead in leads if _dense_ok(es, n0, lead) and _dense_ok(es, n1, lead)]
            out.append(FusedCase(es, "dense_x", ((n0, ny, nz), (n1, ny, nz)), ((lead[0], lead[-1]), (lead[-1], lead[0]))))
    # the layouts the sample may miss, each named by the branch it is there for
    out += [
        FusedCase(4, "self", ((130, 17, 33),), ((12, 12),)),  # overhang: FP32 lead 12, nx = 2 (mod 4)
        FusedCase(4, "self", ((30, 9, 9),), ((12, 12),)),  # overhang
        FusedCase(4, "cut_y", ((66, 8, 9), (66, 7, 9)), ((12, 12), (12, 12))),  # overhang with y pushes
        FusedCase(4, "self", ((32, 8, 9),), ((0, 0),)),  # SHIFT (rows of 136 B) in one strip, x wrap patched into a vector
        FusedCase(4, "self", ((128, 8, 9),), ((0, 0),)),  # SHIFT: tail-column tiles, x wrap in place
        FusedCase(4, "self", ((256, 8, 2),), ((0, 0),)),  # SHIFT: tail-column tiles, y wrap (even ny)
        FusedCase(4, "cut_x", ((128, 8, 9), (256, 8, 9)), ((0, 0), (0, 0))),  # SHIFT: tail column ruled out by the +x push
        FusedCase(4, "self", ((32, 9, 9),), ((8, 8),)),  # pairs on rows alternating in phase, y pushed (odd ny)
        FusedCase(4, "self", ((64, 9, 9),), ((8, 8),)),  # FP32 pairs (rows of 264 B, 8-byte phase)
        FusedCase(4, "self", ((126, 9, 2),), ((4, 4),)),  # FP32 phase 4, tail lane
        FusedCase(4, "self", ((128, 8, 9),), ((4, 0),)),  # scalar, mixed leads; x wrap in place (whole strips of 32)
        FusedCase(4, "null", ((62, 9, 33),), ((0, 8),)),  # pairs with mixed leads, all neighbours NULL
        FusedCase(8, "self", ((30, 9, 9),), ((8, 8),)),  # FP64 phase 8, tail lane, x pushed into its own ghosts
        FusedCase(8, "self", ((64, 8, 1),), ((8, 8),)),  # FP64 x wrap in place, one plane
        FusedCase(8, "self", ((31, 8, 9),), ((0, 0),)),  # FP64 SHIFT (rows of 264 B)
        FusedCase(8, "self", ((31, 7, 9),), ((0, 0),)),  # FP64 scalar, y pushed (odd ny: rows alternate in phase)
        FusedCase(8, "self", ((64, 17, 2),), ((0, 0),)),  # FP64 phase 0: x0a = 0, x pushed
        FusedCase(8, "null", ((33, 9, 9),), ((8, 8),)),  # FP64 scalar (rows of 280 B at an 8-byte phase)
    ]
    return out


def fused_case_branches(c: FusedCase) -> set:
    out = set()
    for parity in (0, 1):
        for pl in c.plans(parity):
            assert pl.error is None, (c.id(), pl.error)
            out |= pl.branches
    return out


# the error paths of sb_jacobi3d_fused (SB_ERR_INVALID) and the message each one must carry
FUSED_ERRORS = {
    "thin": "fused step needs at least 16 cells along x",
    "dense": "a dense received x array needs a 16-byte aligned first compute cell and whole warp strips along x",
    "too_tall": "too tall for the fused kernel's face groups",
}
FUSED_ERROR_CASES: Dict[str, Tuple[int, int, Tuple[int, int, int], Tuple[bool, bool]]] = {
    # name: (es, lead, compute size, x_dense)
    "thin": (8, 8, (15, 8, 8), (False, False)),
    "dense": (8, 8, (66, 8, 8), (True, False)),  # not whole strips of 64 doubles
    "too_tall": (4, 0, (16, 8 * 65, 32 * 64), (False, False)),  # 65 tile rows x 64 chunks of 32 planes > 4096 groups
}
