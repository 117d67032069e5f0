"""CPU-side checks of the product's C ABI: the library loads, exports every symbol the header declares,
and its host-side geometry / partition logic agrees with the reference-generated golden vectors and the
oracle.  No GPU compute is invoked here."""
import ctypes as C
import json
import os
import re

import pytest

import stencil_b200 as sb
from oracle import geometry as g
from stencil_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_geometry.json")))


def radius27(tab):
    r = sb.Radius()
    i = 0
    for z in (-1, 0, 1):
        for y in (-1, 0, 1):
            for x in (-1, 0, 1):
                r.set_dir((x, y, z), tab[i])
                i += 1
    return r


RADII = {k: radius27(v) for k, v in GOLD["radii"].items()}


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "stencil_b200.h")).read()
    declared = set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"sb_status"}
    assert len(declared) >= 30
    L = C.CDLL(sb.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(L, name), name
    # and the ctypes table covers exactly the header
    assert declared == set(_lib._SIGS), declared ^ set(_lib._SIGS)
    assert sb.lib().sb_version() == 2


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libstencil_b200.so")
    with pytest.raises(sb.StencilError):
        _lib.lib()


def test_radius_constructors():
    assert list(sb.Radius.constant(3).c27()) == GOLD["radii"]["c3"]
    assert list(sb.Radius.face_edge_corner(2, 1, 0).c27()) == GOLD["radii"]["f2e1"]
    assert list(sb.Radius.face_edge_corner(3, 2, 1).c27()) == GOLD["radii"]["f3e2c1"]
    r = sb.Radius.constant(0)
    r.set_face(1)
    assert r == sb.Radius.face_edge_corner(1, 0, 0)


def test_halo_geometry_vs_reference():
    for c in GOLD["halo"]:
        sz, r = tuple(c["size"]), RADII[c["radius"]]
        for d in c["dirs"]:
            dv = tuple(d["dir"])
            assert list(sb.halo_pos(dv, sz, r, True)) == d["pos_halo"]
            assert list(sb.halo_pos(dv, sz, r, False)) == d["pos_interior"]
            assert list(sb.halo_extent(dv, sz, r)) == d["extent"]
    for c in GOLD["local_domain"]:
        assert list(sb.raw_size(tuple(c["size"]), RADII[c["radius"]])) == c["raw_size"]


def test_bad_direction_is_an_error():
    with pytest.raises(sb.StencilError):
        sb.halo_pos((2, 0, 0), (4, 4, 4), sb.Radius.constant(1), True)


def test_prime_factors_vs_reference():
    for n, f in GOLD["prime_factors"].items():
        assert sb.prime_factors(int(n)) == f


def test_partitions_vs_reference():
    for c in GOLD["node_partition"]:
        p = sb.Partition(tuple(c["size"]), RADII[c["radius"]], c["nodes"], c["gpus"])
        assert list(p.sys_dim) == c["sys_dim"] and list(p.node_dim) == c["node_dim"]
        for s in c["subdomains"]:
            assert list(p.subdomain_size(tuple(s["idx"]))) == s["size"]
            assert list(p.subdomain_origin(tuple(s["idx"]))) == s["origin"]
    for c in GOLD["rank_partition"]:
        p = sb.Partition(tuple(c["size"]), sb.Radius.constant(0), 1, c["n"], trivial=True)
        assert list(p.dim) == c["dim"]
        for s in c["subdomains"]:
            assert list(p.subdomain_size(tuple(s["idx"]))) == s["size"]
            assert list(p.subdomain_origin(tuple(s["idx"]))) == s["origin"]


def test_interior_exterior_vs_oracle():
    L = sb.lib()
    for name, tab in GOLD["radii"].items():
        r, ro = RADII[name], g.Radius()
        i = 0
        for z in (-1, 0, 1):
            for y in (-1, 0, 1):
                for x in (-1, 0, 1):
                    ro.set_dir((x, y, z), tab[i])
                    i += 1
        for lo, hi in [((0, 0, 0), (512, 512, 512)), ((5, 0, 10), (25, 30, 50)), ((0, 0, 0), (3, 3, 3))]:
            ilo, ihi = _lib.o3(), _lib.o3()
            _lib.check(L.sb_interior(_lib.i3(lo), _lib.i3(hi), r.c27(), ilo, ihi))
            assert (_lib.t3(ilo), _lib.t3(ihi)) == g.get_interior(lo, hi, ro)
            elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
            n = _lib.check(L.sb_exterior(_lib.i3(lo), _lib.i3(hi), r.c27(), elo, ehi))
            got = [(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(n)]
            assert got == g.get_exterior(lo, hi, ro)


def test_neighbor_wrap_vs_reference():
    for p, lim, w in GOLD["wrap"]:
        assert list(sb.get_neighbor(tuple(p), (0, 0, 0), tuple(lim))) == w


def test_fused_schedule_choice_per_partition():
    """Jacobi3D picks how x faces travel in the fused schedule from the partition and the ownership table alone (every
    rank evaluates the same function): direct pushes while x stays inside a rank, dense 256-byte lines across ranks where
    the layout allows it (also on 8 ranks, where y and z faces cross ranks too), else the queued schedule."""
    from stencil_b200.domain import Partition, Radius
    from stencil_b200.jacobi import fused_x_mode

    r = Radius.face_edge_corner(1, 0, 0)

    def owners(part, per_rank):
        return {tuple(idx): (k // per_rank, k % per_rank) for k, idx in enumerate(part.indices())}

    one = Partition((512, 512, 512), r, 1, 1)
    assert fused_x_mode(one, owners(one, 1), 8, r) == "direct"
    two = Partition((1024, 512, 512), r, 1, 2)
    assert tuple(two.dim) == (2, 1, 1)
    assert fused_x_mode(two, owners(two, 2), 8, r) == "direct"  # one process x 2 GPUs: peer access
    assert fused_x_mode(two, owners(two, 1), 8, r) == "dense"  # torchrun, 2 ranks
    four = Partition((1024, 1024, 512), r, 1, 4)
    assert tuple(four.dim) == (2, 2, 1) and fused_x_mode(four, owners(four, 1), 8, r) == "dense"
    eight = Partition((1024, 1024, 1024), r, 1, 8)
    assert tuple(eight.dim) == (2, 2, 2)
    assert fused_x_mode(eight, owners(eight, 1), 8, r) == "dense"
    # 48 cells along x per rank are not whole warp strips (64 FP64 cells): never dense
    small = Partition((96, 48, 48), r, 1, 2)
    assert fused_x_mode(small, owners(small, 1), 8, r) == "queued"
    # FP32: strips of 128 cells, and 514-float rows alternate between two 16-byte phases
    assert fused_x_mode(two, owners(two, 1), 4, r) == "queued"
    # bench.py's default shapes grow along y and z only: x never crosses ranks, either precision runs the fused schedule
    for size, n, dim in (((512, 512, 1024), 2, (1, 1, 2)), ((512, 1024, 1024), 4, (1, 2, 2)), ((512, 1024, 2048), 8, (1, 2, 4))):
        part = Partition(size, r, 1, n)
        assert tuple(part.dim) == dim
        assert fused_x_mode(part, owners(part, 1), 8, r) == "direct" and fused_x_mode(part, owners(part, 1), 4, r) == "direct"


def test_ctypes_structs_match_the_header(tmp_path):
    """The Python mirrors of the C ABI structs have the size the header gives them (gcc compiles a probe against
    include/stencil_b200.h): a field added on one side only would shift every later argument silently."""
    import ctypes as C
    import os
    import subprocess

    from stencil_b200._lib import AstarothParams, BoxCopy, HaloPush, Pitched, StepSync

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "probe.c"
    src.write_text(
        '#include <stdio.h>\n#include "stencil_b200.h"\n'
        'int main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(sb_pitched), sizeof(sb_box_copy), sizeof(sb_halo_push), sizeof(sb_astaroth_params), sizeof(sb_step_sync)); return 0; }\n'
    )
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(Pitched), C.sizeof(BoxCopy), C.sizeof(HaloPush), C.sizeof(AstarothParams), C.sizeof(StepSync)]


def test_astaroth_params_field_order_matches_the_header(tmp_path):
    """sb_astaroth_params is thirteen doubles: two swapped fields keep the size, so compare each field's offset in the
    header with the product's ctypes mirror (stencil_b200._lib.AstarothParams) and the oracle's (oracle.c_oracle.AcParams)."""
    import subprocess

    from oracle.c_oracle import AcParams
    from stencil_b200._lib import AstarothParams

    names = [n for n, _ in AstarothParams._fields_]
    assert len(names) == 13
    src = tmp_path / "probe.c"
    body = "".join(f'  printf("{n} %zu\\n", offsetof(sb_astaroth_params, {n}));\n' for n in names)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "stencil_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    header = {n: int(v) for n, v in (line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())}
    assert len(header) == 13
    for struct in (AstarothParams, AcParams):
        assert {n: getattr(struct, n).offset for n, _ in struct._fields_} == header, struct
    # and the header has no field the mirrors lack: the offsets cover the whole struct
    assert sorted(header.values()) == [8 * k for k in range(13)]


def test_exchange_plan_structs_match_the_header(tmp_path):
    """sb_message and sb_staged hold only int64 fields, so a swapped pair keeps the size: compare each field's offset
    and each struct's size in the header with the ctypes mirrors, and check that the exchange-plan entry points exist."""
    import subprocess

    from stencil_b200._lib import Message, Staged

    structs = {"sb_message": Message, "sb_staged": Staged}
    body = ""
    for cname, struct in structs.items():
        body += f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));\n'
        body += "".join(f'  printf("{cname} {n} %zu\\n", offsetof({cname}, {n}));\n' for n, _ in struct._fields_)
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "stencil_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    header = {}
    for line in subprocess.check_output([str(exe)], text=True).splitlines():
        cname, field, value = line.split()
        header[(cname, field)] = int(value)
    for cname, struct in structs.items():
        assert header[(cname, "sizeof")] == C.sizeof(struct), cname
        for n, _ in struct._fields_:
            assert header[(cname, n)] == getattr(struct, n).offset, (cname, n)
    L = C.CDLL(sb.LIB_PATH)
    assert hasattr(L, "sb_exchange_messages") and hasattr(L, "sb_staging_layout")


def test_allocation_lead_rule(monkeypatch):
    """LocalDomain.lead_bytes (DESIGN.md section 1): when all rows share one 16-byte phase the allocation starts so that
    the first COMPUTE cell is 16-byte aligned; rows with alternating phase (FP32, 514 cells) keep the reference placement."""
    import numpy as np

    from stencil_b200.domain import LocalDomain, Radius

    def lead(n, r, dtype):
        d = LocalDomain((n, n, n), (0, 0, 0), 0)
        d.set_radius(Radius.constant(r))
        d.add_data(dtype)
        return d.lead_bytes(np.dtype(dtype).itemsize)

    assert lead(512, 1, np.float64) == 8  # row = 514 * 8 = 4112 B = 16 * 257; first compute cell 8 B in
    assert lead(512, 2, np.float64) == 0  # already aligned
    assert lead(512, 3, np.float64) == 8
    assert lead(512, 1, np.float32) == 0  # 2056 B rows alternate between two phases: no single lead helps
    assert lead(510, 1, np.float32) == 12  # 512 floats per row: one phase, first compute cell 4 B in
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    assert lead(512, 1, np.float64) == 0
