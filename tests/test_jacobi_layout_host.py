"""The GPU layout sweep (tests/test_gpu_jacobi_layouts.py) reaches every branch of the jacobi launch decisions, in every dtype
where the branch exists.  Runs without a GPU: it evaluates the host-side restatement in tests/jacobi_layout.py over the
GPU case lists, so a later edit of those lists cannot silently drop a layout."""
import pytest

import jacobi_layout as jl

DT = {4: "float32", 8: "float64"}

# FP64 has no 8-byte pairs, and no overhang: its 16-byte vectors are aligned to the row's own phase and a row of 16-byte
# multiples, so the last vector holding compute cells ends at most at the first ghost cell.  (FP32: 4 cells per vector,
# 1 ghost cell.)
SWEEP_WANT = {
    4: {"cell", "phase0", "phase", "shift", "pairs", "scalar", "overhang", "tail_lane", "tail_lane0"},
    8: {"cell", "phase0", "phase", "shift", "scalar", "tail_lane", "tail_lane0"},
}
FUSED_WANT = {
    4: {"phase0", "phase", "shift", "pairs", "scalar", "overhang", "tail_lane", "tail_lane0", "x_wrap", "x_self_push", "y_wrap", "y_self_push",
        "z_wrap", "x_dense", "all_null", "column", "column_with_x_push"},
    8: {"phase0", "phase", "shift", "scalar", "tail_lane", "tail_lane0", "x_wrap", "x_self_push", "y_wrap", "y_self_push", "z_wrap", "x_dense",
        "all_null"},
}


@pytest.mark.parametrize("es", [4, 8], ids=DT.get)
def test_sweep_reaches_every_vector_branch(es):
    got = set()
    for c in jl.sweep_cases():
        if c.es == es:
            got |= jl.sweep_case_branches(c)
    assert got == SWEEP_WANT[es], sorted(got ^ SWEEP_WANT[es])
    print(f"{DT[es]} sb_jacobi3d branches covered: {sorted(got)}")


def test_sweep_has_every_lead_ghost_width_and_both_row_parities():
    cases = jl.sweep_cases()
    for es in (4, 8):
        mine = [c for c in cases if c.es == es]
        assert {c.s_lead for c in mine if c.s_lead == c.d_lead} == set(jl.LEADS[es])
        assert any(c.s_lead != c.d_lead for c in mine)
        assert {c.ghost for c in mine} == set(jl.GHOSTS)
        assert {c.ny % 2 for c in mine} == {0, 1} and {(c.ny + 2 * c.ghost) % 2 for c in mine} == {0, 1}
        assert {c.nx for c in mine} == set(jl.SWEEP_NX)
        # every strip multiple has a neighbour on each side
        for strip in (64, 128):
            assert {strip - 2, strip - 1, strip, strip + 1, strip + 2} <= {c.nx for c in mine}


@pytest.mark.parametrize("es", [4, 8], ids=DT.get)
def test_fused_cases_reach_every_branch(es):
    got = set()
    for c in jl.fused_cases():
        if c.es == es:
            got |= jl.fused_case_branches(c)
    assert got == FUSED_WANT[es], sorted(got ^ FUSED_WANT[es])
    print(f"{DT[es]} sb_jacobi3d_fused branches covered: {sorted(got)}")


def test_fused_cases_cover_the_configurations_and_chunks():
    cases = jl.fused_cases()
    for es in (4, 8):
        mine = [c for c in cases if c.es == es]
        assert {c.config for c in mine} == {"self", "null", "cut_x", "cut_y", "cut_z", "dense_x"}
        for c in mine:
            if c.axis is not None:  # unequal sizes along the cut
                assert c.sizes[0][c.axis] != c.sizes[1][c.axis], c.id()
        assert any(c.leads[0] != c.leads[1] for c in mine if len(c.sizes) == 2)
        nz = {s[2] for c in mine for s in c.sizes}
        assert 1 in nz and any(z % 8 for z in nz if z > 8)  # one-plane subdomains and partial z chunks
        ny = {s[1] for c in mine for s in c.sizes}
        assert 1 in ny and any(y % 8 for y in ny if y > 8)


def test_the_suspected_overhang_layout_is_in_the_fused_cases():
    """FP32, lead 12, nx = 2 (mod 4): the last vector holding compute cells hangs one element over its row, so the launch must
    take the scalar path (pick_vectors) rather than give that lane a stand-in load."""
    pl = jl.fused_plan(4, 12, 12, (130, 17, 33), ("self",) * 6)
    assert (pl.vx, pl.kind) == (1, "overhang")
    assert any(c.es == 4 and (130, 17, 33) in c.sizes and c.leads[0] == (12, 12) for c in jl.fused_cases())


def test_a_tail_lane_that_would_be_lane_0_takes_the_scalar_path():
    """FP64, lead 8, nx = 2 (mod 64): the vector after the last compute cell hangs over the row, and the one before it is lane
    0 of a strip, whose edge scalar is its left neighbour -- march_body's tail_lane cannot serve it.  Both launchers take
    the scalar path, and the sweep and the DistributedDomain test run that layout."""
    for nx in (66, 130):
        assert jl.pick_vectors(8, 8, (nx + 2) * 8, (nx + 2) * 8 * 10, 8, 1, nx + 1, nx + 2) == (1, 1, "tail_lane0")
    assert jl.pick_vectors(8, 8, 514 * 8, 514 * 8 * 514, 8, 1, 513, 514)[:2] == (2, 1)  # 512^3 keeps its vectors (lane 31)
    assert any(c.es == 8 and c.nx in (66, 130) and c.s_lead == 8 for c in jl.sweep_cases())


@pytest.mark.parametrize("name", sorted(jl.FUSED_ERRORS))
def test_fused_error_cases_hit_their_error(name):
    es, lead, size, dense = jl.FUSED_ERROR_CASES[name]
    nbr = ("null",) * 6 if not any(dense) else ("other", "other", "self", "self", "self", "self")
    assert jl.fused_plan(es, lead, lead, size, nbr, dense).error == name
