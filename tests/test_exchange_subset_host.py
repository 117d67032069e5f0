"""CPU tests of the quantity-subset exchange (DESIGN.md section 2.15): the planner's subset staging layout
(sb_staging_layout_subset) is the full layout filtered by quantity, at the full layout's offsets and total, for 1 to 8
subdomains, uneven partitions, periodic and walled axes and asymmetric radii (the full layout itself is checked against
the staging rule by test_exchange_plan.py); the planner's and DistributedDomain.exchange's refusals; the quantities exchange="reads" moves for
each kind of call; and a gloo world of 2 and 4 ranks refusing ranks that pass different subsets."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch.distributed as td
import torch.multiprocessing as mp

import stencil_b200 as sb
from stencil_b200 import _lib
from stencil_b200.domain import grid_args, op_moved_coefs, quantity_mask
from stencil_b200.multigrid import residual_op
from test_exchange_plan import BOUNDARIES, CASES, ELEM_SIZES, RADII, grid, staging_layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = (1 << 64) - 1


def subset_layout(part, topo, r, src, dst, elem_sizes, mask, cap=None):
    cap = 26 * len(elem_sizes) if cap is None else cap
    out, total = (_lib.Staged * max(cap, 1))(), C.c_int64(-1)
    n = _lib.check(sb.lib().sb_staging_layout_subset(*grid_args(part, topo, r), _lib.i3(src), _lib.i3(dst),
                                                     (C.c_int64 * len(elem_sizes))(*elem_sizes), len(elem_sizes), mask, out, cap,
                                                     C.byref(total)))
    return total.value, out, n


@pytest.mark.parametrize("walls", list(BOUNDARIES))
@pytest.mark.parametrize("rname", list(RADII))
@pytest.mark.parametrize("size,n", CASES)
def test_subset_layout_is_the_full_layout_filtered(size, n, rname, walls):
    part, topo, r, sends = grid(size, n, rname, walls)
    for es in ELEM_SIZES:
        nq = len(es)
        masks = [1 << q for q in range(nq)] + [(1 << nq) - 1, 0b101 & ((1 << nq) - 1) or 1]
        for src in part.indices():
            for dst in {m["dst_idx"] for m in sends if m["src_idx"] == src}:
                total, full = staging_layout(part, topo, r, src, dst, list(es))
                for mask in masks:
                    t, out, k = subset_layout(part, topo, r, src, dst, list(es), mask)
                    assert t == total  # the full buffers serve every subset
                    assert [(s.msg, s.q, s.offset) for s in out[:k]] == [e for e in full if (mask >> e[1]) & 1]


def test_subset_layout_refusals():
    part, topo, r, _ = grid((12, 10, 14), 8, "c1", "PPF")
    L = sb.lib()
    es = (C.c_int64 * 2)(4, 8)
    out, total = (_lib.Staged * 64)(), C.c_int64()

    def call(mask):
        return L.sb_staging_layout_subset(*grid_args(part, topo, r), _lib.i3((0, 0, 0)), _lib.i3((1, 0, 0)), es, 2, mask, out, 64, C.byref(total))

    def error():
        return L.sb_last_error().decode()

    assert call(0) == -1 and "empty" in error()  # SB_ERR_INVALID
    assert call(0b100) == -1 and "quantity 2 is not one of the 2 quantities" in error()
    assert call(1 << 63) == -1 and "quantity 63 is not one of the 2 quantities" in error()
    assert call(0b11) >= 0 and call(ALL) >= 0


def domain(nq=4):
    dd = sb.DistributedDomain(16, 16, 16)
    hs = [dd.add_data(np.float64, f"q{i}") for i in range(nq)]
    return dd, hs


def test_exchange_key_and_refusals():
    dd, hs = domain()
    assert dd.exchange_key(None) is None
    assert dd.exchange_key([hs[2], hs[0]]) == (0, 2)
    assert dd.exchange_key(hs[::-1]) is None  # every quantity: the full exchange
    assert quantity_mask((0, 2)) == 0b101 and quantity_mask(None) == ALL
    with pytest.raises(sb.StencilError, match="names no quantity"):
        dd.exchange_key([])
    with pytest.raises(sb.StencilError, match=r"quantity 1 \(q1\) is named twice"):
        dd.exchange_key([hs[1], hs[1]])
    other, ohs = domain()
    with pytest.raises(sb.StencilError, match="not a DataHandle of this domain"):
        dd.exchange_key([ohs[0]])
    with pytest.raises(sb.StencilError, match="not a DataHandle of this domain"):
        dd.exchange_key([sb.DataHandle(7, np.float64)])
    with pytest.raises(sb.StencilError, match="sequence of DataHandles"):
        dd.exchange_key(hs[0])
    with pytest.raises(sb.StencilError, match="call realize"):
        dd.exchange(only=[hs[0]])
    big, bhs = domain(70)
    assert big.exchange_key([bhs[5]]) == (5,)
    with pytest.raises(sb.StencilError, match="quantities 0..63"):
        big.exchange_key([bhs[65]])


def test_read_sets():
    """exchange="reads" moves src and the fields read at a non-zero offset, per kind of call."""
    dd, hs = domain(8)
    sel = lambda reads: dd._exchange_sel("apply", "reads", reads)  # noqa: E731
    u, k = 0, [4, 5, 6]
    lap = sb.StencilOp.laplacian(2, (1.0, 1.0, 1.0), np.float64)
    dg = sb.StencilOp.div_grad((1.0, 1.0, 1.0), np.float64).scaled(-1.0)
    assert op_moved_coefs(lap, []) == []  # plain
    assert sel([u] + op_moved_coefs(lap, [])) == (0,)
    assert op_moved_coefs(dg, k) == [4, 5, 6]  # coefficient: every field is read at p + e_a
    assert op_moved_coefs(lap.relax(1.0), []) == []  # coloured
    assert op_moved_coefs(residual_op(dg), k) == [4, 5, 6]  # fused residual-restriction and diagonal relaxation
    cell = sb.StencilOp([(0, (0, 0, 0), 1.0, 0, (0, 0, 0)), (0, (1, 0, 0), 1.0, 1, (1, 0, 0))], np.float64)
    assert op_moved_coefs(cell, [4, 5]) == [5]  # a field read at offset 0 only stays put
    curl = sb.StencilSystem.curl(-1, (1.0, 1.0, 1.0), np.float64)
    assert curl.moved_inputs() == {0, 1, 2}
    ident = sb.StencilSystem([(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)], np.float64, nin=6)
    assert (ident + curl).moved_inputs() == {0, 1, 2}
    assert sel([]) is False  # nothing read at an offset: no exchange
    assert sel(list(range(8))) is True  # everything: the full exchange
    assert dd._exchange_sel("apply", True, [0]) is True and dd._exchange_sel("apply", False, [0]) is False
    assert dd._exchange_sel("apply", None, [0]) is False and dd._exchange_sel("apply", 1, [0]) is True  # by truth, as before
    import pickle

    assert pickle.loads(pickle.dumps(hs[0])).id == 0  # handles stay picklable
    with pytest.raises(sb.StencilError, match="exchange must be True, False or 'reads'"):
        dd._exchange_sel("apply", "all", [0])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_q):
    try:
        sys.path.insert(0, ROOT)
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        td.init_process_group("gloo", rank=rank, world_size=world)
        import stencil_b200 as sb

        dd = sb.DistributedDomain(16, 16, 16)
        dd.set_gpus([0])
        hs = [dd.add_data(np.float32) for _ in range(3)]
        dd.do_placement()  # no GPU needed
        dd._agree_on_subset(dd.exchange_key([hs[0], hs[2]]))  # the same subset everywhere: agreed, once
        dd._agree_on_subset(dd.exchange_key([hs[0], hs[2]]))  # cached: no collective call
        try:
            dd._agree_on_subset(dd.exchange_key([hs[rank % 2]]))
            out_q.put((rank, "FAIL: a mismatched subset was accepted"))
        except sb.StencilError as e:
            out_q.put((rank, "ok" if "every rank must pass the same subset" in str(e) else f"FAIL: {e}"))
        td.barrier()
        td.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        out_q.put((rank, "FAIL: " + traceback.format_exc()))


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_must_pass_the_same_subset(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(r, "ok") for r in range(world)], results
