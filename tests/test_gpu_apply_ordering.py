"""An operator call reads what the caller queued on its current stream just before the call: the exchange of apply() and
of prolong_from() is ordered after that stream, not only the launches.  The caller's stream is kept busy with
torch.cuda._sleep, then stencil_b200.domain.fill overwrites every compute cell of src on that stream (the faces the
other subdomain reads included), then the call runs with exchange=True on 2 subdomains of one GPU.  An exchange that
did not wait for the caller's stream would copy the old values into the ghost cells while the stream sleeps."""
import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
import stencil_op_oracle as so
import transfer_oracle as to
from gpu_util import oracle_radius
from stencil_b200.domain import fill
from test_gpu_stencil_domain import domain, gather, heat_terms, lo_of, load, same
from test_gpu_transfer_domain import pair

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 200_000_000  # about 0.1 s of GPU clock: far longer than queueing fill() and the call on the host


def fill_on_busy_stream(dd, h, cycles=SLEEP_CYCLES):
    """Subdomain i's compute cells of h (curr) set to i + 1, queued on the caller's current stream behind a sleep; returns
    the global array that results."""
    import torch

    glob = np.empty(dd.size()[::-1], dd.dtypes_[h.id])
    torch.cuda._sleep(cycles)
    for i, d in enumerate(dd.domains()):
        lo, hi = d.get_compute_region()
        fill(d, h, (lo, hi), float(i + 1), stream=torch.cuda.current_stream())
        glob[lo[2] : hi[2], lo[1] : hi[1], lo[0] : hi[0]] = i + 1
    return glob


def warm_up(dd, h):
    """The first launch of a kernel in a process loads its module, which can wait for the work on the device and would
    end the sleep before the call: launch the sleep and fill kernels once beforehand."""
    import torch

    fill_on_busy_stream(dd, h, 1)
    torch.cuda.synchronize()


def test_apply_exchange_follows_caller_stream():
    import torch

    terms = heat_terms()
    op = sb.StencilOp(terms, np.float64)
    dd, (src, dst) = domain(2, sb.Radius.face_edge_corner(2, 0, 0), [np.float64, np.float64])
    try:
        warm_up(dd, src)
        load(dd, src.id, "curr", np.random.default_rng(2).uniform(-1, 1, dd.size()[::-1]))
        dd.apply(op, dst, src)  # builds and caches the plans, so the call below only queues
        with torch.cuda.stream(torch.cuda.Stream()):
            glob = fill_on_busy_stream(dd, src)
            dd.apply(op, dst, src, exchange=True)
        assert same(gather(dd, dst.id, "next"), so.apply_periodic(terms, glob, None))
    finally:
        dd.close()


def test_prolong_exchange_follows_caller_stream():
    import torch

    dtype = np.dtype(np.float64)
    (fd, (u, v)), (cd, (e, w)) = pair(2, dtype)
    try:
        csize = cd.size()
        warm_up(cd, e)
        load(cd, e.id, "curr", np.random.default_rng(3).uniform(-1, 1, csize[::-1]))
        fd.prolong_from(cd, v, e)  # builds and caches the plans
        with torch.cuda.stream(torch.cuda.Stream()):
            coarse = fill_on_busy_stream(cd, e)
            fd.prolong_from(cd, v, e, exchange=True)
        od = bo.Domains(csize, oracle_radius(cd.radius_), [dtype], n_subdomains=1, periodic=[True] * 3)
        rl = lo_of(cd.radius_)
        so._view(od.arrays[(0, 0, 0)][0], rl, csize, (0, 0, 0))[...] = coarse
        od.exchange()
        want = np.empty(fd.size()[::-1], dtype)
        to.prolong_box(want, (0, 0, 0), od.arrays[(0, 0, 0)][0], tuple(-r for r in rl), (0, 0, 0), fd.size())
        assert same(gather(fd, v.id, "next"), want)
    finally:
        fd.close()
        cd.close()
