"""One-process-per-GPU plumbing for DistributedDomain (torch.distributed = rendezvous only).

The reference reaches colocated ranks through CUDA IPC memory/event handles shipped over MPI
(include/stencil/tx_cuda.cuh:225-315, src/tx_ipc.cpp, src/tx_colocated.cu).  Here the handles travel
once, at realize(), through torch.distributed.all_gather_object; after that the data path is the
same fused kernel as in the single-process case, storing into IPC-mapped ghost cells over NVLink,
and completion is a pair of device-side flags per neighbour (ready / done) -- no host barrier and no
NCCL call inside exchange().

Protocol of exchange number e on rank A with neighbour ranks N(A):
    begin :  for B in N(A): ready[B][A] = e      (A's ghost cells may be overwritten for e)
             wait  ready[A][B] >= e for B in N(A)
    copy  :  fused halo write into every neighbour (one launch per local subdomain)
    finish:  for B in N(A): done[B][A] = e        (release, system scope, after the copy)
             wait  done[A][B] >= e for B in N(A)
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Dict, List, Tuple

from ._lib import Pitched, check, lib, stream_ptr

Vec = Tuple[int, int, int]


@dataclass
class World:
    rank: int
    size: int
    local_device: int


def world() -> World:
    try:
        import torch.distributed as td

        if td.is_available() and td.is_initialized():
            rank, size = td.get_rank(), td.get_world_size()
            local = int(os.environ.get("LOCAL_RANK", rank))
            return World(rank, size, local)
    except ImportError:
        pass
    return World(0, 1, 0)


def all_gather_object(obj):
    import torch.distributed as td

    out = [None] * td.get_world_size()
    td.all_gather_object(out, obj)
    return out


class RemoteDomains:
    """IPC mappings of every other rank's allocations + the flag mailboxes."""

    def __init__(self, dd, w: World):
        self.w = w
        self.dev = dd.domains_[0].gpu()
        self._opened: List[int] = []
        n = w.size
        # my mailbox: ready[0..n), done[0..n), then step[0..n) (iteration counters of the fused jacobi schedule)
        p = C.c_void_p()
        check(lib().sb_malloc(C.byref(p), 3 * n * 4, self.dev))
        check(lib().sb_memset(p, 0, 3 * n * 4, self.dev, None))
        check(lib().sb_device_sync(self.dev))
        self.flags = int(p.value)

        def export(ptr: int) -> bytes:
            buf = (C.c_char * 64)()
            check(lib().sb_ipc_export(C.c_void_p(ptr), buf))
            return bytes(buf)

        mine = {
            "rank": w.rank,
            "flags": export(self.flags),
            "recv": {key: export(ptr) for key, ptr in dd._recv_local.items()},
            "domains": {
                dd.domain_idx_[i]: {
                    "raw": d.raw_size(),
                    "elem_sizes": list(d.elem_sizes_),
                    # (handle of the cudaMalloc block, offset of the allocation inside it): LocalDomain.lead_bytes
                    "curr": [(export(d._base_of[p_]), p_ - d._base_of[p_]) for p_ in d.curr_],
                    "next": [(export(d._base_of[p_]), p_ - d._base_of[p_]) for p_ in d.next_],
                }
                for i, d in enumerate(dd.domains_)
            },
        }
        everyone = all_gather_object(mine)

        def open_(handle: bytes) -> int:
            out = C.c_void_p()
            check(lib().sb_ipc_import(handle, self.dev, C.byref(out)))
            self._opened.append(int(out.value))
            return int(out.value)

        self.remote: Dict[Vec, dict] = {}
        self.peer_flags: Dict[int, int] = {}
        self.recv: Dict[tuple, int] = {}  # (src_idx, dst_idx) -> staging buffer in the DST rank's memory
        for info in everyone:
            r = info["rank"]
            if r == w.rank:
                continue
            self.peer_flags[r] = open_(info["flags"])
            for key, h in info["recv"].items():
                if dd._owner[tuple(key[0])][0] == w.rank:  # only buffers one of my subdomains writes into
                    self.recv[(tuple(key[0]), tuple(key[1]))] = open_(h)
            for idx, dom in info["domains"].items():
                self.remote[tuple(idx)] = {
                    "raw": tuple(dom["raw"]),
                    "elem_sizes": dom["elem_sizes"],
                    "curr": [open_(h) + off for h, off in dom["curr"]],
                    "next": [open_(h) + off for h, off in dom["next"]],
                }
        # neighbour ranks: owners of any subdomain adjacent to one of mine (periodic, symmetric)
        from .domain import ALL_DIRS, get_neighbor

        nbrs = set()
        for idx in dd.domain_idx_:
            for d in ALL_DIRS:
                nbrs.add(dd._owner[get_neighbor(idx, d, dd.partition_.dim)][0])
        nbrs.discard(w.rank)
        self.nbrs = sorted(nbrs)
        k = len(self.nbrs)
        self._ready_remote = (C.c_void_p * max(k, 1))(*[self.peer_flags[b] + 4 * w.rank for b in self.nbrs])
        self._done_remote = (C.c_void_p * max(k, 1))(*[self.peer_flags[b] + 4 * (n + w.rank) for b in self.nbrs])
        # local slots to poll, gathered contiguously is not possible (slots are indexed by rank), so wait per slot list
        self._ready_local = [self.flags + 4 * b for b in self.nbrs]
        self._done_local = [self.flags + 4 * (n + b) for b in self.nbrs]
        self._step_remote = (C.c_void_p * max(k, 1))(*[self.peer_flags[b] + 4 * (2 * n + w.rank) for b in self.nbrs])
        self._step_local = [self.flags + 4 * (2 * n + b) for b in self.nbrs]
        # iteration counter of the fused jacobi schedule: lives with the mailboxes (not with a Jacobi3D object) so that
        # the values only ever grow; every rank advances it in lockstep (one per fused iteration)
        self.step_epoch = 0

    def step_slots(self, ranks):
        """(slots in MY mailbox written by `ranks`, my slot in each of their mailboxes) for the in-kernel handshake of
        sb_jacobi3d_fused_sync."""
        n, me = self.w.size, self.w.rank
        return [self.flags + 4 * (2 * n + b) for b in ranks], [self.peer_flags[b] + 4 * (2 * n + me) for b in ranks]

    def pitched(self, idx: Vec, q: int, parity: int) -> Tuple[Pitched, int]:
        dom = self.remote[tuple(idx)]
        base = dom["curr" if parity == 0 else "next"][q]
        return Pitched(base, dom["raw"][0] * dom["elem_sizes"][q], dom["raw"][1]), -1

    def _wait_all(self, slots: List[int], value: int, stream) -> None:
        # contiguous runs of slots are waited on by one kernel
        i = 0
        while i < len(slots):
            j = i
            while j + 1 < len(slots) and slots[j + 1] == slots[j] + 4:
                j += 1
            check(lib().sb_wait(C.c_void_p(slots[i]), j - i + 1, value, self.dev, stream_ptr(stream)))
            i = j + 1

    def begin(self, epoch: int, streams) -> None:
        if not self.nbrs:
            return
        s = streams[0]
        check(lib().sb_signal(self._ready_remote, len(self.nbrs), epoch, self.dev, stream_ptr(s)))
        self._wait_all(self._ready_local, epoch, s)
        # other local streams (several subdomains per rank) start after the handshake
        if len(streams) > 1:
            import torch

            ev = torch.cuda.Event()
            ev.record(s)
            for o in streams[1:]:
                o.wait_event(ev)

    def finish(self, epoch: int, streams) -> None:
        if not self.nbrs:
            return
        s = streams[0]
        if len(streams) > 1:
            import torch

            for o in streams[1:]:
                ev = torch.cuda.Event()
                ev.record(o)
                s.wait_event(ev)
        check(lib().sb_signal(self._done_remote, len(self.nbrs), epoch, self.dev, stream_ptr(s)))
        self._wait_all(self._done_local, epoch, s)

    def raw_of(self, idx: Vec) -> Vec:
        return tuple(self.remote[tuple(idx)]["raw"])

    def signal_step(self, value: int, stream) -> None:
        """Tell every neighbour rank that this rank's iteration `value` has finished (stream-ordered)."""
        if self.nbrs:
            check(lib().sb_signal(self._step_remote, len(self.nbrs), value, self.dev, stream_ptr(stream)))

    def wait_step(self, value: int, stream) -> None:
        """Hold `stream` until every neighbour rank has finished iteration `value`."""
        if self.nbrs:
            self._wait_all(self._step_local, value, stream)

    def close(self) -> None:
        import torch.distributed as td

        # nobody may unmap while a peer could still be writing
        if td.is_initialized():
            td.barrier()
        for p in self._opened:
            lib().sb_ipc_close(C.c_void_p(p), self.dev)
        self._opened = []
        if td.is_initialized():
            td.barrier()
        if self.flags:
            lib().sb_free(C.c_void_p(self.flags), self.dev)
            self.flags = 0


def share_domains(dd, w: World) -> RemoteDomains:
    return RemoteDomains(dd, w)


# --------------------------------------------------------------------------------------------- NCCL fallback
def messages_from(dd, src_rank: int) -> List[dict]:
    """The send plan of ANY rank (pure geometry: every rank can compute every other rank's plan)."""
    from .domain import ALL_DIRS, get_neighbor, halo_extent, halo_pos

    part, radius = dd.partition_, dd.radius_
    out = []
    for idx in part.indices():
        rank, slot = dd._owner[idx]
        if rank != src_rank:
            continue
        sz = part.subdomain_size(idx)
        for d in ALL_DIRS:
            nd = (-d[0], -d[1], -d[2])
            if radius.dir(nd) == 0:
                continue
            dst_idx = get_neighbor(idx, d, part.dim)
            dst_sz = part.subdomain_size(dst_idx)
            ext = halo_extent(nd, dst_sz, radius)
            if ext[0] * ext[1] * ext[2] == 0:
                continue
            out.append(
                dict(src_idx=idx, src_slot=slot, dst_idx=dst_idx, dst_rank=dd._owner[dst_idx][0], dst_slot=dd._owner[dst_idx][1], dir=d,
                     src_pos=halo_pos(d, sz, radius, False), dst_pos=halo_pos(nd, dst_sz, radius, True), ext=ext)
            )
    return out


STAGE_MAX_ROW_BYTES = 64


def staging_layout(dd, src_idx, dst_idx):
    """Messages from subdomain src_idx to subdomain dst_idx (on a DIFFERENT GPU) whose rows are shorter than
    STAGE_MAX_ROW_BYTES (x-faces, x-edges, corners): storing such rows straight into the peer's ghost cells costs one
    tiny NVLink transaction per row (1.6 M 8-byte remote stores per exchange on two GPUs, and a much slower
    interior kernel), so the sender packs them into ONE dense receive buffer in the peer's memory (contiguous 128-byte
    NVLink packets) and the receiver scatters them locally.  Pure geometry: both sides compute the same layout.
    Returns (total_bytes, [dict(dir, q, offset, ext, src_pos, dst_pos, es)])."""
    es = [int(e) for e in dd._elem_sizes()]
    entries, off = [], 0
    src_rank = dd._owner[tuple(src_idx)][0]
    for m in messages_from(dd, src_rank):
        if tuple(m["src_idx"]) != tuple(src_idx) or tuple(m["dst_idx"]) != tuple(dst_idx):
            continue
        n = m["ext"][0] * m["ext"][1] * m["ext"][2]
        for q, e in enumerate(es):
            if m["ext"][0] * e >= STAGE_MAX_ROW_BYTES:
                continue
            off = (off + 15) & ~15
            entries.append(dict(dir=m["dir"], q=q, offset=off, ext=m["ext"], src_pos=m["src_pos"], dst_pos=m["dst_pos"], es=e))
            off += n * e
    return off, entries


def wire_order(msgs: List[dict]) -> List[dict]:
    """Sender and receiver agree on one order per (src rank -> dst rank) buffer: larger messages first, ties by
    (src subdomain, direction) -- Message::by_size of the reference (tx_common.hpp:25-36) extended to several
    subdomains per rank."""
    return sorted(msgs, key=lambda m: (-(m["ext"][0] * m["ext"][1] * m["ext"][2]), m["src_idx"], m["dir"]))


class NcclExchange:
    """Fallback transport where CUDA IPC / peer mapping between two ranks' GPUs is unavailable (or when forced with
    SB_FORCE_NCCL=1): pack -> ncclSend/ncclRecv (torch.distributed P2P ops, one group per exchange) -> unpack, with the
    reference's packed wire format (src/packer.cu: per message, per quantity, offset aligned to the element size).
    This is the analogue of the reference's CudaAwareMpiSender/Recver (tx_cuda.cuh:769-930); it costs two extra HBM
    passes per halo byte compared with the fused direct write and is never used when P2P works."""

    def __init__(self, dd, w: World):
        import torch

        from .domain import CopyPlan, box_copy

        self.dd, self.w = dd, w
        self.dev = dd.domains_[0].gpu()
        es = [d for d in dd.domains_[0].elem_sizes_]

        def layout(msgs):
            off, entries = 0, []
            for m in wire_order(msgs):
                n = m["ext"][0] * m["ext"][1] * m["ext"][2]
                for q, e in enumerate(es):
                    off = (off + e - 1) & ~(e - 1)
                    entries.append((m, q, off))
                    off += n * e
            return off, entries

        mine = messages_from(dd, w.rank)
        self.peers = sorted({m["dst_rank"] for m in mine} - {w.rank})
        self.send_buf, self.recv_buf, self.pack, self.unpack = {}, {}, {}, {}
        for b in self.peers:
            out_total, out_entries = layout([m for m in mine if m["dst_rank"] == b])
            in_total, in_entries = layout([m for m in messages_from(dd, b) if m["dst_rank"] == w.rank])
            self.send_buf[b] = torch.empty(max(out_total, 1), dtype=torch.uint8, device=f"cuda:{self.dev}")
            self.recv_buf[b] = torch.empty(max(in_total, 1), dtype=torch.uint8, device=f"cuda:{self.dev}")
            self.pack[b], self.unpack[b] = [], []
            for parity in (0, 1):
                pk, up = [], []
                for m, q, off in out_entries:
                    d = dd.domains_[m["src_slot"]]
                    src = Pitched((d._curr0 if parity == 0 else d._next0)[q], d.raw_size()[0] * es[q], d.raw_size()[1])
                    dense = Pitched(self.send_buf[b].data_ptr() + off, m["ext"][0] * es[q], m["ext"][1])
                    pk.append(box_copy(dense, (0, 0, 0), src, m["src_pos"], m["ext"], es[q]))
                for m, q, off in in_entries:
                    d = dd.domains_[m["dst_slot"]]
                    dst = Pitched((d._curr0 if parity == 0 else d._next0)[q], d.raw_size()[0] * es[q], d.raw_size()[1])
                    dense = Pitched(self.recv_buf[b].data_ptr() + off, m["ext"][0] * es[q], m["ext"][1])
                    up.append(box_copy(dst, m["dst_pos"], dense, (0, 0, 0), m["ext"], es[q]))
                self.pack[b].append(CopyPlan(self.dev, pk))
                self.unpack[b].append(CopyPlan(self.dev, up))
        self.bytes_per_exchange = sum(t.numel() for t in self.send_buf.values())

    def exchange(self, parity: int, stream) -> None:
        import torch
        import torch.distributed as td

        with torch.cuda.stream(stream):
            for b in self.peers:
                self.pack[b][parity].launch(stream)
            ops = []
            for b in self.peers:
                ops.append(td.P2POp(td.isend, self.send_buf[b], b))
                ops.append(td.P2POp(td.irecv, self.recv_buf[b], b))
            if ops:
                for r in td.batch_isend_irecv(ops):
                    r.wait()
            for b in self.peers:
                self.unpack[b][parity].launch(stream)

    def close(self) -> None:
        for plans in list(self.pack.values()) + list(self.unpack.values()):
            for p in plans:
                p.destroy()
        self.pack, self.unpack = {}, {}
