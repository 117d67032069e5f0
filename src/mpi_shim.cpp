// Node-local implementation of the MPI surface declared in include/mpi_shim/mpi.h (lib/libmpi_shim.a).
//
// A machine need not have an MPI.  This file provides the subset the reference library,
// its drivers and its tests use (SURVEY.md section 2c), for the ranks of ONE node:
//   * started directly            -> a world of one rank (the reference's 1 rank x N GPUs deployment);
//   * started by bin/sb_mpirun -n N -> N processes that share one POSIX shared-memory segment: a sense-reversing
//     barrier, one scratch slot per rank for the collectives (allgather-based), and a single-producer single-consumer
//     ring of 32 KiB fragments per ordered rank pair for point-to-point messages (tag/communicator matching and the
//     unexpected-message queue live on the receiver).  Buffers may be host or device pointers ("CUDA-aware": device
//     memory is staged through the fragments with cudaMemcpy).
// It is a control-plane transport: the halo data of stencil_b200 never travels through it (CUDA-IPC handles do, once).
// If the process was started by some OTHER launcher with more than one rank (mpirun, srun, torchrun), MPI_Init aborts
// instead of letting every rank believe it is rank 0 of 1.
#include "mpi.h"

#include <cuda_runtime_api.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <list>
#include <vector>

#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace {

constexpr uint32_t kMagic = 0x53424d50; // "SBMP"
constexpr size_t kFrag = 32 * 1024;     // bytes per point-to-point fragment
constexpr int kSlots = 8;               // fragments in flight per ordered rank pair
constexpr size_t kColl = 256 * 1024;    // collective scratch bytes per rank

struct Slot {
  int32_t tag, comm;
  uint64_t total, offset;
  uint32_t bytes, pad;
  unsigned char data[kFrag];
};
struct Chan { // src -> dst ring: head written by src, tail by dst
  alignas(64) std::atomic<uint64_t> head;
  alignas(64) std::atomic<uint64_t> tail;
  alignas(64) Slot slot[kSlots];
};
struct Header {
  uint32_t magic, size;
  alignas(64) std::atomic<uint32_t> barCount;
  alignas(64) std::atomic<uint32_t> barGen;
  alignas(64) std::atomic<uint32_t> abortFlag;
};
constexpr size_t kHeaderBytes = 4096;
static_assert(sizeof(Header) <= kHeaderBytes, "header page");

struct Req {
  bool live = false, done = false, isSend = false;
  const unsigned char *sbuf = nullptr;
  unsigned char *rbuf = nullptr;
  size_t bytes = 0, sent = 0;
  int peer = 0, tag = 0, comm = 0;
  int srcSeen = 0;
};
struct Msg { // a complete message waiting for its receive
  int src, tag, comm;
  std::vector<unsigned char> data;
};
struct SelfMsg { // a message of this rank to itself: matched by pointer (host or device memory, one direct copy)
  const unsigned char *ptr; // the user's buffer (MPI_Isend: valid until the request completes) ...
  std::vector<unsigned char> owned; // ... or a private copy (blocking MPI_Send that found no posted receive)
  size_t bytes;
  int tag, comm, reqId;
};

int g_rank = 0, g_size = 1;
bool g_init = false;
unsigned char *g_shm = nullptr;
size_t g_shmBytes = 0;
Header *g_hdr = nullptr;
std::vector<Req> g_reqs(1);                 // id 0 is MPI_REQUEST_NULL
std::vector<std::deque<int>> g_sendq;       // per destination: request ids in posting order
std::deque<int> g_recvq;                    // posted receives, in posting order
std::list<Msg> g_unexpected;                // arrived, unmatched (arrival order)
std::list<SelfMsg> g_self;                  // self-sends, unmatched (posting order)
std::vector<Msg> g_partial;                 // per source: message being assembled
std::vector<bool> g_partialOpen;
const int g_tagUb = (1 << 30) - 1;

inline size_t dt_size(MPI_Datatype dt) { return size_t(dt & 0xFF); }
inline unsigned char *coll_slot(int r) { return g_shm + kHeaderBytes + size_t(r) * kColl; }
inline Chan *chan(int src, int dst) {
  return reinterpret_cast<Chan *>(g_shm + kHeaderBytes + size_t(g_size) * kColl) + (size_t(src) * size_t(g_size) + size_t(dst));
}

[[noreturn]] void fatal(const char *msg) {
  std::fprintf(stderr, "mpi_shim[%d/%d]: %s\n", g_rank, g_size, msg);
  if (g_hdr) g_hdr->abortFlag.store(1);
  std::_Exit(70);
}

void check_abort() {
  if (g_hdr && g_hdr->abortFlag.load(std::memory_order_relaxed)) {
    std::fprintf(stderr, "mpi_shim[%d/%d]: another rank aborted\n", g_rank, g_size);
    std::_Exit(71);
  }
}

bool is_plain_host(const void *p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
    cudaGetLastError(); // no driver / unregistered memory: treat as host
    return true;
  }
  return attr.type == cudaMemoryTypeUnregistered || attr.type == cudaMemoryTypeHost;
}

void copy_any(void *dst, const void *src, size_t n) {
  if (0 == n || dst == src) return;
  if (is_plain_host(dst) && is_plain_host(src)) {
    std::memcpy(dst, src, n);
    return;
  }
  if (cudaMemcpy(dst, src, n, cudaMemcpyDefault) != cudaSuccess) fatal("cudaMemcpy of a message buffer failed");
}

int new_req() {
  for (size_t i = 1; i < g_reqs.size(); ++i)
    if (!g_reqs[i].live) {
      g_reqs[i] = Req{};
      g_reqs[i].live = true;
      return int(i);
    }
  g_reqs.push_back(Req{});
  g_reqs.back().live = true;
  return int(g_reqs.size() - 1);
}

inline bool tag_ok(int want, int have) { return want == MPI_ANY_TAG || want == have; }
inline bool src_ok(int want, int have) { return want == MPI_ANY_SOURCE || want == have; }

void deliver(Req &r, const Msg &m) {
  if (m.data.size() > r.bytes) fatal("message truncated (receive buffer smaller than the message)");
  copy_any(r.rbuf, m.data.data(), m.data.size());
  r.bytes = m.data.size();
  r.tag = m.tag;
  r.srcSeen = m.src;
  r.done = true;
}

// match posted receives (posting order) against arrived messages (arrival order) and pending self-sends
void match() {
  for (auto it = g_recvq.begin(); it != g_recvq.end();) {
    Req &r = g_reqs[size_t(*it)];
    bool hit = false;
    if (src_ok(r.peer, g_rank)) {
      for (auto m = g_self.begin(); m != g_self.end(); ++m) {
        if (m->comm == r.comm && tag_ok(r.tag, m->tag)) {
          if (m->bytes > r.bytes) fatal("message truncated (receive buffer smaller than the message)");
          copy_any(r.rbuf, m->owned.empty() ? m->ptr : m->owned.data(), m->bytes);
          r.bytes = m->bytes, r.tag = m->tag, r.srcSeen = g_rank, r.done = true;
          if (m->reqId) g_reqs[size_t(m->reqId)].done = true;
          g_self.erase(m);
          hit = true;
          break;
        }
      }
    }
    for (auto m = g_unexpected.begin(); !hit && m != g_unexpected.end(); ++m) {
      if (m->comm == r.comm && src_ok(r.peer, m->src) && tag_ok(r.tag, m->tag)) {
        deliver(r, *m);
        g_unexpected.erase(m);
        hit = true;
        break;
      }
    }
    it = hit ? g_recvq.erase(it) : std::next(it);
  }
}

// push fragments of queued sends, drain incoming fragments, match
void progress() {
  if (g_size > 1) {
    for (int dst = 0; dst < g_size; ++dst) {
      std::deque<int> &q = g_sendq[size_t(dst)];
      while (!q.empty()) {
        Req &r = g_reqs[q.front()];
        Chan *c = chan(g_rank, dst);
        bool stalled = false;
        while (r.sent < r.bytes || (0 == r.bytes && !r.done)) {
          const uint64_t head = c->head.load(std::memory_order_relaxed);
          if (head - c->tail.load(std::memory_order_acquire) >= uint64_t(kSlots)) {
            stalled = true;
            break;
          }
          Slot &s = c->slot[head % kSlots];
          const size_t n = std::min(kFrag, r.bytes - r.sent);
          s.tag = r.tag, s.comm = r.comm, s.total = r.bytes, s.offset = r.sent, s.bytes = uint32_t(n);
          copy_any(s.data, r.sbuf + r.sent, n);
          r.sent += n;
          c->head.store(head + 1, std::memory_order_release);
          if (0 == r.bytes) break;
        }
        if (stalled) break;
        r.done = true; // buffered: the user buffer may be reused
        q.pop_front();
      }
    }
    for (int src = 0; src < g_size; ++src) {
      if (src == g_rank) continue;
      Chan *c = chan(src, g_rank);
      uint64_t tail = c->tail.load(std::memory_order_relaxed);
      while (tail < c->head.load(std::memory_order_acquire)) {
        const Slot &s = c->slot[tail % kSlots];
        Msg &p = g_partial[size_t(src)];
        if (0 == s.offset) {
          p.src = src, p.tag = s.tag, p.comm = s.comm;
          p.data.assign(size_t(s.total), 0);
          g_partialOpen[size_t(src)] = true;
        }
        if (s.bytes) std::memcpy(p.data.data() + s.offset, s.data, s.bytes);
        const bool complete = s.offset + s.bytes >= s.total;
        c->tail.store(++tail, std::memory_order_release);
        if (complete) {
          g_unexpected.push_back(std::move(p));
          p = Msg{};
          g_partialOpen[size_t(src)] = false;
        }
      }
    }
  }
  match();
}

void spin_pause(unsigned &spins) {
  check_abort();
  if (++spins > 64) sched_yield();
}

void wait_req(int id) {
  unsigned spins = 0;
  while (!g_reqs[size_t(id)].done) {
    progress();
    if (g_reqs[size_t(id)].done) break;
    if (g_size == 1) fatal("waiting on a request that no other operation of this one-rank world can complete");
    spin_pause(spins);
  }
}

void barrier_world() {
  if (g_size == 1) return;
  const uint32_t gen = g_hdr->barGen.load(std::memory_order_acquire);
  if (g_hdr->barCount.fetch_add(1, std::memory_order_acq_rel) + 1 == uint32_t(g_size)) {
    g_hdr->barCount.store(0, std::memory_order_relaxed);
    g_hdr->barGen.store(gen + 1, std::memory_order_release);
    return;
  }
  unsigned spins = 0;
  while (g_hdr->barGen.load(std::memory_order_acquire) == gen) {
    progress(); // keep draining: a peer may be pushing a long message at us before it reaches the barrier
    spin_pause(spins);
  }
}

bool world_like(MPI_Comm comm) { return comm != MPI_COMM_SELF && g_size > 1; }

// every rank contributes `bytes`; all[r * bytes ..] receives rank r's contribution
void allgather_bytes(const void *mine, size_t bytes, void *all) {
  for (size_t off = 0; off < bytes || (0 == bytes && 0 == off); off += kColl) {
    const size_t n = std::min(kColl, bytes - off);
    copy_any(coll_slot(g_rank), static_cast<const unsigned char *>(mine) + off, n);
    barrier_world();
    for (int r = 0; r < g_size; ++r) copy_any(static_cast<unsigned char *>(all) + size_t(r) * bytes + off, coll_slot(r), n);
    barrier_world();
    if (0 == bytes) break;
  }
}

template <typename T> void reduce_typed(T *acc, const T *in, int count, MPI_Op op) {
  for (int i = 0; i < count; ++i) {
    if (op == MPI_SUM) acc[i] = T(acc[i] + in[i]);
    else if (op == MPI_MAX) acc[i] = in[i] > acc[i] ? in[i] : acc[i];
    else if (op == MPI_MIN) acc[i] = in[i] < acc[i] ? in[i] : acc[i];
  }
}

void reduce_into(void *acc, const void *in, int count, MPI_Datatype dt, MPI_Op op) {
  switch (dt) {
  case MPI_INT: reduce_typed(static_cast<int *>(acc), static_cast<const int *>(in), count, op); break;
  case MPI_UNSIGNED: reduce_typed(static_cast<unsigned *>(acc), static_cast<const unsigned *>(in), count, op); break;
  case MPI_FLOAT: reduce_typed(static_cast<float *>(acc), static_cast<const float *>(in), count, op); break;
  case MPI_DOUBLE: reduce_typed(static_cast<double *>(acc), static_cast<const double *>(in), count, op); break;
  case MPI_INT64_T:
  case MPI_LONG_LONG: reduce_typed(static_cast<long long *>(acc), static_cast<const long long *>(in), count, op); break;
  case MPI_UINT64_T:
  case MPI_UNSIGNED_LONG: reduce_typed(static_cast<unsigned long long *>(acc), static_cast<const unsigned long long *>(in), count, op); break;
  case MPI_BYTE:
  case MPI_CHAR: reduce_typed(static_cast<signed char *>(acc), static_cast<const signed char *>(in), count, op); break;
  default: fatal("reduction on an unsupported datatype");
  }
}

// allreduce on host copies (buffers may be device memory)
void allreduce_bytes(const void *sendbuf, void *recvbuf, int count, MPI_Datatype dt, MPI_Op op) {
  const size_t bytes = size_t(count) * dt_size(dt);
  std::vector<unsigned char> mine(bytes), all(bytes * size_t(g_size));
  copy_any(mine.data(), sendbuf == MPI_IN_PLACE ? recvbuf : sendbuf, bytes);
  allgather_bytes(mine.data(), bytes, all.data());
  std::vector<unsigned char> acc(all.begin(), all.begin() + long(bytes));
  for (int r = 1; r < g_size; ++r) reduce_into(acc.data(), all.data() + size_t(r) * bytes, count, dt, op);
  copy_any(recvbuf, acc.data(), bytes);
}

int env_int(const char *name, int dflt) {
  const char *s = std::getenv(name);
  return (s && *s) ? std::atoi(s) : dflt;
}

void init_world() {
  if (g_init) return;
  g_init = true;
  const int size = env_int("SB_MPI_SIZE", 0);
  if (size <= 1) {
    // not started by sb_mpirun: refuse to run as N independent "rank 0 of 1" worlds under a foreign launcher
    for (const char *v : {"OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "PMIX_SIZE", "SLURM_NTASKS", "WORLD_SIZE"}) {
      if (env_int(v, 1) > 1 && !std::getenv("SB_MPI_ALLOW_FOREIGN_LAUNCHER")) {
        std::fprintf(stderr, "mpi_shim: %s=%d but this binary links stencil_b200's node-local MPI shim, which only forms a "
                             "multi-rank world under bin/sb_mpirun; link a real MPI instead of lib/libmpi_shim.a for that launcher\n", v, env_int(v, 1));
        std::_Exit(72);
      }
    }
    g_rank = 0, g_size = 1;
    g_sendq.assign(1, {});
    return;
  }
  g_size = size;
  g_rank = env_int("SB_MPI_RANK", -1);
  const char *job = std::getenv("SB_MPI_JOB");
  if (g_rank < 0 || g_rank >= g_size || !job) fatal("SB_MPI_SIZE is set but SB_MPI_RANK / SB_MPI_JOB are not: start the program with bin/sb_mpirun");
  const int fd = shm_open(job, O_RDWR, 0600);
  if (fd < 0) fatal("cannot open the job's shared-memory segment");
  g_shmBytes = kHeaderBytes + size_t(g_size) * kColl + size_t(g_size) * size_t(g_size) * sizeof(Chan);
  void *p = mmap(nullptr, g_shmBytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) fatal("cannot map the job's shared-memory segment");
  g_shm = static_cast<unsigned char *>(p);
  g_hdr = reinterpret_cast<Header *>(g_shm);
  if (g_hdr->magic != kMagic || int(g_hdr->size) != g_size) fatal("shared-memory segment does not belong to this job");
  g_sendq.assign(size_t(g_size), {});
  g_partial.assign(size_t(g_size), Msg{});
  g_partialOpen.assign(size_t(g_size), false);
}

void fill_status(MPI_Status *status, const Req &r) {
  if (!status) return;
  status->MPI_SOURCE = r.isSend ? g_rank : r.srcSeen;
  status->MPI_TAG = r.tag;
  status->MPI_ERROR = MPI_SUCCESS;
  status->count_bytes_ = int(r.bytes);
}

} // namespace

// sb_mpirun needs the segment geometry
extern "C" size_t sb_mpi_shim_segment_bytes(int size) {
  return kHeaderBytes + size_t(size) * kColl + size_t(size) * size_t(size) * sizeof(Chan);
}
extern "C" void sb_mpi_shim_segment_init(void *base, int size) {
  Header *h = static_cast<Header *>(base);
  h->magic = kMagic;
  h->size = uint32_t(size);
}
extern "C" void sb_mpi_shim_segment_abort(void *base) { static_cast<Header *>(base)->abortFlag.store(1); }

extern "C" {

int MPI_Init(int *, char ***) {
  init_world();
  return MPI_SUCCESS;
}
int MPI_Init_thread(int *, char ***, int required, int *provided) {
  init_world();
  if (provided) *provided = required;
  return MPI_SUCCESS;
}
int MPI_Initialized(int *flag) {
  *flag = g_init ? 1 : 0;
  return MPI_SUCCESS;
}
int MPI_Finalize(void) {
  if (g_size > 1) barrier_world(); // nobody unmaps while a peer still drains its channels
  return MPI_SUCCESS;
}
int MPI_Abort(MPI_Comm, int errorcode) {
  if (g_hdr) g_hdr->abortFlag.store(1);
  std::_Exit(errorcode ? errorcode : 1);
}

int MPI_Comm_rank(MPI_Comm comm, int *rank) {
  init_world();
  *rank = comm == MPI_COMM_SELF ? 0 : g_rank;
  return MPI_SUCCESS;
}
int MPI_Comm_size(MPI_Comm comm, int *size) {
  init_world();
  *size = comm == MPI_COMM_SELF ? 1 : g_size;
  return MPI_SUCCESS;
}
int MPI_Comm_split_type(MPI_Comm comm, int, int, MPI_Info, MPI_Comm *newcomm) {
  // one node: the shared-memory communicator has the membership (and rank order) of its parent; collective, so every
  // rank draws the same id
  static int next = 16;
  *newcomm = comm == MPI_COMM_SELF ? MPI_COMM_SELF : next++;
  return MPI_SUCCESS;
}
int MPI_Comm_free(MPI_Comm *comm) {
  *comm = MPI_COMM_NULL;
  return MPI_SUCCESS;
}
int MPI_Comm_get_attr(MPI_Comm, int keyval, void *attribute_val, int *flag) {
  if (keyval == MPI_TAG_UB) {
    *reinterpret_cast<const int **>(attribute_val) = &g_tagUb;
    *flag = 1;
  } else {
    *flag = 0;
  }
  return MPI_SUCCESS;
}
int MPI_Get_processor_name(char *name, int *resultlen) {
  if (0 != gethostname(name, MPI_MAX_PROCESSOR_NAME - 1)) std::strcpy(name, "localhost");
  name[MPI_MAX_PROCESSOR_NAME - 1] = 0;
  *resultlen = int(std::strlen(name));
  return MPI_SUCCESS;
}

double MPI_Wtime(void) {
  using clk = std::chrono::steady_clock;
  static const clk::time_point t0 = clk::now();
  return std::chrono::duration<double>(clk::now() - t0).count();
}
int MPI_Barrier(MPI_Comm comm) {
  init_world();
  if (world_like(comm)) barrier_world();
  return MPI_SUCCESS;
}

int MPI_Isend(const void *buf, int count, MPI_Datatype dt, int dest, int tag, MPI_Comm comm, MPI_Request *req) {
  init_world();
  if (comm == MPI_COMM_SELF) dest = g_rank;
  if (dest < 0 || dest >= g_size) fatal("send to a rank outside the world");
  const int id = new_req();
  Req &r = g_reqs[size_t(id)];
  r.isSend = true, r.sbuf = static_cast<const unsigned char *>(buf), r.bytes = size_t(count) * dt_size(dt);
  r.peer = dest, r.tag = tag, r.comm = comm;
  *req = id;
  if (dest == g_rank) { // self-send: matched by pointer, one direct copy (device to device when both are device memory)
    g_self.push_back(SelfMsg{r.sbuf, {}, r.bytes, tag, comm, id});
    match();
    return MPI_SUCCESS;
  }
  g_sendq[size_t(dest)].push_back(id);
  progress();
  return MPI_SUCCESS;
}

int MPI_Irecv(void *buf, int count, MPI_Datatype dt, int source, int tag, MPI_Comm comm, MPI_Request *req) {
  init_world();
  if (comm == MPI_COMM_SELF) source = g_rank;
  const int id = new_req();
  Req &r = g_reqs[size_t(id)];
  r.rbuf = static_cast<unsigned char *>(buf), r.bytes = size_t(count) * dt_size(dt);
  r.peer = source, r.tag = tag, r.comm = comm;
  *req = id;
  g_recvq.push_back(id);
  progress();
  return MPI_SUCCESS;
}

int MPI_Test(MPI_Request *req, int *flag, MPI_Status *status) {
  if (*req == MPI_REQUEST_NULL) {
    *flag = 1;
    return MPI_SUCCESS;
  }
  progress();
  Req &r = g_reqs[size_t(*req)];
  if (r.done) {
    fill_status(status, r);
    r.live = false;
    *req = MPI_REQUEST_NULL;
    *flag = 1;
  } else {
    *flag = 0;
  }
  return MPI_SUCCESS;
}

int MPI_Wait(MPI_Request *req, MPI_Status *status) {
  if (*req == MPI_REQUEST_NULL) return MPI_SUCCESS;
  wait_req(*req);
  Req &r = g_reqs[size_t(*req)];
  fill_status(status, r);
  r.live = false;
  *req = MPI_REQUEST_NULL;
  return MPI_SUCCESS;
}

int MPI_Waitall(int n, MPI_Request *reqs, MPI_Status *statuses) {
  for (int i = 0; i < n; ++i) MPI_Wait(&reqs[i], statuses ? &statuses[i] : MPI_STATUS_IGNORE);
  return MPI_SUCCESS;
}

int MPI_Send(const void *buf, int count, MPI_Datatype dt, int dest, int tag, MPI_Comm comm) {
  MPI_Request q;
  MPI_Isend(buf, count, dt, dest, tag, comm, &q);
  Req &r = g_reqs[size_t(q)];
  if (!r.done && (dest == g_rank || comm == MPI_COMM_SELF)) {
    // blocking self-send with no receive posted yet: the caller may reuse the buffer on return -> keep a private copy
    for (SelfMsg &m : g_self) {
      if (m.reqId == q) {
        m.owned.resize(m.bytes ? m.bytes : 1);
        copy_any(m.owned.data(), m.ptr, m.bytes);
        m.reqId = 0;
      }
    }
    r.live = false;
    return MPI_SUCCESS;
  }
  return MPI_Wait(&q, MPI_STATUS_IGNORE); // remote: returns once the payload is in the ring
}

int MPI_Recv(void *buf, int count, MPI_Datatype dt, int source, int tag, MPI_Comm comm, MPI_Status *status) {
  MPI_Request r;
  MPI_Irecv(buf, count, dt, source, tag, comm, &r);
  return MPI_Wait(&r, status);
}

int MPI_Get_count(const MPI_Status *status, MPI_Datatype dt, int *count) {
  *count = int(size_t(status->count_bytes_) / dt_size(dt));
  return MPI_SUCCESS;
}

int MPI_Allreduce(const void *sendbuf, void *recvbuf, int count, MPI_Datatype dt, MPI_Op op, MPI_Comm comm) {
  init_world();
  if (!world_like(comm)) {
    if (sendbuf != MPI_IN_PLACE && sendbuf != recvbuf) copy_any(recvbuf, sendbuf, size_t(count) * dt_size(dt));
    return MPI_SUCCESS;
  }
  allreduce_bytes(sendbuf, recvbuf, count, dt, op);
  return MPI_SUCCESS;
}
int MPI_Reduce(const void *sendbuf, void *recvbuf, int count, MPI_Datatype dt, MPI_Op op, int root, MPI_Comm comm) {
  init_world();
  if (!world_like(comm)) {
    if (sendbuf != MPI_IN_PLACE && sendbuf != recvbuf && recvbuf) copy_any(recvbuf, sendbuf, size_t(count) * dt_size(dt));
    return MPI_SUCCESS;
  }
  const size_t bytes = size_t(count) * dt_size(dt);
  std::vector<unsigned char> tmp(bytes);
  if (sendbuf == MPI_IN_PLACE) copy_any(tmp.data(), recvbuf, bytes); // root only, by the standard
  allreduce_bytes(sendbuf == MPI_IN_PLACE ? tmp.data() : sendbuf, tmp.data(), count, dt, op);
  if (g_rank == root) copy_any(recvbuf, tmp.data(), bytes);
  return MPI_SUCCESS;
}
int MPI_Allgather(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, int recvcount, MPI_Datatype rdt, MPI_Comm comm) {
  init_world();
  if (!world_like(comm)) {
    if (sendbuf != MPI_IN_PLACE) copy_any(recvbuf, sendbuf, size_t(sendcount) * dt_size(sdt));
    return MPI_SUCCESS;
  }
  const size_t bytes = size_t(recvcount) * dt_size(rdt);
  std::vector<unsigned char> mine(bytes);
  copy_any(mine.data(), sendbuf == MPI_IN_PLACE ? static_cast<unsigned char *>(recvbuf) + size_t(g_rank) * bytes : sendbuf, bytes);
  allgather_bytes(mine.data(), bytes, recvbuf);
  return MPI_SUCCESS;
}
int MPI_Allgatherv(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, const int *recvcounts, const int *displs,
                   MPI_Datatype rdt, MPI_Comm comm) {
  init_world();
  if (!world_like(comm)) {
    if (sendbuf != MPI_IN_PLACE)
      copy_any(static_cast<char *>(recvbuf) + size_t(displs ? displs[0] : 0) * dt_size(rdt), sendbuf, size_t(sendcount) * dt_size(sdt));
    return MPI_SUCCESS;
  }
  size_t mx = 0;
  for (int r = 0; r < g_size; ++r) mx = std::max(mx, size_t(recvcounts[r]) * dt_size(rdt));
  std::vector<unsigned char> mine(mx), all(mx * size_t(g_size));
  const size_t myBytes = size_t(recvcounts[g_rank]) * dt_size(rdt);
  copy_any(mine.data(), sendbuf == MPI_IN_PLACE ? static_cast<unsigned char *>(recvbuf) + size_t(displs[g_rank]) * dt_size(rdt) : sendbuf, myBytes);
  allgather_bytes(mine.data(), mx, all.data());
  for (int r = 0; r < g_size; ++r)
    copy_any(static_cast<unsigned char *>(recvbuf) + size_t(displs[r]) * dt_size(rdt), all.data() + size_t(r) * mx, size_t(recvcounts[r]) * dt_size(rdt));
  return MPI_SUCCESS;
}
int MPI_Gather(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, int, MPI_Datatype, int root, MPI_Comm comm) {
  init_world();
  const size_t bytes = size_t(sendcount) * dt_size(sdt);
  if (!world_like(comm)) {
    if (sendbuf != MPI_IN_PLACE) copy_any(recvbuf, sendbuf, bytes);
    return MPI_SUCCESS;
  }
  std::vector<unsigned char> mine(bytes), all(bytes * size_t(g_size));
  copy_any(mine.data(), sendbuf == MPI_IN_PLACE ? static_cast<unsigned char *>(recvbuf) + size_t(g_rank) * bytes : sendbuf, bytes);
  allgather_bytes(mine.data(), bytes, all.data());
  if (g_rank == root) copy_any(recvbuf, all.data(), all.size());
  return MPI_SUCCESS;
}
int MPI_Bcast(void *buf, int count, MPI_Datatype dt, int root, MPI_Comm comm) {
  init_world();
  if (!world_like(comm)) return MPI_SUCCESS;
  const size_t bytes = size_t(count) * dt_size(dt);
  for (size_t off = 0; off < bytes; off += kColl) {
    const size_t n = std::min(kColl, bytes - off);
    if (g_rank == root) copy_any(coll_slot(root), static_cast<unsigned char *>(buf) + off, n);
    barrier_world();
    if (g_rank != root) copy_any(static_cast<unsigned char *>(buf) + off, coll_slot(root), n);
    barrier_world();
  }
  return MPI_SUCCESS;
}
int MPI_Alltoallv(const void *sendbuf, const int *sendcounts, const int *sdispls, MPI_Datatype sdt, void *recvbuf, const int *recvcounts,
                  const int *rdispls, MPI_Datatype rdt, MPI_Comm comm) {
  init_world();
  const int n = world_like(comm) ? g_size : 1;
  std::vector<MPI_Request> reqs;
  for (int r = 0; r < n; ++r) {
    MPI_Request q;
    MPI_Irecv(static_cast<char *>(recvbuf) + size_t(rdispls[r]) * dt_size(rdt), recvcounts[r], rdt, n == 1 ? g_rank : r, 0x5a5a, comm, &q);
    reqs.push_back(q);
  }
  for (int r = 0; r < n; ++r) {
    MPI_Request q;
    MPI_Isend(static_cast<const char *>(sendbuf) + size_t(sdispls[r]) * dt_size(sdt), sendcounts[r], sdt, n == 1 ? g_rank : r, 0x5a5a, comm, &q);
    reqs.push_back(q);
  }
  return MPI_Waitall(int(reqs.size()), reqs.data(), MPI_STATUSES_IGNORE);
}

} // extern "C"
