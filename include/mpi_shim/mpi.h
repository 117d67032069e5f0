/* mpi.h -- single-process MPI shim shipped with stencil_b200.
 *
 * A machine need not have an MPI installation, yet every public
 * header of cwpearson/stencil includes <mpi.h> (reference include/stencil/stencil.hpp:10) and
 * every driver calls MPI_Init / MPI_Wtime / MPI_Allreduce directly (bin/jacobi3d.cu:139,298,371).
 * This header declares exactly the MPI surface the reference library, drivers and tests use
 * (SURVEY.md 2c) for a world of ONE rank that drives all GPUs of the node -- a deployment the
 * reference already supports (src/stencil.cu:74-85).  Point-to-point calls are self-sends matched
 * by (communicator, tag); buffers may be host or device pointers.
 *
 * Implementation: src/mpi_shim.cpp (part of libstencil).  Put this directory on the include
 * path only when no real MPI is present.
 */
#pragma once

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STENCIL_B200_MPI_SHIM 1

typedef int MPI_Comm;
typedef int MPI_Datatype;
typedef int MPI_Op;
typedef int MPI_Info;
typedef int MPI_Request;

typedef struct MPI_Status {
  int MPI_SOURCE;
  int MPI_TAG;
  int MPI_ERROR;
  int count_bytes_;
} MPI_Status;

#define MPI_SUCCESS 0
#define MPI_ERR_OTHER 15

#define MPI_COMM_NULL ((MPI_Comm)0)
#define MPI_COMM_WORLD ((MPI_Comm)1)
#define MPI_COMM_SELF ((MPI_Comm)2)

#define MPI_INFO_NULL ((MPI_Info)0)
#define MPI_REQUEST_NULL ((MPI_Request)0)
#define MPI_STATUS_IGNORE ((MPI_Status *)0)
#define MPI_STATUSES_IGNORE ((MPI_Status *)0)
#define MPI_IN_PLACE ((void *)-1)
#define MPI_ANY_SOURCE (-2)
#define MPI_ANY_TAG (-1)

#define MPI_MAX_PROCESSOR_NAME 256
#define MPI_COMM_TYPE_SHARED 1
#define MPI_TAG_UB 1

#define MPI_THREAD_SINGLE 0
#define MPI_THREAD_FUNNELED 1
#define MPI_THREAD_SERIALIZED 2
#define MPI_THREAD_MULTIPLE 3

/* datatypes: the value encodes the element size in the low byte */
#define MPI_BYTE ((MPI_Datatype)0x0101)
#define MPI_CHAR ((MPI_Datatype)0x0201)
#define MPI_INT ((MPI_Datatype)0x0304)
#define MPI_UNSIGNED ((MPI_Datatype)0x0404)
#define MPI_FLOAT ((MPI_Datatype)0x0504)
#define MPI_DOUBLE ((MPI_Datatype)0x0608)
#define MPI_INT64_T ((MPI_Datatype)0x0708)
#define MPI_UINT64_T ((MPI_Datatype)0x0808)
#define MPI_LONG_LONG ((MPI_Datatype)0x0908)
#define MPI_UNSIGNED_LONG ((MPI_Datatype)0x0A08)

#define MPI_MAX ((MPI_Op)1)
#define MPI_MIN ((MPI_Op)2)
#define MPI_SUM ((MPI_Op)3)

int MPI_Init(int *argc, char ***argv);
int MPI_Init_thread(int *argc, char ***argv, int required, int *provided);
int MPI_Initialized(int *flag);
int MPI_Finalize(void);
int MPI_Abort(MPI_Comm comm, int errorcode);

int MPI_Comm_rank(MPI_Comm comm, int *rank);
int MPI_Comm_size(MPI_Comm comm, int *size);
int MPI_Comm_split_type(MPI_Comm comm, int split_type, int key, MPI_Info info, MPI_Comm *newcomm);
int MPI_Comm_free(MPI_Comm *comm);
int MPI_Comm_get_attr(MPI_Comm comm, int keyval, void *attribute_val, int *flag);
int MPI_Get_processor_name(char *name, int *resultlen);

double MPI_Wtime(void);
int MPI_Barrier(MPI_Comm comm);

int MPI_Isend(const void *buf, int count, MPI_Datatype dt, int dest, int tag, MPI_Comm comm, MPI_Request *req);
int MPI_Irecv(void *buf, int count, MPI_Datatype dt, int source, int tag, MPI_Comm comm, MPI_Request *req);
int MPI_Send(const void *buf, int count, MPI_Datatype dt, int dest, int tag, MPI_Comm comm);
int MPI_Recv(void *buf, int count, MPI_Datatype dt, int source, int tag, MPI_Comm comm, MPI_Status *status);
int MPI_Wait(MPI_Request *req, MPI_Status *status);
int MPI_Waitall(int n, MPI_Request *reqs, MPI_Status *statuses);
int MPI_Test(MPI_Request *req, int *flag, MPI_Status *status);
int MPI_Get_count(const MPI_Status *status, MPI_Datatype dt, int *count);

int MPI_Reduce(const void *sendbuf, void *recvbuf, int count, MPI_Datatype dt, MPI_Op op, int root, MPI_Comm comm);
int MPI_Allreduce(const void *sendbuf, void *recvbuf, int count, MPI_Datatype dt, MPI_Op op, MPI_Comm comm);
int MPI_Allgather(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, int recvcount, MPI_Datatype rdt,
                  MPI_Comm comm);
int MPI_Allgatherv(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, const int *recvcounts,
                   const int *displs, MPI_Datatype rdt, MPI_Comm comm);
int MPI_Gather(const void *sendbuf, int sendcount, MPI_Datatype sdt, void *recvbuf, int recvcount, MPI_Datatype rdt,
               int root, MPI_Comm comm);
int MPI_Bcast(void *buf, int count, MPI_Datatype dt, int root, MPI_Comm comm);
int MPI_Alltoallv(const void *sendbuf, const int *sendcounts, const int *sdispls, MPI_Datatype sdt, void *recvbuf,
                  const int *recvcounts, const int *rdispls, MPI_Datatype rdt, MPI_Comm comm);

#ifdef __cplusplus
}
#endif
