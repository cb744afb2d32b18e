// hnh/comm.h -- the communicator abstraction that replaces raw MPI in the host classes.
//
// The reference talks MPI everywhere (MPI_Sendrecv ring shifts, distributed_sparse.h:351-361;
// MPI_Isend/Irecv CSR shifts, SpmatLocal.hpp:200-259; MPI_Allgather / MPI_Reduce_scatter
// replication, 15D_dense_shift.hpp:194,240,310,378; MPI_Alltoallv redistribution,
// SpmatLocal.hpp:425,451; MPI_Comm_split grids, FlexibleGrid.hpp:80-88).  Here one rank is one
// process that owns one GPU, and a `Comm` offers exactly those operations:
//   * on DEVICE buffers, stream-ordered (enqueued on a CUDA stream, no host synchronisation):
//     NCCL send/recv, all-gather, reduce-scatter over NVLink 5 / NVSwitch;
//   * on HOST buffers, blocking (setup path only: tuple redistribution, nnz counts).
// Transports: Self (world of 1: plain copies), Nccl (the product's multi-GPU path), External
// (caller-supplied C callbacks on host buffers -- torch.distributed/gloo in the CPU tests, or a
// real MPI in a maintainer's integration; device buffers are staged through pinned memory).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "hnh_b200_driver.h"

namespace hnh {

class Transport;

class Comm {
public:
    // One (send, recv) segment of a grouped exchange with a single (dst, src) pair.
    struct Seg {
        const void *send;
        size_t send_bytes;
        void *recv;
        size_t recv_bytes;
    };

    ~Comm();
    int rank() const { return rank_; }
    int size() const { return size_; }
    const std::string &transport_name() const;

    // ---- device buffers, enqueued on `s` ------------------------------------------------
    void sendrecv(const void *send, size_t send_bytes, int dst, void *recv, size_t recv_bytes,
                  int src, cudaStream_t s);
    void sendrecv_multi(const Seg *segs, int nsegs, int dst, int src, cudaStream_t s);
    // recv holds size()*bytes_each; rank i's contribution lands at offset i*bytes_each
    void allgather(const void *send, void *recv, size_t bytes_each, cudaStream_t s);
    // send holds size()*count_each doubles; rank i receives the sum of everyone's i-th chunk
    void reduce_scatter_sum_f64(const double *send, double *recv, size_t count_each, cudaStream_t s);
    void allreduce_sum_f64(double *buf, size_t count, cudaStream_t s);
    void allreduce_max_f64(double *buf, size_t count, cudaStream_t s);  // element-wise maximum over the ranks
    // MPI_Alltoallv on device buffers (byte counts / displacements per rank)
    void alltoallv(const void *send, const size_t *send_bytes, const size_t *send_displs, void *recv,
                   const size_t *recv_bytes, const size_t *recv_displs, cudaStream_t s);

    // ---- host buffers, blocking (setup path) ---------------------------------------------
    void host_sendrecv(const void *send, size_t send_bytes, int dst, void *recv, size_t recv_bytes, int src);
    void host_allgather(const void *send, void *recv, size_t bytes_each);
    void host_alltoallv(const void *send, const size_t *send_bytes, const size_t *send_displs,
                        void *recv, const size_t *recv_bytes, const size_t *recv_displs);
    void host_allreduce_sum_f64(double *buf, size_t count);
    void barrier();

    // MPI_Comm_split semantics: ranks with equal color form a communicator, ordered by key.
    std::shared_ptr<Comm> split(int color, int key);

    // ---- process world --------------------------------------------------------------------
    static std::shared_ptr<Comm> world();  // throws if no world was initialised
    static bool world_initialised();
    static void init_self();
    static void init_nccl(int rank, int size, const char unique_id[HNHD_NCCL_ID_BYTES]);
    static void init_external(int rank, int size, const hnhd_external_transport_t *cb);
    static void nccl_unique_id(char out[HNHD_NCCL_ID_BYTES]);
    static void finalize();

    // bytes moved through device-buffer operations since the last reset (per rank, sent side)
    uint64_t device_bytes_sent() const { return bytes_sent_; }
    void reset_counters() { bytes_sent_ = 0; }

private:
    friend class Transport;
    Comm(std::shared_ptr<Transport> t, int rank, int size);
    std::shared_ptr<Transport> t_;
    int rank_, size_;
    uint64_t bytes_sent_ = 0;
    static std::shared_ptr<Comm> &world_slot();
};

}  // namespace hnh
