// comm.cpp -- hnh::Comm and its three transports (Self, Nccl, External).  See hnh/comm.h.
#include "hnh/comm.h"

#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "hnh/runtime.h"
#include "hnh_b200.h"

namespace hnh {

// ------------------------------------------------------------------ transport interface --
class Transport {
public:
    virtual ~Transport() {}
    virtual const std::string &name() const = 0;
    virtual void sendrecv_multi(int rank, const Comm::Seg *segs, int n, int dst, int src, cudaStream_t s) = 0;
    virtual void allgather(int rank, int size, const void *send, void *recv, size_t bytes_each, cudaStream_t s) = 0;
    virtual void reduce_scatter(int rank, int size, const double *send, double *recv, size_t count_each, cudaStream_t s) = 0;
    virtual void allreduce(double *buf, size_t count, cudaStream_t s) = 0;
    virtual void allreduce_max(int size, double *buf, size_t count, cudaStream_t s) = 0;
    // default: through host memory with the transport's host all-to-all
    virtual void alltoallv(int rank, int size, const void *send, const size_t *sb, const size_t *sd, void *recv, const size_t *rb,
                           const size_t *rd, cudaStream_t s) {
        size_t stot = 0, rtot = 0;
        for (int i = 0; i < size; i++) {
            stot = std::max(stot, sd[i] + sb[i]);
            rtot = std::max(rtot, rd[i] + rb[i]);
        }
        std::vector<char> hs(std::max<size_t>(stot, 1)), hr(std::max<size_t>(rtot, 1));
        if (stot) cuda_check(cudaMemcpyAsync(hs.data(), send, stot, cudaMemcpyDeviceToHost, s), "alltoallv d2h");
        cuda_check(cudaStreamSynchronize(s), "alltoallv sync");
        host_alltoallv(rank, size, hs.data(), sb, sd, hr.data(), rb, rd);
        if (rtot) cuda_check(cudaMemcpyAsync(recv, hr.data(), rtot, cudaMemcpyHostToDevice, s), "alltoallv h2d");
        cuda_check(cudaStreamSynchronize(s), "alltoallv sync");
    }
    virtual void host_sendrecv(int rank, const void *send, size_t sb, int dst, void *recv, size_t rb, int src) = 0;
    virtual void host_allgather(int rank, int size, const void *send, void *recv, size_t bytes_each) = 0;
    virtual void host_alltoallv(int rank, int size, const void *send, const size_t *sb, const size_t *sd,
                                void *recv, const size_t *rb, const size_t *rd) = 0;
    virtual void host_allreduce(double *buf, size_t count) = 0;
    virtual void barrier() = 0;
    virtual std::shared_ptr<Transport> split(int color, int key, int *new_rank, int *new_size) = 0;

protected:
    static std::shared_ptr<Comm> make_comm(std::shared_ptr<Transport> t, int rank, int size);
};

static void copy_d2d(void *dst, const void *src, size_t bytes, cudaStream_t s) {
    if (bytes && dst != src)
        cuda_check(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s), "cudaMemcpyAsync d2d");
}

// ------------------------------------------------------------------ Self -----------------
class SelfTransport : public Transport {
public:
    const std::string &name() const override { static std::string n = "self"; return n; }
    void sendrecv_multi(int, const Comm::Seg *segs, int n, int, int, cudaStream_t s) override {
        for (int i = 0; i < n; i++) {
            if (segs[i].send_bytes != segs[i].recv_bytes)
                throw Error(HNH_E_COMM, "self sendrecv: send/recv size mismatch");
            copy_d2d(segs[i].recv, segs[i].send, segs[i].send_bytes, s);
        }
    }
    void allgather(int, int, const void *send, void *recv, size_t b, cudaStream_t s) override { copy_d2d(recv, send, b, s); }
    void reduce_scatter(int, int, const double *send, double *recv, size_t c, cudaStream_t s) override {
        copy_d2d(recv, send, c * sizeof(double), s);
    }
    void allreduce(double *, size_t, cudaStream_t) override {}
    void allreduce_max(int, double *, size_t, cudaStream_t) override {}
    void alltoallv(int, int, const void *send, const size_t *sb, const size_t *sd, void *recv, const size_t *rb, const size_t *rd,
                   cudaStream_t s) override {
        if (sb[0] != rb[0]) throw Error(HNH_E_COMM, "self alltoallv: size mismatch");
        copy_d2d((char *)recv + rd[0], (const char *)send + sd[0], sb[0], s);
    }
    void host_sendrecv(int, const void *send, size_t sb, int, void *recv, size_t rb, int) override {
        if (sb != rb) throw Error(HNH_E_COMM, "self sendrecv: size mismatch");
        if (recv != send) std::memcpy(recv, send, sb);
    }
    void host_allgather(int, int, const void *send, void *recv, size_t b) override {
        if (recv != send) std::memcpy(recv, send, b);
    }
    void host_alltoallv(int, int, const void *send, const size_t *sb, const size_t *sd, void *recv,
                        const size_t *rb, const size_t *rd) override {
        if (sb[0] != rb[0]) throw Error(HNH_E_COMM, "self alltoallv: size mismatch");
        std::memcpy((char *)recv + rd[0], (const char *)send + sd[0], sb[0]);
    }
    void host_allreduce(double *, size_t) override {}
    void barrier() override {}
    std::shared_ptr<Transport> split(int, int, int *nr, int *ns) override {
        *nr = 0; *ns = 1;
        return std::make_shared<SelfTransport>();
    }
};

// ------------------------------------------------------------------ NCCL -----------------
static void nccl_check(ncclResult_t r, const char *what) {
    if (r != ncclSuccess && r != ncclInProgress)
        throw Error(HNH_E_COMM, std::string(what) + ": " + ncclGetErrorString(r));
}

class NcclTransport : public Transport {
public:
    NcclTransport(ncclComm_t c, int rank, int size) : comm_(c), rank_(rank), size_(size) {}
    ~NcclTransport() override {
        if (comm_) ncclCommDestroy(comm_);
    }
    const std::string &name() const override { static std::string n = "nccl"; return n; }

    void sendrecv_multi(int rank, const Comm::Seg *segs, int n, int dst, int src, cudaStream_t s) override {
        if (dst == rank && src == rank) {
            for (int i = 0; i < n; i++) copy_d2d(segs[i].recv, segs[i].send, segs[i].send_bytes, s);
            return;
        }
        nccl_check(ncclGroupStart(), "ncclGroupStart");
        for (int i = 0; i < n; i++) {
            if (segs[i].send_bytes)
                nccl_check(ncclSend(segs[i].send, segs[i].send_bytes, ncclChar, dst, comm_, s), "ncclSend");
            if (segs[i].recv_bytes)
                nccl_check(ncclRecv(segs[i].recv, segs[i].recv_bytes, ncclChar, src, comm_, s), "ncclRecv");
        }
        nccl_check(ncclGroupEnd(), "ncclGroupEnd");
    }
    void allgather(int, int, const void *send, void *recv, size_t b, cudaStream_t s) override {
        nccl_check(ncclAllGather(send, recv, b, ncclChar, comm_, s), "ncclAllGather");
    }
    void reduce_scatter(int, int, const double *send, double *recv, size_t c, cudaStream_t s) override {
        nccl_check(ncclReduceScatter(send, recv, c, ncclDouble, ncclSum, comm_, s), "ncclReduceScatter");
    }
    void allreduce(double *buf, size_t count, cudaStream_t s) override {
        nccl_check(ncclAllReduce(buf, buf, count, ncclDouble, ncclSum, comm_, s), "ncclAllReduce");
    }
    void allreduce_max(int, double *buf, size_t count, cudaStream_t s) override {
        nccl_check(ncclAllReduce(buf, buf, count, ncclDouble, ncclMax, comm_, s), "ncclAllReduce");
    }

    void alltoallv(int rank, int size, const void *send, const size_t *sb, const size_t *sd, void *recv, const size_t *rb,
                   const size_t *rd, cudaStream_t s) override {
        copy_d2d((char *)recv + rd[rank], (const char *)send + sd[rank], sb[rank], s);
        nccl_check(ncclGroupStart(), "ncclGroupStart");
        for (int i = 0; i < size; i++) {
            if (i == rank) continue;
            if (sb[i]) nccl_check(ncclSend((const char *)send + sd[i], sb[i], ncclChar, i, comm_, s), "ncclSend");
            if (rb[i]) nccl_check(ncclRecv((char *)recv + rd[i], rb[i], ncclChar, i, comm_, s), "ncclRecv");
        }
        nccl_check(ncclGroupEnd(), "ncclGroupEnd");
    }
    // host buffers are staged through device memory (setup path only)
    void host_sendrecv(int rank, const void *send, size_t sb, int dst, void *recv, size_t rb, int src) override {
        if (dst == rank && src == rank) {
            if (recv != send) std::memcpy(recv, send, sb);
            return;
        }
        cudaStream_t s = Runtime::get().comm_stream();
        stage_a_.resize(sb);
        stage_b_.resize(rb);
        if (sb) cuda_check(cudaMemcpyAsync(stage_a_.data(), send, sb, cudaMemcpyHostToDevice, s), "h2d");
        nccl_check(ncclGroupStart(), "ncclGroupStart");
        if (sb) nccl_check(ncclSend(stage_a_.data(), sb, ncclChar, dst, comm_, s), "ncclSend");
        if (rb) nccl_check(ncclRecv(stage_b_.data(), rb, ncclChar, src, comm_, s), "ncclRecv");
        nccl_check(ncclGroupEnd(), "ncclGroupEnd");
        if (rb) cuda_check(cudaMemcpyAsync(recv, stage_b_.data(), rb, cudaMemcpyDeviceToHost, s), "d2h");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    void host_allgather(int, int size, const void *send, void *recv, size_t b) override {
        cudaStream_t s = Runtime::get().comm_stream();
        stage_a_.resize(b);
        stage_b_.resize(b * size);
        cuda_check(cudaMemcpyAsync(stage_a_.data(), send, b, cudaMemcpyHostToDevice, s), "h2d");
        nccl_check(ncclAllGather(stage_a_.data(), stage_b_.data(), b, ncclChar, comm_, s), "ncclAllGather");
        cuda_check(cudaMemcpyAsync(recv, stage_b_.data(), b * size, cudaMemcpyDeviceToHost, s), "d2h");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    void host_alltoallv(int, int size, const void *send, const size_t *sb, const size_t *sd, void *recv,
                        const size_t *rb, const size_t *rd) override {
        cudaStream_t s = Runtime::get().comm_stream();
        size_t stot = 0, rtot = 0;
        for (int i = 0; i < size; i++) {
            stot = std::max(stot, sd[i] + sb[i]);
            rtot = std::max(rtot, rd[i] + rb[i]);
        }
        stage_a_.resize(stot);
        stage_b_.resize(rtot);
        if (stot) cuda_check(cudaMemcpyAsync(stage_a_.data(), send, stot, cudaMemcpyHostToDevice, s), "h2d");
        nccl_check(ncclGroupStart(), "ncclGroupStart");
        for (int i = 0; i < size; i++) {
            if (sb[i]) nccl_check(ncclSend(stage_a_.data() + sd[i], sb[i], ncclChar, i, comm_, s), "ncclSend");
            if (rb[i]) nccl_check(ncclRecv(stage_b_.data() + rd[i], rb[i], ncclChar, i, comm_, s), "ncclRecv");
        }
        nccl_check(ncclGroupEnd(), "ncclGroupEnd");
        if (rtot) cuda_check(cudaMemcpyAsync(recv, stage_b_.data(), rtot, cudaMemcpyDeviceToHost, s), "d2h");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    void host_allreduce(double *buf, size_t count) override {
        cudaStream_t s = Runtime::get().comm_stream();
        stage_a_.resize(count * sizeof(double));
        cuda_check(cudaMemcpyAsync(stage_a_.data(), buf, count * sizeof(double), cudaMemcpyHostToDevice, s), "h2d");
        nccl_check(ncclAllReduce(stage_a_.data(), stage_a_.data(), count, ncclDouble, ncclSum, comm_, s), "ncclAllReduce");
        cuda_check(cudaMemcpyAsync(buf, stage_a_.data(), count * sizeof(double), cudaMemcpyDeviceToHost, s), "d2h");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    void barrier() override {
        double one = 1.0;
        Runtime::get().sync_all();
        host_allreduce(&one, 1);
    }
    std::shared_ptr<Transport> split(int color, int key, int *nr, int *ns) override {
        ncclComm_t sub = nullptr;
        nccl_check(ncclCommSplit(comm_, color, key, &sub, nullptr), "ncclCommSplit");
        nccl_check(ncclCommUserRank(sub, nr), "ncclCommUserRank");
        nccl_check(ncclCommCount(sub, ns), "ncclCommCount");
        return std::make_shared<NcclTransport>(sub, *nr, *ns);
    }

private:
    ncclComm_t comm_;
    int rank_, size_;
    DeviceBuffer<char> stage_a_, stage_b_;
};

// ------------------------------------------------------------------ External -------------
class ExternalTransport : public Transport {
public:
    ExternalTransport(const hnhd_external_transport_t &cb, int comm, int rank, int size)
        : cb_(cb), id_(comm), rank_(rank), size_(size) {}
    ~ExternalTransport() override {
        Runtime::get().free_pinned(pin_a_);
        Runtime::get().free_pinned(pin_b_);
    }
    const std::string &name() const override { static std::string n = "external"; return n; }

    void sendrecv_multi(int, const Comm::Seg *segs, int n, int dst, int src, cudaStream_t s) override {
        for (int i = 0; i < n; i++) {
            const Comm::Seg &g = segs[i];
            char *hs = pinned_a(g.send_bytes), *hr = pinned_b(g.recv_bytes);
            d2h(hs, g.send, g.send_bytes, s);
            call(cb_.sendrecv(cb_.ctx, id_, hs, g.send_bytes, dst, hr, g.recv_bytes, src), "sendrecv");
            h2d(g.recv, hr, g.recv_bytes, s);
        }
    }
    void allgather(int, int size, const void *send, void *recv, size_t b, cudaStream_t s) override {
        char *hs = pinned_a(b), *hr = pinned_b(b * size);
        d2h(hs, send, b, s);
        call(cb_.allgather(cb_.ctx, id_, hs, hr, b), "allgather");
        h2d(recv, hr, b * size, s);
    }
    void reduce_scatter(int, int size, const double *send, double *recv, size_t c, cudaStream_t s) override {
        char *hs = pinned_a(c * size * sizeof(double)), *hr = pinned_b(c * sizeof(double));
        d2h(hs, send, c * size * sizeof(double), s);
        call(cb_.reduce_scatter_f64(cb_.ctx, id_, (const double *)hs, (double *)hr, c), "reduce_scatter");
        h2d(recv, hr, c * sizeof(double), s);
    }
    void allreduce(double *buf, size_t count, cudaStream_t s) override {
        char *hs = pinned_a(count * sizeof(double));
        d2h(hs, buf, count * sizeof(double), s);
        call(cb_.allreduce_f64(cb_.ctx, id_, (double *)hs, count), "allreduce");
        h2d(buf, hs, count * sizeof(double), s);
    }
    // the callback table has no max reduction: every rank gathers all contributions and takes the maximum of
    // each element in rank order (the same result everywhere)
    void allreduce_max(int size, double *buf, size_t count, cudaStream_t s) override {
        const size_t b = count * sizeof(double);
        char *hs = pinned_a(b), *hr = pinned_b(b * size);
        d2h(hs, buf, b, s);
        call(cb_.allgather(cb_.ctx, id_, hs, hr, b), "allgather");
        double *out = (double *)hs;
        const double *all = (const double *)hr;
        for (size_t i = 0; i < count; i++) {
            double m = all[i];
            for (int q = 1; q < size; q++) m = std::max(m, all[(size_t)q * count + i]);
            out[i] = m;
        }
        h2d(buf, hs, b, s);
    }
    void host_sendrecv(int, const void *send, size_t sb, int dst, void *recv, size_t rb, int src) override {
        call(cb_.sendrecv(cb_.ctx, id_, send, sb, dst, recv, rb, src), "sendrecv");
    }
    void host_allgather(int, int, const void *send, void *recv, size_t b) override {
        call(cb_.allgather(cb_.ctx, id_, send, recv, b), "allgather");
    }
    void host_alltoallv(int, int, const void *send, const size_t *sb, const size_t *sd, void *recv,
                        const size_t *rb, const size_t *rd) override {
        call(cb_.alltoallv(cb_.ctx, id_, send, sb, sd, recv, rb, rd), "alltoallv");
    }
    void host_allreduce(double *buf, size_t count) override {
        call(cb_.allreduce_f64(cb_.ctx, id_, buf, count), "allreduce");
    }
    void barrier() override {
        if (Runtime::get().has_device()) Runtime::get().sync_all();
        call(cb_.barrier(cb_.ctx, id_), "barrier");
    }
    std::shared_ptr<Transport> split(int color, int key, int *nr, int *ns) override {
        int nc = -1;
        call(cb_.split(cb_.ctx, id_, color, key, &nc, nr, ns), "split");
        return std::make_shared<ExternalTransport>(cb_, nc, *nr, *ns);
    }

private:
    static void call(int rc, const char *what) {
        if (rc != 0) throw Error(HNH_E_COMM, std::string("external transport callback failed: ") + what);
    }
    char *pinned_a(size_t n) { return grow(pin_a_, cap_a_, n); }
    char *pinned_b(size_t n) { return grow(pin_b_, cap_b_, n); }
    static char *grow(void *&p, size_t &cap, size_t n) {
        if (n > cap) {
            Runtime::get().free_pinned(p);
            p = Runtime::get().alloc_pinned(n);
            cap = n;
        }
        return (char *)p;
    }
    static void d2h(void *h, const void *d, size_t n, cudaStream_t s) {
        if (n) cuda_check(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s), "d2h");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    static void h2d(void *d, const void *h, size_t n, cudaStream_t s) {
        if (n) cuda_check(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s), "h2d");
        cuda_check(cudaStreamSynchronize(s), "sync");
    }
    hnhd_external_transport_t cb_;
    int id_, rank_, size_;
    void *pin_a_ = nullptr, *pin_b_ = nullptr;
    size_t cap_a_ = 0, cap_b_ = 0;
};

// ------------------------------------------------------------------ Comm -----------------
std::shared_ptr<Comm> Transport::make_comm(std::shared_ptr<Transport> t, int rank, int size) {
    return std::shared_ptr<Comm>(new Comm(std::move(t), rank, size));
}

struct CommFactory : Transport {  // access to the protected maker
    static std::shared_ptr<Comm> make(std::shared_ptr<Transport> t, int r, int s) { return make_comm(std::move(t), r, s); }
};

Comm::Comm(std::shared_ptr<Transport> t, int rank, int size) : t_(std::move(t)), rank_(rank), size_(size) {}
Comm::~Comm() {}
const std::string &Comm::transport_name() const { return t_->name(); }

void Comm::sendrecv(const void *send, size_t sb, int dst, void *recv, size_t rb, int src, cudaStream_t s) {
    Seg g{send, sb, recv, rb};
    sendrecv_multi(&g, 1, dst, src, s);
}
void Comm::sendrecv_multi(const Seg *segs, int n, int dst, int src, cudaStream_t s) {
    if (dst < 0 || dst >= size_ || src < 0 || src >= size_) throw Error(HNH_E_COMM, "sendrecv: peer out of range");
    for (int i = 0; i < n; i++) bytes_sent_ += segs[i].send_bytes;
    t_->sendrecv_multi(rank_, segs, n, dst, src, s);
}
void Comm::allgather(const void *send, void *recv, size_t b, cudaStream_t s) {
    bytes_sent_ += b * (size_ - 1);
    t_->allgather(rank_, size_, send, recv, b, s);
}
void Comm::reduce_scatter_sum_f64(const double *send, double *recv, size_t c, cudaStream_t s) {
    bytes_sent_ += c * sizeof(double) * (size_ - 1);
    t_->reduce_scatter(rank_, size_, send, recv, c, s);
}
void Comm::alltoallv(const void *send, const size_t *sb, const size_t *sd, void *recv, const size_t *rb, const size_t *rd,
                     cudaStream_t s) {
    for (int i = 0; i < size_; i++)
        if (i != rank_) bytes_sent_ += sb[i];
    t_->alltoallv(rank_, size_, send, sb, sd, recv, rb, rd, s);
}
void Comm::allreduce_sum_f64(double *buf, size_t count, cudaStream_t s) {
    if (size_ > 1) bytes_sent_ += 2 * count * sizeof(double) * (size_ - 1) / size_;
    t_->allreduce(buf, count, s);
}
void Comm::allreduce_max_f64(double *buf, size_t count, cudaStream_t s) {
    if (size_ > 1) bytes_sent_ += 2 * count * sizeof(double) * (size_ - 1) / size_;
    t_->allreduce_max(size_, buf, count, s);
}
void Comm::host_sendrecv(const void *send, size_t sb, int dst, void *recv, size_t rb, int src) {
    t_->host_sendrecv(rank_, send, sb, dst, recv, rb, src);
}
void Comm::host_allgather(const void *send, void *recv, size_t b) { t_->host_allgather(rank_, size_, send, recv, b); }
void Comm::host_alltoallv(const void *send, const size_t *sb, const size_t *sd, void *recv, const size_t *rb,
                          const size_t *rd) {
    t_->host_alltoallv(rank_, size_, send, sb, sd, recv, rb, rd);
}
void Comm::host_allreduce_sum_f64(double *buf, size_t count) { t_->host_allreduce(buf, count); }
void Comm::barrier() { t_->barrier(); }

std::shared_ptr<Comm> Comm::split(int color, int key) {
    int nr = 0, ns = 1;
    auto nt = t_->split(color, key, &nr, &ns);
    return CommFactory::make(nt, nr, ns);
}

std::shared_ptr<Comm> &Comm::world_slot() {
    static std::shared_ptr<Comm> w;
    return w;
}
bool Comm::world_initialised() { return (bool)world_slot(); }
std::shared_ptr<Comm> Comm::world() {
    if (!world_slot())
        throw Error(HNH_E_COMM, "no world: call hnhd_init_self / hnhd_init_nccl / hnhd_init_external "
                                "(the MPI_Init of this library) first");
    return world_slot();
}
void Comm::init_self() { world_slot() = CommFactory::make(std::make_shared<SelfTransport>(), 0, 1); }
void Comm::nccl_unique_id(char out[HNHD_NCCL_ID_BYTES]) {
    static_assert(sizeof(ncclUniqueId) <= HNHD_NCCL_ID_BYTES, "ncclUniqueId does not fit");
    ncclUniqueId id;
    nccl_check(ncclGetUniqueId(&id), "ncclGetUniqueId");
    std::memset(out, 0, HNHD_NCCL_ID_BYTES);
    std::memcpy(out, &id, sizeof(id));
}
void Comm::init_nccl(int rank, int size, const char uid[HNHD_NCCL_ID_BYTES]) {
    Runtime::get().compute_stream();  // bind the device first
    ncclUniqueId id;
    std::memcpy(&id, uid, sizeof(id));
    ncclComm_t c = nullptr;
    nccl_check(ncclCommInitRank(&c, size, id, rank), "ncclCommInitRank");
    world_slot() = CommFactory::make(std::make_shared<NcclTransport>(c, rank, size), rank, size);
}
void Comm::init_external(int rank, int size, const hnhd_external_transport_t *cb) {
    if (!cb || !cb->sendrecv || !cb->allgather || !cb->reduce_scatter_f64 || !cb->allreduce_f64 ||
        !cb->alltoallv || !cb->barrier || !cb->split)
        throw Error(HNH_E_INVALID, "init_external: incomplete callback table");
    world_slot() = CommFactory::make(std::make_shared<ExternalTransport>(*cb, 0, rank, size), rank, size);
}
void Comm::finalize() { world_slot().reset(); }

}  // namespace hnh
