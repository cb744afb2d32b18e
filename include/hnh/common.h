// hnh/common.h -- common types of the H100-native HnH host library.
//
// Mirrors the public surface of the reference's common.h / common.cpp (DenseMatrix, MatMode,
// spcoord_t, BufferPair, pMod, divideAndRoundUp, divideIntoSegments, start_clock /
// stop_clock_get_elapsed; reference common.h:13-93, common.cpp:6-84) with one decisive
// difference: DenseMatrix and VectorXd own DEVICE memory (HBM) and every operation on them is a
// stream-ordered CUDA launch on hnh::Runtime::compute_stream().  The reference's DenseMatrix is
// an Eigen row-major host matrix (common.h:13); only the subset of the Eigen API that the
// reference's own callers use on the hot path and in the ALS application is provided
// (SURVEY.md 8b lists it).  `data()` returns a device pointer.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <string>
#include <vector>

#include "hnh/runtime.h"

using namespace std;  // the reference's headers do this and its drivers rely on it

typedef chrono::time_point<std::chrono::steady_clock> my_timer_t;
my_timer_t start_clock();
double stop_clock_get_elapsed(my_timer_t &start);

typedef enum { Amat, Bmat } MatMode;

int pMod(int num, int denom);
int divideAndRoundUp(int num, int denom);
// Roughly equal segments; segment_starts has num_segments + 1 entries (common.cpp:68-84).
void divideIntoSegments(int total, int num_segments, vector<int> &segment_starts,
                        vector<int> &segment_sizes);

struct spcoord_t {
    uint64_t r;
    uint64_t c;
    double value;
    string string_rep() const;
};
bool column_major(const spcoord_t &a, const spcoord_t &b);  // sort by (c, r)
bool row_major(const spcoord_t &a, const spcoord_t &b);     // sort by (r, c)
inline void initialize_mpi_datatypes() {}  // SPCOORD is sent as raw bytes here (common.cpp:37-47)

class DenseMatrix;

// Device vector of doubles (the reference's Eigen::VectorXd of SValues / sddmm_result).
class VectorXd {
public:
    VectorXd() = default;
    explicit VectorXd(int64_t n) : buf_((size_t)n), n_(n) {}
    VectorXd(const VectorXd &o);
    VectorXd &operator=(const VectorXd &o);
    VectorXd(VectorXd &&) = default;
    VectorXd &operator=(VectorXd &&) = default;
    static VectorXd Constant(int64_t n, double value);

    int64_t size() const { return n_; }
    double *data() { hnh::host_access_fence(); return buf_.data(); }
    const double *data() const { hnh::host_access_fence(); return buf_.data(); }
    void resize(int64_t n) { buf_.resize((size_t)n); n_ = n; }
    void setZero() { setConstant(0.0); }
    void setConstant(double v);
    // Element access from the HOST (`scale_vector[i]`, als_conjugate_gradients.cpp:21): only in host-access mode
    // (hnh::Runtime::managed_mode), where the storage is managed memory; throws otherwise.
    double &operator[](int64_t i);
    double operator[](int64_t i) const { return const_cast<VectorXd &>(*this)[i]; }
    // `v.array() += c` of the reference (als_conjugate_gradients.cpp:96-97): the array view is the vector itself
    VectorXd &array() { return *this; }

    VectorXd cwiseProduct(const VectorXd &o) const;
    VectorXd cwiseQuotient(const VectorXd &o) const;
    VectorXd operator+(const VectorXd &o) const;
    VectorXd operator-(const VectorXd &o) const;
    VectorXd &operator+=(double c);  // `.array() += c` of the reference
    double squaredNorm() const;      // synchronises and returns the host value
    double sum() const;
    // this[i] = (a[i] + ca) / (b[i] + cb): the alpha/coeff updates of cg_optimizer
    void setQuotient(const VectorXd &a, double ca, const VectorXd &b, double cb);
    // this[i] = max(this[i], 0) + alpha * min(this[i], 0)
    // (`v = v.array().max(0) + v.array().min(0) * alpha` of gat.hpp:98)
    void leakyRelu(double alpha);
    // this[i] = this[i] > 0 ? 1 : alpha: the derivative of leakyRelu at the values it was applied to
    void leakyReluGrad(double alpha);

    // host interop (not in Eigen; the data lives in HBM)
    static VectorXd from_host(const double *h, int64_t n);
    vector<double> to_host() const;
    void copy_from_host(const double *h);
    void swap(VectorXd &o) { buf_.swap(o.buf_); std::swap(n_, o.n_); }

private:
    hnh::DeviceBuffer<double> buf_;
    int64_t n_ = 0;
};

// A contiguous block of rows of a DenseMatrix (what Eigen's middleRows returns).
struct RowBlock {
    double *ptr;
    int64_t nrows, ncols;
    RowBlock &operator=(const DenseMatrix &m);  // copy m into the block
    double *data() const { return ptr; }
    int64_t rows() const { return nrows; }
    int64_t cols() const { return ncols; }
    int64_t size() const { return nrows * ncols; }
};

// Row-major dense matrix of doubles in HBM, leading dimension = cols().
class DenseMatrix {
public:
    DenseMatrix() = default;
    DenseMatrix(int64_t rows, int64_t cols) : buf_((size_t)(rows * cols)), rows_(rows), cols_(cols) {}
    DenseMatrix(const DenseMatrix &o);
    DenseMatrix &operator=(const DenseMatrix &o);
    DenseMatrix(DenseMatrix &&) = default;
    DenseMatrix &operator=(DenseMatrix &&) = default;
    DenseMatrix(const RowBlock &b);  // copy out of a block
    DenseMatrix &operator=(const RowBlock &b);
    static DenseMatrix Constant(int64_t rows, int64_t cols, double value);
    // Non-owning view of rows x cols doubles at device pointer p (e.g. a row block of another
    // matrix): lets a kernel work on part of a matrix without the copies Eigen's
    // `tmp = X.middleRows(...)` / `X.middleRows(...) = tmp` make (15D_sparse_shift.hpp:232-249).
    static DenseMatrix view(double *p, int64_t rows, int64_t cols) {
        DenseMatrix m;
        m.buf_.adopt(p, (size_t)(rows * cols));
        m.rows_ = rows;
        m.cols_ = cols;
        return m;
    }
    DenseMatrix rowsView(int64_t start, int64_t n) { return view(buf_.data() + start * cols_, n, cols_); }

    int64_t rows() const { return rows_; }
    int64_t cols() const { return cols_; }
    int64_t size() const { return rows_ * cols_; }
    double *data() { hnh::host_access_fence(); return buf_.data(); }
    const double *data() const { hnh::host_access_fence(); return buf_.data(); }
    void resize(int64_t rows, int64_t cols);
    void setZero() { setConstant(0.0); }
    void setConstant(double v);
    void setRandom(uint64_t seed);  // uniform(-1, 1), counter-based (Eigen::setRandom)
    void setRandom();               // the same with the next seed of a per-process sequence (Eigen's signature)
    RowBlock middleRows(int64_t start, int64_t n) {
        return RowBlock{buf_.data() + start * cols_, n, cols_};
    }

    DenseMatrix &operator*=(double s);
    DenseMatrix &operator/=(double s) { return *this *= (1.0 / s); }
    DenseMatrix &operator+=(const DenseMatrix &o);
    DenseMatrix &operator-=(const DenseMatrix &o);
    DenseMatrix operator+(const DenseMatrix &o) const;
    DenseMatrix operator-(const DenseMatrix &o) const;
    // `A.cwiseProduct(B)`: a lazy product, so that the reference's `A.cwiseProduct(B).rowwise().sum()`
    // (als_conjugate_gradients.cpp:9-11) is ONE batched-dot kernel; converts to a DenseMatrix anywhere else.
    struct CwiseProduct {
        const DenseMatrix &a, &b;
        operator DenseMatrix() const;
        struct Rowwise {
            const DenseMatrix &a, &b;
            VectorXd sum() const;
        };
        Rowwise rowwise() const { return Rowwise{a, b}; }
        double squaredNorm() const { return DenseMatrix(*this).squaredNorm(); }
    };
    CwiseProduct cwiseProduct(const DenseMatrix &o) const;
    double squaredNorm() const;

    // matrix product (gat.hpp:90 `buffers[i] * wMats[j]`): this library's DMMA GEMM (hnh_dgemm_f64) on the compute stream
    DenseMatrix operator*(const DenseMatrix &o) const;
    // this.middleCols(start, m.cols()) = m.array().max(0)   (gat.hpp:104)
    void setMiddleColsRelu(int64_t start, const DenseMatrix &m);
    // the GAT backward products (GAT::backwardPass), on this library's DMMA GEMMs:
    //   this = a^T * b                        (hnh_dgemm_tn_f64; a and b have the same row count)
    //   this = a * b^T, or this += a * b^T    (hnh_dgemm_nt_f64; a and b have the same column count)
    void setTransposeTimes(const DenseMatrix &a, const DenseMatrix &b);
    void setTimesTranspose(const DenseMatrix &a, const DenseMatrix &b, bool accumulate);
    // this = grad.middleCols(start, w) where out.middleCols(start, w) > 0, else 0; w = cols() (the ReLU gradient of
    // setMiddleColsRelu: grad and out are the gradient and the value of the matrix the ReLU wrote into)
    void setMiddleColsReluGrad(const DenseMatrix &grad, const DenseMatrix &out, int64_t start);

    // this = c + alpha * diag(s) * m  (row-scaled axpy; s empty == all ones). In place allowed.
    void setRowAxpy(const DenseMatrix &c, double alpha, const VectorXd *s, const DenseMatrix &m);

    static DenseMatrix from_host(const double *h, int64_t rows, int64_t cols);
    vector<double> to_host() const;
    void copy_from_host(const double *h);
    void copy_to_host(double *h) const;  // synchronises
    bool owns_storage() const { return buf_.owns(); }
    // *this = o without reallocating when `o` can give its storage away (both own theirs and have one shape):
    // a swap; otherwise (a view on either side) a device-to-device copy, like the reference's `*Arole = buffer`.
    void take(DenseMatrix &o);
    // Exchange storage with `o`.  The algorithm classes use this to hand a result back without a copy, so data()
    // pointers (and view() / rowsView() windows) taken before an operation are invalid after it.  A non-owning
    // view cannot take part: it would end up owning, or freeing, memory that belongs to somebody else.
    void swap(DenseMatrix &o) {
        if (!buf_.owns() || !o.buf_.owns()) throw hnh::Error(-1, "DenseMatrix::swap: non-owning view");
        buf_.swap(o.buf_);
        std::swap(rows_, o.rows_);
        std::swap(cols_, o.cols_);
    }

private:
    hnh::DeviceBuffer<double> buf_;
    int64_t rows_ = 0, cols_ = 0;
};

DenseMatrix operator*(double s, const DenseMatrix &m);  // `lambda * A` (als_conjugate_gradients.cpp:286,298)

// batch_dot_product / scale_matrix_rows of als_conjugate_gradients.cpp:9-29 on the device
VectorXd batch_dot_product(const DenseMatrix &A, const DenseMatrix &B);
DenseMatrix scale_matrix_rows(const VectorXd &scale_vector, const DenseMatrix &mat);

// Double buffer for ring shifts (reference common.h:49-93).  `extra` comes from the caching
// allocator; sync_active() swaps storage instead of copying when the live data ended up in
// `extra`.
class BufferPair {
public:
    DenseMatrix *original;
    DenseMatrix *extra;
    int switchVal;

    explicit BufferPair(DenseMatrix *buf)
        : original(buf), extra(new DenseMatrix(buf->rows(), buf->cols())), switchVal(0) {}
    ~BufferPair() { delete extra; }
    BufferPair(const BufferPair &) = delete;
    BufferPair &operator=(const BufferPair &) = delete;
    DenseMatrix *getActive() { return switchVal == 0 ? original : extra; }
    DenseMatrix *getPassive() { return switchVal == 0 ? extra : original; }
    void swapActive() { switchVal = 1 - switchVal; }
    void sync_active() {
        if (switchVal == 1) {
            original->take(*extra);  // swap, or a copy when the caller's matrix is a non-owning view
            switchVal = 0;
        }
    }
};
