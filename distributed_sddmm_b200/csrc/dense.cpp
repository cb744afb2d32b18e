// dense.cpp -- device-resident DenseMatrix / VectorXd and the small helpers of hnh/common.h.
#include "hnh/common.h"
#include "hnh_b200.h"

using hnh::abi_check;
using hnh::cuda_check;
using hnh::Runtime;

static cudaStream_t cs() { return Runtime::get().compute_stream(); }

my_timer_t start_clock() { return std::chrono::steady_clock::now(); }
double stop_clock_get_elapsed(my_timer_t &start) {
    std::chrono::duration<double> diff = std::chrono::steady_clock::now() - start;
    return diff.count();
}

int pMod(int num, int denom) { return ((num % denom) + denom) % denom; }
int divideAndRoundUp(int num, int denom) { return num / denom + (num % denom > 0 ? 1 : 0); }

void divideIntoSegments(int total, int num_segments, vector<int> &segment_starts, vector<int> &segment_sizes) {
    const int share = divideAndRoundUp(total, num_segments);
    segment_starts.clear();
    for (int i = 0; i < num_segments; i++) segment_starts.push_back(std::min(share * i, total));
    segment_starts.push_back(total);
    for (int i = 0; i < num_segments; i++) segment_sizes.push_back(segment_starts[i + 1] - segment_starts[i]);
}

string spcoord_t::string_rep() const { return to_string(r) + " " + to_string(c) + " " + to_string(value); }
bool column_major(const spcoord_t &a, const spcoord_t &b) { return a.c == b.c ? a.r < b.r : a.c < b.c; }
bool row_major(const spcoord_t &a, const spcoord_t &b) { return a.r == b.r ? a.c < b.c : a.r < b.r; }

static void d2d(double *dst, const double *src, int64_t n) {
    if (n > 0 && dst != src)
        cuda_check(cudaMemcpyAsync(dst, src, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, cs()), "d2d copy");
}
static void require(bool ok, const char *what) {
    if (!ok) throw hnh::Error(HNH_E_INVALID, what);
}

// ------------------------------------------------------------------ VectorXd -------------
VectorXd::VectorXd(const VectorXd &o) : buf_((size_t)o.n_), n_(o.n_) { d2d(data(), o.data(), n_); }
VectorXd &VectorXd::operator=(const VectorXd &o) {
    if (this != &o) {
        resize(o.n_);
        d2d(data(), o.data(), n_);
    }
    return *this;
}
VectorXd VectorXd::Constant(int64_t n, double value) {
    VectorXd v(n);
    v.setConstant(value);
    return v;
}
void VectorXd::setConstant(double v) { abi_check(hnh_fill_f64(data(), n_, v, cs()), "fill"); }
double &VectorXd::operator[](int64_t i) {
    if (!hnh::Runtime::managed_mode())
        throw hnh::Error(HNH_E_INVALID, "VectorXd::operator[]: element access from the host needs host-access mode "
                                        "(HNH_MANAGED_MEMORY=1 / the compat <Eigen/Dense>); the vector lives in HBM");
    if (i < 0 || i >= n_) throw hnh::Error(HNH_E_INVALID, "VectorXd::operator[]: index out of range");
    return data()[i];
}
VectorXd VectorXd::cwiseProduct(const VectorXd &o) const {
    require(o.n_ == n_, "cwiseProduct: size mismatch");
    VectorXd r(n_);
    abi_check(hnh_hadamard_f64(r.data(), data(), o.data(), n_, cs()), "hadamard");
    return r;
}
VectorXd VectorXd::cwiseQuotient(const VectorXd &o) const {
    require(o.n_ == n_, "cwiseQuotient: size mismatch");
    VectorXd r(n_);
    abi_check(hnh_vec_quotient_f64(r.data(), data(), 0.0, o.data(), 0.0, n_, cs()), "quotient");
    return r;
}
void VectorXd::setQuotient(const VectorXd &a, double ca, const VectorXd &b, double cb) {
    require(a.n_ == b.n_, "setQuotient: size mismatch");
    resize(a.n_);
    abi_check(hnh_vec_quotient_f64(data(), a.data(), ca, b.data(), cb, n_, cs()), "quotient");
}
VectorXd VectorXd::operator+(const VectorXd &o) const {
    require(o.n_ == n_, "operator+: size mismatch");
    VectorXd r(n_);
    abi_check(hnh_axpby_f64(r.data(), 1.0, data(), 1.0, o.data(), n_, cs()), "axpby");
    return r;
}
VectorXd VectorXd::operator-(const VectorXd &o) const {
    require(o.n_ == n_, "operator-: size mismatch");
    VectorXd r(n_);
    abi_check(hnh_axpby_f64(r.data(), 1.0, data(), -1.0, o.data(), n_, cs()), "axpby");
    return r;
}
VectorXd &VectorXd::operator+=(double c) {
    abi_check(hnh_vec_quotient_f64(data(), data(), c, nullptr, 0.0, n_, cs()), "add scalar");
    return *this;
}
double VectorXd::squaredNorm() const {
    hnh::DeviceBuffer<double> out(1);
    abi_check(hnh_squared_norm_f64(out.data(), data(), n_, cs()), "squared_norm");
    return out.to_host(1, cs())[0];
}
double VectorXd::sum() const {
    vector<double> h = to_host();
    double s = 0.0;
    for (double x : h) s += x;
    return s;
}
VectorXd VectorXd::from_host(const double *h, int64_t n) {
    VectorXd v(n);
    v.copy_from_host(h);
    return v;
}
void VectorXd::copy_from_host(const double *h) {
    if (n_) cuda_check(cudaMemcpyAsync(data(), h, sizeof(double) * (size_t)n_, cudaMemcpyHostToDevice, cs()), "h2d");
    cuda_check(cudaStreamSynchronize(cs()), "sync");
}
vector<double> VectorXd::to_host() const { return buf_.to_host((size_t)n_, cs()); }

// ------------------------------------------------------------------ DenseMatrix ----------
RowBlock &RowBlock::operator=(const DenseMatrix &m) {
    require(m.rows() == nrows && m.cols() == ncols, "middleRows assignment: shape mismatch");
    d2d(ptr, m.data(), m.size());
    return *this;
}
DenseMatrix::DenseMatrix(const DenseMatrix &o) : buf_((size_t)o.size()), rows_(o.rows_), cols_(o.cols_) {
    d2d(data(), o.data(), size());
}
DenseMatrix &DenseMatrix::operator=(const DenseMatrix &o) {
    if (this != &o) {
        resize(o.rows_, o.cols_);
        d2d(data(), o.data(), size());
    }
    return *this;
}
DenseMatrix::DenseMatrix(const RowBlock &b) : buf_((size_t)b.size()), rows_(b.nrows), cols_(b.ncols) {
    d2d(data(), b.ptr, size());
}
DenseMatrix &DenseMatrix::operator=(const RowBlock &b) {
    resize(b.nrows, b.ncols);
    d2d(data(), b.ptr, size());
    return *this;
}
DenseMatrix DenseMatrix::Constant(int64_t rows, int64_t cols, double value) {
    DenseMatrix m(rows, cols);
    m.setConstant(value);
    return m;
}
void DenseMatrix::resize(int64_t rows, int64_t cols) {
    if (rows * cols != rows_ * cols_) buf_.resize((size_t)(rows * cols));
    rows_ = rows;
    cols_ = cols;
}
void DenseMatrix::take(DenseMatrix &o) {
    if (buf_.owns() && o.buf_.owns()) {
        swap(o);
        return;
    }
    require(o.size() == size(), "take: shape mismatch on a non-owning view");
    if (size())
        hnh::cuda_check(cudaMemcpyAsync(data(), o.data(), sizeof(double) * (size_t)size(), cudaMemcpyDeviceToDevice, cs()),
                        "DenseMatrix::take");
}
void DenseMatrix::setConstant(double v) { abi_check(hnh_fill_f64(data(), size(), v, cs()), "fill"); }
void DenseMatrix::setRandom(uint64_t seed) { abi_check(hnh_random_uniform_f64(data(), size(), seed, cs()), "random"); }
DenseMatrix &DenseMatrix::operator*=(double s) {
    abi_check(hnh_axpby_f64(data(), s, data(), 0.0, nullptr, size(), cs()), "scale");
    return *this;
}
DenseMatrix &DenseMatrix::operator+=(const DenseMatrix &o) {
    require(o.size() == size(), "operator+=: shape mismatch");
    abi_check(hnh_axpby_f64(data(), 1.0, data(), 1.0, o.data(), size(), cs()), "axpby");
    return *this;
}
DenseMatrix &DenseMatrix::operator-=(const DenseMatrix &o) {
    require(o.size() == size(), "operator-=: shape mismatch");
    abi_check(hnh_axpby_f64(data(), 1.0, data(), -1.0, o.data(), size(), cs()), "axpby");
    return *this;
}
DenseMatrix DenseMatrix::operator+(const DenseMatrix &o) const {
    DenseMatrix r(*this);
    r += o;
    return r;
}
DenseMatrix DenseMatrix::operator-(const DenseMatrix &o) const {
    DenseMatrix r(*this);
    r -= o;
    return r;
}
DenseMatrix::CwiseProduct DenseMatrix::cwiseProduct(const DenseMatrix &o) const {
    require(o.rows() == rows_ && o.cols() == cols_, "cwiseProduct: shape mismatch");
    return CwiseProduct{*this, o};
}
DenseMatrix::CwiseProduct::operator DenseMatrix() const {
    DenseMatrix r(a.rows(), a.cols());
    abi_check(hnh_hadamard_f64(r.data(), a.data(), b.data(), a.size(), cs()), "hadamard");
    return r;
}
VectorXd DenseMatrix::CwiseProduct::Rowwise::sum() const { return batch_dot_product(a, b); }
DenseMatrix operator*(double s, const DenseMatrix &m) {
    DenseMatrix r(m);
    r *= s;
    return r;
}
void DenseMatrix::setRandom() {
    // Eigen's setRandom() draws from the C library generator; here: the next seed of a fixed per-process sequence
    static uint64_t next = 0x5EED0000ull;
    setRandom(next++);
}
double DenseMatrix::squaredNorm() const {
    hnh::DeviceBuffer<double> out(1);
    abi_check(hnh_squared_norm_f64(out.data(), data(), size(), cs()), "squared_norm");
    return out.to_host(1, cs())[0];
}
void DenseMatrix::setRowAxpy(const DenseMatrix &c, double alpha, const VectorXd *s, const DenseMatrix &m) {
    require(c.rows() == m.rows() && c.cols() == m.cols(), "setRowAxpy: shape mismatch");
    require(!s || s->size() == m.rows(), "setRowAxpy: scale vector length");
    resize(c.rows(), c.cols());
    abi_check(hnh_row_axpy_f64(data(), c.data(), alpha, s ? s->data() : nullptr, m.data(), rows_, (int)cols_, cs()),
              "row_axpy");
}
DenseMatrix DenseMatrix::from_host(const double *h, int64_t rows, int64_t cols) {
    DenseMatrix m(rows, cols);
    m.copy_from_host(h);
    return m;
}
void DenseMatrix::copy_from_host(const double *h) {
    if (size()) cuda_check(cudaMemcpyAsync(data(), h, sizeof(double) * (size_t)size(), cudaMemcpyHostToDevice, cs()), "h2d");
    cuda_check(cudaStreamSynchronize(cs()), "sync");
}
void DenseMatrix::copy_to_host(double *h) const {
    if (size()) cuda_check(cudaMemcpyAsync(h, data(), sizeof(double) * (size_t)size(), cudaMemcpyDeviceToHost, cs()), "d2h");
    cuda_check(cudaStreamSynchronize(cs()), "sync");
}
vector<double> DenseMatrix::to_host() const { return buf_.to_host((size_t)size(), cs()); }

void VectorXd::leakyRelu(double alpha) {
    abi_check(hnh_leaky_relu_f64(data(), data(), n_, alpha, cs()), "leaky_relu");
}
DenseMatrix DenseMatrix::operator*(const DenseMatrix &o) const {
    require(cols_ == o.rows(), "matrix product: inner dimensions differ");
    DenseMatrix res(rows_, o.cols());
    abi_check(hnh_dgemm_f64(res.data(), data(), o.data(), rows_, o.cols(), cols_, cs()), "dgemm");
    return res;
}
void DenseMatrix::setMiddleColsRelu(int64_t start, const DenseMatrix &m) {
    require(m.rows() == rows_ && start >= 0 && start + m.cols() <= cols_, "middleCols assignment: shape mismatch");
    abi_check(hnh_relu_cols_f64(data(), cols_, start, m.data(), m.rows(), m.cols(), cs()), "relu_cols");
}
void VectorXd::leakyReluGrad(double alpha) {
    abi_check(hnh_leaky_relu_grad_f64(data(), data(), n_, alpha, cs()), "leaky_relu_grad");
}
void DenseMatrix::setTransposeTimes(const DenseMatrix &a, const DenseMatrix &b) {
    require(a.rows() == b.rows(), "transposed product: row counts differ");
    require(buf_.owns() || (rows_ == a.cols() && cols_ == b.cols()), "transposed product: shape mismatch on a view");
    resize(a.cols(), b.cols());
    const int64_t ws = hnh_dgemm_tn_workspace_bytes(a.cols(), b.cols(), a.rows());
    if (ws < 0) abi_check((int)ws, "dgemm_tn");
    hnh::DeviceBuffer<char> workspace((size_t)ws);  // from the caching allocator, released stream-ordered
    abi_check(hnh_dgemm_tn_f64(data(), a.data(), b.data(), a.cols(), b.cols(), a.rows(), workspace.data(), (size_t)ws, cs()),
              "dgemm_tn");
}
void DenseMatrix::setTimesTranspose(const DenseMatrix &a, const DenseMatrix &b, bool accumulate) {
    require(a.cols() == b.cols(), "product with a transpose: inner dimensions differ");
    if (accumulate || !buf_.owns())
        require(rows_ == a.rows() && cols_ == b.rows(), "product with a transpose: shape mismatch");
    resize(a.rows(), b.rows());
    abi_check(hnh_dgemm_nt_f64(data(), a.data(), b.data(), a.rows(), b.rows(), a.cols(), accumulate ? 1 : 0, cs()), "dgemm_nt");
}
void DenseMatrix::setMiddleColsReluGrad(const DenseMatrix &grad, const DenseMatrix &out, int64_t start) {
    require(grad.rows() == out.rows() && grad.cols() == out.cols() && rows_ == out.rows() && start >= 0 &&
                start + cols_ <= out.cols(),
            "middleCols ReLU gradient: shape mismatch");
    abi_check(hnh_relu_cols_backward_f64(data(), grad.data(), out.data(), out.cols(), start, rows_, cols_, cs()),
              "relu_cols_backward");
}

VectorXd batch_dot_product(const DenseMatrix &A, const DenseMatrix &B) {
    require(A.rows() == B.rows() && A.cols() == B.cols(), "batch_dot_product: shape mismatch");
    VectorXd r(A.rows());
    abi_check(hnh_batch_dot_f64(r.data(), A.data(), B.data(), A.rows(), (int)A.cols(), cs()), "batch_dot");
    return r;
}
DenseMatrix scale_matrix_rows(const VectorXd &scale_vector, const DenseMatrix &mat) {
    require(scale_vector.size() == mat.rows(), "scale_matrix_rows: scale vector length");
    DenseMatrix res(mat.rows(), mat.cols());
    abi_check(hnh_row_axpy_f64(res.data(), nullptr, 1.0, scale_vector.data(), mat.data(), mat.rows(),
                               (int)mat.cols(), cs()), "row_axpy");
    return res;
}
