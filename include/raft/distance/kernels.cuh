// raft::distance::kernels -- header-only shim of the removed raft/distance/kernels.cuh ([RECALLED], <= 25.12): the kernel
// Gram matrices of cuML's SVM, dispatching through b2d_gram_matrix (include/raft_b200.h).  For x1 [n1, k], x2 [n2, k]:
//   GramMatrixBase       out = <x1_i, x2_j>                              (the linear kernel)
//   PolynomialKernel     out = (gain <x1_i, x2_j> + offset)^exponent     (integer exponent >= 0)
//   TanhKernel           out = tanh(gain <x1_i, x2_j> + offset)
//   RBFKernel            out = exp(-gain ||x1_i - x2_j||^2)
// Dense inputs only (the CSR overloads are not provided).  Row- or column-major, with leading dimensions; float (fp32
// on the tensor path, parameters used as float) or double (the fp64 path).  Asynchronous like every shim call.
#pragma once
#include "distance.cuh"

namespace raft {
namespace distance {
namespace kernels {

template <typename math_t>
class GramMatrixBase {
 public:
  GramMatrixBase() = default;
  virtual ~GramMatrixBase() = default;

  /**
   * mdspan form: out [n1, n2] = K(x1 [n1, k], x2 [n2, k]) on the handle's stream, scratch from its workspace.  x1, x2 and
   * out share one layout (row- or column-major; strided views with unit stride along one dimension).  norm_x1 / norm_x2
   * are accepted for source compatibility and ignored: the squared norms are computed with the operands.
   */
  template <typename IdxT, typename Layout1, typename Layout2, typename LayoutO>
  void operator()(raft::resources const& handle, raft::device_matrix_view<const math_t, IdxT, Layout1> x1,
                  raft::device_matrix_view<const math_t, IdxT, Layout2> x2, raft::device_matrix_view<math_t, IdxT, LayoutO> out,
                  math_t* norm_x1 = nullptr, math_t* norm_x2 = nullptr)
  {
    (void)norm_x1;
    (void)norm_x2;
    RAFT_EXPECTS(x1.extent(1) == x2.extent(1), "Number of columns must be equal.");
    RAFT_EXPECTS(out.extent(0) == x1.extent(0) && out.extent(1) == x2.extent(0), "out must be [rows of x1, rows of x2]");
    bool r1, r2, ro;
    int64_t ld1, ld2, ldo;
    raft::distance::detail::view_layout(x1, r1, ld1);
    raft::distance::detail::view_layout(x2, r2, ld2);
    raft::distance::detail::view_layout(out, ro, ldo);
    RAFT_EXPECTS(r1 == r2 && r1 == ro, "gram matrix: x1, x2 and out must share one layout (all row- or all column-major)");
    const int64_t n1 = x1.extent(0), n2 = x2.extent(0), k = x1.extent(1);
    const size_t need = workspace_bytes(n1, n2, k);
    raft::b200::scoped_workspace ws(handle, need);
    run(raft::resource::get_cuda_stream(handle), x1.data_handle(), ld1, x2.data_handle(), ld2, out.data_handle(), ldo, n1,
        n2, k, r1, ws.data(), need);
  }

  /**
   * Legacy pointer form: out [n1, n2] = K(x1 [n1, n_cols], x2 [n2, n_cols]) on `stream`, leading dimensions ld1 / ld2 /
   * ld_out (0: dense).  It takes no handle, so its scratch is allocated stream-ordered on `stream`
   * (raft::b200::scoped_workspace).
   */
  void evaluate(const math_t* x1, int n1, int n_cols, const math_t* x2, int n2, math_t* out, bool is_row_major,
                cudaStream_t stream, int ld1 = 0, int ld2 = 0, int ld_out = 0)
  {
    if (ld1 <= 0) ld1 = is_row_major ? n_cols : n1;
    if (ld2 <= 0) ld2 = is_row_major ? n_cols : n2;
    if (ld_out <= 0) ld_out = is_row_major ? n2 : n1;
    const size_t need = workspace_bytes(n1, n2, n_cols);
    raft::b200::scoped_workspace ws(stream, need);
    run(stream, x1, ld1, x2, ld2, out, ld_out, n1, n2, n_cols, is_row_major, ws.data(), need);
  }

 protected:
  GramMatrixBase(int kernel, int degree, double gamma, double coef0)
    : kernel_(kernel), degree_(degree), gamma_(gamma), coef0_(coef0)
  {
  }

 private:
  size_t workspace_bytes(int64_t n1, int64_t n2, int64_t k) const
  {
    const size_t need = b2d_gram_matrix_workspace_bytes(kernel_, raft::distance::detail::b2d_dtype<math_t>(), n1, n2, k);
    RAFT_EXPECTS(need != SIZE_MAX, "gram matrix: invalid extents");
    return need;
  }
  void run(cudaStream_t stream, const math_t* x1, int64_t ld1, const math_t* x2, int64_t ld2, math_t* out, int64_t ldo,
           int64_t n1, int64_t n2, int64_t k, bool row_major, void* ws, size_t ws_bytes) const
  {
    raft::distance::detail::b2d_check(b2d_gram_matrix(stream, kernel_, degree_, gamma_, coef0_,
                                                      raft::distance::detail::b2d_dtype<math_t>(), x1, ld1, x2, ld2, out, ldo,
                                                      n1, n2, k, row_major ? 1 : 0, ws_bytes ? ws : nullptr, ws_bytes));
  }

  int kernel_    = B2D_KERNEL_LINEAR;
  int degree_    = 0;
  double gamma_  = 1.0;
  double coef0_  = 0.0;
};

template <typename math_t, typename exp_t>
class PolynomialKernel : public GramMatrixBase<math_t> {
 public:
  PolynomialKernel(exp_t exponent, math_t gain, math_t offset)
    : GramMatrixBase<math_t>(B2D_KERNEL_POLYNOMIAL, static_cast<int>(exponent), gain, offset)
  {
  }
};

template <typename math_t>
class TanhKernel : public GramMatrixBase<math_t> {
 public:
  TanhKernel(math_t gain, math_t offset) : GramMatrixBase<math_t>(B2D_KERNEL_TANH, 0, gain, offset) {}
};

template <typename math_t>
class RBFKernel : public GramMatrixBase<math_t> {
 public:
  explicit RBFKernel(math_t gain) : GramMatrixBase<math_t>(B2D_KERNEL_RBF, 0, gain, 0.0) {}
};

template <typename math_t>
class KernelFactory {
 public:
  // a new kernel object for params (the caller deletes it, as with the reference's factory)
  static GramMatrixBase<math_t>* create(KernelParams params)
  {
    switch (params.kernel) {
      case LINEAR: return new GramMatrixBase<math_t>();
      case POLYNOMIAL:
        return new PolynomialKernel<math_t, int>(params.degree, static_cast<math_t>(params.gamma),
                                                 static_cast<math_t>(params.coef0));
      case TANH: return new TanhKernel<math_t>(static_cast<math_t>(params.gamma), static_cast<math_t>(params.coef0));
      case RBF: return new RBFKernel<math_t>(static_cast<math_t>(params.gamma));
      default: throw raft::logic_error("Kernel not implemented");
    }
  }
};

}  // namespace kernels
}  // namespace distance
}  // namespace raft
