// raft::distance::fusedL2NNMinReduce -- shim over b2d_fused_l2_nn (include/raft_b200.h).
// Signature of the removed raft/distance/fused_l2_nn.cuh (SURVEY.md 8(a5)); OutT is
// raft::KeyValuePair<IdxT, DataT> (cpp/include/raft/core/kvp.hpp:20-62) with IdxT = int,
// DataT = float; xn / yn are the SQUARED row norms; `workspace` (the reference's per-row mutex
// array) is accepted and ignored -- this implementation needs no mutex.
#pragma once
#include "distance.cuh"

namespace raft {
namespace distance {

template <typename DataT, typename OutT, typename IdxT>
void fusedL2NNMinReduce(OutT* min, const DataT* x, const DataT* y, const DataT* xn, const DataT* yn, IdxT m, IdxT n,
                        IdxT k, void* /*workspace*/, bool sqrt, bool initOutBuffer, raft::resources const& handle)
{
  static_assert(std::is_same<DataT, float>::value && sizeof(OutT) == sizeof(b2d_kvp_if),
                "raft_b200: fusedL2NN is provided for <float, KeyValuePair<int,float>, int>");
  const size_t need = b2d_fused_l2_nn_workspace_bytes(m, n, k);
  raft::b200::scoped_workspace ws(handle, need);
  detail::b2d_check(b2d_fused_l2_nn(raft::resource::get_cuda_stream(handle), reinterpret_cast<b2d_kvp_if*>(min), x, k, y,
                                    k, xn, yn, m, n, k, sqrt ? 1 : 0, initOutBuffer ? 1 : 0, ws.data(), need));
}

// Legacy stream-only signature (no handle): fusedL2NNMinReduce(min, x, y, xn, yn, m, n, k, workspace,
// sqrt, initOutBuffer, stream) as listed in SURVEY.md 8(a5).  The reference's `workspace` holds m
// ints for its per-row mutexes -- too small for the packed operands this engine stages -- so the
// scratch comes from the stream-ordered allocator and is returned to it behind the kernels.
template <typename DataT, typename OutT, typename IdxT>
void fusedL2NNMinReduce(OutT* min, const DataT* x, const DataT* y, const DataT* xn, const DataT* yn, IdxT m, IdxT n,
                        IdxT k, void* /*workspace*/, bool sqrt, bool initOutBuffer, cudaStream_t stream)
{
  static_assert(std::is_same<DataT, float>::value && sizeof(OutT) == sizeof(b2d_kvp_if),
                "raft_b200: fusedL2NN is provided for <float, KeyValuePair<int,float>, int>");
  const size_t need = b2d_fused_l2_nn_workspace_bytes(m, n, k);
  raft::b200::scoped_workspace ws(stream, need);
  detail::b2d_check(b2d_fused_l2_nn(stream, reinterpret_cast<b2d_kvp_if*>(min), x, k, y, k, xn, yn, m, n, k, sqrt ? 1 : 0,
                                    initOutBuffer ? 1 : 0, ws.data(), need));
}

// ---------------------------------------------------------------------------------------------
// Generic form: fusedL2NN<DataT, OutT, IdxT, ReduceOpT, KVPReduceOpT> (SURVEY.md 8(a5); existence / shape:
// cpp/include/raft/linalg/contractions.cuh:170-175, CHANGELOG.md:1371-1372,1525).  OutT is
// raft::KeyValuePair<IdxT, DataT> or DataT; redOp(row, OutT* out, KVP candidate) folds a candidate into out and
// redOp.init(OutT* out, DataT maxVal) resets it ([RECALLED] functor protocol of the removed header; the two stock
// functors are restated below).  A functor cannot cross the C ABI, so the engine computes the per-row
// {arg-min, min} (ties -> smaller index, raft::argmin_op) and the caller's redOp is applied ONCE per row to that
// winner, on the device, on the same stream.  That equals folding every candidate for any reduction that keeps the
// minimum-distance candidate -- MinAndDistanceReduceOp, MinReduceOp and user functors built on them; pairRedOp (the
// in-tile KVP reduction of the reference kernel) is accepted for signature compatibility and must be a minimum too.
template <typename LabelT, typename DataT>
struct KVPMinReduce {
  typedef raft::KeyValuePair<LabelT, DataT> KVP;
  __host__ __device__ KVP operator()(LabelT, const KVP& a, const KVP& b) const
  {
    return (b.value < a.value || (b.value == a.value && b.key < a.key)) ? b : a;
  }
};
template <typename LabelT, typename DataT>
struct MinAndDistanceReduceOp {
  typedef raft::KeyValuePair<LabelT, DataT> KVP;
  __host__ __device__ void operator()(LabelT, KVP* out, const KVP& other) const
  {
    if (other.value < out->value || (other.value == out->value && other.key < out->key)) *out = other;
  }
  __host__ __device__ void operator()(LabelT, DataT* out, const KVP& other) const
  {
    if (other.value < *out) *out = other.value;
  }
  __host__ __device__ void init(DataT* out, DataT maxVal) const { *out = maxVal; }
  __host__ __device__ void init(KVP* out, DataT maxVal) const { out->key = 0; out->value = maxVal; }
};
template <typename LabelT, typename DataT>
struct MinReduceOp {
  typedef raft::KeyValuePair<LabelT, DataT> KVP;
  __host__ __device__ void operator()(LabelT, DataT* out, const KVP& other) const
  {
    if (other.value < *out) *out = other.value;
  }
  __host__ __device__ void init(DataT* out, DataT maxVal) const { *out = maxVal; }
};

#ifdef __CUDACC__
namespace detail {
template <typename OutT, typename IdxT, typename DataT, typename ReduceOpT>
__global__ void b2d_apply_reduce_kernel(OutT* min, const b2d_kvp_if* nn, IdxT m, ReduceOpT redOp, bool init, DataT maxVal)
{
  const IdxT i = static_cast<IdxT>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  if (init) redOp.init(min + i, maxVal);
  if (nn[i].key == 0x7fffffff) return;  // no candidate (n == 0)
  raft::KeyValuePair<IdxT, DataT> c;
  c.key   = static_cast<IdxT>(nn[i].key);
  c.value = nn[i].value;
  redOp(i, min + i, c);
}
}  // namespace detail

template <typename DataT, typename OutT, typename IdxT, typename ReduceOpT, typename KVPReduceOpT>
void fusedL2NN(OutT* min, const DataT* x, const DataT* y, const DataT* xn, const DataT* yn, IdxT m, IdxT n, IdxT k,
               void* /*workspace*/, ReduceOpT redOp, KVPReduceOpT /*pairRedOp*/, bool sqrt, bool initOutBuffer,
               cudaStream_t stream)
{
  static_assert(std::is_same<DataT, float>::value && sizeof(IdxT) == 4, "raft_b200: fusedL2NN is provided for DataT = float, 32-bit IdxT");
  const size_t need = b2d_fused_l2_nn_workspace_bytes(m, n, k);
  const size_t kvpb = (static_cast<size_t>(m) * sizeof(b2d_kvp_if) + 255) / 256 * 256;
  raft::b200::scoped_workspace ws(stream, kvpb + need);   // the per-row arg-min in front of the engine's scratch
  char* base     = static_cast<char*>(ws.data());
  b2d_kvp_if* nn = reinterpret_cast<b2d_kvp_if*>(base);
  const int st   = b2d_fused_l2_nn(stream, nn, x, k, y, k, xn, yn, m, n, k, sqrt ? 1 : 0, 1, base + kvpb, need);
  if (st == B2D_OK && m > 0)
    detail::b2d_apply_reduce_kernel<OutT, IdxT, DataT, ReduceOpT><<<static_cast<unsigned>((m + 255) / 256), 256, 0, stream>>>(
      min, nn, m, redOp, initOutBuffer, 3.402823466e+38f);
  detail::b2d_check(st);
}
#endif  // __CUDACC__

// raft::distance::fusedDistanceNNMinReduce: L2 (sqrt flag) or cosine, SURVEY.md 8(f1)
template <typename DataT, typename OutT, typename IdxT>
void fusedDistanceNNMinReduce(OutT* min, const DataT* x, const DataT* y, const DataT* xn, const DataT* yn, IdxT m, IdxT n,
                              IdxT k, void* /*workspace*/, bool sqrt, bool initOutBuffer, bool /*isRowMajor*/,
                              raft::distance::DistanceType metric, float /*metric_arg*/, raft::resources const& handle)
{
  static_assert(std::is_same<DataT, float>::value && sizeof(OutT) == sizeof(b2d_kvp_if), "float / KeyValuePair<int,float>");
  int mt = static_cast<int>(metric);
  if (metric == DistanceType::L2Expanded && sqrt) mt = static_cast<int>(DistanceType::L2SqrtExpanded);
  const size_t need = b2d_fused_l2_nn_workspace_bytes(m, n, k);
  raft::b200::scoped_workspace ws(handle, need);
  detail::b2d_check(b2d_fused_distance_nn(raft::resource::get_cuda_stream(handle), reinterpret_cast<b2d_kvp_if*>(min), mt,
                                          x, k, y, k, xn, yn, m, n, k, initOutBuffer ? 1 : 0, ws.data(), need));
}

}  // namespace distance
}  // namespace raft
