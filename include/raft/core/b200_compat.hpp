// Minimal stand-in for the parts of raft/core that the distance shim needs, used ONLY when the real
// RAFT headers are not on the include path (RMM / CCCL 3 are not installable offline; SURVEY.md
// hard part F).  With real RAFT present, define RAFT_B200_USE_REAL_RAFT: the shim then includes
// <raft/core/resources.hpp>, <raft/core/resource/cuda_stream.hpp>, <raft/core/device_mdspan.hpp>,
// <raft/core/kvp.hpp>, <raft/core/error.hpp> itself and this file defines nothing
// (tests/test_cpp_shim.py compiles that configuration against tests/cpp/mock_raft, a header tree with the
// reference's signatures and NO members beyond them).
//
//   raft::resources + raft::resource::get_cuda_stream   cpp/include/raft/core/resources.hpp:38-128,
//                                                       cpp/include/raft/core/resource/cuda_stream.hpp:58-64
//   raft::row_major / col_major / device_matrix_view     cpp/include/raft/core/mdspan_types.hpp:19-32,
//                                                       cpp/include/raft/core/device_mdspan.hpp:94-97,169-176
//                                                       (aliases of cuda::std::mdspan, as here)
//   raft::KeyValuePair                                  cpp/include/raft/core/kvp.hpp:20-62
//   raft::logic_error / raft::cuda_error / RAFT_EXPECTS cpp/include/raft/core/error.hpp:218-239
// Temporaries: include/raft/core/b200_workspace.hpp (the counterpart of the handle's workspace resource).
#pragma once
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#include <raft/core/error.hpp>
#include <raft/core/kvp.hpp>
#include <raft/core/resource/cuda_stream.hpp>
#include <raft/core/resources.hpp>
#else
#include <cuda/std/mdspan>
#include <cuda_runtime_api.h>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>

namespace raft {

struct exception : std::runtime_error { using std::runtime_error::runtime_error; };
struct logic_error : exception { using exception::exception; };
struct cuda_error : exception { using exception::exception; };

#define RAFT_EXPECTS(cond, msg)                                   \
  do {                                                            \
    if (!(cond)) throw ::raft::logic_error(std::string("RAFT failure: ") + (msg)); \
  } while (0)

using cuda::std::dynamic_extent;
using cuda::std::extents;
using cuda::std::layout_left;
using cuda::std::layout_right;
using cuda::std::layout_stride;
using row_major = layout_right;
using col_major = layout_left;
template <typename IndexType>
using matrix_extent = cuda::std::extents<IndexType, dynamic_extent, dynamic_extent>;

// device_matrix_view<T, IdxT, Layout>: a 2-d cuda::std::mdspan (the reference adds an accessor that tags the
// memory as device memory; data_handle() / extent(i) / stride(i) are what the shim uses)
template <typename T, typename IdxT = std::uint32_t, typename Layout = row_major>
using device_matrix_view = cuda::std::mdspan<T, matrix_extent<IdxT>, Layout>;

template <typename T, typename IdxT = std::uint32_t, typename Layout = row_major>
auto constexpr make_device_matrix_view(T* p, IdxT rows, IdxT cols)
{
  return device_matrix_view<T, IdxT, Layout>{p, matrix_extent<IdxT>{rows, cols}};
}
// row-major view with a leading dimension (raft::make_device_strided_matrix_view, device_mdspan.hpp:178-199)
template <typename T, typename IdxT = std::uint32_t>
auto make_device_strided_matrix_view(T* p, IdxT rows, IdxT cols, IdxT ld)
{
  cuda::std::array<IdxT, 2> strides{ld, IdxT(1)};
  return device_matrix_view<T, IdxT, layout_stride>{
    p, typename layout_stride::template mapping<matrix_extent<IdxT>>{matrix_extent<IdxT>{rows, cols}, strides}};
}

// device_vector_view<T, IdxT, Layout>: a 1-d cuda::std::mdspan (device_mdspan.hpp, make_device_vector_view)
using layout_c_contiguous = row_major;
template <typename IndexType>
using vector_extent = cuda::std::extents<IndexType, dynamic_extent>;
template <typename T, typename IdxT = std::uint32_t, typename Layout = row_major>
using device_vector_view = cuda::std::mdspan<T, vector_extent<IdxT>, Layout>;

template <typename T, typename IdxT = std::uint32_t>
auto constexpr make_device_vector_view(T* p, IdxT n)
{
  return device_vector_view<T, IdxT>{p, vector_extent<IdxT>{n}};
}

template <typename K, typename V>
struct KeyValuePair {
  K key;
  V value;
};

// raft::resources: here just the stream (the reference keeps every resource behind get_*() free functions)
class resources {
 public:
  explicit resources(cudaStream_t s = nullptr) : stream_(s) {}
  resources(const resources&) = delete;
  cudaStream_t b200_stream() const { return stream_; }
 private:
  cudaStream_t stream_;
};
using device_resources = resources;
using handle_t         = resources;

namespace resource {
inline cudaStream_t get_cuda_stream(resources const& h) { return h.b200_stream(); }
inline void sync_stream(resources const& h)
{
  if (cudaStreamSynchronize(get_cuda_stream(h)) != cudaSuccess) throw cuda_error("cudaStreamSynchronize failed");
}
}  // namespace resource
}  // namespace raft
#endif
