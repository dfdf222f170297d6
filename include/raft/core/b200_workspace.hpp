// Customization point for the temporaries of one shim call.  The C ABI never allocates; the reference's rule
// is that a primitive takes its scratch from the handle's workspace memory resource
// (cpp/include/raft/core/resource/device_memory_resource.hpp:100-129,187-203: a limiting adaptor over the
// current device resource, 1/4 of device memory by default).  So:
//   with real RAFT (RAFT_B200_USE_REAL_RAFT): an rmm::device_uvector<char> on
//       raft::resource::get_workspace_resource_ref(handle), stream-ordered on the handle's stream -- it is released
//       behind the kernels the call enqueued, exactly like the reference's own temporaries;
//   stand-alone: cudaMallocAsync / cudaFreeAsync on the same stream (the default pool keeps the memory, so the
//       steady state costs no driver call).
// Entry points without a handle (epsUnexpL2SqNeighborhood) take the stand-alone way on their stream in either build.
// Either way nothing synchronises and the scratch lives until the work enqueued so far has run.
#pragma once
#include <optional>

#include "b200_compat.hpp"
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/resource/device_memory_resource.hpp>
#include <rmm/device_uvector.hpp>
#endif

namespace raft {
namespace b200 {

class scoped_workspace {
 public:
#ifdef RAFT_B200_USE_REAL_RAFT
  scoped_workspace(raft::resources const& handle, std::size_t bytes)
  {
    buf_.emplace(bytes + 256, raft::resource::get_cuda_stream(handle), raft::resource::get_workspace_resource_ref(handle));
  }
#else
  scoped_workspace(raft::resources const& handle, std::size_t bytes)
    : scoped_workspace(raft::resource::get_cuda_stream(handle), bytes)
  {
  }
#endif
  // entry points that take a stream and no handle (the reference's pointer forms): cudaMallocAsync / cudaFreeAsync on
  // that stream, in either build
  scoped_workspace(cudaStream_t stream, std::size_t bytes) : stream_(stream)
  {
    if (bytes && cudaMallocAsync(&p_, bytes + 256, stream_) != cudaSuccess)
      throw raft::cuda_error("raft_b200: workspace allocation failed");
  }
  ~scoped_workspace()
  {
    if (p_) cudaFreeAsync(p_, stream_);
  }
  void* data()
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    if (buf_) return align(buf_->data());
#endif
    return align(p_);
  }
  scoped_workspace(const scoped_workspace&)            = delete;
  scoped_workspace& operator=(const scoped_workspace&) = delete;

 private:
  static void* align(void* p)  // the C ABI wants 256-byte aligned scratch
  {
    return reinterpret_cast<void*>((reinterpret_cast<std::uintptr_t>(p) + 255) & ~static_cast<std::uintptr_t>(255));
  }
  cudaStream_t stream_ = nullptr;
  void* p_             = nullptr;
#ifdef RAFT_B200_USE_REAL_RAFT
  std::optional<rmm::device_uvector<char>> buf_;
#endif
};

}  // namespace b200
}  // namespace raft
