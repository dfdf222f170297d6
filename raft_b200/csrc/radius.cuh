// Small kernels and iterator functors of radius_neighbors (radius.cu); the pairs themselves are found in the epilogue of
// the tensor kernel (expanded_tc.cuh, EPI_RADIUS).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "nn_key.cuh"

namespace b2d {

// a row degree (uint32) as the int64 the scan into indptr adds up
struct RadiusDeg64 {
  __host__ __device__ __forceinline__ long long operator()(unsigned d) const { return static_cast<long long>(d); }
};

// offset of CSR row i for the segmented sort, clipped to the nnz slots the caller gave: a segment never reaches past nnz
struct RadiusRowStart {
  const int64_t* indptr;
  long long nnz;
  __host__ __device__ __forceinline__ long long operator()(int64_t i) const
  {
    const long long v = indptr[i];
    return v < nnz ? v : nnz;
  }
};

// the sorted keys split into column indices and distances (keys may alias indices: each thread reads its key first)
__global__ void radius_split_kernel(const long long* keys, int64_t* indices, float* distances, int64_t nnz)
{
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < nnz;
       e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const long long key = keys[e];
    indices[e]          = key_index(key);
    distances[e]        = key_dist(key);
  }
}

}  // namespace b2d
