// The packed arg-min key of the NN kernels: (ordered bits of the distance) << 32 | (32-bit index of the row of y).  Signed
// 64-bit key order is the (distance, index) order of raft::argmin_op, so an atomicMin, a sort or an NCCL MIN exchange
// keeps the smallest distance and, among equal ones, the smallest index.  KEY_EMPTY: no candidate yet.  (Python model:
// oracle.pack_minloc.)
#pragma once
#include <cuda_runtime.h>

namespace b2d {

constexpr long long KEY_EMPTY = 0x7FFFFFFFFFFFFFFFll;

// float -> int whose signed order equals the float order (its own inverse)
__device__ __forceinline__ int ordered_bits(float v)
{
  int b = __float_as_int(v);
  return b < 0 ? (b ^ 0x7FFFFFFF) : b;
}
__device__ __forceinline__ long long key_pack(float d, long long idx)
{
  return (static_cast<long long>(ordered_bits(d)) << 32) | (idx & 0xFFFFFFFFll);
}
__device__ __forceinline__ float key_dist(long long key) { return __int_as_float(ordered_bits(__int_as_float(static_cast<int>(key >> 32)))); }
__device__ __forceinline__ long long key_index(long long key) { return key & 0xFFFFFFFFll; }
// the distance as an upper bound of the row's minimum: +inf while the row has no candidate
__device__ __forceinline__ float key_bound(long long key)
{
  float d = key_dist(key);
  if (key == KEY_EMPTY) d = __int_as_float(0x7f800000);
  return d;
}

// raft::KeyValuePair<int, float> as the 1-NN entry points write it
struct KvpIF {
  int key;
  float value;
};

}  // namespace b2d
