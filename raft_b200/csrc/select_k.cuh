// raft::matrix::select_k: exact per-row top-k of an fp32 matrix by radix selection (DESIGN.md section 2, K9).
//
// Order: the float order with -0.0 == +0.0 and every NaN above +inf; select_min takes the smallest, !select_min the
// largest, and among equal values the smaller column wins.  Both directions become one ascending order on the 64-bit
// word (select_key(v) << 32) | column, which has no ties, so the k-th word is unique and the k results are exactly
// the words <= it.  The k-th word is found one digit at a time, most significant first, in 11/11/10/11/11/10-bit
// passes; the three column passes only run for rows whose k-th key value is shared by more elements than are still
// needed.  A pass histograms the digit over the live words (those matching every digit fixed so far) and picks the
// bucket holding the k-th one; the words below that bucket are taken by the next read, the ones in it stay live.  A row
// is done as soon as its chosen bucket is taken whole.  The k results are then sorted as words, so every row comes out
// best first, equal values in ascending column order; the returned values are re-read from the input, bit for bit.
#pragma once
#include <cooperative_groups.h>
#include <cstdint>
#include <cstring>
#include <cub/block/block_scan.cuh>
#include <cuda_runtime.h>

namespace b2d {

// The selection order as an unsigned key: ascending key order is the order of the selection (so it is inverted for a
// max selection).  -0.0 maps to the key of +0.0 and every NaN to the key above +inf.  The one definition of the order.
__host__ __device__ __forceinline__ uint32_t select_key(float v, bool select_min)
{
  uint32_t b;
#ifdef __CUDA_ARCH__
  b = __float_as_uint(v);
#else
  std::memcpy(&b, &v, sizeof b);
#endif
  uint32_t key;
  if ((b & 0x7fffffffu) > 0x7f800000u) {
    key = 0xffffffffu;
  } else {
    if (b == 0x80000000u) b = 0;
    key = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  }
  return select_min ? key : ~key;
}

constexpr int kSkPasses   = 6;
constexpr int kSkBuckets  = 2048;
constexpr int kSkThreads  = 512;      // block of every radix kernel (4 buckets per thread in the scan)
constexpr int kSkSortMax  = 4096;     // k up to this is sorted in shared memory; above, by cub's segmented radix sort
constexpr int kSkRowSort  = 2048;     // rows up to this long are sorted whole in shared memory
constexpr int kSkRowSmem  = 100 * 1024;   // shared memory of the one-CTA-per-row radix kernel (two CTAs per SM)

__host__ __device__ constexpr int sk_shift(int p) { return p == 0 ? 53 : p == 1 ? 42 : p == 2 ? 32 : p == 3 ? 21 : p == 4 ? 10 : 0; }
__host__ __device__ constexpr int sk_bits(int p) { return (p == 2 || p == 5) ? 10 : 11; }

__device__ __forceinline__ uint64_t sk_word(float v, uint32_t col, bool select_min)
{
  return (static_cast<uint64_t>(select_key(v, select_min)) << 32) | col;
}

// Per-row selection state.  npass digits of `tgt` are fixed; k_rem of the words still live are needed; done: every live
// word is taken (the last chosen bucket held exactly k_rem words).  nout counts the words emitted so far.
struct SkState {
  uint64_t tgt;
  uint32_t k_rem;
  uint32_t npass;
  uint32_t done;
  uint32_t nout;
};

// How a word stands after the passes of `st`: 0 rejected or taken by an earlier read, 1 taken now, 2 live.  fin: the
// selection is complete (done), so every live word is taken.
struct SkClass {
  uint64_t t, tpre;
  int sh, bits;
  bool all_live, fin;
  __device__ __forceinline__ SkClass(const SkState& st, bool final_read)
  {
    all_live = st.npass == 0;
    fin      = final_read;
    const int L = all_live ? 0 : static_cast<int>(st.npass) - 1;
    sh = sk_shift(L);
    bits = sk_bits(L);
    t    = st.tgt >> sh;
    tpre = t >> bits;
  }
  __device__ __forceinline__ int operator()(uint64_t v) const
  {
    if (all_live) return fin ? 1 : 2;
    const uint64_t hi = v >> sh;
    if ((hi >> bits) != tpre) return 0;
    if (hi < t) return 1;
    if (hi == t) return fin ? 1 : 2;
    return 0;
  }
};

// warp-aggregated slot reservation: one shared or global atomic per group of converged lanes
__device__ __forceinline__ uint32_t sk_reserve(uint32_t* counter)
{
  namespace cg = cooperative_groups;
  cg::coalesced_group g = cg::coalesced_threads();
  uint32_t base = 0;
  if (g.thread_rank() == 0) base = atomicAdd(counter, g.size());
  return g.shfl(base, 0) + g.thread_rank();
}

// histogram count, aggregated over the converged lanes that hit the same bucket (rows of equal values would otherwise
// serialise on one shared-memory address)
__device__ __forceinline__ void sk_count(uint32_t* hist, uint32_t b)
{
  namespace cg = cooperative_groups;
  cg::coalesced_group peers = cg::labeled_partition(cg::coalesced_threads(), b);
  if (peers.thread_rank() == 0) atomicAdd(hist + b, peers.size());
}

__device__ __forceinline__ uint32_t sk_digit(uint64_t v, int p)
{
  return static_cast<uint32_t>(v >> sk_shift(p)) & ((1u << sk_bits(p)) - 1);
}

// f(value, column) for every column of x in [c0, c1): the block's threads, 16-byte loads, four in flight per thread
template <class F>
__device__ __forceinline__ void sk_for_each(const float* __restrict__ x, int64_t c0, int64_t c1, F&& f)
{
  const int64_t mis = static_cast<int64_t>((reinterpret_cast<uintptr_t>(x + c0) >> 2) & 3);
  const int64_t h   = c0 + ((4 - mis) & 3) < c1 ? c0 + ((4 - mis) & 3) : c1;
  for (int64_t i = c0 + threadIdx.x; i < h; i += blockDim.x) f(x[i], static_cast<uint32_t>(i));
  const int64_t nv    = (c1 - h) >> 2;
  const float4* xv    = reinterpret_cast<const float4*>(x + h);
  const int64_t bd    = blockDim.x;
  int64_t j = threadIdx.x;
  for (; j + 3 * bd < nv; j += 4 * bd) {
    float4 q[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) q[u] = xv[j + u * bd];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const uint32_t c = static_cast<uint32_t>(h + 4 * (j + u * bd));
      f(q[u].x, c);
      f(q[u].y, c + 1);
      f(q[u].z, c + 2);
      f(q[u].w, c + 3);
    }
  }
  for (; j < nv; j += bd) {
    const float4 q   = xv[j];
    const uint32_t c = static_cast<uint32_t>(h + 4 * j);
    f(q.x, c);
    f(q.y, c + 1);
    f(q.z, c + 2);
    f(q.w, c + 3);
  }
  for (int64_t i = h + 4 * nv + threadIdx.x; i < c1; i += blockDim.x) f(x[i], static_cast<uint32_t>(i));
}

// The bucket of the k_rem-th live word of a 2048-bucket histogram in shared memory: out = {bucket, live words in the
// buckets below it, words in it}.  Every thread of the (kSkThreads) block calls it; out is valid after it returns.
__device__ __forceinline__ void sk_find_bucket(const uint32_t* hist, uint32_t k_rem, uint32_t* out)
{
  constexpr int per = kSkBuckets / kSkThreads;
  using Scan = cub::BlockScan<uint32_t, kSkThreads>;
  __shared__ typename Scan::TempStorage tmp;
  uint32_t c[per], sum = 0;
#pragma unroll
  for (int j = 0; j < per; ++j) {
    c[j] = hist[threadIdx.x * per + j];
    sum += c[j];
  }
  uint32_t before;
  Scan(tmp).ExclusiveSum(sum, before);
  if (before < k_rem && k_rem <= before + sum) {
#pragma unroll
    for (int j = 0; j < per; ++j) {
      if (k_rem <= before + c[j]) {
        out[0] = threadIdx.x * per + j;
        out[1] = before;
        out[2] = c[j];
        break;
      }
      before += c[j];
    }
  }
  __syncthreads();
}

// fix digit p of the state from the bucket found in its histogram
__device__ __forceinline__ void sk_advance(SkState& st, int p, const uint32_t* found)
{
  st.tgt |= static_cast<uint64_t>(found[0]) << sk_shift(p);
  st.k_rem -= found[1];
  st.npass = p + 1;
  st.done  = found[2] == st.k_rem;
}

// block-wide ascending bitonic sort of n (a power of two) words in shared memory; the caller has synchronised
__device__ __forceinline__ void sk_bitonic(uint64_t* s, int n)
{
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < n / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const uint64_t a = s[lo], b = s[hi];
        if ((a > b) == up) {
          s[lo] = b;
          s[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

// k sorted words of one row -> values (re-read from the row, so the input bits come back unchanged) and indices
__device__ __forceinline__ void sk_write_row(const uint64_t* w, int64_t k, const float* x, const int64_t* idx, float* ov,
                                             int64_t* oi)
{
  for (int64_t i = threadIdx.x; i < k; i += blockDim.x) {
    const uint32_t col = static_cast<uint32_t>(w[i]);
    ov[i] = x[col];
    oi[i] = idx ? idx[col] : static_cast<int64_t>(col);
  }
}

__host__ __device__ constexpr int sk_pow2(int64_t n)
{
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// Rows of at most kSkRowSort elements: the whole row is sorted as words in shared memory (n = its power-of-two size).
__global__ void __launch_bounds__(1024) select_k_sort_row_kernel(const float* __restrict__ in, int64_t ld, int64_t len,
                                                                 int64_t k, int select_min, const int64_t* __restrict__ in_idx,
                                                                 float* __restrict__ out_val, int64_t* __restrict__ out_idx,
                                                                 int n)
{
  extern __shared__ __align__(16) unsigned char sk_sm_sort[];
  uint64_t* s = reinterpret_cast<uint64_t*>(sk_sm_sort);
  const int64_t row = blockIdx.x;
  const float* x    = in + row * ld;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    s[i] = i < len ? sk_word(x[i], static_cast<uint32_t>(i), select_min) : ~0ull;
  __syncthreads();
  sk_bitonic(s, n);
  sk_write_row(s, k, x, in_idx ? in_idx + row * ld : nullptr, out_val + row * k, out_idx + row * k);
}

// One CTA per row.  Shared memory: the histogram, the sort area (sort_n words; 0 when the results go to `list`) and a
// buffer of `cap` live words.  The first read whose live words fit the buffer copies them there, and every later read
// takes the buffer instead of the row: a row of at most `cap` elements is read from memory once, a longer row twice
// when the live words after the first digit fit.
__global__ void __launch_bounds__(kSkThreads, 2) select_k_radix_row_kernel(
  const float* __restrict__ in, int64_t ld, int64_t len, int64_t k, int select_min, const int64_t* __restrict__ in_idx,
  float* __restrict__ out_val, int64_t* __restrict__ out_idx, int sort_n, int cap, uint64_t* __restrict__ list)
{
  extern __shared__ __align__(16) unsigned char sk_sm_row[];
  uint32_t* hist = reinterpret_cast<uint32_t*>(sk_sm_row);
  uint64_t* res  = reinterpret_cast<uint64_t*>(hist + kSkBuckets);
  uint64_t* buf  = res + sort_n;
  __shared__ SkState st;
  __shared__ uint32_t found[3], nbuf, live;
  __shared__ int buf_ok;
  const int64_t row = blockIdx.x;
  const float* x    = in + row * ld;
  uint64_t* out     = list ? list + row * k : res;
  if (threadIdx.x == 0) {
    st     = SkState{0, static_cast<uint32_t>(k), 0, 0, 0};
    live   = static_cast<uint32_t>(len);
    nbuf   = 0;
    buf_ok = 0;
  }
  for (int p = 0; p <= kSkPasses; ++p) {
    for (int b = threadIdx.x; b < kSkBuckets; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    const bool fin  = p == kSkPasses || st.done;
    const bool fill = !fin && !buf_ok && live <= static_cast<uint32_t>(cap);
    const SkClass cls(st, fin);
    auto visit = [&](uint64_t v) {
      const int c = cls(v);
      if (c == 1) {
        out[sk_reserve(&st.nout)] = v;
      } else if (c == 2) {
        sk_count(hist, sk_digit(v, p));
        if (fill) buf[sk_reserve(&nbuf)] = v;
      }
    };
    if (buf_ok) {
      for (uint32_t i = threadIdx.x; i < nbuf; i += blockDim.x) visit(buf[i]);
    } else {
      sk_for_each(x, 0, len, [&](float v, uint32_t col) { visit(sk_word(v, col, select_min)); });
    }
    __syncthreads();
    if (fin) break;
    if (fill && threadIdx.x == 0) buf_ok = 1;
    sk_find_bucket(hist, st.k_rem, found);
    if (threadIdx.x == 0) {
      sk_advance(st, p, found);
      live = found[2];
    }
    __syncthreads();
  }
  if (list) return;
  for (int i = static_cast<int>(k) + threadIdx.x; i < sort_n; i += blockDim.x) res[i] = ~0ull;
  __syncthreads();
  sk_bitonic(res, sort_n);
  sk_write_row(res, k, x, in_idx ? in_idx + row * ld : nullptr, out_val + row * k, out_idx + row * k);
}

// Few long rows: each row is split over gridDim.x CTAs of `chunk` columns, the histograms are merged in global memory
// and every pass is one launch of this kernel (pass = kSkPasses: the final read) and one of select_k_split_scan_kernel.
// A row that is done skips the remaining passes; the launch sequence itself is fixed.
__global__ void __launch_bounds__(kSkThreads) select_k_split_read_kernel(const float* __restrict__ in, int64_t ld,
                                                                         int64_t len, int64_t chunk, int64_t k,
                                                                         int select_min, SkState* st, uint32_t* ghist,
                                                                         uint64_t* __restrict__ list, int p)
{
  __shared__ uint32_t hist[kSkBuckets];
  const int64_t row = blockIdx.y;
  const SkState s   = st[row];
  const bool fin    = p == kSkPasses;
  if (!fin && s.done) return;
  const int64_t c0 = blockIdx.x * chunk, c1 = c0 + chunk < len ? c0 + chunk : len;
  for (int b = threadIdx.x; b < kSkBuckets; b += blockDim.x) hist[b] = 0;
  __syncthreads();
  const SkClass cls(s, fin);
  uint64_t* out = list + row * k;
  sk_for_each(in + row * ld, c0, c1, [&](float v, uint32_t col) {
    const uint64_t w = sk_word(v, col, select_min);
    const int c      = cls(w);
    if (c == 1)
      out[sk_reserve(&st[row].nout)] = w;
    else if (c == 2)
      sk_count(hist, sk_digit(w, p));
  });
  if (fin) return;
  __syncthreads();
  uint32_t* g = ghist + row * kSkBuckets;
  for (int b = threadIdx.x; b < kSkBuckets; b += blockDim.x)
    if (hist[b]) atomicAdd(g + b, hist[b]);
}

// pass p of the split layout: one CTA per row picks the bucket from the merged histogram and clears it for pass p + 1
__global__ void __launch_bounds__(kSkThreads) select_k_split_scan_kernel(SkState* st, uint32_t* ghist, int64_t k, int p)
{
  __shared__ uint32_t hist[kSkBuckets];
  __shared__ uint32_t found[3];
  const int64_t row = blockIdx.x;
  SkState s         = st[row];
  if (s.done) return;
  uint32_t* g = ghist + row * kSkBuckets;
  for (int b = threadIdx.x; b < kSkBuckets; b += blockDim.x) {
    hist[b] = g[b];
    g[b]    = 0;
  }
  if (p == 0) s.k_rem = static_cast<uint32_t>(k);
  __syncthreads();
  sk_find_bucket(hist, s.k_rem, found);
  if (threadIdx.x == 0) {
    sk_advance(s, p, found);
    st[row] = s;
  }
}

// the k unsorted words of every row in `list` -> sorted in shared memory (sort_n >= k, a power of two) and written out
__global__ void __launch_bounds__(kSkThreads) select_k_sort_list_kernel(const uint64_t* __restrict__ list,
                                                                        const float* __restrict__ in, int64_t ld, int64_t k,
                                                                        const int64_t* __restrict__ in_idx,
                                                                        float* __restrict__ out_val,
                                                                        int64_t* __restrict__ out_idx, int sort_n)
{
  extern __shared__ __align__(16) unsigned char sk_sm_list[];
  uint64_t* s       = reinterpret_cast<uint64_t*>(sk_sm_list);
  const int64_t row = blockIdx.x;
  for (int i = threadIdx.x; i < sort_n; i += blockDim.x) s[i] = i < k ? list[row * k + i] : ~0ull;
  __syncthreads();
  sk_bitonic(s, sort_n);
  sk_write_row(s, k, in + row * ld, in_idx ? in_idx + row * ld : nullptr, out_val + row * k, out_idx + row * k);
}

// rows [r0, r0 + rows) whose words cub sorted into `w` ([rows, k]) -> values and indices
__global__ void select_k_gather_kernel(const uint64_t* __restrict__ w, const float* __restrict__ in, int64_t ld, int64_t k,
                                       const int64_t* __restrict__ in_idx, float* __restrict__ out_val,
                                       int64_t* __restrict__ out_idx, int64_t r0, int64_t rows)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= rows * k) return;
  const int64_t row = r0 + i / k;
  const uint32_t col = static_cast<uint32_t>(w[i]);
  out_val[r0 * k + i] = in[row * ld + col];
  out_idx[r0 * k + i] = in_idx ? in_idx[row * ld + col] : static_cast<int64_t>(col);
}

__global__ void select_k_offsets_kernel(int* off, int64_t n, int64_t k)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i <= n) off[i] = static_cast<int>(i * k);
}

}  // namespace b2d
