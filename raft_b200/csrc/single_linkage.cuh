// raft::cluster::single_linkage (DESIGN.md section 2, K13): single-linkage clustering on the kNN graph.  This file holds
// the edge-list Borůvka MST and the small kernels of connect_components; the kNN graph comes from the fused kNN
// (EPI_TOPK), the 1-NN across components from the masked arg-min (EPI_MINLOC_MASKED), the sort of the rows by component
// from the k-means counting sort (kmeans.cuh).
//
// Edge order: edge e of weight w has the key key_pack(w, e) = (ordered_bits(w) << 32) | e, a strict total order, so
// the minimum spanning forest is unique and every atomicMin below is order independent.
// One Borůvka round (every kernel returns at once when the run word is 0):
//   sl_round_begin_kernel   best[v] <- KEY_EMPTY, jump flags <- 0
//   sl_edge_kernel          every edge between two components: atomicMin of its key into both components' slots
//   sl_hook_kernel          every component with an edge hooks to the other side; in a mutual pair the smaller id stays
//                           root.  The edge is appended to the forest once (by the side that is not the larger id of a
//                           mutual pair).
//   sl_jump_kernel          pointer jumping on the hook forest; launch j returns at once when launch j - 1 changed nothing
//   sl_relabel_kernel       colour[v] <- root of colour[v]
//   sl_round_end_kernel     no edge appended in this round: the run word goes to 0
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "nn_key.cuh"

namespace b2d {

constexpr int kSlMaxJumps = 40;   // jump launches per round: ceil(log2 n) + 1 <= 32 for n < 2^31

struct SlCtrl {
  unsigned run;     // 1 while rounds still merge (the run word of every round kernel)
  unsigned n_mst;   // forest edges chosen so far
  unsigned prev;    // n_mst at the end of the previous round
  unsigned bad;     // single_linkage: bit 0 a non-finite value in X, bit 1 a component without a connecting edge
  unsigned jump[kSlMaxJumps];   // jump launch j of this round changed a parent
};

__device__ __forceinline__ bool sl_running(const SlCtrl* c) { return *reinterpret_cast<const volatile unsigned*>(&c->run) != 0u; }

// every vertex its own component, the forest's key list empty, counters 0, run word 1
__global__ void sl_mst_init_kernel(SlCtrl* ctrl, int* colour, long long* mst_keys, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) {
    colour[v]   = static_cast<int>(v);
    mst_keys[v] = KEY_EMPTY;
  }
  if (v == 0) { ctrl->run = 1u; ctrl->n_mst = 0u; ctrl->prev = 0u; ctrl->bad = 0u; }
}

// run word 1 again before the rounds over newly appended edges
__global__ void sl_rearm_kernel(SlCtrl* ctrl)
{
  ctrl->run  = 1u;
  ctrl->prev = ctrl->n_mst;
}

__global__ void sl_round_begin_kernel(SlCtrl* ctrl, long long* best, int64_t n)
{
  if (!sl_running(ctrl)) return;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) best[v] = KEY_EMPTY;
  if (v < kSlMaxJumps) ctrl->jump[v] = 0u;
}

// edges [e0, e1); an edge with an endpoint outside [0, n) is no edge
__global__ void sl_edge_kernel(const SlCtrl* ctrl, const int* src, const int* dst, const float* w, int64_t e0, int64_t e1,
                               int64_t n, const int* colour, long long* best)
{
  if (!sl_running(ctrl)) return;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t e = e0 + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < e1; e += stride) {
    const int a = src[e], b = dst[e];
    if (a < 0 || b < 0 || a >= n || b >= n) continue;
    const int ca = colour[a], cb = colour[b];
    if (ca == cb) continue;
    const long long key = key_pack(w[e], e);
    atomicMin(&best[ca], key);
    atomicMin(&best[cb], key);
  }
}

__global__ void sl_hook_kernel(SlCtrl* ctrl, const int* src, const int* dst, const int* colour, const long long* best,
                               int* parent, long long* mst_keys, int64_t n)
{
  if (!sl_running(ctrl)) return;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= n || colour[v] != v) return;
  const long long b = best[v];
  if (b == KEY_EMPTY) { parent[v] = static_cast<int>(v); return; }
  const int64_t e   = key_index(b);
  const int ca      = colour[src[e]];
  const int other   = ca == v ? colour[dst[e]] : ca;
  const bool mutual = best[other] == b;
  parent[v]         = (mutual && v < other) ? static_cast<int>(v) : other;
  if (!mutual || v < other) mst_keys[atomicAdd(&ctrl->n_mst, 1u)] = b;
}

// launch j of a round: parent[v] <- parent[parent[v]] for every component root v
__global__ void sl_jump_kernel(SlCtrl* ctrl, const int* colour, int* parent, int64_t n, int j)
{
  if (!sl_running(ctrl)) return;
  if (j > 0 && *reinterpret_cast<volatile unsigned*>(&ctrl->jump[j - 1]) == 0u) return;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool changed    = false;
  if (v < n && colour[v] == v) {
    const int p = parent[v], pp = parent[p];
    if (pp != p) { parent[v] = pp; changed = true; }
  }
  if (__syncthreads_or(changed) && threadIdx.x == 0) ctrl->jump[j] = 1u;
}

__global__ void sl_relabel_kernel(const SlCtrl* ctrl, int* colour, const int* parent, int64_t n)
{
  if (!sl_running(ctrl)) return;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) colour[v] = parent[colour[v]];
}

__global__ void sl_round_end_kernel(SlCtrl* ctrl)
{
  if (!sl_running(ctrl)) return;
  if (ctrl->n_mst == ctrl->prev) ctrl->run = 0u;
  ctrl->prev = ctrl->n_mst;
}

// forest edge t (in key order) of the sorted keys: endpoints and weight (sqrt: the root of the weight); count <- n_mst
__global__ void sl_emit_kernel(const SlCtrl* ctrl, const long long* sorted, const int* src, const int* dst, const float* w,
                               int64_t cap, int do_sqrt, int* out_src, int* out_dst, float* out_w, int* out_count)
{
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t cnt = ctrl->n_mst;
  if (t == 0 && out_count) *out_count = static_cast<int>(cnt);
  if (t >= cnt || t >= cap) return;
  const int64_t e = key_index(sorted[t]);
  out_src[t]      = src[e];
  out_dst[t]      = dst[e];
  if (out_w) out_w[t] = do_sqrt ? sqrtf(w[e]) : w[e];
}

// out_colour[v] = the smallest vertex of v's tree (minv: [n] scratch, INT_MAX on entry)
__global__ void sl_min_vertex_kernel(const int* colour, int* minv, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) atomicMin(&minv[colour[v]], static_cast<int>(v));
}

__global__ void sl_colour_out_kernel(const int* colour, const int* minv, int* out_colour, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) out_colour[v] = minv[colour[v]];
}

__global__ void sl_fill_kernel(int* a, int v, int64_t n)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// ---- single_linkage

// bit 0 of ctrl->bad when some value of x [m, d] is not finite
__global__ void sl_finite_kernel(const float* x, int64_t ldx, int64_t m, int d, SlCtrl* ctrl)
{
  bool bad = false;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < m * d; t += stride)
    bad |= !isfinite(x[(t / d) * ldx + t % d]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(&ctrl->bad, 1u);
}

// edge i * n_nb + s = (i, idx[i, s], dist[i, s]); the row's edge to itself stays in place as a self-loop, which no
// round ever chooses (so the positions, and with them the key order, are those of the kNN output)
__global__ void sl_knn_edges_kernel(const int64_t* idx, const float* dist, int64_t m, int n_nb, int* src, int* dst, float* w)
{
  const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= m * n_nb) return;
  const int i = static_cast<int>(e / n_nb);
  const int64_t j = idx[e];
  src[e] = i;
  dst[e] = j < 0 ? i : static_cast<int>(j);
  w[e]   = dist[e];
}

// The dense component ids of a connect round, numbered in order of each component's smallest row (the root of a
// component is not always its smallest row): minv[r] <- r for every root r, then sl_min_vertex_kernel lowers it to the
// component's smallest row (only the roots' entries are written or read).
__global__ void sl_tree_min_init_kernel(const int* colour, int* minv, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n && colour[v] == v) minv[v] = static_cast<int>(v);
}

// flags[v] = 1 for the smallest row of a component (scanned in place into the dense component ids), then lab[v] = the
// id of v's component
__global__ void sl_root_flags_kernel(const int* colour, const int* minv, unsigned* flags, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) flags[v] = minv[colour[v]] == v ? 1u : 0u;
}

__global__ void sl_dense_label_kernel(const int* colour, const int* minv, const unsigned* ids, int* lab, int64_t n)
{
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) lab[v] = static_cast<int>(ids[minv[colour[v]]]);
}

// the end of every component in the sorted rows (km_scatter_kernel's cursors): the group_idxs of the masked arg-min
__global__ void sl_ends_kernel(const unsigned* cur, int64_t nblk, int64_t c, int* ends)
{
  const int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g < c) ends[g] = static_cast<int>(cur[g * nblk + nblk - 1]);
}

// adj[i, g] = (component of sorted row r0 + i) != g, for the rows [r0, r0 + rows) of one chunk
__global__ void sl_adj_kernel(const int* slab, int64_t r0, int64_t rows, int64_t c, uint8_t* adj)
{
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < rows * c; t += stride)
    adj[t] = slab[r0 + t / c] != t % c ? 1 : 0;
}

// best[g] = min over the sorted rows p of component g of (d_p, p), d_p the row's masked nearest distance (clamped at 0)
__global__ void sl_comp_best_kernel(const long long* keys, const int* slab, int64_t m, long long* best)
{
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const long long key = keys[p];
  if (key == KEY_EMPTY) return;
  atomicMin(&best[slab[p]], key_pack(fmaxf(key_dist(key), 0.f), p));
}

// edge e0 + g connects component g to its nearest other component: (row, its masked nearest row, distance), original
// row ids.  A component without a candidate (or a nearest row of its own component) sets bit 1 of ctrl->bad and gets a
// self-loop.
__global__ void sl_connect_kernel(const long long* best, const long long* keys, const int* perm, const int* slab, int64_t c,
                                  int64_t e0, int* src, int* dst, float* w, SlCtrl* ctrl)
{
  const int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= c) return;
  const long long b = best[g];
  const int64_t p   = key_index(b);
  const int64_t j   = b == KEY_EMPTY ? p : key_index(keys[p]);
  if (b == KEY_EMPTY || slab[j] == g) {
    atomicOr(&ctrl->bad, 2u);
    src[e0 + g] = 0; dst[e0 + g] = 0; w[e0 + g] = 0.f;
    return;
  }
  src[e0 + g] = perm[p];
  dst[e0 + g] = perm[j];
  w[e0 + g]   = key_dist(b);
}

}  // namespace b2d
