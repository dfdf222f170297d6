// Hierarchical balanced k-means (kmeans_balanced.cuh; DESIGN.md section 2, K16): G = min(nc, max(1, round(sqrt(nc))))
// mesoclusters by balanced EM on all rows, nc fine clusters allocated to them by size, balanced EM on every mesocluster
// at once with the masked arg-min, then a short balanced-EM pass over all rows and all centroids.  Every launch size is
// known on the host: nothing synchronises, and a whole fit can be captured in a CUDA graph.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>

#include "host.cuh"
#include "kmeans_balanced.cuh"

using namespace b2d;

namespace {
enum KbStage : int { KB_MESO = 0, KB_FINE = 1, KB_FINAL = 2 };

int64_t kb_groups(int64_t nc)
{
  return std::min<int64_t>(nc, std::max<int64_t>(1, std::llround(std::sqrt(static_cast<double>(nc)))));
}

char* at(void* base, size_t off) { return base ? static_cast<char*>(base) + off : nullptr; }

// Regions every stage reads, then two phases that share their bytes: the mesocluster stage, and the fine and final
// stages (one k-means layout for nc clusters: the fine stage's operand is xs, the final stage's is x).
struct KbLayout {
  int64_t G;
  int* vperm;       // [m] the finite rows in row order (the row order of the mesocluster and final stages)
  int* nvalid;      // [1] their count
  int* alloc;       // [G] fine clusters per mesocluster
  int* E;           // [G] ends of the mesoclusters' rows in xs
  int* F;           // [G] ends of their fine centroids
  float* cmeso;     // [G, k] mesocluster centroids
  float* xs;        // [m, k] the finite rows sorted by mesocluster (stably), zero rows after them
  KmLayout meso;    // phase 1: (m, k, G) on x
  KmLayout fine;    // phase 2: (m, k, nc) on xs, then on x
  unsigned* bits;   // [ceil(m/32)][G] rows of xs adjacent to mesocluster g
  uint8_t* cls;     // tile classes of (xs, centroids)
  int* grp;         // [nc] mesocluster of every fine centroid
  unsigned* bad;    // [8] zero: the group ends are valid by construction
  size_t bytes;
};

KbLayout kb_layout(void* base, int64_t m, int64_t k, int64_t nc)
{
  KbLayout L{};
  L.G = kb_groups(nc);
  Carve c(base, 1024);
  L.vperm  = c.take<int>(m);
  L.nvalid = c.take<int>(8);
  L.alloc  = c.take<int>(L.G);
  L.E      = c.take<int>(L.G);
  L.F      = c.take<int>(L.G);
  L.cmeso  = c.take<float>(static_cast<size_t>(L.G) * k);
  L.xs     = c.take<float>(static_cast<size_t>(m) * k);
  L.meso   = km_layout(at(base, c.bytes), m, k, L.G);
  L.fine   = km_layout(at(base, c.bytes), m, k, nc);
  Carve b(at(base, c.bytes + L.fine.bytes), 1024);
  L.bits  = b.take<unsigned>(static_cast<size_t>((m + 31) / 32) * L.G);
  L.cls   = b.take<uint8_t>(static_cast<size_t>((m + TC_BM - 1) / TC_BM) * ((nc + TC_BN - 1) / TC_BN));
  L.grp   = b.take<int>(nc);
  L.bad   = b.take<unsigned>(8);
  L.bytes = c.bytes + std::max(L.meso.bytes, L.fine.bytes + b.bytes);
  return L;
}

// the masked arg-min's tables of the fine stage
struct KbMask {
  const int* grp;
  const unsigned* bits;
  const uint8_t* cls;
  const int* F;
  int64_t G;
};

// The masked arg-min's tables for rows sorted into the groups [E[g-1], E[g]) against centroids grouped as
// [F[g-1], F[g]): the group of every centroid, the adjacency bits straight from the row ranges, the tile classes.
int kb_fine_tables(cudaStream_t s, const KbLayout& L, const int* E, const int* F, int64_t G, int64_t m, int64_t nc,
                   KbMask* M)
{
  masked_group_map(s, sl_grid(nc), L.grp, F, G, nc);
  B2D_CUDA(cudaMemsetAsync(L.bad, 0, 8 * sizeof(unsigned), s));
  kb_bits_kernel<<<km_grid((m + 31) / 32 * G, 256), 256, 0, s>>>(L.bits, E, G, m);
  B2D_CUDA(cudaGetLastError());
  int rc = masked_classify(s, L.cls, L.bits, F, G, m, nc, L.bad);
  if (rc) return rc;
  *M = KbMask{L.grp, L.bits, L.cls, F, G};
  return B2D_OK;
}

// The fine stage's assignment: every row's arg-min among the centroids c [nc, k] of its group, from the prepared
// operands of L (x side prepared, the centroids prepared here), into labels with L's label histogram
int kb_fine_assign(cudaStream_t s, const KmLayout& L, const KbMask& M, int64_t m, int64_t k, int64_t nc, const float* c,
                   int* labels)
{
  int rc = km_assign_prep(s, L, m, k, nc, c, nullptr, true, true);
  if (rc) return rc;
  rc = masked_launch(s, L.tc, L.tc.keys, M.grp, M.bits, M.cls, M.G, m, nc, k);
  if (rc) return rc;
  return km_assign_labels(s, L, m, nc, nullptr, labels, nullptr, true);
}

// `iters` iterations of balanced EM on the problems q with centroids c [q.nc, k], from the prepared operands of L (x
// side: q.x): the arg-min (masked by M when given), the k-means update, and the adjust step after every iteration but
// the last, so the centroids returned are the update of the last labels.
int kb_em(cudaStream_t s, const KmLayout& L, const KbProblems& q, const KbMask* M, int64_t m, int64_t k, float* c,
          int* labels, int iters, uint64_t seed, int stage)
{
  const int64_t nc = q.nc;
  for (int it = 0; it < iters; ++it) {
    int rc = M ? kb_fine_assign(s, L, *M, m, k, nc, c, labels) : km_assign(s, L, m, k, nc, c, nullptr, labels, nullptr, true, true);
    if (rc) return rc;
    rc = km_update(s, L, q.x, q.ldx, m, k, nc, nullptr, labels, c, c, nullptr, nullptr);
    if (rc) return rc;
    if (it + 1 < iters) {
      kb_adjust_kernel<<<static_cast<unsigned>(nc), 128, 0, s>>>(q, labels, L.sort.hist, L.P.nblk, c, static_cast<int>(k),
                                                                 seed, stage, it);
      B2D_CUDA(cudaGetLastError());
    }
  }
  return B2D_OK;
}

int kb_fit(cudaStream_t s, const KbLayout& L, const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc, int n_iters,
           uint64_t seed, float* centroids, int32_t* labels, int32_t* sizes)
{
  const int64_t G = L.G;
  const int kk = static_cast<int>(k);
  const KmLayout& A = L.meso;
  const KmLayout& B = L.fine;
  int rc;
  {  // stage 0 (each stage is one measured region between b2d_profile_begin and b2d_profile_end)
    ProfileScope prof(s);
    // the finite rows, in row order: a counting sort by the label 0 (finite) / -1
    B2D_CUDA(cudaMemsetAsync(L.nvalid, 0, sizeof(int), s));
    kb_valid_kernel<<<static_cast<unsigned>((m + 7) / 8), 256, 0, s>>>(x, ldx, kk, m, A.labels, L.nvalid);
    B2D_CUDA(cudaGetLastError());
    const KmSortPlan P1 = km_sort_plan(m, 1);
    KmSort V = A.sort;
    V.perm = L.vperm;
    rc = km_sort_count(s, V, P1, A.labels, m, 1);
    if (rc) return rc;
    rc = km_sort_scatter(s, nullptr, V, P1, A.labels, m, 1);
    if (rc) return rc;
    // mesoclusters: one problem, G centroids
    const KbProblems meso{x, ldx, L.vperm, L.nvalid, nullptr, 1, static_cast<int>(G)};
    kb_init_kernel<<<static_cast<unsigned>(G), 128, 0, s>>>(meso, L.cmeso, kk);
    B2D_CUDA(cudaGetLastError());
    rc = launch_prep<float>(s, A.tc, x, ldx, 1, m, L.cmeso, k, 1, G, k, nullptr, nullptr, TC_L2);
    if (rc) return rc;
    rc = kb_em(s, A, meso, nullptr, m, k, L.cmeso, A.labels, n_iters, seed, KB_MESO);
    if (rc) return rc;
  }
  {  // stage 1 (its masked arg-min launches are measured regions of their own, inside this one)
    ProfileScope prof(s);
    // fine allocation, and the rows sorted by mesocluster (the last update's counting sort)
    kb_alloc_kernel<<<1, kKbAllocThreads, 0, s>>>(A.sort.hist, A.P.nblk, static_cast<int>(G), nc, L.alloc, L.E, L.F);
    kb_gather_kernel<<<static_cast<unsigned>(m), 128, 0, s>>>(x, ldx, kk, A.sort.perm, L.E, static_cast<int>(G), L.xs);
    B2D_CUDA(cudaGetLastError());
    // G problems on xs, each row's arg-min restricted to the centroids of its mesocluster
    KbMask M;
    rc = kb_fine_tables(s, L, L.E, L.F, G, m, nc, &M);
    if (rc) return rc;
    const KbProblems fine{L.xs, k, nullptr, L.E, L.F, static_cast<int>(G), static_cast<int>(nc)};
    kb_init_kernel<<<static_cast<unsigned>(nc), 128, 0, s>>>(fine, centroids, kk);
    B2D_CUDA(cudaGetLastError());
    rc = launch_prep<float>(s, B.tc, L.xs, k, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, TC_L2);
    if (rc) return rc;
    rc = kb_em(s, B, fine, &M, m, k, centroids, B.labels, n_iters, seed, KB_FINE);
    if (rc) return rc;
  }
  // stage 2: one problem, all centroids, x in the caller's row order
  ProfileScope prof(s);
  const KbProblems all{x, ldx, L.vperm, L.nvalid, nullptr, 1, static_cast<int>(nc)};
  rc = launch_prep<float>(s, B.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  int* lab = labels ? labels : B.labels;
  rc = kb_em(s, B, all, nullptr, m, k, centroids, lab, std::max(n_iters / 10, 2), seed, KB_FINAL);
  if (rc) return rc;
  if (sizes) {
    kb_sizes_kernel<<<sl_grid(nc), 256, 0, s>>>(B.sort.hist, B.P.nblk, static_cast<int>(nc), sizes);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}
}  // namespace

size_t b2d_kmeans_balanced_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters)
{
  if (m < 0 || k < 0 || n_clusters < 0) return static_cast<size_t>(-1);
  return kb_layout(nullptr, m, k, n_clusters).bytes;
}

int b2d_kmeans_balanced_fit(void* stream, int n_clusters, int n_iters, uint64_t seed, const float* x, int64_t ldx, int64_t m,
                            int64_t k, float* centroids, int32_t* labels, int32_t* sizes, void* workspace,
                            size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  if (n_iters < 1) return fail(B2D_ERR_INVALID_ARG, "n_iters must be >= 1");
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, kb_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  return kb_fit(s, kb_layout(workspace, m, k, nc), x, ldx, m, k, nc, n_iters, seed, centroids, labels, sizes);
}

int b2d_debug_kmeans_balanced_fine_assign(void* stream, const float* x, int64_t ldx, int64_t m, int64_t k,
                                          const int32_t* row_ends, const float* centroids, int n_clusters,
                                          const int32_t* centroid_ends, int64_t num_groups, int32_t* labels,
                                          void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  const int64_t nc = n_clusters, G = num_groups;
  if (G < 1 || G > kb_groups(nc)) return fail(B2D_ERR_INVALID_ARG, "num_groups must be in [1, round(sqrt(n_clusters))]");
  if (!row_ends || !centroid_ends || !labels) return fail(B2D_ERR_INVALID_ARG, "null row_ends / centroid_ends / labels");
  rc = check_workspace(workspace, workspace_bytes, kb_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KbLayout L = kb_layout(workspace, m, k, nc);
  rc = launch_prep<float>(s, L.fine.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  KbMask M;
  rc = kb_fine_tables(s, L, row_ends, centroid_ends, G, m, nc, &M);
  if (rc) return rc;
  return kb_fine_assign(s, L.fine, M, m, k, nc, centroids, labels);
}
