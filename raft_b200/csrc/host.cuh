// Host code shared by the C-ABI families (one .cu per family under csrc/): this header is the list of what crosses a
// file.  A name used by one file only stays static in that file.  Nothing here is exported from the library.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <functional>
#include <string>

#include "../../include/raft_b200.h"
#include "ball_cover_types.cuh"
#include "kmeans_types.cuh"
#include "prep.cuh"   // PrepMode (its kernels are templates, instantiated by launch_prep alone)
#include "tc_params.cuh"

#pragma GCC visibility push(hidden)

namespace b2d {

// ------------------------------------------------------------------------------------------
// host.cu: error state, workspace check, tensor-map encoder, device check, profiling ring

int fail(int code, const std::string& msg);
#define B2D_CUDA(call)                                                                       \
  do {                                                                                       \
    cudaError_t e__ = (call);                                                                \
    if (e__ != cudaSuccess)                                                                  \
      return fail(B2D_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));        \
  } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Cuts a caller's workspace into consecutive regions, each rounded up to `align` bytes.  With a null base it only
// counts the bytes (the *_workspace_bytes queries): every region is then null, and no pointer is formed from null.
struct Carve {
  char* base;
  size_t align;
  size_t bytes = 0;
  Carve(void* b, size_t a) : base(static_cast<char*>(b)), align(a) {}
  template <typename T>
  T* take(size_t count)
  {
    T* at = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += align_up(count * sizeof(T), align);
    return at;
  }
};

// the caller's workspace holds `need` bytes (none needed: anything goes) and starts on an `align`-byte boundary
int check_workspace(const void* ws, size_t bytes, size_t need, size_t align = 256);

// a row-major matrix [rows][cols] of `dtype` with a row pitch of pitch_bytes, in boxes of box_cols x box_rows;
// `tag` names the map in the error message
int encode_2d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int64_t cols, int64_t rows,
              int64_t pitch_bytes, unsigned box_cols, unsigned box_rows, CUtensorMapSwizzle swizzle,
              CUtensorMapL2promotion promotion, const char* tag);
// the same for a 3-D view: dims and box innermost first, pitch_bytes of dimensions 1 and 2
int encode_3d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, const int64_t (&dims)[3],
              const int64_t (&pitch_bytes)[2], const unsigned (&box)[3], CUtensorMapSwizzle swizzle,
              CUtensorMapL2promotion promotion, const char* tag);

// SM count of the current device; every kernel of the library is built for sm_90a only, so any other device is an error
int device_sms(int* sms);

// CUDA events on the call's stream around the main kernel(s) of a call, between b2d_profile_begin and b2d_profile_end
struct ProfileScope {
  cudaStream_t s;
  int slot = -1;
  explicit ProfileScope(cudaStream_t st);
  ~ProfileScope();
};

// ------------------------------------------------------------------------------------------
// tensor_launch.cu: the tensor-core path

// workspace layout of the tensor-core path
struct TcWorkspace {
  __half* xop;
  __half* yop;
  float* xt;
  float* yt;
  float* xsc;        // [m] per-row scale 2^(E - e_row) of x (1 unless the row took its own exponent, prep.cuh)
  float* ysc;        // [n] the same for y
  unsigned* nonuni;  // [2] some row of x / y took its own exponent
  long long* keys;
  unsigned* gmax;  // [2]
  float* coef;     // [1]
  unsigned* has_lo;  // [1]
  float4* aux;       // [m]    screened NN: per-row (bound - |x|^2, |x|, |x - hi part|, -)
  float* xlo;        // [m]    screened NN: |x_i - hi part| (prep.cuh lvec)
  float* ylo;        // [n]
  int2* cand;        // [cap]  screened NN: candidate list
  unsigned* cand_cnt;  // [1] (+ overflow flag right behind it)
  unsigned cand_cap;
  // screened NN: the database chunk is worked through in the order of its squared row norms (screen_tc.cuh)
  unsigned* sort_key[2];  // [min(n, 2^20)] each
  int* sort_val[2];       // [min(n, 2^20)] each: position -> source row
  void* sort_tmp;
  size_t bytes;      // end of these regions in the workspace
};
constexpr int64_t kNnChunkRows  = 1 << 20;   // database rows per screened chunk
constexpr size_t kSortTmpBytes  = 4u << 20;  // cub::DeviceRadixSort scratch for <= 2^20 pairs (checked at run time)

// the tensor-core path's regions at the front of `c` (1024-byte alignment); with_keys: the screened arg-min's too
TcWorkspace tc_layout(Carve& c, int64_t m, int64_t n, int64_t k, bool with_keys);
TcWorkspace tc_layout(void* base, int64_t m, int64_t n, int64_t k, bool with_keys);
// w with side 0 (x) or side 1 (y) starting at prepared row r0: the operand, t and scale rows the tensor kernels read
TcWorkspace tc_rows(TcWorkspace w, int side, int64_t r0, int64_t k);

// How the tensor path computes an expanded metric: the operand preparation (PrepParams: mode, center, xform, coef_mul,
// tx_const) and the epilogue's post-processing (TcPost)
struct TcMetric {
  int mode, center, post, xform;
  float coef_mul, tx_const;
};
constexpr TcMetric TC_L2{PREP_L2, 0, POST_CLAMP, 0, 1.f, 0.f};   // L2Expanded
// *out for `metric` with k columns; false: the metric is not on the tensor path
bool tc_metric(int metric, int64_t k, TcMetric* out);
// TcParams::diag_off of the operands x [m] and y [n] (element strides as launch_prep takes them): 0 when they are the same
// matrix and the metric's distance is the clamped L2 one (d(i, i) = 0 exactly), TC_NO_DIAG otherwise
int64_t tc_self_diag(const TcMetric& tm, const void* x, int64_t xrs, int64_t xcs, int64_t m, const void* y, int64_t yrs,
                     int64_t ycs, int64_t n);

// operand preparation (prep.cuh) of x [m, k] and y [n, k] into w; T is float or __half.  x_only (with n == 0): the rows
// of x alone, against the y side an earlier launch prepared (the seeds of every mean-shift iteration)
template <typename T>
int launch_prep(cudaStream_t s, const TcWorkspace& w, const void* x, int64_t xrs, int64_t xcs, int64_t m,
                const void* y, int64_t yrs, int64_t ycs, int64_t n, int64_t k, const float* xn, const float* yn,
                const TcMetric& tm, const int* y_gather = nullptr, bool y_only = false, const unsigned* run_flag = nullptr,
                bool x_only = false);

// one expanded_tc_kernel launch (K chunk [kb0, kb0 + nkb_chunk) when nkb_chunk > 0)
int launch_tc(cudaStream_t s, const TcWorkspace& w, TcParams p, int64_t k, int epi, int post, int kb0 = 0,
              int nkb_chunk = 0);

// coarse screening pass of the screened fusedL2NN (screen_tc.cuh) over the y blocks with
// sel_lo <= index % sel_s < sel_hi
int launch_screen(cudaStream_t s, const TcWorkspace& w, int64_t m, int64_t n, int64_t k, int sel_s, int sel_lo,
                  int sel_hi, unsigned* overflow, const unsigned* run_flag, int unit_norm, const int* col_map);

// ------------------------------------------------------------------------------------------
// nearest.cu: the 1-NN kernels single linkage also runs

// The masked arg-min of the prepared x rows (w's x side) against the prepared y rows into keys (KEY_EMPTY or earlier
// minima on entry), for a valid group_idxs whose group map of y is grp: adjacency bits, tile classes, the
// EPI_MINLOC_MASKED launch
int masked_keys(cudaStream_t s, const TcWorkspace& w, long long* keys, const int* grp, unsigned* bits, uint8_t* cls,
                const unsigned* bad, const uint8_t* adj, int64_t ld_adj, const int32_t* group_idxs, int64_t G,
                int64_t m, int64_t n, int64_t k);
// masked_keys in two steps, for callers that build the adjacency bits themselves and reuse the tile classes: the tile
// classes cls of (x, y) from the bits (all MASK_NONE when *bad), then the EPI_MINLOC_MASKED launch
int masked_classify(cudaStream_t s, uint8_t* cls, const unsigned* bits, const int32_t* group_idxs, int64_t G, int64_t m,
                    int64_t n, const unsigned* bad);
int masked_launch(cudaStream_t s, const TcWorkspace& w, long long* keys, const int* grp, const unsigned* bits,
                  const uint8_t* cls, int64_t G, int64_t m, int64_t n, int64_t k);
// launches of minloc_init_kernel / masked_group_map_kernel, 256 threads per block
void minloc_init(cudaStream_t s, unsigned grid, long long* keys, int64_t m);
void masked_group_map(cudaStream_t s, unsigned grid, int* grp, const int* group_idxs, int64_t G, int64_t n);

// ------------------------------------------------------------------------------------------
// neighbors.cu: the kNN workspace, which single linkage sizes its kNN phase with

// The tensor-core workspace with keys, then the kNN's own regions.  Two regions of the tensor workspace are borrowed:
// thr and cnt live in aux ([m] floats, then [m] counters: 8 of its 16 bytes per row), and the per-row candidate lists
// (KNN_CAP entries of 8 bytes per row) in cand, which b2d_knn guards with m * KNN_CAP <= cand_cap.
struct KnnLayout {
  TcWorkspace w;
  long long* topk;      // [m][n_neighbors]
  float* thr;           // [m]
  unsigned* cnt;        // [m]
  long long* dropmin;   // [m] best key that did not fit into a row's list this pass
  int* dirty;           // [m] rows to redo for the current pass
  unsigned* repaired;   // [m] 1 once a row has been repaired in some pass
  int* rep_list;        // [m] the repaired rows ...
  unsigned* dirty_cnt;  // [64] one counter per pass
  unsigned* rep_cnt;    // [1] ... and their count, right behind dirty_cnt
  size_t bytes;
};

KnnLayout knn_layout(void* base, int64_t m, int64_t n, int64_t k, int64_t n_neighbors);

// ------------------------------------------------------------------------------------------
// kmeans.cu: the stable counting sort of rows by label and the scan, which single linkage and DBSCAN run too

// The stable counting sort of m rows by a label in [0, nc) (km_assign_kernel's histogram, km_scan_*, km_scatter_kernel):
// row blocks of 2048 rows, or more when nc x blocks would exceed kKmHistCap words.  A function of (m, nc) only, so the
// summation order of k-means never depends on the device.
struct KmSortPlan {
  int64_t rb, nblk, nhist;
};

KmSortPlan km_sort_plan(int64_t m, int64_t nc);

// the sort's regions in the workspace
struct KmSort {
  unsigned* hist;   // label counts per (label, row block), scanned in place into the sort cursors
  unsigned* tiles;  // scan tile sums
  int* perm;        // [m] row ids sorted by label
  int* slab;        // [m] their labels
  KmCtrl* ctrl;     // receives the scan total
};

// Sized for the plan of exactly nc labels, or with any_count for the plan of any label count up to nc:
// km_sort_plan(m, c).nhist <= min(c * ceil(m / 2048), max(c, kKmHistCap)), which grows with c.  The histogram holds at
// least nc words, so its tiles also serve a scan of nc words (km_scan).
KmSort km_sort_regions(Carve& c, int64_t m, int64_t nc, bool any_count);

inline unsigned km_grid(int64_t n, int per = 256) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + per - 1) / per, 1 << 16))); }

// exclusive scan of the words a[0, n) in place, the total into ctrl->total
int km_scan(cudaStream_t s, const unsigned* run, unsigned* a, int64_t n, unsigned* tiles, KmCtrl* ctrl);
// the histogram of given labels (km_assign fuses it into the arg-min)
int km_sort_count(cudaStream_t s, const KmSort& S, const KmSortPlan& P, const int* labels, int64_t m, int64_t nc);
// the histogram scanned into the sort cursors, then the rows scattered into perm / slab
int km_sort_scatter(cudaStream_t s, const unsigned* run, const KmSort& S, const KmSortPlan& P, const int* labels,
                    int64_t m, int64_t nc);
// launch of km_gather_rows_kernel<int>: rows idx[0, nc) of x into out [nc, k], one 128-thread block per row
void km_gather_rows(cudaStream_t s, unsigned grid, const float* x, int64_t ldx, int k, const int* idx, int nc, float* out);

// The workspace of one k-means call on m rows, k columns and nc clusters (b2d_kmeans_workspace_bytes)
struct KmLayout {
  TcWorkspace tc;   // x (side 0) and the centroids (side 1) of the arg-min, keys[m]
  KmSortPlan P;
  KmSort sort;
  KmCtrl* ctrl;     // the fit's control words: sort.ctrl
  int* labels;      // [m]
  float* w;         // [m] the normalised weights
  float* rowf;      // [m] k-means++ D^2 / Random: the uniforms
  double *sums, *wsums, *part, *wpart, *shift, *ipart, *bs;
  float* best;      // [nc * k] n_init: the best centroids so far
  float* sk_val;    // Random: select_k outputs and workspace
  int64_t* sk_idx;
  void* sk_ws;
  size_t sk_bytes;
  int64_t nchunks, nb;
  size_t bytes;
};

KmLayout km_layout(void* base, int64_t m, int64_t k, int64_t nc);
// the argument checks every k-means entry shares (c: the centroids)
int km_args(const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc, const void* c);
// the arguments of a fit besides km_args
int km_fit_args(const double* inertia, const int32_t* n_iter, int max_iter, double tol, int init, int n_init);
// arg-min of every row against the centroids c [nc, k] (prepared first when prep_y): labels, inertia partials, label
// histogram (when hist)
int km_assign(cudaStream_t s, const KmLayout& L, int64_t m, int64_t k, int64_t nc, const float* c, const float* w,
              int* labels, const unsigned* run, bool prep_y, bool hist);
// km_assign in two halves around the arg-min launch, for a caller with its own (masked) launch: keys <- KEY_EMPTY and
// the histogram zeroed, the centroids prepared when prep_y; then the labels, inertia partials and histogram from the keys
int km_assign_prep(cudaStream_t s, const KmLayout& L, int64_t m, int64_t k, int64_t nc, const float* c, const unsigned* run,
                   bool prep_y, bool hist);
int km_assign_labels(cudaStream_t s, const KmLayout& L, int64_t m, int64_t nc, const float* w, int* labels,
                     const unsigned* run, bool hist);
// new centroids (and, when wpc, the fp32 weight per cluster) from the histogram km_assign left
int km_update(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc,
              const float* w, const int* labels, const float* old_c, float* out_c, float* wpc, const unsigned* run);
// the weights of a fit (normalize: scaled to sum to m) or null; marks L.ctrl bad for negative / NaN weights or a zero sum
const float* km_weights(cudaStream_t s, const KmLayout& L, const float* w, int64_t m, bool normalize);
// greedy k-means++ seeding of c [nc, k] from the rows of x
int km_plus_plus(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
                 int64_t nc, uint64_t seed, float* c);
// A fit after its checks, its km_ctrl_init_kernel and its weights: `runs` times seed_run(r) (which writes the initial
// centroids) then Lloyd's loop; with runs > 1 the first run of strictly lowest inertia is kept.  inertia / n_iter may be
// null.
int km_fit_runs(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
                int64_t nc, int max_iter, double tol, int inertia_check, int runs, float* centroids, double* inertia,
                int32_t* n_iter, const std::function<int(int)>& seed_run);
// launch of km_ctrl_init_kernel: the control words at the start of a fit
void km_ctrl_init(cudaStream_t s, KmCtrl* ctrl);
// k-means|| launches (kmeans.cuh): km_par_keys_kernel over m rows and km_par_take_kernel for n candidates
void km_par_keys(cudaStream_t s, const long long* fold_keys, float* d2, const float* w, int64_t m, uint64_t seed, int round,
                 float* key);
void km_par_take(cudaStream_t s, const float* x, int64_t ldx, int k, const int64_t* idx, int n, float* cand, int* ids,
                 float* d2);

// ------------------------------------------------------------------------------------------
// radius.cu: the CSR row sort, which the ball cover's epsilon query runs too

// scratch of the segmented sort below: it is given both key buffers and needs next to nothing else
constexpr size_t kRowSortBytes = static_cast<size_t>(1) << 20;
// The packed (distance, index) keys of CSR rows at indices[0, nnz) sorted row by row (segments clipped to the nnz slots;
// alt: a second key buffer of nnz entries, sort_tmp: sort_bytes >= kRowSortBytes of scratch), then split into the
// indices and distances.
int radius_sort_split(cudaStream_t s, const int64_t* indptr, int64_t m, int64_t nnz, int64_t* indices, float* distances,
                      long long* alt, void* sort_tmp, size_t sort_bytes);

// ------------------------------------------------------------------------------------------
// ball_cover.cu: the index, its build and the walk launch, which DBSCAN's ball-cover fit and the EMST run too

// n_landmarks, or ceil(sqrt(n)) for 0
int64_t bc_landmarks(int64_t n, int64_t nl);

// the index's regions (256-byte aligned)
struct BcLayout {
  BcIndex ix;
  size_t bytes;
};
BcLayout bc_layout(void* base, int64_t n, int64_t d, int64_t nl);

// Scratch bound of a onesweep radix sort of n items: its digit counters and one 1 KiB look-back row per tile of at least
// 256 items of a 2^28-item portion.  CUB reports its scratch only with a device present, so the sorts check it at run time.
inline size_t bc_sort_bytes(int64_t n)
{
  return 4 * static_cast<size_t>(std::min<int64_t>(n, int64_t(1) << 28)) + (static_cast<size_t>(1) << 20);
}

// The build's workspace: two key and two value buffers of the radix sorts, and their scratch (bc_sort_bytes).
struct BcBuildLayout {
  unsigned long long* keys[2];
  int* vals[2];
  void* tmp;
  size_t tmp_bytes;
  size_t bytes;
};
BcBuildLayout bc_build_layout(void* base, int64_t n);

// The workspace of a call that builds its own index: the index, then one region that holds first the build's scratch and,
// once the index is built, the caller's arrays, carved from `rest` (256-byte aligned) over that scratch.
struct BcOverlay {
  BcIndex ix;
  BcBuildLayout build;
  size_t index_bytes;
  Carve rest;

  BcOverlay(void* base, int64_t n, int64_t d, int64_t nl)
      : rest(nullptr, 256)
  {
    const BcLayout I = bc_layout(base, n, d, nl);
    ix               = I.ix;
    index_bytes      = I.bytes;   // a multiple of 256
    rest.base        = base ? static_cast<char*>(base) + I.bytes : nullptr;
    build            = bc_build_layout(rest.base, n);
  }
  size_t bytes() const { return index_bytes + std::max(build.bytes, rest.bytes); }
};

// the index of x [n][D] (pitch ldx) with nl landmarks into ix, scratch W (D = 2 and 3 are instantiated)
template <int D>
int bc_build(cudaStream_t s, const BcIndex& ix, const BcBuildLayout& W, const float* x, int64_t ldx, int n, int nl,
             uint64_t seed);

constexpr size_t kBcSmemMax = 64 << 10;   // landmarks staged in shared memory up to this many bytes per block

// One launch of a walk kernel of ball_cover.cuh (or of a walk built on it) over `items` queries or index positions:
// one warp each, kBcWarps per block, with the nl landmarks of d coordinates and their rhi in dynamic shared memory when
// they fit in kBcSmemMax.  The kernel takes args followed by the staging flag.
template <typename Kernel, typename... Args>
int bc_walk_launch(cudaStream_t s, Kernel kernel, int64_t items, int64_t nl, int64_t d, Args... args)
{
  size_t smem = static_cast<size_t>(nl) * (d + 1) * sizeof(float);
  if (smem > kBcSmemMax) smem = 0;
  B2D_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)));
  kernel<<<static_cast<unsigned>((items + kBcWarps - 1) / kBcWarps), kBcWarps * 32, smem, s>>>(args..., smem > 0);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// single_linkage.cu

inline unsigned sl_grid(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, (n + 255) / 256)); }

}  // namespace b2d

#pragma GCC visibility pop
