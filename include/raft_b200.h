/* raft_b200 -- C ABI of the H100-native pairwise-distance / fusedL2NN engine.
 *
 * This is the drop-in boundary: every entry point below is what a RAFT-side binding for the
 * distance path would call.  Reference interfaces replaced (all relative to the reference snapshot;
 * the distance sources themselves were deleted upstream in raft 26.02, CHANGELOG.md:59, so the
 * citations are the surviving call sites / patterns -- see SURVEY.md section 8(a),(b)):
 *
 *   b2d_pairwise_distance      raft::distance::pairwise_distance(handle, x, y, dist, m, n, k,
 *                              metric, isRowMajor, metric_arg)
 *                              call shape: cpp/include/raft/stats/detail/silhouette_score.cuh:205-206,
 *                              cpp/include/raft/stats/detail/trustworthiness_score.cuh:152-153;
 *                              runtime-ABI pattern: cpp/include/raft_runtime/random/
 *                              rmat_rectangular_generator.hpp:18-34
 *   b2d_fused_l2_nn            raft::distance::fusedL2NN / fusedL2NNMinReduce (out = KeyValuePair
 *                              <int,float>[m]); KVP type cpp/include/raft/core/kvp.hpp:20-62,
 *                              tie-break cpp/include/raft/core/operators.hpp:187-194
 *   b2d_fused_l2_nn_keys /     the per-GPU half and the post-exchange half of the multi-GPU
 *   b2d_fused_l2_nn_finalize   fusedL2NN (db row-sharded, packed min-loc all-reduce:
 *                              comms_t::allreduce(INT64, MIN), cpp/include/raft/core/comms.hpp:335,
 *                              cpp/include/raft/comms/detail/std_comms.hpp:365-374)
 *   b2d_row_norm               raft::linalg::rowNorm / norm<ALONG_ROWS>
 *                              cpp/include/raft/linalg/norm.cuh:50-58,118-147
 *   b2d_select_k               raft::matrix::select_k(handle, in_val, in_idx, out_val, out_idx, select_min,
 *                              sorted, algo), cpp/include/raft/matrix/select_k.cuh:72-106: exact per-row
 *                              top-k, the selection step after pairwise_distance in a brute-force kNN
 *
 * Conventions (same as the reference's, cpp/docs developer_guide.md:396-433): every call only
 * enqueues work on `stream` (a cudaStream_t passed as void*), never synchronises, never
 * allocates device memory (temporaries come from the caller's `workspace`, sized by the
 * *_workspace_bytes query -- the counterpart of the handle's workspace memory resource,
 * cpp/include/raft/core/resource/device_memory_resource.hpp:100-129), is thread-safe, and
 * returns a status code instead of throwing.  There is no CPU fallback: on a machine without
 * an sm_90 GPU every compute entry point returns B2D_ERR_CUDA.
 */
#ifndef RAFT_B200_H_
#define RAFT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* status codes */
enum {
  B2D_OK              = 0,
  B2D_ERR_INVALID_ARG = 1, /* -> raft::logic_error  (cpp/include/raft/core/error.hpp:218-239) */
  B2D_ERR_CUDA        = 2, /* -> raft::cuda_error   (cpp/include/raft/util/cuda_rt_essentials.hpp:23-52) */
  B2D_ERR_UNSUPPORTED = 3,
  B2D_ERR_WORKSPACE   = 4
};

/* raft::distance::DistanceType values (SURVEY.md 8(a1)) */
enum {
  B2D_L2Expanded          = 0,
  B2D_L2SqrtExpanded      = 1,
  B2D_CosineExpanded      = 2,
  B2D_L1                  = 3,
  B2D_L2Unexpanded        = 4,
  B2D_L2SqrtUnexpanded    = 5,
  B2D_InnerProduct        = 6,
  B2D_Linf                = 7,
  B2D_Canberra            = 8,
  B2D_LpUnexpanded        = 9,
  B2D_CorrelationExpanded = 10,
  B2D_JaccardExpanded     = 11, /* 1 - <x,y> / (|x|^2 + |y|^2 - <x,y>): Jaccard distance on indicator data */
  B2D_HellingerExpanded   = 12,
  B2D_BrayCurtis          = 14, /* sum |x - y| / sum |x + y| */
  B2D_JensenShannon       = 15,
  B2D_HammingUnexpanded   = 16,
  B2D_KLDivergence        = 17, /* 0.5 sum x log(x / y), 0 log 0 = 0; +inf where y = 0 < x (the mathematical value; pinned by
                                   tests/golden); operand roles follow (x, y) of the call in row- AND column-major order */
  B2D_RusselRaoExpanded   = 18,
  B2D_DiceExpanded        = 19  /* 1 - 2 <x,y> / (|x|^2 + |y|^2): Dice dissimilarity on indicator data */
};

/* element types of x / y: fp32 (dist fp32), fp16 (fp32 accumulate, dist fp32), fp64 (dist fp64: a SIMT double-precision
 * path for every metric; workspace = per-row statistics, 16 (m + n) bytes) */
enum { B2D_F32 = 0, B2D_F16 = 1, B2D_F64 = 2 };

/* raft::KeyValuePair<int,float> (cpp/include/raft/core/kvp.hpp:20-62) */
typedef struct {
  int32_t key;
  float value;
} b2d_kvp_if;

/* norm types of b2d_row_norm (raft::linalg::NormType, cpp/include/raft/linalg/norm_types.hpp:12-23) */
enum { B2D_L0PseudoNorm = 0, B2D_L1Norm = 1, B2D_L2Norm = 2, B2D_LinfNorm = 3 };

int b2d_version(void);
/* Process-wide tuning / test hooks (nothing on the hot path reads the environment):
 *   "nn_screen"  0 forces the exact arg-min kernel for fusedL2NN (default 1: screened search where it applies)
 *   "nn_tau"     candidates per row above which the trial pass calls screening off (default 6) */
int b2d_set_option(const char* name, double value);
/* Diagnostic -- SYNCHRONISES `stream`: control words of the last screened fusedL2NN chunk in `workspace`:
 * [0] list slots in use (one incumbent per row + the blocks of 64 the screen reserved), [1] list overflow, [2] go_screen,
 * [3] go_exact, [4] (unused), [5] candidates after the trial pass, [6] candidates found by the screen.  `out7`: 7 words. */
int b2d_debug_nn_stats(void* stream, const void* workspace, int64_t m, int64_t n, int64_t k, unsigned* out7);
/* thread-local description of the last non-zero status returned on this thread */
const char* b2d_last_error(void);

/* Bytes of device scratch b2d_pairwise_distance needs for this problem (0 for the unexpanded
 * metrics).  Returns (size_t)-1 for an unsupported metric / dtype. */
size_t b2d_pairwise_workspace_bytes(int metric, int dtype, int64_t m, int64_t n, int64_t k);

/* dist[i,j] = metric(x_i, y_j).  x:[m,k], y:[n,k], dist:[m,n]; row_major != 0: C order with
 * leading dimensions ldx, ldy, ldd (elements, >= k / k / n); row_major == 0: Fortran order
 * (ld >= m / n / m).  x and y may alias.  metric_arg = p of LpUnexpanded. */
int b2d_pairwise_distance(void* stream, int metric, int dtype, const void* x, int64_t ldx,
                          const void* y, int64_t ldy, void* dist /* float*, or double* for B2D_F64 */, int64_t ldd, int64_t m,
                          int64_t n, int64_t k, int row_major, float metric_arg, void* workspace,
                          size_t workspace_bytes);

/* Diagnostic, host arithmetic only (no device, nothing is dereferenced): the kernels b2d_pairwise_distance would run for
 * these arguments, which it also validates in the same way.  x, y and dist matter through their alignment.  out:
 *   [0] path (B2D_PLAN_*)
 *   [1] tensor path: 1 if the tiles leave through TMA stores, 0 from registers
 *   [2] tensor path, register stores: 1 if tiles wholly inside dist go out as 8-byte vectors, 0 all scalar
 *   [3], [4] fp32 unexpanded kernels: 16-byte loads of the kernel's first / second operand (in Fortran order the
 *            first operand is y)
 *   [5] number of launches L of the main kernel (the tensor path accumulates K in chunks when k > 320)
 *   [6 + 4 i ...] launch i < L, as far as out_len allows: first k-block (32 columns each), k-blocks, accumulation
 *            mode (0 single pass, 1 first chunk: store, 2 middle: add, 3 last: add and finish), 1 if the resident
 *            kernel (<= 4 k-blocks) runs it, 0 the streaming one
 * out_len >= 6. */
enum { B2D_PLAN_NONE = 0, B2D_PLAN_TENSOR = 1, B2D_PLAN_F32_SIMT = 2, B2D_PLAN_F32_TMA = 3, B2D_PLAN_F64_SIMT = 4 };
int b2d_debug_pairwise_plan(int metric, int dtype, const void* x, int64_t ldx, const void* y, int64_t ldy,
                            const void* dist, int64_t ldd, int64_t m, int64_t n, int64_t k, int row_major, int* out,
                            int out_len);

size_t b2d_fused_l2_nn_workspace_bytes(int64_t m, int64_t n, int64_t k);

/* out[i] = {argmin_j, min_j} ||x_i - y_j||^2 (sqrt != 0: of the Euclidean distance); ties go to
 * the smaller j.  xn / yn: optional precomputed squared row norms (NULL: computed here).
 * init_out == 0: reduce into the existing contents of out (initOutBuffer=false). */
int b2d_fused_l2_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y,
                    int64_t ldy, const float* xn, const float* yn, int64_t m, int64_t n, int64_t k,
                    int do_sqrt, int init_out, void* workspace, size_t workspace_bytes);

/* raft::distance::fusedDistanceNN[MinReduce] (SURVEY.md 8(f1)): the same fused arg-min for
 * metric in {L2Expanded, L2SqrtExpanded, CosineExpanded, CorrelationExpanded}; out[i].value is the
 * distance in that metric.  xn / yn (optional) are squared L2 row norms and are used by the L2 metrics.
 * All four metrics take the screened search described at b2d_fused_l2_nn_keys when 64 < k <= 128. */
int b2d_fused_distance_nn(void* stream, b2d_kvp_if* out, int metric, const float* x, int64_t ldx,
                          const float* y, int64_t ldy, const float* xn, const float* yn, int64_t m,
                          int64_t n, int64_t k, int init_out, void* workspace, size_t workspace_bytes);

/* raft::distance::masked_l2_nn: b2d_fused_l2_nn restricted by a row x group adjacency mask.  Group g holds the rows
 * [group_idxs[g-1], group_idxs[g]) of y (group_idxs[-1] = 0: group_idxs is the inclusive scan of the group sizes);
 * rows at or after group_idxs[num_groups-1] are in no group.  adj [m][num_groups] bytes, row pitch ld_adj >= num_groups,
 * nonzero = adjacent (a C++ bool array qualifies).  out[i] = {argmin_j, min_j} ||x_i - y_j||^2 (do_sqrt: Euclidean)
 * over the rows j whose group is adjacent to row i, ties to the smaller j; a row without any such j gets
 * {0x7fffffff, FLT_MAX} (init_out == 0: the caller's value stays).  Always the exact arg-min kernel, which skips the
 * MMAs of tiles the mask rules out.  group_idxs must be non-decreasing and inside [0, n]; this is checked on the device
 * without a synchronisation: when it fails, every row of out becomes {0x7fffffff, NaN}.  xn / yn: optional squared row
 * norms.  m, n, num_groups < 2^31. */
size_t b2d_masked_l2_nn_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t num_groups);
int b2d_masked_l2_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                     const float* xn, const float* yn, const uint8_t* adj, int64_t ld_adj, const int32_t* group_idxs,
                     int64_t num_groups, int64_t m, int64_t n, int64_t k, int do_sqrt, int init_out, void* workspace,
                     size_t workspace_bytes);

/* Multi-GPU building blocks.  keys[i] = (order-preserving bits of ||x_i - y_j||^2 << 32)
 * | (j + idx_offset), reduced with signed 64-bit MIN: over this GPU's y shard here, then across
 * GPUs by the caller's all-reduce(INT64, MIN).  init_keys != 0 resets keys to +max first;
 * init_keys == 0 continues from the keys an earlier call or another GPU left (they also serve as
 * starting bounds of the screened search, so exchanging keys early makes the rest of a shard
 * cheaper -- INTEGRATION.md section 3).  b2d_fused_l2_nn_finalize unpacks (clamp at 0, optional sqrt).
 * For 64 < k <= 128 and n >= 16384 the result is produced by a screened search (y worked through in norm-ordered
 * chunks of 2^20 rows: exact tensor pass on 1/32 of a chunk, 1-product lower-bound screen on all of it, exact fp32
 * re-evaluation of the candidates, device-side fallback to the exact pass): same answer, about a third of the
 * work.  Row indices in the keys are always the caller's (source) rows. */
int b2d_fused_l2_nn_keys(void* stream, int64_t* keys, const float* x, int64_t ldx, const float* y,
                         int64_t ldy, const float* xn, const float* yn, int64_t m, int64_t n,
                         int64_t k, int64_t idx_offset, int init_keys, void* workspace,
                         size_t workspace_bytes);
int b2d_fused_l2_nn_finalize(void* stream, b2d_kvp_if* out, const int64_t* keys, int64_t m,
                             int do_sqrt, const void* workspace, size_t workspace_bytes);

/* Single-process multi-GPU fusedL2NN (SURVEY.md 8(e); the reference's SNMG pattern: one ncclComm_t per device from a
 * grouped ncclCommInitRank / ncclCommInitAll, cpp/include/raft/core/resource/nccl_comm.hpp:43-62,
 * cpp/include/raft/core/device_resources_snmg.hpp:35-154).  Device g holds the replicated queries x[g] [m,k], its
 * database row block y[g] [n_shard[g],k] (global index of its first row: idx_offset[g]), keys[g] [m] and a workspace of
 * b2d_fused_l2_nn_workspace_bytes(m, n_shard[g], k) bytes; streams[g] is a cudaStream_t of device devices[g] and
 * comms[g] the ncclComm_t of that device (NULL array allowed for ngpu == 1).  Work is only enqueued: per exchange
 * step one ncclAllReduce(int64, min) of the m packed keys per device inside a ncclGroupStart/End (a 32768-row head of
 * every shard, then sub-chunks growing x4: the screened search starts each from GLOBAL bounds), then out[g] [m] is
 * written on every device (identical results).  NCCL is resolved at run time from the libnccl.so.2 already loaded. */
int b2d_fused_l2_nn_multi(int ngpu, const int* devices, void* const* streams, void* const* comms, b2d_kvp_if* const* out,
                          const float* const* x, int64_t ldx, const float* const* y, int64_t ldy, const int64_t* n_shard,
                          const int64_t* idx_offset, int64_t m, int64_t k, int do_sqrt, int64_t* const* keys,
                          void* const* workspace, const size_t* workspace_bytes);

/* Fused brute-force kNN for the L2 metrics (SURVEY.md 8(f2); replaces raft::neighbors::brute_force::knn /
 * fused_l2_knn, removed with the distance package -- CHANGELOG.md:59-60 -- and the pair
 * pairwise_distance + raft::matrix::select_k, cpp/include/raft/matrix/select_k.cuh:73-106):
 * out_idx[i, 0..n_neighbors) = rows of y nearest to x_i in ascending (distance, index) order,
 * out_dist the squared (do_sqrt != 0: Euclidean) distances.  The m x n matrix is never written.
 * n_neighbors <= 64, k <= 320.  Asynchronous like every other entry point: a pass whose per-row candidate lists overflowed
 * in a way that matters (database ordered by decreasing distance, ...) is repaired on the device.  A slot that
 * cannot be filled (fewer than n_neighbors comparable rows: NaN distances) holds index -1, distance +inf. */
size_t b2d_knn_l2_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t n_neighbors);
/* the same for metric in {L2Expanded, L2Unexpanded, L2SqrtExpanded, L2SqrtUnexpanded, CosineExpanded,
 * CorrelationExpanded} (workspace: b2d_knn_l2_workspace_bytes) */
int b2d_knn(void* stream, int64_t* out_idx, float* out_dist, int metric, const float* x, int64_t ldx, const float* y,
            int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, void* workspace,
            size_t workspace_bytes);
int b2d_knn_l2(void* stream, int64_t* out_idx, float* out_dist, const float* x, int64_t ldx, const float* y,
               int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, int do_sqrt,
               void* workspace, size_t workspace_bytes);

/* raft::stats::silhouette_score (cpp/include/raft/stats/detail/silhouette_score.cuh:186-328), a caller of
 * the distance path (SURVEY.md 8(f3)): *score (device) = mean over samples of (b - a) / max(a, b);
 * per_sample (device, [n]) optional.  labels: int32 in [0, n_labels).  metric: any metric of
 * b2d_pairwise_distance (the reference's default is L2Unexpanded).  The n x n matrix is produced and
 * consumed in [chunk_rows x n] slabs (0 = about 1 GiB per slab), like the reference's batched variant
 * (detail/batched/silhouette_score.cuh:213-243).  Never synchronises: labels are validated on the device, a label
 * outside [0, n_labels) makes *score (and the per-sample value of that row) NaN, and so do labels that leave fewer
 * than two non-empty clusters (*score only). */
size_t b2d_silhouette_score_workspace_bytes(int64_t n, int64_t k, int n_labels, int metric, int64_t chunk_rows);
int b2d_silhouette_score(void* stream, float* score, float* per_sample, const float* x, int64_t ldx,
                         const int* labels, int64_t n, int64_t k, int n_labels, int metric, float metric_arg,
                         int64_t chunk_rows, void* workspace, size_t workspace_bytes);

/* raft::stats::trustworthiness_score (cpp/include/raft/stats/detail/trustworthiness_score.cuh:113-211), the
 * other dangling caller (SURVEY.md 8(f3)): x [n, m] original space, x_embedded [n, d]; neighbours in the
 * embedded space from the fused kNN and ranks in the original space both under `metric` (the reference's
 * distance_type template parameter; L2 / L2Sqrt (Expanded or Unexpanded), CosineExpanded, CorrelationExpanded),
 * ranks counted over [batch_rows x n] slabs (0 = about 1 GiB).  Every sample has exactly n_neighbors embedded
 * neighbours: itself excluded, ties by index.  *score is a DEVICE double; the call never synchronises.
 * n_neighbors <= 63. */
size_t b2d_trustworthiness_score_workspace_bytes(int64_t n, int64_t m, int64_t d, int n_neighbors, int metric,
                                                 int64_t batch_rows);
int b2d_trustworthiness_score(void* stream, double* score, const float* x, int64_t ldx,
                              const float* x_embedded, int64_t lde, int64_t n, int64_t m, int64_t d,
                              int n_neighbors, int metric, int64_t batch_rows, void* workspace,
                              size_t workspace_bytes);

/* Measurement aid (bench.py's roofline): between b2d_profile_begin(capacity) and b2d_profile_end every
 * b2d_pairwise_distance (and b2d_gram_matrix) call on the tensor path records a CUDA-event pair on ITS stream around its main
 * kernel launch(es) (operand preparation excluded).  Nothing synchronises until b2d_profile_end, which
 * waits for the recorded events and returns the durations in call order (milliseconds). */
int b2d_profile_begin(int capacity);
int b2d_profile_end(float* ms, int max_count, int* count);

/* out[r] = norm of row r of x:[rows,k] (L2Norm = sum of squares; do_sqrt applies sqrt_op as
 * fin_op, cpp/include/raft/linalg/norm.cuh:118-147). */
int b2d_row_norm(void* stream, float* out, const float* x, int64_t ldx, int64_t rows, int64_t k,
                 int norm_type, int do_sqrt);

/* raft::matrix::argmin (cpp/include/raft/matrix/argmin.cuh:25-37; cpp/include/raft/matrix/detail/math.cuh:290-343):
 * out[r] = column of the minimum of row r of in:[rows,n] (row pitch ld), ties -> smaller index, a row without any
 * value below +inf (all NaN / +inf) -> 0.  The separate-pass form of the arg-min that fusedL2NN fuses (SURVEY.md a9);
 * one read of the matrix. */
int b2d_row_argmin(void* stream, int32_t* out, const float* in, int64_t ld, int64_t rows, int64_t n);

/* raft::matrix::select_k (cpp/include/raft/matrix/select_k.cuh:72-106): for every row r of in_val:[rows,len] (row pitch
 * ld), out_val[r, 0..k) / out_idx[r, 0..k) = the k smallest (select_min != 0) or largest values and their columns, or
 * in_idx[r, column] when in_idx (int64, same pitch) is given.  Order: the float order with -0.0 == +0.0 and every NaN
 * above +inf (so NaNs come first in a max selection, last in a min selection); among equal values the smaller column
 * wins.  Every row is written sorted, best first, equal values in ascending column order.  The values are the input
 * bits unchanged (-0.0 stays -0.0, a NaN keeps its payload).  1 <= k <= len (else B2D_ERR_INVALID_ARG); rows, len <
 * 2^31 (else B2D_ERR_UNSUPPORTED); rows == 0 does nothing.  Exact radix selection on the (value, column) order
 * (DESIGN.md K9).  The workspace query returns SIZE_MAX for invalid extents. */
size_t b2d_select_k_workspace_bytes(int64_t rows, int64_t len, int64_t k);
int b2d_select_k(void* stream, const float* in_val, int64_t ld, const int64_t* in_idx, int64_t rows, int64_t len, int64_t k,
                 int select_min, float* out_val, int64_t* out_idx, void* workspace, size_t workspace_bytes);

/* raft::neighbors::epsilon_neighborhood::eps_neighbors_l2sq / epsUnexpL2SqNeighborhood ([RECALLED]; removed upstream with
 * neighbors/, CHANGELOG.md:59): the epsilon neighbourhood of the rows of x:[m,k] among the rows of y:[n,k] (fp32,
 * row-major, pitches ldx / ldy), the vertex-degree step of DBSCAN.  eps is the SQUARED radius.
 *   adj[i * ld_adj + j] = (d(i, j) <= eps) as a 0 / 1 byte (a C++ bool array qualifies), ld_adj >= n, where d(i, j) is
 *     exactly the value b2d_pairwise_distance(L2Expanded) returns for the pair: the call equals that matrix compared with
 *     eps, bit for bit, without writing it.  A NaN distance is never adjacent; a NaN or negative eps makes nothing adjacent.
 *   Self pairs: when y is x or a window of its rows (same buffer, ldx == ldy, y == x + off * ldx for an integer off), the
 *     pairs i == j + off have d = 0, adjacent for every eps >= 0 (the tensor form alone does not give exactly 0 there).  A
 *     copy of x in other memory gets no such rule.
 *   vd[j] += #{i : adj[i, j]} for j < n and vd[n] += the total: PER-COLUMN degrees, length n + 1, as the reference's kernel
 *     summed them ([RECALLED] updateVertexDegree; its doc comment said m + 1, and cuML swapped the operands to get row
 *     degrees).  vd is int32 (wrapping modulo 2^32 like the reference's int) or, vd_int64 != 0, int64.  init_vd != 0 zeroes
 *     vd first; init_vd == 0 adds to its contents (the reference atomicAdd-ed without clearing, [RECALLED]).
 *   adj == NULL: count only; vd == NULL: adjacency only; both NULL is B2D_ERR_INVALID_ARG.
 * k <= 320 (the whole distance at once; else B2D_ERR_UNSUPPORTED), m, n < 2^31.  m == 0 or n == 0 only zeroes vd when
 * init_vd is set.  Workspace: the size of b2d_pairwise_workspace_bytes(L2Expanded, F32, m, n, k); SIZE_MAX for negative
 * extents. */
size_t b2d_eps_neighbors_l2sq_workspace_bytes(int64_t m, int64_t n, int64_t k);
int b2d_eps_neighbors_l2sq(void* stream, uint8_t* adj, int64_t ld_adj, void* vd, int vd_int64, int init_vd,
                           const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m, int64_t n, int64_t k,
                           float eps, void* workspace, size_t workspace_bytes);

/* Radius neighbours (sklearn.neighbors.NearestNeighbors.radius_neighbors(sort_results=True); a project API, no upstream
 * signature): for every row i of x:[m,k] the rows j of y:[n,k] with d(i, j) <= radius, as CSR, without the m x n matrix.
 * fp32, row-major, pitches ldx / ldy >= k.
 *   d(i, j) is exactly the fp32 value b2d_pairwise_distance(metric) returns for the pair, metric one of L2Expanded (radius
 *     is then a squared distance), L2SqrtExpanded, CosineExpanded and CorrelationExpanded (else B2D_ERR_UNSUPPORTED),
 *     including its self-pair rule: under an L2 metric with x == y, m == n and ldx == ldy, d(i, i) = 0.  A NaN distance
 *     (NaN element, zero-norm row under cosine, constant row under correlation) is never in the result; a NaN or negative
 *     radius gives no pairs; radius = +inf gives every non-NaN pair.
 *   Output: indptr int64 [m + 1] (indptr[m] = nnz), indices int64 [nnz] (rows of y) and distances float [nnz].  Each row is
 *     sorted by the packed (distance, index) key of the 1-NN and kNN entry points: ascending distance, equal distances by
 *     ascending index, -0.0 before +0.0.  The result is reproducible byte for byte.
 * Two calls: b2d_radius_neighbors_count writes indptr (the row degrees, scanned); the caller reads nnz = indptr[m],
 * allocates and calls b2d_radius_neighbors_fill with the same inputs and that nnz (<= 2^31 - 1, else
 * B2D_ERR_UNSUPPORTED: split the queries).  fill never writes past nnz entries: called with other inputs or a smaller nnz,
 * its result is unspecified but stays inside the caller's buffers.  k <= 320 (else B2D_ERR_UNSUPPORTED); k == 0, ld < k,
 * m or n >= 2^31, a negative extent or nnz and null pointers are B2D_ERR_INVALID_ARG; m == 0 or n == 0 give nnz = 0.  Both
 * calls only enqueue work (no synchronisation, no allocation) and can be captured in a CUDA graph.  Workspace: the query
 * with nnz = 0 for the count call and with the call's nnz for fill; SIZE_MAX for negative arguments. */
size_t b2d_radius_neighbors_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t nnz);
int b2d_radius_neighbors_count(void* stream, int64_t* indptr, int metric, const float* x, int64_t ldx, const float* y,
                               int64_t ldy, int64_t m, int64_t n, int64_t k, float radius, void* workspace,
                               size_t workspace_bytes);
int b2d_radius_neighbors_fill(void* stream, const int64_t* indptr, int64_t nnz, int64_t* indices, float* distances,
                              int metric, const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m, int64_t n,
                              int64_t k, float radius, void* workspace, size_t workspace_bytes);

/* kernels of b2d_kde_score_samples, in the order of sklearn.neighbors.KernelDensity's kernel names */
enum {
  B2D_KDE_GAUSSIAN     = 0,
  B2D_KDE_TOPHAT       = 1,
  B2D_KDE_EPANECHNIKOV = 2,
  B2D_KDE_EXPONENTIAL  = 3,
  B2D_KDE_LINEAR       = 4,
  B2D_KDE_COSINE       = 5
};

/* Kernel density estimation (sklearn.neighbors.KernelDensity(kernel, bandwidth = h, atol = 0, rtol = 0).fit(dataset,
 * sample_weight).score_samples(queries); a project API, no upstream signature): for fp32 dataset y:[n,d] and queries
 * x:[m,d] (row-major, pitches ldy / ldx >= d), the log densities out (double, device, [m]):
 *   out[i] = log(sum_j w_j K(d_ij; h)) - log(sum_j w_j) + log_norm(kernel, h, d)
 *   d^2_ij is exactly the fp32 value of b2d_pairwise_distance(L2Expanded) for the pair, including its self-pair rule: with
 *     x == y (same pointer, m == n, ldx == ldy), d^2_ii = 0; a copy of the data gets no such rule.  d_ij = sqrt(d^2_ij).
 *   K: gaussian exp(-d^2 / 2h^2), tophat 1, epanechnikov 1 - d^2 / h^2, exponential exp(-d / h), linear 1 - d / h, cosine
 *     cos(pi d / 2h).  The four compact kernels (tophat, epanechnikov, linear, cosine) count only the pairs with
 *     d^2_ij < h2 = fp32(h h) (h h formed in fp64): sklearn's strict dist < h, decided exactly by the engine's d^2.
 *   log_norm: sklearn's _log_kernel_norm for gaussian, tophat, epanechnikov, exponential and linear; for cosine the exact
 *     -log(S_(d-1) int_0^1 t^(d-1) cos(pi t / 2) dt) - d log h, S_(d-1) = 2 pi^(d/2) / Gamma(d/2) (sklearn's value is wrong
 *     at every even d), by a series without cancellation, within 1e-12 relative of quadrature for d = 1 ... 320.
 *   Range: gaussian and exponential carry a per-row maximum of log K (log-sum-exp), so every finite input gives a finite
 *     result however far a query lies from the data.  A compact kernel with no dataset row in its support gives -inf.
 *   Weights: sample_weight [n] (device) or NULL (every weight 1); finite and >= 0, a weight of 0 removes its row.  A
 *     negative or non-finite weight, or a total of 0, makes EVERY output NaN (checked on the device, no synchronisation).
 *   NaN: a NaN distance in a row makes that row NaN, for every kernel: a NaN query row poisons itself, a NaN dataset row
 *     every query.
 *   Results are bit-identical from run to run and independent of the device's SM count and of batch_cols (no
 *     floating-point atomics): the distances are reduced in the epilogue of the tensor kernel to one partial per row and
 *     128-column half (8 bytes), folded in fp64 in ascending column order.
 * batch_cols: dataset columns per slab, rounded up to the 256-column y block; 0 means as many as keep the partials at
 * about 1 GiB.  d <= 320 (else B2D_ERR_UNSUPPORTED).  B2D_ERR_INVALID_ARG: n == 0 or d == 0, a bandwidth that is not
 * finite or not > 0 or whose 0.5 / h2 is not finite in fp32, an unknown kernel, m or n >= 2^31, ld < d, a negative extent
 * or batch_cols, null dataset / queries / out.  m == 0 does nothing.  The call only enqueues work (no allocation, no
 * synchronisation) and can be captured in a CUDA graph.  The workspace query returns SIZE_MAX for negative arguments. */
size_t b2d_kde_workspace_bytes(int64_t m, int64_t n, int64_t d, int64_t batch_cols);
int b2d_kde_score_samples(void* stream, int kernel, double bandwidth, const float* dataset, int64_t ldy,
                          const float* sample_weight, const float* queries, int64_t ldx, int64_t m, int64_t n, int64_t d,
                          int64_t batch_cols, double* out, void* workspace, size_t workspace_bytes);

/* raft::distance::kernels::KernelType ([RECALLED] raft/distance/distance_types.hpp, <= 25.12) */
enum { B2D_KERNEL_LINEAR = 0, B2D_KERNEL_POLYNOMIAL = 1, B2D_KERNEL_RBF = 2, B2D_KERNEL_TANH = 3 };

/* raft::distance::kernels Gram matrices (GramMatrixBase / PolynomialKernel / RBFKernel / TanhKernel, [RECALLED] removed
 * with the distance package, CHANGELOG.md:59), the kernel evaluations of cuML's SVM.  For x:[m,k], y:[n,k]:
 *   LINEAR      out[i,j] = <x_i, y_j>, bit-identical to b2d_pairwise_distance(InnerProduct)
 *   POLYNOMIAL  (gamma <x_i, y_j> + coef0)^degree, integer degree >= 0 by repeated squaring (degree 0: 1 everywhere)
 *   RBF         exp(-gamma ||x_i - y_j||^2), the squared distance of b2d_pairwise_distance(L2Expanded); when x and y are
 *               the same matrix (same pointer, m == n, ldx == ldy) the diagonal is exactly 1
 *   TANH        tanh(gamma <x_i, y_j> + coef0)
 * The transform runs in the epilogue of the distance kernel, so the matrix is written once.  Layout, leading dimensions,
 * dtypes and the workspace are those of b2d_pairwise_distance (row_major == 0: Fortran order, out [m,n] with ldo >= m);
 * out is float for fp32 / fp16 inputs and double for fp64.  gamma and coef0 are used as float for fp32 / fp16 inputs and
 * as double for fp64, and must be finite in that precision; degree is read for POLYNOMIAL only.  An unknown kernel, a
 * non-finite gamma / coef0, a negative POLYNOMIAL degree, k == 0 are B2D_ERR_INVALID_ARG; m == 0 or n == 0 does nothing.
 * No precomputed norms: the operand preparation computes them.  The workspace query returns SIZE_MAX for an unknown
 * kernel or dtype and for negative extents. */
size_t b2d_gram_matrix_workspace_bytes(int kernel, int dtype, int64_t m, int64_t n, int64_t k);
int b2d_gram_matrix(void* stream, int kernel, int degree, double gamma, double coef0, int dtype, const void* x, int64_t ldx,
                    const void* y, int64_t ldy, void* out /* float*, or double* for B2D_F64 */, int64_t ldo, int64_t m,
                    int64_t n, int64_t k, int row_major, void* workspace, size_t workspace_bytes);

/* raft::cluster::kmeans InitMethod ([RECALLED] raft/cluster/kmeans_types.hpp, <= 25.12) */
enum { B2D_KMEANS_INIT_PLUS_PLUS = 0, B2D_KMEANS_INIT_RANDOM = 1, B2D_KMEANS_INIT_ARRAY = 2 };

/* raft::cluster::kmeans ([RECALLED] removed with distance/, CHANGELOG.md:59): Lloyd's k-means under L2Expanded for fp32
 * x:[m,k] (row-major, pitch ldx), centroids:[n_clusters,k] contiguous.
 *   Assignment: label_i = argmin_j ||x_i - c_j||^2 by the exact arg-min of b2d_fused_l2_nn (the distance bits of its
 *     unscreened kernel; ties to the smaller j).  A row with a NaN distance gets no label (-1) and makes the inertia NaN.
 *   Update: c_j = sum_{label_i = j} w_i x_i / sum_{label_i = j} w_i, accumulated in fp64 in a fixed order and rounded once
 *     to fp32; a cluster of zero weight keeps its previous centroid bit for bit; labels outside [0, n_clusters) are
 *     skipped.  Results are bit-identical from run to run (no floating-point atomics).
 *   fit: iteration t assigns with C_t and computes C_{t+1}; it stops when sum ||C_{t+1} - C_t||^2 < tol (fp64) or, with
 *     inertia_check, after the first iteration when inertia_t / inertia_{t-1} > 1 - tol; at most max_iter iterations,
 *     *n_iter = the iterations that ran.  *inertia = sum_i w_i ||x_i - c_{label_i}||^2 for the returned centroids, in fp64 in the difference
 *     form (0 for a row equal to its centroid; inertia_check uses the arg-min's fp32 distances).  init:
 *     ARRAY uses centroids as given (n_init ignored); RANDOM takes n_clusters distinct rows; PLUS_PLUS is greedy
 *     k-means++ with 2 + floor(ln n_clusters) trials per round.  n_init > 1 runs seeds seed + r and keeps the first run of
 *     strictly lowest inertia.  The loop runs on the device: max_iter iterations are enqueued and the ones after
 *     convergence return at once.
 *   Weights (optional, NULL = 1): fit and predict (normalize_weight != 0) scale them to sum to m; update_centroids uses
 *     them as given.  A negative weight or a zero sum makes the inertia NaN.
 *   predict: labels (int32, optional) and *inertia (optional) for the given centroids.  update_centroids: new_centroids
 *     from given labels, weight_per_cluster[j] = the fp64 weight sum rounded to fp32 (optional).  init_plus_plus: the
 *     k-means++ seeding alone, weights as given.
 * 1 <= n_clusters <= m < 2^31 and 1 <= k <= 2^24 (the accuracy caveat of b2d_fused_l2_nn above k = 320 applies), else
 * B2D_ERR_INVALID_ARG; m == 0 does nothing.  inertia and n_iter are device pointers.  No call synchronises or allocates,
 * so every call can be captured in a CUDA graph.  The workspace query returns SIZE_MAX for negative extents. */
size_t b2d_kmeans_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters);
int b2d_kmeans_fit(void* stream, int n_clusters, int max_iter, double tol, int init, int n_init, uint64_t seed,
                   int inertia_check, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                   float* centroids, double* inertia, int32_t* n_iter, void* workspace, size_t workspace_bytes);
int b2d_kmeans_predict(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                       const float* centroids, int n_clusters, int32_t* labels, double* inertia, int normalize_weight,
                       void* workspace, size_t workspace_bytes);
int b2d_kmeans_update_centroids(void* stream, const float* x, int64_t ldx, const float* sample_weight, const int32_t* labels,
                                int64_t m, int64_t k, const float* old_centroids, int n_clusters, float* new_centroids,
                                float* weight_per_cluster, void* workspace, size_t workspace_bytes);
int b2d_kmeans_init_plus_plus(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                              int n_clusters, uint64_t seed, float* centroids, void* workspace, size_t workspace_bytes);

/* k-means|| seeding (scalable k-means++, Bahmani et al. 2012; [RECALLED] RAFT InitMethod::KMeansPlusPlus with
 * oversampling_factor > 0) for the k-means above.  f = oversampling_factor must be finite and > 0.
 *   Sizes: L = min(m, max(ceil(f n_clusters), ceil((n_clusters - 1) / 8))) rows per round over R = 8 rounds, so the
 *     candidate set has exactly C = 1 + 8L >= n_clusters rows and no call synchronises.  C > 2^31 - 1 is
 *     B2D_ERR_UNSUPPORTED.  Departure: the reference runs min(8, ceil(ln psi)) rounds (psi: the initial cost) of
 *     independent Bernoulli draws and tops a short candidate set up with random rows; here R and C are fixed.
 *   Draws: fixed-size weighted sampling without replacement (Efraimidis-Spirakis).  Round r gives row i the key
 *     ln(E_ir) - ln(p_i), E_ir = -ln(u_ir), u_ir uniform in (0, 1) from Philox4x32-10 keyed by (seed, r, i), computed in
 *     fp64 logs and rounded to fp32.  Round 0 has p_i = w_i and takes the smallest key; rounds 1..8 have
 *     p_i = w_i D2_i and take the L smallest (b2d_select_k: ties to the smaller row).  Mass 0 (w_i <= 0, D2_i = 0, a row
 *     already taken) gives +inf; a row with NaN distances a NaN key, ranked after +inf.  So a row without mass is taken
 *     only once every row with mass has been.
 *   D2: after each round D2_i = min(D2_i, squared distance of x_i to the nearest candidate of the round), by the exact
 *     arg-min of b2d_fused_l2_nn; the rows taken get D2 = 0.
 *   Candidate weights: W_c = sum of w_i over the rows whose arg-min among all C candidates is c, in fp64 in a fixed
 *     order, rounded once to fp32: weight_per_cluster of b2d_kmeans_update_centroids.  A duplicate candidate loses its
 *     ties to the earlier copy and gets weight 0.
 *   Recluster: greedy k-means++ (as PLUS_PLUS) on the C candidate rows with weights W, then b2d_kmeans_fit's loop on them
 *     with max_iter 300, tol 1e-4 and no inertia check.  The centroids are weighted means of candidates, not
 *     necessarily rows of x.  Results are bit-identical from run to run; no floating-point atomics.
 * init_scalable: the seeding alone, weights as given; optional device outputs candidates [C] (row ids) and
 *   candidate_weights [C] (W): a weighted coreset of x.  fit_scalable: b2d_kmeans_fit with init = PLUS_PLUS and this
 *   seeding in place of greedy k-means++ (run r seeded with seed + r; weights scaled to sum to m, also for the seeding).
 * Argument checks are those of b2d_kmeans_fit, plus B2D_ERR_INVALID_ARG for an oversampling_factor that is not finite or
 * not > 0; m == 0 does nothing.  The workspace query covers both calls and returns SIZE_MAX for negative extents, an
 * invalid oversampling_factor or C > 2^31 - 1; it is at least b2d_kmeans_workspace_bytes(m, k, n_clusters). */
size_t b2d_kmeans_scalable_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters, double oversampling_factor);
int b2d_kmeans_init_scalable(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                             int n_clusters, double oversampling_factor, uint64_t seed, float* centroids,
                             int32_t* candidates /* optional [C] row ids */, float* candidate_weights /* optional [C] */,
                             void* workspace, size_t workspace_bytes);
int b2d_kmeans_fit_scalable(void* stream, int n_clusters, int max_iter, double tol, double oversampling_factor, int n_init,
                            uint64_t seed, int inertia_check, const float* x, int64_t ldx, const float* sample_weight,
                            int64_t m, int64_t k, float* centroids, double* inertia, int32_t* n_iter,
                            void* workspace, size_t workspace_bytes);

/* Hierarchical balanced k-means ([RECALLED] raft::cluster::kmeans_balanced::fit, L2Expanded, fp32): n_clusters
 * centroids [n_clusters, k] of x [m, k] in three stages of balanced EM, with G = min(n_clusters,
 * max(1, round(sqrt(n_clusters)))) mesoclusters.  Labels are predicted with b2d_kmeans_predict.
 *   Balanced EM on a problem (a set of rows and a set of centroids): every iteration assigns each row to its nearest
 *     centroid of the problem (ties to the smaller index), updates the centroids (b2d_kmeans_update_centroids: fp64 sums
 *     in a fixed order; an empty cluster keeps its centroid), then adjusts them: with a = rows / centroids of the
 *     problem, a centroid j of size s_j < a / 4 draws a donor row d uniformly from the problem's rows (Philox4x32-10,
 *     counter (j, iteration, stage, 0), key seed; position floor(((w0 << 32) | w1) * rows / 2^64)); when the donor's
 *     cluster has size >= a, c_j <- (w c_j + x_d) / (w + 1) with w = min(s_j, 7), in fp64 rounded once.  The last
 *     iteration of a problem has no adjust.  Initial centroid t of a problem with R rows and C centroids is its row
 *     floor(t R / C) in the problem's row order.
 *   Stage 0: the G mesoclusters, one problem on all finite rows in row order, n_iters iterations.
 *   Allocation: mesocluster g of S_g rows (R in all) gets floor(n_clusters S_g / R) fine clusters, plus one for the
 *     largest remainders n_clusters S_g mod R (ties to the lower g) until they sum to n_clusters; a non-empty
 *     mesocluster left with none takes one from the mesocluster of the largest count / S_g holding at least two (ties to
 *     the lower g).  Mesocluster g owns the fine centroids [F_{g-1}, F_g).  With R >= n_clusters no mesocluster gets
 *     more fine clusters than rows.
 *   Stage 1: every mesocluster is a problem of its rows and its fine centroids, n_iters iterations, all at once on the
 *     rows sorted stably by mesocluster with the masked fused arg-min (b2d_masked_l2_nn's kernel).
 *   Stage 2: one problem on all finite rows and all n_clusters centroids in the caller's row order,
 *     max(n_iters / 10, 2) iterations.  So the centroids returned are b2d_kmeans_update_centroids(x, labels) bit for
 *     bit, with labels [m] (optional output) the assignment that update used and sizes [n_clusters] (optional output)
 *     its cluster sizes.
 * A row with a non-finite element gets label -1, belongs to no problem and is never a donor; every centroid is finite.
 * Results are bit-identical from run to run and independent of the device's SM count; nothing synchronises, so a fit
 * can be captured in a CUDA graph.  Argument checks are those of b2d_kmeans_fit (n_clusters in [1, m], ...) plus
 * n_iters >= 1; m == 0 does nothing.  The workspace query returns SIZE_MAX for negative extents. */
size_t b2d_kmeans_balanced_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters);
int b2d_kmeans_balanced_fit(void* stream, int n_clusters, int n_iters, uint64_t seed, const float* x, int64_t ldx,
                            int64_t m, int64_t k, float* centroids, int32_t* labels /* optional [m] */,
                            int32_t* sizes /* optional [n_clusters] */, void* workspace, size_t workspace_bytes);
/* The assignment step of the fit's stage 1 on its own, for tests: x [m, k] holds G = num_groups groups of rows
 * [row_ends[g-1], row_ends[g]) and centroids [n_clusters, k] the groups [centroid_ends[g-1], centroid_ends[g])
 * (row_ends[-1] = centroid_ends[-1] = 0; device arrays, non-decreasing, row_ends[G-1] <= m and centroid_ends[G-1] <=
 * n_clusters, not checked).  labels[i] = the nearest centroid of row i's group (ties to the smaller index), -1 for a row
 * in no group or with NaN distances.  Same kernels and tables as the fit: adjacency bits from the row ranges, tile
 * classes, one EPI_MINLOC_MASKED launch.  Argument checks of b2d_kmeans_balanced_fit, plus num_groups in
 * [1, round(sqrt(n_clusters))]; the workspace is b2d_kmeans_balanced_workspace_bytes(m, k, n_clusters). */
int b2d_debug_kmeans_balanced_fine_assign(void* stream, const float* x, int64_t ldx, int64_t m, int64_t k,
                                          const int32_t* row_ends, const float* centroids, int n_clusters,
                                          const int32_t* centroid_ends, int64_t num_groups, int32_t* labels,
                                          void* workspace, size_t workspace_bytes);

/* Minimum spanning forest of an edge list (the MST step of raft::cluster::single_linkage, [RECALLED]
 * raft::sparse::solver::mst): Borůvka on the device.  Edge e = (src[e], dst[e], w[e]) (int32 vertices, fp32 weights) is
 * ordered by (w[e], e): this order is strict, so the forest is unique.  Self-loops, duplicate and reversed edges are
 * allowed; an edge with an endpoint outside [0, n_vertices) is ignored; a NaN weight orders by its bits (a positive NaN
 * after +inf).  Outputs (device pointers): *out_count (int32) forest edges in (w, e) order in out_src / out_dst / out_w
 * (capacity n_vertices - 1; each edge as given), and out_colour[v] = the smallest vertex of v's tree.  n_vertices < 2^30
 * and n_edges < 2^32 - 1, else B2D_ERR_UNSUPPORTED.  Only enqueues work: the rounds run on the device and the ones after
 * the last merge return at once.  The workspace query returns SIZE_MAX for negative extents. */
size_t b2d_mst_workspace_bytes(int64_t n_vertices, int64_t n_edges);
int b2d_mst(void* stream, const int32_t* src, const int32_t* dst, const float* w, int64_t n_vertices, int64_t n_edges,
            int32_t* out_src, int32_t* out_dst, float* out_w, int32_t* out_colour, int32_t* out_count, void* workspace,
            size_t workspace_bytes);

/* raft::cluster::single_linkage with LinkageDistance::KNN_GRAPH ([RECALLED], <= 25.12) for fp32 x:[m,d] (row-major, pitch
 * ldx), metric B2D_L2Expanded or B2D_L2SqrtExpanded (else B2D_ERR_UNSUPPORTED):
 *   1. the kNN graph of x with n_nb = min(m, max(2, floor(log2 m) + c)) neighbours (the fused kNN), edge i n_nb + s =
 *      (i, idx[i, s], squared distance); a row's edge to itself is never used;
 *   2. edges ordered by (squared weight, position): the tree and the merge order do not depend on the metric;
 *   3. its minimum spanning forest by Borůvka (b2d_mst);
 *   4. connect_components while the forest has more than one tree: every tree's row i of smallest (d_i, i), d_i the
 *      squared distance to i's nearest row of another tree (the masked 1-NN), gives the edge (i, that row), appended
 *      after the edges so far; Borůvka again;
 *   5. the m - 1 edges in key order, merged on the host: merge t creates cluster m + t; children[t] = the two merged ids,
 *      smaller first; deltas[t] = its weight (its square root for L2SqrtExpanded); sizes[t] = the new cluster's size
 *      (scipy.cluster.hierarchy.linkage's conventions).  labels[i] = the cluster of row i after the first
 *      m - n_clusters merges, numbered 0 .. n_clusters - 1 in order of each cluster's smallest row.
 * children [m-1][2], deltas [m-1], sizes [m-1], labels [m] (int32 / fp32) are device pointers; *n_components_out (host)
 * = the number of trees of the kNN graph's forest (before step 4).  1 <= n_clusters <= m, m >= 1, d >= 1 and a finite x
 * (else B2D_ERR_INVALID_ARG, the last one found on the device); d <= 320, n_nb <= 64, m < 2^30 and m (n_nb + 1) < 2^32 - 1
 * (else B2D_ERR_UNSUPPORTED).  The call synchronises its stream: once after step 3, once per connect round and twice
 * for the dendrogram.  The workspace depends on (m, d, n_nb) only; the query returns SIZE_MAX for negative extents and
 * for an unsupported n_nb or m. */
size_t b2d_single_linkage_workspace_bytes(int64_t m, int64_t d, int c);
int b2d_single_linkage(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int c, int n_clusters,
                       int32_t* children, float* deltas, int32_t* sizes, int32_t* labels, int32_t* n_components_out,
                       void* workspace, size_t workspace_bytes);

/* DBSCAN (cuML's DBSCAN(eps, min_samples, metric, max_mbytes_per_batch), sklearn.cluster.DBSCAN's labels_ and
 * core_sample_indices_) for fp32 x:[m,d] (row-major, pitch ldx), on the epsilon neighbourhood of b2d_eps_neighbors_l2sq.
 * A is the m x m matrix one call b2d_eps_neighbors_l2sq(x, x, e) returns, bit for bit, for metric
 *   B2D_L2SqrtExpanded  squared L2 distance <= e = fp32(eps^2), eps^2 formed in fp64
 *   B2D_L2Expanded      squared L2 distance <= e = fp32(eps)
 *   B2D_CosineExpanded  the distance of b2d_pairwise_distance(CosineExpanded) <= e = fp32(eps)
 * with d(i, i) = 0 (every row is its own neighbour for eps >= 0); a NaN distance, a NaN or negative eps match nothing.
 * deg(j) = #{i : A[i, j]}; j is core iff deg(j) >= min_samples.  Core i and j are linked iff A[i, j] or A[j, i]; clusters
 * are the connected components of the core rows, numbered 0, 1, ... in order of their smallest row.  A non-core row b
 * takes the smallest cluster number of the core rows c with A[b, c], or -1 (noise).  When A is symmetric this is
 * sklearn.cluster.DBSCAN's result exactly.  Outputs (device pointers): labels [m]; core_sample_indices [m] (optional)
 * the core rows ascending, then -1 up to m; *n_clusters (optional, int32).
 * A is formed in batches of b = min(m, max(256, floor(max_bytes_per_batch / m / 256) * 256)) columns (0 means 2^30
 * bytes) of the once-prepared x, in three passes (degrees; links; border), or once when b = m.  The results do not
 * depend on the batch size, the device or the scheduling: the only atomics are an integer CAS and atomicMin.
 * Precondition: x finite (a non-finite x is safe, its labels are unspecified).  metric outside the three above and
 * d > 320 are B2D_ERR_UNSUPPORTED; m >= 2^31, d < 1, min_samples < 1, ldx < d, a negative max_bytes_per_batch and a null
 * x / labels are B2D_ERR_INVALID_ARG; m == 0 does nothing.  Only enqueues work (no synchronisation, no allocation), so
 * the call can be captured in a CUDA graph.  The workspace depends on (m, d, max_bytes_per_batch) only; the query returns
 * SIZE_MAX for negative arguments. */
size_t b2d_dbscan_workspace_bytes(int64_t m, int64_t d, int64_t max_bytes_per_batch);
int b2d_dbscan_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, double eps,
                   int64_t min_samples, int64_t max_bytes_per_batch, int32_t* labels /* [m] */,
                   int32_t* core_sample_indices /* [m] or NULL */, int32_t* n_clusters /* device, or NULL */,
                   void* workspace, size_t workspace_bytes);

/* Mean shift (sklearn.cluster.MeanShift(bandwidth = h, seeds, bin_seeding, min_bin_freq, cluster_all, max_iter).fit(x)
 * with sklearn's test dist <= h replaced by the engine's rule; a project API, no upstream signature) for fp32 x:[n,d]
 * (row-major, pitch ldx >= d, d <= 320):
 *   Neighbourhood: row j of x is within h of a point p when d^2(p, x_j) <= e = fp32(h^2), h^2 formed in fp64, d^2 the
 *     value b2d_eps_neighbors_l2sq computes for the pair with the points as x and the data as y (DBSCAN's
 *     L2SqrtExpanded rule).
 *   Seeds: seeds:[n_seeds,d] (pitch lds >= d) when not NULL; else with bin_seeding sklearn's get_bin_seeds: the bin of a
 *     row is rint(x / h) per coordinate (fp64 division, ties to even), the bins holding >= min_bin_freq rows are seeds
 *     at fp32(bin) * fp32(h) (one fp32 product), and when that makes every row a seed the seeds are the rows of x;
 *     else the seeds are the rows of x.  Bin seeding runs on the device.
 *   Iteration (sklearn's _mean_shift_single_seed), per seed: N = the neighbourhood of the current mean; an empty N drops
 *     the seed; else the new mean is the mean of x over N (fp64, rounded once to fp32); the seed stops when
 *     ||new - old||_2 <= 1e-3 h (fp64) or after max_iter completed iterations, else its count goes up by one.  So
 *     max_iter = 0 still moves every seed once.  A stopped seed is frozen with intensity |N| of its last step;
 *     *n_iter = the largest completed count over all seeds, dropped ones included.
 *   Centres: surviving seeds with bitwise-equal means merge (intensity: the largest); they are ordered by (intensity,
 *     coordinates lexicographically by their fp32 order) descending and walked greedily: a centre no earlier kept centre
 *     suppresses is kept and suppresses every later one within h of it, where i and j are within h when d^2(c_i, c_j)
 *     <= e or d^2(c_j, c_i) <= e (the symmetric rule, from the candidates prepared once as both operands).
 *   Labels: the nearest kept centre of every row by the fused L2 arg-min (b2d_fused_l2_nn's distance, ties to the
 *     smaller centre index); with cluster_all == 0 a row whose squared distance to it is > e gets -1.
 * Outputs (device): centers [n_seeds or n][d], kept centres first in walk order; *n_centers (int32; 0: no seed had a
 * neighbour, labels all -1); labels [n] (int32); *n_iter (int32, may be NULL).  Results are bit-identical from run to run
 * and independent of max_bytes_per_batch, the device's SM count and the seed order: every sum is fp64 over fp32 partials
 * of fixed chunks of 2048 data rows, folded in ascending order; the only atomics are integer ones.
 * The adjacency is formed for batches of b = min(S rounded up to 128, max(128, floor(max_bytes_per_batch / ld / 128) *
 * 128)) seeds (S the seed capacity, ld = max(n, S) rounded up to 16; 0 means 2^30 bytes).  The iterations are enqueued
 * without a host round trip (the ones after every seed has stopped return at once); the call synchronises its stream
 * after bin seeding, after the iterations and after the walk, to size what follows.  d > 320 is B2D_ERR_UNSUPPORTED;
 * n == 0, n or n_seeds >= 2^31, d < 1, a bandwidth that is not finite or > 0 or whose square is not finite in fp32,
 * max_iter < 0, seeds without n_seeds or the reverse, lds < d, ldx < d, bin_seeding with min_bin_freq < 1, a negative
 * max_bytes_per_batch and null x / centers / labels / n_centers are B2D_ERR_INVALID_ARG.  Precondition: x and seeds
 * finite.  The workspace depends on (n, d, n_seeds, max_bytes_per_batch) only (n_seeds = 0: no caller seeds); the
 * query returns SIZE_MAX for negative arguments. */
size_t b2d_mean_shift_fit_workspace_bytes(int64_t n, int64_t d, int64_t n_seeds, int64_t max_bytes_per_batch);
int b2d_mean_shift_fit(void* stream, const float* x, int64_t ldx, int64_t n, int64_t d, double bandwidth,
                       const float* seeds /* [n_seeds][lds] or NULL */, int64_t lds, int64_t n_seeds, int bin_seeding,
                       int64_t min_bin_freq, int cluster_all, int max_iter, int64_t max_bytes_per_batch,
                       float* centers, int32_t* n_centers, int32_t* labels, int32_t* n_iter /* or NULL */,
                       void* workspace, size_t workspace_bytes);

#ifdef __cplusplus
}
#endif
#endif /* RAFT_B200_H_ */
