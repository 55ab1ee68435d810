/*
 * bigclam_b200.h — C ABI of the H100-native BigCLAM F-gradient / line-search step.
 *
 * The reference (thangdnsf/BigCLAM-ApacheSpark) has no FFI or plugin interface; its boundary is
 * the implicit signature of one spark-shell function and the globals it touches:
 *
 *     def backtrackingLineSearchs(uset: List[Long]): Double      codes/bigclam4-7.scala:152
 *       reads   collectNeighbor / Neightborbc (adjacency)         codes/bigclam4-7.scala:50-51
 *               K, liststepSizeRDD, alpha, MIN_P_/MAX_P_/MIN_F_/MAX_F_   :134,:28-34,:22,:39-43
 *       reads+writes  F (N x K affiliation rows), sumF (K)        codes/bigclam4-7.scala:36,38,190,192
 *       returns the log-likelihood after the update               codes/bigclam4-7.scala:196-222
 *
 * Every entry point below names the reference lines it replaces.  A JVM binding (JNI) that the
 * Scala driver would use is shown in INTEGRATION.md; the Python ctypes binding used by the tests
 * lives in bigclam_apachespark_b200/_lib.py.
 *
 * Conventions: plain C, no exceptions cross the boundary.  Every function returns 0 on success
 * and a negative BIGCLAM_E* code on failure; bigclam_last_error() gives the message.  The caller
 * owns all host buffers; the context owns all device memory.  A context is driven by one thread
 * at a time; distinct contexts are independent.  All calls are synchronous on return unless noted.
 * There is NO CPU fallback: creating a context without a usable CUDA device fails.
 */
#ifndef BIGCLAM_B200_H
#define BIGCLAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BIGCLAM_OK            0
#define BIGCLAM_EINVAL      (-1)   /* bad argument */
#define BIGCLAM_ECUDA       (-2)   /* CUDA runtime / driver error, or no device */
#define BIGCLAM_ENOMEM      (-3)   /* host or device allocation failed */
#define BIGCLAM_EIO         (-4)   /* edge-list file unreadable / malformed */
#define BIGCLAM_EUNSUPPORTED (-5)  /* parameter combination the kernels do not cover */

typedef struct bigclam_ctx bigclam_ctx;

/* Script-level variables of the reference, one field each. */
typedef struct {
    int32_t k;           /* K.value: number of communities            bigclam4-7.scala:134,249 */
    int32_t max_inter;   /* MaxInter = 15 -> 16 step sizes            bigclam4-7.scala:26-34   */
    double  alpha;       /* 0.05  Armijo slope                        bigclam4-7.scala:22      */
    double  beta;        /* 0.1   step shrink factor                  bigclam4-7.scala:24      */
    double  min_p;       /* MIN_P_ = 0.0001                           bigclam4-7.scala:40      */
    double  max_p;       /* MAX_P_ = 0.9999                           bigclam4-7.scala:41      */
    double  min_f;       /* MIN_F_ = 0.0                              bigclam4-7.scala:42      */
    double  max_f;       /* MAX_F_ = 1000.0                           bigclam4-7.scala:43      */
    int32_t device;      /* CUDA ordinal; -1 = the calling thread's current device */
    int32_t flags;       /* BIGCLAM_F_* */
} bigclam_params;

#define BIGCLAM_F_TIME_KERNELS   1   /* record CUDA events around every step-kernel launch */
#define BIGCLAM_F_RECORD_ACCEPTED 2  /* keep the accepted step index per node (diagnostics/tests) */
#define BIGCLAM_F_SPARSE_ROWS     4  /* keep F as sparse rows on the device (like the reference's BSV[Double],
                                        bigclam4-7.scala:97-104): k <= 16384, min_f == 0, n < 2^28.  The dense entry
                                        points still work (bigclam_set_F / bigclam_get_F convert on the device);
                                        bigclam_set_F_csr / bigclam_get_F_csr never build a dense image.
                                        Above k = 1024 the step runs a wide variant: no tiles (bigclam_get_tile_stats
                                        reports n_tiles == 0), the per-warp K-sized vectors in a device scratch of
                                        (resident warps x 28 bytes x k), per-node passes over the touched components
                                        only, and no line-search bounds on the general path (BIGCLAM_LS_PRUNE=2). */

#define BIGCLAM_F_LS_EXHAUSTIVE   8  /* sparse rows: evaluate all max_inter+1 candidates of every node like the reference
                                        does (bigclam4-7.scala:172-181).  Default: a candidate that a bound on the node's
                                        objective proves unable to pass the Armijo test (:181) is not evaluated — same
                                        accepted steps, same rows, same LLH bits (DESIGN.md (d), tests/test_gpu_prune.py). */

/* Fills *p with the reference's constants for a given K. */
int bigclam_default_params(bigclam_params *p, int32_t k);

/* The 16 candidate step sizes, built by repeated `*= beta` exactly as bigclam4-7.scala:28-34
 * (out[0] = 1.0, out[j] = out[j-1]*beta; max_inter+1 values). */
int bigclam_step_sizes(double beta, int32_t max_inter, double *out);

/*
 * Context = the hot path's resident state: CSR adjacency (collectNeighbor, :50-51), F double
 * buffer, sumF.  rowptr has n+1 entries, col has rowptr[n] entries in [0,n); neighbour lists are
 * taken as given (multiplicity and order preserved, like collectNeighborIds(Either)): repeated entries,
 * self loops, unsorted and one-sided lists are tested on every step engine in tests/test_gpu_graphx_lists.py.
 * Replaces: Neightborbc broadcast (:51) and the per-call Fbc broadcast (:154).
 * Limits on k: 1024 for dense rows, 16384 with BIGCLAM_F_SPARSE_ROWS; above them BIGCLAM_EUNSUPPORTED (checked
 * before any device is touched).
 */
int bigclam_create(bigclam_ctx **out, int64_t n, const int64_t *rowptr, const int32_t *col,
                   const bigclam_params *params);
void bigclam_destroy(bigclam_ctx *ctx);
const char *bigclam_last_error(const bigclam_ctx *ctx);   /* ctx may be NULL: last create error */

/* F <- host row-major n x k; sumF <- exact column sums (initNeighborComF, :105-107). */
int bigclam_set_F(bigclam_ctx *ctx, const double *F);
/* Optional: inject a sumF that has drifted from colsum(F) (the reference never recomputes it, :192). */
int bigclam_set_sumF(bigclam_ctx *ctx, const double *sumF);
int bigclam_get_F(bigclam_ctx *ctx, double *F_out);        /* n x k row-major */
int bigclam_get_sumF(bigclam_ctx *ctx, double *sumF_out);  /* k */

/*
 * One call of backtrackingLineSearchs(uset)  (bigclam4-7.scala:152-223): PRE (:157-169), 16-candidate
 * Armijo line search keeping the max passing step (:172-184), Jacobi row swap + incremental sumF
 * (:186-193), LLH with the new F and sumF (:196-219, returned).  node_mask: NULL = all vertices
 * (the reference always passes all, :227); otherwise n bytes, u is in uset iff node_mask[u] != 0.
 * Nodes with an empty neighbour list are never updated (the reference would throw, see DESIGN.md).
 * The returned LLH is the PRE sum of the next call, so the next call's step kernel (same uset) is launched
 * speculatively to obtain it; a following bigclam_step with the same uset just commits that result.  Every
 * other entry point that reads or writes the state sees exactly the state after this call.
 */
int bigclam_step(bigclam_ctx *ctx, const uint8_t *node_mask, double *llh_out, int64_t *n_updated_out);

/* loglikelihood() (bigclamv3-7.scala:106-120, Bigclamv2.scala:187-200) on the current F, sumF. */
int bigclam_loglikelihood(bigclam_ctx *ctx, double *llh_out);

/*
 * Outer loop on the device, LLH of step t taken from step t+1's PRE pass (they are the same sum).
 *   variant 4: SGDFindC  (bigclam4-7.scala:225-243)  LLHold = first step; returns LLHold as coded at :242
 *   variant 3: MBSGD     (bigclamv3-7.scala:206-222) LLHold = 0.0
 *   variant 2: MBSGD     (Bigclamv2.scala:203-219)   LLHold = loglikelihood()
 * Stops when |1 - new/old| < rel_tol (:237) or after max_outer hot-path calls (0 = unbounded, like
 * the reference).  llh_trace (optional, trace_cap doubles) receives every call's returned LLH.
 * On return F/sumF are exactly the state after `*calls_out` calls.
 */
int bigclam_run(bigclam_ctx *ctx, int32_t variant, double rel_tol, int64_t max_outer,
                double *llh_out, int64_t *calls_out, double *llh_trace, int64_t trace_cap);

/* Diagnostics (BIGCLAM_F_RECORD_ACCEPTED): index of the accepted step size per node for the
 * most recent step, -1 = row unchanged. */
int bigclam_get_accepted(bigclam_ctx *ctx, int8_t *accepted_out);

/* Timing of the most recent bigclam_step / bigclam_run (BIGCLAM_F_TIME_KERNELS), CUDA events on
 * the context's stream: total device ms of the step kernels and how many were launched. */
int bigclam_get_kernel_time(bigclam_ctx *ctx, double *step_kernel_ms_sum, int64_t *step_kernel_launches,
                            int64_t *all_kernel_launches);

/* Interop with the host framework's plumbing (torch streams / NCCL buffers): use an existing
 * cudaStream_t, and expose device pointers of the current F (n x ld doubles, ld = row pitch) and sumF. */
/* Sparse rows (BIGCLAM_F_SPARSE_ROWS): how the small nodes were processed since the
 * context was created / the counters were last read — tiles done on the tile path, tiles that did not fit the
 * warp's shared memory and went node by node through the general path; the tile layout of the current order
 * (tiles, nodes on the general path, split hubs).  The two counters count from the previous read. */
int bigclam_get_tile_stats(bigclam_ctx *ctx, int64_t *tiles_done, int64_t *tiles_fallback, int64_t *n_tiles,
                           int64_t *n_general_nodes, int64_t *n_split_hubs);

/* Sparse rows, line search by bounds: of the nodes that asked for a line search since the previous read (split hubs not
 * counted), how many had at least one candidate that the bounds could not exclude (and were therefore evaluated). */
int bigclam_get_ls_stats(bigclam_ctx *ctx, int64_t *nodes_asked, int64_t *nodes_searched);

/* Sparse rows: re-cut the tiles of small nodes for the current average row size (rows grow or shrink while the solver
 * runs; bigclam_run does this by itself between its batches, bigclam_set_F* always).  Synchronises the stream. */
int bigclam_retile(bigclam_ctx *ctx);

int bigclam_set_stream(bigclam_ctx *ctx, void *cuda_stream);
int bigclam_device_state(bigclam_ctx *ctx, void **F_dev, void **F_next_dev, void **sumF_dev, int64_t *ld);
/* Device pointer of the per-node accepted-step index (int8, n entries; BIGCLAM_F_RECORD_ACCEPTED):
 * lets a multi-GPU caller exchange only the rows that changed. */
int bigclam_device_accepted(bigclam_ctx *ctx, void **accepted_dev);

/*
 * Multi-GPU (node-partitioned) pieces: a context created with an owned node range only updates
 * rows [lo,hi); rows outside are halo (read-only copies refreshed by the caller's collective).
 * See DESIGN.md (e).  bigclam_step_local runs PRE+LS+row swap for owned rows and leaves the partial
 * reductions [sum(old-new) (ld) | unused (ld) | llh_pre | n_updated] in a device buffer of 2*ld+2 doubles
 * (ld = row pitch, see bigclam_device_state) that
 * the caller all-reduces; bigclam_finish_local applies the reduced values (sumF update, :192).
 */
int bigclam_set_owned_range(bigclam_ctx *ctx, int64_t lo, int64_t hi);
int bigclam_set_owned_nodes(bigclam_ctx *ctx, const int32_t *nodes, int64_t count);   /* arbitrary owned set */
int bigclam_set_uset(bigclam_ctx *ctx, const uint8_t *node_mask);   /* uset of the following bigclam_step_local calls (NULL = all) */
int bigclam_step_local(bigclam_ctx *ctx, void **partials_dev /* 2*ld+2 doubles */);
int bigclam_finish_local(bigclam_ctx *ctx, double *llh_pre_out, int64_t *n_updated_out);  /* both NULL: asynchronous, no host sync */
int bigclam_collect_timing(bigclam_ctx *ctx);   /* sync + sum the kernel timings recorded since the last collection */
int bigclam_llh_local(bigclam_ctx *ctx, void **partials_dev /* llh at [2*ld] */);
/* Undo the most recent bigclam_finish_local (the previous F and sumF are still intact in the other
 * halves of the double buffers): used to drop the speculative step of a pipelined convergence loop. */
int bigclam_rollback(bigclam_ctx *ctx);

/*
 * Peer replicas over NVLink (one process per GPU on one box).  bigclam_ipc_export writes the two CUDA IPC
 * handles (2 x 64 bytes) of this context's F double buffer; the caller all-gathers them over its own
 * plumbing and hands all of them (world x 2 x 64 bytes, rank order) to bigclam_ipc_open_peers.  From then
 * on bigclam_step_local pushes every owned row that this step or the previous one changed straight into
 * the peers' replicas (plain stores to peer memory inside the step kernel): the row exchange that
 * replaces the reference's re-broadcast of F (bigclam4-7.scala:154) is fused into the compute kernel and
 * only the all-reduce of the partials remains.  bigclam_mark_all_changed forces a full publish (after
 * bigclam_set_F).
 */
int bigclam_ipc_export(bigclam_ctx *ctx, void *handles_out);
int bigclam_ipc_open_peers(bigclam_ctx *ctx, int32_t world, int32_t rank, const void *all_handles);
int bigclam_mark_all_changed(bigclam_ctx *ctx);
/*
 * With BIGCLAM_F_SPARSE_ROWS the replicas are (header, pool) pairs: bigclam_ipc_handle_count() handles per rank
 * (4 instead of 2) travel through bigclam_ipc_export / bigclam_ipc_open_peers, every rank allocates its owned
 * rows inside its own part of the output pool (bigclam_set_pool_region: disjoint parts, 8-byte words) and the
 * step kernel writes each owned row to the same offset of every replica — all owned rows, every step (the
 * output pool is rebuilt per step, so there is no changed-row bookkeeping).
 */
int bigclam_ipc_handle_count(const bigclam_ctx *ctx);
/*
 * Fused collective of the node-partitioned path (sparse rows): instead of an all-reduce by the host framework, the
 * reduction kernel behind every step kernel stores this rank's sums [sum(old-new) | llh | n_updated] into its slot
 * of every rank's exchange buffer (peer memory over NVLink) and raises a flag there; bigclam_finish_local /
 * bigclam_llh_finish_local then wait for all flags on the device and add the slots up in rank order (every rank
 * gets the same bits).  bigclam_xchg_export allocates the buffers and writes their 2 CUDA IPC handles (2 x 64
 * bytes); the caller all-gathers them and passes all of them (world x 2 x 64 bytes, rank order) to
 * bigclam_xchg_open_peers.  Replaces the driver-side reduce of bigclam4-7.scala:191-192 and :219.
 */
int bigclam_xchg_export(bigclam_ctx *ctx, int32_t world, int32_t rank, void *handles_out);
int bigclam_xchg_open_peers(bigclam_ctx *ctx, const void *all_handles);
int bigclam_llh_finish_local(bigclam_ctx *ctx, double *llh_out);

/*
 * All the GPUs of one box behind ONE handle, driven by one host thread — what a JVM/JNI caller uses (INTEGRATION.md):
 * one context per device (sparse rows), nodes dealt over the ranks by degree, each rank's new rows stored straight
 * into every replica by the step kernel, sums combined by the fused collective above.  No NCCL, no Python.
 * devices: `world` CUDA ordinals, NULL = 0 .. world-1.  The entry points mirror the single-GPU ones
 * (same reference lines); rank selects the replica a getter reads (they are identical).
 */
typedef struct bigclam_multi bigclam_multi;
int  bigclam_multi_create(bigclam_multi **out, int64_t n, const int64_t *rowptr, const int32_t *col,
                          const bigclam_params *params, int32_t world, const int32_t *devices);
void bigclam_multi_destroy(bigclam_multi *m);
const char *bigclam_multi_last_error(const bigclam_multi *m);     /* m may be NULL: last create error */
int  bigclam_multi_world(const bigclam_multi *m);
int  bigclam_multi_set_F(bigclam_multi *m, const double *F);
int  bigclam_multi_set_F_csr(bigclam_multi *m, const int64_t *indptr, const int32_t *indices, const double *values);
int  bigclam_multi_set_sumF(bigclam_multi *m, const double *sumF);
int  bigclam_multi_get_F(bigclam_multi *m, int32_t rank, double *F_out);
int  bigclam_multi_get_sumF(bigclam_multi *m, int32_t rank, double *sumF_out);
int  bigclam_multi_get_F_nnz(bigclam_multi *m, int64_t *nnz_out);
int  bigclam_multi_get_F_csr(bigclam_multi *m, int64_t *indptr_out, int32_t *indices_out, double *values_out);
int  bigclam_multi_step(bigclam_multi *m, const uint8_t *node_mask, double *llh_out, int64_t *n_updated_out);
int  bigclam_multi_loglikelihood(bigclam_multi *m, double *llh_out);
int  bigclam_multi_run(bigclam_multi *m, int32_t variant, double rel_tol, int64_t max_outer, double *llh_out,
                       int64_t *calls_out, double *llh_trace, int64_t trace_cap);
int  bigclam_multi_get_kernel_time(bigclam_multi *m, double *max_rank_ms_sum, int64_t *step_kernel_launches);
int  bigclam_multi_get_ls_stats(bigclam_multi *m, int64_t *nodes_asked, int64_t *nodes_searched);   /* bigclam_get_ls_stats summed over the ranks */

/*
 * F as CSR rows, the shape of the reference's RDD[(Long, BSV[Double])] (bigclam4-7.scala:97-104): indptr[n + 1],
 * indices (component of each entry, any order inside a row), values.  sumF becomes the column sums (:105-106).
 * With BIGCLAM_F_SPARSE_ROWS no dense n x K image is ever built.  bigclam_get_F_nnz sizes the output of
 * bigclam_get_F_csr (ascending indices inside a row, explicit zeros never stored).
 */
int bigclam_set_F_csr(bigclam_ctx *ctx, const int64_t *indptr, const int32_t *indices, const double *values);
int bigclam_get_F_nnz(bigclam_ctx *ctx, int64_t *nnz_out);
int bigclam_get_F_csr(bigclam_ctx *ctx, int64_t *indptr_out, int32_t *indices_out, double *values_out);
int bigclam_set_pool_region(bigclam_ctx *ctx, int64_t base_words, int64_t cap_words);
int bigclam_get_pool_capacity(bigclam_ctx *ctx, int64_t *words_out);   /* words of each row pool (what the regions partition) */

/*
 * Edge-list reader with GraphX semantics (GraphLoader.edgeListFile, bigclam4-7.scala:45;
 * collectNeighborIds(EdgeDirection.Either), :50): '#' and blank lines skipped, whitespace split,
 * CRLF safe; each edge line adds dst to src's list and src to dst's list.  Vertex ids are relabelled
 * to 0..n-1 in ascending id order (ids_out gives the original id of each dense index).
 * multiplicity: 0 = keep (literal GraphX), 1 = dedup (simple undirected graph, self loops dropped).
 * Neighbour lists are sorted ascending.  Buffers are malloc'ed by the library; release with
 * bigclam_graph_free.
 */
typedef struct {
    int64_t  n;
    int64_t  nnz;
    int64_t *rowptr;   /* n+1 */
    int32_t *col;      /* nnz */
    int64_t *ids;      /* n: original vertex id of dense index i */
    int64_t  n_edge_lines;
} bigclam_graph;

int  bigclam_graph_read_edgelist(const char *path, int32_t multiplicity, bigclam_graph *out,
                                 char *errbuf, int64_t errbuf_len);
void bigclam_graph_free(bigclam_graph *g);

/*
 * The caller behind the hot path: community extraction, Bigclamv2.scala:223-230 (SURVEY.md §8f-3).
 * member_out[u*k + c] = 1 iff F_uc >= delta, or, when the row maximum is below delta, iff F_uc equals the
 * row maximum (ties included, as coded at :227).  delta is computed by the caller:
 * sqrt(-log(1 - e)) with e = 2*count/(N*(N-1)) (:223-224; `count` there is the number of vertices that
 * have edges, not |E|).  fmax_out (optional, n) gets the row maxima.
 *
 * Membership, the one definition of this call and bigclam_extract_grouped (:225-228): with fmax_u the maximum of row u
 * over ALL k components (the zeros a sparse row does not store included), u is a member of community c iff
 *   fmax_u <  delta:  F_uc == fmax_u   (ties included)
 *   fmax_u >= delta:  F_uc >= delta.
 * bigclam_extract reads the rows where they live (sparse or dense) in batches of rows whose n_b x k bytes stay within
 * the smaller of 1 GiB and 10 % of the free device memory; no dense image of F is built.
 */
int bigclam_extract(bigclam_ctx *ctx, double delta, uint8_t *member_out, double *fmax_out);

/*
 * The communities grouped by community (the flatMap / groupByKey of :229-230), without an n x k image anywhere.
 * delta must be > 0 and not NaN (+inf is allowed: every row goes to its maximum entries), else BIGCLAM_EINVAL before
 * any device work; with delta <= 0 every zero entry would be a membership.  F must have no negative entry (the step
 * never leaves one, bigclam_set_F can): a row with one gives BIGCLAM_EUNSUPPORTED naming the smallest such row.  Then
 * every row is one of two kinds:
 *   all zero (fmax_u = 0 < delta): as coded a member of every community; listed ONCE, in zero_rows_out (ascending),
 *                                  and left out of the per-community lists;
 *   any other row:                 its memberships are among its non-zero entries.
 * The output is a CSR over communities: comptr_out (k + 1, int64), members_out (nnz, int32, each community's nodes
 * ascending, zero rows excluded), zero_rows_out (z, int32, ascending).  It depends on (F bits, delta) only: not on the
 * row layout, the batch cut, the number of GPUs or the device.
 *
 * bigclam_extract_nnz gives nnz and z; bigclam_extract_grouped fills the three outputs (sized with them; it counts
 * again, nothing is kept between the calls).  Both read F only, like the calls below: no state changes (F, sumF,
 * accepted indices, a speculative step), the context's stream, synchronous.  A NULL output (also for nnz = 0 or z = 0)
 * gives BIGCLAM_EINVAL.  The communities are filled in consecutive ranges whose members stay within the smaller of
 * 1 GiB and 10 % of the free device memory (a longer community gets a range of its own); BIGCLAM_ENOMEM, naming the
 * community, when even that cannot be allocated.
 */
int bigclam_extract_nnz(bigclam_ctx *ctx, double delta, int64_t *nnz_out, int64_t *n_zero_rows_out);
int bigclam_extract_grouped(bigclam_ctx *ctx, double delta, int64_t *comptr_out /* k + 1 */, int32_t *members_out /* nnz */,
                            int32_t *zero_rows_out /* z */);
/* The same for a multi-GPU handle: rank 0's replica is read, errors go to bigclam_multi_last_error. */
int bigclam_multi_extract_nnz(bigclam_multi *m, double delta, int64_t *nnz_out, int64_t *n_zero_rows_out);
int bigclam_multi_extract_grouped(bigclam_multi *m, double delta, int64_t *comptr_out, int32_t *members_out, int32_t *zero_rows_out);

/*
 * A score for every community of the current F, with no ground truth needed.  Membership is the rule above (delta > 0
 * and not NaN, +inf allowed, else BIGCLAM_EINVAL before any device work; a negative entry gives BIGCLAM_EUNSUPPORTED
 * naming the smallest such row).  As coded an all-zero row belongs to every community; zero_rows chooses:
 *   1: the zero rows are in every community, as coded;   0: they are in no community;   anything else: BIGCLAM_EINVAL.
 * With S_c the member set of community c and the graph the context was created with (deg(u) = rowptr[u + 1] - rowptr[u],
 * list entries counted with their multiplicity, self-loop entries included; the graph need not be symmetric):
 *   size_out[c]        = |S_c|
 *   volume_out[c]      = sum over u in S_c of deg(u)
 *   internal_out[c]    = the list entries u -> v with u and v in S_c (vol_S of bigclam4-7.scala:65; for a symmetric
 *                        graph without repeated entries, twice the edges inside S_c).  The cut is volume - internal.
 *   conductance_out[c] (optional) = conductanceLocalMin's formula (:64-67, bigclam::conductance_formula below) with
 *                        cut_S = volume - internal, vol_S = internal, sigma = rowptr[n]:
 *                        vol_T = sigma - vol_S - 2 cut_S;  0 if vol_S == 0, else 1 if vol_T == 0, else cut_S / min(vol_S, vol_T).
 *                        So an empty community (and any community without an internal entry) scores 0, and on multigraph
 *                        input vol_T, and with it the score, can be negative, as coded.  The textbook conductance is
 *                        cut / min(volume, sigma - volume); it is not an output.
 * An ego net scored this way equals conductanceLocalMin's score of its centre when the centre's own list has no repeated
 * entry and no self loop: :63 walks a repeated neighbour's list once per repetition, a set walks it once.
 *
 * Output (k values each) depends on (F bits, delta, graph, zero_rows) only: not on the row layout, the number of GPUs
 * or the device.  Device scratch is O(n + k), nothing n x k (BIGCLAM_ENOMEM when even that cannot be allocated).  Reads F
 * only (no state changes: F, sumF, accepted indices, a speculative step), on the context's stream, synchronous.  A NULL
 * required output gives BIGCLAM_EINVAL; n = 0 gives zeros.  The multi-GPU call reads rank 0's replica; its errors go to
 * bigclam_multi_last_error.
 */
int bigclam_community_stats(bigclam_ctx *ctx, double delta, int32_t zero_rows, int64_t *size_out /* k */, int64_t *volume_out /* k */,
                            int64_t *internal_out /* k */, double *conductance_out /* k, optional */);
int bigclam_multi_community_stats(bigclam_multi *m, double delta, int32_t zero_rows, int64_t *size_out, int64_t *volume_out,
                                  int64_t *internal_out, double *conductance_out);

/*
 * The communities of the current F scored against a known cover: Avg-F1 and overlapping NMI.
 *
 * Detected cover X: the communities of bigclam_extract_grouped at delta (the rule above), the all-zero rows in every
 * community (zero_rows = 1, as coded) or in none (0); X_c is community c, and only non-empty ones take part.  It is
 * the cover communities.group(..., zero_rows_everywhere) returns.  Truth cover Y: q communities as a CSR, truth_ptr
 * (q + 1, int64, truth_ptr[0] = 0, non-decreasing) and truth_members (int32 ids in [0, n)); members may come in any
 * order and a repeated id counts once.  Y may be a ground truth or the group() output of another fit.
 *
 * For a non-empty X_c and a non-empty Y_t, with x = |X_c|, y = |Y_t|, a = |X_c ∩ Y_t| and n the context's node count:
 *   F1(c, t) = (2.0 * a) / (double)(x + y)                  (the integer sum exact; communities.avg_f1's expression)
 *   f1_det[c]    = max over t of F1(c, t);  match_det[c] = the smallest t attaining it.  An empty c, or a best F1 of 0,
 *                  gives 0 and -1.  f1_truth[t] / match_truth[t]: the same in the other direction; an empty Y_t gives
 *                  0 and -1 and still counts in the mean.
 *   scores_out[0] avg_f1 = 0.5 * (mean of f1_det over the non-empty c + mean of f1_truth over all q); 0 when there is
 *                  no non-empty c or q = 0 (as communities.avg_f1).
 * Overlapping NMI (Lancichinetti, Fortunato & Kertész 2009), natural logarithms, h of an integer count m:
 *   h(m)          = m == 0 ? 0 : -(p * log(p)),  p = (double)m / (double)n
 *   H(X_c)        = h(x) + h(n - x)
 *   H(X_c | Y_t)  = max(0, ((h(a) + h(x - a)) + h(y - a)) + h(n - x - y + a) - (h(y) + h(n - y)))
 *   (c, t) is admissible iff h(a) + h(n - x - y + a) > h(x - a) + h(y - a)   (symmetric in X and Y)
 *   hcond_det[c]  = H*(X_c | Y) = the minimum of H(X_c | Y_t) over the admissible t, or H(X_c) when none is;
 *                   hcond_truth[t] = H*(Y_t | X) the same in the other direction (x and y, X and Y swapped).
 *                   Only communities with 0 < size < n enter the NMI; the others get NaN.
 *   scores_out[1] nmi_lfk = 1 - 0.5 * (mean_c H*(X_c|Y) / H(X_c) + mean_t H*(Y_t|X) / H(Y_t))
 *   scores_out[2] nmi_max = 0.5 * ((ΣH(X_c) - ΣH*(X_c|Y)) + (ΣH(Y_t) - ΣH*(Y_t|X))) / max(ΣH(X_c), ΣH(Y_t))
 *                 (McDaid, Greene & Hurley 2011).  Either NMI is NaN when one side has no community of size in (0, n).
 * Every mean and sum is a left fold in ascending id.  Scoring a fit against its own group() output in the same mode
 * gives exactly 1.0 for all three scores (the max(0, .) makes the self pair exactly 0).
 *
 * f1_det, match_det (k each), f1_truth, match_truth (q each, may be NULL when q = 0) and scores_out (3) are required;
 * hcond_det (k) and hcond_truth (q) are optional.  BIGCLAM_EINVAL before any device work for delta <= 0 or NaN (+inf
 * allowed), zero_rows not 0 or 1, q < 0 or q >= 2^31, truth_ptr[0] != 0, a decreasing truth_ptr, an id outside [0, n)
 * (naming the truth community) or a NULL required argument; a negative entry of F gives BIGCLAM_EUNSUPPORTED naming the
 * smallest such row.  The outputs depend on (F bits, delta, zero_rows, the truth sets) only: not on the row layout, the
 * order of truth members or repeats, the number of GPUs or the device.  Device scratch is O(n + k + q + Σ|Y_t|), nothing
 * n x k (BIGCLAM_ENOMEM when even that cannot be allocated).  Reads F only (no state changes), on the context's stream,
 * synchronous.  The multi-GPU call reads rank 0's replica; its errors go to bigclam_multi_last_error.
 */
int bigclam_cover_scores(bigclam_ctx *ctx, double delta, int32_t zero_rows, int64_t q, const int64_t *truth_ptr /* q + 1 */,
                         const int32_t *truth_members /* truth_ptr[q] */, double *f1_det /* k */, int32_t *match_det /* k */,
                         double *f1_truth /* q */, int32_t *match_truth /* q */, double *hcond_det /* k, optional */,
                         double *hcond_truth /* q, optional */, double *scores_out /* 3: avg_f1, nmi_lfk, nmi_max */);
int bigclam_multi_cover_scores(bigclam_multi *m, double delta, int32_t zero_rows, int64_t q, const int64_t *truth_ptr,
                               const int32_t *truth_members, double *f1_det, int32_t *match_det, double *f1_truth,
                               int32_t *match_truth, double *hcond_det, double *hcond_truth, double *scores_out);

/*
 * How the communities of the current F overlap each other: the shared members of every overlapping pair.
 *
 * Membership is the rule above (delta > 0 and not NaN, +inf allowed; F >= 0).  M_c is the set of NON-ZERO rows that are
 * members of community c, and z the number of all-zero rows; as coded, each of those is a member of every community.
 * For c != d:
 *   shared(c, d) = |M_c ∩ M_d|          (non-zero rows only)
 * The output lists, for every community c, the communities d != c with shared(c, d) >= min_shared (min_shared >= 1),
 * as a CSR over communities: ovptr_out (k + 1, int64), other_out (nnz, int32, d ascending within a row) and shared_out
 * (nnz, int32, shared(c, d)).  It is symmetric (d is in row c exactly when c is in row d, with the same count) and never
 * lists the diagonal.  size_out (k, int64, optional) gets |M_c|, and bigclam_community_overlaps_nnz's n_zero_rows_out
 * gets z.  Zero rows are kept out of every count and reported once, as bigclam_extract_grouped reports them, so the
 * caller decides what they mean:
 *   as coded (zero rows in every community): a pair's intersection is shared + z and a size is |M_c| + z; a pair that
 *     is not listed still shares the z zero rows;
 *   zero rows in no community: both are taken as they are.
 * Every number is an exact integer, and the output depends on (F bits, delta, min_shared) only: not on the row layout,
 * the range cut, the number of GPUs or the device.
 *
 * bigclam_community_overlaps_nnz gives nnz and z; bigclam_community_overlaps fills the outputs (sized with them; it
 * counts again, nothing is kept between the calls).  BIGCLAM_EINVAL before any device work for delta <= 0 or NaN,
 * min_shared < 1 or a NULL required output (other_out and shared_out also for nnz = 0); a negative entry of F gives
 * BIGCLAM_EUNSUPPORTED naming the smallest such row; n = 0 gives zeros.  Device scratch is O(n + k + the memberships of
 * the non-zero rows), nothing n x k; the rows are filled in consecutive ranges of communities whose output stays within
 * the smaller of 1 GiB and 10 % of the free device memory (a row has at most k - 1 entries, so a range always holds
 * one); BIGCLAM_ENOMEM, naming the community, when even one row's room cannot be allocated.  Reads F only (no state
 * changes: F, sumF, accepted indices, a speculative step), on the context's stream, synchronous.  The cost of a pass is
 * sum over the non-zero rows u of m_u^2 (m_u = the communities u is in) shared-memory increments, plus O(k) per
 * community.  The multi-GPU calls read rank 0's replica; their errors go to bigclam_multi_last_error.
 */
int bigclam_community_overlaps_nnz(bigclam_ctx *ctx, double delta, int32_t min_shared, int64_t *nnz_out, int64_t *n_zero_rows_out);
int bigclam_community_overlaps(bigclam_ctx *ctx, double delta, int32_t min_shared, int64_t *ovptr_out /* k + 1 */, int32_t *other_out /* nnz */,
                               int32_t *shared_out /* nnz */, int64_t *size_out /* k, optional */);
int bigclam_multi_community_overlaps_nnz(bigclam_multi *m, double delta, int32_t min_shared, int64_t *nnz_out, int64_t *n_zero_rows_out);
int bigclam_multi_community_overlaps(bigclam_multi *m, double delta, int32_t min_shared, int64_t *ovptr_out, int32_t *other_out,
                                     int32_t *shared_out, int64_t *size_out);

/*
 * The fitted model as a model of edges (the clamp of bigclam4-7.scala:166, the edge term of :218), on the current F:
 *   x_uv = sum of F_uc * F_vc over the components c that are non-zero in both rows, folded left in ascending c with
 *          every product and every sum rounded on its own (the same bits for sparse and dense rows and for (v, u));
 *   p_uv = 1 - clamp(exp(-x_uv), min_p, max_p), so log(p_uv) + x_uv is the per-edge term of the LLH.
 * Both calls read F only: no state changes (F, sumF, accepted indices, a speculative step of bigclam_step), no dense
 * n x k image; they run on the context's stream and are synchronous.  Host buffers in and out; ids outside [0, n),
 * count < 0, m < 1 or a NULL required buffer give BIGCLAM_EINVAL before any device work.  count == 0 is a no-op.
 *
 * bigclam_pair_affinity: x_out[i] = x(u[i], v[i]); p_out (optional) the p of the same pairs.  Any count (the pairs are
 * moved in bounded chunks).
 */
int bigclam_pair_affinity(bigclam_ctx *ctx, const int32_t *u, const int32_t *v, int64_t count,
                          double *x_out, double *p_out /* optional */);
/*
 * bigclam_recommend: for each query node u (nodes NULL = all n nodes in id order, then count must be n), the m nodes v
 * at distance 2 (a neighbour of a neighbour, not u and not in N(u); repeated or unsorted neighbour lists are fine) with
 * the largest x_uv > 0, by x descending, then v ascending.  A pair with x = 0 has the floor probability 1 - max_p and is
 * never returned.  v_out / x_out: count x m, row i padded with -1 / 0 after its found_out[i] (optional) entries.  Two-hop
 * lists are built in batches whose scratch stays within the smaller of 1 GiB and 10 % of the free device memory; a node
 * whose list alone is longer gets scratch of its own, and BIGCLAM_ENOMEM (naming the node) only when that fails.
 */
int bigclam_recommend(bigclam_ctx *ctx, const int32_t *nodes /* NULL = all n */, int64_t count, int32_t m,
                      int32_t *v_out /* count x m, -1 padded */, double *x_out /* count x m, 0 padded */,
                      int32_t *found_out /* count, optional */);
/* The same for a multi-GPU handle: rank 0's replica is read, errors go to bigclam_multi_last_error. */
int bigclam_multi_pair_affinity(bigclam_multi *m, const int32_t *u, const int32_t *v, int64_t count,
                                double *x_out, double *p_out);
int bigclam_multi_recommend(bigclam_multi *m, const int32_t *nodes, int64_t count, int32_t mm,
                            int32_t *v_out, double *x_out, int32_t *found_out);

/*
 * A graph sampled from the model, on the current F.  For every unordered pair u < v of the n nodes:
 *   shared      rows u and v have at least one component that is non-zero in both: p_uv = the p of
 *               bigclam_pair_affinity (the same bits, its floor 1 - max_p included);
 *   not shared  p_uv = eps, a background probability, 0 <= eps < 1: 1 - max_p gives the model as coded (the clamp of
 *               bigclam4-7.scala:166 applied to every pair), 0 gives community edges only;
 * and the pair is an edge iff r(seed, u, v) < p_uv, where
 *   key = (uint64_t)u << 32 | v,   h = mix(seed ^ mix(key)),   r = (h >> 11) * 2^-53,
 *   mix(z) = the splitmix64 step: z += 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 *            z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31)   (all mod 2^64).
 * The result is a function of (F, seed, eps, min_p, max_p) only: not of the row layout (sparse or dense), the batch
 * cut, the number of GPUs or the device.  It is a symmetric CSR, the shape bigclam_create takes: rowptr_out (n + 1) and
 * col_out (nnz), every row ascending, no self loops, no duplicates.
 *
 * bigclam_sample_graph_nnz gives nnz; bigclam_sample_graph fills rowptr_out and col_out (sized with the nnz of the
 * same F, seed and eps; it counts again, nothing is kept between the calls).  Both read F only, like the calls above:
 * no state changes, no dense n x k image, the context's stream, synchronous.  eps NaN, negative or >= 1, or a NULL
 * output (col_out included, also for nnz = 0) gives BIGCLAM_EINVAL before any device work.  The rows are decided in
 * batches whose output stays within the smaller of 1 GiB and 10 % of the free device memory (a longer row gets a batch
 * of its own); BIGCLAM_ENOMEM when a batch's buffer cannot be allocated.
 */
int bigclam_sample_graph_nnz(bigclam_ctx *ctx, uint64_t seed, double eps, int64_t *nnz_out);
int bigclam_sample_graph(bigclam_ctx *ctx, uint64_t seed, double eps, int64_t *rowptr_out /* n + 1 */, int32_t *col_out /* nnz */);
/* The same for a multi-GPU handle: rank 0's replica is read, errors go to bigclam_multi_last_error. */
int bigclam_multi_sample_graph_nnz(bigclam_multi *m, uint64_t seed, double eps, int64_t *nnz_out);
int bigclam_multi_sample_graph(bigclam_multi *m, uint64_t seed, double eps, int64_t *rowptr_out, int32_t *col_out);

/*
 * Fold-in: the rows of q NEW nodes (arrived after the fit), with the context's F and sumF held fixed.  Query node u
 * comes with its neighbour list among the n fitted nodes, as a CSR: rowptr (q + 1) and col (rowptr[q] ids in [0, n));
 * repeats and any order are allowed, as in bigclam_create.  Its objective is the step's (bigclam4-7.scala:157-184) for u
 * appended to the graph, with every other row fixed:
 *   l_u(f) = sum_{v in N(u)} [log(1 - clamp(exp(-f.F_v), min_p, max_p)) + f.F_v] - f.sumF
 * (sumF the fitted one; the candidates are scored with sumF - f_old + f_new as at :176-180).  For each query node on its
 * own:
 *   start from f_0 = 0, l_0 = l_u(0);  for t = 1 .. max_iter: the reference's line search from f_{t-1} over the step
 *   sizes of bigclam_step_sizes(beta, max_inter), candidates clamp(f + s g, 0, max_f), keeping the largest s with
 *   l_u(cand) >= l_{t-1} + alpha s |g|^2 (|g|^2 over all k components, :181).  No candidate passes: stop at f_{t-1}.
 *   Otherwise f_t = the candidate; stop if |1 - l_t / l_{t-1}| < rel_tol (:237 for one node).
 * iters = the number of accepted steps; the row returned is the last one accepted, llh = l_u of it.  A node with an
 * empty list gets a zero row, llh = 0 and iters = 0.  Query nodes never see each other: a node's results are the same
 * bits whatever the other nodes of the call, their order or the batches they are cut into.
 *
 * The rows come in bigclam_get_F_csr's form (indptr q + 1, ascending indices, no stored zeros), ready for
 * bigclam_set_F_csr of a context over the extended graph.  bigclam_fold_in_nnz gives their total nnz; bigclam_fold_in
 * fills indptr_out, indices_out and values_out (sized with that nnz; the rows are computed again, nothing is kept
 * between the calls) and, optionally, llh_out (q) and iters_out (q).  Both read F only, like the calls above: no state
 * changes (F, sumF, accepted indices, a speculative step), no dense n x k or q x k image, the context's stream,
 * synchronous.  q < 0, max_iter < 1, rel_tol negative or NaN, a NULL required buffer, rowptr[0] != 0, a decreasing
 * rowptr or an id outside [0, n) give BIGCLAM_EINVAL before any device work; a context with min_f != 0 gives
 * BIGCLAM_EUNSUPPORTED.  q == 0 is a no-op (nnz 0).  The nodes go in batches whose scratch stays within the smaller of
 * 1 GiB and 10 % of the free device memory (a node that needs more gets a batch of its own); BIGCLAM_ENOMEM, naming the
 * node, when even that cannot be allocated.
 */
int bigclam_fold_in_nnz(bigclam_ctx *ctx, int64_t q, const int64_t *rowptr, const int32_t *col, int32_t max_iter, double rel_tol,
                        int64_t *nnz_out);
int bigclam_fold_in(bigclam_ctx *ctx, int64_t q, const int64_t *rowptr, const int32_t *col, int32_t max_iter, double rel_tol,
                    int64_t *indptr_out /* q + 1 */, int32_t *indices_out, double *values_out,
                    double *llh_out /* q, optional: l_u of the returned row */, int32_t *iters_out /* q, optional */);
/* The same for a multi-GPU handle: rank 0's replica is read, errors go to bigclam_multi_last_error. */
int bigclam_multi_fold_in_nnz(bigclam_multi *m, int64_t q, const int64_t *rowptr, const int32_t *col, int32_t max_iter,
                              double rel_tol, int64_t *nnz_out);
int bigclam_multi_fold_in(bigclam_multi *m, int64_t q, const int64_t *rowptr, const int32_t *col, int32_t max_iter, double rel_tol,
                          int64_t *indptr_out, int32_t *indices_out, double *values_out, double *llh_out, int32_t *iters_out);

/*
 * Callers in front of the hot path (host side, one-off integer graph work; SURVEY.md §8f-2).
 * bigclam_conductance_seeds = conductanceLocalMin() (bigclam4-7.scala:58-73): ego-net conductance of every
 * node, candidates = the min-id neighbour of each node (tuple .min at :70), ranked by conductance ascending
 * (ties by id).  seeds_out has room for n ids; *n_seeds_out receives the number of candidates.
 * bigclam_init_neighbor_com_F = initNeighborComF(K) (bigclam4-7.scala:81-108): column c of F is the
 * indicator of the neighbours of the c-th (in id order) of the first K ranked seeds; include_self adds the
 * seed (Bigclamv2.scala:70); missing columns are random 0/1 from a seeded xorshift64* (the reference's
 * Random is unseeded).  The result goes to bigclam_set_F.
 */
int bigclam_conductance_seeds(int64_t n, const int64_t *rowptr, const int32_t *col, double *conductance_out,
                              int32_t *seeds_out, int64_t *n_seeds_out);
/* The same ranking with the ego-net conductances computed on the GPU (one warp per node, csrc/initf_gpu.cu); device:
 * CUDA ordinal, -1 = current.  Fails without a CUDA device (BIGCLAM_ECUDA): bigclam_conductance_seeds is the host path. */
int bigclam_conductance_seeds_gpu(int64_t n, const int64_t *rowptr, const int32_t *col, int32_t device,
                                  double *conductance_out, int32_t *seeds_out, int64_t *n_seeds_out);
int bigclam_init_neighbor_com_F(int64_t n, const int64_t *rowptr, const int32_t *col, int32_t k,
                                const int32_t *ranked_seeds, int64_t n_ranked, int32_t include_self,
                                uint64_t pad_seed, double *F_out);
/*
 * bigclam_init_F = initNeighborComF(K) (bigclam4-7.scala:81-108) built on the context's device, straight into the
 * context, from the graph it was created with: the F rows and sumF bits that bigclam_init_neighbor_com_F(n, rowptr, col,
 * K, ranked_seeds, n_ranked, include_self, pad_seed, F0) followed by bigclam_set_F(ctx, F0) leave, padding draws
 * included, without an n x K array on either side (device scratch O(nnz(F0) + n + K)).  Column c of the first
 * min(K, n_ranked) seeds in id order marks the entries of that seed's own neighbour list (any CSR: repeated entries and
 * seeds allowed).  A seed outside [0, n) gives BIGCLAM_EINVAL, rows that do not fit the row pool BIGCLAM_ENOMEM; either
 * way F and sumF stay as they were.  bigclam_multi_init_F builds the same rows on every rank.
 */
int bigclam_init_F(bigclam_ctx *ctx, const int32_t *ranked_seeds, int64_t n_ranked, int32_t include_self, uint64_t pad_seed);
int bigclam_multi_init_F(bigclam_multi *m, const int32_t *ranked_seeds, int64_t n_ranked, int32_t include_self, uint64_t pad_seed);

/* Library / device probe (no compute): returns the number of visible CUDA devices or <0. */
int bigclam_device_count(void);
const char *bigclam_version(void);

#ifdef __cplusplus
}

#include <math.h>
#if defined(__CUDACC__)
#define BIGCLAM_HD __host__ __device__
#else
#define BIGCLAM_HD
#endif
namespace bigclam {
/* The conductance of conductanceLocalMin (bigclam4-7.scala:64-67) from cut_S, vol_S and sigma (integers as doubles):
 * the ego nets of bigclam_conductance_seeds_gpu and the communities of bigclam_community_stats score through it. */
BIGCLAM_HD inline double conductance_formula(double cut_S, double vol_S, double sigma) {
    const double vol_T = sigma - vol_S - cut_S * 2;                                   /* :66 */
    return (vol_S == 0) ? 0.0 : (vol_T == 0) ? 1.0 : cut_S / fmin(vol_S, vol_T);    /* :67 */
}
}  // namespace bigclam
#undef BIGCLAM_HD
#endif
#endif /* BIGCLAM_B200_H */
