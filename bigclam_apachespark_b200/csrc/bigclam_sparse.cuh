// bigclam_sparse.cuh — the step (codes/bigclam4-7.scala:152-223) over SPARSE rows of F: layout, the general
// one-warp-per-node path (any degree, any row length, K <= 16384) and the split-hub phases.  The tile path for
// small nodes and the kernels themselves are in bigclam_tile.cuh.
//
// Why: the reference keeps F as Breeze sparse vectors (`BSV[Double]`, bigclam4-7.scala:97-104) because the rows
// ARE sparse: on the bench workload (com-amazon, K = 200) a row holds ~9 non-zeros of 200 through the whole
// run and ~17 components are "active" in a line search.  A row is (count, ascending component indices, values)
// in a per-step pool, every neighbour row is read once per step (~112 bytes instead of 1.6 KB), and all
// per-edge work is proportional to the row's non-zeros.
//
// Layout (per F buffer; double-buffered like the dense F):
//   hdr[u]      uint64: (offset in 8-byte words << 24) | count
//   pool        row block at `offset` (16-byte aligned, a multiple of 16 bytes — one bulk copy moves it):
//               vpad(count) doubles, then ipad(count) uint16 indices (ascending);  vpad = count rounded up to 2,
//               ipad = count rounded up to 8.  A node whose step was accepted is followed by its DELTA block in
//               the same format: the non-zero (old - new) components (:191-192), dcnt[u] of them.
//   pool_top    bump allocator of the OUTPUT pool (words), zeroed before every step.  The input pool is only
//               read (Jacobi), so a step whose pool overflowed can simply be repeated with a larger pool.
//
// Per-node results (no floating-point atomics anywhere: the sums over nodes are taken afterwards, in a fixed
// order, by reduce_kernel — bit-identical from run to run):
//   node_llh[u]  llh_u of the PRE block (:168)          accepted[u]  accepted step index, -1 = row kept
//   dcnt[u]      entries of the delta block
//
// General path, per node (one warp), with fu scattered into a dense shared-memory vector fu_d[ld]:
//   PRE   the entries of up to 32 neighbour rows are staged in shared memory; lane e walks row e:
//         x_e = sum_i val_i * fu_d[idx_i]; the gradient sum g_d[idx] += w_e * val goes neighbour by neighbour;
//   scan  one pass over the ld components turns g_d into the gradient (:168), sums |g|^2 and lists the
//         active components (fu > 0 or g > 0);
//   LS    lane (trial j, edge parity h) walks the staged entries of its edges:
//         D = sum_i clamp(fu_d[idx_i] + s_j * g_d[idx_i]) * val_i — an inactive component clamps to 0 and adds
//         exactly nothing; two edges per lane in flight;
//   SWAP  the accepted candidate's non-zeros are compacted (ascending) into the staging buffer, a block is
//         taken from the output pool, the row, its delta block and its header are written.
//
// Wide rows (ld > 1024, the `kWide` variant of the step kernel): the K-sized vectors of a warp (fu_d, g_d, the entry
// buffer, aidx) no longer fit shared memory, so they live in the warp's slice of a global scratch that the context
// allocates and zeroes once (sp_wide_warp_bytes); sumF is read from global memory.  Every node is a general-path item
// (no tiles).  The per-node passes cover only the components the node TOUCHES (its own non-zeros and its neighbours'),
// kept in a per-warp bitmask in shared memory: the gradient scan, the active list and the clears visit its set bits.
// An untouched component has fu = 0 and gradient -sumF_c <= 0: it is inactive and enters |g|^2 through
// S2_all - sum_touched sumF_c^2 (the identity of the tile path).  The line-search bounds of the general path
// (BIGCLAM_LS_PRUNE=2) are not compiled into the wide variant.  The scratch is all zero between nodes and launches.
//
// Limits: ld <= 1024 (ld <= kSpMaxK with the wide variant), MIN_F_ == 0.
#pragma once
#include "bigclam_kernels.cuh"

namespace bigclam {

#ifndef BIGCLAM_GEN_BOUNDS          // 1: the line-search bounds of the general path are compiled in (used when SparseArgs::ls_prune > 1)
#define BIGCLAM_GEN_BOUNDS 1
#endif
#ifndef BIGCLAM_GEN_INLINE          // how the general path (one node / one hub item per call, a single call site each) is compiled into the kernel
#define BIGCLAM_GEN_INLINE __forceinline__
#endif

constexpr int kSpBlocksPerSM = 2;
constexpr int kSpWarps = 8;            // warps per block at most; wide rows run fewer (sp_warps_per_block)
constexpr int kSpThreads = kSpWarps * 32;
// staged neighbour entries per chunk of the general path: at least one full row always fits
__host__ __device__ inline int sp_entries(int ld) { return ld > 512 ? ld : 512; }

__host__ __device__ inline uint64_t sp_pack(uint64_t off8, uint32_t cnt) { return (off8 << 24) | (uint64_t)cnt; }
__host__ __device__ inline uint32_t sp_cnt(uint64_t h) { return (uint32_t)(h & 0xffffffull); }
__host__ __device__ inline uint64_t sp_off8(uint64_t h) { return h >> 24; }
__host__ __device__ inline uint32_t sp_vpad(uint32_t cnt) { return (cnt + 1u) & ~1u; }
__host__ __device__ inline uint32_t sp_ipad(uint32_t cnt) { return (cnt + 7u) & ~7u; }
__host__ __device__ inline uint64_t sp_words(uint32_t cnt) { return (uint64_t)sp_vpad(cnt) + sp_ipad(cnt) / 4u; }   // 8-byte words of a block
__host__ __device__ inline const unsigned short *sp_idx(const double *vals, uint32_t cnt) {
    return reinterpret_cast<const unsigned short *>(vals + sp_vpad(cnt));
}
__host__ __device__ inline unsigned short *sp_idx(double *vals, uint32_t cnt) {
    return reinterpret_cast<unsigned short *>(vals + sp_vpad(cnt));
}

struct TileMeta {   // a group of consecutive small nodes of the processing order handled together by one warp
    int32_t pos0;   // first position (index into StepArgs::meta)
    int32_t ecol0;  // first entry of the tile in SparseArgs::tcol
    int32_t nn;     // nodes (<= kTlMaxNodes)
    int32_t ne;     // edges (<= kTlMaxEdges)
};

struct SparseArgs {
    const uint64_t *hdr_in;
    const double *pool_in;
    uint64_t *hdr_out;
    double *pool_out;
    unsigned long long *pool_top;      // words used of this rank's region of pool_out
    uint64_t pool_cap8;                // capacity of that region in words
    uint64_t region_base8;             // where the region starts in pool_out (0 on a single GPU)
    int32_t *overflow;                 // set when a row did not fit (the step must be repeated with a larger pool)
    // per-node results (see the header comment)
    double *node_llh;
    unsigned short *dcnt;
    int8_t *accepted;                  // always written by a line-search launch
    // node-partitioned multi-GPU: the owners' new rows go to the same offsets of every replica's output pool
    // (plain stores to IPC-mapped peer memory over NVLink); each rank allocates only inside its own region, so
    // all replicas end up with the same layout and no remote atomics are needed.
    int32_t n_peers;
    uint64_t *peer_hdr[7];
    double *peer_pool[7];
    unsigned int *hub_work;            // next hub item to hand out (zeroed per launch); items: StepArgs::hub_items
    // work list after the hubs: n_gen nodes for the general path (positions n_hubs ..), then the tiles
    int32_t n_gen;
    int32_t ntiles;
    const TileMeta *tiles;
    const int32_t *tcol;               // per tile edge: neighbour id | (node index within the tile << 28)
    unsigned int *stats;               // optional [tiles done on the tile path, tiles that fell back, nodes line-searched, nodes that asked for it]
    // line search by bounds (bigclam_tile.cuh, H2): 0 = every candidate of every node is evaluated (BIGCLAM_F_LS_EXHAUSTIVE),
    // 1 = bounds on the tile path only, 2 = on the general path too
    int32_t ls_prune;
    float pr_xlo, pr_kinv, pr_cap;     // x_lo rounded down, 1 / (1 - MAX_P_) and S_hi - S_lo rounded up
    unsigned char *wide_scratch;       // wide rows: sp_wide_warp_bytes(ld) per resident warp, all zero between launches
#ifdef BIGCLAM_TL_PHASE_CLOCKS
    unsigned long long *phase_clocks;  // phase profile of the tile path (bigclam_tile.cuh, kTlPcBuckets)
#endif
};

// The dense per-warp vectors are padded to a multiple of 32 components (zeros: a padding component has
// fu = sumF = 0, hence gradient 0, never active), so that the loops over components need no bounds checks.
__host__ __device__ inline int sp_ldp(int ld) { return (ld + 31) & ~31; }
// general path, per-warp shared memory:
//   fu_d[ldp] | g_d[ldp] | ent_val[E] | ent_idx[E] u16 | aidx[max(ld, 256)] u16 | poff[40] u16 | cbal[32] u32 | ccum[32] u16
__host__ __device__ inline size_t sp_gen_warp_bytes(int ld) {
    return sizeof(double) * 2 * (size_t)sp_ldp(ld) + (size_t)sp_entries(ld) * 10 + 2 * (size_t)(ld > 256 ? ld : 256) + 2 * 40 + 4 * 32 + 2 * 32;
}
// wide rows: the largest K of a sparse-row context (component ids, dcnt, poff and aidx are uint16), and the ld above
// which the wide variant runs
constexpr int kSpMaxK = 16384;
constexpr int kSpWideLd = 1024;
__host__ __device__ inline bool sp_wide(int ld) { return ld > kSpWideLd; }
// wide rows, per warp: global scratch  fu_d[ldp] | g_d[ldp] | ent_val[E] | ent_idx[E] u16 | aidx[ld] u16
__host__ __device__ inline size_t sp_wide_warp_bytes(int ld) {
    return (sizeof(double) * 2 * (size_t)sp_ldp(ld) + (size_t)sp_entries(ld) * 10 + 2 * (size_t)ld + 15) & ~(size_t)15;
}
// ... and shared memory  tmask[ldp / 32] u32 | cbal[E / 32] u32 | poff[40] u16 | ccum[E / 32] u16  (a chunk of the entry
// buffer may hold E = ld entries: compact_active keeps one ballot per 32 of them)
__host__ __device__ inline size_t sp_wide_smem_warp_bytes(int ld) {
    return (4 * (size_t)(sp_ldp(ld) / 32) + 6 * (size_t)(sp_ldp(sp_entries(ld)) / 32) + 2 * 40 + 15) & ~(size_t)15;
}
// block: steps[kMaxSteps] | wpb x warp region
__host__ __device__ inline size_t sp_wide_block_smem_bytes(int ld, int wpb) {
    return sizeof(double) * kMaxSteps + (size_t)wpb * sp_wide_smem_warp_bytes(ld);
}

// Split hubs.  A node whose neighbour list is long enough to dominate a launch when one warp walks it is split
// into segments of kSpHubSeg edges that different warps work on; the pieces meet in a global scratch row per
// hub (G[ld] | S1 | ST[16], stride ld + 32 doubles, two counters per hub):
//   phase 1  PRE of one segment: its share of sum_v w_v fv and of S1 into the segment's own slot of the scratch
//            (no atomics: the hub's warps add the slots up in slot order, so the result is reproducible);
//   phase 2  line search of one segment, once all phase-1 segments of the hub are in;
//   phase 3  once per hub, after its phase-2 segments: gradient, active set, Armijo decision, new row.
// Items are handed out in that order by one counter and every warp holds one item at a time on a grid whose
// warps are all resident, so a waiting warp only waits for items that are being processed: no deadlock.
constexpr int kSpHubSeg = 96;
constexpr int kSpHubMaxSlices = 192;      // very large hubs get longer segments: the slot sums are taken by one warp per hub
// scratch of one hub: (nslices + 1) x (ld + 32) doubles: slice sl holds  G_sl[ld] | S1_sl | ST_sl[16], the last
// slot the sums over the slices (G | S1)
__host__ __device__ inline size_t sp_hub_stride(int ld) { return (size_t)ld + 32; }

// ---------------------------------------------------------------------------------------------------------------
// Line search by bounds (derivation: bigclam_tile.cuh, phase H2): the per-node terms of the bound
//   phi(nf_j) - phi(fu) <= min(s Qn, R3) + min(s Qp, G1) - kappa s Mp + c0 + s c1 + Hs_j
// and the test that excludes candidate j.  Shared by the tile path and the general path.
struct LsBound {
    double Qn, Qp, Mp, G1, R3;
    float c0, c1, kap0;
    __device__ __forceinline__ bool cannot_pass(double sj, float Hs, double alpha, double G2node) const {
        const float sfu = __double2float_ru(sj);
        const float kap = fminf(1.0f, __fdividef(kap0, sfu) * 0.9999f);
        const double bound = fmin(sj * Qn, R3) + fmin(sj * Qp, G1) - sj * ((double)kap * Mp) + (double)(fmaf(Hs, 1.00001f, c0) + sfu * c1);
        return bound < (alpha * sj) * G2node * (1.0 - 1.0e-9);
    }
};
// One edge's share Hs of candidate ln(s) = lns given the edge's code (lnthr, Lp): 0 up to lnthr; beyond it
// min(cap, lns + Lp) for an edge that is clamped flat, or the constant -1000 - Lp (an edge next to x_lo, Lp < -500).
__device__ __forceinline__ float ls_edge_share(float lns, float lnthr, float Lp, float cap) {
    if (!(lns > lnthr)) return 0.0f;
    return (Lp < -500.0f) ? (-1000.0f - Lp) : fminf(cap, fmaxf(lns + Lp, 0.0f));
}
// The code of an edge that is clamped flat (x <= x_lo): Dp = sum_c max(g_c, 0) fv_c > 0.
__device__ __forceinline__ void ls_code_flat(float xf, double Dp, float xlo_f, float kinv_f, float &lnthr, float &Lp) {
    const float Df = __double2float_ru(Dp) * 1.000001f;
    const float sthr = (xlo_f - xf) / Df * 0.99999f;                    // x + s Dp stays below x_lo up to here
    if (sthr > 0.0f) {
        const float t1 = __log2f(sthr), t2 = __log2f(kinv_f * (Df + xf / sthr));
        lnthr = t1 * 0.69314718f - fmaf(1.0e-6f, fabsf(t1), 1.0e-4f);
        Lp = t2 * 0.69314718f + fmaf(1.0e-6f, fabsf(t2), 1.0e-4f);
    } else {
        lnthr = -3.0e38f;                                               // (always at the cap)
        Lp = 3.0e38f;
    }
}
// The code of an edge in range next to x_lo with violation `vnear`: charged from x + s En < x_lo on (En < 0).
__device__ __forceinline__ void ls_code_near(double x, double x_lo, double En, float vnear, float &lnthr, float &Lp) {
    const float sthr = __double2float_rd((x - x_lo) / (-En)) * 0.99999f;
    if (sthr > 0.0f) {
        const float t1 = __log2f(sthr);
        lnthr = t1 * 0.69314718f - fmaf(1.0e-6f, fabsf(t1), 1.0e-4f);
    } else {
        lnthr = -3.0e38f;
    }
    Lp = -1000.0f - vnear;
}

struct RowSrc {                    // the rows of the current F: sparse (hdr, pool) when hdr != nullptr, else dense (F, ld)
    const uint64_t *hdr;
    const double *pool;
    const double *F;
    int32_t k, ld;
};

// ---------------------------------------------------------------------------------------------------------------
// The general path: everything one warp needs to process one node (or one hub item).  kWide: wide rows (see the
// header comment): K-sized vectors in global scratch, sumF in global memory, touched-only per-node passes.
// kFold: the phases as fold-in runs them (FoldGen): rows from `rs`, sparse or dense, and sumF' = sumF + f.
template <bool kWide, bool kFold = false>
struct SpGen {
    // launch-wide
    const StepArgs *a;
    const SparseArgs *sp;
    const RowSrc *rs;                // fold-in: the fitted rows
    const double *s_steps;
    const double *s_sumF;            // (wide rows: the global sumF)
    const float *s_lns;              // upper bounds of ln(step size), 16 values (line search by bounds)
    double S2_all;                   // wide rows: sum_c sumF_c^2 (fixed order)
    EdgeConst ec;
    // per warp
    double *fu_d, *g_d, *ent_val;
    unsigned short *ent_idx, *aidx, *poff, *ccum;
    unsigned int *cbal;
    unsigned int *tmask;             // wide rows: the components the current node touches, one bit each
    int lane, ld, ldp, ecap;
    unsigned lt_mask;

    // wide rows: the K-sized vectors in the warp's slice `gbase` of the global scratch, the rest in shared memory
    __device__ __forceinline__ void carve_wide(unsigned char *gbase, unsigned char *sbase, int ld_, int lane_) {
        ld = ld_;
        ldp = sp_ldp(ld_);
        ecap = sp_entries(ld_);
        lane = lane_;
        lt_mask = (1u << lane_) - 1u;
        fu_d = reinterpret_cast<double *>(gbase);
        g_d = fu_d + ldp;
        ent_val = g_d + ldp;
        ent_idx = reinterpret_cast<unsigned short *>(ent_val + ecap);
        aidx = ent_idx + ecap;
        tmask = reinterpret_cast<unsigned int *>(sbase);
        cbal = tmask + ldp / 32;
        poff = reinterpret_cast<unsigned short *>(cbal + sp_ldp(ecap) / 32);
        ccum = poff + 40;
    }
    __device__ __forceinline__ void touch(int c) { atomicOr(tmask + (c >> 5), 1u << (c & 31)); }

    __device__ __forceinline__ void carve(unsigned char *wbase, int ld_, int lane_) {
        ld = ld_;
        ldp = sp_ldp(ld_);
        ecap = sp_entries(ld_);
        lane = lane_;
        lt_mask = (1u << lane_) - 1u;
        fu_d = reinterpret_cast<double *>(wbase);
        g_d = fu_d + ldp;
        ent_val = g_d + ldp;
        ent_idx = reinterpret_cast<unsigned short *>(ent_val + ecap);
        aidx = ent_idx + ecap;
        poff = aidx + (ld > 256 ? ld : 256);
        cbal = reinterpret_cast<unsigned int *>(poff + 40);
        ccum = reinterpret_cast<unsigned short *>(cbal + 32);
    }
    // the tile path uses the same bytes: the dense vectors must be zero whenever the general path starts
    __device__ __forceinline__ void clear_dense() {
#pragma unroll 1
        for (int i = lane; i < ldp; i += 32) { fu_d[i] = 0.0; g_d[i] = 0.0; }
        __syncwarp();
    }

    // Stages the rows of up to 32 neighbours (ids colp[0 .. cnt32), the low 28 bits when `tagged`) of one node
    // into the entry buffer: the longest prefix of them whose entries fit (at least one: a row has at most
    // ld <= ecap entries).  Returns the number ne of staged neighbours; poff[e] .. poff[e + 1] is row e's range.
    __device__ __forceinline__ int stage_chunk(const int32_t *__restrict__ colp, int cnt32) {
        const uint64_t *__restrict__ hdr_in = sp->hdr_in;
        const double *__restrict__ pool_in = sp->pool_in;
        const int v = (lane < cnt32) ? (colp[lane] & 0x0fffffff) : 0;
        const uint64_t hv = (lane < cnt32) ? __ldg(hdr_in + v) : 0ull;
        const int cv = (int)sp_cnt(hv);
        int incl = cv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        const unsigned fit = __ballot_sync(0xffffffffu, (lane < cnt32) && (incl <= ecap));
        const int ne = __popc(fit);                     // incl is monotone: the fitting lanes are 0 .. ne-1
        if (lane == 0) poff[0] = 0;
        if (lane < ne) poff[lane + 1] = (unsigned short)incl;
        __syncwarp();
        // the T entries of the ne rows, 32 at a time, one per lane: all loads of a round are in flight together
        const int T = (ne > 0) ? __shfl_sync(0xffffffffu, incl, ne - 1) : 0;
#pragma unroll 1
        for (int base = 0; base < T; base += 32) {
            const int j = base + lane;
            int lo = 0, hi = ne;                                   // row of entry j: the largest e with poff[e] <= j
#pragma unroll
            for (int s = 0; s < 5; ++s) {
                const int mid = (lo + hi) >> 1;
                const bool le = (int)poff[mid] <= j;
                if (hi - lo > 1) { if (le) lo = mid; else hi = mid; }
            }
            const uint64_t he = __shfl_sync(0xffffffffu, hv, lo);
            if (j < T) {
                const int ce = (int)sp_cnt(he);
                const double *vals = pool_in + sp_off8(he);
                const int i = j - (int)poff[lo];
                ent_val[j] = __ldg(vals + i);
                ent_idx[j] = __ldg(sp_idx(vals, (uint32_t)ce) + i);
            }
        }
        __syncwarp();
        return ne;
    }
    // Fold-in over dense rows: the same, each row compacted to its non-zeros by the whole warp, row after row, while
    // the rows fit.
    __device__ __forceinline__ int stage_dense(const int32_t *__restrict__ colp, int cnt32) {
        int total = 0, ne = 0;
        if (lane == 0) poff[0] = 0;
#pragma unroll 1
        for (; ne < cnt32; ++ne) {
            const double *row = rs->F + (size_t)colp[ne] * rs->ld;
            int cv = 0;
#pragma unroll 1
            for (int c0 = 0; c0 < rs->k; c0 += 32)
                cv += __popc(__ballot_sync(0xffffffffu, c0 + lane < rs->k && __ldg(row + c0 + lane) != 0.0));
            if (total + cv > ecap) break;                 // (never for the first row: k <= ecap)
#pragma unroll 1
            for (int c0 = 0; c0 < rs->k; c0 += 32) {
                const int c = c0 + lane;
                const double v = (c < rs->k) ? __ldg(row + c) : 0.0;
                const unsigned bal = __ballot_sync(0xffffffffu, v != 0.0);
                if (v != 0.0) {
                    const int p = total + __popc(bal & lt_mask);
                    ent_val[p] = v;
                    ent_idx[p] = (unsigned short)c;
                }
                total += __popc(bal);
            }
            if (lane == 0) poff[ne + 1] = (unsigned short)total;
        }
        __syncwarp();
        return ne;
    }
    __device__ __forceinline__ int stage(const int32_t *colp, int cnt32) {
        if constexpr (kFold)
            if (rs->hdr == nullptr) return stage_dense(colp, cnt32);
        return stage_chunk(colp, cnt32);
    }

    // PRE over the edges [eb, ee) of a node whose fu is in fu_d: returns this lane's share of S1 (lane e holds the
    // terms of the chunks' e-th rows); with `axpy` the weighted neighbour rows are added into g_d, and with `mark`
    // their components are set in tmask.
    __device__ __forceinline__ double pre_range(const int32_t *colbase, int eb, int ee, bool axpy, int &nchunks, int &ne_last,
                                                bool mark = kWide) {
        double S1 = 0.0;
        nchunks = 0;
        ne_last = 0;
#pragma unroll 1
        for (int cb = eb; cb < ee;) {
            const int ne = stage(colbase + cb, min(32, ee - cb));
            double x = 0.0;
            if (lane < ne) {
                const int end = poff[lane + 1];
#pragma unroll 1
                for (int i = poff[lane]; i < end; ++i) x = fma(ent_val[i], fu_d[ent_idx[i]], x);
            }
            double w;
            const double t = edge_term<true>(x, ec, w);
            S1 += (lane < ne) ? t : 0.0;
            if (axpy) {
#pragma unroll 1
                for (int e = 0; e < ne; ++e) {
                    const double we = __shfl_sync(0xffffffffu, w, e);
                    const int pe = poff[e], pn = poff[e + 1];
#pragma unroll 1
                    for (int i = pe + lane; i < pn; i += 32) {
                        const int c = ent_idx[i];
                        g_d[c] = fma(we, ent_val[i], g_d[c]);
                        if (mark) touch(c);
                    }
                    __syncwarp();
                }
            }
            cb += ne;
            ne_last = ne;
            ++nchunks;
        }
        return S1;
    }
    // g_d (sum of weighted neighbour rows) -> gradient (:168) in place; returns |g|^2, lists the active
    // components in aidx (m of them) and tells whether any candidate can reach MAX_F_.
    __device__ __forceinline__ double scan_gradient(int &m, bool &need_hi) {
        double G2 = 0.0;
        bool hi_lane = false;
        m = 0;
        const double max_f = a->max_f;
#pragma unroll 1
        for (int c0 = 0; c0 < ldp; c0 += 32) {          // (padding components: f = g = 0, inactive)
            const int c = c0 + lane;
            const double f = fu_d[c];
            const double g = (g_d[c] - ((kWide && c >= ld) ? 0.0 : s_sumF[c])) + f;     // (the global sumF has ld entries)
            g_d[c] = g;
            G2 = fma(g, g, G2);
            const bool act = (f > 0.0 || g > 0.0);
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            if (act) {
                aidx[m + __popc(bal & lt_mask)] = (unsigned short)c;
                hi_lane |= (f + g > max_f);
            }
            m += __popc(bal);
        }
        G2 = warp_sum(G2);
        need_hi = __any_sync(0xffffffffu, hi_lane);
        __syncwarp();
        return G2;
    }
    // Wide rows: the same over the TOUCHED components only (ascending, from the bitmask); the others are inactive and
    // enter |g|^2 through S2_all - sum_touched sumF_c^2.  The touched list is built in aidx and compacted in place to
    // the active list.
    __device__ __forceinline__ double scan_touched(int &m, bool &need_hi) {
        const int W = ldp >> 5;
        int nt = 0;
#pragma unroll 1
        for (int w0 = 0; w0 < W; w0 += 32) {
            const int w = w0 + lane;
            unsigned bits = (w < W) ? tmask[w] : 0u;
            const int pc = __popc(bits);
            int incl = pc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            int p = nt + incl - pc;
            while (bits) {
                aidx[p++] = (unsigned short)(32 * w + __ffs(bits) - 1);
                bits &= bits - 1u;
            }
            nt += __shfl_sync(0xffffffffu, incl, 31);
        }
        __syncwarp();
        double G2 = 0.0, SF2 = 0.0;
        bool hi_lane = false;
        m = 0;
        const double max_f = a->max_f;
#pragma unroll 1
        for (int t0 = 0; t0 < nt; t0 += 32) {
            const int t = t0 + lane;
            const bool ok = t < nt;
            const int c = ok ? (int)aidx[t] : 0;
            double f = 0.0, g = 0.0;
            if (ok) {
                const double sf = s_sumF[c];
                f = fu_d[c];
                g = (g_d[c] - sf) + f;
                g_d[c] = g;
                G2 = fma(g, g, G2);
                SF2 = fma(sf, sf, SF2);
            }
            const bool act = ok && (f > 0.0 || g > 0.0);
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            __syncwarp();                                 // this round's reads are done; the writes land at or below them
            if (act) {
                aidx[m + __popc(bal & lt_mask)] = (unsigned short)c;
                hi_lane |= (f + g > max_f);
            }
            m += __popc(bal);
        }
        G2 = warp_sum(G2);
        SF2 = warp_sum(SF2);
        need_hi = __any_sync(0xffffffffu, hi_lane);
        __syncwarp();
        return (S2_all - SF2) + G2;
    }
    // Fold-in: the components set in tmask, ascending, into `list` (once per node); returns their number.
    __device__ __forceinline__ int list_touched(unsigned short *list) {
        const int W = ldp >> 5;
        int nt = 0;
#pragma unroll 1
        for (int w0 = 0; w0 < W; w0 += 32) {
            const int w = w0 + lane;
            unsigned bits = (w < W) ? tmask[w] : 0u;
            const int pc = __popc(bits);
            int incl = pc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            int p = nt + incl - pc;
            while (bits) {
                list[p++] = (unsigned short)(32 * w + __ffs(bits) - 1);
                bits &= bits - 1u;
            }
            nt += __shfl_sync(0xffffffffu, incl, 31);
        }
        __syncwarp();
        return nt;
    }
    // Fold-in: scan_touched over the nt components of `list`, which is kept, with sumF' = sumF + f in the gradient.
    // (The step keeps its own fused scan_touched: written as these two parts, its wide kernels compile to different
    // instructions.)
    __device__ __forceinline__ double scan_list(const unsigned short *list, int nt, int &m, bool &need_hi) {
        double G2 = 0.0, SF2 = 0.0;
        bool hi_lane = false;
        m = 0;
        const double max_f = a->max_f;
#pragma unroll 1
        for (int t0 = 0; t0 < nt; t0 += 32) {
            const int t = t0 + lane;
            const bool ok = t < nt;
            const int c = ok ? (int)list[t] : 0;
            double f = 0.0, g = 0.0;
            if (ok) {
                const double sf = __ldg(s_sumF + c);
                f = fu_d[c];
                g = (g_d[c] - (sf + f)) + f;
                g_d[c] = g;
                G2 = fma(g, g, G2);
                SF2 = fma(sf, sf, SF2);
            }
            const bool act = ok && (f > 0.0 || g > 0.0);
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            if (act) {
                aidx[m + __popc(bal & lt_mask)] = (unsigned short)c;
                hi_lane |= (f + g > max_f);
            }
            m += __popc(bal);
        }
        G2 = warp_sum(G2);
        SF2 = warp_sum(SF2);
        need_hi = __any_sync(0xffffffffu, hi_lane);
        __syncwarp();
        return (S2_all - SF2) + G2;
    }
    // Wide rows: g_d of the touched components back to zero (when it was written) and the bitmask cleared.
    __device__ __forceinline__ void clear_touched(bool clear_g) {
        const int W = ldp >> 5;
#pragma unroll 1
        for (int w = lane; w < W; w += 32) {
            unsigned bits = tmask[w];
            if (bits == 0u) continue;
            if (clear_g)
                while (bits) {
                    g_d[32 * w + __ffs(bits) - 1] = 0.0;
                    bits &= bits - 1u;
                }
            tmask[w] = 0u;
        }
        __syncwarp();
    }
    // The staged entries of `ne` rows shrink, in place, to those on ACTIVE components (fu > 0 or grad > 0): only
    // they can contribute to a candidate's dot.  Order inside a row is kept, poff is rewritten.
    __device__ __forceinline__ void compact_active(int ne) {
        const int T = poff[ne];
        int total = 0;
#pragma unroll 1
        for (int base = 0; base < T; base += 32) {
            const int j = base + lane;
            const bool in = j < T;
            const int c = in ? (int)ent_idx[j] : 0;
            const double v = in ? ent_val[j] : 0.0;
            const bool act = in && (fu_d[c] > 0.0 || g_d[c] > 0.0);
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            if (lane == 0) { cbal[base >> 5] = bal; ccum[base >> 5] = (unsigned short)total; }
            __syncwarp();                       // this block's reads are done; writes land at or below them
            if (act) {
                const int p = total + __popc(bal & lt_mask);
                ent_idx[p] = (unsigned short)c;
                ent_val[p] = v;
            }
            total += __popc(bal);
        }
        __syncwarp();
        int newp = 0;
        if (lane < ne) {
            const int p = poff[lane];
            newp = (p >= T) ? total : (int)ccum[p >> 5] + __popc(cbal[p >> 5] & ((1u << (p & 31)) - 1u));
        }
        __syncwarp();
        if (lane < ne) poff[lane] = (unsigned short)newp;
        if (lane == 0) poff[ne] = (unsigned short)total;
        __syncwarp();
    }
    // Line search over the edges [eb, ee): lane (j, h) returns the sum over its edges of the clamped edge term
    // for candidate step s; `staged` rows of a single chunk may still be in the buffer from PRE.
    __device__ __forceinline__ double ls_range(const int32_t *colbase, int eb, int ee, double s, bool need_hi, int staged) {
        const int h = lane >> 4;
        const double max_f = a->max_f;
        double sumterms = 0.0;
#pragma unroll 1
        for (int cb = eb; cb < ee;) {
            const int ne = (staged > 0) ? staged : stage(colbase + cb, min(32, ee - cb));
            compact_active(ne);
#pragma unroll 1
            for (int e2 = 0; e2 < ne; e2 += 4) {
                const int eA = e2 + h, eB = e2 + 2 + h;
                const bool vA = eA < ne, vB = eB < ne;
                const int iA = vA ? (int)poff[eA] : 0, nA = vA ? (int)poff[eA + 1] - iA : 0;
                const int iB = vB ? (int)poff[eB] : 0, nB = vB ? (int)poff[eB + 1] - iB : 0;
                const int nmax = max(nA, nB);
                double DA = 0.0, DB = 0.0;
#pragma unroll 1
                for (int k = 0; k < nmax; ++k) {
                    const bool ka = k < nA, kb = k < nB;
                    const int ca = ka ? (int)ent_idx[iA + k] : 0, cb2 = kb ? (int)ent_idx[iB + k] : 0;
                    const double pa = ka ? ent_val[iA + k] : 0.0, pb = kb ? ent_val[iB + k] : 0.0;
                    const double fa = fu_d[ca], ga = g_d[ca], fb = fu_d[cb2], gb = g_d[cb2];
                    if (need_hi) {
                        DA = fma(clamp_step0(fa, s, ga, max_f), pa, DA);
                        DB = fma(clamp_step0(fb, s, gb, max_f), pb, DB);
                    } else {
                        DA = fma(clamp_step0_lo(fa, s, ga), pa, DA);
                        DB = fma(clamp_step0_lo(fb, s, gb), pb, DB);
                    }
                }
                double tA, tB;
                edge_term2(DA, DB, ec, tA, tB);
                sumterms += vA ? tA : 0.0;
                sumterms += vB ? tB : 0.0;
            }
            __syncwarp();
            cb += ne;
        }
        return sumterms;
    }
    // Armijo decision for the 16 candidates tg .. tg+15 given each lane's edge-term sum (already summed over h).
    __device__ __forceinline__ int decide(int tg, double s, bool jok, double sumterms, int m, bool need_hi, double llh_u, double G2, unsigned surv = 0xffffu) {
        const int h = lane >> 4;
        const double max_f = a->max_f;
        // - newfu.sfT + newfu.newfu with sfT = (sumF - fu) + newfu   (:176,:180; fold-in: sumF' = sumF + fu)
        double oa = 0.0, ob = 0.0;
#pragma unroll 1
        for (int t = h; t < m; t += 2) {
            const int c = aidx[t];
            const double f = fu_d[c], g = g_d[c];
            const double nf = need_hi ? clamp_step0(f, s, g, max_f) : clamp_step0_lo(f, s, g);
            const double sf = ((kFold ? __ldg(s_sumF + c) + f : s_sumF[c]) - f) + nf;
            oa = fma(nf, sf, oa);
            ob = fma(nf, nf, ob);
        }
        oa += __shfl_xor_sync(0xffffffffu, oa, 16);
        ob += __shfl_xor_sync(0xffffffffu, ob, 16);
        const double result = (sumterms - oa) + ob;
        const double rhs = llh_u + (a->alpha * s) * G2;
        const unsigned pass = __ballot_sync(0xffffffffu, jok && (result >= rhs)) & 0xffffu & surv;
        return pass ? tg + __ffs(pass) - 1 : -1;          // lowest j == largest step (:182 max)
    }
    // SWAP (:183-190): the accepted candidate's non-zeros (or the old row) go to the output pool(s), followed by
    // the delta block (old - new, :191-192) of an accepted node.
    template <bool kPush>
    __device__ __forceinline__ void swap_row(int64_t u, int jstar, int m, int cu, const double *uval, const unsigned short *uidx) {
        const double max_f = a->max_f;
        int cnt_new = 0, nd = 0;
        double s = 0.0;
        __syncwarp();                     // the entry buffers are reused: every lane is done reading the staged rows (PRE, bounds, LS)
        if (jstar >= 0) {
            s = s_steps[jstar];
#pragma unroll 1
            for (int t0 = 0; t0 < m; t0 += 32) {
                const int t = t0 + lane;
                const bool ok = t < m;
                const int c = ok ? (int)aidx[t] : 0;
                const double f = fu_d[c], g = g_d[c];
                const double nr = clamp_step(f, s, g, a->min_f, max_f);
                const bool nz = ok && (nr != 0.0);
                const unsigned bal = __ballot_sync(0xffffffffu, nz);
                if (nz) {
                    const int p = cnt_new + __popc(bal & lt_mask);
                    ent_val[p] = nr;
                    ent_idx[p] = (unsigned short)c;
                }
                cnt_new += __popc(bal);
                nd += __popc(__ballot_sync(0xffffffffu, ok && (f != nr)));
            }
        } else {
#pragma unroll 1
            for (int i = lane; i < cu; i += 32) {
                ent_val[i] = __ldg(uval + i);
                ent_idx[i] = __ldg(uidx + i);
            }
            cnt_new = cu;
        }
        __syncwarp();
        const unsigned long long wrow = sp_words((uint32_t)cnt_new);
        const unsigned long long words = wrow + (nd > 0 ? sp_words((uint32_t)nd) : 0ull);
        unsigned long long rel = 0;
        if (lane == 0 && words > 0) rel = atomicAdd(sp->pool_top, words);
        rel = __shfl_sync(0xffffffffu, rel, 0);
        if (rel + words > sp->pool_cap8) {
            if (lane == 0) { *sp->overflow = 1; sp->hdr_out[u] = sp_pack(0, 0); sp->dcnt[u] = 0; }
            return;
        }
        const unsigned long long off = sp->region_base8 + rel;
        const uint64_t hnew = sp_pack(off, (uint32_t)cnt_new);
        double *ov = sp->pool_out + off;
        unsigned short *oi = sp_idx(ov, (uint32_t)cnt_new);
#pragma unroll 1
        for (int i = lane; i < cnt_new; i += 32) {
            ov[i] = ent_val[i];
            oi[i] = ent_idx[i];
        }
        if (lane == 0) { sp->hdr_out[u] = hnew; sp->dcnt[u] = (unsigned short)nd; }
        if (kPush) {
#pragma unroll 1
            for (int pr = 0; pr < sp->n_peers; ++pr) {
                double *pv = sp->peer_pool[pr] + off;
                unsigned short *pi = sp_idx(pv, (uint32_t)cnt_new);
#pragma unroll 1
                for (int i = lane; i < cnt_new; i += 32) {
                    pv[i] = ent_val[i];
                    pi[i] = ent_idx[i];
                }
                if (lane == 0) sp->peer_hdr[pr][u] = hnew;
            }
        }
        if (nd > 0) {                                    // delta block (local only: the owner reduces it)
            double *dv = ov + wrow;
            unsigned short *di = sp_idx(dv, (uint32_t)nd);
            int q = 0;
#pragma unroll 1
            for (int t0 = 0; t0 < m; t0 += 32) {
                const int t = t0 + lane;
                const bool ok = t < m;
                const int c = ok ? (int)aidx[t] : 0;
                const double f = fu_d[c], g = g_d[c];
                const double nr = clamp_step(f, s, g, a->min_f, max_f);
                const bool ch = ok && (f != nr);
                const unsigned bal = __ballot_sync(0xffffffffu, ch);
                if (ch) {
                    const int p = q + __popc(bal & lt_mask);
                    dv[p] = f - nr;
                    di[p] = (unsigned short)c;
                }
                q += __popc(bal);
            }
        }
    }

    // own row -> fu_d; returns fu.sumF and fu.fu through the references
    __device__ __forceinline__ void scatter_own(int cu, const double *uval, const unsigned short *uidx, double &fusf, double &fufu) {
        fusf = 0.0;
        fufu = 0.0;
#pragma unroll 1
        for (int i = lane; i < cu; i += 32) {
            const double v = __ldg(uval + i);
            const int c = __ldg(uidx + i);
            fu_d[c] = v;
            if constexpr (kWide) touch(c);
            fusf = fma(v, s_sumF[c], fusf);
            fufu = fma(v, v, fufu);
        }
        fusf = warp_sum(fusf);
        fufu = warp_sum(fufu);
        __syncwarp();
    }

    // Line search by bounds for a node on the general path (gradient in g_d, m active components in aidx): the mask of
    // the candidates 0 .. 15 that the bound cannot exclude.  `staged`: rows of the node's only chunk that are still
    // staged from PRE (0: the chunks are staged again).  Next to x_lo the violation is taken at its cap (w_lo - 1) x.
    __device__ __forceinline__ unsigned bound_mask(const int32_t *colp, int deg, int m, double G2node, double llh_u, double fusf, double fufu, int staged) {
        const int nsteps = a->nsteps;
        const int j = lane & 15, h = lane >> 4;
        // active components: |g|^2 split by sign, R3, G1, max g, sum sumF^2
        float g2n = 0.0f, g2p = 0.0f, r3 = 0.0f, g1p = 0.0f, gmx = 0.0f, sf2 = 0.0f;
#pragma unroll 1
        for (int t = lane; t < m; t += 32) {
            const int c = aidx[t];
            const double f = fu_d[c], g = g_d[c];
            const float ga = __double2float_ru(fabs(g)), ff = __double2float_ru(f), sff = __double2float_ru(fabs(s_sumF[c]));
            r3 = fmaf(ff, fmaf(2.0f, ga, sff) + 3.0f * ff, r3);
            sf2 = fmaf(sff, sff, sf2);
            if (g > 0.0) {
                g2p = fmaf(ga, ga, g2p);
                g1p += ga;
                gmx = fmaxf(gmx, ga);
            } else {
                g2n = fmaf(ga, ga, g2n);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            g2n += __shfl_xor_sync(0xffffffffu, g2n, o);
            g2p += __shfl_xor_sync(0xffffffffu, g2p, o);
            r3 += __shfl_xor_sync(0xffffffffu, r3, o);
            g1p += __shfl_xor_sync(0xffffffffu, g1p, o);
            sf2 += __shfl_xor_sync(0xffffffffu, sf2, o);
            gmx = fmaxf(gmx, __shfl_xor_sync(0xffffffffu, gmx, o));
        }
        // edges, chunk by chunk: x, Dp, En per edge (lane = edge), then every candidate lane (j, h) collects its share
        const float lns = (j < nsteps) ? s_lns[j] : -3.0e38f;
        const float cap_f = sp->pr_cap;
        double sDp = 0.0, sEn = 0.0;
        float sV = 0.0f, Hs = 0.0f;
#pragma unroll 1
        for (int cb = 0; cb < deg;) {
            const int ne = (staged > 0) ? staged : stage_chunk(colp + cb, min(32, deg - cb));
            double x = 0.0, Dp = 0.0, En = 0.0;
            if (lane < ne) {
                const int end = poff[lane + 1];
#pragma unroll 1
                for (int i = poff[lane]; i < end; ++i) {
                    const int c = ent_idx[i];
                    const double v = ent_val[i], f = fu_d[c], g = g_d[c];
                    x = fma(v, f, x);
                    Dp = fma(v, g > 0.0 ? g : 0.0, Dp);
                    En = fma(v, (g < 0.0 && f > 0.0) ? g : 0.0, En);
                }
            }
            float lnthr = 3.0e38f, Lp = 0.0f, violf = 0.0f;
            if (lane < ne) {
                if (x <= ec.x_lo) {
                    if (Dp > 0.0) ls_code_flat(__double2float_ru(x), Dp, sp->pr_xlo, sp->pr_kinv, lnthr, Lp);
                } else {
                    if (x >= ec.x_hi) violf = __double2float_ru((ec.w_hi - 1.0) * (x - ec.x_hi)) * 1.000001f;
                    else if (x < 4.0 * ec.x_lo && En < 0.0)             // (beyond e * x_lo the tangent never fails)
                        ls_code_near(x, ec.x_lo, En, __double2float_ru((ec.w_lo - 1.0) * x) * 1.000001f, lnthr, Lp);
                    Dp = 0.0;
                    En = 0.0;
                }
            }
            sDp += Dp;
            sEn += En;
            sV += violf;
#pragma unroll 1
            for (int r0 = 0; r0 < ne; r0 += 2) {                     // (the two half-warps take alternate edges)
                const int r = r0 + h;
                const float tx = __shfl_sync(0xffffffffu, lnthr, r & 31), ty = __shfl_sync(0xffffffffu, Lp, r & 31);
                if (r < ne) Hs += ls_edge_share(lns, tx, ty, cap_f);
            }
            cb += ne;
        }
        sDp = warp_sum(sDp);
        sEn = warp_sum(sEn);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sV += __shfl_xor_sync(0xffffffffu, sV, o);
        Hs += __shfl_xor_sync(0xffffffffu, Hs, 16);
        LsBound B;
        const double m_lo = ec.w_lo - 1.0;
        B.Qn = (double)(g2n * 1.000001f) - m_lo * sEn;
        B.Qp = (double)(g2p * 1.000001f);
        B.Mp = m_lo * sDp;
        B.G1 = (double)(__double2float_ru(a->max_f) * g1p * 1.0001f);
        B.R3 = (double)(r3 * 1.0001f);
        const float fuf = __double2float_ru(fabs(fusf)), fff = __double2float_ru(fufu), g2f = __double2float_ru(G2node);
        const float r4 = fmaf(2.0f, g2f, sqrtf(g2f) * sqrtf(fmaf(2.0f, sf2, 18.0f * fff)) * 1.0001f);
        const float base = fmaf(2.0f * cap_f, (float)deg, __double2float_ru(fabs(llh_u))) + 2.0f * (fuf + fff) + r3;
        const float nops = 2.3e-16f * (float)(4 * deg + 3 * m + 16);
        B.c0 = fmaf(nops, base, sV) * 1.0001f;
        B.c1 = nops * fmaf(2.0f, r4, __double2float_ru(sDp)) * 1.0001f;
        B.kap0 = (gmx > 0.0f) ? __fdividef(fmaxf(__double2float_rd(a->max_f) - sqrtf(fff) * 1.000001f, 0.0f), gmx) * 0.9999f : 3.0e38f;
        const bool keep = (j < nsteps) && !B.cannot_pass(s_steps[j < nsteps ? j : 0], Hs, a->alpha, G2node);
        return __ballot_sync(0xffffffffu, keep) & 0xffffu;
    }

    // One node, start to finish.  colp: the node's neighbour list (ids in the low 28 bits when it comes from tcol).
    template <bool kPush>
    __device__ BIGCLAM_GEN_INLINE void node(int64_t u, int deg, const int32_t *colp) {
        const uint64_t hu = __ldg(sp->hdr_in + u);
        const int cu = (int)sp_cnt(hu);
        const double *uval = sp->pool_in + sp_off8(hu);
        const unsigned short *uidx = sp_idx(uval, (uint32_t)cu);
        double fusf, fufu;
        scatter_own(cu, uval, uidx, fusf, fufu);
        const bool in_uset = (a->node_mask == nullptr) || (a->node_mask[u] != 0);
        const bool want_ls = a->do_linesearch && in_uset && deg > 0;
        const int nsteps = a->nsteps;
        const int j16 = lane & 15;

        // ---------------- PRE (:157-169) ----------------
        int nchunks, ne_last;
        const double S1 = warp_sum(pre_range(colp, 0, deg, want_ls, nchunks, ne_last));
        const double llh_u = (S1 - fusf) + fufu;
        int jstar = -1, m = 0;
        if (want_ls) {
            bool need_hi;
            double G2;
            if constexpr (kWide) G2 = scan_touched(m, need_hi);
            else G2 = scan_gradient(m, need_hi);
            // ---------------- LS (:172-182): only if the bounds leave a candidate that can pass ----------------
            unsigned surv = 0xffffu;
            if constexpr (!kWide)           // (wide rows: no bounds on the general path)
                if (BIGCLAM_GEN_BOUNDS && sp->ls_prune > 1 && nsteps <= 16) surv = bound_mask(colp, deg, m, G2, llh_u, fusf, fufu, nchunks == 1 ? ne_last : 0);
            if (sp->stats != nullptr && lane == 0) {
                atomicAdd(sp->stats + 3, 1u);
                if (surv != 0u) atomicAdd(sp->stats + 2, 1u);
            }
#pragma unroll 1
            for (int tg = 0; tg < nsteps && jstar < 0 && surv != 0u; tg += 16) {
                const int j = tg + j16;
                const bool jok = j < nsteps;
                const double s = s_steps[jok ? j : 0];
                // a node whose neighbours fitted one chunk still has them staged from PRE
                double sumterms = ls_range(colp, 0, deg, s, need_hi, (nchunks == 1 && tg == 0) ? ne_last : 0);
                sumterms += __shfl_xor_sync(0xffffffffu, sumterms, 16);
                jstar = decide(tg, s, jok, sumterms, m, need_hi, llh_u, G2, surv);
            }
        }
        if (lane == 0) sp->node_llh[u] = llh_u;
        if (a->do_linesearch) {
            swap_row<kPush>(u, jstar, m, cu, uval, uidx);
            if (lane == 0) sp->accepted[u] = (int8_t)jstar;
        }
        // ---- leave the dense vectors at zero for the next node ----
        __syncwarp();
#pragma unroll 1
        for (int i = lane; i < cu; i += 32) fu_d[__ldg(uidx + i)] = 0.0;
        if constexpr (kWide) {
            clear_touched(want_ls);
        } else {
            if (want_ls)
#pragma unroll 1
                for (int c = lane; c < ldp; c += 32) g_d[c] = 0.0;
        }
        __syncwarp();
    }

    // One item of a split hub (see above).
    template <bool kPush>
    __device__ BIGCLAM_GEN_INLINE void hub_item(const HubItem item) {
        const NodeMeta nm = a->meta[item.hub];
        const int64_t u = nm.u, e0 = nm.e0;
        const int deg = nm.deg;
        const size_t hstride = sp_hub_stride(ld);
        double *scr0 = a->hub_scratch + (size_t)item.mslot * hstride;            // mslot: first scratch slot of the hub
        unsigned int *cnt = a->hub_counters + 2 * (size_t)item.hub;
        const int sb = item.slice * item.seg, se = min(deg, sb + item.seg);
        const uint64_t hu = __ldg(sp->hdr_in + u);
        const int cu = (int)sp_cnt(hu);
        const double *uval = sp->pool_in + sp_off8(hu);
        const unsigned short *uidx = sp_idx(uval, (uint32_t)cu);
        double fusf, fufu;
        scatter_own(cu, uval, uidx, fusf, fufu);
        const bool in_uset = (a->node_mask == nullptr) || (a->node_mask[u] != 0);
        const bool want_ls = a->do_linesearch && in_uset;
        const int j16 = lane & 15;
        const int32_t *colp = a->col + e0;
        double *tot = scr0 + (size_t)item.nslices * hstride;                      // the hub's combined slot
        if (item.phase == 1) {
            int nch, nel;
            const double S1 = warp_sum(pre_range(colp, sb, se, want_ls, nch, nel));
            double *scr = scr0 + (size_t)item.slice * hstride;
            if (want_ls) {
#pragma unroll 1
                for (int c = lane; c < ld; c += 32) { scr[c] = g_d[c]; g_d[c] = 0.0; }
            }
            if (lane == 0) scr[ld] = S1;
            __threadfence();
            __syncwarp();
            unsigned int old = 0;
            if (lane == 0) old = atomicAdd(cnt, 1u);
            old = __shfl_sync(0xffffffffu, old, 0);
            if (old == (unsigned int)item.nslices - 1u) {
                // the last segment to arrive adds the slots up, in slot order: whichever warp does it, the sums
                // are the same bits
                __threadfence();
                if (want_ls) {
#pragma unroll 1
                    for (int c = lane; c < ld; c += 32) {
                        double v = 0.0;
#pragma unroll 1
                        for (int sl = 0; sl < item.nslices; ++sl) v += __ldcg(scr0 + (size_t)sl * hstride + c);
                        tot[c] = v;
                    }
                }
                if (lane == 0) {
                    double v = 0.0;
#pragma unroll 1
                    for (int sl = 0; sl < item.nslices; ++sl) v += __ldcg(scr0 + (size_t)sl * hstride + ld);
                    tot[ld] = v;
                }
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(cnt, 1u);
            }
        } else {
            if (lane == 0) {
                const unsigned int *c = cnt + (item.phase == 2 ? 0 : 1);
                const unsigned int target = (unsigned int)item.nslices + (item.phase == 2 ? 1u : 0u);
                while (*reinterpret_cast<const volatile unsigned int *>(c) < target) __nanosleep(200);
                __threadfence();
            }
            __syncwarp();
            const double llh_u = (__ldcg(tot + ld) - fusf) + fufu;
            int m = 0, jstar = -1;
            bool need_hi = false;
            double G2 = 0.0;
            if (want_ls) {
#pragma unroll 1
                for (int c = lane; c < ldp; c += 32) g_d[c] = (c < ld) ? __ldcg(tot + c) : 0.0;
                __syncwarp();
                G2 = scan_gradient(m, need_hi);
            }
            const int nsteps = a->nsteps;
            const double s = s_steps[j16 < nsteps ? j16 : 0];       // hubs are only split when nsteps <= 16
            if (item.phase == 2) {
                if (want_ls) {
                    double st = ls_range(colp, sb, se, s, need_hi, 0);
                    st += __shfl_xor_sync(0xffffffffu, st, 16);
                    if (lane < 16) scr0[(size_t)item.slice * hstride + ld + 1 + lane] = st;
                }
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(cnt + 1, 1u);
            } else {
                if (want_ls) {
                    double st = 0.0;
#pragma unroll 1
                    for (int sl = 0; sl < item.nslices; ++sl) st += __ldcg(scr0 + (size_t)sl * hstride + ld + 1 + j16);
                    jstar = decide(0, s, j16 < nsteps, st, m, need_hi, llh_u, G2);
                }
                if (lane == 0) sp->node_llh[u] = llh_u;
                if (a->do_linesearch) {
                    swap_row<kPush>(u, jstar, m, cu, uval, uidx);
                    if (lane == 0) sp->accepted[u] = (int8_t)jstar;
                }
            }
            __syncwarp();
            if (want_ls)
#pragma unroll 1
                for (int c = lane; c < ldp; c += 32) g_d[c] = 0.0;
        }
        __syncwarp();
#pragma unroll 1
        for (int i = lane; i < cu; i += 32) fu_d[__ldg(uidx + i)] = 0.0;
        if constexpr (kWide) {            // (the hub phases loop over all components: only the bitmask is left to clear)
#pragma unroll 1
            for (int w = lane; w < (ldp >> 5); w += 32) tmask[w] = 0u;
        }
        __syncwarp();
    }
};

// Dense n x ld rows -> sparse rows (one warp per row; non-zeros in ascending component order).
__global__ void dense_to_sparse_kernel(const double *F, int64_t n, int ld, uint64_t *hdr, double *pool,
                                       unsigned long long *pool_top, uint64_t pool_cap8, int32_t *overflow) {
    const int lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= n) return;
    const unsigned lt_mask = (1u << lane) - 1u;
    const double *row = F + (size_t)u * ld;
    int cnt = 0;
    for (int c0 = 0; c0 < ld; c0 += 32) {
        const int c = c0 + lane;
        cnt += __popc(__ballot_sync(0xffffffffu, c < ld && row[c] != 0.0));
    }
    const unsigned long long words = sp_words((uint32_t)cnt);
    unsigned long long off = 0;
    if (lane == 0 && cnt > 0) off = atomicAdd(pool_top, words);
    off = __shfl_sync(0xffffffffu, off, 0);
    if (off + words > pool_cap8) {
        if (lane == 0) { *overflow = 1; hdr[u] = sp_pack(0, 0); }
        return;
    }
    double *ov = pool + off;
    unsigned short *oi = sp_idx(ov, (uint32_t)cnt);
    int p = 0;
    for (int c0 = 0; c0 < ld; c0 += 32) {
        const int c = c0 + lane;
        const double v = (c < ld) ? row[c] : 0.0;
        const unsigned bal = __ballot_sync(0xffffffffu, v != 0.0);
        if (v != 0.0) {
            const int q = p + __popc(bal & lt_mask);
            ov[q] = v;
            oi[q] = (unsigned short)c;
        }
        p += __popc(bal);
    }
    if (lane == 0) hdr[u] = sp_pack(off, (uint32_t)cnt);
}

// Host side of the layout: rows given as CSR (indptr, ascending-or-not indices, values; explicit zeros are dropped)
// -> header + pool image, and back.  Used by bigclam_set_F_csr / bigclam_get_F_csr (and by the emulation tests).
// Returns the number of 8-byte words used, or -1 for an index outside [0, k) / a row longer than ld.
inline int64_t sp_host_pack(int64_t n, int32_t k, int32_t ld, const int64_t *indptr, const int32_t *indices, const double *values,
                            uint64_t *hdr, double *pool, uint64_t pool_cap8, double *colsum /* k, optional */) {
    uint64_t top = 0;
    if (colsum != nullptr)
        for (int32_t c = 0; c < k; ++c) colsum[c] = 0.0;
    for (int64_t u = 0; u < n; ++u) {
        uint32_t cnt = 0;
        for (int64_t i = indptr[u]; i < indptr[u + 1]; ++i) {
            if (indices[i] < 0 || indices[i] >= k) return -1;
            if (values[i] != 0.0) ++cnt;
        }
        if (cnt > (uint32_t)ld) return -1;
        const uint64_t words = sp_words(cnt);
        if (top + words > pool_cap8) return -2;
        double *ov = pool + top;
        unsigned short *oi = sp_idx(ov, cnt);
        for (uint64_t z = 0; z < words; ++z) ov[z] = 0.0;
        uint32_t q = 0;
        for (int64_t i = indptr[u]; i < indptr[u + 1]; ++i) {
            if (values[i] == 0.0) continue;
            // insertion keeps the indices ascending (rows arrive sorted in practice: one comparison per entry)
            uint32_t p = q;
            while (p > 0 && oi[p - 1] > (unsigned short)indices[i]) { oi[p] = oi[p - 1]; ov[p] = ov[p - 1]; --p; }
            oi[p] = (unsigned short)indices[i];
            ov[p] = values[i];
            ++q;
            if (colsum != nullptr) colsum[indices[i]] += values[i];
        }
        hdr[u] = sp_pack(cnt ? top : 0, cnt);
        top += words;
    }
    return (int64_t)top;
}

inline int64_t sp_host_nnz(int64_t n, const uint64_t *hdr) {
    int64_t t = 0;
    for (int64_t u = 0; u < n; ++u) t += sp_cnt(hdr[u]);
    return t;
}

inline void sp_host_unpack(int64_t n, const uint64_t *hdr, const double *pool, int64_t *indptr, int32_t *indices, double *values) {
    int64_t t = 0;
    for (int64_t u = 0; u < n; ++u) {
        indptr[u] = t;
        const uint32_t cnt = sp_cnt(hdr[u]);
        const double *ov = pool + sp_off8(hdr[u]);
        const unsigned short *oi = sp_idx(ov, cnt);
        for (uint32_t i = 0; i < cnt; ++i) { indices[t] = oi[i]; values[t] = ov[i]; ++t; }
    }
    indptr[n] = t;
}

// Sparse rows -> dense n x ld (rows are zeroed here, no separate memset).
__global__ void sparse_to_dense_kernel(const uint64_t *hdr, const double *pool, int64_t n, int ld, double *F) {
    const int lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= n) return;
    double *row = F + (size_t)u * ld;
    for (int c = lane; c < ld; c += 32) row[c] = 0.0;
    __syncwarp();
    const uint64_t h = hdr[u];
    const int cnt = (int)sp_cnt(h);
    const double *vals = pool + sp_off8(h);
    const unsigned short *idx = sp_idx(vals, (uint32_t)cnt);
    for (int i = lane; i < cnt; i += 32) row[idx[i]] = vals[i];
}

// ---------------------------------------------------------------------------------------------------------------
// Edge probabilities and link recommendations from the current F (read only; bigclam_pair_affinity / bigclam_recommend).
//
// The affinity x_uv is the sum of F_uc F_vc over the components c that are non-zero in BOTH rows, folded left in
// ascending c with every product and every sum rounded on its own: the same bits for sparse and dense rows, for (u, v)
// and (v, u), and for a NumPy restatement.  p_uv = 1 - clamp(exp(-x), MIN_P_, MAX_P_), the clamp of
// bigclam4-7.scala:166, so log(p_uv) + x_uv is the per-edge term of the LLH (:218).
struct PairConst {                 // the clamp of p, with the step kernel's exact shortcuts (fill_args)
    double min_p, max_p, x_lo, x_hi;
};

__device__ __forceinline__ double pair_x(const RowSrc &s, int64_t u, int64_t v) {
    double x = 0.0;
    if (s.hdr != nullptr) {        // merge of the two ascending index lists
        const uint64_t hu = s.hdr[u], hv = s.hdr[v];
        const uint32_t cu = sp_cnt(hu), cv = sp_cnt(hv);
        const double *au = s.pool + sp_off8(hu), *av = s.pool + sp_off8(hv);
        const unsigned short *iu = sp_idx(au, cu), *iv = sp_idx(av, cv);
        uint32_t i = 0, j = 0;
        while (i < cu && j < cv) {
            const unsigned short a = iu[i], b = iv[j];
            if (a == b) { x = __dadd_rn(x, __dmul_rn(au[i], av[j])); ++i; ++j; }
            else if (a < b) ++i;
            else ++j;
        }
        return x;
    }
    const double *fu = s.F + (size_t)u * s.ld, *fv = s.F + (size_t)v * s.ld;
    for (int c = 0; c < s.k; ++c) {
        const double a = fu[c], b = fv[c];
        if (a != 0.0 && b != 0.0) x = __dadd_rn(x, __dmul_rn(a, b));
    }
    return x;
}

__device__ __forceinline__ double pair_p(double x, const PairConst &c) {
    double e;
    if (x <= c.x_lo) e = c.max_p;
    else if (x >= c.x_hi) e = c.min_p;
    else e = fmin(fmax(exp_neg(x), c.min_p), c.max_p);      // (next to the shortcuts the clamp may still bite)
    return 1.0 - e;
}

// One lane per pair.
__global__ void pair_affinity_kernel(RowSrc s, PairConst pc, const int32_t *__restrict__ u, const int32_t *__restrict__ v,
                                     int64_t count, double *__restrict__ x_out, double *__restrict__ p_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const double x = pair_x(s, u[i], v[i]);
    x_out[i] = x;
    if (p_out != nullptr) p_out[i] = pair_p(x, pc);
}

// Recommendations, one warp per query node u of a batch.  The two-hop list of u is, in one segment of a key scratch:
// 2u and 2w for every w in N(u) (entries that exclude a node), then 2v + 1 for every v in N(w), w in N(u) (candidates).
// Sorted ascending, the first key of every run of equal v >> 1 tells whether v is excluded: repeated and unsorted
// neighbour lists need no preparation.
//   count  entries of u's segment: 1 + deg(u) + sum_{w in N(u)} deg(w)
__global__ void rec_count_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                 const int32_t *__restrict__ q, int64_t nq, int64_t *__restrict__ cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= nq) return;                                     // (warp-uniform)
    const int64_t u = q[i], e0 = rowptr[u], e1 = rowptr[u + 1];
    long long t = 0;
    for (int64_t e = e0 + lane; e < e1; e += 32) {
        const int32_t w = col[e];
        t += rowptr[w + 1] - rowptr[w];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) cnt[i] = 1 + (e1 - e0) + t;
}

//   fill   the segment at off[i] (offsets relative to the batch's scratch)
__global__ void rec_fill_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                const int32_t *__restrict__ q, int64_t nq, const int64_t *__restrict__ off,
                                uint32_t *__restrict__ keys) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= nq) return;
    const int64_t u = q[i], e0 = rowptr[u], e1 = rowptr[u + 1];
    uint32_t *seg = keys + off[i];
    if (lane == 0) seg[0] = 2u * (uint32_t)u;
    for (int64_t e = e0 + lane; e < e1; e += 32) seg[1 + (e - e0)] = 2u * (uint32_t)col[e];
    int64_t pos = 1 + (e1 - e0);
    for (int64_t e = e0; e < e1; ++e) {
        const int32_t w = col[e];
        const int64_t f0 = rowptr[w], f1 = rowptr[w + 1];
        for (int64_t f = f0 + lane; f < f1; f += 32) seg[pos + (f - f0)] = 2u * (uint32_t)col[f] + 1u;
        pos += f1 - f0;
    }
}

// (x, v) ranks before (y, w): larger affinity first, then the smaller node id
__device__ __forceinline__ bool rec_better(double x, int32_t v, double y, int32_t w) { return x > y || (x == y && v < w); }

// Sorts seg[0, L) ascending in place, by the whole warp: a bitonic network whose comparators all put the smaller key
// first, so the keys beyond the segment's end act as +inf and never move.  Ends with the warp in step.
__device__ __forceinline__ void warp_sort_u32(uint32_t *seg, int64_t L, int lane) {
    int lgp = 0;
    while (((int64_t)1 << lgp) < L) ++lgp;
    const int64_t npairs = ((int64_t)1 << lgp) >> 1;
    for (int lg = 1; lg <= lgp; ++lg) {
        const int64_t size = (int64_t)1 << lg, hmask = (size >> 1) - 1;
        for (int64_t t = lane; t < npairs; t += 32) {             // the flip: j <-> size - 1 - j inside a block of size
            const int64_t base = (t >> (lg - 1)) << lg, j = t & hmask;
            const int64_t lo = base + j, hi = base + size - 1 - j;
            if (hi < L) {
                const uint32_t a = seg[lo], c = seg[hi];
                if (a > c) { seg[lo] = c; seg[hi] = a; }
            }
        }
        __syncwarp();
        for (int ls = lg - 2; ls >= 0; --ls) {                    // half-cleaners: j <-> j + stride
            const int64_t stride = (int64_t)1 << ls;
            for (int64_t t = lane; t < npairs; t += 32) {
                const int64_t lo = ((t >> ls) << (ls + 1)) + (t & (stride - 1)), hi = lo + stride;
                if (hi < L) {
                    const uint32_t a = seg[lo], c = seg[hi];
                    if (a > c) { seg[lo] = c; seg[hi] = a; }
                }
            }
            __syncwarp();
        }
    }
}

//   rank   sort the segment (warp_sort_u32), then score every candidate that survives (pair_x) and keep the m best with
//          x > 0 in v_out / x_out (rows of m, padded with -1 / 0); found = how many were kept
__global__ void rec_rank_kernel(RowSrc s, const int32_t *__restrict__ q, int64_t nq, const int64_t *__restrict__ off,
                                uint32_t *__restrict__ keys, int32_t m, int32_t *__restrict__ v_out, double *__restrict__ x_out,
                                int32_t *__restrict__ found) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= nq) return;
    const int64_t u = q[i];
    uint32_t *seg = keys + off[i];
    const int64_t L = off[i + 1] - off[i];
    warp_sort_u32(seg, L, lane);
    int32_t *vo = v_out + (size_t)i * m;
    double *xo = x_out + (size_t)i * m;
    for (int t = lane; t < m; t += 32) { vo[t] = -1; xo[t] = 0.0; }
    __syncwarp();
    int kept = 0;                                            // (warp-uniform)
    double xw = 0.0;                                         // the last kept entry, once the list is full
    int32_t vw = 0;
    for (int64_t t0 = 0; t0 < L; t0 += 32) {
        const int64_t t = t0 + lane;
        const uint32_t key = (t < L) ? seg[t] : 0u;
        const bool cand = (t < L) && (key & 1u) && (t == 0 || (seg[t - 1] >> 1) != (key >> 1));
        const int32_t v = (int32_t)(key >> 1);
        const double x = cand ? pair_x(s, u, v) : 0.0;
        unsigned want = __ballot_sync(0xffffffffu, cand && x > 0.0 && (kept < m || rec_better(x, v, xw, vw)));
        while (want) {                                       // insertions in lane order, by lane 0
            const int l = __ffs(want) - 1;
            want &= want - 1u;
            const double xb = __shfl_sync(0xffffffffu, x, l);
            const int32_t vb = __shfl_sync(0xffffffffu, v, l);
            if (lane == 0 && (kept < m || rec_better(xb, vb, xo[m - 1], vo[m - 1]))) {
                int p = (kept < m) ? kept : m - 1;
                while (p > 0 && rec_better(xb, vb, xo[p - 1], vo[p - 1])) { xo[p] = xo[p - 1]; vo[p] = vo[p - 1]; --p; }
                xo[p] = xb;
                vo[p] = vb;
                if (kept < m) ++kept;
            }
            kept = __shfl_sync(0xffffffffu, kept, 0);
        }
        __syncwarp();
        if (kept == m) { xw = xo[m - 1]; vw = vo[m - 1]; }
    }
    if (lane == 0 && found != nullptr) found[i] = kept;
}

// ---------------------------------------------------------------------------------------------------------------
// A graph sampled from the model (read only; bigclam_sample_graph).  For every unordered pair u < v of the n nodes:
//   shared      rows u and v have a component that is non-zero in both: p_uv = pair_p(pair_x(u, v)), the bits of
//               bigclam_pair_affinity's p (its floor 1 - MAX_P_ included);
//   not shared  p_uv = eps, the caller's background probability (0 <= eps < 1);
// and the pair is an edge iff r(seed, u, v) < p_uv, with
//   key = (uint64)u << 32 | v,  h = mix(seed ^ mix(key)),  r = (h >> 11) * 2^-53,
// mix = the splitmix64 step.  The result is a function of (F bits, seed, eps, min_p, max_p) only.
//
// Row u decides all of its pairs, v < u and v > u, so every pair is decided twice, once from each end, with the same
// bits (x, p and r are symmetric): no transpose and no symmetrisation, and any cut of the rows into batches works.
//   co-member pairs  for c in supp(u), v in M_c (the column index below), v != u: one merge of the two rows gives x_uv
//                    and the first shared component; the pair is taken at that component only, so once per row;
//   background       (eps > 0) lanes stride over all v != u and hash first; only a hit (an eps fraction) pays the merge
//                    that checks the two rows share nothing.
// count gives the row's degree; fill writes the row at its offset, then sorts it (warp_sort_u32).
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ double sample_r(uint64_t seed, int64_t u, int64_t v) {
    const uint64_t lo = (uint64_t)(u < v ? u : v), hi = (uint64_t)(u < v ? v : u);
    const uint64_t h = splitmix64(seed ^ splitmix64(lo << 32 | hi));
    return (double)(h >> 11) * 0x1.0p-53;
}

// pair_x's fold (the same bits) and the first component that is non-zero in both rows (-1: none)
__device__ __forceinline__ double pair_x_first(const RowSrc &s, int64_t u, int64_t v, int &first) {
    double x = 0.0;
    first = -1;
    if (s.hdr != nullptr) {
        const uint64_t hu = s.hdr[u], hv = s.hdr[v];
        const uint32_t cu = sp_cnt(hu), cv = sp_cnt(hv);
        const double *au = s.pool + sp_off8(hu), *av = s.pool + sp_off8(hv);
        const unsigned short *iu = sp_idx(au, cu), *iv = sp_idx(av, cv);
        uint32_t i = 0, j = 0;
        while (i < cu && j < cv) {
            const unsigned short a = iu[i], b = iv[j];
            if (a == b) {
                if (first < 0 && au[i] != 0.0 && av[j] != 0.0) first = a;
                x = __dadd_rn(x, __dmul_rn(au[i], av[j]));
                ++i;
                ++j;
            } else if (a < b) ++i;
            else ++j;
        }
        return x;
    }
    const double *fu = s.F + (size_t)u * s.ld, *fv = s.F + (size_t)v * s.ld;
    for (int c = 0; c < s.k; ++c) {
        const double a = fu[c], b = fv[c];
        if (a != 0.0 && b != 0.0) {
            if (first < 0) first = c;
            x = __dadd_rn(x, __dmul_rn(a, b));
        }
    }
    return x;
}

// Row u as stored: cnt entries vals[0, cnt) at components idx[i] (sparse rows) or i (dense rows, cnt = k).  The k - cnt
// components a sparse row does not store are zeros.
struct RowView {
    const double *vals;
    const unsigned short *idx;         // nullptr: dense row
    int cnt;
};
__device__ __forceinline__ RowView row_view(const RowSrc &s, int64_t u) {
    if (s.hdr == nullptr) return RowView{s.F + (size_t)u * s.ld, nullptr, s.k};
    const uint64_t hu = s.hdr[u];
    const double *vals = s.pool + sp_off8(hu);
    return RowView{vals, sp_idx(vals, sp_cnt(hu)), (int)sp_cnt(hu)};
}

// ---------------------------------------------------------------------------------------------------------------
// Community membership, Bigclamv2.scala:225-228 (bigclam_extract, bigclam_extract_grouped).  With fmax_u the maximum of
// row u over all k components (the zeros a sparse row does not store included), u is a member of community c iff
//   fmax_u <  delta:  F_uc == fmax_u   (ties included, `value == Fmax` at :227)
//   fmax_u >= delta:  F_uc >= delta.
// row_fmax is warp-uniform; every lane gets the same bits whatever the layout.
__device__ __forceinline__ double row_fmax(const RowSrc &s, const RowView &r, int lane) {
    double mx = r.cnt < s.k ? 0.0 : -INFINITY;
    for (int i = lane; i < r.cnt; i += 32) mx = fmax2(mx, r.vals[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax2(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    return mx;
}
__host__ __device__ __forceinline__ bool is_member(double v, double fmax, double delta) { return fmax < delta ? v == fmax : v >= delta; }

#ifdef BIGCLAM_EMU          // host emulation (tests/emu): no atomicMin / atomicMax there
template <bool kMax, class T>
inline void atomic_extreme(T *p, T v) {
    T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while ((kMax ? v > old : v < old) && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
    }
}
inline void atomic_min_u64(unsigned long long *p, unsigned long long v) { atomic_extreme<false>(p, v); }
inline void atomic_max_u64(unsigned long long *p, unsigned long long v) { atomic_extreme<true>(p, v); }
inline void atomic_min_u32(unsigned int *p, unsigned int v) { atomic_extreme<false>(p, v); }
#else
__device__ __forceinline__ void atomic_min_u64(unsigned long long *p, unsigned long long v) { atomicMin(p, v); }
__device__ __forceinline__ void atomic_max_u64(unsigned long long *p, unsigned long long v) { atomicMax(p, v); }
__device__ __forceinline__ void atomic_min_u32(unsigned int *p, unsigned int v) { atomicMin(p, v); }
#endif

// Which entries of a row the column index lists (colidx_kernel's predicate).  row() runs once per row with the whole
// warp and gives the row's state; take(state, v) says whether an entry v != 0 is listed; whole(state) names a column
// that takes the row itself (-1: none).
struct NonZeroPred {               // every non-zero (the sampler's M_c)
    struct Row {};
    __device__ __forceinline__ Row row(const RowSrc &, const RowView &, int64_t, int) const { return Row{}; }
    __device__ __forceinline__ bool take(const Row &, double) const { return true; }
    __device__ __forceinline__ int whole(const Row &) const { return -1; }
};
// Membership for delta > 0 and F >= 0 (bigclam_extract_grouped): a row with a non-zero entry has its members among its
// non-zeros; an all-zero row (fmax = 0 < delta) is a member of every community and goes, once, to column k.  neg (count
// pass only) takes the smallest row with a negative entry, for which the rule above does not hold.
struct MemberPred {
    double delta;
    int k;
    unsigned long long *neg;
    double *fmax = nullptr;            // (optional) fmax[u] = row_fmax, for community_stats_kernel
    struct Row {
        double fmax;
    };
    __device__ __forceinline__ Row row(const RowSrc &s, const RowView &r, int64_t u, int lane) const {
        if (neg != nullptr) {
            bool any = false;
            for (int i = lane; i < r.cnt; i += 32) any |= r.vals[i] < 0.0;
            if (any) atomic_min_u64(neg, (unsigned long long)u);
        }
        const double mx = row_fmax(s, r, lane);
        if (fmax != nullptr && lane == 0) fmax[u] = mx;
        return Row{mx};
    }
    __device__ __forceinline__ bool take(const Row &st, double v) const { return is_member(v, st.fmax, delta); }
    __device__ __forceinline__ int whole(const Row &st) const { return st.fmax == 0.0 ? k : -1; }
};

// Column index of the current rows under a predicate P: colptr and members, list c = members[colptr[c], colptr[c + 1])
// ascending.  Built by count, scan (host) and fill, one warp per row; the fill takes slots in any order and the sort
// makes the lists ascending, so the index is the same from run to run.  Only the columns [c0, c1) are counted or
// filled: count adds to colcnt[c], fill writes members[colpos[c - c0]++] (positions relative to the caller's buffer).
template <bool kFill, class P>
__global__ void colidx_kernel(RowSrc s, int64_t n, P pred, int32_t c0, int32_t c1, unsigned int *__restrict__ colcnt,
                              unsigned long long *__restrict__ colpos, int32_t *__restrict__ members) {
    const int lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= n) return;
    const RowView r = row_view(s, u);
    const typename P::Row st = pred.row(s, r, u, lane);
    auto list = [&](int c) {
        if (c < c0 || c >= c1) return;
        if (kFill) members[atomicAdd(&colpos[c - c0], 1ull)] = (int32_t)u;
        else atomicAdd(&colcnt[c], 1u);
    };
    const int w = pred.whole(st);
    if (w >= 0) {
        if (lane == 0) list(w);
        return;
    }
    for (int i = lane; i < r.cnt; i += 32) {
        const double v = r.vals[i];
        if (v == 0.0 || !pred.take(st, v)) continue;
        list(r.idx != nullptr ? (int)r.idx[i] : i);
    }
}

// Sorts each list c < nc of members[colptr[c] - base, colptr[c + 1] - base), one warp per list.
__global__ void colidx_sort_kernel(const int64_t *__restrict__ colptr, int32_t nc, int64_t base, int32_t *__restrict__ members) {
    const int lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (c >= nc) return;
    warp_sort_u32(reinterpret_cast<uint32_t *>(members + (colptr[c] - base)), colptr[c + 1] - colptr[c], lane);
}

// bigclam_extract's n x k bytes for the rows [r0, r1), one warp per row: member[(u - r0) k + c] = is_member(F_uc), and
// fmax[u - r0] = row_fmax.  A sparse row writes its implicit zeros' verdict first, then its stored entries.
__global__ void extract_rows_kernel(RowSrc s, int64_t r0, int64_t r1, double delta, uint8_t *__restrict__ member,
                                    double *__restrict__ fmax) {
    const int lane = threadIdx.x & 31;
    const int64_t u = r0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= r1) return;
    const RowView r = row_view(s, u);
    const double mx = row_fmax(s, r, lane);
    uint8_t *m = member + (size_t)(u - r0) * s.k;
    if (r.idx != nullptr) {
        const uint8_t z = is_member(0.0, mx, delta);
        for (int c = lane; c < s.k; c += 32) m[c] = z;
        __syncwarp();
    }
    for (int i = lane; i < r.cnt; i += 32) m[r.idx != nullptr ? (int)r.idx[i] : i] = is_member(r.vals[i], mx, delta);
    if (lane == 0) fmax[u - r0] = mx;
}

// Community scores (bigclam_community_stats): volume[c] and internal[c] over the members M(u) of is_member, with
// fmax[u] = row_fmax from the count pass (colidx_kernel with MemberPred, which also checks F >= 0); fmax 0 marks a zero
// row, whose memberships are not walked.  One warp per row u, the lanes over u's list entries u -> v:
//   u not a zero row  M(u) goes to the warp's bitmap of k bits in shared memory; volume[c] += deg(u) for c in M(u).  A lane
//                     walks the stored entries of each v that is not a zero row: internal[c] += 1 for each c in M(v)
//                     whose bit is set.  zero_rows: the entries to zero rows add their count to internal[c], c in M(u);
//   u a zero row      (zero_rows only) internal[c] += 1 for c in M(v) of every entry to a v that is not a zero row;
//                     scal[0] += deg(u) and scal[1] += the entries to zero rows, which the host adds to every c.
// The work is O(entries x stored row length), never O(k x zero-row degree).
constexpr int kStatWarps = 8;
__global__ void community_stats_kernel(RowSrc s, const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col, int64_t n,
                                       const double *__restrict__ fmax, double delta, bool zero_rows,
                                       unsigned long long *__restrict__ volume, unsigned long long *__restrict__ internal,
                                       unsigned long long *__restrict__ scal) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= n) return;                                      // (warp-uniform)
    const double fu = fmax[u];
    const int64_t e0 = rowptr[u], e1 = rowptr[u + 1];
    if (fu == 0.0) {
        if (!zero_rows) return;
        unsigned long long zz = 0;
        for (int64_t e = e0 + lane; e < e1; e += 32) {
            const int32_t v = col[e];
            const double fv = fmax[v];
            if (fv == 0.0) {
                ++zz;
                continue;
            }
            const RowView r = row_view(s, v);
            for (int i = 0; i < r.cnt; ++i)
                if (is_member(r.vals[i], fv, delta)) atomicAdd(&internal[r.idx != nullptr ? (int)r.idx[i] : i], 1ull);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) zz += __shfl_xor_sync(0xffffffffu, zz, o);
        if (lane == 0) {
            atomicAdd(&scal[0], (unsigned long long)(e1 - e0));
            if (zz != 0) atomicAdd(&scal[1], zz);
        }
        return;
    }
    const int words = (s.k + 31) >> 5;
    unsigned int *bits = reinterpret_cast<unsigned int *>(smem_raw) + (threadIdx.x >> 5) * words;
    for (int i = lane; i < words; i += 32) bits[i] = 0u;
    __syncwarp();
    const RowView ru = row_view(s, u);
    for (int i = lane; i < ru.cnt; i += 32)
        if (is_member(ru.vals[i], fu, delta)) {
            const int c = ru.idx != nullptr ? (int)ru.idx[i] : i;
            atomicOr(&bits[c >> 5], 1u << (c & 31));
            atomicAdd(&volume[c], (unsigned long long)(e1 - e0));
        }
    __syncwarp();
    unsigned long long zn = 0;
    for (int64_t e = e0 + lane; e < e1; e += 32) {
        const int32_t v = col[e];
        const double fv = fmax[v];
        if (fv == 0.0) {
            ++zn;
            continue;
        }
        const RowView r = row_view(s, v);
        for (int i = 0; i < r.cnt; ++i) {
            const int c = r.idx != nullptr ? (int)r.idx[i] : i;
            if (((bits[c >> 5] >> (c & 31)) & 1u) && is_member(r.vals[i], fv, delta)) atomicAdd(&internal[c], 1ull);
        }
    }
    if (!zero_rows) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) zn += __shfl_xor_sync(0xffffffffu, zn, o);
    if (zn == 0) return;                                     // (warp-uniform)
    for (int i = lane; i < ru.cnt; i += 32)
        if (is_member(ru.vals[i], fu, delta)) atomicAdd(&internal[ru.idx != nullptr ? (int)ru.idx[i] : i], zn);
}

// ---------------------------------------------------------------------------------------------------------------
// The member-counting loop of cover_scores_kernel and community_overlaps_kernel: the warps of a block walk the rows
// list[i0, i1), one row per warp (warp w of kWarps takes i0 + w, i0 + w + kWarps, ...), and add 1 to cnt[c] (shared
// memory) for each c in M(u), read with row_view + is_member; fmax[u] = row_fmax from the count pass.  A zero row
// (fmax 0) is never expanded: the returned value (the same on every lane) is the number of zero rows the warp met.
template <int kWarps>
__device__ __forceinline__ unsigned int count_memberships(const RowSrc &s, const double *__restrict__ fmax, double delta,
                                                          const int32_t *__restrict__ list, int64_t i0, int64_t i1,
                                                          unsigned int *cnt) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned int zeros = 0;
    for (int64_t i = i0 + warp; i < i1; i += kWarps) {
        const int32_t u = list[i];
        const double fu = fmax[u];
        if (fu == 0.0) {                                     // (warp-uniform)
            ++zeros;
            continue;
        }
        const RowView r = row_view(s, u);
        for (int j = lane; j < r.cnt; j += 32)
            if (is_member(r.vals[j], fu, delta)) atomicAdd(&cnt[r.idx != nullptr ? (int)r.idx[j] : j], 1u);
    }
    return zeros;
}

// ---------------------------------------------------------------------------------------------------------------
// Cover scores (bigclam_cover_scores): the detected cover X (the communities of is_member, the zero rows in every
// community or in none) against a truth cover Y given as a CSR of distinct members.  Non-negative doubles order as their
// bits, so the per-community maxima and minima over t are 64-bit integer atomics and come out the same in any order.
__device__ __forceinline__ unsigned long long dbl_bits(double d) {
    return ((unsigned long long)(unsigned)__double2hiint(d) << 32) | (unsigned)__double2loint(d);
}
__device__ __forceinline__ double bits_dbl(unsigned long long b) { return __hiloint2double((int)(b >> 32), (int)(unsigned)b); }

// h[m] = -(p log p) with p = m / n, m = 0 .. n (h[0] = 0): the one table every entropy of the cover scores reads.
__global__ void cover_h_kernel(int64_t n, double *__restrict__ h) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m > n) return;
    const double p = (double)m / (double)n;
    h[m] = m == 0 ? 0.0 : -(p * log(p));
}

// hs[i] = H(S_i) = h(s) + h(n - s) for the sizes s = size[i], i < cnt.
__global__ void cover_hsize_kernel(const double *__restrict__ h, int64_t n, const int64_t *__restrict__ size, int64_t cnt,
                                   double *__restrict__ hs) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cnt) hs[i] = h[size[i]] + h[n - size[i]];
}

struct CoverArgs {
    RowSrc s;
    const double *fmax;                // row_fmax from the count pass; 0: a zero row
    const int64_t *tptr;               // truth community t = tmem[tptr[t], tptr[t + 1]), distinct ids
    const int32_t *tmem;
    const int64_t *xs;                 // |X_c| (the zero rows counted in when zero_rows); 0: an empty community
    const double *h;                   // cover_h_kernel's table
    int64_t n;
    double delta;
    bool zero_rows;
    unsigned long long *f1_det;        // per c: bits of max_t F1(c, t), from 0
    unsigned long long *hc_det;        // per c: bits of min over admissible t of H(X_c | Y_t), from +inf
    unsigned int *match_det;           // per c (kTies): the smallest t with F1(c, t) == f1_det[c] > 0, from ~0u
    double *f1_t, *hc_t, *hy_t;        // per t: max_c F1(c, t); min over admissible c of H(Y_t | X_c) (+inf: none); H(Y_t)
    int32_t *match_t;                  // per t: the smallest c attaining f1_t, -1 when f1_t = 0
};

// One block per truth community t (empty ones return).  count_memberships walks t's members u: a zero row adds 1 to
// z_t, any other row adds 1 to cnt[c] (k counters in shared memory) for each c in M(u), so zero rows are never
// expanded.  Then every non-empty c is a pair (c, t)
// with a = cnt[c] (+ z_t when zero_rows), x = xs[c], y = |Y_t|:
//   !kTies  F1 = 2a / (x + y) goes to f1_det[c] (atomicMax on its bits, after a read that skips what cannot improve)
//           and to the block's maximum (smallest c on ties); an admissible pair's H(X_c | Y_t) goes to hc_det[c]
//           (atomicMin likewise) and its H(Y_t | X_c) to the block's minimum.  The k x q pairs with a = 0 are evaluated
//           too: one with x + y > n / 2 can be admissible.
//   kTies   (after the !kTies launch) every pair whose F1 equals f1_det[c] > 0 offers t to match_det[c] (atomicMin).
// No floating-point sum depends on the order of the atomics or of the threads.
constexpr int kCoverWarps = 8;
template <bool kTies>
__global__ void __launch_bounds__(32 * kCoverWarps) cover_scores_kernel(CoverArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned int s_zt;
    __shared__ double s_f1[kCoverWarps], s_hc[kCoverWarps];
    __shared__ int s_c[kCoverWarps];
    unsigned int *cnt = reinterpret_cast<unsigned int *>(smem_raw);
    const int64_t t = blockIdx.x;
    const int64_t m0 = a.tptr[t], m1 = a.tptr[t + 1];
    if (m0 == m1) return;                                    // (block-uniform)
    const int k = a.s.k, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x; c < k; c += blockDim.x) cnt[c] = 0u;
    if (threadIdx.x == 0) s_zt = 0u;
    __syncthreads();
    const unsigned int zeros = count_memberships<kCoverWarps>(a.s, a.fmax, a.delta, a.tmem, m0, m1, cnt);
    if (lane == 0 && zeros != 0u) atomicAdd(&s_zt, zeros);
    __syncthreads();
    const int64_t n = a.n, y = m1 - m0, zt = a.zero_rows ? (int64_t)s_zt : 0;
    const double *h = a.h;
    const double hy = h[y] + h[n - y];
    double best = 0.0, hmin = INFINITY;
    int bc = -1;
    for (int c = threadIdx.x; c < k; c += blockDim.x) {
        const int64_t x = a.xs[c];
        if (x == 0) continue;
        const int64_t ai = (int64_t)cnt[c] + zt;
        const double f1 = (2.0 * (double)ai) / (double)(x + y);
        if (kTies) {
            if (ai > 0 && dbl_bits(f1) == __ldcg(&a.f1_det[c])) atomic_min_u32(&a.match_det[c], (unsigned int)t);
            continue;
        }
        if (f1 > best) {
            best = f1;
            bc = c;
        }
        if (ai > 0) {
            const unsigned long long b = dbl_bits(f1);
            if (b > __ldcg(&a.f1_det[c])) atomic_max_u64(&a.f1_det[c], b);
        }
        const double ha = h[ai], hxa = h[x - ai], hya = h[y - ai], hd = h[n - x - y + ai];
        if (ha + hd > hxa + hya) {                           // admissible (symmetric in X and Y)
            const double hx = h[x] + h[n - x];
            const unsigned long long b = dbl_bits(fmax(0.0, ((ha + hxa) + hya) + hd - hy));   // H(X_c | Y_t)
            if (b < __ldcg(&a.hc_det[c])) atomic_min_u64(&a.hc_det[c], b);
            hmin = fmin(hmin, fmax(0.0, ((ha + hya) + hxa) + hd - hx));                     // H(Y_t | X_c)
        }
    }
    if (kTies) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o), oh = __shfl_xor_sync(0xffffffffu, hmin, o);
        const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
        if (ob > best || (ob == best && (unsigned)oc < (unsigned)bc)) {
            best = ob;
            bc = oc;
        }
        hmin = fmin(hmin, oh);
    }
    if (lane == 0) {
        s_f1[warp] = best;
        s_c[warp] = bc;
        s_hc[warp] = hmin;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 1; w < kCoverWarps; ++w) {
        if (s_f1[w] > best || (s_f1[w] == best && (unsigned)s_c[w] < (unsigned)bc)) {
            best = s_f1[w];
            bc = s_c[w];
        }
        hmin = fmin(hmin, s_hc[w]);
    }
    a.f1_t[t] = best;
    a.match_t[t] = best > 0.0 ? bc : -1;
    a.hc_t[t] = hmin;
    a.hy_t[t] = hy;
}

// ---------------------------------------------------------------------------------------------------------------
// Community overlaps (bigclam_community_overlaps): shared(c, d) = |M_c ∩ M_d| over the non-zero rows, for every pair
// c != d with shared(c, d) >= min_shared.
struct OverlapArgs {
    RowSrc s;
    const double *fmax;                // row_fmax from the count pass
    const int64_t *colptr;             // the column index of the memberships (colidx_kernel with MemberPred, columns < k:
    const int32_t *members;            //   no zero rows), any order within a column
    double delta;
    unsigned int min_shared;
    int32_t c0;                        // block b works on community c0 + b
    unsigned int *rowcnt;              // count launch: rowcnt[c] = the entries of row c
    const int64_t *ovptr;              // fill launch: row c goes to other / shared [ovptr[c - c0] - base, ...)
    int64_t base;
    int32_t *other, *shared;
};

// One block per community c.  count_memberships walks c's members u and adds 1 to cnt[d] (k counters in shared memory)
// for each d in M(u), so cnt[d] = shared(c, d) (cnt[c] = |M_c|).  Then one block-wide ordered compaction over the
// counters, blockDim.x of them per round: a ballot per warp, the warps' totals in shared memory, a running offset.  The
// count launch (!kFill) keeps the total, the fill launch writes each kept d and its count at its rank, so every row
// comes out ascending in d with no sort.  Everything is integer: any order of the atomics gives the same output.
constexpr int kOverlapWarps = 8;
template <bool kFill>
__global__ void __launch_bounds__(32 * kOverlapWarps) community_overlaps_kernel(OverlapArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned int s_wsum[kOverlapWarps];
    unsigned int *cnt = reinterpret_cast<unsigned int *>(smem_raw);
    const int c = a.c0 + (int)blockIdx.x;
    const int k = a.s.k, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = threadIdx.x; d < k; d += blockDim.x) cnt[d] = 0u;
    __syncthreads();
    count_memberships<kOverlapWarps>(a.s, a.fmax, a.delta, a.members, a.colptr[c], a.colptr[c + 1], cnt);
    __syncthreads();
    const int64_t out0 = kFill ? a.ovptr[c - a.c0] - a.base : 0;
    unsigned int done = 0;                                   // (block-uniform) entries kept in the rounds before
    for (int d0 = 0; d0 < k; d0 += blockDim.x) {
        const int d = d0 + (int)threadIdx.x;
        const unsigned int v = d < k ? cnt[d] : 0u;
        const bool keep = d < k && d != c && v >= a.min_shared;
        const unsigned int m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_wsum[warp] = (unsigned int)__popc(m);
        __syncthreads();
        unsigned int before = 0, round = 0;
        for (int w = 0; w < kOverlapWarps; ++w) {
            const unsigned int x = s_wsum[w];
            before += w < warp ? x : 0u;
            round += x;
        }
        if (kFill && keep) {
            const int64_t p = out0 + done + before + (unsigned int)__popc(m & ((1u << lane) - 1u));
            a.other[p] = d;
            a.shared[p] = (int32_t)v;
        }
        done += round;
        __syncthreads();                                     // (s_wsum is rewritten by the next round)
    }
    if (!kFill && threadIdx.x == 0) a.rowcnt[c] = done;
}

struct SampleArgs {
    RowSrc s;
    PairConst pc;
    const int64_t *colptr;             // the column index (colidx_kernel)
    const int32_t *members;
    int64_t n;
    uint64_t seed;
    double eps;
};

// One warp per row u of [r0, r1).  count: deg[u - r0] = the row's degree.  fill: the row goes to out[rowptr[u] - base ..),
// ascending.
template <bool kFill>
__global__ void sample_rows_kernel(SampleArgs a, int64_t r0, int64_t r1, int64_t *__restrict__ deg, const int64_t *__restrict__ rowptr,
                                   int64_t base, int32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t u = r0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (u >= r1) return;                                     // (warp-uniform)
    const unsigned lt_mask = (1u << lane) - 1u;
    int32_t *seg = kFill ? out + (rowptr[u] - base) : nullptr;
    int64_t taken = 0;                                       // (warp-uniform)
    auto emit = [&](bool take, int64_t v) {
        const unsigned bal = __ballot_sync(0xffffffffu, take);
        if (kFill && take) seg[taken + __popc(bal & lt_mask)] = (int32_t)v;
        taken += __popc(bal);
    };
    const RowSrc &s = a.s;
    const bool sparse = s.hdr != nullptr;
    const uint64_t hu = sparse ? s.hdr[u] : 0;
    const int cnt = sparse ? (int)sp_cnt(hu) : s.k;
    const double *vals = sparse ? s.pool + sp_off8(hu) : s.F + (size_t)u * s.ld;
    const unsigned short *idx = sparse ? sp_idx(vals, (uint32_t)cnt) : nullptr;
    for (int i = 0; i < cnt; ++i) {                          // co-member pairs, component by component
        if (vals[i] == 0.0) continue;
        const int c = sparse ? (int)idx[i] : i;
        const int64_t m0 = a.colptr[c], m1 = a.colptr[c + 1];
        for (int64_t t0 = m0; t0 < m1; t0 += 32) {
            const int64_t t = t0 + lane;
            const int64_t v = (t < m1) ? a.members[t] : u;
            bool take = false;
            if (v != u) {
                int first;
                const double x = pair_x_first(s, u, v, first);
                take = first == c && sample_r(a.seed, u, v) < pair_p(x, a.pc);
            }
            emit(take, v);
        }
    }
    if (a.eps > 0.0) {                                       // background pairs
        for (int64_t v0 = 0; v0 < a.n; v0 += 32) {
            const int64_t v = v0 + lane;
            bool take = false;
            if (v < a.n && v != u && sample_r(a.seed, u, v) < a.eps) {
                int first;
                (void)pair_x_first(s, u, v, first);
                take = first < 0;
            }
            emit(take, v);
        }
    }
    if (!kFill) {
        if (lane == 0) deg[u - r0] = taken;
        return;
    }
    __syncwarp();
    warp_sort_u32(reinterpret_cast<uint32_t *>(seg), taken, lane);
}

// ---------------------------------------------------------------------------------------------------------------
// Fold-in (read only; bigclam_fold_in): the row f of a NEW node u, given its neighbour list N(u) among the n fitted
// nodes, with every fitted row and sumF held fixed.  u's objective is the step's own (bigclam4-7.scala:157-184) for u
// appended to the graph, whose sumF is then sumF' = sumF + f:
//   l_u(f) = sum_{v in N(u)} [log(1 - clamp(exp(-f.F_v))) + f.F_v] - f.sumF' + f.f,   grad = sum_v w_v F_v - sumF' + f,
// and a candidate nf is scored with sumF' - f + nf (:176-180), every sum rounded as the step rounds it.  From f = 0, at
// most max_iter line searches over the 16 candidates, each taking the largest step that passes; it stops when none
// passes or when |1 - l_t / l_{t-1}| < rel_tol (:237 for one node).
//
// One warp per query node.  The phases are the general path's own, compiled for fold-in (SpGen<kWide, true>): PRE
// (pre_range), the line search (ls_range) and the Armijo decision (decide), with the staging of sparse rows, a dense-row
// stager and the active-entry compaction; the gradient scan over the touched components is SpGen::scan_list.  ptxas:
// 80 registers (ld <= 1024) and 94 (wide rows), no spills.  Only the components the node TOUCHES
// (its neighbours' non-zeros; its own row stays inside them) are visited: an untouched component has f = 0 and
// gradient -sumF_c <= 0, never moves, and enters |g|^2 through S2_all - sum_touched sumF_c^2 (the identity of the tile
// and wide paths).  The first PRE marks the touched components and they are listed once, ascending, in `tl` for the
// node's whole run.  Every sum has a fixed order and there are no floating-point atomics: a node's results are the
// same bits whatever the batch around it.  The step's constants (steps, alpha, max_f, the edge term's clamp) come
// from the context's StepArgs; FoldArgs holds the batch.
struct FoldArgs {
    RowSrc s;
    double S2_all;               // sum_c sumF_c^2 over the k components, ascending c
    const int64_t *rowptr;       // the batch's lists: node i has col[rowptr[i] .. rowptr[i + 1])
    const int32_t *col;
    int64_t nq;
    int32_t max_iter;
    double rel_tol;
    const int64_t *slot;         // fill: node i's row goes to out_idx / out_val from slot[i] (nullptr: count only)
    int32_t *out_idx;
    double *out_val;
    int32_t *cnt;                // per node: non-zeros of the row, l_u of the row, accepted steps
    double *llh;
    int32_t *iters;
    unsigned char *scratch;      // wide rows: fold_warp_bytes(ld) per warp of the grid, all zero between nodes
};

constexpr int kFoldWarps = 4;    // warps per block
// per warp: fu_d[ldp] | g_d[ldp] | ent_val[E] | cbal[E/32] u32 | tmask[ldp/32] u32 | ent_idx[E] u16 | tl[ldp] u16 |
//           aidx[ldp] u16 | poff[40] u16 | ccum[E/32] u16      (shared memory for ld <= 1024, else global scratch)
__host__ __device__ inline size_t fold_warp_bytes(int ld) {
    const size_t ldp = (size_t)sp_ldp(ld), E = (size_t)sp_entries(ld), Ew = (size_t)sp_ldp(sp_entries(ld)) / 32;
    return (16 * ldp + 10 * E + 4 * Ew + ldp / 8 + 4 * ldp + 80 + 2 * Ew + 15) & ~(size_t)15;
}

template <bool kWide>
struct FoldGen {
    SpGen<kWide, true> g;
    const FoldArgs *a;
    unsigned short *tl;          // the touched components, ascending

    __device__ __forceinline__ void carve(unsigned char *base, int ld, int lane) {
        g.ld = ld;
        g.ldp = sp_ldp(ld);
        g.ecap = sp_entries(ld);
        g.lane = lane;
        g.lt_mask = (1u << lane) - 1u;
        const int Ew = sp_ldp(g.ecap) / 32;
        g.fu_d = reinterpret_cast<double *>(base);
        g.g_d = g.fu_d + g.ldp;
        g.ent_val = g.g_d + g.ldp;
        g.cbal = reinterpret_cast<unsigned int *>(g.ent_val + g.ecap);
        g.tmask = g.cbal + Ew;
        g.ent_idx = reinterpret_cast<unsigned short *>(g.tmask + g.ldp / 32);
        tl = g.ent_idx + g.ecap;
        g.aidx = tl + g.ldp;
        g.poff = g.aidx + g.ldp;
        g.ccum = g.poff + 40;
    }

    // Query node i, start to finish.  Leaves fu_d, g_d and tmask at zero.
    __device__ __forceinline__ void node(int64_t i) {
        const int lane = g.lane;
        const int64_t e0 = a->rowptr[i];
        const int deg = (int)(a->rowptr[i + 1] - e0);
        const int32_t *colp = a->col + e0;
        const int nsteps = g.a->nsteps;
        double l = 0.0, lprev = 0.0;
        int it = 0, nt = 0;
#pragma unroll 1
        while (deg > 0) {
            // ---------------- PRE of f_it: l_it and the weighted neighbour sum ----------------
            int nchunks, ne_last;
            const double S1 = warp_sum(g.pre_range(colp, 0, deg, true, nchunks, ne_last, it == 0));
            if (it == 0) nt = g.list_touched(tl);
            double fusf = 0.0, fufu = 0.0;
#pragma unroll 1
            for (int t = lane; t < nt; t += 32) {
                const int c = tl[t];
                const double f = g.fu_d[c];
                fusf = fma(f, __ldg(g.s_sumF + c) + f, fusf);
                fufu = fma(f, f, fufu);
            }
            l = (S1 - warp_sum(fusf)) + warp_sum(fufu);
            const bool go = !(it > 0 && fabs(1.0 - l / lprev) < a->rel_tol) && it < a->max_iter;
            // ---------------- LS from f_it ----------------
            int jstar = -1, m = 0;
            if (go) {
                bool need_hi;
                const double G2 = g.scan_list(tl, nt, m, need_hi);
#pragma unroll 1
                for (int tg = 0; tg < nsteps && jstar < 0; tg += 16) {
                    const int j = tg + (lane & 15);
                    const bool jok = j < nsteps;
                    const double s = g.s_steps[jok ? j : 0];
                    double st = g.ls_range(colp, 0, deg, s, need_hi, (nchunks == 1 && tg == 0) ? ne_last : 0);
                    st += __shfl_xor_sync(0xffffffffu, st, 16);
                    jstar = g.decide(tg, s, jok, st, m, need_hi, l, G2);
                }
            }
            if (jstar >= 0) {                              // f_{it+1}: the accepted candidate, in place (one lane per component)
                const double s = g.s_steps[jstar];
#pragma unroll 1
                for (int t = lane; t < m; t += 32) {
                    const int c = g.aidx[t];
                    g.fu_d[c] = clamp_step0(g.fu_d[c], s, g.g_d[c], g.a->max_f);
                }
                __syncwarp();                              // (every lane is done reading g_d)
            }
#pragma unroll 1
            for (int t = lane; t < nt; t += 32) g.g_d[tl[t]] = 0.0;
            __syncwarp();
            if (jstar < 0) break;
            lprev = l;
            ++it;
        }
        // ---------------- the row: non-zeros of fu_d, ascending ----------------
        int cnt = 0;
#pragma unroll 1
        for (int t0 = 0; t0 < nt; t0 += 32) {
            const int t = t0 + lane;
            const int c = (t < nt) ? (int)tl[t] : 0;
            const double v = (t < nt) ? g.fu_d[c] : 0.0;
            const unsigned bal = __ballot_sync(0xffffffffu, v != 0.0);
            if (a->slot != nullptr && v != 0.0) {
                const int64_t p = a->slot[i] + cnt + __popc(bal & g.lt_mask);
                a->out_idx[p] = c;
                a->out_val[p] = v;
            }
            cnt += __popc(bal);
        }
        if (lane == 0) {
            a->cnt[i] = cnt;
            a->llh[i] = l;
            a->iters[i] = it;
        }
        __syncwarp();
#pragma unroll 1
        for (int t = lane; t < nt; t += 32) g.fu_d[tl[t]] = 0.0;
#pragma unroll 1
        for (int w = lane; w < (g.ldp >> 5); w += 32) g.tmask[w] = 0u;
        __syncwarp();
    }
};

// Grid-stride over the batch's query nodes, one warp each.  a: the context's step arguments (fill_args).  kWide: the
// per-warp vectors live in FoldArgs::scratch.
template <bool kWide>
__global__ void fold_in_kernel(const __grid_constant__ StepArgs a, const __grid_constant__ FoldArgs fa, const __grid_constant__ SparseArgs sp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * kFoldWarps + wib, nw = (int64_t)gridDim.x * kFoldWarps;
    const size_t wb = fold_warp_bytes(a.ld);
    unsigned char *base = kWide ? fa.scratch + (size_t)gw * wb : smem_raw + (size_t)wib * wb;
    FoldGen<kWide> fg;
    fg.a = &fa;
    fg.g.a = &a;
    fg.g.sp = &sp;
    fg.g.rs = &fa.s;
    fg.g.s_steps = a.steps;
    fg.g.s_sumF = a.sumF;
    fg.g.S2_all = fa.S2_all;
    fg.g.ec = {a.x_lo, a.x_hi, a.t_lo, a.t_hi, a.w_lo, a.w_hi};
    fg.carve(base, a.ld, lane);
    if constexpr (!kWide) {
        fg.g.clear_dense();
#pragma unroll 1
        for (int w = lane; w < (fg.g.ldp >> 5); w += 32) fg.g.tmask[w] = 0u;
        __syncwarp();
    }
#pragma unroll 1
    for (int64_t i = gw; i < fa.nq; i += nw) fg.node(i);
}

// An upper bound of the row length of each query node: min(k, the non-zeros of its neighbours' rows), one warp per node.
__global__ void fold_bound_kernel(RowSrc s, const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col, int64_t nq,
                                  int64_t *__restrict__ bound) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= nq) return;
    long long t = 0;
    for (int64_t e = rowptr[i] + lane; e < rowptr[i + 1]; e += 32) t += (s.hdr != nullptr) ? (long long)sp_cnt(s.hdr[col[e]]) : (long long)s.k;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) bound[i] = t < s.k ? t : s.k;
}

// ------------------------------------------------------------------------------------------------
// initNeighborComF(K) (bigclam4-7.scala:81-108) built as rows on the device (bigclam_init_F), bit for bit the n x K F0
// of the host (bigclam_init_neighbor_com_F, initf.cpp) without ever holding it.  S = the selected seeds in id order:
//   * column c < |S| is 1.0 on every entry of S[c]'s own neighbour list (and on S[c] with include_self): the pairs
//     (row, c) are scattered from the seeds' lists (the CSR need not be symmetric; repeated entries and seeds allowed),
//     then each row's columns are de-duplicated and sorted through a bitmap of |S| bits;
//   * column c >= |S| is bit 33 of xorshift64*'s output for draw m = (c - |S|) n + u, i.e. of state s_(m+1).  The state
//     update T is linear over GF(2): row u starts from T^(u+1) s_0 (byte tables of T^(2^j)) and moves from one padding
//     column to the next with T^n, so every row draws exactly the host's bits, in ascending column order.
// Counts and offsets come before anything is written (the pool check), and offsets are exclusive scans of the counts
// in row order: the layout and pool_top follow from the rows alone.

constexpr uint64_t kXsMul = 2685821657736338717ULL;   // xorshift64* output multiplier (initf.cpp)
constexpr int kGf2Tab = 8 * 256;                      // byte tables of one 64 x 64 GF(2) matrix

__host__ __device__ inline uint64_t xs_next(uint64_t s) {
    s ^= s >> 12;
    s ^= s << 25;
    s ^= s >> 27;
    return s;
}
__host__ __device__ inline uint64_t gf2_apply(const uint64_t *tab, uint64_t v) {
    uint64_t r = 0;
#pragma unroll
    for (int b = 0; b < 8; ++b) r ^= tab[b * 256 + (int)((v >> (8 * b)) & 255u)];
    return r;
}

// (row, column) pairs of the seeds' lists, one warp per seed: counted per row (kScatter = false), then written to the
// row's segment of raw (taken[] zeroed again in between).
template <bool kScatter>
__global__ void initf_seed_pairs_kernel(int ns, const int32_t *__restrict__ S, const int64_t *__restrict__ rowptr,
                                        const int32_t *__restrict__ col, int include_self, unsigned *taken,
                                        const uint64_t *__restrict__ rawoff, unsigned short *raw) {
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (c >= ns) return;
    const int32_t s = S[c];
    const int64_t e0 = rowptr[s], e1 = rowptr[s + 1];
    for (int64_t e = e0 + lane; e < e1 + (include_self ? 1 : 0); e += 32) {
        const int32_t v = e < e1 ? col[e] : s;
        const unsigned q = atomicAdd(taken + v, 1u);
        if constexpr (kScatter) raw[rawoff[v] + q] = (unsigned short)c;
    }
}

// One warp per row: its seed columns de-duplicated and ascending, written back to the front of its segment of raw.
constexpr int kInitWarps = 8;
__global__ void initf_seed_rows_kernel(int64_t n, int ns, const uint64_t *__restrict__ rawoff, unsigned short *raw,
                                       unsigned *seedcnt) {
    __shared__ unsigned bm_all[kInitWarps][kSpMaxK / 32];
    __shared__ unsigned part_all[kInitWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t u = (int64_t)blockIdx.x * kInitWarps + w;
    if (u >= n) return;
    const uint64_t e0 = rawoff[u], e1 = rawoff[u + 1];
    if (e0 == e1) {
        if (lane == 0) seedcnt[u] = 0;
        return;
    }
    unsigned *bm = bm_all[w], *part = part_all[w];
    const int nw = (ns + 31) >> 5, per = (nw + 31) >> 5;
    for (int i = lane; i < nw; i += 32) bm[i] = 0u;
    __syncwarp();
    for (uint64_t e = e0 + lane; e < e1; e += 32) atomicOr(bm + (raw[e] >> 5), 1u << (raw[e] & 31));
    __syncwarp();
    const int w0 = min(nw, lane * per), w1 = min(nw, w0 + per);   // lane's words
    unsigned mine = 0;
    for (int i = w0; i < w1; ++i) mine += (unsigned)__popc(bm[i]);
    part[lane] = mine;
    __syncwarp();
    unsigned q = 0, tot = 0;
    for (int i = 0; i < 32; ++i) {
        q += i < lane ? part[i] : 0u;
        tot += part[i];
    }
    for (int i = w0; i < w1; ++i)
        for (unsigned x = bm[i]; x != 0u; x &= x - 1u) raw[e0 + q++] = (unsigned short)(i * 32 + __ffs(x) - 1);
    if (lane == 0) seedcnt[u] = tot;
}

struct InitRows {
    int64_t n;
    int32_t ns, npad, ld, njump;
    uint64_t s0;                        // the padding sequence's seed state
    const uint64_t *tabs;               // xs_jump_tables
    const uint64_t *rawoff;             // n + 1
    const unsigned short *raw;          // the rows' seed columns (initf_seed_rows_kernel)
    const unsigned *seedcnt;            // n
    unsigned *cnt;                      // n: written by the count pass, read by the fill pass
    const uint64_t *woff;               // sparse rows: n + 1, the exclusive scan of sp_words(cnt)
    uint64_t *hdr;
    double *pool;
    double *F;                          // dense rows (ld stride), zeroed before the fill pass
    unsigned *colcnt;                   // ld, zeroed: the column counts (fill pass)
};

// One thread per row: the seed columns, then the padding bits.  The count pass (kFill = false) counts the row; the
// fill pass writes it and adds its entries to the column counts.  Every thread of a block runs the padding loop
// (the column counts are taken per warp).
template <bool kFill>
__global__ void initf_rows_kernel(InitRows r) {
    __shared__ uint64_t stride_tab[kGf2Tab];
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = u < r.n;
    if (r.npad > 0) {
        for (int i = threadIdx.x; i < kGf2Tab; i += blockDim.x) stride_tab[i] = r.tabs[(size_t)r.njump * kGf2Tab + i];
        __syncthreads();
    }
    const unsigned nseed = live ? r.seedcnt[u] : 0u;
    double *ov = nullptr, *frow = nullptr;
    unsigned short *oi = nullptr;
    unsigned q = 0;
    if (kFill && live) {
        if (r.F != nullptr) {
            frow = r.F + (size_t)u * r.ld;
        } else {
            const unsigned cnt = r.cnt[u];
            const uint64_t off = r.woff[u];
            ov = r.pool + off;
            oi = sp_idx(ov, cnt);
            for (unsigned i = cnt; i < sp_vpad(cnt); ++i) ov[i] = 0.0;
            for (unsigned i = cnt; i < sp_ipad(cnt); ++i) oi[i] = 0;
            r.hdr[u] = sp_pack(cnt ? off : 0, cnt);
        }
        const unsigned short *sc = r.raw + (live && nseed ? r.rawoff[u] : 0);
        for (unsigned i = 0; i < nseed; ++i) {
            const int c = sc[i];
            if (frow != nullptr) frow[c] = 1.0;
            else { ov[q] = 1.0; oi[q] = (unsigned short)c; ++q; }
            atomicAdd(r.colcnt + c, 1u);
        }
    }
    unsigned npad_set = 0;
    if (r.npad > 0) {
        uint64_t s = r.s0;
        const uint64_t v = live ? (uint64_t)u + 1 : 0;
        for (int j = 0; j < r.njump; ++j)
            if ((v >> j) & 1u) s = gf2_apply(r.tabs + (size_t)j * kGf2Tab, s);
        const int lane = threadIdx.x & 31;
#pragma unroll 1
        for (int j = 0; j < r.npad; ++j) {                  // s = state s_(j n + u + 1)
            const bool bit = live && (((s * kXsMul) >> 33) & 1u);
            npad_set += bit ? 1u : 0u;
            if constexpr (kFill) {
                const int c = r.ns + j;
                if (bit) {
                    if (frow != nullptr) frow[c] = 1.0;
                    else { ov[q] = 1.0; oi[q] = (unsigned short)c; ++q; }
                }
                const unsigned b = __ballot_sync(0xffffffffu, bit);
                if (lane == 0 && b != 0u) atomicAdd(r.colcnt + c, (unsigned)__popc(b));
            }
            s = gf2_apply(stride_tab, s);
        }
    }
    if (!kFill && live) r.cnt[u] = nseed + npad_set;
}

__global__ void initf_sumF_kernel(const unsigned *__restrict__ colcnt, int ld, double *sumF) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < ld) sumF[c] = (double)colcnt[c];
}

// Exclusive scan of n counts (or of sp_words(count)) into out[0 .. n], out[n] = the total: chunk sums, a scan of the
// chunk sums in one block, then each chunk with its base.
constexpr int kScanThreads = 256, kScanChunk = 4 * kScanThreads;
__device__ inline uint64_t block_exclusive_scan(uint64_t x, uint64_t *sh, uint64_t *total) {
    const int t = threadIdx.x;
    sh[t] = x;
    __syncthreads();
    for (int off = 1; off < kScanThreads; off <<= 1) {
        const uint64_t y = t >= off ? sh[t - off] : 0;
        __syncthreads();
        sh[t] += y;
        __syncthreads();
    }
    const uint64_t incl = sh[t];
    *total = sh[kScanThreads - 1];
    __syncthreads();
    return incl - x;
}
__device__ inline uint64_t scan_item(const unsigned *cnt, int64_t n, int words, int64_t i) {
    if (i >= n) return 0;
    return words ? sp_words(cnt[i]) : (uint64_t)cnt[i];
}
__global__ void scan_chunks_kernel(const unsigned *__restrict__ cnt, int64_t n, int words, uint64_t *chunk_sum) {
    __shared__ uint64_t sh[kScanThreads];
    const int64_t i0 = (int64_t)blockIdx.x * kScanChunk + 4 * threadIdx.x;
    uint64_t x = 0, total = 0;
    for (int k = 0; k < 4; ++k) x += scan_item(cnt, n, words, i0 + k);
    block_exclusive_scan(x, sh, &total);
    if (threadIdx.x == 0) chunk_sum[blockIdx.x] = total;
}
__global__ void scan_top_kernel(uint64_t *chunk_sum, int64_t nchunks, uint64_t *grand_total) {
    __shared__ uint64_t sh[kScanThreads];
    uint64_t carry = 0;
    for (int64_t b0 = 0; b0 < nchunks; b0 += kScanThreads) {
        const int64_t i = b0 + threadIdx.x;
        const uint64_t x = i < nchunks ? chunk_sum[i] : 0;
        uint64_t total = 0;
        const uint64_t ex = block_exclusive_scan(x, sh, &total);
        if (i < nchunks) chunk_sum[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *grand_total = carry;
}
__global__ void scan_apply_kernel(const unsigned *__restrict__ cnt, int64_t n, int words, const uint64_t *__restrict__ chunk_base,
                                  uint64_t *out) {
    __shared__ uint64_t sh[kScanThreads];
    const int64_t i0 = (int64_t)blockIdx.x * kScanChunk + 4 * threadIdx.x;
    uint64_t v[4], x = 0, total = 0;
    for (int k = 0; k < 4; ++k) { v[k] = scan_item(cnt, n, words, i0 + k); x += v[k]; }
    uint64_t p = chunk_base[blockIdx.x] + block_exclusive_scan(x, sh, &total);
    for (int k = 0; k < 4; ++k) {
        if (i0 + k < n) out[i0 + k] = p;
        p += v[k];
    }
}

}  // namespace bigclam
