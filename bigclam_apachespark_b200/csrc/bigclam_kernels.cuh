// bigclam_kernels.cuh — sm_90a kernels of the BigCLAM hot path (one warp per node).
//
// What one launch of step_kernel computes, per node u (reference: codes/bigclam4-7.scala):
//   PRE   :157-169  x_uv = fu.fv, p = clamp(exp(-x)), grad_u = sum_v fv/(1-p) - sumF + fu,
//                   llh_u = sum_v (log(1-p)+x) - fu.sumF + fu.fu
//   LS    :172-182  16 candidates s_j, nf_j = clamp(fu + s_j*grad), Armijo test, max passing s
//   SWAP  :183-190  F_out[u] = nf_{j*} (or fu when nothing passes)  — Jacobi: only F_in is read
//   partial reductions for :191-192 (sum over accepted nodes of old - new rows) and for the LLH
//   (sum_u llh_u == the LLH the previous call returns, :196-219).
//
// Layout: F is n x ld fp64 row-major, ld = K rounded up to a multiple of 4 (32-byte sectors,
// 16-byte double2 loads); padding columns are zero and stay zero.  Lane l of the warp owns the
// double2 chunks q = l + 32c (components 2q, 2q+1), so a row load is C2 coalesced LDG.128.
//
// Memory pipeline: nodes are visited hubs-first through a packed 16-byte NodeMeta record handed
// out by an atomic work counter two nodes ahead.  Neighbour rows arrive in batches of R (4 for K <= 256)
// through a per-warp shared-memory staging buffer filled by cp.async (LDGSTS): while batch k is processed
// from registers, batch k+1 — or, during the line search, the next node's first batch — is in flight, so
// the HBM latency of the gather is off the dependent chain.  (L2 prefetches, per line or TMA bulk, were
// measured useless-to-harmful here and are not used.)
//
// Hubs: nodes whose serial chain would dominate a launch are processed by whole blocks, very large ones
// by several blocks in three ordered phases (hub_phase below).
//
// Line search ("pair list"): a component can only matter in nf_j . fv if nf_j can be non-zero,
// i.e. fu_i > 0 or grad_i > 0 (MIN_F_ = 0).  Those m "active" components are compacted into shared
// memory; for every edge the warp gathers fv at the active components with one LDG per 32 of them
// and keeps only the non-zero products' operands (t, fv_t) — typically ~3 per edge.  Lanes then
// re-map to (trial j, edge parity) and each lane accumulates its own trial's dot over the pairs
// and evaluates exp/log for it: every point of the 16 x deg grid is computed by exactly one lane.
// Rows with more active components than the shared-memory lists hold, or MIN_F_ != 0, take the
// dense path (lane-owned components, one candidate at a time, early exit).
//
// exp/log: the clamped edge term is only evaluated for x in (x_lo, x_hi) = (-log MAX_P, -log MIN_P)
// (outside, the clamp makes it a constant + x), so exp(-x) and log(1-p) see a small, benign domain
// and are written branch-free here (Estrin evaluation; <= 2 ulp, see the NumPy twin of these formulas in
// tests/test_explog_twin.py) instead of paying for libdevice's special-case handling.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bigclam {

constexpr int kWarpsPerBlock = 6;      // 12 warps/SM at ~168 registers: the point where ptxas stops spilling
constexpr int kBlockThreads = kWarpsPerBlock * 32;
constexpr int kHubDegree = 48;      // floor of the degree from which a node is shared by the warps of a block
constexpr int kMaxSteps = 64;       // MaxInter + 1 <= kMaxSteps
constexpr int kMaxActiveCap = 256;  // upper bound of the active-set lists (and of pair-list t)
constexpr int kMaxPairs = 512;      // capacity of the pair list of one line-search chunk (<= 32 edges)

struct NodeMeta {   // one record per visited node, in processing order
    int32_t u;
    int32_t deg;
    int64_t e0;
};

struct HubItem;
struct StepArgs {
    int64_t n;
    const int64_t *rowptr;
    const int32_t *col;
    const double *F_in;
    double *F_out;
    const double *sumF;
    int32_t k, ld;
    int32_t nsteps;
    int32_t maxm;             // capacity of the active-set / pair lists (per warp)
    double steps[kMaxSteps];
    double alpha, min_p, max_p, min_f, max_f;
    // thresholds/constants of the clamped edge term (exact shortcuts, see edge_term)
    double x_lo, x_hi, t_lo, t_hi, w_lo, w_hi;
    const NodeMeta *meta;     // processing order (degree descending) over the owned nodes
    int64_t order_n;
    int32_t n_hubs;           // the first n_hubs positions are hub nodes (skipped by the warp-per-node loop)
    int32_t n_hub_items;      // block-cooperative work items over those hubs (see hub_phase)
    const struct HubItem *hub_items;
    double *hub_scratch;
    unsigned int *hub_counters;
    unsigned int *work_counter;   // next position to hand out (host sets it to 4 * #warps)
    const uint8_t *node_mask; // optional uset
    double *partials;         // [D(ld) = sum(old - new) | unused(ld) | llh | n_updated]
    int8_t *accepted;         // optional, n
    const int32_t *done_flag; // optional: non-zero -> the launch is a no-op
    int32_t do_linesearch;    // 0: PRE/LLH only (loglikelihood())
    // node-partitioned multi-GPU: replicas of F_out on the other GPUs of the box (peer memory over
    // NVLink, opened through CUDA IPC).  A row is pushed to every peer when this step or the previous one
    // changed it (the previous one makes the peers' copy in this half of the double buffer stale).
    int32_t n_peers;
    double *peer_out[7];
    int8_t *changed;          // n: 1 if the node's row changed in the most recent step (read: previous step)
    long long *dbg;           // optional debug scratch (unused in this build)
};

// Shared-memory carve-up.  Everything whose size does not depend on K sits at compile-time offsets
// (so the compiler never recomputes list pointers from kernel parameters inside the loops):
//   block: steps[kMaxSteps] f64 | kWarpsPerBlock x WarpLists | sumF[ld] f64 | kWarpsPerBlock x D[ld] f64
struct __align__(16) WarpLists {
    double2 afg[kMaxActiveCap];          // (fu_t, g_t) of the active components
    double pval[kMaxPairs];              // pair list: fv value
    unsigned short aidx[kMaxActiveCap];  // component index of active t
    unsigned short poff[40];             // pair-list offsets per edge of the chunk (33 used)
    unsigned char pt[kMaxPairs];         // pair list: active index t
};
// Rows per staged batch (the R of step_kernel) for a row of C2 double2 chunks per lane.
template <int C2>
struct RowsInFlight { static constexpr int value = (C2 <= 4) ? 4 : (C2 <= 8 ? 2 : 1); };
__host__ __device__ inline size_t block_smem_bytes(int ld, int /*maxm*/) {
    const int stage = (ld <= 256) ? RowsInFlight<4>::value : (ld <= 512 ? RowsInFlight<8>::value : RowsInFlight<16>::value);
    // ... | sumF[ld] | W x D[ld] | W x rows[4][ld] (cp.async staging of one batch of neighbour rows)
    return sizeof(double) * kMaxSteps + (size_t)kWarpsPerBlock * sizeof(WarpLists) +
           sizeof(double) * (size_t)ld * (1 + kWarpsPerBlock + stage * kWarpsPerBlock);
}

__device__ __forceinline__ double fmax2(double a, double b) { return a > b ? a : b; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double2 ldg2(const double *p) {
    return __ldg(reinterpret_cast<const double2 *>(p));
}

// ---------------------------------------------------------------------------------------------
// exp(-x) for x in (0, ~9.3): n = rint(-x log2 e), r = -x - n ln2 (two-step FMA reduction),
// degree-13 Taylor of e^r on |r| <= ln2/2 (truncation 4e-18), scale by adding n to the exponent.
__device__ __forceinline__ double exp_neg(double x) {
    const double kMagic = 6755399441055744.0;                       // 1.5 * 2^52
    const double t = fma(-x, 1.4426950408889634, kMagic);
    const int n = __double2loint(t);
    const double nf = t - kMagic;
    double r = fma(nf, -0.6931471805599453094, -x);
    r = fma(nf, -2.3190468138462996e-17, r);
    // Estrin evaluation (depth 4 instead of 13 dependent FMAs)
    const double r2 = r * r, r4 = r2 * r2, r8 = r4 * r4;
    const double a0 = r + 1.0;
    const double a1 = fma(0.16666666666666666, r, 0.5);
    const double a2 = fma(0.008333333333333333, r, 0.041666666666666664);
    const double a3 = fma(0.0001984126984126984, r, 0.001388888888888889);
    const double a4 = fma(2.7557319223985893e-06, r, 2.48015873015873e-05);
    const double a5 = fma(2.505210838544172e-08, r, 2.755731922398589e-07);
    const double a6 = fma(1.6059043836821613e-10, r, 2.08767569878681e-09);
    const double b0 = fma(a1, r2, a0), b1 = fma(a3, r2, a2), b2 = fma(a5, r2, a4);
    const double d0 = fma(b1, r4, b0), d1 = fma(a6, r4, b2);
    const double p = fma(d1, r8, d0);
    return __hiloint2double(__double2hiint(p) + (n << 20), __double2loint(p));
}

// 1/d for normal positive d: rcp.approx (2^-23) + two Newton steps.
__device__ __forceinline__ double rcp_pos(double d) {
    double y;
#ifdef BIGCLAM_EMU          // host emulation of the kernels (tests/emu): no PTX, same accuracy class of the seed
    y = (double)(1.0f / (float)d);
#else
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
#endif
    double e = fma(-d, y, 1.0);
    y = fma(y, e, y);
    e = fma(-d, y, 1.0);
    return fma(y, e, y);
}

// log(y) for normal y in (0, 1]: y = 2^e m, m in [sqrt(1/2), sqrt 2], s = (m-1)/(m+1),
// log m = 2s + s z (2/3 + 2/5 z + ... + 2/23 z^10), z = s^2 <= 0.0295 (truncation 6e-19).
__device__ __forceinline__ double log_pos(double y) {
    const int hi = __double2hiint(y);
    int e = (hi >> 20) - 1023;
    int mh = (hi & 0x000fffff) | 0x3ff00000;
    if (mh > 0x3ff6a09e) { mh -= 0x00100000; e += 1; }
    const double m = __hiloint2double(mh, __double2loint(y));
    const double f = m - 1.0, d = m + 1.0;
    const double rd = rcp_pos(d);
    double s = f * rd;
    s = fma(fma(-d, s, f), rd, s);
    const double z = s * s;
    const double z2 = z * z, z4 = z2 * z2, z8 = z4 * z4;
    const double a0 = fma(0.4, z, 0.6666666666666666);                     // 2/5, 2/3
    const double a1 = fma(0.2222222222222222, z, 0.2857142857142857);      // 2/9, 2/7
    const double a2 = fma(0.15384615384615385, z, 0.18181818181818182);    // 2/13, 2/11
    const double a3 = fma(0.11764705882352941, z, 0.13333333333333333);    // 2/17, 2/15
    const double a4 = fma(0.09523809523809523, z, 0.10526315789473684);    // 2/21, 2/19
    const double b0 = fma(a1, z2, a0), b1 = fma(a3, z2, a2), b2 = fma(0.08695652173913043, z2, a4);   // 2/23
    const double q = fma(b2, z8, fma(b1, z4, b0));
    const double ed = (double)e;
    const double inner = fma(ed, 2.3190468138462996e-17, (s * z) * q);
    return fma(ed, 0.6931471805599453094, fma(2.0, s, inner));
}

// Constants of the clamped edge term kept in registers.
struct EdgeConst {
    double x_lo, x_hi, t_lo, t_hi, w_lo, w_hi;
};

// log(1 - clamp(exp(-x), MIN_P, MAX_P)) + x and 1/(1 - p)   (bigclam4-7.scala:166-167).
// Exact shortcuts: x <= x_lo gives p == MAX_P after the clamp, x >= x_hi gives p == MIN_P
// (x_lo/x_hi carry a 1e-12 safety margin so the clamp outcome is never in doubt); in between the
// clamp is a no-op.  Must be called by all 32 lanes (warp-uniform skip of the transcendental).
template <bool kNeedW>
__device__ __forceinline__ double edge_term(double x, const EdgeConst &c, double &w) {
    const bool low = x <= c.x_lo;
    const bool need = !low && (x < c.x_hi);
    double t = low ? c.t_lo : c.t_hi;
    if (kNeedW) w = low ? c.w_lo : c.w_hi;
    if (__any_sync(0xffffffffu, need)) {
        const double xs = need ? x : 1.0;
        const double omp = 1.0 - exp_neg(xs);
        const double tf = log_pos(omp);
        t = need ? tf : t;
        if (kNeedW) {
            const double wf = rcp_pos(omp);
            w = need ? wf : w;
        }
    }
    return t + x;
}

// Two independent edge terms per lane (ILP 2): same arithmetic as edge_term<false>.
__device__ __forceinline__ void edge_term2(double xa, double xb, const EdgeConst &c, double &ta, double &tb) {
    const bool lowa = xa <= c.x_lo, lowb = xb <= c.x_lo;
    const bool needa = !lowa && (xa < c.x_hi), needb = !lowb && (xb < c.x_hi);
    ta = lowa ? c.t_lo : c.t_hi;
    tb = lowb ? c.t_lo : c.t_hi;
    if (__any_sync(0xffffffffu, needa || needb)) {
        const double ompa = 1.0 - exp_neg(needa ? xa : 1.0);
        const double ompb = 1.0 - exp_neg(needb ? xb : 1.0);
        const double fa = log_pos(ompa);
        const double fb = log_pos(ompb);
        ta = needa ? fa : ta;
        tb = needb ? fb : tb;
    }
    ta += xa;
    tb += xb;
}

// step(), bigclam4-7.scala:110-113: product and sum rounded separately (the JVM never fuses).
__device__ __forceinline__ double clamp_step(double f, double s, double g, double lo, double hi) {
    double x = __dadd_rn(f, __dmul_rn(s, g));
    x = (x < lo) ? lo : x;
    return (x > hi) ? hi : x;
}
// Same with MIN_F_ == 0: the lower clamp is a sign test (also maps -0.0 to +0.0 like Math.max).
__device__ __forceinline__ double clamp_step0(double f, double s, double g, double hi) {
    double x = __dadd_rn(f, __dmul_rn(s, g));
    x = (__double2hiint(x) < 0) ? 0.0 : x;
    return (x > hi) ? hi : x;
}

// Lower clamp only (used when no active component of the node can reach MAX_F_ at step 1).
__device__ __forceinline__ double clamp_step0_lo(double f, double s, double g) {
    const double x = __dadd_rn(f, __dmul_rn(s, g));
    return (__double2hiint(x) < 0) ? 0.0 : x;
}

// cp.async staging of up to 4 neighbour rows (edges first .. first+3 of the id register `ids`) into the
// warp's shared-memory row buffer; lane l copies the same 16-byte chunks it later reads back.
#ifdef BIGCLAM_EMU          // host emulation (tests/emu): the copy happens at once
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) { memcpy(smem_dst, gsrc, 16); }
__device__ __forceinline__ void cp_async_commit() {}
__device__ __forceinline__ void cp_async_wait_all() {}
#else
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
#endif
template <int C2, int RB>
__device__ __forceinline__ void stage_rows(double *buf, const double *__restrict__ F, int ld, int ld2, int lane,
                                           int ids, int first, int cnt) {
#pragma unroll
    for (int r = 0; r < RB; ++r) {
        const int e = first + r;
        const int v = __shfl_sync(0xffffffffu, ids, e & 31);
        if (e < cnt) {
            const double *fv = F + (size_t)v * ld;
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) cp_async16(buf + r * ld + 2 * q, fv + 2 * q);
            }
        }
    }
    cp_async_commit();
}

// Transposed butterfly over RB per-lane partials (RB = 4, 2 or 1): afterwards the lanes of group
// r = lane / (32 / RB) hold the warp total of part[r].
template <int RB>
__device__ __forceinline__ double batch_reduce(const double (&part)[RB], int lane) {
    double kx;
    if constexpr (RB == 4) {
        const bool b4 = lane & 16, b3 = lane & 8;
        double k0 = b4 ? part[2] : part[0], k1 = b4 ? part[3] : part[1];
        const double s0 = b4 ? part[0] : part[2], s1 = b4 ? part[1] : part[3];
        k0 += __shfl_xor_sync(0xffffffffu, s0, 16);
        k1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        kx = b3 ? k1 : k0;
        const double sd = b3 ? k0 : k1;
        kx += __shfl_xor_sync(0xffffffffu, sd, 8);
    } else if constexpr (RB == 2) {
        const bool b4 = lane & 16;
        kx = b4 ? part[1] : part[0];
        const double sd = b4 ? part[0] : part[1];
        kx += __shfl_xor_sync(0xffffffffu, sd, 16);
        kx += __shfl_xor_sync(0xffffffffu, kx, 8);
    } else {
        kx = part[0];
        kx += __shfl_xor_sync(0xffffffffu, kx, 16);
        kx += __shfl_xor_sync(0xffffffffu, kx, 8);
    }
    kx += __shfl_xor_sync(0xffffffffu, kx, 4);
    kx += __shfl_xor_sync(0xffffffffu, kx, 2);
    kx += __shfl_xor_sync(0xffffffffu, kx, 1);
    return kx;
}

// Sum R per-lane partials across the warp; the total of partial r is returned to lane (eb + r).
template <int R>
__device__ __forceinline__ double reduce_to_lanes(double (&part)[R], int lane, int eb, double myx) {
    if constexpr (R == 4) {
        // transposed butterfly: 6 shuffles instead of 20
        const bool b4 = lane & 16, b3 = lane & 8;
        double k0 = b4 ? part[2] : part[0], k1 = b4 ? part[3] : part[1];
        const double s0 = b4 ? part[0] : part[2], s1 = b4 ? part[1] : part[3];
        k0 += __shfl_xor_sync(0xffffffffu, s0, 16);
        k1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        double k = b3 ? k1 : k0;
        const double sd = b3 ? k0 : k1;
        k += __shfl_xor_sync(0xffffffffu, sd, 8);
        k += __shfl_xor_sync(0xffffffffu, k, 4);
        k += __shfl_xor_sync(0xffffffffu, k, 2);
        k += __shfl_xor_sync(0xffffffffu, k, 1);
        // total of part[r] now sits in the lanes with (bit4, bit3) == (r >> 1, r & 1)
        const int r = (lane - eb) & 3;
        const double got = __shfl_sync(0xffffffffu, k, ((r & 2) << 3) | ((r & 1) << 3));
        return ((unsigned)(lane - eb) < 4u) ? got : myx;
    } else {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
            for (int r = 0; r < R; ++r) part[r] += __shfl_xor_sync(0xffffffffu, part[r], o);
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
            if (lane == eb + r) myx = part[r];
        return myx;
    }
}

// Dots of `vec` (lane-owned components) with the rows of up to 32 neighbours; lane e returns
// the dot for neighbour e of the chunk.  R rows are in flight per batch.
template <int C2, int R>
__device__ __forceinline__ double chunk_dots(const double2 (&vec)[C2], const double *__restrict__ F,
                                             int ld, int ld2, int lane, int myv, int cnt) {
    double myx = 0.0;
    for (int eb = 0; eb < cnt; eb += R) {
        double part[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int e = eb + r;
            const int v = __shfl_sync(0xffffffffu, myv, e & 31);
            const double *fv = F + (size_t)v * ld;
            double p = 0.0;
            if (e < cnt) {
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
                    if (q < ld2) {
                        const double2 x = ldg2(fv + 2 * q);
                        p = fma(vec[c].x, x.x, p);
                        p = fma(vec[c].y, x.y, p);
                    }
                }
            }
            part[r] = p;
        }
        myx = reduce_to_lanes<R>(part, lane, eb, myx);
    }
    return myx;
}

// Line search, edge range [ebeg, eend) of one node: per-lane sum over the range's edges e = (chunk edge)
// with parity h of  log(1 - clamp(exp(-nf_j . fv_e))) + nf_j . fv_e  for the lane's own trial j (step s).
// Builds the (t, fv_t) pair lists of up to 32 edges at a time in the warp's shared memory, then walks them.
struct LsLists {
    double2 *afg;
    double *pval;
    unsigned short *aidx;
    unsigned short *poff;
    unsigned char *pt;
};
__device__ __forceinline__ double ls_edge_range(const double *__restrict__ F, const int32_t *__restrict__ colp,
                                                int ebeg, int eend, int ld, int m, int my_idx0, unsigned lt_mask,
                                                int lane, int h, double s, bool need_hi, double max_f,
                                                const EdgeConst &ec, const LsLists &L) {
    double2 *s_afg = L.afg;
    double *s_pval = L.pval;
    unsigned short *s_aidx = L.aidx;
    unsigned short *s_poff = L.poff;
    unsigned char *s_pt = L.pt;
    const int mdiv = max(m, 1);
    double sumterms = 0.0;
    // groups of 32 edges (one coalesced load of neighbour ids), split into chunks whose
    // pairs fit the list
    for (int gb = ebeg; gb < eend; gb += 32) {
      const int gcnt = min(32, eend - gb);
      const int cv = (lane < gcnt) ? colp[gb + lane] : 0;
      int ge = 0;
      while (ge < gcnt) {
        int np = 0, ce = 0;
        if (lane == 0) s_poff[0] = 0;
        // build: for every edge keep (t, fv[idx_t]) with fv != 0
        if (m <= 32) {
            while (ge + ce < gcnt) {
                int nb = min(4, gcnt - ge - ce);
                if (np + nb * m > kMaxPairs) {
                    nb = (kMaxPairs - np) / mdiv;
                    if (nb == 0) break;
                }
                double val[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) {          // up to 4 gathers in flight
                    const int v = __shfl_sync(0xffffffffu, cv, (ge + ce + r) & 31);
                    val[r] = (r < nb && lane < m) ? __ldg(F + (size_t)v * ld + my_idx0) : 0.0;
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (r < nb) {
                        const unsigned bal = __ballot_sync(0xffffffffu, val[r] != 0.0);
                        if (val[r] != 0.0) {
                            const int pp = np + __popc(bal & lt_mask);
                            s_pval[pp] = val[r];
                            s_pt[pp] = (unsigned char)lane;
                        }
                        np += __popc(bal);
                        if (lane == 0) s_poff[ce + r + 1] = (unsigned short)np;
                    }
                }
                ce += nb;
            }
        } else {
            // hubs / dense rows: up to 8 gather rounds per edge, all issued before the ballots;
            // the list is filled optimistically and the last edge rolled back if it overflows
            while (ge + ce < gcnt) {
                const int v = __shfl_sync(0xffffffffu, cv, (ge + ce) & 31);
                const double *fv = F + (size_t)v * ld;
                double vv[kMaxActiveCap / 32];
#pragma unroll
                for (int r = 0; r < kMaxActiveCap / 32; ++r) {
                    const int t = 32 * r + lane;
                    vv[r] = (t < m) ? __ldg(fv + s_aidx[t]) : 0.0;
                }
                const int np0 = np;
#pragma unroll
                for (int r = 0; r < kMaxActiveCap / 32; ++r) {
                    if (32 * r < m) {
                        const unsigned bal = __ballot_sync(0xffffffffu, vv[r] != 0.0);
                        if (vv[r] != 0.0) {
                            const int pp = np + __popc(bal & lt_mask);
                            if (pp < kMaxPairs) {
                                s_pval[pp] = vv[r];
                                s_pt[pp] = (unsigned char)(32 * r + lane);
                            }
                        }
                        np += __popc(bal);
                    }
                }
                if (np > kMaxPairs) { np = np0; break; }      // does not fit: flush first
                if (lane == 0) s_poff[ce + 1] = (unsigned short)np;
                ++ce;
            }
        }
        __syncwarp();
        // consume: lane (j, h) walks the pairs of edges e2 + h and e2 + 2 + h together (two independent
        // LDS -> clamp -> FMA chains in flight, then two exp/log chains)
#pragma unroll 1
        for (int e2 = 0; e2 < ce; e2 += 4) {
            const int eA = e2 + h, eB = e2 + 2 + h;
            const bool vA = eA < ce, vB = eB < ce;
            const int iA = vA ? (int)s_poff[eA] : 0, nA = vA ? (int)s_poff[eA + 1] - iA : 0;
            const int iB = vB ? (int)s_poff[eB] : 0, nB = vB ? (int)s_poff[eB + 1] - iB : 0;
            const int nmax = max(nA, nB);
            double DA = 0.0, DB = 0.0;
#pragma unroll 1
            for (int k = 0; k < nmax; ++k) {
                const bool ka = k < nA, kb = k < nB;
                const int ia = ka ? iA + k : 0, ib = kb ? iB + k : 0;        // entry 0 is always readable
                const double2 fa = s_afg[s_pt[ia]], fb = s_afg[s_pt[ib]];
                const double pa = ka ? s_pval[ia] : 0.0, pb = kb ? s_pval[ib] : 0.0;
                if (need_hi) {
                    DA = fma(clamp_step0(fa.x, s, fa.y, max_f), pa, DA);
                    DB = fma(clamp_step0(fb.x, s, fb.y, max_f), pb, DB);
                } else {
                    DA = fma(clamp_step0_lo(fa.x, s, fa.y), pa, DA);
                    DB = fma(clamp_step0_lo(fb.x, s, fb.y), pb, DB);
                }
            }
            double tA, tB;
            edge_term2(DA, DB, ec, tA, tB);
            sumterms += vA ? tA : 0.0;
            sumterms += vB ? tB : 0.0;
        }
        __syncwarp();
        ge += ce;
      }
    }
    return sumterms;
}

// Dense line search (cold path): lane-owned components, candidates in descending order, early exit.
// fu is re-read from F_in and the gradient from `grow` (the caller parks it in the node's F_out row,
// which it owns and overwrites afterwards) so that no register array has its address taken.
template <int C2, int R>
__device__ __noinline__ int dense_linesearch(const double *__restrict__ F, const int32_t *__restrict__ colp,
                                             int ld, int nsteps, const double *s_steps, double alpha,
                                             double min_f, double max_f, EdgeConst ec,
                                             const double *frow, const double *grow,
                                             const double *s_sumF, int deg, int lane,
                                             double llh_u, double G2) {
    const int ld2 = ld >> 1;
    for (int j = 0; j < nsteps; ++j) {
        const double s = s_steps[j];
        double2 nf[C2];
        double oa = 0.0, ob = 0.0;
#pragma unroll
        for (int c = 0; c < C2; ++c) {
            const int q = lane + 32 * c;
            nf[c] = make_double2(0.0, 0.0);
            if (q < ld2) {
                const double2 sf = *reinterpret_cast<const double2 *>(s_sumF + 2 * q);
                const double2 fu = ldg2(frow + 2 * q);
                const double2 g = *reinterpret_cast<const double2 *>(grow + 2 * q);
                nf[c].x = clamp_step(fu.x, s, g.x, min_f, max_f);
                nf[c].y = clamp_step(fu.y, s, g.y, min_f, max_f);
                oa = fma(nf[c].x, (sf.x - fu.x) + nf[c].x, oa);
                oa = fma(nf[c].y, (sf.y - fu.y) + nf[c].y, oa);
                ob = fma(nf[c].x, nf[c].x, ob);
                ob = fma(nf[c].y, nf[c].y, ob);
            }
        }
        oa = warp_sum(oa);
        ob = warp_sum(ob);
        double sumterms = 0.0;
        for (int cb = 0; cb < deg; cb += 32) {
            const int cnt = min(32, deg - cb);
            const int myv = (lane < cnt) ? colp[cb + lane] : 0;
            const double myx = chunk_dots<C2, R>(nf, F, ld, ld2, lane, myv, cnt);
            double w;
            const double t = edge_term<false>(myx, ec, w);
            sumterms += warp_sum(lane < cnt ? t : 0.0);
        }
        const double result = (sumterms - oa) + ob;
        const double rhs = llh_u + (alpha * s) * G2;
        if (result >= rhs) return j;
    }
    return -1;
}

// ------------------------------------------------------------------------------------------------
// Hub phase: high-degree nodes are shared by the warps of a BLOCK, very high-degree ones by several blocks.
// A node's edges are independent in PRE (sum over edges) and in the line search (sum over edges per
// trial), so the warps take contiguous slices of the neighbour list, exchange the partial gradient / the
// partial per-trial sums through shared memory, and every warp redundantly derives the (identical)
// gradient, active set and decision; warp 0 writes the row.
//
// Work items (host-built, processed by block b in the order b, b + grid, ...):
//   phase 0  a hub of at most kHubSlice edges, done completely by one block;
//   phase 1  PRE of one kHubSlice-edge slice of a mega hub -> partial gradient / S1 added to global scratch;
//   phase 2  line search of one slice (waits until all phase-1 slices of the hub are in) -> partial
//            per-trial sums added to global scratch;
//   phase 3  decision + row write of a mega hub (waits for its phase-2 slices).
// All phase-1 items precede all phase-2 items precede all phase-3 items and the grid is persistent (every
// block resident), so a waiting block only ever waits for items that are being processed: no deadlock.
constexpr int kHubSlice = 384;

struct HubItem {
    int32_t hub;      // position in meta[]
    int32_t slice;    // slice index (phases 1, 2)
    int32_t phase;
    int32_t mslot;    // scratch / counter slot of the mega hub (0 for phase-0 hubs)
    int32_t nslices;
    int32_t seg;      // edges per slice (sparse engine: kSpHubSeg, more for very large hubs)
    int32_t pad[2];
};

struct HubArgs {
    const NodeMeta *meta;
    const int32_t *col;
    const double *F_in;
    double *F_out;
    const uint8_t *node_mask;
    int8_t *accepted;
    int8_t *changed;
    double *peer_out[7];
    const HubItem *items;
    double *scratch;            // per mega hub: G[ld] | S1 | ST[16] | pad  (stride ld + 32 doubles)
    unsigned int *counters;     // per mega hub: [phase-1 slices done, phase-2 slices done]
    int32_t n_peers, n_items, ld, nsteps, do_linesearch;
    double alpha, min_f, max_f;
};

__device__ __forceinline__ void hub_wait(const unsigned int *counter, unsigned int target) {
    if (threadIdx.x == 0) {
        while (*reinterpret_cast<const volatile unsigned int *>(counter) < target) __nanosleep(200);
        __threadfence();
    }
    __syncthreads();
}

template <int C2>
__device__ __noinline__ void hub_phase(const HubArgs ha, const EdgeConst ec, const double *s_sumF, const double *s_steps,
                                       double *s_D, double *s_rows_all, const LsLists lists, double *hub_small,
                                       double *llh_acc_io, double *nupd_acc_io) {
    const int ld = ha.ld, ld2 = ha.ld >> 1;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    const double *__restrict__ F = ha.F_in;
    double *my_part = s_rows_all + (size_t)wib * 4 * ld;           // this warp's partial gradient
    double *hub_S1 = hub_small;                                     // [kWarpsPerBlock]
    double *hub_st = hub_small + kWarpsPerBlock;                    // [kWarpsPerBlock][32]
    int *hub_j = reinterpret_cast<int *>(hub_small + kWarpsPerBlock * 33);
    const double max_f = ha.max_f;
    const int j16 = lane & 15, h = lane >> 4;

    for (int it = blockIdx.x; it < ha.n_items; it += gridDim.x) {
        const HubItem item = ha.items[it];
        const int phase = item.phase;
        const NodeMeta nm = ha.meta[item.hub];
        const int64_t u = nm.u, e0 = nm.e0;
        const int deg = nm.deg;
        const int32_t *colp = ha.col + e0;
        double *scr = ha.scratch + (size_t)item.mslot * (ld + 32);
        unsigned int *cnt = ha.counters + 2 * (size_t)item.mslot;
        // edge range of this item, then of this warp inside it
        const int blk_beg = (phase == 1 || phase == 2) ? item.slice * kHubSlice : 0;
        const int blk_end = (phase == 1 || phase == 2) ? min(deg, blk_beg + kHubSlice) : deg;
        const int per = ((((blk_end - blk_beg) + kWarpsPerBlock - 1) / kWarpsPerBlock) + 3) & ~3;
        const int ebeg = min(blk_end, blk_beg + wib * per), eend = min(blk_end, ebeg + per);

        double2 fu[C2];
        double fusf = 0.0, fufu = 0.0;
#pragma unroll
        for (int c = 0; c < C2; ++c) {
            const int q = lane + 32 * c;
            fu[c] = (q < ld2) ? ldg2(F + (size_t)u * ld + 2 * q) : make_double2(0.0, 0.0);
            if (q < ld2) {
                const double2 sf = *reinterpret_cast<const double2 *>(s_sumF + 2 * q);
                fusf = fma(fu[c].x, sf.x, fusf); fusf = fma(fu[c].y, sf.y, fusf);
                fufu = fma(fu[c].x, fu[c].x, fufu); fufu = fma(fu[c].y, fu[c].y, fufu);
            }
        }
        fusf = warp_sum(fusf);
        fufu = warp_sum(fufu);

        double2 g[C2];
#pragma unroll
        for (int c = 0; c < C2; ++c) g[c] = make_double2(0.0, 0.0);
        double S1 = 0.0;

        if (phase <= 1) {
            // ---- PRE over this warp's slice: batches of 4 rows through the warp's cp.async staging buffer
            // (the same buffer later carries this warp's partial gradient), next batch in flight ----
            const int rsel = (lane >> 3) & 3;
            int gb = ebeg;
            int cnt32 = min(32, max(0, eend - gb));
            int myv = (lane < cnt32) ? colp[gb + lane] : 0;
            if (cnt32 > 0) stage_rows<C2, 4>(my_part, F, ld, ld2, lane, myv, 0, cnt32);
            while (gb < eend) {
                const int cnt2 = min(32, max(0, eend - gb - 32));
                const int myv2 = (lane < cnt2) ? colp[gb + 32 + lane] : 0;
                for (int eb = 0; eb < cnt32; eb += 4) {
                    cp_async_wait_all();
                    __syncwarp();
                    double2 x[4][C2];
                    double part[4];
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const bool ok = eb + r < cnt32;
                        double p = 0.0;
#pragma unroll
                        for (int c = 0; c < C2; ++c) {
                            const int q = lane + 32 * c;
                            x[r][c] = (ok && q < ld2) ? *reinterpret_cast<const double2 *>(my_part + r * ld + 2 * q)
                                                      : make_double2(0.0, 0.0);
                            p = fma(fu[c].x, x[r][c].x, p);
                            p = fma(fu[c].y, x[r][c].y, p);
                        }
                        part[r] = p;
                    }
                    __syncwarp();
                    if (eb + 4 < cnt32) stage_rows<C2, 4>(my_part, F, ld, ld2, lane, myv, eb + 4, cnt32);
                    else if (cnt2 > 0) stage_rows<C2, 4>(my_part, F, ld, ld2, lane, myv2, 0, cnt2);
                    const double kx = batch_reduce<4>(part, lane);
                    double w;
                    double t = edge_term<true>(kx, ec, w);
                    t = (eb + rsel < cnt32) ? t : 0.0;
                    t += __shfl_xor_sync(0xffffffffu, t, 8);
                    t += __shfl_xor_sync(0xffffffffu, t, 16);
                    S1 += t;
                    if (ha.do_linesearch) {
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const double we = __shfl_sync(0xffffffffu, w, 8 * r);
#pragma unroll
                            for (int c = 0; c < C2; ++c) {
                                g[c].x = fma(we, x[r][c].x, g[c].x);
                                g[c].y = fma(we, x[r][c].y, g[c].y);
                            }
                        }
                    }
                }
                gb += 32;
                cnt32 = cnt2;
                myv = myv2;
            }
            __syncwarp();
            // ---- combine the partial gradient and S1 over the block ----
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) *reinterpret_cast<double2 *>(my_part + 2 * q) = g[c];
            }
            if (lane == 0) hub_S1[wib] = S1;
            __syncthreads();
            S1 = 0.0;
#pragma unroll
            for (int c = 0; c < C2; ++c) g[c] = make_double2(0.0, 0.0);
            for (int w = 0; w < kWarpsPerBlock; ++w) {
                S1 += hub_S1[w];
                const double *pw = s_rows_all + (size_t)w * 4 * ld;
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
                    if (q < ld2) {
                        const double2 v = *reinterpret_cast<const double2 *>(pw + 2 * q);
                        g[c].x += v.x;
                        g[c].y += v.y;
                    }
                }
            }
            __syncthreads();
            if (phase == 1) {
                // publish this slice's partial sums, then signal
                if (wib == 0) {
#pragma unroll
                    for (int c = 0; c < C2; ++c) {
                        const int q = lane + 32 * c;
                        if (q < ld2) {
                            atomicAdd(scr + 2 * q, g[c].x);
                            atomicAdd(scr + 2 * q + 1, g[c].y);
                        }
                    }
                    if (lane == 0) atomicAdd(scr + ld, S1);
                    __threadfence();
                }
                __syncthreads();
                if (threadIdx.x == 0) atomicAdd(cnt, 1u);
                continue;
            }
        } else {
            // phases 2 and 3: the whole node's gradient sum and S1 come from the scratch
            hub_wait(cnt + (phase == 2 ? 0 : 1), (unsigned int)item.nslices);
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) g[c] = __ldcg(reinterpret_cast<const double2 *>(scr + 2 * q));
            }
            S1 = __ldcg(scr + ld);
        }

        const double llh_u = (S1 - fusf) + fufu;
        const bool in_uset = (ha.node_mask == nullptr) || (ha.node_mask[u] != 0);
        int jstar = -1;
        if (ha.do_linesearch && in_uset) {
            double G2 = 0.0;
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) {
                    const double2 sf = *reinterpret_cast<const double2 *>(s_sumF + 2 * q);
                    g[c].x = (g[c].x - sf.x) + fu[c].x;
                    g[c].y = (g[c].y - sf.y) + fu[c].y;
                    G2 = fma(g[c].x, g[c].x, G2);
                    G2 = fma(g[c].y, g[c].y, G2);
                }
            }
            G2 = warp_sum(G2);
            int m = 0;
            const bool sparse_ok = (ha.min_f == 0.0);
            if (sparse_ok) {
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const double fval = hh ? fu[c].y : fu[c].x;
                        const double gval = hh ? g[c].y : g[c].x;
                        const bool act = (q < ld2) && (fval > 0.0 || gval > 0.0);
                        const unsigned bal = __ballot_sync(0xffffffffu, act);
                        if (bal) {
                            if (act) {
                                const int posn = m + __popc(bal & lt_mask);
                                if (posn < kMaxActiveCap) {
                                    lists.afg[posn] = make_double2(fval, gval);
                                    lists.aidx[posn] = (unsigned short)(2 * q + hh);
                                }
                            }
                            m += __popc(bal);
                        }
                    }
                }
                __syncwarp();
            }
            if (sparse_ok && m <= kMaxActiveCap) {
                const int my_idx0 = (lane < m) ? (int)lists.aidx[lane] : 0;
                bool hi_lane = false;
                for (int t = lane; t < m; t += 32) {
                    const double2 fg = lists.afg[t];
                    hi_lane |= (fg.x + fg.y > max_f);
                }
                const bool need_hi = __any_sync(0xffffffffu, hi_lane);
                // mega hubs are restricted (host side) to nsteps <= 16, i.e. a single trial group
                for (int tg = 0; tg < ha.nsteps && jstar < 0; tg += 16) {
                    const int j = tg + j16;
                    const bool jok = j < ha.nsteps;
                    const double s = s_steps[jok ? j : 0];
                    double sumterms = 0.0;
                    if (phase != 3) {
                        double st = ls_edge_range(F, colp, ebeg, eend, ld, m, my_idx0, lt_mask, lane, h, s, need_hi, max_f, ec, lists);
                        st += __shfl_xor_sync(0xffffffffu, st, 16);
                        hub_st[wib * 32 + lane] = st;
                        __syncthreads();
                        for (int w = 0; w < kWarpsPerBlock; ++w) sumterms += hub_st[w * 32 + lane];
                        __syncthreads();
                        if (phase == 2) {
                            if (wib == 0 && lane < 16) atomicAdd(scr + ld + 1 + lane, sumterms);
                            break;
                        }
                    } else {
                        sumterms = __ldcg(scr + ld + 1 + j16);
                    }
                    double oa = 0.0, ob = 0.0;
                    for (int t = h; t < m; t += 2) {
                        const double2 fg = lists.afg[t];
                        const double nf = need_hi ? clamp_step0(fg.x, s, fg.y, max_f) : clamp_step0_lo(fg.x, s, fg.y);
                        const double sf = (s_sumF[lists.aidx[t]] - fg.x) + nf;
                        oa = fma(nf, sf, oa);
                        ob = fma(nf, nf, ob);
                    }
                    oa += __shfl_xor_sync(0xffffffffu, oa, 16);
                    ob += __shfl_xor_sync(0xffffffffu, ob, 16);
                    const double result = (sumterms - oa) + ob;
                    const double rhs = llh_u + (ha.alpha * s) * G2;
                    const unsigned pass = __ballot_sync(0xffffffffu, jok && (result >= rhs)) & 0xffffu;
                    if (pass) jstar = tg + __ffs(pass) - 1;
                }
            } else if (phase != 2) {
                // MIN_F_ != 0 or more active components than the lists hold: warp 0 runs the dense search
                double *orow = ha.F_out + (size_t)u * ld;
                if (wib == 0) {
#pragma unroll
                    for (int c = 0; c < C2; ++c) {
                        const int q = lane + 32 * c;
                        if (q < ld2) *reinterpret_cast<double2 *>(orow + 2 * q) = g[c];
                    }
                    __syncwarp();
                    const int jd = dense_linesearch<C2, 4>(F, colp, ld, ha.nsteps, s_steps, ha.alpha, ha.min_f, max_f, ec,
                                                            F + (size_t)u * ld, orow, s_sumF, deg, lane, llh_u, G2);
                    if (lane == 0) hub_j[0] = jd;
                }
                __syncthreads();
                jstar = hub_j[0];
                __syncthreads();
            }
        }
        if (phase == 2) {
            // this slice's per-trial sums are in the scratch (or there is nothing to add): signal
            __threadfence();
            __syncthreads();
            if (threadIdx.x == 0) atomicAdd(cnt + 1, 1u);
            continue;
        }
        // ---- SWAP by warp 0 (phases 0 and 3) ----
        if (wib == 0) {
            double *orow = ha.F_out + (size_t)u * ld;
            const bool push = (ha.n_peers > 0) && ha.do_linesearch && ((jstar >= 0) || (ha.changed[u] != 0));
            __syncwarp();      // every lane has read the flag before lane 0 rewrites it below
            if (ha.do_linesearch) {
                const double s = (jstar >= 0) ? s_steps[jstar] : 0.0;
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
                    if (q < ld2) {
                        double2 nr = fu[c];
                        if (jstar >= 0) {
                            nr.x = clamp_step(fu[c].x, s, g[c].x, ha.min_f, max_f);
                            nr.y = clamp_step(fu[c].y, s, g[c].y, ha.min_f, max_f);
                            double2 *pd = reinterpret_cast<double2 *>(s_D + 2 * q);
                            double2 vd = *pd;
                            vd.x += fu[c].x - nr.x;
                            vd.y += fu[c].y - nr.y;
                            *pd = vd;
                        }
                        *reinterpret_cast<double2 *>(orow + 2 * q) = nr;
                        if (push) {
                            for (int pr = 0; pr < ha.n_peers; ++pr)
                                *reinterpret_cast<double2 *>(ha.peer_out[pr] + (size_t)u * ld + 2 * q) = nr;
                        }
                    }
                }
                if (jstar >= 0) *nupd_acc_io += 1.0;
            }
            *llh_acc_io += llh_u;
            if (ha.accepted != nullptr && lane == 0) ha.accepted[u] = (int8_t)jstar;
            if (ha.n_peers > 0 && ha.do_linesearch && lane == 0) ha.changed[u] = (jstar >= 0) ? 1 : 0;
        }
        __syncthreads();
    }
}

// kHub: the launch has block-cooperative hub nodes; kPush: peers' replicas are written (multi-GPU).
// Both are compile-time so that the single-GPU, hub-free launch carries none of that code.
template <int C2, int R, bool kHub, bool kPush>
__global__ void __launch_bounds__(kBlockThreads, (C2 <= 4) ? 2 : 1) step_kernel(const StepArgs a) {
    if (a.done_flag != nullptr && *a.done_flag != 0) return;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int ld = a.ld, ld2 = a.ld >> 1;
    constexpr int maxm = kMaxActiveCap;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double *s_steps = reinterpret_cast<double *>(smem_raw);
    WarpLists *wl = reinterpret_cast<WarpLists *>(smem_raw + sizeof(double) * kMaxSteps) + wib;
    double *s_sumF = reinterpret_cast<double *>(smem_raw + sizeof(double) * kMaxSteps + kWarpsPerBlock * sizeof(WarpLists));
    double *s_D = s_sumF + (size_t)ld * (1 + wib);
    double *s_rows = s_sumF + (size_t)ld * (1 + kWarpsPerBlock) + (size_t)wib * R * ld;
    double2 *s_afg = wl->afg;
    double *s_pval = wl->pval;
    unsigned short *s_aidx = wl->aidx;
    unsigned short *s_poff = wl->poff;
    unsigned char *s_pt = wl->pt;
    const LsLists lists = {s_afg, s_pval, s_aidx, s_poff, s_pt};

    for (int i = threadIdx.x; i < ld; i += kBlockThreads) s_sumF[i] = a.sumF[i];
    for (int i = threadIdx.x; i < kMaxSteps; i += kBlockThreads) s_steps[i] = a.steps[i];
    for (int i = lane; i < ld; i += 32) s_D[i] = 0.0;
    __syncthreads();

    const EdgeConst ec = {a.x_lo, a.x_hi, a.t_lo, a.t_hi, a.w_lo, a.w_hi};
    const double max_f = a.max_f;
    const int nsteps = a.nsteps;
    const int64_t order_n = a.order_n;
    double llh_acc = 0.0;
    double nupd_acc = 0.0;
    const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
    const double *__restrict__ F = a.F_in;
    const unsigned lt_mask = (1u << lane) - 1u;

    // ---------------- hub phase (block-cooperative), then one warp per node ----------------
    __shared__ double hub_small[kWarpsPerBlock * 33 + 2];
    if constexpr (kHub && C2 <= 4) {
        if (a.n_hubs > 0) {
            HubArgs ha;
            ha.meta = a.meta; ha.col = a.col; ha.F_in = a.F_in; ha.F_out = a.F_out; ha.node_mask = a.node_mask;
            ha.accepted = a.accepted; ha.changed = a.changed;
            for (int r = 0; r < 7; ++r) ha.peer_out[r] = a.peer_out[r];
            ha.items = a.hub_items; ha.scratch = a.hub_scratch; ha.counters = a.hub_counters;
            ha.n_peers = a.n_peers; ha.n_items = a.n_hub_items; ha.ld = ld; ha.nsteps = nsteps; ha.do_linesearch = a.do_linesearch;
            ha.alpha = a.alpha; ha.min_f = a.min_f; ha.max_f = max_f;
            double hub_llh = 0.0, hub_nupd = 0.0;
            hub_phase<C2>(ha, ec, s_sumF, s_steps, s_D, s_sumF + (size_t)ld * (1 + kWarpsPerBlock), lists, hub_small, &hub_llh, &hub_nupd);
            llh_acc += hub_llh;
            nupd_acc += hub_nupd;
        }
    }

    // software pipeline: cur (being processed), nxt (meta in registers; ids + own row loaded at the
    // top of cur's iteration, rows prefetched to L2), pos_nn (position handed out for the node after)
    int64_t pos = (int64_t)a.n_hubs + (int64_t)blockIdx.x * kWarpsPerBlock + wib;
    int64_t pos_n = pos + nwarps, pos_nn = pos + 2 * nwarps;
    NodeMeta cur = {0, 0, 0}, nxt = {0, 0, 0};
    if (pos < order_n) cur = a.meta[pos];
    if (pos_n < order_n) nxt = a.meta[pos_n];
    int myv = (lane < min(32, cur.deg)) ? a.col[cur.e0 + lane] : 0;
    double2 fu[C2];
#pragma unroll
    for (int c = 0; c < C2; ++c) {
        const int q = lane + 32 * c;
        fu[c] = (pos < order_n && q < ld2) ? ldg2(F + (size_t)cur.u * ld + 2 * q) : make_double2(0.0, 0.0);
    }
    stage_rows<C2, R>(s_rows, F, ld, ld2, lane, myv, 0, min(32, cur.deg));

    while (pos < order_n) {
        const int64_t u = cur.u;
        const int64_t e0 = cur.e0;
        const int deg = cur.deg;
        double *orow = a.F_out + (size_t)u * ld;

        // ---- issue the next nodes' loads (consumed at the bottom of this iteration) ----
        const bool has_next = pos_n < order_n;
        NodeMeta nn = {0, 0, 0};
        if (pos_nn < order_n) nn = a.meta[pos_nn];
        unsigned int fetched = 0;
        if (lane == 0) fetched = atomicAdd(a.work_counter, 1u);
        const int ncnt = has_next ? min(32, nxt.deg) : 0;
        const int nmyv = (lane < ncnt) ? a.col[nxt.e0 + lane] : 0;
        double fusf = 0.0, fufu = 0.0;
#pragma unroll
        for (int c = 0; c < C2; ++c) {
            const int q = lane + 32 * c;
            if (q < ld2) {
                const double2 sf = *reinterpret_cast<const double2 *>(s_sumF + 2 * q);
                fusf = fma(fu[c].x, sf.x, fusf); fusf = fma(fu[c].y, sf.y, fusf);
                fufu = fma(fu[c].x, fu[c].x, fufu); fufu = fma(fu[c].y, fu[c].y, fufu);
            }
        }
        fusf = warp_sum(fusf);
        fufu = warp_sum(fufu);

        // ---------------- PRE (:157-169) ----------------
        double2 g[C2];
#pragma unroll
        for (int c = 0; c < C2; ++c) g[c] = make_double2(0.0, 0.0);
        double S1 = 0.0;
        for (int cb = 0; cb < deg; cb += 32) {
            const int cnt = min(32, deg - cb);
            // neighbour ids of the chunk after this one (hubs): loaded now, prefetched after the first batch
            const int cnt2 = min(32, max(0, deg - cb - 32));
            const int myv2 = (lane < cnt2) ? a.col[e0 + cb + 32 + lane] : 0;
            {
                // batches of R rows kept in registers: dots -> exp/log (each group of 32/R lanes evaluates one
                // of the R edges) -> axpy from the same registers: every neighbour row is loaded once here
                constexpr int GL = 32 / R;                    // lanes per edge group
                const int rsel = lane / GL;
                for (int eb = 0; eb < cnt; eb += R) {
                    // this batch was staged in shared memory one batch (or one node) ago
                    cp_async_wait_all();
                    __syncwarp();
                    double2 x[R][C2];
                    double part[R];
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        const bool ok = eb + r < cnt;
                        double p = 0.0;
#pragma unroll
                        for (int c = 0; c < C2; ++c) {
                            const int q = lane + 32 * c;
                            x[r][c] = (ok && q < ld2) ? *reinterpret_cast<const double2 *>(s_rows + r * ld + 2 * q)
                                                      : make_double2(0.0, 0.0);
                            p = fma(fu[c].x, x[r][c].x, p);
                            p = fma(fu[c].y, x[r][c].y, p);
                        }
                        part[r] = p;
                    }
                    __syncwarp();
                    // stage the following batch while this one is processed: same 32-group, next group of
                    // this node, or the first batch of the next node
                    if (eb + R < cnt) stage_rows<C2, R>(s_rows, F, ld, ld2, lane, myv, eb + R, cnt);
                    else if (cnt2 > 0) stage_rows<C2, R>(s_rows, F, ld, ld2, lane, myv2, 0, cnt2);
                    else stage_rows<C2, R>(s_rows, F, ld, ld2, lane, nmyv, 0, ncnt);
                    const double kx = batch_reduce<R>(part, lane);
                    double w;
                    double t = edge_term<true>(kx, ec, w);
                    t = (eb + rsel < cnt) ? t : 0.0;
                    if constexpr (R >= 4) t += __shfl_xor_sync(0xffffffffu, t, 8);
                    if constexpr (R >= 2) t += __shfl_xor_sync(0xffffffffu, t, 16);
                    S1 += t;
                    if (a.do_linesearch) {
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            const double we = __shfl_sync(0xffffffffu, w, GL * r);
#pragma unroll
                            for (int c = 0; c < C2; ++c) {
                                g[c].x = fma(we, x[r][c].x, g[c].x);
                                g[c].y = fma(we, x[r][c].y, g[c].y);
                            }
                        }
                    }
                }
            }
            myv = myv2;
        }
        if (deg == 0) stage_rows<C2, R>(s_rows, F, ld, ld2, lane, nmyv, 0, ncnt);
        const double llh_u = (S1 - fusf) + fufu;
        llh_acc += llh_u;

        // own row of the next node: loaded here, after the row registers of PRE are dead, and
        // consumed when the pipeline rotates (the whole line search hides the latency)
        double2 nfu[C2];
#pragma unroll
        for (int c = 0; c < C2; ++c) {
            const int q = lane + 32 * c;
            nfu[c] = (has_next && q < ld2) ? ldg2(F + (size_t)nxt.u * ld + 2 * q) : make_double2(0.0, 0.0);
        }

        const bool in_uset = (a.node_mask == nullptr) || (a.node_mask[u] != 0);
        int jstar = -1;

        if (a.do_linesearch && in_uset && deg > 0) {
            // grad = (sum - sumF) + fu  (:168);  G2 = grad.grad for the Armijo slope (:181)
            double G2 = 0.0;
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) {
                    const double2 sf = *reinterpret_cast<const double2 *>(s_sumF + 2 * q);
                    g[c].x = (g[c].x - sf.x) + fu[c].x;
                    g[c].y = (g[c].y - sf.y) + fu[c].y;
                    G2 = fma(g[c].x, g[c].x, G2);
                    G2 = fma(g[c].y, g[c].y, G2);
                }
            }
            G2 = warp_sum(G2);

            // ---- active set: components whose candidate value can be non-zero ----
            int m = 0;
            const bool sparse_ok = (a.min_f == 0.0);
            if (sparse_ok) {
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const double fval = hh ? fu[c].y : fu[c].x;
                        const double gval = hh ? g[c].y : g[c].x;
                        const bool act = (q < ld2) && (fval > 0.0 || gval > 0.0);
                        const unsigned bal = __ballot_sync(0xffffffffu, act);
                        if (bal) {
                            if (act) {
                                const int posn = m + __popc(bal & lt_mask);
                                if (posn < maxm) {
                                    s_afg[posn] = make_double2(fval, gval);
                                    s_aidx[posn] = (unsigned short)(2 * q + hh);
                                }
                            }
                            m += __popc(bal);
                        }
                    }
                }
                __syncwarp();
            }

            if (sparse_ok && m <= maxm) {
                // ---------------- LS, pair-list path ----------------
                const int j16 = lane & 15, h = lane >> 4;
                const int my_idx0 = (lane < m) ? (int)s_aidx[lane] : 0;
                const int mdiv = max(m, 1);
                bool hi_lane = false;
                for (int t = lane; t < m; t += 32) {
                    const double2 fg = s_afg[t];
                    hi_lane |= (fg.x + fg.y > max_f);      // step sizes are <= 1 and fu <= MAX_F_
                }
                const bool need_hi = __any_sync(0xffffffffu, hi_lane);
                for (int tg = 0; tg < nsteps && jstar < 0; tg += 16) {
                    const int j = tg + j16;
                    const bool jok = j < nsteps;
                    const double s = s_steps[jok ? j : 0];
                    double sumterms = ls_edge_range(F, a.col + e0, 0, deg, ld, m, my_idx0, lt_mask, lane, h, s, need_hi, max_f, ec, lists);
                    sumterms += __shfl_xor_sync(0xffffffffu, sumterms, 16);
                    // - newfu.sfT + newfu.newfu with sfT = (sumF - fu) + newfu   (:176,:180)
                    double oa = 0.0, ob = 0.0;
#pragma unroll 2
                    for (int t = h; t < m; t += 2) {
                        const double2 fg = s_afg[t];
                        const double nf = need_hi ? clamp_step0(fg.x, s, fg.y, max_f) : clamp_step0_lo(fg.x, s, fg.y);
                        const double sf = (s_sumF[s_aidx[t]] - fg.x) + nf;
                        oa = fma(nf, sf, oa);
                        ob = fma(nf, nf, ob);
                    }
                    oa += __shfl_xor_sync(0xffffffffu, oa, 16);
                    ob += __shfl_xor_sync(0xffffffffu, ob, 16);
                    const double result = (sumterms - oa) + ob;
                    const double rhs = llh_u + (a.alpha * s) * G2;
                    const unsigned pass = __ballot_sync(0xffffffffu, jok && (result >= rhs)) & 0xffffu;
                    if (pass) jstar = tg + __ffs(pass) - 1;   // lowest j == largest step (:182 max)
                }
            } else {
#pragma unroll
                for (int c = 0; c < C2; ++c) {
                    const int q = lane + 32 * c;
                    if (q < ld2) *reinterpret_cast<double2 *>(orow + 2 * q) = g[c];
                }
                __syncwarp();
                jstar = dense_linesearch<C2, R>(F, a.col + e0, ld, nsteps, s_steps, a.alpha, a.min_f, max_f, ec,
                                                F + (size_t)u * ld, orow, s_sumF, deg, lane, llh_u, G2);
            }
        }

        // ---------------- SWAP (:183-190) + partial sums for :191-192 ----------------
        // fused exchange: the new row goes to the local replica and, over NVLink, straight into the
        // peers' replicas (plain stores to IPC-mapped peer memory) while other warps keep computing
        if (jstar >= 0) {
            const double s = s_steps[jstar];
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) {
                    double2 nr;
                    nr.x = clamp_step(fu[c].x, s, g[c].x, a.min_f, max_f);
                    nr.y = clamp_step(fu[c].y, s, g[c].y, a.min_f, max_f);
                    *reinterpret_cast<double2 *>(orow + 2 * q) = nr;
                    double2 *pd = reinterpret_cast<double2 *>(s_D + 2 * q);
                    double2 vd = *pd;
                    vd.x += fu[c].x - nr.x;
                    vd.y += fu[c].y - nr.y;
                    *pd = vd;
                    fu[c] = nr;                 // fu is dead after this point: reuse it for the pushes below
                }
            }
            nupd_acc += 1.0;
        } else if (a.do_linesearch) {
#pragma unroll
            for (int c = 0; c < C2; ++c) {
                const int q = lane + 32 * c;
                if (q < ld2) *reinterpret_cast<double2 *>(orow + 2 * q) = fu[c];
            }
        }
        if (kPush && a.n_peers > 0 && a.do_linesearch) {
            // multi-GPU launches only (compile-time flag)
            const bool push_row = (jstar >= 0) || (a.changed[u] != 0);
            __syncwarp();      // every lane has read the flag before lane 0 rewrites it below
            if (push_row) {
                for (int pr = 0; pr < a.n_peers; ++pr) {
                    double *prow = a.peer_out[pr] + (size_t)u * ld;
#pragma unroll
                    for (int c = 0; c < C2; ++c) {
                        const int q = lane + 32 * c;
                        if (q < ld2) *reinterpret_cast<double2 *>(prow + 2 * q) = fu[c];
                    }
                }
            }
            if (lane == 0) a.changed[u] = (jstar >= 0) ? 1 : 0;
        }
        if (a.accepted != nullptr && lane == 0) a.accepted[u] = (int8_t)jstar;

        // ---- rotate the pipeline ----
        cur = nxt;
        nxt = nn;
        myv = nmyv;
#pragma unroll
        for (int c = 0; c < C2; ++c) fu[c] = nfu[c];
        pos = pos_n;
        pos_n = pos_nn;
        pos_nn = (int64_t)__shfl_sync(0xffffffffu, fetched, 0);
    }

    // ---------------- block reduction of the partials, one RED per address per block ----------------
    __syncthreads();
    if (a.do_linesearch) {
        for (int i = threadIdx.x; i < ld; i += kBlockThreads) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < kWarpsPerBlock; ++w) v += s_sumF[(size_t)ld * (1 + w) + i];
            if (v != 0.0) atomicAdd(a.partials + i, v);
        }
    }
    __shared__ double s_red[2 * kWarpsPerBlock];
    if (lane == 0) { s_red[wib] = llh_acc; s_red[kWarpsPerBlock + wib] = nupd_acc; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double l = 0.0, c = 0.0;
#pragma unroll
        for (int w = 0; w < kWarpsPerBlock; ++w) { l += s_red[w]; c += s_red[kWarpsPerBlock + w]; }
        atomicAdd(a.partials + 2 * ld, l);
        if (c != 0.0) atomicAdd(a.partials + 2 * ld + 1, c);
    }
}

// Device-side bookkeeping between two step kernels (single block).
struct RunState {
    double llhold;          // LLHold of the reference's loop
    double last_llh;        // most recent call's LLH
    double ret_llh;         // value the loop returns
    long long calls_seen;   // number of calls whose LLH is known
    long long conv_call;    // call index at which |1 - new/old| < tol, or 0
    long long n_updated;    // of the most recent applied step
    int done;
    int pad;
};

struct FinishArgs {
    double *partials;        // [A | B | llh | nupd] of the kernel that just ran
    const double *sumF_cur;
    double *sumF_next;
    int32_t ld;
    RunState *st;
    int32_t *done_flag;
    double *trace;           // optional device trace
    long long trace_cap;
    long long kernel_index;  // c: this is the finish of step kernel c (1-based); 0 = plain apply
    int32_t variant;
    double rel_tol;
    int32_t apply;           // apply the sumF update of this kernel
    int32_t llh_is_final;    // partials.llh is the LLH of the final state (tail LLH kernel)
};

__global__ void finish_kernel(const FinishArgs f) {
    __shared__ int s_done;
    const int ld = f.ld;
    if (threadIdx.x == 0) {
        RunState *st = f.st;
        // a plain apply (kernel_index == 0: bigclam_step, bigclam_finish_local) is not part of a device-side loop: a
        // `done` left behind by an earlier converged bigclam_run must not turn it into a no-op
        int done = (f.kernel_index > 0) ? st->done : 0;
        if (!done && f.kernel_index > 0) {
            // partials.llh == LLH(state before kernel c) == LLH returned by call c-1
            const double L = f.partials[2 * ld];
            const long long call = f.llh_is_final ? f.kernel_index : f.kernel_index - 1;
            if (call == 0) {
                if (f.variant == 2) st->llhold = L;          // LLHold = loglikelihood()
            } else {
                if (f.trace != nullptr && call - 1 < f.trace_cap) f.trace[call - 1] = L;
                st->last_llh = L;
                st->calls_seen = call;
                bool test = true;
                if (f.variant == 4 && call == 1) { st->llhold = L; test = false; }   // :228
                if (f.variant == 3 && call == 1) { st->llhold = 0.0; }               // v3 :207
                if (test) {
                    if (fabs(1.0 - L / st->llhold) < f.rel_tol) {                    // :237
                        done = 1;
                        st->done = 1;
                        st->conv_call = call;
                        st->ret_llh = (f.variant == 4) ? st->llhold : L;             // :242
                        *f.done_flag = 1;
                    } else {
                        st->llhold = L;
                    }
                }
                if (!done) st->ret_llh = L;
            }
        }
        s_done = done;
        if (!done && f.apply) st->n_updated = (long long)(f.partials[2 * ld + 1] + 0.5);
    }
    __syncthreads();
    if (s_done) return;
    if (f.apply) {
        const bool any = f.partials[2 * ld + 1] > 0.0;
        for (int i = threadIdx.x; i < ld; i += blockDim.x) {
            const double sf = f.sumF_cur[i];
            // sumF = sumF - (changeFu._1 - changeFu._2)   (:192); partials[i] = sum over accepted nodes of (old - new)
            f.sumF_next[i] = any ? sf - f.partials[i] : sf;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * ld + 2; i += blockDim.x) f.partials[i] = 0.0;
}

// Column sums of F (initial sumF, bigclam4-7.scala:105-106): pass 1 sums row chunks of kColsumRows rows
// per block into part[chunk][col] (coalesced: 32 lanes = 32 consecutive columns), pass 2 adds the chunks
// in chunk order.  Deterministic.
constexpr int kColsumRows = 2048;
__global__ void colsum_partial_kernel(const double *F, int64_t n, int ld, double *part) {
    const int col = blockIdx.x * 32 + (threadIdx.x & 31);
    const int rlane = threadIdx.x >> 5;             // 0..7
    const int64_t r0 = (int64_t)blockIdx.y * kColsumRows;
    const int64_t r1 = min(n, r0 + kColsumRows);
    double acc = 0.0;
    if (col < ld)
        for (int64_t r = r0 + rlane; r < r1; r += 8) acc += F[(size_t)r * ld + col];
    __shared__ double s[8][33];
    s[rlane][threadIdx.x & 31] = acc;
    __syncthreads();
    if (rlane == 0 && col < ld) {
        double v = 0.0;
        for (int i = 0; i < 8; ++i) v += s[i][threadIdx.x & 31];
        part[(size_t)blockIdx.y * ld + col] = v;
    }
}
__global__ void colsum_final_kernel(const double *part, int nchunks, int ld, double *out) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= ld) return;
    double v = 0.0;
    for (int c = 0; c < nchunks; ++c) v += part[(size_t)c * ld + col];
    out[col] = v;
}

}  // namespace bigclam
