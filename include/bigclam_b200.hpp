// bigclam_b200.hpp — header-only C++17 mirror of the reference's spark-shell surface over the C ABI (bigclam_b200.h).
//
// The reference's host side is JVM code (three Scala scripts); the image has no JVM, so the compiled host mirror is C++
// (the Python one is bigclam_apachespark_b200/driver.py — same names, same argument meaning).  Script-level names are
// kept so that a driver reads like the script:
//
//   script (codes/bigclam4-7.scala)                              here
//   numCore/minCom/maxCom/divCom/alpha/beta/MaxInter  :14-26     public members of BigClam (same defaults)
//   GraphLoader.edgeListFile + collectNeighborIds     :45,50-51  load_edge_list / set_graph
//   conductanceLocalMin()                             :58-73     conductanceLocalMin()
//   initNeighborComF(K)                               :81-108    initNeighborComF(K)
//   Kset()                                            :116-133   Kset()
//   backtrackingLineSearchs(uset)                     :152-223   backtrackingLineSearchs(uset)
//   loglikelihood()           bigclamv3-7.scala:106-120          loglikelihood()
//   SGDFindC()                                        :225-243   SGDFindC()
//   MBSGD()       bigclamv3-7.scala:206-222, Bigclamv2.scala:203-219   MBSGD(version)
//   K sweep                                           :244-266   sweep_K()
//   community extraction         Bigclamv2.scala:223-230         delta_threshold(), extract(delta),
//                                                                extract_grouped(delta, ...)
//   community scores, the formula of conductanceLocalMin :64-67  community_stats(delta, zero_rows_everywhere)
//   Avg-F1 (thesis p.21) and overlapping NMI against a known cover  score_against(truth, delta, zero_rows_everywhere)
//   the shared members of every overlapping pair of communities  community_overlaps(delta, min_shared,
//                                                                zero_rows_everywhere)
//   the model P(u,v) = 1 - exp(-F_u.F_v), clamp of :166          edge_probability(u, v), recommend(nodes, m),
//                                                                sample_graph(seed, eps)
//   rows for new nodes, the fit held fixed (:157-184 per node)    fold_in(rowptr, col, max_iter, rel_tol, ...)
//
// Errors: the reference throws JVM exceptions; here every negative return code of the C ABI becomes a bigclam::Error
// (std::runtime_error carrying the code and bigclam_last_error()).  There is no CPU path: without a CUDA device
// set_K() throws BIGCLAM_ECUDA.  One BigClam is driven by one thread at a time (like the script's driver thread).
#ifndef BIGCLAM_B200_HPP
#define BIGCLAM_B200_HPP

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <iterator>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "bigclam_b200.h"

namespace bigclam {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &msg) : std::runtime_error("bigclam_b200 error " + std::to_string(c) + ": " + msg), code(c) {}
};

// Geometric grid of K values (:116-133).  `maxCom / minCom` is an Int division in the script (both are Int vars): the
// pasted REPL value at :268 is only reproduced with that quirk, so it is the default.
inline std::vector<int> Kset(int minCom, int maxCom, int divCom, bool int_division = true) {
    const double ratio = int_division ? (double)(maxCom / minCom) : (double)maxCom / (double)minCom;
    const double conGap = std::exp(std::log(ratio) / divCom);
    std::vector<int> ks{minCom};
    for (int x = minCom;;) {
        int next = (int)(x * conGap);
        if (next == x) ++next;
        x = next;
        if (x >= maxCom) break;
        ks.push_back(x);
    }
    ks.push_back(maxCom);
    return ks;
}

class BigClam {
public:
    // script variables (:14-26), the script's values as defaults
    int numCore = 36;                                // :14 (Spark parallelism; informational here: numGPUs plays that role)
    int minCom = 1000, maxCom = 9000, divCom = 100;
    double alpha = 0.05, beta = 0.1;
    int MaxInter = 15;
    // outcome of the most recent call
    int64_t last_n_updated = 0, last_calls = 0;
    std::vector<double> last_trace;                  // LLH returned by every hot-path call of the last SGDFindC / MBSGD

    explicit BigClam(int numGPUs = 1, int device = 0, bool sparse_rows = true, bool exhaustive_linesearch = false)
        : world_(numGPUs), device_(device),
          flags_((sparse_rows || numGPUs > 1 ? BIGCLAM_F_SPARSE_ROWS : 0) | (exhaustive_linesearch ? BIGCLAM_F_LS_EXHAUSTIVE : 0)) {}
    BigClam(const BigClam &) = delete;
    BigClam &operator=(const BigClam &) = delete;
    ~BigClam() { close(); }

    void close() {
        if (ctx_ != nullptr) bigclam_destroy(ctx_);
        if (multi_ != nullptr) bigclam_multi_destroy(multi_);
        ctx_ = nullptr;
        multi_ = nullptr;
    }

    // GraphLoader.edgeListFile + collectNeighborIds(Either) (:45,50-51).  dedup: simple undirected graph; false = one
    // neighbour entry per edge line and endpoint (literal GraphX).  Vertex ids are relabelled 0..n-1 in ascending order.
    BigClam &load_edge_list(const std::string &path, bool dedup = true) {
        bigclam_graph g{};
        char err[512] = {0};
        const int rc = bigclam_graph_read_edgelist(path.c_str(), dedup ? 1 : 0, &g, err, (int64_t)sizeof(err));
        if (rc != BIGCLAM_OK) throw Error(rc, err);
        ids.assign(g.ids, g.ids + g.n);
        set_graph(g.n, g.rowptr, g.col);
        bigclam_graph_free(&g);
        return *this;
    }
    BigClam &set_graph(int64_t n, const int64_t *rowptr, const int32_t *col) {
        close();
        n_ = n;
        rowptr_.assign(rowptr, rowptr + n + 1);
        col_.assign(col, col + rowptr[n]);
        Sbc.clear();
        return *this;
    }

    // K = sc.broadcast(i) (:249): (re)creates the device context for this K.
    BigClam &set_K(int K) {
        close();
        bigclam_params p;
        check(bigclam_default_params(&p, K), "bigclam_default_params");
        p.alpha = alpha;
        p.beta = beta;
        p.max_inter = MaxInter;
        p.device = device_;
        p.flags = flags_ | (K > 1024 ? BIGCLAM_F_SPARSE_ROWS : 0);      // (the dense engine stops at K = 1024)
        if (world_ > 1) {
            const int rc = bigclam_multi_create(&multi_, n_, rowptr_.data(), col_.data(), &p, world_, nullptr);
            if (rc != BIGCLAM_OK) throw Error(rc, str(bigclam_multi_last_error(nullptr)));
        } else {
            const int rc = bigclam_create(&ctx_, n_, rowptr_.data(), col_.data(), &p);
            if (rc != BIGCLAM_OK) throw Error(rc, str(bigclam_last_error(nullptr)));
        }
        K_ = K;
        return *this;
    }

    // F <- n x K row-major; sumF <- column sums (:105-107), or an injected sumF (the script never recomputes it, :192)
    BigClam &set_F(const std::vector<double> &F, const std::vector<double> *sumF = nullptr) {
        need();
        if ((int64_t)F.size() != n_ * K_) throw Error(BIGCLAM_EINVAL, "F must be n x K");
        call("set_F", bigclam_set_F, bigclam_multi_set_F, F.data());
        if (sumF != nullptr) call("set_sumF", bigclam_set_sumF, bigclam_multi_set_sumF, sumF->data());
        return *this;
    }
    std::vector<double> F() {
        need();
        std::vector<double> out((size_t)(n_ * K_));
        check(multi_ ? bigclam_multi_get_F(multi_, 0, out.data()) : bigclam_get_F(ctx_, out.data()), "get_F");
        return out;
    }
    std::vector<double> sumF() {
        need();
        std::vector<double> out((size_t)K_);
        check(multi_ ? bigclam_multi_get_sumF(multi_, 0, out.data()) : bigclam_get_sumF(ctx_, out.data()), "get_sumF");
        return out;
    }

    // conductanceLocalMin() (:58-73): ranked seed candidates `Sbc` (:75) and every vertex's ego-net conductance.
    const std::vector<int32_t> &conductanceLocalMin(bool on_gpu = true) {
        conductance.assign((size_t)n_, 0.0);
        Sbc.assign((size_t)n_, 0);
        int64_t cnt = 0;
        const int rc = on_gpu ? bigclam_conductance_seeds_gpu(n_, rowptr_.data(), col_.data(), device_, conductance.data(), Sbc.data(), &cnt)
                              : bigclam_conductance_seeds(n_, rowptr_.data(), col_.data(), conductance.data(), Sbc.data(), &cnt);
        if (rc != BIGCLAM_OK) throw Error(rc, "bigclam_conductance_seeds failed");
        Sbc.resize((size_t)cnt);
        return Sbc;
    }
    // initNeighborComF(K) (:81-108) built on the device, straight into the context: the F and sumF bits that loading
    // the host's n x K F0 gives (:105-107), with nothing n x K allocated on either side.
    BigClam &init_F(int K, bool include_self = false, uint64_t pad_seed = 1234) {
        if (Sbc.empty()) conductanceLocalMin();
        if (K != K_ || (ctx_ == nullptr && multi_ == nullptr)) set_K(K);
        const int32_t inc = include_self ? 1 : 0;
        call("init_F", bigclam_init_F, bigclam_multi_init_F, Sbc.data(), (int64_t)Sbc.size(), inc, pad_seed);
        return *this;
    }
    // initNeighborComF(K) (:81-108): builds F0 from the ranked seeds, loads it and returns it (n x K).
    std::vector<double> initNeighborComF(int K, bool include_self = false, uint64_t pad_seed = 1234) {
        init_F(K, include_self, pad_seed);
        return F();
    }

    // ---- the hot path (:152-223).  uset: nullptr = all vertices (what the script always passes, :227)
    double backtrackingLineSearchs(const std::vector<int64_t> *uset = nullptr) {
        need();
        std::vector<uint8_t> mask;
        if (uset != nullptr) {
            mask.assign((size_t)n_, 0);
            for (int64_t u : *uset) mask.at((size_t)u) = 1;
        }
        double llh = 0.0;
        const uint8_t *m = uset != nullptr ? mask.data() : nullptr;
        call("step", bigclam_step, bigclam_multi_step, m, &llh, &last_n_updated);
        return llh;
    }
    double loglikelihood() {
        need();
        double llh = 0.0;
        call("loglikelihood", bigclam_loglikelihood, bigclam_multi_loglikelihood, &llh);
        return llh;
    }
    // :225-243: one call for LLHold, then until |1 - new/old| < 1e-4; returns what the script returns (:242).
    double SGDFindC(double rel_tol = 1e-4, int64_t max_outer = 0) { return run(4, rel_tol, max_outer); }
    void MBSGD(int version = 3, double rel_tol = 1e-4, int64_t max_outer = 0) {
        if (version != 2 && version != 3) throw Error(BIGCLAM_EINVAL, "version must be 2 or 3");
        run(version, rel_tol, max_outer);
    }

    // Community extraction as coded in Bigclamv2.scala:223-230.  delta_threshold: `e = 2.0*count/(N*(N-1)); sqrt(-log(1-e))`
    // (:223-224; in the script `count` is the number of vertices that have edges, the thesis uses |E|: pass what you mean).
    // extract(): communities[c] = vertices u with F_uc >= delta, or, when the row maximum is below delta, with F_uc equal to
    // the row maximum (:227), ascending; an all-zero row is in every community, as coded.  The flatMap / groupByKey of
    // :229-230 runs on the GPU (bigclam_extract_grouped: delta > 0, F >= 0).  Works for multi-GPU handles too.
    static double delta_threshold(int64_t n_vertices, int64_t count) {
        const double e = 2.0 * (double)count / ((double)n_vertices * ((double)n_vertices - 1.0));
        return std::sqrt(-std::log(1.0 - e));
    }
    std::vector<std::vector<int32_t>> extract(double delta) {
        std::vector<int64_t> comptr;
        std::vector<int32_t> members, zero_rows;
        extract_grouped(delta, comptr, members, zero_rows);
        std::vector<std::vector<int32_t>> comms((size_t)K_);
        for (int c = 0; c < K_; ++c) {
            auto &out = comms[(size_t)c];
            out.reserve((size_t)(comptr[(size_t)c + 1] - comptr[(size_t)c]) + zero_rows.size());
            std::merge(members.begin() + comptr[(size_t)c], members.begin() + comptr[(size_t)c + 1], zero_rows.begin(), zero_rows.end(),
                       std::back_inserter(out));
        }
        return comms;
    }
    // The same communities as a CSR over communities (bigclam_extract_grouped): community c is
    // members[comptr[c] .. comptr[c + 1]) ascending, and the all-zero rows are listed once, ascending, in zero_rows.
    void extract_grouped(double delta, std::vector<int64_t> &comptr, std::vector<int32_t> &members, std::vector<int32_t> &zero_rows) {
        need();
        int64_t nnz = 0, z = 0;
        call("extract", bigclam_extract_nnz, bigclam_multi_extract_nnz, delta, &nnz, &z);
        comptr.assign((size_t)K_ + 1, 0);
        members.assign((size_t)std::max<int64_t>(nnz, 1), 0);
        zero_rows.assign((size_t)std::max<int64_t>(z, 1), 0);
        call("extract", bigclam_extract_grouped, bigclam_multi_extract_grouped, delta, comptr.data(), members.data(), zero_rows.data());
        members.resize((size_t)nnz);
        zero_rows.resize((size_t)z);
    }

    // A label-free score of every community of extract(delta) (bigclam_community_stats): size |S_c|, volume (sum of deg(u)
    // over S_c), internal (list entries u -> v with u, v in S_c; the cut is volume - internal) and conductanceLocalMin's
    // formula of :64-67 on them.  zero_rows_everywhere: all-zero rows in every community (as coded) or in none.  Works
    // for multi-GPU handles too.
    struct CommunityStats {
        std::vector<int64_t> size, volume, internal;
        std::vector<double> conductance;
    };
    CommunityStats community_stats(double delta, bool zero_rows_everywhere = true) {
        need();
        CommunityStats s;
        s.size.assign((size_t)K_, 0);
        s.volume.assign((size_t)K_, 0);
        s.internal.assign((size_t)K_, 0);
        s.conductance.assign((size_t)K_, 0.0);
        const int32_t zr = zero_rows_everywhere ? 1 : 0;
        call("community_stats", bigclam_community_stats, bigclam_multi_community_stats, delta, zr, s.size.data(), s.volume.data(),
             s.internal.data(), s.conductance.data());
        return s;
    }

    // The communities of extract(delta) scored against a known cover (bigclam_cover_scores, whose header comment defines
    // every output): truth is a list of node-id lists (any order; a repeated id counts once).  Avg-F1 and the two
    // overlapping NMIs, and per community of either side its best F1, the smallest id attaining it (-1: none) and
    // H*(X_c | Y) / H*(Y_t | X) (NaN outside the NMI).  zero_rows_everywhere: all-zero rows in every detected community
    // (as coded) or in none.  Works for multi-GPU handles too.
    struct CoverScores {
        double avg_f1 = 0.0, nmi_lfk = 0.0, nmi_max = 0.0;
        std::vector<double> f1_detected, f1_truth, hcond_detected, hcond_truth;
        std::vector<int32_t> match_detected, match_truth;
    };
    CoverScores score_against(const std::vector<std::vector<int32_t>> &truth, double delta, bool zero_rows_everywhere = true) {
        need();
        const size_t q = truth.size();
        std::vector<int64_t> ptr(q + 1, 0);
        for (size_t t = 0; t < q; ++t) ptr[t + 1] = ptr[t] + (int64_t)truth[t].size();
        std::vector<int32_t> members;
        members.reserve((size_t)ptr[q]);
        for (const auto &y : truth) members.insert(members.end(), y.begin(), y.end());
        CoverScores s;
        s.f1_detected.assign((size_t)K_, 0.0);
        s.hcond_detected.assign((size_t)K_, 0.0);
        s.match_detected.assign((size_t)K_, -1);
        s.f1_truth.assign(std::max<size_t>(q, 1), 0.0);
        s.hcond_truth.assign(std::max<size_t>(q, 1), 0.0);
        s.match_truth.assign(std::max<size_t>(q, 1), -1);
        double scores[3] = {0.0, 0.0, 0.0};
        const int32_t zr = zero_rows_everywhere ? 1 : 0;
        const int32_t *mp = members.empty() ? nullptr : members.data();
        call("score_against", bigclam_cover_scores, bigclam_multi_cover_scores, delta, zr, (int64_t)q, ptr.data(), mp, s.f1_detected.data(),
             s.match_detected.data(), s.f1_truth.data(), s.match_truth.data(), s.hcond_detected.data(), s.hcond_truth.data(), scores);
        s.f1_truth.resize(q);
        s.hcond_truth.resize(q);
        s.match_truth.resize(q);
        s.avg_f1 = scores[0];
        s.nmi_lfk = scores[1];
        s.nmi_max = scores[2];
        return s;
    }

    // How the communities of extract(delta) overlap each other (bigclam_community_overlaps, whose header comment defines
    // the counts): row c lists other[ptr[c] .. ptr[c + 1]) ascending, the communities d != c sharing at least min_shared
    // non-zero rows with c, with the shared members and the Jaccard index shared / (size_c + size_d - shared) of each
    // pair; symmetric.  zero_rows_everywhere: the zero_rows all-zero rows are in every community (as coded: shared and
    // size include them, and a pair that is not listed still shares them) or in none.  Works for multi-GPU handles too.
    struct CommunityOverlaps {
        std::vector<int64_t> ptr, size;
        std::vector<int32_t> other, shared;
        std::vector<double> jaccard;
        int64_t zero_rows = 0;
    };
    CommunityOverlaps community_overlaps(double delta, int32_t min_shared = 1, bool zero_rows_everywhere = true) {
        need();
        int64_t nnz = 0;
        CommunityOverlaps s;
        call("community_overlaps", bigclam_community_overlaps_nnz, bigclam_multi_community_overlaps_nnz, delta, min_shared, &nnz, &s.zero_rows);
        s.ptr.assign((size_t)K_ + 1, 0);
        s.size.assign((size_t)K_, 0);
        s.other.assign((size_t)std::max<int64_t>(nnz, 1), 0);
        s.shared.assign((size_t)std::max<int64_t>(nnz, 1), 0);
        call("community_overlaps", bigclam_community_overlaps, bigclam_multi_community_overlaps, delta, min_shared, s.ptr.data(),
             s.other.data(), s.shared.data(), s.size.data());
        s.other.resize((size_t)nnz);
        s.shared.resize((size_t)nnz);
        const int64_t z = zero_rows_everywhere ? s.zero_rows : 0;
        for (auto &x : s.shared) x += (int32_t)z;
        for (auto &x : s.size) x += z;
        s.jaccard.resize((size_t)nnz);
        for (int c = 0; c < K_; ++c)
            for (int64_t i = s.ptr[(size_t)c]; i < s.ptr[(size_t)c + 1]; ++i) {
                const int64_t a = s.shared[(size_t)i];
                s.jaccard[(size_t)i] = (double)a / (double)(s.size[(size_t)c] + s.size[(size_t)s.other[(size_t)i]] - a);
            }
        return s;
    }

    // The fitted model as a model of edges, P(u,v) = 1 - exp(-F_u.F_v) with the clamp of :166 (bigclam_pair_affinity):
    // x[i] = F_u[i].F_v[i] and p[i] = 1 - clamp(exp(-x[i]), MIN_P_, MAX_P_).  Works for multi-GPU handles too.
    void edge_probability(const std::vector<int32_t> &u, const std::vector<int32_t> &v, std::vector<double> &x, std::vector<double> &p) {
        need();
        if (u.size() != v.size()) throw Error(BIGCLAM_EINVAL, "edge_probability: u and v differ in length");
        x.assign(u.size(), 0.0);
        p.assign(u.size(), 0.0);
        const int64_t cnt = (int64_t)u.size();
        call("edge_probability", bigclam_pair_affinity, bigclam_multi_pair_affinity, u.data(), v.data(), cnt, x.data(), p.data());
    }
    // For each query node (empty = all nodes) the m nodes at distance 2, not yet linked, with the largest affinity x > 0
    // (x descending, then id ascending): v and x are nodes.size() x m row-major, padded with -1 and 0 (bigclam_recommend).
    void recommend(const std::vector<int32_t> &nodes, int m, std::vector<int32_t> &v, std::vector<double> &x) {
        need();
        const int64_t cnt = nodes.empty() ? n_ : (int64_t)nodes.size();
        const int32_t *q = nodes.empty() ? nullptr : nodes.data();
        v.assign((size_t)(cnt * std::max(m, 0)), -1);
        x.assign((size_t)(cnt * std::max(m, 0)), 0.0);
        call("recommend", bigclam_recommend, bigclam_multi_recommend, q, cnt, m, v.data(), x.data(), nullptr);
    }
    // A graph sampled from the model (bigclam_sample_graph): pairs that share a component are edges with probability
    // p_uv (edge_probability's p), the others with probability eps; a symmetric CSR, rows ascending, the shape set_graph
    // takes.  The same (F, seed, eps) gives the same graph.  Works for multi-GPU handles too.
    void sample_graph(uint64_t seed, double eps, std::vector<int64_t> &rowptr, std::vector<int32_t> &col) {
        need();
        int64_t nnz = 0;
        call("sample_graph", bigclam_sample_graph_nnz, bigclam_multi_sample_graph_nnz, seed, eps, &nnz);
        rowptr.assign((size_t)n_ + 1, 0);
        col.assign((size_t)std::max<int64_t>(nnz, 1), 0);
        call("sample_graph", bigclam_sample_graph, bigclam_multi_sample_graph, seed, eps, rowptr.data(), col.data());
        col.resize((size_t)nnz);
    }
    // Rows for new nodes with the fitted F and sumF held fixed (bigclam_fold_in): query node i has the neighbour list
    // col[rowptr[i] .. rowptr[i + 1]) among the fitted nodes.  The rows come as a CSR (indptr, indices, values: ascending,
    // no zeros, the shape set_F_csr takes), with each row's LLH term and accepted steps.  Works for multi-GPU handles too.
    void fold_in(const std::vector<int64_t> &rowptr, const std::vector<int32_t> &col, int32_t max_iter, double rel_tol,
                 std::vector<int64_t> &indptr, std::vector<int32_t> &indices, std::vector<double> &values, std::vector<double> &llh,
                 std::vector<int32_t> &iters) {
        need();
        if (rowptr.empty()) throw Error(BIGCLAM_EINVAL, "fold_in: rowptr needs q + 1 entries");
        const int64_t q = (int64_t)rowptr.size() - 1;
        if (rowptr.back() > (int64_t)col.size()) throw Error(BIGCLAM_EINVAL, "fold_in: rowptr goes beyond col");
        int64_t nnz = 0;
        call("fold_in", bigclam_fold_in_nnz, bigclam_multi_fold_in_nnz, q, rowptr.data(), col.data(), max_iter, rel_tol, &nnz);
        indptr.assign((size_t)q + 1, 0);
        indices.assign((size_t)std::max<int64_t>(nnz, 1), 0);
        values.assign((size_t)std::max<int64_t>(nnz, 1), 0.0);
        llh.assign((size_t)q, 0.0);
        iters.assign((size_t)q, 0);
        call("fold_in", bigclam_fold_in, bigclam_multi_fold_in, q, rowptr.data(), col.data(), max_iter, rel_tol, indptr.data(), indices.data(),
             values.data(), llh.data(), iters.data());
        indices.resize((size_t)nnz);
        values.resize((size_t)nnz);
    }

    std::vector<int> Kset() const { return bigclam::Kset(minCom, maxCom, divCom); }
    // The K sweep (:244-266): for K in Kset: initNeighborComF(K) (init_F), SGDFindC(); stops at the first K whose gain
    // `1 - new/old` is below 0.1 %.  As coded LLHKold starts at 0.0, so the first K never stops the sweep.
    // Returns KforC (0 when the grid ran out, :245) and fills hist with (K, LLH).
    int sweep_K(std::vector<std::pair<int, double>> *hist = nullptr, double rel_gain = 0.001, int64_t max_outer = 0) {
        double LLHKold = 0.0;
        for (int k : Kset()) {
            init_F(k);
            const double LLHKnew = SGDFindC(1e-4, max_outer);
            if (hist != nullptr) hist->emplace_back(k, LLHKnew);
            if (1.0 - LLHKnew / LLHKold < rel_gain) return k;          // (x / 0.0 = -inf or nan: never below, like the JVM)
            LLHKold = LLHKnew;
        }
        return 0;
    }

    int64_t n() const { return n_; }
    int K() const { return K_; }
    std::vector<int64_t> ids;                         // original vertex id of dense index i (load_edge_list)
    std::vector<int32_t> Sbc;                         // ranked seeds (:75)
    std::vector<double> conductance;

private:
    double run(int variant, double rel_tol, int64_t max_outer) {
        need();
        std::vector<double> trace(65536);
        double llh = 0.0;
        call("run", bigclam_run, bigclam_multi_run, variant, rel_tol, max_outer, &llh, &last_calls, trace.data(), (int64_t)trace.size());
        trace.resize((size_t)std::min<int64_t>(last_calls, (int64_t)trace.size()));
        last_trace = std::move(trace);
        return llh;
    }
    void need() const {
        if (ctx_ == nullptr && multi_ == nullptr) throw Error(BIGCLAM_EINVAL, "no context: call set_graph()/load_edge_list() and set_K() first");
    }
    static std::string str(const char *s) { return s != nullptr ? s : "unknown error"; }
    // The same C call on whichever handle this instance holds, its error thrown as an Error prefixed with `what`.
    template <typename Single, typename Multi, typename... A>
    void call(const char *what, Single single_fn, Multi multi_fn, A... args) const {
        check(multi_ ? multi_fn(multi_, args...) : single_fn(ctx_, args...), what);
    }
    void check(int rc, const char *what) const {
        if (rc == BIGCLAM_OK) return;
        const char *msg = multi_ ? bigclam_multi_last_error(multi_) : bigclam_last_error(ctx_);
        throw Error(rc, std::string(what) + ": " + str(msg));
    }

    int world_, device_, flags_;
    int64_t n_ = 0;
    int K_ = 0;
    std::vector<int64_t> rowptr_;
    std::vector<int32_t> col_;
    bigclam_ctx *ctx_ = nullptr;
    bigclam_multi *multi_ = nullptr;
};

}  // namespace bigclam
#endif  // BIGCLAM_B200_HPP
