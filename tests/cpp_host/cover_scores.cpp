// Scores the communities against a truth cover through the C++ mirror (include/bigclam_b200.hpp,
// BigClam::score_against), for tests/test_gpu_cover_scores.py.
//
//   cover_scores IN OUT WORLD
//
// IN:  int64 n, nnz, K, cases, q; int64 rowptr[n + 1]; int32 col[nnz]; double F[n * K] (row-major); double delta[cases];
//      int64 truth_ptr[q + 1]; int32 truth_members[truth_ptr[q]].
// OUT: per case, zero rows everywhere then nowhere: double avg_f1, nmi_lfk, nmi_max; double f1_detected[K];
//      int32 match_detected[K]; double hcond_detected[K]; double f1_truth[q]; int32 match_truth[q]; double hcond_truth[q].
// stdout: the error code of a call with delta = 0 (BIGCLAM_EINVAL expected).
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>

#include "bigclam_b200.hpp"

template <class T>
static std::vector<T> rd(FILE *f, size_t n) {
    std::vector<T> v(n);
    if (n > 0 && std::fread(v.data(), sizeof(T), n, f) != n) throw std::runtime_error("short input");
    return v;
}

template <class T>
static void wr(FILE *o, const std::vector<T> &v) {
    if (!v.empty()) std::fwrite(v.data(), sizeof(T), v.size(), o);
}

int main(int argc, char **argv) {
    if (argc != 4) {
        std::fprintf(stderr, "usage: cover_scores IN OUT WORLD\n");
        return 2;
    }
    FILE *f = std::fopen(argv[1], "rb");
    if (f == nullptr) return 2;
    try {
        const auto hd = rd<int64_t>(f, 5);
        const auto rp = rd<int64_t>(f, (size_t)hd[0] + 1);
        const auto col = rd<int32_t>(f, (size_t)hd[1]);
        const auto F = rd<double>(f, (size_t)(hd[0] * hd[2]));
        const auto deltas = rd<double>(f, (size_t)hd[3]);
        const auto tptr = rd<int64_t>(f, (size_t)hd[4] + 1);
        const auto tmem = rd<int32_t>(f, (size_t)tptr.back());
        std::fclose(f);
        std::vector<std::vector<int32_t>> truth;
        for (size_t t = 0; t + 1 < tptr.size(); ++t) truth.emplace_back(tmem.begin() + tptr[t], tmem.begin() + tptr[t + 1]);
        bigclam::BigClam b(std::atoi(argv[3]), 0, true);
        b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
        FILE *o = std::fopen(argv[2], "wb");
        if (o == nullptr) return 2;
        for (double delta : deltas)
            for (bool everywhere : {true, false}) {
                const auto s = b.score_against(truth, delta, everywhere);
                const double sc[3] = {s.avg_f1, s.nmi_lfk, s.nmi_max};
                std::fwrite(sc, 8, 3, o);
                wr(o, s.f1_detected);
                wr(o, s.match_detected);
                wr(o, s.hcond_detected);
                wr(o, s.f1_truth);
                wr(o, s.match_truth);
                wr(o, s.hcond_truth);
            }
        std::fclose(o);
        try {
            b.score_against(truth, 0.0);
        } catch (const bigclam::Error &e) {
            std::printf("%d\n", e.code);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
