// Scores communities through the C++ mirror (include/bigclam_b200.hpp, BigClam::community_stats), for
// tests/test_gpu_community_stats.py.
//
//   community_stats IN OUT WORLD
//
// IN:  int64 n, nnz, K, cases; int64 rowptr[n + 1]; int32 col[nnz]; double F[n * K] (row-major); double delta[cases].
// OUT: per case, zero rows everywhere then nowhere: int64 size[K], volume[K], internal[K]; double conductance[K].
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

int main(int argc, char **argv) {
    if (argc != 4) {
        std::fprintf(stderr, "usage: community_stats IN OUT WORLD\n");
        return 2;
    }
    FILE *f = std::fopen(argv[1], "rb");
    if (f == nullptr) return 2;
    const auto hd = rd<int64_t>(f, 4);
    const auto rp = rd<int64_t>(f, (size_t)hd[0] + 1);
    const auto col = rd<int32_t>(f, (size_t)hd[1]);
    const auto F = rd<double>(f, (size_t)(hd[0] * hd[2]));
    const auto deltas = rd<double>(f, (size_t)hd[3]);
    std::fclose(f);
    try {
        bigclam::BigClam b(std::atoi(argv[3]), 0, true);
        b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
        FILE *o = std::fopen(argv[2], "wb");
        if (o == nullptr) return 2;
        for (double delta : deltas)
            for (bool everywhere : {true, false}) {
                const auto s = b.community_stats(delta, everywhere);
                std::fwrite(s.size.data(), 8, s.size.size(), o);
                std::fwrite(s.volume.data(), 8, s.volume.size(), o);
                std::fwrite(s.internal.data(), 8, s.internal.size(), o);
                std::fwrite(s.conductance.data(), 8, s.conductance.size(), o);
            }
        std::fclose(o);
        try {
            b.community_stats(0.0);
        } catch (const bigclam::Error &e) {
            std::printf("%d\n", e.code);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
