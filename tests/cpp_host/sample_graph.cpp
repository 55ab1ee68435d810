// Samples graphs from a model through the C++ mirror (include/bigclam_b200.hpp, BigClam::sample_graph), for
// tests/test_gpu_sample.py.
//
//   sample_graph IN OUT WORLD
//
// IN:  int64 n, nnz, K, cases; int64 rowptr[n + 1]; int32 col[nnz]; double F[n * K] (row-major);
//      then per case: uint64 seed, double eps.
// OUT: per case: int64 nnz; int64 rowptr[n + 1]; int32 col[nnz].
// stdout: the error code of a call with eps = 1 (BIGCLAM_EINVAL expected).
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
        std::fprintf(stderr, "usage: sample_graph IN OUT WORLD\n");
        return 2;
    }
    FILE *f = std::fopen(argv[1], "rb");
    if (f == nullptr) return 2;
    const auto hd = rd<int64_t>(f, 4);
    const auto rp = rd<int64_t>(f, (size_t)hd[0] + 1);
    const auto col = rd<int32_t>(f, (size_t)hd[1]);
    const auto F = rd<double>(f, (size_t)(hd[0] * hd[2]));
    std::vector<uint64_t> seeds;
    std::vector<double> eps;
    for (int64_t i = 0; i < hd[3]; ++i) {
        seeds.push_back(rd<uint64_t>(f, 1)[0]);
        eps.push_back(rd<double>(f, 1)[0]);
    }
    std::fclose(f);
    try {
        bigclam::BigClam b(std::atoi(argv[3]), 0, true);
        b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
        FILE *o = std::fopen(argv[2], "wb");
        if (o == nullptr) return 2;
        std::vector<int64_t> srp;
        std::vector<int32_t> scol;
        for (size_t i = 0; i < seeds.size(); ++i) {
            b.sample_graph(seeds[i], eps[i], srp, scol);
            const int64_t nnz = (int64_t)scol.size();
            std::fwrite(&nnz, 8, 1, o);
            std::fwrite(srp.data(), 8, srp.size(), o);
            std::fwrite(scol.data(), 4, scol.size(), o);
        }
        std::fclose(o);
        try {
            b.sample_graph(1, 1.0, srp, scol);
        } catch (const bigclam::Error &e) {
            std::printf("%d\n", e.code);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
