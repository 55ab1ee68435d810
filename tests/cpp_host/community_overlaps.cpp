// Lists the overlaps between the communities through the C++ mirror (include/bigclam_b200.hpp,
// BigClam::community_overlaps), for tests/test_gpu_community_overlaps.py.
//
//   community_overlaps IN OUT WORLD
//
// IN:  int64 n, nnz, K, cases; int64 rowptr[n + 1]; int32 col[nnz]; double F[n * K] (row-major); double delta[cases];
//      int32 min_shared[cases].
// OUT: per case, zero rows everywhere then nowhere: int64 nnz, zero_rows; int64 ptr[K + 1]; int64 size[K];
//      int32 other[nnz]; int32 shared[nnz]; double jaccard[nnz].
// stdout: the error code of a call with min_shared = 0 (BIGCLAM_EINVAL expected).
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
        std::fprintf(stderr, "usage: community_overlaps IN OUT WORLD\n");
        return 2;
    }
    FILE *f = std::fopen(argv[1], "rb");
    if (f == nullptr) return 2;
    try {
        const auto hd = rd<int64_t>(f, 4);
        const auto rp = rd<int64_t>(f, (size_t)hd[0] + 1);
        const auto col = rd<int32_t>(f, (size_t)hd[1]);
        const auto F = rd<double>(f, (size_t)(hd[0] * hd[2]));
        const auto deltas = rd<double>(f, (size_t)hd[3]);
        const auto min_shared = rd<int32_t>(f, (size_t)hd[3]);
        std::fclose(f);
        bigclam::BigClam b(std::atoi(argv[3]), 0, true);
        b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
        FILE *o = std::fopen(argv[2], "wb");
        if (o == nullptr) return 2;
        for (size_t i = 0; i < deltas.size(); ++i)
            for (bool everywhere : {true, false}) {
                const auto s = b.community_overlaps(deltas[i], min_shared[i], everywhere);
                const int64_t hdr[2] = {(int64_t)s.other.size(), s.zero_rows};
                std::fwrite(hdr, 8, 2, o);
                wr(o, s.ptr);
                wr(o, s.size);
                wr(o, s.other);
                wr(o, s.shared);
                wr(o, s.jaccard);
            }
        std::fclose(o);
        try {
            b.community_overlaps(0.5, 0);
        } catch (const bigclam::Error &e) {
            std::printf("%d\n", e.code);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
