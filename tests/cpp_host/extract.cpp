// Extracts communities through the C++ mirror (include/bigclam_b200.hpp, BigClam::extract_grouped and BigClam::extract),
// for tests/test_gpu_extract.py.
//
//   extract IN OUT WORLD
//
// IN:  int64 n, nnz, K, cases; int64 rowptr[n + 1]; int32 col[nnz]; double F[n * K] (row-major); double delta[cases].
// OUT: per case: int64 comptr[K + 1]; int64 z; int32 members[comptr[K]]; int32 zero_rows[z];
//      then extract(delta): per community c < K, int64 len and int32 nodes[len].
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
        std::fprintf(stderr, "usage: extract IN OUT WORLD\n");
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
        std::vector<int64_t> comptr;
        std::vector<int32_t> members, zero_rows;
        for (double delta : deltas) {
            b.extract_grouped(delta, comptr, members, zero_rows);
            const int64_t z = (int64_t)zero_rows.size();
            std::fwrite(comptr.data(), 8, comptr.size(), o);
            std::fwrite(&z, 8, 1, o);
            std::fwrite(members.data(), 4, members.size(), o);
            std::fwrite(zero_rows.data(), 4, zero_rows.size(), o);
            for (const auto &c : b.extract(delta)) {
                const int64_t len = (int64_t)c.size();
                std::fwrite(&len, 8, 1, o);
                std::fwrite(c.data(), 4, c.size(), o);
            }
        }
        std::fclose(o);
        try {
            b.extract_grouped(0.0, comptr, members, zero_rows);
        } catch (const bigclam::Error &e) {
            std::printf("%d\n", e.code);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
