// Driver of bigclam::BigClam::fold_in (include/bigclam_b200.hpp), run by tests/test_gpu_fold_in.py: reads a graph, F and
// query lists, writes the folded rows.
#include <cstdio>
#include <vector>
#include "bigclam_b200.hpp"
template <class T> static std::vector<T> rd(FILE *f, size_t n) { std::vector<T> v(n); if (fread(v.data(), sizeof(T), n, f) != n) throw 1; return v; }
int main(int, char **argv) {
    FILE *f = fopen(argv[1], "rb");
    int64_t hd[5];                                   // n, nnz, K, q, query entries
    if (fread(hd, 8, 5, f) != 5) return 2;
    auto rp = rd<int64_t>(f, hd[0] + 1);
    auto col = rd<int32_t>(f, hd[1]);
    auto F = rd<double>(f, hd[0] * hd[2]);
    auto qrp = rd<int64_t>(f, hd[3] + 1);
    auto qcol = rd<int32_t>(f, hd[4]);
    fclose(f);
    bigclam::BigClam b(1, 0, true);
    b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
    std::vector<int64_t> ip;
    std::vector<int32_t> ix, it;
    std::vector<double> vl, llh;
    b.fold_in(qrp, qcol, 100, 1e-4, ip, ix, vl, llh, it);
    FILE *o = fopen(argv[2], "wb");
    fwrite(ip.data(), 8, ip.size(), o); fwrite(ix.data(), 4, ix.size(), o); fwrite(vl.data(), 8, vl.size(), o);
    fwrite(llh.data(), 8, llh.size(), o); fwrite(it.data(), 4, it.size(), o);
    fclose(o);
    try { b.fold_in(qrp, qcol, 0, 1e-4, ip, ix, vl, llh, it); } catch (const bigclam::Error &e) { std::printf("%d\n", e.code); }
    return 0;
}
