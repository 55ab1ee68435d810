// initf_gpu.cu — conductanceLocalMin() (codes/bigclam4-7.scala:58-73) on the GPU: the ego-net conductance of every
// node is integer set work (for every member u of the ego net of x, count the entries of u's neighbour list that
// fall inside the ego net), one warp per node, membership by binary search in x's sorted neighbour list.  The host
// version (initf.cpp, same quirks, documented there) takes 0.5-1.8 s on com-amazon — longer than a whole converged
// run of the hot path; the seed ranking that follows (one sort of the candidates) stays on the host.
#include "../../include/bigclam_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

void bigclam_select_seeds_internal(int64_t n, const int64_t *rowptr, const int32_t *col, const double *cond,
                                   int32_t *seeds_out, int64_t *n_seeds_out);

namespace {

// col: neighbour lists as given (members and z are walked in this order, with multiplicity);
// scol: the same lists sorted ascending (membership tests)
__global__ void conductance_kernel(int64_t n, const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                   const int32_t *__restrict__ scol, double sigma, double *__restrict__ cond) {
    const int lane = threadIdx.x & 31;
    const int64_t x = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (x >= n) return;
    const int64_t b0 = rowptr[x];
    const int deg = (int)(rowptr[x + 1] - b0);
    const int32_t *ego = scol + b0;
    long long zsize = 0, inside = 0;
    for (int m = -1; m < deg; ++m) {                       // y = [x] ++ neighbours(x)   (:54-56, :62)
        const int64_t u = (m < 0) ? x : (int64_t)col[b0 + m];
        const int64_t e0 = rowptr[u], e1 = rowptr[u + 1];
        for (int64_t e = e0 + lane; e < e1; e += 32) {     // z = y.flatMap(neighbours)   (:63)
            const int32_t i = __ldg(col + e);
            bool in = (i == (int32_t)x);
            int lo = 0, hi = deg;
            while (!in && lo < hi) {
                const int mid = (lo + hi) >> 1;
                const int32_t v = __ldg(ego + mid);
                if (v == i) in = true;
                else if (v < i) lo = mid + 1;
                else hi = mid;
            }
            ++zsize;
            inside += in ? 1 : 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        zsize += __shfl_xor_sync(0xffffffffu, zsize, o);
        inside += __shfl_xor_sync(0xffffffffu, inside, o);
    }
    if (lane == 0) {
        cond[x] = bigclam::conductance_formula((double)(zsize - inside), (double)inside, sigma);   // :64-67
    }
}

}  // namespace

extern "C" int bigclam_conductance_seeds_gpu(int64_t n, const int64_t *rowptr, const int32_t *col, int32_t device,
                                             double *conductance_out /* n, optional */, int32_t *seeds_out /* n */,
                                             int64_t *n_seeds_out) {
    if (n <= 0 || rowptr == nullptr || seeds_out == nullptr || n_seeds_out == nullptr) return BIGCLAM_EINVAL;
    const int64_t nnz = rowptr[n];
    if (nnz > 0 && col == nullptr) return BIGCLAM_EINVAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { (void)cudaGetLastError(); return BIGCLAM_ECUDA; }   // no CPU fallback here
    if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return BIGCLAM_ECUDA;
    // sorted copy of the lists for the membership tests (readers deliver them sorted already: then it is the same array)
    bool sorted = true;
    for (int64_t u = 0; u < n && sorted; ++u)
        for (int64_t e = rowptr[u] + 1; e < rowptr[u + 1]; ++e)
            if (col[e - 1] > col[e]) { sorted = false; break; }
    std::vector<int32_t> scol_h;
    if (!sorted) {
        scol_h.assign(col, col + nnz);
        for (int64_t u = 0; u < n; ++u) std::sort(scol_h.begin() + rowptr[u], scol_h.begin() + rowptr[u + 1]);
    }
    int64_t *d_rp = nullptr;
    int32_t *d_col = nullptr, *d_scol = nullptr;
    double *d_cond = nullptr;
    std::vector<double> cond((size_t)n);
    cudaError_t e = cudaMalloc(&d_rp, sizeof(int64_t) * ((size_t)n + 1));
    if (e == cudaSuccess) e = cudaMalloc(&d_col, sizeof(int32_t) * std::max<size_t>(1, (size_t)nnz));
    if (e == cudaSuccess && !sorted) e = cudaMalloc(&d_scol, sizeof(int32_t) * std::max<size_t>(1, (size_t)nnz));
    if (e == cudaSuccess) e = cudaMalloc(&d_cond, sizeof(double) * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_rp, rowptr, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && nnz > 0) e = cudaMemcpy(d_col, col, sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !sorted) e = cudaMemcpy(d_scol, scol_h.data(), sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        const int wpb = 8;
        conductance_kernel<<<(unsigned)((n + wpb - 1) / wpb), wpb * 32, 0, 0>>>(n, d_rp, d_col, sorted ? d_col : d_scol, (double)nnz, d_cond);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(cond.data(), d_cond, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost);
    cudaFree(d_rp); cudaFree(d_col); cudaFree(d_scol); cudaFree(d_cond);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return BIGCLAM_ECUDA; }
    if (conductance_out != nullptr) std::copy(cond.begin(), cond.end(), conductance_out);
    bigclam_select_seeds_internal(n, rowptr, col, cond.data(), seeds_out, n_seeds_out);
    return BIGCLAM_OK;
}
