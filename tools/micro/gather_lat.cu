// Microbenchmark: latency of gathering 4 random rows (1600 B each) per warp from a 536 MB matrix,
// 16 warps/SM, with no prefetch / per-line prefetch.global.L2 / cp.async.bulk.prefetch.L2 issued one
// "node" ahead.  Prints average cycles per batch and achieved GB/s.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

template <int MODE>   // 0 none, 1 per-line L2 prefetch, 2 bulk L2 prefetch
__global__ void __launch_bounds__(256, 2) k(const double *F, const int *idx, int nbatch_per_warp, int ld, long long *cyc, double *sink, int work) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int *my = idx + (size_t)warp * nbatch_per_warp * 4;
    double acc = 0.0;
    long long tot = 0;
    for (int b = 0; b < nbatch_per_warp; ++b) {
        if (MODE != 0 && b + 1 < nbatch_per_warp && lane < 4) {
            const char *row = (const char *)(F + (size_t)my[(b + 1) * 4 + lane] * ld);
            if (MODE == 1) { for (int off = 0; off < ld * 8; off += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + off)); }
            else asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(row), "r"(ld * 8) : "memory");
        }
        // simulated compute between batches (dependent FMA chain)
        double w = acc;
        for (int i = 0; i < work; ++i) w = fma(w, 1.0000001, 1e-9);
        acc = w;
        const long long t0 = clock64();
        double2 x[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const double *fv = F + (size_t)my[b * 4 + r] * ld;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int q = lane + 32 * c;
                x[r][c] = (q < ld / 2) ? __ldg((const double2 *)(fv + 2 * q)) : make_double2(0, 0);
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc += x[r][c].x + x[r][c].y;
        tot += clock64() - t0;
    }
    if (lane == 0) cyc[warp] = tot;
    if (acc == 123.456) sink[0] = acc;
}

int main(int argc, char **argv) {
    const int n = 334863, ld = 200;
    const int work = argc > 1 ? atoi(argv[1]) : 2000;
    const int dense = argc > 2 ? atoi(argv[2]) : 1;
    double *F; CK(cudaMalloc(&F, sizeof(double) * (size_t)n * ld)); { std::vector<double> hf((size_t)n * ld); unsigned long long st = 88172645463325252ULL; for (auto &v : hf) { st ^= st << 13; st ^= st >> 7; st ^= st << 17; v = ((st >> 11) * (1.0 / 9007199254740992.0)) * (((st & 31) == 0) ? 1.0 : (dense ? 1.0 : 0.0)); } CK(cudaMemcpy(F, hf.data(), hf.size() * 8, cudaMemcpyHostToDevice)); }
    const int blocks = 132 * 2, warps = blocks * 8, nb = 200;
    std::vector<int> h((size_t)warps * nb * 4);
    srand(1);
    for (auto &v : h) v = (int)(((long long)rand() * 32768 + rand()) % n);
    int *idx; CK(cudaMalloc(&idx, h.size() * 4)); CK(cudaMemcpy(idx, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    long long *cyc; CK(cudaMalloc(&cyc, warps * 8)); double *sink; CK(cudaMalloc(&sink, 8));
    std::vector<long long> hc(warps);
    for (int mode = 0; mode < 3; ++mode) {
        for (int rep = 0; rep < 2; ++rep) {
            cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
            cudaEventRecord(e0);
            if (mode == 0) k<0><<<blocks, 256>>>(F, idx, nb, ld, cyc, sink, work);
            if (mode == 1) k<1><<<blocks, 256>>>(F, idx, nb, ld, cyc, sink, work);
            if (mode == 2) k<2><<<blocks, 256>>>(F, idx, nb, ld, cyc, sink, work);
            cudaEventRecord(e1); CK(cudaDeviceSynchronize());
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            CK(cudaMemcpy(hc.data(), cyc, warps * 8, cudaMemcpyDeviceToHost));
            double s = 0; for (auto v : hc) s += v;
            if (rep == 1) printf("work %d mode %d: %.3f ms, avg load-wait %.0f cycles per batch of 4 rows, %.0f GB/s\n", work, mode, ms,
                   s / warps / nb, (double)warps * nb * 4 * ld * 8 / ms / 1e6);
        }
    }
    return 0;
}
