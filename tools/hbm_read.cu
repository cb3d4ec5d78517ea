// Read-only HBM stream: the ceiling the substring scan (k_substr_scan) is measured against.  Built and run by tools/hbm_ceiling.py.
//
//     hbm_read <GiB> <runs>      -> one line "bytes=<B> median_ms=<t> gbs=<GB/s> min_ms=<t> max_ms=<t> device=<name>"
//
// Every thread of a resident persistent grid keeps 8 independent 16-byte loads in flight and folds them into an XOR that is written only
// when it equals a value no input produces, so the loads cannot be dropped.  The buffer (>= 32 GiB) is far larger than the 50 MB L2.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

static constexpr int kThreads = 256, kUnroll = 8;

__global__ void __launch_bounds__(kThreads) k_read(const uint4* __restrict__ p, size_t n, unsigned* __restrict__ sink) {
    const size_t stride = (size_t)gridDim.x * kThreads;
    size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
    unsigned acc = 0;
    for (; i + (kUnroll - 1) * stride < n; i += kUnroll * stride) {
        uint4 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) v[u] = __ldg(p + i + u * stride);
#pragma unroll
        for (int u = 0; u < kUnroll; u++) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    for (; i < n; i += stride) { const uint4 v = __ldg(p + i); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
    if (acc == 0x9e3779b9u) *sink = acc;   // never true for the 0x5a fill
}

int main(int argc, char** argv) {
    const double gib = argc > 1 ? atof(argv[1]) : 32.0;
    const int runs = argc > 2 ? atoi(argv[2]) : 10;
    const size_t bytes = (size_t)(gib * (1ull << 30)) & ~(size_t)15, n = bytes / 16;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_read, kThreads, 0));
    uint4* buf = nullptr; unsigned* sink = nullptr;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMalloc(&sink, 4));
    CK(cudaMemset(buf, 0x5a, bytes));
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    const int grid = prop.multiProcessorCount * std::max(occ, 1);
    for (int w = 0; w < 2; w++) k_read<<<grid, kThreads>>>(buf, n, sink);
    CK(cudaDeviceSynchronize());
    std::vector<float> ms;
    for (int r = 0; r < runs; r++) {
        CK(cudaEventRecord(a));
        k_read<<<grid, kThreads>>>(buf, n, sink);
        CK(cudaEventRecord(b));
        CK(cudaEventSynchronize(b));
        float t = 0; CK(cudaEventElapsedTime(&t, a, b)); ms.push_back(t);
    }
    CK(cudaGetLastError());
    std::vector<float> s = ms; std::sort(s.begin(), s.end());
    const double med = runs % 2 ? s[runs / 2] : 0.5 * (s[runs / 2 - 1] + s[runs / 2]);
    printf("bytes=%zu median_ms=%.4f gbs=%.1f min_ms=%.4f max_ms=%.4f grid=%d device=%s\n", bytes, med, bytes / 1e9 / (med / 1e3), s.front(), s.back(), grid, prop.name);
    cudaFree(buf); cudaFree(sink);
    return 0;
}
