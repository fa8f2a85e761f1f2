// cub_sort.cu -- CALIBRATION ONLY (never linked into libgsr): cub::DeviceRadixSort::SortPairs / SortKeys on the c5 key
// distribution, timed with CUDA events, so that the hand-written Onesweep of csrc/radix_sort.cu can be read against what the
// vendor library reaches on the same box.  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o ubench/cub_sort ubench/cub_sort.cu
#include <cub/cub.cuh>
#include <cstdio>
#include <cstdlib>
#include <vector>

__global__ void fill(uint32_t *k, uint32_t *v, size_t n, uint32_t tiles) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x = (uint32_t)i * 2654435761u; x ^= x >> 15; x *= 2246822519u; x ^= x >> 13; x *= 3266489917u; x ^= x >> 16;
    uint32_t y = x * 747796405u + 2891336453u; y ^= y >> 16;
    k[i] = ((x % tiles) << 16) | (52000u + (y % 9500u));
    v[i] = (uint32_t)i;
}

int main(int argc, char **argv) {
    std::vector<size_t> sizes;
    for (int i = 1; i < argc; ++i) sizes.push_back((size_t)atoll(argv[i]));
    if (sizes.empty()) sizes = {1u << 20, 1u << 22, 9600000u, 1u << 24, 1u << 26, 1u << 28};
    printf("{");
    for (size_t si = 0; si < sizes.size(); ++si) {
        const size_t n = sizes[si];
        uint32_t *k0, *k1, *v0, *v1;
        cudaMalloc(&k0, 4 * n); cudaMalloc(&k1, 4 * n); cudaMalloc(&v0, 4 * n); cudaMalloc(&v1, 4 * n);
        void *tmp = nullptr; size_t tb = 0;
        cub::DoubleBuffer<uint32_t> dk(k0, k1), dv(v0, v1);
        cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)n);
        cudaMalloc(&tmp, tb);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        float best_p = 1e30f, best_k = 1e30f;
        for (int it = 0; it < 5; ++it) {
            fill<<<(unsigned)((n + 255) / 256), 256>>>(k0, v0, n, 8160u);
            cub::DoubleBuffer<uint32_t> a(k0, k1), b(v0, v1);
            cudaEventRecord(e0);
            cub::DeviceRadixSort::SortPairs(tmp, tb, a, b, (int)n);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (it && ms < best_p) best_p = ms;
        }
        for (int it = 0; it < 5; ++it) {
            fill<<<(unsigned)((n + 255) / 256), 256>>>(k0, v0, n, 8160u);
            cub::DoubleBuffer<uint32_t> a(k0, k1);
            cudaEventRecord(e0);
            cub::DeviceRadixSort::SortKeys(tmp, tb, a, (int)n);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (it && ms < best_k) best_k = ms;
        }
        printf("%s\"%zu\": {\"pairs_ms\": %.4f, \"gpairs_s\": %.2f, \"keys_ms\": %.4f, \"gkeys_s\": %.2f}", si ? ", " : "", n, best_p, n / best_p / 1e6, best_k,
               n / best_k / 1e6);
        cudaFree(k0); cudaFree(k1); cudaFree(v0); cudaFree(v1); cudaFree(tmp);
    }
    printf("}\n");
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { fprintf(stderr, "cuda error: %s\n", cudaGetErrorString(e)); return 1; }
    return 0;
}
