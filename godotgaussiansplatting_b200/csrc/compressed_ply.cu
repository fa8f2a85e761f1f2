// compressed_ply.cu -- export of the store as a SuperSplat / PlayCanvas compressed PLY (gsr_export_compressed_ply; include/gsr.h
// "Compressed PLY"; DESIGN.md section 5.24).  The decode (gsr_upload_compressed_ply) is compressed_to_soa_kernel in ingest.cu.
//
// Three passes over the store and one sort:
//   1. compress_bounds_kernel: the count of exported splats and the bounds of their positions (order-preserving words, integer atomics);
//   2. compress_key_kernel: one (key, slot) pair per slot of [0, n): the Morton code (or 0 for store order) of an exported splat,
//      CPLY_NOT_EXPORTED for every other slot.  The library's Onesweep sort of the pairs is stable, so it gives the file's row order and
//      the compaction at once: the exported slots come first, in key order, ties in ascending slot;
//   3. compress_chunk_kernel: one 256-thread CTA per chunk.  Each thread gathers its row's splat and decomposes its covariance with
//      gsr_export_ply's float64 Jacobi (export_scale_rot), the CTA reduces the chunk's 18 bounds, each thread packs its row into shared
//      memory, and the CTA stores its words, floats and SH bytes as contiguous runs.
// The arithmetic follows the library's deterministic math (-fmad=false): one rounding per operator, in the order of include/gsr.h.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int CPLY_THREADS = 256;
static_assert(CPLY_THREADS == (int)CPLY_CHUNK, "one thread per row of a chunk");
constexpr int CPLY_WARPS = CPLY_THREADS / 32;

// The inverse of depth_order_word
__device__ __forceinline__ float order_word_float(uint32_t w) { return __uint_as_float(w ^ ((w >> 31) ? 0x80000000u : 0xFFFFFFFFu)); }
__device__ __forceinline__ uint32_t float_order_word(float f) { return depth_order_word(__float_as_uint(f)); }

__device__ __forceinline__ uint32_t warp_min_u32(uint32_t v) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) { const uint32_t o = __shfl_xor_sync(0xffffffffu, v, m); v = o < v ? o : v; }
    return v;
}
__device__ __forceinline__ uint32_t warp_max_u32(uint32_t v) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) { const uint32_t o = __shfl_xor_sync(0xffffffffu, v, m); v = o > v ? o : v; }
    return v;
}

// Slot s (< n) is exported: in scope and plane-0 x, y, z finite (so not vacant).  p0 is read only for a slot in scope.
__device__ __forceinline__ bool cply_exported(const CompressArgs &a, uint64_t s, float4 &p0) {
    if (a.hidden && (a.selected_only ? !mask_bit(a.selected, s) : mask_bit(a.hidden, s))) return false;
    p0 = __ldg(a.soa + s);
    return fabsf(p0.x) <= 3.402823466e38f && fabsf(p0.y) <= 3.402823466e38f && fabsf(p0.z) <= 3.402823466e38f;
}

// Pass 1: a warp per 32 consecutive slots (grid-stride), warp-reduced, one set of atomics per warp and round
__global__ void __launch_bounds__(CPLY_THREADS) compress_bounds_kernel(const __grid_constant__ CompressArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warps = (uint64_t)gridDim.x * CPLY_WARPS;
    for (uint64_t base = ((uint64_t)blockIdx.x * CPLY_WARPS + (threadIdx.x >> 5)) * 32ull; base < a.n; base += warps * 32ull) {
        const uint64_t s = base + lane;
        float4 p0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        const bool in = s < a.n && cply_exported(a, s, p0);
        const uint32_t bits = __ballot_sync(0xffffffffu, in);
        if (!bits) continue;
        const float p[3] = {p0.x, p0.y, p0.z};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint32_t w = float_order_word(p[k]);
            const uint32_t lo = warp_min_u32(in ? w : 0xFFFFFFFFu), hi = warp_max_u32(in ? w : 0u);
            if (lane == 0u) { atomicMin(a.bounds->lo + k, lo); atomicMax(a.bounds->hi + k, hi); }
        }
        if (lane == 0u) atomicAdd(&a.bounds->count, (unsigned long long)__popc(bits));
    }
}

// 10 bits spread to every third bit
__device__ __forceinline__ uint32_t part1by2(uint32_t v) {
    v &= 0x3FFu;
    v = (v | (v << 16)) & 0x030000FFu;
    v = (v | (v << 8)) & 0x0300F00Fu;
    v = (v | (v << 4)) & 0x030C30C3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}
__device__ __forceinline__ uint32_t morton_cell(float p, float lo, float hi) {
    if (hi == lo) return 0u;
    const double c = floor(((double)p - (double)lo) / ((double)hi - (double)lo) * 1024.0);
    return c >= 1023.0 ? 1023u : (uint32_t)c;
}

// Pass 2: one thread per slot
__global__ void __launch_bounds__(CPLY_THREADS) compress_key_kernel(const __grid_constant__ CompressArgs a) {
    const uint64_t s = (uint64_t)blockIdx.x * CPLY_THREADS + threadIdx.x;
    if (s == 0) *a.sort_n = (uint32_t)a.n;
    if (s >= a.n) return;
    float4 p0;
    uint32_t key = CPLY_NOT_EXPORTED;
    if (cply_exported(a, s, p0)) {
        key = 0u;
        if (a.morton) {
            const CompressBounds &b = *a.bounds;
            key = part1by2(morton_cell(p0.z, order_word_float(b.lo[2]), order_word_float(b.hi[2]))) << 2 |
                  part1by2(morton_cell(p0.y, order_word_float(b.lo[1]), order_word_float(b.hi[1]))) << 1 |
                  part1by2(morton_cell(p0.x, order_word_float(b.lo[0]), order_word_float(b.hi[0])));
        }
    }
    a.keys[s] = key;
    a.vals[s] = (uint32_t)s;
}

__device__ __forceinline__ double cply_norm(float x, float lo, float hi) {
    if (x <= lo) return 0.0;
    if (x >= hi) return 1.0;
    const double r = (double)hi - (double)lo;
    if (r < 1e-5) return 0.0;
    return ((double)x - (double)lo) / r;
}
__device__ __forceinline__ uint32_t cply_unorm(double v, int b) {
    const double t = (double)((1u << b) - 1u), f = floor(v * t + 0.5);
    return (uint32_t)(f < 0.0 ? 0.0 : f > t ? t : f);
}
__device__ __forceinline__ uint32_t cply_pack111011(const float *v, const float *lo, const float *hi) {
    return cply_unorm(cply_norm(v[0], lo[0], hi[0]), 11) << 21 | cply_unorm(cply_norm(v[1], lo[1], hi[1]), 10) << 11 |
           cply_unorm(cply_norm(v[2], lo[2], hi[2]), 11);
}
__device__ __forceinline__ uint32_t cply_sh_byte(float v) {
    if (v != v) return 128u;
    const double t = trunc(((double)v / 8.0 + 0.5) * 256.0);
    return t < 0.0 ? 0u : t > 255.0 ? 255u : (uint32_t)t;
}
// q = (w, x, y, z): the largest component's index and the other three, sign-fixed, at 10 bits each
__device__ __forceinline__ uint32_t cply_pack_rotation(const float *q) {
    uint32_t i = 0u;
    float m = fabsf(q[0]), qi = q[0];
#pragma unroll
    for (int k = 1; k < 4; ++k)
        if (fabsf(q[k]) > m) { m = fabsf(q[k]); qi = q[k]; i = (uint32_t)k; }
    uint32_t word = i << 30, shift = 20u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if ((uint32_t)k == i) continue;
        const float v = qi < 0.0f ? -q[k] : q[k];
        word |= cply_unorm((double)v * 0.7071067811865476 + 0.5, 10) << shift;
        shift -= 10u;
    }
    return word;
}

// Pass 3: chunk blockIdx.x, row r = 256 chunk + thread, splat vals[r]
constexpr int CPLY_SH_BYTES_MAX = 45;   // cply_sh_bytes(3)
template <int BANDS, bool HALF>
__global__ void __launch_bounds__(CPLY_THREADS) compress_chunk_kernel(const __grid_constant__ CompressArgs a) {
    constexpr int K = sh_coeffs(BANDS), P = sh_planes(BANDS, HALF);
    __shared__ uint32_t s_words[CPLY_THREADS * 4];
    __shared__ uint32_t s_sh[CPLY_THREADS * CPLY_SH_BYTES_MAX / 4];
    __shared__ uint32_t s_red[CPLY_WARPS][18];
    __shared__ float s_chunk[18];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint64_t row0 = (uint64_t)blockIdx.x * CPLY_CHUNK;
    const uint32_t here = (uint32_t)(a.rows - row0 < CPLY_CHUNK ? a.rows - row0 : CPLY_CHUNK);
    const bool live = tid < here;
    const int Kd = (a.degree + 1) * (a.degree + 1), Pd = HALF ? (3 * Kd + 7) / 8 : (3 * Kd + 3) / 4;
    const uint32_t SB = cply_sh_bytes(a.degree);
    // v[0..2] position, v[3..5] log-scales, v[6..8] colour: the sanitised values of the chunk statistics
    float v[9], alpha = 0.0f, q[4] = {1.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = 0.0f;
    if (live) {
        const uint64_t s = a.vals[row0 + tid], st = a.plane_stride;
        const float4 *src = a.soa + s;
        const float4 p0 = __ldg(src), p1 = __ldg(src + st), p2 = __ldg(src + 2 * st);
        float c[HALF ? 8 * P : 4 * P];
#pragma unroll
        for (int k = 0; k < P; ++k) {
            float4 w = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            if (k < Pd) w = __ldg(src + (uint64_t)(3 + k) * st);
            if constexpr (HALF) {
                const uint32_t u[4] = {__float_as_uint(w.x), __float_as_uint(w.y), __float_as_uint(w.z), __float_as_uint(w.w)};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    c[8 * k + 2 * j] = half_bits_to_float(u[j] & 0xFFFFu);
                    c[8 * k + 2 * j + 1] = half_bits_to_float(u[j] >> 16);
                }
            } else {
                c[4 * k + 0] = w.x; c[4 * k + 1] = w.y; c[4 * k + 2] = w.z; c[4 * k + 3] = w.w;
            }
        }
        float sr[7];
        export_scale_rot(p1, p2, sr);
        v[0] = p0.x; v[1] = p0.y; v[2] = p0.z;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float ls = sr[k];
            v[3 + k] = ls != ls ? -20.0f : ls < -20.0f ? -20.0f : ls > 20.0f ? 20.0f : ls;
            const float col = (float)((double)c[k] * 0.28209479177387814 + 0.5);
            v[6 + k] = col != col ? 0.5f : col < -64.0f ? -64.0f : col > 64.0f ? 64.0f : col;
        }
        q[0] = sr[3]; q[1] = sr[4]; q[2] = sr[5]; q[3] = sr[6];
        alpha = p2.z != p2.z ? 0.0f : p2.z < 0.0f ? 0.0f : p2.z > 1.0f ? 1.0f : p2.z;
        // SH bytes, channel-major: byte ch (Kd - 1) + (k - 1) holds coefficient k of channel ch
        unsigned char *b = reinterpret_cast<unsigned char *>(s_sh) + (size_t)tid * SB;
#pragma unroll
        for (int k = 1; k < K; ++k) {
            if (k < Kd) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) b[ch * (Kd - 1) + (k - 1)] = (unsigned char)cply_sh_byte(c[3 * k + ch]);
            }
        }
    }
    // the chunk's bounds: order-preserving words, a warp butterfly, then across the warps
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        const uint32_t w = float_order_word(v[k]);
        const uint32_t lo = warp_min_u32(live ? w : 0xFFFFFFFFu), hi = warp_max_u32(live ? w : 0u);
        if (lane == 0u) { s_red[warp][(k / 3) * 6 + k % 3] = lo; s_red[warp][(k / 3) * 6 + 3 + k % 3] = hi; }
    }
    __syncthreads();
    if (tid < 18u) {
        const bool is_max = (tid % 6u) >= 3u;
        uint32_t r = s_red[0][tid];
        for (uint32_t w = 1; w < (uint32_t)CPLY_WARPS; ++w) {
            const uint32_t o = s_red[w][tid];
            r = is_max ? (o > r ? o : r) : (o < r ? o : r);
        }
        s_chunk[tid] = order_word_float(r);
    }
    __syncthreads();
    if (live) {
        const float *ck = s_chunk;
        uint32_t *w = s_words + 4 * tid;
        w[0] = cply_pack111011(v, ck + 0, ck + 3);
        w[1] = cply_pack_rotation(q);
        w[2] = cply_pack111011(v + 3, ck + 6, ck + 9);
        w[3] = cply_unorm(cply_norm(v[6], ck[12], ck[15]), 8) << 24 | cply_unorm(cply_norm(v[7], ck[13], ck[16]), 8) << 16 |
               cply_unorm(cply_norm(v[8], ck[14], ck[17]), 8) << 8 | cply_unorm((double)alpha, 8);
    }
    __syncthreads();
    if (tid < CPLY_CHUNK_FLOATS) a.chunks[(uint64_t)blockIdx.x * CPLY_CHUNK_FLOATS + tid] = s_chunk[tid];
    uint32_t *pk = a.packed + row0 * 4ull;
    for (uint32_t i = tid; i < 4u * here; i += CPLY_THREADS) pk[i] = s_words[i];
    if (SB) {
        const uint32_t bytes = here * SB;
        uint8_t *dst = a.sh + row0 * SB;
        const unsigned char *sb = reinterpret_cast<const unsigned char *>(s_sh);
        uint32_t done = 0u;
        if ((reinterpret_cast<uintptr_t>(dst) & 3u) == 0u) {   // (row0 SB is a multiple of 4: only the base pointer decides)
            uint32_t *dw = reinterpret_cast<uint32_t *>(dst);
            for (uint32_t i = tid; i < bytes / 4u; i += CPLY_THREADS) dw[i] = s_sh[i];
            done = bytes & ~3u;
        }
        for (uint32_t i = done + tid; i < bytes; i += CPLY_THREADS) dst[i] = sb[i];
    }
}

}  // namespace

#ifndef GSR_CPU_EMU  // host side: CUDA only (tests/compressed_reference drives the kernels above itself)

namespace {
template <int BANDS, bool HALF>
void launch_chunk_variant(const CompressArgs &a, uint32_t blocks, cudaStream_t stream) {
    compress_chunk_kernel<BANDS, HALF><<<blocks, CPLY_THREADS, 0, stream>>>(a);
}
}  // namespace

int launch_compress_bounds(const CompressArgs &a, cudaStream_t stream) {
    GSR_CUDA_TRY(cudaMemsetAsync(a.bounds->lo, 0xFF, sizeof a.bounds->lo, stream));
    GSR_CUDA_TRY(cudaMemsetAsync(a.bounds->hi, 0, sizeof(CompressBounds) - offsetof(CompressBounds, hi), stream));
    const uint64_t warps = (a.n + 31ull) / 32ull, need = (warps + CPLY_WARPS - 1) / CPLY_WARPS;
    if (!need) return GSR_OK;
    compress_bounds_kernel<<<(uint32_t)(need < 2048ull ? need : 2048ull), CPLY_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_compress_keys(const CompressArgs &a, cudaStream_t stream) {
    const uint64_t blocks = (a.n + CPLY_THREADS - 1) / CPLY_THREADS;
    compress_key_kernel<<<(uint32_t)(blocks ? blocks : 1ull), CPLY_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_compress_chunks(const CompressArgs &a, int bands, bool sh_half, cudaStream_t stream) {
    const uint64_t blocks = (a.rows + CPLY_CHUNK - 1) / CPLY_CHUNK;
    if (!blocks) return GSR_OK;
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: launch_chunk_variant<1, false>(a, (uint32_t)blocks, stream); break;
        case 3: launch_chunk_variant<1, true>(a, (uint32_t)blocks, stream); break;
        case 4: launch_chunk_variant<2, false>(a, (uint32_t)blocks, stream); break;
        case 5: launch_chunk_variant<2, true>(a, (uint32_t)blocks, stream); break;
        case 6: launch_chunk_variant<3, false>(a, (uint32_t)blocks, stream); break;
        case 7: launch_chunk_variant<3, true>(a, (uint32_t)blocks, stream); break;
        case 8: launch_chunk_variant<4, false>(a, (uint32_t)blocks, stream); break;
        default: launch_chunk_variant<4, true>(a, (uint32_t)blocks, stream); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

// Force-load this file's kernels (the lazy-loading rule of DESIGN.md section 6)
int preload_compressed_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_bounds_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_key_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<1, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<1, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<2, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<2, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<3, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<3, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<4, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compress_chunk_kernel<4, true>));
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
