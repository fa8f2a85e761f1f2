// ingest.cu -- AoS -> SoA transposition of uploaded splats.
//
// The reference keeps the 60-float std430 `Splat` struct in one AoS storage buffer
// (gsplat_projection.glsl:33-40, written by util/ply_file.gd:71).  libgsr accepts exactly that struct at the
// boundary (gsr_upload_splats_aos) and stores it as 15 float4 planes (fewer for a store of a lower SH degree) so that the projection kernel issues
// coalesced 128-bit loads and culled splats touch one plane only.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int SPLATS_PER_BLOCK = 128;

// `planes` = soa_planes(store bands): the SH planes past them are not stored, and the floats of the last stored SH plane past the store's
// 3K coefficients are written as 0 (the AoS struct holds the next degree's coefficients there).
// HALF (GSR_FLAG_SH_HALF; planes = soa_planes(store bands, true)): SH plane p holds the 8 values 8p .. 8p + 7 of the struct's SH floats
// rounded to binary16 (sh_half), values past 3K as +0.
template <bool HALF = false>
__global__ void __launch_bounds__(256) aos_to_soa_kernel(const float4 *__restrict__ aos, uint64_t count, float4 *__restrict__ soa,
                                                         uint64_t plane_stride, uint64_t first, int planes = NUM_PLANES) {
    __shared__ float4 s[SPLATS_PER_BLOCK * NUM_PLANES];
    const uint64_t s0 = (uint64_t)blockIdx.x * SPLATS_PER_BLOCK;
    const uint32_t here = (uint32_t)((count - s0) < (uint64_t)SPLATS_PER_BLOCK ? (count - s0) : SPLATS_PER_BLOCK);
    const float4 *src = aos + s0 * NUM_PLANES;
    for (uint32_t i = threadIdx.x; i < here * NUM_PLANES; i += blockDim.x) s[i] = src[i];  // coalesced AoS read
    __syncthreads();
    if constexpr (HALF) {
        // SH values of the store: 3K = 3, 12, 27, 48 for 1..4 bands
        const uint32_t nvals = planes == soa_planes(1, true) ? 3u : planes == soa_planes(2, true) ? 12u : planes == soa_planes(3, true) ? 27u : 48u;
        const float *sf = reinterpret_cast<const float *>(s);
        for (uint32_t i = threadIdx.x; i < here * (uint32_t)planes; i += blockDim.x) {
            const uint32_t plane = i / here, k = i - plane * here;
            float4 v;
            if (plane < 3u) {
                v = s[k * NUM_PLANES + plane];
            } else {
                const uint32_t v0 = 8u * (plane - 3u);
                const float *c = sf + (size_t)k * (4 * NUM_PLANES) + 12u + v0;   // the struct's SH floats start at float 12
                uint32_t w[4];
#pragma unroll
                for (uint32_t j = 0; j < 4; ++j)
                    w[j] = sh_half2(v0 + 2u * j < nvals ? c[2 * j] : 0.0f, v0 + 2u * j + 1u < nvals ? c[2 * j + 1] : 0.0f);
                v = make_float4(__uint_as_float(w[0]), __uint_as_float(w[1]), __uint_as_float(w[2]), __uint_as_float(w[3]));
            }
            soa[(uint64_t)plane * plane_stride + first + s0 + k] = v;
        }
        return;
    }
    // valid floats of the last stored plane: 3K - 4(P - 1) = 3, 4, 3, 4 for 1..4 bands
    const uint32_t tail = (planes == soa_planes(1) || planes == soa_planes(3)) ? 3u : 4u;
    for (uint32_t i = threadIdx.x; i < here * (uint32_t)planes; i += blockDim.x) {
        const uint32_t plane = i / here, k = i - plane * here;  // consecutive threads -> consecutive splats of one plane
        float4 v = s[k * NUM_PLANES + plane];
        if (plane == (uint32_t)planes - 1u && tail == 3u) v.w = 0.0f;
        soa[(uint64_t)plane * plane_stride + first + s0 + k] = v;
    }
}

// ---- scope row f1: PLY vertex -> Splat on the device (util/ply_file.gd:44-69) -------------------------------------
// One thread per vertex; a CTA stages its 128 vertices (nprops floats each, standard 3DGS property order) through
// shared memory so that the AoS read is coalesced, then every thread evaluates exp(scale) and the sigmoid in float64
// (GDScript floats are doubles; the results are narrowed when they enter Vector3 / PackedFloat32Array), builds
// Basis(Quaternion).transposed(), Sigma = (S R)^T (S R) with Godot's Basis*Basis operation order (including the
// structurally-zero products, so signed zeros match), re-interleaves the SH coefficients and writes the stored SoA planes (15 for a degree-3 store).
constexpr int INGEST_SPLATS = 128;

__device__ __forceinline__ void godot_basis_mul(const float a[3][3], const float b[3][3], float o[3][3]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) o[i][j] = (b[0][j] * a[i][0] + b[1][j] * a[i][1]) + b[2][j] * a[i][2];
}

// The stored planes of splat `id` from the float values of its PLY vertex, the rule of gsr_upload_ply after exp(scale) and the sigmoid
// (sc0..2 and opacity): Basis(Quaternion(pr[1], pr[2], pr[3], pr[0])).transposed(), Sigma = (S R)^T (S R) with Godot's Basis*Basis
// operation order (including the structurally-zero products, so signed zeros match), then the SH re-interleave.  pf[i] is f_rest value i
// of a file of SH degree `degree`, channel-major (value c rest + k is coefficient k + 1 of channel c, rest = (degree + 1)^2 - 1); it is
// read only for k < rest.  This is the per-splat half of ply_to_soa_kernel, statement for statement, for compressed_to_soa_kernel; the
// older kernel keeps its own copy of the text because routing it through this function changes its register allocation, and the
// library keeps the SASS of its existing kernels unchanged when it adds new ones.  tests/test_compressed_ply.py holds both to the same rule.
template <bool HALF, class RestValues>
__device__ __forceinline__ void store_ply_splat(float4 *__restrict__ soa, uint64_t plane_stride, uint64_t id, int planes, const float *px,
                                                float creation_time, float sc0, float sc1, float sc2, float opacity, const float *pr,
                                                const float *pd, uint32_t degree, RestValues pf) {
    const float qx = pr[1], qy = pr[2], qz = pr[3], qw = pr[0];  // Quaternion(rot_1, rot_2, rot_3, rot_0)
    const float d = ((qx * qx + qy * qy) + qz * qz) + qw * qw;
    const float s = 2.0f / d;
    const float xs = qx * s, ys = qy * s, zs = qz * s;
    const float wx = qw * xs, wy = qw * ys, wz = qw * zs;
    const float xx = qx * xs, xy = qx * ys, xz = qx * zs;
    const float yy = qy * ys, yz = qy * zs, zz = qz * zs;
    const float Bq[3][3] = {{1.0f - (yy + zz), xy - wz, xz + wy}, {xy + wz, 1.0f - (xx + zz), yz - wx}, {xz - wy, yz + wx, 1.0f - (xx + yy)}};
    float R[3][3], M[3][3], Mt[3][3], Cv[3][3];
    const float S[3][3] = {{sc0, 0.0f, 0.0f}, {0.0f, sc1, 0.0f}, {0.0f, 0.0f, sc2}};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[r][c] = Bq[c][r];  // .transposed()
    godot_basis_mul(S, R, M);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) Mt[r][c] = M[c][r];
    godot_basis_mul(Mt, M, Cv);

    soa[0 * plane_stride + id] = make_float4(px[0], px[1], px[2], creation_time);
    soa[1 * plane_stride + id] = make_float4(Cv[0][0], Cv[0][1], Cv[0][2], Cv[1][1]);
    soa[2 * plane_stride + id] = make_float4(Cv[1][2], Cv[2][2], opacity, 0.0f);
    // coefficient-major RGB: DC, then f_rest R | G | B (rest = K_file - 1 floats per channel) re-interleaved (:65-69)
    const uint32_t rest = (degree + 1u) * (degree + 1u) - 1u;
    const uint32_t kept = (uint32_t)(planes - 3) == (uint32_t)sh_planes(4, HALF) ? 16u : (uint32_t)(planes - 3) == (uint32_t)sh_planes(3, HALF) ? 9u
                        : (uint32_t)(planes - 3) == (uint32_t)sh_planes(2, HALF) ? 4u : 1u;   // K of the store
    float sh[48];
    sh[0] = pd[0]; sh[1] = pd[1]; sh[2] = pd[2];
#pragma unroll
    for (uint32_t k = 0; k < 15; ++k) {
        const bool in = k < rest && k + 1u < kept;
        const uint32_t kr = in ? k : 0u;
        sh[3 + 3 * k + 0] = in ? pf[kr] : 0.0f;
        sh[3 + 3 * k + 1] = in ? pf[rest + kr] : 0.0f;
        sh[3 + 3 * k + 2] = in ? pf[2 * rest + kr] : 0.0f;
    }
    if constexpr (HALF) {   // (every value past the store's 3K is 0 already)
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (k < planes - 3)
                soa[(uint64_t)(3 + k) * plane_stride + id] = make_float4(__uint_as_float(sh_half2(sh[8 * k], sh[8 * k + 1])), __uint_as_float(sh_half2(sh[8 * k + 2], sh[8 * k + 3])),
                                                                         __uint_as_float(sh_half2(sh[8 * k + 4], sh[8 * k + 5])), __uint_as_float(sh_half2(sh[8 * k + 6], sh[8 * k + 7])));
        return;
    }
#pragma unroll
    for (int k = 0; k < 12; ++k)
        if (k < planes - 3) soa[(uint64_t)(3 + k) * plane_stride + id] = make_float4(sh[4 * k], sh[4 * k + 1], sh[4 * k + 2], sh[4 * k + 3]);
}

// `lay` names the property groups of a vertex (gsr_ply_layout; default: the standard 62-property layout) and `planes` = soa_planes(store
// bands) the planes written.  SH coefficients above the file's degree are stored as 0, those above the store's degree are dropped.
// HALF (GSR_FLAG_SH_HALF; planes = soa_planes(store bands, true)): the SH planes are written as packed binary16 values (sh_half), 8 per
// plane in the same coefficient-major order, values past 3K as +0.
// FILTER3D (gsr_upload_ply_filtered): property `filter_3d` is Mip-Splatting's per-splat 3D filter f.  With f > 0 the splat is stored
// with the filter folded in, in float64 and narrowed once: q_i = exp(scale_i)^2, q'_i = q_i + f*f, scale_i = sqrt(q'_i) and opacity =
// sigmoid * sqrt((q_0 q_1 q_2) / (q'_0 q'_1 q'_2)).  f <= 0 or NaN: stored exactly as without the filter.
template <bool FILTER3D = false, bool HALF = false>
__global__ void __launch_bounds__(INGEST_SPLATS) ply_to_soa_kernel(const float *__restrict__ ply, uint32_t nprops, uint64_t count, float creation_time,
                                                                  float4 *__restrict__ soa, uint64_t plane_stride, uint64_t first,
                                                                  const gsr_ply_layout lay = PLY_LAYOUT_3DGS, int planes = NUM_PLANES,
                                                                  int32_t filter_3d = -1) {
#ifndef GSR_CPU_EMU
    extern __shared__ float s_v[];  // [INGEST_SPLATS][nprops]
#else  // tests/kernel_emu (CPU logic pre-flight): nprops <= 256 (gsr_upload_ply rejects more)
    __shared__ float s_v[INGEST_SPLATS * 256];
#endif
    const uint64_t s0 = (uint64_t)blockIdx.x * INGEST_SPLATS;
    const uint32_t here = (uint32_t)((count - s0) < (uint64_t)INGEST_SPLATS ? (count - s0) : INGEST_SPLATS);
    const float *src = ply + s0 * nprops;
    for (uint32_t i = threadIdx.x; i < here * nprops; i += blockDim.x) s_v[i] = src[i];
    __syncthreads();
    if (threadIdx.x >= here) return;
    const float *p = s_v + (size_t)threadIdx.x * nprops;
    const uint64_t id = first + s0 + threadIdx.x;

    const float *ps = p + lay.scale, *pr = p + lay.rot, *px = p + lay.x, *pd = p + lay.f_dc;
    const double e0 = exp((double)ps[0]), e1 = exp((double)ps[1]), e2 = exp((double)ps[2]);
    const double sigmoid = 1.0 / (1.0 + exp(-(double)p[lay.opacity]));
    float sc0 = (float)e0, sc1 = (float)e1, sc2 = (float)e2, opacity = (float)sigmoid;
    if constexpr (FILTER3D) {
        const double f = (double)p[filter_3d];
        if (f > 0.0) {
            const double q0 = e0 * e0, q1 = e1 * e1, q2 = e2 * e2, ff = f * f;
            const double g0 = q0 + ff, g1 = q1 + ff, g2 = q2 + ff;
            sc0 = (float)sqrt(g0); sc1 = (float)sqrt(g1); sc2 = (float)sqrt(g2);
            opacity = (float)(sigmoid * sqrt(((q0 * q1) * q2) / ((g0 * g1) * g2)));
        }
    }
    const float qx = pr[1], qy = pr[2], qz = pr[3], qw = pr[0];  // Quaternion(rot_1, rot_2, rot_3, rot_0)
    const float d = ((qx * qx + qy * qy) + qz * qz) + qw * qw;
    const float s = 2.0f / d;
    const float xs = qx * s, ys = qy * s, zs = qz * s;
    const float wx = qw * xs, wy = qw * ys, wz = qw * zs;
    const float xx = qx * xs, xy = qx * ys, xz = qx * zs;
    const float yy = qy * ys, yz = qy * zs, zz = qz * zs;
    const float Bq[3][3] = {{1.0f - (yy + zz), xy - wz, xz + wy}, {xy + wz, 1.0f - (xx + zz), yz - wx}, {xz - wy, yz + wx, 1.0f - (xx + yy)}};
    float R[3][3], M[3][3], Mt[3][3], Cv[3][3];
    const float S[3][3] = {{sc0, 0.0f, 0.0f}, {0.0f, sc1, 0.0f}, {0.0f, 0.0f, sc2}};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[r][c] = Bq[c][r];  // .transposed()
    godot_basis_mul(S, R, M);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) Mt[r][c] = M[c][r];
    godot_basis_mul(Mt, M, Cv);

    soa[0 * plane_stride + id] = make_float4(px[0], px[1], px[2], creation_time);
    soa[1 * plane_stride + id] = make_float4(Cv[0][0], Cv[0][1], Cv[0][2], Cv[1][1]);
    soa[2 * plane_stride + id] = make_float4(Cv[1][2], Cv[2][2], opacity, 0.0f);
    // coefficient-major RGB: DC, then f_rest R | G | B (rest = K_file - 1 floats per channel) re-interleaved (:65-69)
    const uint32_t rest = (lay.sh_degree + 1u) * (lay.sh_degree + 1u) - 1u;
    const uint32_t kept = (uint32_t)(planes - 3) == (uint32_t)sh_planes(4, HALF) ? 16u : (uint32_t)(planes - 3) == (uint32_t)sh_planes(3, HALF) ? 9u
                        : (uint32_t)(planes - 3) == (uint32_t)sh_planes(2, HALF) ? 4u : 1u;   // K of the store
    const float *pf = p + (lay.f_rest < 0 ? 0 : lay.f_rest);   // every index below stays inside the vertex, also for a coefficient not read
    float sh[48];
    sh[0] = pd[0]; sh[1] = pd[1]; sh[2] = pd[2];
#pragma unroll
    for (uint32_t k = 0; k < 15; ++k) {
        const bool in = k < rest && k + 1u < kept;
        const uint32_t kr = in ? k : 0u;
        sh[3 + 3 * k + 0] = in ? pf[kr] : 0.0f;
        sh[3 + 3 * k + 1] = in ? pf[rest + kr] : 0.0f;
        sh[3 + 3 * k + 2] = in ? pf[2 * rest + kr] : 0.0f;
    }
    if constexpr (HALF) {   // (every value past the store's 3K is 0 already)
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (k < planes - 3)
                soa[(uint64_t)(3 + k) * plane_stride + id] = make_float4(__uint_as_float(sh_half2(sh[8 * k], sh[8 * k + 1])), __uint_as_float(sh_half2(sh[8 * k + 2], sh[8 * k + 3])),
                                                                         __uint_as_float(sh_half2(sh[8 * k + 4], sh[8 * k + 5])), __uint_as_float(sh_half2(sh[8 * k + 6], sh[8 * k + 7])));
        return;
    }
#pragma unroll
    for (int k = 0; k < 12; ++k)
        if (k < planes - 3) soa[(uint64_t)(3 + k) * plane_stride + id] = make_float4(sh[4 * k], sh[4 * k + 1], sh[4 * k + 2], sh[4 * k + 3]);
}

// ---- gsr_upload_compressed_ply: compressed PLY rows -> the stored planes (include/gsr.h "Compressed PLY") ----
// One CTA per chunk, one thread per row.  The CTA stages its chunk floats, packed words and SH bytes through shared memory (contiguous
// loads), every thread decodes its row into the float values of a 3DGS vertex in float32, one IEEE operation at a time, and stores
// them with ply_to_soa_kernel's per-splat code; the alpha is stored directly.  BANDS, HALF: the store's.
constexpr int CPLY_DECODE_THREADS = 256;
static_assert(CPLY_DECODE_THREADS == (int)CPLY_CHUNK, "one thread per row of a chunk");
__device__ __forceinline__ float cply_lerp(float lo, float hi, float u) { return lo + (hi - lo) * u; }
// A row's SH bytes as the f_rest values of store_ply_splat: the midpoint of bin q
struct ShBins {
    const unsigned char *q;
    __device__ __forceinline__ float operator[](uint32_t i) const { return ((float)q[i] + 0.5f) * 0.03125f - 4.0f; }
};
template <int BANDS, bool HALF>
__global__ void __launch_bounds__(CPLY_DECODE_THREADS) compressed_to_soa_kernel(const __grid_constant__ DecompressArgs a) {
    __shared__ uint32_t s_words[CPLY_DECODE_THREADS * 4];
    __shared__ uint32_t s_sh[CPLY_DECODE_THREADS * 45 / 4];
    __shared__ float s_chunk[18];
    const uint32_t tid = threadIdx.x, cf = a.chunk_floats;
    const uint64_t row0 = (uint64_t)blockIdx.x * CPLY_CHUNK;
    const uint32_t here = (uint32_t)(a.rows - row0 < CPLY_CHUNK ? a.rows - row0 : CPLY_CHUNK);
    const uint32_t rest = (uint32_t)((a.degree + 1) * (a.degree + 1) - 1), SB = 3u * rest;
    if (tid < cf) s_chunk[tid] = a.chunks[(uint64_t)blockIdx.x * cf + tid];
    const uint32_t *pk = a.packed + row0 * 4ull;
    for (uint32_t i = tid; i < 4u * here; i += CPLY_DECODE_THREADS) s_words[i] = pk[i];
    if (SB) {
        const uint32_t bytes = here * SB;
        const uint8_t *src = a.sh + row0 * SB;
        unsigned char *sb = reinterpret_cast<unsigned char *>(s_sh);
        uint32_t done = 0u;
        if ((reinterpret_cast<uintptr_t>(src) & 3u) == 0u) {   // (row0 SB is a multiple of 4: only the base pointer decides)
            const uint32_t *sw = reinterpret_cast<const uint32_t *>(src);
            for (uint32_t i = tid; i < bytes / 4u; i += CPLY_DECODE_THREADS) s_sh[i] = sw[i];
            done = bytes & ~3u;
        }
        for (uint32_t i = done + tid; i < bytes; i += CPLY_DECODE_THREADS) sb[i] = src[i];
    }
    __syncthreads();
    if (tid >= here) return;
    const float *ck = s_chunk;
    const uint32_t *w = s_words + 4 * tid;
    const uint32_t wp = w[0], wr = w[1], ws = w[2], wc = w[3];
    const float px[3] = {cply_lerp(ck[0], ck[3], (float)(wp >> 21) / 2047.0f), cply_lerp(ck[1], ck[4], (float)((wp >> 11) & 1023u) / 1023.0f),
                         cply_lerp(ck[2], ck[5], (float)(wp & 2047u) / 2047.0f)};
    const float ls[3] = {cply_lerp(ck[6], ck[9], (float)(ws >> 21) / 2047.0f), cply_lerp(ck[7], ck[10], (float)((ws >> 11) & 1023u) / 1023.0f),
                         cply_lerp(ck[8], ck[11], (float)(ws & 2047u) / 2047.0f)};
    float pd[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float u = (float)((wc >> (24 - 8 * k)) & 255u) / 255.0f;
        const float c = cf == 18u ? cply_lerp(ck[12 + k], ck[15 + k], u) : u;
        pd[k] = (c - 0.5f) / 0.28209479177387814f;
    }
    const float alpha = (float)(wc & 255u) / 255.0f;
    const uint32_t i = wr >> 30;
    const float qa = ((float)((wr >> 20) & 1023u) / 1023.0f - 0.5f) * 1.41421356f, qb = ((float)((wr >> 10) & 1023u) / 1023.0f - 0.5f) * 1.41421356f,
                qc = ((float)(wr & 1023u) / 1023.0f - 0.5f) * 1.41421356f;
    const float t = 1.0f - ((qa * qa + qb * qb) + qc * qc), m = sqrtf(t > 0.0f ? t : 0.0f);
    const float pr[4] = {i == 0u ? m : qa, i == 0u ? qa : i == 1u ? m : qb, i <= 1u ? qb : i == 2u ? m : qc, i == 3u ? m : qc};
    const float sc0 = (float)exp((double)ls[0]), sc1 = (float)exp((double)ls[1]), sc2 = (float)exp((double)ls[2]);
    store_ply_splat<HALF>(a.soa, a.plane_stride, a.first + row0 + tid, soa_planes(BANDS, HALF), px, a.creation_time, sc0, sc1, sc2, alpha, pr, pd,
                          (uint32_t)a.degree, ShBins{reinterpret_cast<const unsigned char *>(s_sh) + (size_t)tid * SB});
}

}  // namespace

#ifndef GSR_CPU_EMU  // host side: CUDA only
// Force-load this file's kernels (CUDA loads modules lazily; a first launch that has to load code while another context's
// kernel spins on a flag this launch would satisfy can stall the host: see gsr_group_attach).
int preload_ingest_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, aos_to_soa_kernel<false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<false, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<true, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, aos_to_soa_kernel<true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<1, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<1, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<2, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<2, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<3, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<3, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<4, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compressed_to_soa_kernel<4, true>));
    return GSR_OK;
}
template <bool FILTER3D, bool HALF>
int launch_ply_variant(const float *ply, const gsr_ply_layout &layout, uint64_t count, float creation_time, float4 *soa, uint64_t plane_stride,
                       uint64_t first, int planes, cudaStream_t stream, int32_t filter_3d) {
    const size_t smem = sizeof(float) * (size_t)INGEST_SPLATS * layout.nprops;
    const uint32_t blocks = (uint32_t)((count + INGEST_SPLATS - 1) / INGEST_SPLATS);
    if (smem > 48 * 1024) GSR_CUDA_TRY(cudaFuncSetAttribute(ply_to_soa_kernel<FILTER3D, HALF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ply_to_soa_kernel<FILTER3D, HALF><<<blocks, INGEST_SPLATS, smem, stream>>>(ply, layout.nprops, count, creation_time, soa, plane_stride, first, layout, planes,
                                                                               filter_3d);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
int launch_ply_to_soa(const float *ply, const gsr_ply_layout &layout, uint64_t count, float creation_time, float4 *soa, uint64_t plane_stride,
                      uint64_t first, int planes, cudaStream_t stream, int32_t filter_3d, bool sh_half) {
    if (count == 0) return GSR_OK;
    if (sh_half) {
        return filter_3d >= 0 ? launch_ply_variant<true, true>(ply, layout, count, creation_time, soa, plane_stride, first, planes, stream, filter_3d)
                              : launch_ply_variant<false, true>(ply, layout, count, creation_time, soa, plane_stride, first, planes, stream, -1);
    }
    const size_t smem = sizeof(float) * (size_t)INGEST_SPLATS * layout.nprops;
    const uint32_t blocks = (uint32_t)((count + INGEST_SPLATS - 1) / INGEST_SPLATS);
    if (filter_3d >= 0) {
        if (smem > 48 * 1024) GSR_CUDA_TRY(cudaFuncSetAttribute(ply_to_soa_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ply_to_soa_kernel<true><<<blocks, INGEST_SPLATS, smem, stream>>>(ply, layout.nprops, count, creation_time, soa, plane_stride, first, layout, planes,
                                                                         filter_3d);
    } else {
        if (smem > 48 * 1024) GSR_CUDA_TRY(cudaFuncSetAttribute(ply_to_soa_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ply_to_soa_kernel<false><<<blocks, INGEST_SPLATS, smem, stream>>>(ply, layout.nprops, count, creation_time, soa, plane_stride, first, layout, planes);
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_aos_to_soa(const float4 *aos, uint64_t count, float4 *soa, uint64_t plane_stride, uint64_t first, int planes, cudaStream_t stream,
                      bool sh_half) {
    if (count == 0) return GSR_OK;
    const uint32_t blocks = (uint32_t)((count + SPLATS_PER_BLOCK - 1) / SPLATS_PER_BLOCK);
    if (sh_half) aos_to_soa_kernel<true><<<blocks, 256, 0, stream>>>(aos, count, soa, plane_stride, first, planes);
    else aos_to_soa_kernel<false><<<blocks, 256, 0, stream>>>(aos, count, soa, plane_stride, first, planes);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
namespace {
template <int BANDS, bool HALF>
void launch_decompress_variant(const DecompressArgs &a, uint32_t blocks, cudaStream_t stream) {
    compressed_to_soa_kernel<BANDS, HALF><<<blocks, CPLY_DECODE_THREADS, 0, stream>>>(a);
}
}  // namespace

int launch_compressed_to_soa(const DecompressArgs &a, int bands, bool sh_half, cudaStream_t stream) {
    const uint64_t blocks = (a.rows + CPLY_CHUNK - 1) / CPLY_CHUNK;
    if (!blocks) return GSR_OK;
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: launch_decompress_variant<1, false>(a, (uint32_t)blocks, stream); break;
        case 3: launch_decompress_variant<1, true>(a, (uint32_t)blocks, stream); break;
        case 4: launch_decompress_variant<2, false>(a, (uint32_t)blocks, stream); break;
        case 5: launch_decompress_variant<2, true>(a, (uint32_t)blocks, stream); break;
        case 6: launch_decompress_variant<3, false>(a, (uint32_t)blocks, stream); break;
        case 7: launch_decompress_variant<3, true>(a, (uint32_t)blocks, stream); break;
        case 8: launch_decompress_variant<4, false>(a, (uint32_t)blocks, stream); break;
        default: launch_decompress_variant<4, true>(a, (uint32_t)blocks, stream); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
