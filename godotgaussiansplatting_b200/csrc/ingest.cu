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
__global__ void __launch_bounds__(256) aos_to_soa_kernel(const float4 *__restrict__ aos, uint64_t count, float4 *__restrict__ soa,
                                                         uint64_t plane_stride, uint64_t first, int planes = NUM_PLANES) {
    __shared__ float4 s[SPLATS_PER_BLOCK * NUM_PLANES];
    const uint64_t s0 = (uint64_t)blockIdx.x * SPLATS_PER_BLOCK;
    const uint32_t here = (uint32_t)((count - s0) < (uint64_t)SPLATS_PER_BLOCK ? (count - s0) : SPLATS_PER_BLOCK);
    const float4 *src = aos + s0 * NUM_PLANES;
    for (uint32_t i = threadIdx.x; i < here * NUM_PLANES; i += blockDim.x) s[i] = src[i];  // coalesced AoS read
    __syncthreads();
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

// `lay` names the property groups of a vertex (gsr_ply_layout; default: the standard 62-property layout) and `planes` = soa_planes(store
// bands) the planes written.  SH coefficients above the file's degree are stored as 0, those above the store's degree are dropped.
// FILTER3D (gsr_upload_ply_filtered): property `filter_3d` is Mip-Splatting's per-splat 3D filter f.  With f > 0 the splat is stored
// with the filter folded in, in float64 and narrowed once: q_i = exp(scale_i)^2, q'_i = q_i + f*f, scale_i = sqrt(q'_i) and opacity =
// sigmoid * sqrt((q_0 q_1 q_2) / (q'_0 q'_1 q'_2)).  f <= 0 or NaN: stored exactly as without the filter.
template <bool FILTER3D = false>
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
    const uint32_t kept = (uint32_t)(planes - 3) == (uint32_t)sh_planes(4) ? 16u : (uint32_t)(planes - 3) == (uint32_t)sh_planes(3) ? 9u
                        : (uint32_t)(planes - 3) == (uint32_t)sh_planes(2) ? 4u : 1u;   // K of the store
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
#pragma unroll
    for (int k = 0; k < 12; ++k)
        if (k < planes - 3) soa[(uint64_t)(3 + k) * plane_stride + id] = make_float4(sh[4 * k], sh[4 * k + 1], sh[4 * k + 2], sh[4 * k + 3]);
}

}  // namespace

#ifndef GSR_CPU_EMU  // host side: CUDA only
// Force-load this file's kernels (CUDA loads modules lazily; a first launch that has to load code while another context's
// kernel spins on a flag this launch would satisfy can stall the host: see gsr_group_attach).
int preload_ingest_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, ply_to_soa_kernel<true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, aos_to_soa_kernel));
    return GSR_OK;
}
int launch_ply_to_soa(const float *ply, const gsr_ply_layout &layout, uint64_t count, float creation_time, float4 *soa, uint64_t plane_stride,
                      uint64_t first, int planes, cudaStream_t stream, int32_t filter_3d) {
    if (count == 0) return GSR_OK;
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

int launch_aos_to_soa(const float4 *aos, uint64_t count, float4 *soa, uint64_t plane_stride, uint64_t first, int planes, cudaStream_t stream) {
    if (count == 0) return GSR_OK;
    const uint32_t blocks = (uint32_t)((count + SPLATS_PER_BLOCK - 1) / SPLATS_PER_BLOCK);
    aos_to_soa_kernel<<<blocks, 256, 0, stream>>>(aos, count, soa, plane_stride, first, planes);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
