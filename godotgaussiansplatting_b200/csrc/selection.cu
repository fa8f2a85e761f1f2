// selection.cu -- the splat-mask operations of gsr_select_* (include/gsr.h "Splat selection"; DESIGN.md section 5.17).
//
// The masks are one bit per source splat, 32 splats per uint32 word.  The region operations (all, polygon, volume) give every mask word to
// one warp: lane l tests splat 32 w + l, a ballot forms the word's `inside` bits and lane 0 combines them with the word it owns, so no
// update is atomic, even for an instance range that starts inside a word.  The grid covers every word of [0, max_splats): SET clears the
// splats outside the tested range.  The ID-plane operation scatters into a scratch mask with atomicOr (pixels share splats) and a
// second kernel combines it.  Every kernel ends a word with selected &= ~hidden.
// The arithmetic follows the library's deterministic math (-fmad=false): one rounding per operator, in the order of include/gsr.h.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int SEL_THREADS = 256;
constexpr int SEL_WARPS = SEL_THREADS / 32;

__device__ __forceinline__ uint32_t combine_op(uint32_t op, uint32_t selected, uint32_t inside) {
    switch (op) {
        case GSR_SELECT_SET: return inside;
        case GSR_SELECT_ADD: return selected | inside;
        case GSR_SELECT_SUBTRACT: return selected & ~inside;
        default: return selected ^ inside;   // GSR_SELECT_TOGGLE
    }
}

// pix(M, q) of include/gsr.h (the projection's image_pos without the load-in term); w = clip[3]
__device__ __forceinline__ void select_pix(const float *M, float q0, float q1, float q2, float fw, float fh, float &x, float &y, float &w) {
    const float *V = M, *P = M + 16;
    float view[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) view[r] = ((V[0 + r] * q0 + V[4 + r] * q1) + V[8 + r] * q2) + V[12 + r] * 1.0f;
    const float c0 = ((P[0] * view[0] + P[4] * view[1]) + P[8] * view[2]) + P[12] * view[3];
    const float c1 = ((P[1] * view[0] + P[5] * view[1]) + P[9] * view[2]) + P[13] * view[3];
    w = ((P[3] * view[0] + P[7] * view[1]) + P[11] * view[2]) + P[15] * view[3];
    x = ((c0 / w + 1.0f) * 0.5f) * fw;
    y = ((c1 / w + 1.0f) * 0.5f) * fh;
}

// even-odd rule: for every edge a -> b that straddles py, x = (((b.x - a.x) (py - a.y)) / (b.y - a.y)) + a.x, and px < x toggles.
// A NaN px or py never toggles (every comparison is false), so it is outside.
__device__ __forceinline__ bool polygon_inside(const SelectArgs &a, float px, float py) {
    bool in = false;
    float2 p = a.xy[a.n - 1];
#pragma unroll 1
    for (uint32_t i = 0; i < a.n; ++i) {
        const float2 q = a.xy[i];
        if ((p.y > py) != (q.y > py)) {
            const float x = (((q.x - p.x) * (py - p.y)) / (q.y - p.y)) + p.x;
            if (px < x) in = !in;
        }
        p = q;
    }
    return in;
}

template <int KIND>
__global__ void __launch_bounds__(SEL_THREADS) select_region_kernel(const __grid_constant__ SelectArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t w = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5);
    if (w >= a.words) return;   // warp-uniform
    const uint64_t s = 32ull * w + lane;
    bool in = s < a.max_splats && s >= a.first && s - a.first < a.count;
    if constexpr (KIND != SELECT_ALL) {
        if (in) {
            const float4 pt = __ldg(a.plane0 + s);
            const float sp0 = pt.x * a.model_scale, sp1 = pt.y * a.model_scale, sp2 = pt.z * a.model_scale;
            float q0 = sp0, q1 = sp1, q2 = sp2;
            if (a.instanced) {
                q0 = ((a.A[0] * sp0 + a.A[3] * sp1) + a.A[6] * sp2) + a.A[9];
                q1 = ((a.A[1] * sp0 + a.A[4] * sp1) + a.A[7] * sp2) + a.A[10];
                q2 = ((a.A[2] * sp0 + a.A[5] * sp1) + a.A[8] * sp2) + a.A[11];
            }
            if constexpr (KIND == SELECT_POLYGON) {
                float x, y, cw;
                select_pix(a.vp, q0, q1, q2, a.fw, a.fh, x, y, cw);
                in = cw > 0.0f && polygon_inside(a, x, y);
            } else {
                const bool src = (a.vol.kind & 2) != 0;   // GSR_CUTOUT_SOURCE
                in = cutout_inside(a.vol, src ? sp0 : q0, src ? sp1 : q1, src ? sp2 : q2);
            }
        }
    }
    const uint32_t inside = __ballot_sync(0xffffffffu, in);
    if (lane == 0) a.selected[w] = combine_op(a.op, a.selected[w], inside) & ~a.hidden[w];
}

struct IdScatterArgs {
    const uint32_t *ids;
    int32_t width, x0, y0, x1, y1;
    const uint32_t *warp_inst;
    const InstanceDesc *desc;
    uint32_t drawn_warps;
    uint64_t max_splats;
    uint32_t *scratch;
};

__global__ void __launch_bounds__(SEL_THREADS) select_ids_scatter_kernel(const __grid_constant__ IdScatterArgs a) {
    const int32_t rw = a.x1 - a.x0;
    const uint64_t i = (uint64_t)blockIdx.x * SEL_THREADS + threadIdx.x;
    if (i >= (uint64_t)rw * (uint64_t)(a.y1 - a.y0)) return;
    const int32_t x = a.x0 + (int32_t)(i % (uint64_t)rw), y = a.y0 + (int32_t)(i / (uint64_t)rw);
    const uint32_t v = __ldg(a.ids + 2ull * ((uint64_t)y * (uint64_t)a.width + (uint64_t)x));
    if (v == NO_ID) return;
    uint64_t s = v;
    if (a.warp_inst) {   // drawn id v of instance k is source splat first_k + (v - 32 w_k); ids outside the layout are ignored
        if ((v >> 5) >= a.drawn_warps) return;
        const uint32_t k = __ldg(a.warp_inst + (v >> 5));
        if (k == NO_ID) return;
        const InstanceDesc d = a.desc[k];
        const uint32_t j = v - 32u * d.warp0;
        if (j >= d.count) return;
        s = d.first + j;
    }
    if (s >= a.max_splats) return;
    atomicOr(a.scratch + (s >> 5), 1u << (uint32_t)(s & 31u));
}

__global__ void __launch_bounds__(SEL_THREADS) select_combine_kernel(uint32_t *scratch, uint32_t *selected, const uint32_t *hidden, uint32_t words,
                                                                     uint32_t op) {
    const uint32_t w = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (w >= words) return;
    const uint32_t inside = scratch[w];
    scratch[w] = 0u;
    selected[w] = combine_op(op, selected[w], inside) & ~hidden[w];
}

__global__ void __launch_bounds__(SEL_THREADS) hide_selection_kernel(uint32_t *hidden, uint32_t *selected, uint32_t words) {
    const uint32_t w = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (w >= words) return;
    hidden[w] |= selected[w];
    selected[w] = 0u;
}

__global__ void __launch_bounds__(SEL_THREADS) mask_counts_kernel(const uint32_t *selected, const uint32_t *hidden, uint32_t words,
                                                                  unsigned long long *counts) {
    uint32_t ns = 0u, nh = 0u;
    for (uint32_t w = blockIdx.x * SEL_THREADS + threadIdx.x; w < words; w += gridDim.x * SEL_THREADS) {
        ns += __popc(selected[w]);
        nh += __popc(hidden[w]);
    }
    ns = __reduce_add_sync(0xffffffffu, ns);
    nh = __reduce_add_sync(0xffffffffu, nh);
    if ((threadIdx.x & 31u) == 0u) {
        if (ns) atomicAdd(counts + 0, (unsigned long long)ns);
        if (nh) atomicAdd(counts + 1, (unsigned long long)nh);
    }
}

}  // namespace

#ifndef GSR_CPU_EMU
namespace {
uint32_t word_blocks(uint32_t words) { return (words + SEL_THREADS - 1) / SEL_THREADS; }
}  // namespace

int launch_select_region(const SelectArgs &a, int kind, cudaStream_t stream) {
    if (a.words == 0) return GSR_OK;
    const uint32_t blocks = (a.words + SEL_WARPS - 1) / SEL_WARPS;
    switch (kind) {
        case SELECT_ALL: select_region_kernel<SELECT_ALL><<<blocks, SEL_THREADS, 0, stream>>>(a); break;
        case SELECT_POLYGON: select_region_kernel<SELECT_POLYGON><<<blocks, SEL_THREADS, 0, stream>>>(a); break;
        default: select_region_kernel<SELECT_VOLUME><<<blocks, SEL_THREADS, 0, stream>>>(a); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_select_ids(const uint32_t *ids, int32_t width, int32_t x0, int32_t y0, int32_t x1, int32_t y1, const uint32_t *warp_inst,
                      const InstanceDesc *desc, uint32_t drawn_warps, uint64_t max_splats, uint32_t *scratch, uint32_t *selected,
                      const uint32_t *hidden, uint32_t words, uint32_t op, cudaStream_t stream) {
    const uint64_t pixels = (uint64_t)(x1 - x0) * (uint64_t)(y1 - y0);
    if (pixels) {
        IdScatterArgs s{ids, width, x0, y0, x1, y1, warp_inst, desc, drawn_warps, max_splats, scratch};
        select_ids_scatter_kernel<<<(uint32_t)((pixels + SEL_THREADS - 1) / SEL_THREADS), SEL_THREADS, 0, stream>>>(s);
        GSR_CUDA_TRY(cudaGetLastError());
    }
    if (words) {
        select_combine_kernel<<<word_blocks(words), SEL_THREADS, 0, stream>>>(scratch, selected, hidden, words, op);
        GSR_CUDA_TRY(cudaGetLastError());
    }
    return GSR_OK;
}

int launch_hide_selection(uint32_t *hidden, uint32_t *selected, uint32_t words, cudaStream_t stream) {
    if (!words) return GSR_OK;
    hide_selection_kernel<<<word_blocks(words), SEL_THREADS, 0, stream>>>(hidden, selected, words);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_mask_counts(const uint32_t *selected, const uint32_t *hidden, uint32_t words, unsigned long long *counts, cudaStream_t stream) {
    GSR_CUDA_TRY(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), stream));
    if (!words) return GSR_OK;
    const uint32_t blocks = word_blocks(words) < 1024u ? word_blocks(words) : 1024u;
    mask_counts_kernel<<<blocks, SEL_THREADS, 0, stream>>>(selected, hidden, words, counts);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int preload_selection_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_region_kernel<SELECT_ALL>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_region_kernel<SELECT_POLYGON>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_region_kernel<SELECT_VOLUME>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_ids_scatter_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_combine_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, hide_selection_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, mask_counts_kernel));
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
