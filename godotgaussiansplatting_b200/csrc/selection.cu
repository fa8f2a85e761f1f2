// selection.cu -- the splat-mask operations of gsr_select_* (include/gsr.h "Splat selection"; DESIGN.md section 5.17).
//
// The masks are one bit per source splat, 32 splats per uint32 word.  The region operations (all, polygon, volume) give every mask word to
// one warp: lane l tests splat 32 w + l, a ballot forms the word's `inside` bits and lane 0 combines them with the word it owns, so no
// update is atomic, even for an instance range that starts inside a word.  The grid covers every word of [0, max_splats): SET clears the
// splats outside the tested range.  The ID-plane operation scatters into a scratch mask with atomicOr (pixels share splats) and a
// second kernel combines it.  Every kernel ends a word with selected &= ~hidden.  Delete and duplicate (compact_store_kernel) move whole
// splats between indices with one chained scan over the mask words; export (export_ply_kernel) places its PLY rows with the same scan and
// decomposes each covariance in float64.  Property selection (select_where_kernel) has the region
// operations' shape and tests the stored words; the property histogram (splat_histogram_kernel) is a grid-stride pass with the same reads.
// The arithmetic follows the library's deterministic math (-fmad=false): one rounding per operator, in the order of include/gsr.h.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int SEL_THREADS = 256;
constexpr int SEL_WARPS = SEL_THREADS / 32;

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

// The SH planes of one splat in the edit kernels: `src` / `dst` point at plane 0 of the splat, P = sh_planes(BANDS, HALF) planes follow
// plane 2.  Unpack: every stored value into c[] (a binary16 half widened, which is exact), and the raw words holding binary16 values 0-3.
template <int BANDS, bool HALF>
__device__ __forceinline__ void sh_unpack(const float4 *src, uint64_t st, float (&c)[HALF ? 8 * sh_planes(BANDS, HALF) : 4 * sh_planes(BANDS, HALF)],
                                          uint32_t (&dc_words)[2]) {
    constexpr int P = sh_planes(BANDS, HALF);
#pragma unroll
    for (int k = 0; k < P; ++k) {
        const float4 v = src[(uint64_t)(3 + k) * st];
        if constexpr (HALF) {
            const uint32_t u[4] = {__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w)};
            if (k == 0) { dc_words[0] = u[0]; dc_words[1] = u[1]; }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                c[8 * k + 2 * j] = half_bits_to_float(u[j] & 0xFFFFu);
                c[8 * k + 2 * j + 1] = half_bits_to_float(u[j] >> 16);
            }
        } else {
            c[4 * k + 0] = v.x; c[4 * k + 1] = v.y; c[4 * k + 2] = v.z; c[4 * k + 3] = v.w;
        }
    }
}

// Pack: c[] back into the planes, binary16 values as h(c) (sh_half: the upload's rounding), the slots past 3K +0.  KEEP_DC: a binary16
// store's DC halves are written from dc_words as they were stored (a float store's DC values are c[0..2] either way).
template <int BANDS, bool HALF, bool KEEP_DC>
__device__ __forceinline__ void sh_pack(float4 *dst, uint64_t st, const float (&c)[HALF ? 8 * sh_planes(BANDS, HALF) : 4 * sh_planes(BANDS, HALF)],
                                        const uint32_t (&dc_words)[2]) {
    constexpr int NV = 3 * sh_coeffs(BANDS), P = sh_planes(BANDS, HALF), DC = KEEP_DC ? 3 : 0;
#pragma unroll
    for (int k = 0; k < P; ++k) {
        uint32_t u[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (HALF) {
                const int i = 8 * k + 2 * j;
                const uint32_t lo = i < DC ? (dc_words[i >> 1] & 0xFFFFu) : i < NV ? sh_half(c[i]) : 0u;
                const uint32_t hi = i + 1 < DC ? (dc_words[(i + 1) >> 1] >> 16) : i + 1 < NV ? sh_half(c[i + 1]) : 0u;
                u[j] = lo | (hi << 16);
            } else {
                u[j] = 4 * k + j < NV ? __float_as_uint(c[4 * k + j]) : 0u;
            }
        }
        dst[(uint64_t)(3 + k) * st] = make_float4(__uint_as_float(u[0]), __uint_as_float(u[1]), __uint_as_float(u[2]), __uint_as_float(u[3]));
    }
}

// gsr_transform_selection: every selected splat s of the store is rewritten from its planes in `src` (include/gsr.h "Splat transform
// edits").  Like the region kernels a warp owns one mask word: a warp whose word is 0 leaves after that one load, and the lanes of a
// selected warp read consecutive 16-byte words of every plane.  Unselected splats are never written (a hidden splat is never selected).
// In float32, one rounding per operation, no contraction: position L x + t, covariance (L S) L^T (the six stored entries), SH band l
// c'_j = sum_i c_i M~_l[i][j] left to right per channel; creation time, opacity, plane-2 pad and DC copied bit for bit, slots past 3K +0.
template <int BANDS, bool HALF>
__global__ void __launch_bounds__(SEL_THREADS) transform_selection_kernel(const __grid_constant__ TransformArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t w = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5);
    if (w >= a.words) return;   // warp-uniform
    const uint32_t word = a.selected[w];
    if (((word >> lane) & 1u) == 0u) return;
    const uint64_t s = 32ull * w + lane, st = a.plane_stride;
    const float4 *src = a.src + s;
    float4 *dst = a.dst + s;
    const float *L = a.m;
    const float4 p0 = src[0], p1 = src[st], p2 = src[2 * st];
    const float x[3] = {p0.x, p0.y, p0.z};
    float q[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        q[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L[r], x[0]), __fmul_rn(L[3 + r], x[1])), __fmul_rn(L[6 + r], x[2])), L[9 + r]);
    const float S[3][3] = {{p1.x, p1.y, p1.z}, {p1.y, p1.w, p2.x}, {p1.z, p2.x, p2.y}};
    float G[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            G[r][c] = __fadd_rn(__fadd_rn(__fmul_rn(L[r], S[0][c]), __fmul_rn(L[3 + r], S[1][c])), __fmul_rn(L[6 + r], S[2][c]));
    float E[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c)
            E[r][c] = __fadd_rn(__fadd_rn(__fmul_rn(G[r][0], L[c]), __fmul_rn(G[r][1], L[3 + c])), __fmul_rn(G[r][2], L[6 + c]));
    dst[0] = make_float4(q[0], q[1], q[2], p0.w);
    dst[st] = make_float4(E[0][0], E[0][1], E[0][2], E[1][1]);
    dst[2 * st] = make_float4(E[1][2], E[2][2], p2.z, p2.w);

    constexpr int P = sh_planes(BANDS, HALF);
    float c[HALF ? 8 * P : 4 * P];
    uint32_t dc_words[2] = {0u, 0u};   // binary16: the words holding values 0-3 (the DC halves are copied as stored)
    sh_unpack<BANDS, HALF>(src, st, c, dc_words);
#pragma unroll
    for (int l = 1; l < BANDS; ++l) {
        const int n = 2 * l + 1, k0 = l * l;
        const float *M = a.m + edit_matrix_offset(l);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float in[7];
#pragma unroll
            for (int i = 0; i < n; ++i) in[i] = c[3 * (k0 + i) + ch];
#pragma unroll
            for (int j = 0; j < n; ++j) {
                float acc = __fmul_rn(in[0], M[j]);
#pragma unroll
                for (int i = 1; i < n; ++i) acc = __fadd_rn(acc, __fmul_rn(in[i], M[i * n + j]));
                c[3 * (k0 + j) + ch] = acc;
            }
        }
    }
    sh_pack<BANDS, HALF, true>(dst, st, c, dc_words);
}

// gsr_recolor_selection: every selected splat s of the store is rewritten from its planes in `src` (include/gsr.h "Splat colour
// edits"), with the skeleton of transform_selection_kernel.  In float32, one rounding per operation, no contraction, per coefficient k
// (an RGB triple c): DC c'_i = ((A[i][0] c_r + A[i][1] c_g) + A[i][2] c_b) + d_i, band l >= 1 the same without d and with N~_l for A;
// opacity u = (o s) + t, o' = 1 above 1, u above 0, else +0 (NaN included).  Planes 0-1, plane-2 x, y, w copied bit for bit (in place
// planes 0-1 are neither read nor written), slots past 3K +0.
template <int BANDS, bool HALF>
__global__ void __launch_bounds__(SEL_THREADS) recolor_selection_kernel(const __grid_constant__ RecolorArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t w = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5);
    if (w >= a.words) return;   // warp-uniform
    const uint32_t word = a.selected[w];
    if (((word >> lane) & 1u) == 0u) return;
    const uint64_t s = 32ull * w + lane, st = a.plane_stride;
    const float4 *src = a.src + s;
    float4 *dst = a.dst + s;
    if (a.src != a.dst) {   // uniform: from a snapshot
        dst[0] = src[0];
        dst[st] = src[st];
    }
    float4 p2 = src[2 * st];
    const float u = __fadd_rn(__fmul_rn(p2.z, a.k[EDIT_COLOR_S]), a.k[EDIT_COLOR_S + 1]);
    p2.z = u > 1.0f ? 1.0f : (u > 0.0f ? u : 0.0f);
    dst[2 * st] = p2;

    constexpr int K = sh_coeffs(BANDS), P = sh_planes(BANDS, HALF);
    float c[HALF ? 8 * P : 4 * P];
    uint32_t dc_words[2] = {0u, 0u};   // not used: the DC halves are edited
    sh_unpack<BANDS, HALF>(src, st, c, dc_words);
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float *M = a.k + (k == 0 ? 0 : edit_color_band_offset(k < 4 ? 1 : k < 9 ? 2 : 3));
        const float r = c[3 * k], g = c[3 * k + 1], b = c[3 * k + 2];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float v = __fadd_rn(__fadd_rn(__fmul_rn(M[3 * i], r), __fmul_rn(M[3 * i + 1], g)), __fmul_rn(M[3 * i + 2], b));
            c[3 * k + i] = k == 0 ? __fadd_rn(v, a.k[EDIT_COLOR_D + i]) : v;
        }
    }
    sh_pack<BANDS, HALF, false>(dst, st, c, dc_words);
}

// ---- gsr_delete_hidden / gsr_duplicate_selection: a chained scan with decoupled look-back over the mask words of [0, n) ----
// A tile's status word is a flag | count: EARLY (its count, published right after its ballots), AGG (its count, published after every
// load of its moved splats has returned) or PREFIX (the inclusive count of tiles 0 .. t, published after AGG and a look-back over AGG /
// PREFIX words).  So a PREFIX of tile t also says that every tile up to t has read its sources.
constexpr unsigned long long CS_EARLY = 1ull << 61, CS_AGG = 1ull << 62, CS_PREFIX = 1ull << 63, CS_VALUE = CS_EARLY - 1ull;

struct CompactShared {
    uint32_t tile;
    uint32_t warp_count[COMPACT_TILE_WORDS];
    uint32_t sel[COMPACT_TILE_WORDS];   // DELETE: the selected bits of the kept splats, by CTA rank
    unsigned long long excl;
};
// The CPU kernel emulator runs several CTAs of one launch at once and gives each its own copy of the CTA's shared state.
#ifndef COMPACT_CTA_SHARED
#define COMPACT_CTA_SHARED(T, name) __shared__ T name
#endif

// Warp 0: the exclusive count of tiles [0, tile), walking back 32 status words at a time and spinning on a word until its flag is in
// `ready`; the walk ends at the nearest PREFIX.
__device__ __forceinline__ unsigned long long lookback_exclusive(volatile unsigned long long *status, uint32_t tile, unsigned long long ready) {
    const uint32_t lane = threadIdx.x & 31u;
    unsigned long long excl = 0ull;
    for (int64_t hi = (int64_t)tile - 1; hi >= 0; hi -= 32) {
        const int64_t t = hi - (int64_t)lane;
        unsigned long long v = CS_PREFIX;   // before tile 0: a prefix of 0
        if (t >= 0) {
            while (((v = status[t]) & ready) == 0ull) __nanosleep(32);
        }
        const uint32_t pre = __ballot_sync(0xffffffffu, (v & CS_PREFIX) != 0ull);
        const uint32_t last = pre ? (uint32_t)(__ffs(pre) - 1) : 31u;   // the highest tile with a PREFIX ends the walk
        unsigned long long c = lane <= last ? (v & CS_VALUE) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        excl += c;
        if (pre) break;
    }
    __threadfence();   // acquire: what the tiles did before publishing the words read above comes before what this CTA does next
    return excl;
}

// One pass: the splats of [0, n) whose bit is set (DELETE: hidden clear, the kept splats; DUPLICATE: selected set) move, in order and
// bit for bit (all 3 + P planes), to prefix (DELETE, in place) or n + prefix (DUPLICATE), prefix = the number of set bits below them.
// A CTA owns COMPACT_TILE_WORDS consecutive mask words, one splat per thread, and takes its tile from an atomic ticket, so every
// predecessor it waits on holds an earlier ticket and is resident or done.  A splat whose destination is its own index is neither read
// nor written (a DELETE below the first hidden splat touches no plane).
// In-place DELETE: destinations never exceed sources, but a CTA's destinations can overlap the sources of earlier CTAs.  The exact
// destinations come from a first look-back over EARLY words (reads are always safe); the CTA then loads its moved splats into registers,
// and publishes AGG only after every one of those loads has returned (loads, __syncthreads, fence, flag store).  Its second look-back
// waits for AGG / PREFIX words down to the nearest PREFIX, so when it publishes its own PREFIX and starts to store (flag acquire, then
// stores), every tile at or below it has read its sources: a destination is only ever written after the splat that lived there was
// read.  Inside a CTA every load comes before any store.  DUPLICATE writes only at or above n, where no source lives, so it publishes
// its PREFIX right after the first look-back.
template <int BANDS, bool HALF, int MODE>
__global__ void __launch_bounds__(COMPACT_THREADS) compact_store_kernel(const __grid_constant__ CompactArgs a) {
    constexpr int PL = soa_planes(BANDS, HALF);
    COMPACT_CTA_SHARED(CompactShared, sh);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t nw = (uint32_t)((a.n + 31ull) >> 5), tiles = (nw + COMPACT_TILE_WORDS - 1) / COMPACT_TILE_WORDS;
    volatile unsigned long long *status = a.lookback;
    if (tid == 0) sh.tile = (uint32_t)atomicAdd(a.lookback + tiles, 1ull);
    if (tid < COMPACT_TILE_WORDS) sh.sel[tid] = 0u;
    __syncthreads();
    const uint32_t tile = sh.tile, w = tile * COMPACT_TILE_WORDS + warp;
    const uint64_t s = 32ull * w + lane, st = a.plane_stride;
    uint32_t bits = 0u, sel = 0u;
    if (w < nw) {
        const uint32_t valid = 32ull * (w + 1) <= a.n ? 0xffffffffu : (1u << (uint32_t)(a.n & 31ull)) - 1u;
        if constexpr (MODE == COMPACT_DELETE) {
            bits = ~a.hidden[w] & valid;
            sel = a.selected[w] & bits;
        } else {
            bits = a.selected[w] & valid;
        }
    }
    if (lane == 0) sh.warp_count[warp] = (uint32_t)__popc(bits);
    __syncthreads();
    uint32_t rank = (uint32_t)__popc(bits & ((1u << lane) - 1u)), agg = 0u;
#pragma unroll
    for (uint32_t i = 0; i < COMPACT_TILE_WORDS; ++i) {
        const uint32_t c = sh.warp_count[i];
        rank += i < warp ? c : 0u;
        agg += c;
    }
    const bool mine = (bits >> lane) & 1u;
    if constexpr (MODE == COMPACT_DELETE) {
        if (mine && ((sel >> lane) & 1u)) atomicOr(&sh.sel[rank >> 5], 1u << (rank & 31u));
    }
    if (tid == 0) status[tile] = CS_EARLY | agg;
    if (warp == 0) {
        const unsigned long long e = tile ? lookback_exclusive(status, tile, CS_EARLY | CS_AGG | CS_PREFIX) : 0ull;
        if (lane == 0) {
            sh.excl = e;
            if constexpr (MODE == COMPACT_DUPLICATE) {
                status[tile] = CS_PREFIX | (e + agg);
                if (tile == tiles - 1) *a.total = e + agg;
            }
        }
    }
    __syncthreads();
    const unsigned long long excl = sh.excl;
    const uint64_t dst = (MODE == COMPACT_DUPLICATE ? a.n : 0ull) + excl + rank;
    const bool move = mine && dst != s;
    float4 v[PL];
    if (move) {
#pragma unroll
        for (int p = 0; p < PL; ++p) v[p] = a.soa[(uint64_t)p * st + s];
    }
    if constexpr (MODE == COMPACT_DELETE) {
        __syncthreads();   // every load of this tile's moved splats has returned
        if (tid == 0) {
            __threadfence();
            status[tile] = (tile == 0 ? CS_PREFIX : CS_AGG) | agg;
        }
        if (warp == 0 && tile) {
            const unsigned long long e = lookback_exclusive(status, tile, CS_AGG | CS_PREFIX);   // == excl
            if (lane == 0) {
                __threadfence();
                status[tile] = CS_PREFIX | (e + agg);
            }
        }
        if (tid == 0 && tile == tiles - 1) *a.total = excl + agg;
        __syncthreads();
        // the selected bits of the destinations [excl, excl + agg): word j of the CTA's rank bits lands at bit offset excl & 31
        if (tid <= COMPACT_TILE_WORDS && agg) {
            const uint32_t off = (uint32_t)(excl & 31ull);
            const uint32_t val = (tid < COMPACT_TILE_WORDS ? sh.sel[tid] << off : 0u) | (tid > 0 && off ? sh.sel[tid - 1] >> (32u - off) : 0u);
            const uint64_t ow = (excl >> 5) + tid;
            if (val) {
                if (32ull * ow >= excl && 32ull * ow + 32ull <= excl + agg) a.sel_out[ow] = val;   // no other CTA writes this word
                else atomicOr(a.sel_out + ow, val);
            }
        }
    }
    if (move) {
#pragma unroll
        for (int p = 0; p < PL; ++p) a.soa[(uint64_t)p * st + dst] = v[p];
    }
}

// After a delete that kept k of n splats: selected = the moved bits (scratch, zeroed again), hidden = 0 over every word, and the slots
// [k, n) vacant: plane-0 x, y, z the quiet NaN 0x7FC00000, every other word +0.
__global__ void __launch_bounds__(SEL_THREADS) delete_finish_kernel(float4 *soa, uint64_t st, int planes, uint64_t k, uint64_t n, uint32_t *hidden,
                                                                    uint32_t *selected, uint32_t *scratch, uint32_t words) {
    const uint64_t i = (uint64_t)blockIdx.x * SEL_THREADS + threadIdx.x;
    if (i < words) {
        selected[i] = scratch[i];
        scratch[i] = 0u;
        hidden[i] = 0u;
    }
    if (i < n - k) {
        const float qnan = __uint_as_float(0x7FC00000u);
        soa[k + i] = make_float4(qnan, qnan, qnan, 0.0f);
#pragma unroll 1
        for (int p = 1; p < planes; ++p) soa[(uint64_t)p * st + k + i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
}

// After a duplicate of S splats behind n: selected = exactly [n, n + S), hidden cleared there
__global__ void __launch_bounds__(SEL_THREADS) duplicate_finish_kernel(uint64_t n, uint64_t S, uint32_t *hidden, uint32_t *selected, uint32_t words) {
    const uint32_t w = blockIdx.x * SEL_THREADS + threadIdx.x;
    if (w >= words) return;
    const uint64_t lo = 32ull * w, a = n > lo ? n : lo, b = n + S < lo + 32ull ? n + S : lo + 32ull;
    uint32_t m = 0u;
    if (a < b) {
        const uint32_t i0 = (uint32_t)(a - lo), c = (uint32_t)(b - a);
        m = (c == 32u ? 0xffffffffu : (1u << c) - 1u) << i0;
    }
    selected[w] = m;
    hidden[w] &= ~m;
}

// counts[0] += the selected bits below n (the bounded count of gsr_duplicate_selection; mask_counts_kernel counts every word)
__global__ void __launch_bounds__(SEL_THREADS) count_selected_kernel(const uint32_t *selected, uint64_t n, unsigned long long *counts) {
    const uint32_t nw = (uint32_t)((n + 31ull) >> 5);
    uint32_t ns = 0u;
    for (uint32_t w = blockIdx.x * SEL_THREADS + threadIdx.x; w < nw; w += gridDim.x * SEL_THREADS) {
        const uint32_t valid = 32ull * (w + 1) <= n ? 0xffffffffu : (1u << (uint32_t)(n & 31ull)) - 1u;
        ns += __popc(selected[w] & valid);
    }
    ns = __reduce_add_sync(0xffffffffu, ns);
    if ((threadIdx.x & 31u) == 0u && ns) atomicAdd(counts, (unsigned long long)ns);
}

// A tested splat counts only if none of its plane-0 x, y, z is NaN (a vacant slot never counts).
__device__ __forceinline__ bool splat_vacant(const float4 &p0) { return p0.x != p0.x || p0.y != p0.y || p0.z != p0.z; }

// ---- gsr_export_ply: the exported splats of [0, n) as 3DGS vertex rows (include/gsr.h "Splat export") ----
// The exported bits of mask word w (< ceil(n / 32)): lane l tests splat 32 w + l.  Plane 0 is read only for a splat in scope.
__device__ __forceinline__ uint32_t export_bits(const ExportArgs &a, uint32_t w, uint32_t lane) {
    const uint32_t valid = 32ull * (w + 1) <= a.n ? 0xffffffffu : (1u << (uint32_t)(a.n & 31ull)) - 1u;
    const uint32_t scope = a.hidden ? (a.selected_only ? a.selected[w] : ~a.hidden[w]) & valid : valid;
    bool in = (scope >> lane) & 1u;
    if (in) in = !splat_vacant(__ldg(a.soa + 32ull * w + lane));
    return __ballot_sync(0xffffffffu, in);
}

// *count += the exported splats: a warp per mask word (grid-stride), one atomic per warp
__global__ void __launch_bounds__(SEL_THREADS) export_count_kernel(const __grid_constant__ ExportArgs a) {
    const uint32_t lane = threadIdx.x & 31u, nw = (uint32_t)((a.n + 31ull) >> 5);
    uint32_t c = 0u;
    for (uint32_t w = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5); w < nw; w += gridDim.x * SEL_WARPS) c += (uint32_t)__popc(export_bits(a, w, lane));
    if (lane == 0u && c) atomicAdd(a.count, (unsigned long long)c);
}

// The writing pass.  A CTA owns COMPACT_TILE_WORDS consecutive mask words (one splat per thread, its tile from an atomic ticket like
// compact_store_kernel), ranks its exported splats, publishes its count and looks back for its prefix excl (the pass only reads the
// store, so it publishes its PREFIX right after).  Each exported splat reads planes 1, 2 and the SH planes of degree d and writes its
// row into shared memory at its rank; the CTA's rows [excl, excl + agg) are one contiguous range of dst, stored with consecutive threads
// on consecutive 4-byte words.
#ifndef EXPORT_CTA_ROWS
#ifndef GSR_CPU_EMU
#define EXPORT_CTA_ROWS(name) extern __shared__ float name[]
#else  // tests/kernel_emu, one CTA at a time: the largest row buffer
#define EXPORT_CTA_ROWS(name) __shared__ float name[COMPACT_THREADS * export_row_floats(3)]
#endif
#endif
template <int BANDS, bool HALF>
__global__ void __launch_bounds__(COMPACT_THREADS) export_ply_kernel(const __grid_constant__ ExportArgs a) {
    constexpr int K = sh_coeffs(BANDS), P = sh_planes(BANDS, HALF);
    COMPACT_CTA_SHARED(CompactShared, sh);
    EXPORT_CTA_ROWS(rows);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t nw = (uint32_t)((a.n + 31ull) >> 5), tiles = (nw + COMPACT_TILE_WORDS - 1) / COMPACT_TILE_WORDS;
    volatile unsigned long long *status = a.lookback;
    if (tid == 0) sh.tile = (uint32_t)atomicAdd(a.lookback + tiles, 1ull);
    __syncthreads();
    const uint32_t tile = sh.tile, w = tile * COMPACT_TILE_WORDS + warp;
    const uint32_t bits = w < nw ? export_bits(a, w, lane) : 0u;
    if (lane == 0) sh.warp_count[warp] = (uint32_t)__popc(bits);
    __syncthreads();
    uint32_t rank = (uint32_t)__popc(bits & ((1u << lane) - 1u)), agg = 0u;
#pragma unroll
    for (uint32_t i = 0; i < COMPACT_TILE_WORDS; ++i) {
        const uint32_t c = sh.warp_count[i];
        rank += i < warp ? c : 0u;
        agg += c;
    }
    if (tid == 0) status[tile] = CS_EARLY | agg;
    if (warp == 0) {
        const unsigned long long e = tile ? lookback_exclusive(status, tile, CS_EARLY | CS_AGG | CS_PREFIX) : 0ull;
        if (lane == 0) {
            sh.excl = e;
            status[tile] = CS_PREFIX | (e + agg);
        }
    }
    const uint32_t RW = export_row_floats(a.degree);
    if ((bits >> lane) & 1u) {
        const int Kd = (a.degree + 1) * (a.degree + 1), Pd = HALF ? (3 * Kd + 7) / 8 : (3 * Kd + 3) / 4;
        const uint64_t s = 32ull * w + lane, st = a.plane_stride;
        const float4 *src = a.soa + s;
        const float4 p0 = __ldg(src), p1 = __ldg(src + st), p2 = __ldg(src + 2 * st);
        float c[HALF ? 8 * P : 4 * P];
#pragma unroll
        for (int k = 0; k < P; ++k) {
            float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            if (k < Pd) v = __ldg(src + (uint64_t)(3 + k) * st);
            if constexpr (HALF) {
                const uint32_t u[4] = {__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w)};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    c[8 * k + 2 * j] = half_bits_to_float(u[j] & 0xFFFFu);
                    c[8 * k + 2 * j + 1] = half_bits_to_float(u[j] >> 16);
                }
            } else {
                c[4 * k + 0] = v.x; c[4 * k + 1] = v.y; c[4 * k + 2] = v.z; c[4 * k + 3] = v.w;
            }
        }
        float *r = rows + (size_t)rank * RW;
        r[0] = p0.x; r[1] = p0.y; r[2] = p0.z;
        r[3] = r[4] = r[5] = 0.0f;
        r[6] = c[0]; r[7] = c[1]; r[8] = c[2];
#pragma unroll
        for (int k = 1; k < K; ++k) {
            if (k < Kd) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) r[9 + ch * (Kd - 1) + (k - 1)] = c[3 * k + ch];
            }
        }
        float *t = r + 9 + 3 * (Kd - 1);
        const double o = (double)p2.z;
        double logit = log(o) - log1p(-o);
        logit = logit != logit ? 0.0 : logit < -104.0 ? -104.0 : logit > 104.0 ? 104.0 : logit;
        t[0] = (float)logit;
        export_scale_rot(p1, p2, t + 1);
    }
    __syncthreads();
    const unsigned long long excl = sh.excl;
    float *dst = a.dst + excl * RW;
    for (uint32_t i = tid; i < agg * RW; i += COMPACT_THREADS) dst[i] = rows[i];
}

// ---- gsr_select_where / gsr_splat_histogram: per-splat properties of the stored words (include/gsr.h "Splat property selection") ----
// The planes of one splat beyond plane 0, each loaded the first time a property needs it, so a splat that failed an earlier filter
// reads nothing more.  PL: the prop_planes bits of the filter set (a plane outside PL is never read); HALF: the SH format of plane 3.
// Every value in float32, one rounding per operation, in the order of include/gsr.h.  PROP_PC in PL: the contribution properties are
// read from the splat's record `rec` of the contribution buffer.
template <bool PC> struct ContribRec {};
template <> struct ContribRec<true> { const gsr_splat_contribution *rec = nullptr; };
template <bool HALF, int PL>
struct SplatProps : ContribRec<(PL & PROP_PC) != 0> {
    const float4 *src;   // plane 0 of the splat
    uint64_t st;
    float4 p1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), p2 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float dc[3] = {0.0f, 0.0f, 0.0f};
    int have = 0;
    __device__ __forceinline__ SplatProps(const float4 *s, uint64_t stride) : src(s), st(stride) {}

    __device__ __forceinline__ float value(const gsr_splat_filter &f) {
        if constexpr ((PL & PROP_PC) != 0) {
            const int32_t p = f.property;
            if (p == GSR_PROP_CONTRIBUTION) return __fmul_rn((float)__ldg(reinterpret_cast<const unsigned long long *>(&this->rec->weight)), 0x1p-24f);
            if (p == GSR_PROP_PEAK_CONTRIBUTION) return __ldg(&this->rec->peak);
            if (p == GSR_PROP_VIEWS) return (float)__ldg(&this->rec->views);
            if (p == GSR_PROP_CONTRIBUTING_PIXELS) return (float)__ldg(reinterpret_cast<const unsigned long long *>(&this->rec->pixels));
        }
        const int need = prop_planes(f.property) & ~have;
        if constexpr ((PL & PROP_P1) != 0) if (need & PROP_P1) p1 = __ldg(src + st);
        if constexpr ((PL & PROP_P2) != 0) if (need & PROP_P2) p2 = __ldg(src + 2 * st);
        if constexpr ((PL & PROP_P3) != 0) {
            if (need & PROP_P3) {
                const float4 v = __ldg(src + 3 * st);
                if constexpr (HALF) {   // values 0, 1 in word x, value 2 in the low half of word y
                    dc[0] = half_bits_to_float(__float_as_uint(v.x) & 0xFFFFu);
                    dc[1] = half_bits_to_float(__float_as_uint(v.x) >> 16);
                    dc[2] = half_bits_to_float(__float_as_uint(v.y) & 0xFFFFu);
                } else {
                    dc[0] = v.x; dc[1] = v.y; dc[2] = v.z;
                }
            }
        }
        have |= need;
        const int32_t p = f.property;
        if (p == GSR_PROP_OPACITY) return p2.z;
        if (p == GSR_PROP_COLOR_DISTANCE) {
            float d2 = 0.0f;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float d = __fsub_rn(__fadd_rn(0.5f, __fmul_rn(dc[i], SH_C0)), f.rgb[i]);
                d2 = i == 0 ? __fmul_rn(d, d) : __fadd_rn(d2, __fmul_rn(d, d));
            }
            return d2;
        }
        const float S00 = p1.x, S01 = p1.y, S02 = p1.z, S11 = p1.w, S12 = p2.x, S22 = p2.y;
        const float t = __fadd_rn(__fadd_rn(S00, S11), S22);
        if (p == GSR_PROP_SIZE) return t;
        const float det = __fadd_rn(__fsub_rn(__fmul_rn(S00, __fsub_rn(__fmul_rn(S11, S22), __fmul_rn(S12, S12))),
                                              __fmul_rn(S01, __fsub_rn(__fmul_rn(S01, S22), __fmul_rn(S12, S02)))),
                                    __fmul_rn(S02, __fsub_rn(__fmul_rn(S01, S12), __fmul_rn(S11, S02))));
        if (p == GSR_PROP_VOLUME) return det;
        return __fdiv_rn(__fmul_rn(27.0f, det), __fmul_rn(__fmul_rn(t, t), t));   // GSR_PROP_ISOTROPY
    }
};

// gsr_select_where: the shape of select_region_kernel -- a warp per mask word, a lane per splat, a ballot, lane 0 combines.  Lanes
// outside the tested range read nothing; a lane leaves the filter loop at its first failed filter.
template <bool HALF, int PL>
__global__ void __launch_bounds__(SEL_THREADS) select_where_kernel(const __grid_constant__ WhereArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t w = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5);
    if (w >= a.words) return;   // warp-uniform
    const uint64_t s = 32ull * w + lane;
    bool in = s >= a.first && s - a.first < a.count;
    if (in) {
        const float4 *src = a.soa + s;
        in = !splat_vacant(__ldg(src));
        SplatProps<HALF, PL> sp(src, a.plane_stride);
        if constexpr ((PL & PROP_PC) != 0) sp.rec = a.contrib + s;
#pragma unroll 1
        for (uint32_t i = 0; in && i < a.n; ++i) {
            const float v = sp.value(a.f[i]);
            in = a.f[i].lo <= v && v <= a.f[i].hi;
        }
    }
    const uint32_t inside = __ballot_sync(0xffffffffu, in);
    if (lane == 0) a.selected[w] = combine_op(a.op, a.selected[w], inside) & ~a.hidden[w];
}

// gsr_splat_histogram: a grid-stride pass over the tested range.  Each CTA keeps the edges and a private bins + 3 histogram in shared
// memory, finds a value's bin by a branch-free binary search (the largest i < bins with e_i <= v; the comparisons place below, above
// and NaN), and adds its non-zero counters to the 64-bit global ones once at the end.  The least and greatest ord(v) of the non-NaN
// values are reduced per warp (a shuffle butterfly), then go to the global keys with one atomicMax each per warp: max of
// signed_key(~lo) for the least, max of signed_key(hi) for the greatest (signed_key orders an unsigned key as an int).  Launched only while something can count (not for
// GSR_HISTOGRAM_SELECTED while the masks are not in use).
constexpr int PROP_HIST_THREADS = 512;
struct PropHistShared {
    uint32_t count[HIST_COUNTS];
    float edge[GSR_MAX_HISTOGRAM_BINS + 1];
};
// The CPU kernel emulator runs several CTAs of one launch at once and gives each its own copy of the CTA's shared state.
#ifndef HIST_CTA_SHARED
#define HIST_CTA_SHARED(T, name) __shared__ T name
#endif

template <bool HALF, int PL>
__global__ void __launch_bounds__(PROP_HIST_THREADS) splat_histogram_kernel(const __grid_constant__ HistArgs a) {
    HIST_CTA_SHARED(PropHistShared, sh);
    const uint32_t tid = threadIdx.x, B = a.bins;
    for (uint32_t i = tid; i < B + 3; i += PROP_HIST_THREADS) sh.count[i] = 0u;
    for (uint32_t i = tid; i <= B; i += PROP_HIST_THREADS) sh.edge[i] = __ldg(a.edges + i);
    __syncthreads();
    const float e0 = sh.edge[0], eb = sh.edge[B];
    uint32_t lo = 0xFFFFFFFFu, hi = 0u;
    for (uint64_t i = (uint64_t)blockIdx.x * PROP_HIST_THREADS + tid; i < a.count; i += (uint64_t)gridDim.x * PROP_HIST_THREADS) {
        const uint64_t s = a.first + i;
        if (a.hidden) {
            const uint32_t bit = 1u << (uint32_t)(s & 31u);
            if ((__ldg(a.hidden + (s >> 5)) & bit) || (a.selected_only && !(__ldg(a.selected + (s >> 5)) & bit))) continue;
        }
        const float4 *src = a.soa + s;
        if (splat_vacant(__ldg(src))) continue;
        SplatProps<HALF, PL> sp(src, a.plane_stride);
        if constexpr ((PL & PROP_PC) != 0) sp.rec = a.contrib + s;
        const float v = sp.value(a.prop);
        uint32_t k = 0u;
        for (uint32_t step = a.top; step; step >>= 1) {
            const uint32_t j = k + step;
            k = (j < B && sh.edge[j] <= v) ? j : k;
        }
        const bool nan = v != v;
        atomicAdd(&sh.count[nan ? B + 2 : v < e0 ? B : v > eb ? B + 1 : k], 1u);
        if (!nan) {
            const uint32_t key = depth_order_word(__float_as_uint(v));
            lo = key < lo ? key : lo;
            hi = key > hi ? key : hi;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint32_t l = __shfl_xor_sync(0xffffffffu, lo, o), h = __shfl_xor_sync(0xffffffffu, hi, o);
        lo = l < lo ? l : lo;
        hi = h > hi ? h : hi;
    }
    if ((tid & 31u) == 0u && lo <= hi) {   // lo > hi: no value in this warp
        atomicMax(a.keys, hist_signed_key(~lo));
        atomicMax(a.keys + 1, hist_signed_key(hi));
    }
    __syncthreads();
    for (uint32_t i = tid; i < B + 3; i += PROP_HIST_THREADS) {
        const uint32_t c = sh.count[i];
        if (c) atomicAdd(a.counts + i, (unsigned long long)c);
    }
}

}  // namespace

// ---- the host's float64 matrices of gsr_transform_selection (also compiled into the CPU kernel emulator) ----
namespace {
// P_l(d): the polynomials that multiply coefficients l^2 .. l^2 + 2l in sh_color (projection.cu), signs included, with the float64
// values of its constants
void sh_band_poly(int l, const double d[3], double *p) {
    const double x = d[0], y = d[1], z = d[2], xx = x * x, yy = y * y, zz = z * z;
    if (l == 1) {
        const double c1 = 0.4886025119029199;
        p[0] = -c1 * y; p[1] = c1 * z; p[2] = -c1 * x;
    } else if (l == 2) {
        p[0] = 1.0925484305920792 * x * y; p[1] = -1.0925484305920792 * y * z; p[2] = 0.31539156525252005 * (2.0 * zz - xx - yy);
        p[3] = -1.0925484305920792 * x * z; p[4] = 0.5462742152960396 * (xx - yy);
    } else {
        p[0] = -0.5900435899266435 * y * (3.0 * xx - yy); p[1] = 2.890611442640554 * x * y * z;
        p[2] = -0.4570457994644658 * y * (4.0 * zz - xx - yy); p[3] = 0.3731763325901154 * z * (2.0 * zz - 3.0 * xx - 3.0 * yy);
        p[4] = -0.4570457994644658 * x * (4.0 * zz - xx - yy); p[5] = 1.445305721320277 * z * (xx - yy);
        p[6] = -0.5900435899266435 * x * (xx - 3.0 * yy);
    }
}

double det3(const double X[3][3]) {
    return X[0][0] * (X[1][1] * X[2][2] - X[1][2] * X[2][1]) - X[0][1] * (X[1][0] * X[2][2] - X[1][2] * X[2][0]) +
           X[0][2] * (X[1][0] * X[2][1] - X[1][1] * X[2][0]);
}

// Solves A X = B in place (A n x n, B n x m, row-major), Gaussian elimination with partial pivoting
void solve(double *A, double *B, int n, int m) {
    for (int k = 0; k < n; ++k) {
        int piv = k;
        for (int r = k + 1; r < n; ++r) if (fabs(A[r * n + k]) > fabs(A[piv * n + k])) piv = r;
        if (piv != k) {
            for (int c = 0; c < n; ++c) { const double t = A[k * n + c]; A[k * n + c] = A[piv * n + c]; A[piv * n + c] = t; }
            for (int c = 0; c < m; ++c) { const double t = B[k * m + c]; B[k * m + c] = B[piv * m + c]; B[piv * m + c] = t; }
        }
        for (int r = k + 1; r < n; ++r) {
            const double f = A[r * n + k] / A[k * n + k];
            for (int c = k; c < n; ++c) A[r * n + c] -= f * A[k * n + c];
            for (int c = 0; c < m; ++c) B[r * m + c] -= f * B[k * m + c];
        }
    }
    for (int k = n - 1; k >= 0; --k) {
        for (int c = 0; c < m; ++c) {
            double v = B[k * m + c];
            for (int j = k + 1; j < n; ++j) v -= A[k * n + j] * B[j * m + c];
            B[k * m + c] = v / A[k * n + k];
        }
    }
}

// Q = the orthogonal polar factor of L (U V^T of its SVD; improper when det L < 0) by Newton's iteration X <- (g X + (g X)^-T) / 2,
// with the determinant scaling g = |det X|^(-1/3) while X is far from orthogonal.
void polar_factor(const double L[3][3], double X[3][3]) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) X[r][c] = L[r][c];
    for (int it = 0; it < 100; ++it) {
        const double d = det3(X);
        double cof[3][3];   // X^-T = cof(X) / det X
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
                cof[r][c] = X[r1][c1] * X[r2][c2] - X[r1][c2] * X[r2][c1];
            }
        double err = 0.0;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) { const double e = X[r][c] - cof[r][c] / d; err += e * e; }
        const double g = err > 1e-4 ? pow(fabs(d), -1.0 / 3.0) : 1.0;
        double diff = 0.0;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                const double y = 0.5 * (g * X[r][c] + cof[r][c] / (g * d));
                diff += (y - X[r][c]) * (y - X[r][c]);
                X[r][c] = y;
            }
        if (diff < 1e-30) break;
    }
}

// M_l (row-major (2l+1)^2) with P_l(Q^T d) = M_l P_l(d) for every d: the least-squares solution over 64 directions of a Fibonacci
// sphere (the relation is exact, so the fit is too), M_l A = B with A = sum P_l(d) P_l(d)^T and B = sum P_l(Q^T d) P_l(d)^T.
void band_matrix(const double Q[3][3], int l, double *M) {
    const int n = 2 * l + 1;
    double A[49] = {}, B[49] = {};
    for (int k = 0; k < 64; ++k) {
        const double z = 1.0 - (2.0 * k + 1.0) / 64.0, rr = sqrt(1.0 - z * z), phi = 2.399963229728653 * k;
        const double d[3] = {rr * cos(phi), rr * sin(phi), z};
        const double qd[3] = {Q[0][0] * d[0] + Q[1][0] * d[1] + Q[2][0] * d[2], Q[0][1] * d[0] + Q[1][1] * d[1] + Q[2][1] * d[2],
                              Q[0][2] * d[0] + Q[1][2] * d[1] + Q[2][2] * d[2]};   // Q^T d
        double p[7], pq[7];
        sh_band_poly(l, d, p);
        sh_band_poly(l, qd, pq);
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) { A[i * n + j] += p[i] * p[j]; B[i * n + j] += pq[i] * p[j]; }
    }
    double Bt[49];   // M A = B with A symmetric: A M^T = B^T
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) Bt[i * n + j] = B[j * n + i];
    solve(A, Bt, n, n);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) M[i * n + j] = Bt[j * n + i];
}
}  // namespace

// The 95 floats: to_source, then M~_l = M_l(polar factor of L) with entries below 1e-9 in magnitude set to +0, rounded to float32.
int edit_transform_matrices(const float to_source[12], float out[EDIT_TRANSFORM_FLOATS]) {
    double L[3][3], Q[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) L[r][c] = (double)to_source[3 * c + r];
    const double det = det3(L);
    if (!(det != 0.0 && fabs(det) <= 1.7976931348623157e308)) return GSR_ERR_INVALID;
    polar_factor(L, Q);
    for (int e = 0; e < 12; ++e) out[e] = to_source[e];
    for (int l = 1; l <= 3; ++l) {
        double M[49];
        band_matrix(Q, l, M);
        float *o = out + edit_matrix_offset(l);
        for (int i = 0; i < (2 * l + 1) * (2 * l + 1); ++i) o[i] = fabs(M[i]) < 1e-9 ? 0.0f : (float)M[i];
    }
    return GSR_OK;
}

// The 41 floats of gsr_recolor_selection, each computed in float64 from the float inputs and rounded to float32 once: A row-major,
// d_i = ((((A[i][0] / 2 + A[i][1] / 2) + A[i][2] / 2) + b_i) - 1/2) / C0 with C0 the projection's SH_C0, N~_l = band_scale[l-1] A (the
// double product of two floats is exact), s, t.  colour' = A colour + b on 0.5 + C0 c_0 + sum_k P_k(d) c_k is c_0' = A c_0 + d and
// c_k' = A c_k: every such map is an exact map of the coefficients.
void edit_color_constants(const gsr_color_edit *e, float out[EDIT_COLOR_FLOATS]) {
    const double c0 = (double)SH_C0;
    for (int i = 0; i < 3; ++i) {
        const double A0 = e->matrix[i], A1 = e->matrix[3 + i], A2 = e->matrix[6 + i];
        out[3 * i] = (float)A0; out[3 * i + 1] = (float)A1; out[3 * i + 2] = (float)A2;
        out[EDIT_COLOR_D + i] = (float)(((((A0 * 0.5 + A1 * 0.5) + A2 * 0.5) + (double)e->matrix[9 + i]) - 0.5) / c0);
        for (int l = 1; l <= 3; ++l)
            for (int j = 0; j < 3; ++j) out[edit_color_band_offset(l) + 3 * i + j] = (float)((double)e->band_scale[l - 1] * (double)e->matrix[3 * j + i]);
    }
    out[EDIT_COLOR_S] = e->opacity_scale;
    out[EDIT_COLOR_S + 1] = e->opacity_offset;
}

#ifndef GSR_CPU_EMU
namespace {
uint32_t word_blocks(uint32_t words) { return (words + SEL_THREADS - 1) / SEL_THREADS; }

template <int BANDS, bool HALF>
void launch_transform_variant(const TransformArgs &a, uint32_t blocks, cudaStream_t stream) {
    transform_selection_kernel<BANDS, HALF><<<blocks, SEL_THREADS, 0, stream>>>(a);
}
}  // namespace

int launch_transform_selection(const TransformArgs &a, int bands, bool sh_half, cudaStream_t stream) {
    if (a.words == 0) return GSR_OK;
    const uint32_t blocks = (a.words + SEL_WARPS - 1) / SEL_WARPS;
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: launch_transform_variant<1, false>(a, blocks, stream); break;
        case 3: launch_transform_variant<1, true>(a, blocks, stream); break;
        case 4: launch_transform_variant<2, false>(a, blocks, stream); break;
        case 5: launch_transform_variant<2, true>(a, blocks, stream); break;
        case 6: launch_transform_variant<3, false>(a, blocks, stream); break;
        case 7: launch_transform_variant<3, true>(a, blocks, stream); break;
        case 8: launch_transform_variant<4, false>(a, blocks, stream); break;
        default: launch_transform_variant<4, true>(a, blocks, stream); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

namespace {
template <int BANDS, bool HALF>
void launch_recolor_variant(const RecolorArgs &a, uint32_t blocks, cudaStream_t stream) {
    recolor_selection_kernel<BANDS, HALF><<<blocks, SEL_THREADS, 0, stream>>>(a);
}
}  // namespace

int launch_recolor_selection(const RecolorArgs &a, int bands, bool sh_half, cudaStream_t stream) {
    if (a.words == 0) return GSR_OK;
    const uint32_t blocks = (a.words + SEL_WARPS - 1) / SEL_WARPS;
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: launch_recolor_variant<1, false>(a, blocks, stream); break;
        case 3: launch_recolor_variant<1, true>(a, blocks, stream); break;
        case 4: launch_recolor_variant<2, false>(a, blocks, stream); break;
        case 5: launch_recolor_variant<2, true>(a, blocks, stream); break;
        case 6: launch_recolor_variant<3, false>(a, blocks, stream); break;
        case 7: launch_recolor_variant<3, true>(a, blocks, stream); break;
        case 8: launch_recolor_variant<4, false>(a, blocks, stream); break;
        default: launch_recolor_variant<4, true>(a, blocks, stream); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

namespace {
template <int BANDS, bool HALF>
void launch_compact_variant(const CompactArgs &a, int mode, uint32_t blocks, cudaStream_t stream) {
    if (mode == COMPACT_DELETE) compact_store_kernel<BANDS, HALF, COMPACT_DELETE><<<blocks, COMPACT_THREADS, 0, stream>>>(a);
    else compact_store_kernel<BANDS, HALF, COMPACT_DUPLICATE><<<blocks, COMPACT_THREADS, 0, stream>>>(a);
}
}  // namespace

int launch_compact_store(const CompactArgs &a, int mode, int bands, bool sh_half, cudaStream_t stream) {
    if (a.n == 0) return GSR_OK;
    const uint32_t words = (uint32_t)((a.n + 31ull) >> 5);
    const uint32_t blocks = (uint32_t)compact_lookback_words(words) - 1u;
    GSR_CUDA_TRY(cudaMemsetAsync(a.lookback, 0, sizeof(unsigned long long) * compact_lookback_words(words), stream));
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: launch_compact_variant<1, false>(a, mode, blocks, stream); break;
        case 3: launch_compact_variant<1, true>(a, mode, blocks, stream); break;
        case 4: launch_compact_variant<2, false>(a, mode, blocks, stream); break;
        case 5: launch_compact_variant<2, true>(a, mode, blocks, stream); break;
        case 6: launch_compact_variant<3, false>(a, mode, blocks, stream); break;
        case 7: launch_compact_variant<3, true>(a, mode, blocks, stream); break;
        case 8: launch_compact_variant<4, false>(a, mode, blocks, stream); break;
        default: launch_compact_variant<4, true>(a, mode, blocks, stream); break;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_delete_finish(float4 *soa, uint64_t plane_stride, int planes, uint64_t k, uint64_t n, uint32_t *hidden, uint32_t *selected,
                         uint32_t *scratch, uint32_t words, cudaStream_t stream) {
    const uint64_t items = words > n - k ? (uint64_t)words : n - k;
    if (!items) return GSR_OK;
    delete_finish_kernel<<<(uint32_t)((items + SEL_THREADS - 1) / SEL_THREADS), SEL_THREADS, 0, stream>>>(soa, plane_stride, planes, k, n, hidden,
                                                                                                         selected, scratch, words);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_duplicate_finish(uint64_t n, uint64_t S, uint32_t *hidden, uint32_t *selected, uint32_t words, cudaStream_t stream) {
    if (!words) return GSR_OK;
    duplicate_finish_kernel<<<word_blocks(words), SEL_THREADS, 0, stream>>>(n, S, hidden, selected, words);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_count_selected(const uint32_t *selected, uint64_t n, unsigned long long *counts, cudaStream_t stream) {
    GSR_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(unsigned long long), stream));
    const uint32_t words = (uint32_t)((n + 31ull) >> 5);
    if (!words) return GSR_OK;
    const uint32_t blocks = word_blocks(words) < 1024u ? word_blocks(words) : 1024u;
    count_selected_kernel<<<blocks, SEL_THREADS, 0, stream>>>(selected, n, counts);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_export_count(const ExportArgs &a, cudaStream_t stream) {
    GSR_CUDA_TRY(cudaMemsetAsync(a.count, 0, sizeof(unsigned long long), stream));
    const uint32_t words = (uint32_t)((a.n + 31ull) >> 5);
    if (!words) return GSR_OK;
    const uint32_t need = (words + SEL_WARPS - 1) / SEL_WARPS, blocks = need < 2048u ? need : 2048u;
    export_count_kernel<<<blocks, SEL_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

namespace {
template <int BANDS, bool HALF>
int launch_export_variant(const ExportArgs &a, uint32_t blocks, cudaStream_t stream) {
    const size_t smem = export_shared_bytes(a.degree);
    if (smem > 48 * 1024) GSR_CUDA_TRY(cudaFuncSetAttribute(export_ply_kernel<BANDS, HALF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    export_ply_kernel<BANDS, HALF><<<blocks, COMPACT_THREADS, smem, stream>>>(a);
    return GSR_OK;
}
}  // namespace

int launch_export_rows(const ExportArgs &a, int bands, bool sh_half, cudaStream_t stream) {
    if (a.n == 0) return GSR_OK;
    const uint32_t words = (uint32_t)((a.n + 31ull) >> 5);
    const uint32_t blocks = (uint32_t)compact_lookback_words(words) - 1u;
    GSR_CUDA_TRY(cudaMemsetAsync(a.lookback, 0, sizeof(unsigned long long) * compact_lookback_words(words), stream));
    int rc;
    switch (bands * 2 + (sh_half ? 1 : 0)) {
        case 2: rc = launch_export_variant<1, false>(a, blocks, stream); break;
        case 3: rc = launch_export_variant<1, true>(a, blocks, stream); break;
        case 4: rc = launch_export_variant<2, false>(a, blocks, stream); break;
        case 5: rc = launch_export_variant<2, true>(a, blocks, stream); break;
        case 6: rc = launch_export_variant<3, false>(a, blocks, stream); break;
        case 7: rc = launch_export_variant<3, true>(a, blocks, stream); break;
        case 8: rc = launch_export_variant<4, false>(a, blocks, stream); break;
        default: rc = launch_export_variant<4, true>(a, blocks, stream); break;
    }
    if (rc) return rc;
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

namespace {
template <bool HALF, int PL>
void launch_property_variant(const WhereArgs &a, uint32_t blocks, cudaStream_t stream) {
    select_where_kernel<HALF, PL><<<blocks, SEL_THREADS, 0, stream>>>(a);
}
template <bool HALF, int PL>
void launch_property_variant(const HistArgs &a, uint32_t blocks, cudaStream_t stream) {
    splat_histogram_kernel<HALF, PL><<<blocks, PROP_HIST_THREADS, 0, stream>>>(a);
}

// The variants: the plane sets a filter set can need (plane 1 always comes with plane 2), and the SH format only where plane 3 is read.
// A set that reads the contribution buffer takes the contribution-only variant, or with other properties the variant that can read
// every plane (a plane is still loaded only when a filter needs it).
constexpr int PROP_ALL = PROP_P1 | PROP_P2 | PROP_P3 | PROP_PC;
template <class Args>
int launch_property(const Args &a, int planes, bool sh_half, uint32_t blocks, cudaStream_t stream) {
    if (planes & PROP_PC) {
        if (planes == PROP_PC) launch_property_variant<false, PROP_PC>(a, blocks, stream);
        else if (sh_half) launch_property_variant<true, PROP_ALL>(a, blocks, stream);
        else launch_property_variant<false, PROP_ALL>(a, blocks, stream);
        GSR_CUDA_TRY(cudaGetLastError());
        return GSR_OK;
    }
    switch (planes | (sh_half && (planes & PROP_P3) ? 8 : 0)) {
        case PROP_P2: launch_property_variant<false, PROP_P2>(a, blocks, stream); break;
        case PROP_P1 | PROP_P2: launch_property_variant<false, PROP_P1 | PROP_P2>(a, blocks, stream); break;
        case PROP_P3: launch_property_variant<false, PROP_P3>(a, blocks, stream); break;
        case PROP_P2 | PROP_P3: launch_property_variant<false, PROP_P2 | PROP_P3>(a, blocks, stream); break;
        case PROP_P1 | PROP_P2 | PROP_P3: launch_property_variant<false, PROP_P1 | PROP_P2 | PROP_P3>(a, blocks, stream); break;
        case 8 | PROP_P3: launch_property_variant<true, PROP_P3>(a, blocks, stream); break;
        case 8 | PROP_P2 | PROP_P3: launch_property_variant<true, PROP_P2 | PROP_P3>(a, blocks, stream); break;
        case 8 | PROP_P1 | PROP_P2 | PROP_P3: launch_property_variant<true, PROP_P1 | PROP_P2 | PROP_P3>(a, blocks, stream); break;
        default: set_last_error("splat property kernels: no variant for plane set %d", planes); return GSR_ERR_INVALID;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
}  // namespace

int launch_select_where(const WhereArgs &a, int planes, bool sh_half, cudaStream_t stream) {
    if (a.words == 0) return GSR_OK;
    return launch_property(a, planes, sh_half, (a.words + SEL_WARPS - 1) / SEL_WARPS, stream);
}

int launch_splat_histogram(const HistArgs &a, int planes, bool sh_half, int sm_count, cudaStream_t stream) {
    if (a.count == 0) return GSR_OK;
    const uint64_t need = (a.count + PROP_HIST_THREADS - 1) / PROP_HIST_THREADS, most = 4ull * (uint64_t)(sm_count > 0 ? sm_count : 1);   // 4 CTAs of 512 per SM
    return launch_property(a, planes, sh_half, (uint32_t)(need < most ? need : most), stream);
}

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
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<1, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<1, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<2, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<2, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<3, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<3, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<4, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, transform_selection_kernel<4, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<1, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<1, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<2, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<2, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<3, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<3, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<4, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, recolor_selection_kernel<4, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<1, false, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<1, true, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<2, false, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<2, true, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<3, false, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<3, true, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<4, false, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<4, true, COMPACT_DELETE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<1, false, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<1, true, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<2, false, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<2, true, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<3, false, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<3, true, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<4, false, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, compact_store_kernel<4, true, COMPACT_DUPLICATE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, delete_finish_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, duplicate_finish_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, count_selected_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_count_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<1, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<1, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<2, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<2, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<3, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<3, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<4, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, export_ply_kernel<4, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_P2>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_P1 | PROP_P2>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_P1 | PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<true, PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<true, PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<true, PROP_P1 | PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_P2>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_P1 | PROP_P2>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_P1 | PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<true, PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<true, PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<true, PROP_P1 | PROP_P2 | PROP_P3>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_PC>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<false, PROP_ALL>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, select_where_kernel<true, PROP_ALL>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_PC>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<false, PROP_ALL>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, splat_histogram_kernel<true, PROP_ALL>));
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
