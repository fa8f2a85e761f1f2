// common.cuh -- shared declarations of libgsr (sm_90a).  Product code: never includes anything from oracle/.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gsr.h"

namespace gsr {

constexpr int TILE = 16;            // rasterizer.gd:4 TILE_SIZE
constexpr int NUM_PLANES = 15;      // 60-float Splat = 15 float4 planes in SoA
constexpr int PROJ_THREADS = 256;   // gsplat_projection.glsl:31 local_size_x

// SH storage by degree (gsr_config.sh_bands): B bands = degree + 1 hold K = B^2 coefficients per channel, stored coefficient-major RGB in
// P = ceil(3K / 4) float4 planes after planes 0-2.  B = 1, 2, 3, 4 -> P = 1, 3, 7, 12 (64 / 96 / 160 / 240 B per splat).
// A binary16 store (GSR_FLAG_SH_HALF, `half`) packs the same 3K values as IEEE halves, 8 per 16-byte plane: value i in SH plane i >> 3,
// slot i & 7 (slot 0 = the low half of the plane's first word), slots past 3K = +0.  P_h = ceil(3K / 8) = 1, 2, 4, 6 (64 / 80 / 112 /
// 144 B per splat).  Every plane of either format is 16 B per splat, so plane k of splat s is always float4 k * plane_stride + s.
constexpr int SH_BANDS_MAX = 4;
__host__ __device__ constexpr int sh_coeffs(int bands) { return bands * bands; }
__host__ __device__ constexpr int sh_planes(int bands, bool half = false) { return half ? (3 * bands * bands + 7) / 8 : (3 * bands * bands + 3) / 4; }
__host__ __device__ constexpr int soa_planes(int bands, bool half = false) { return 3 + sh_planes(bands, half); }
static_assert(soa_planes(SH_BANDS_MAX) == NUM_PLANES, "a degree-3 store is the 60-float Splat");
static_assert(soa_planes(SH_BANDS_MAX, true) * 16 == 144, "a degree-3 binary16 store is 144 B per splat");
// The DC factor of the projection's SH colour, colour = 0.5 + SH_C0 c_0 + ... (also the colour edits' host constants)
constexpr float SH_C0 = 0.28209479177387814f;

// binary16 SH store: h(c) = c rounded to binary16 (round to nearest even, subnormals and signed zeros kept); finite or infinite values
// beyond +-65504 saturate to +-65504, NaN stays a NaN.  The decode of a half is exact.
#ifndef GSR_CPU_EMU
__device__ __forceinline__ uint32_t half_bits_rn(float x) {   // IEEE conversion: overflow gives +-inf, NaN a NaN
    unsigned short h;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(x));
    return h;
}
__device__ __forceinline__ float half_bits_to_float(uint32_t h) {   // the low 16 bits
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"((unsigned short)h));
    return f;
}
#else  // tests/kernel_emu (CPU logic pre-flight): the same two conversions in integer arithmetic, bit for bit
inline uint32_t half_bits_rn(float x) {   // round to nearest even, subnormal halves kept, overflow to +-inf, NaN to a quiet NaN
    const uint32_t u = __float_as_uint(x), s = (u >> 16) & 0x8000u, a = u & 0x7FFFFFFFu;
    if (a > 0x7F800000u) return s | 0x7E00u | ((a >> 13) & 0x3FFu);
    if (a >= 0x477FF000u) return s | 0x7C00u;                      // |x| >= 65520 (and inf) rounds to inf
    if (a < 0x38800000u) {                                         // below 2^-14: a subnormal half (or zero), in units of 2^-24
        const uint32_t m = (a >> 23) ? ((a & 0x7FFFFFu) | 0x800000u) : (a & 0x7FFFFFu);
        const int e = (a >> 23) ? (int)(a >> 23) : 1;              // x = m * 2^(e - 150) = m * 2^(e - 126) units
        const int sh = 126 - e;                                    // >= 14
        if (sh > 24) return s;                                     // below 2^-25 (a tie at 2^-25 rounds to even 0 too)
        const uint32_t q = m >> sh, rem = m & ((1u << sh) - 1u), half = 1u << (sh - 1);
        return s | (q + ((rem > half || (rem == half && (q & 1u))) ? 1u : 0u));
    }
    uint32_t h = (a - 0x38000000u) >> 13;                          // rebias 127 -> 15, keep 10 mantissa bits
    const uint32_t rem = a & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) h += 1u;   // a carry moves into the exponent, as it should
    return s | h;
}
inline float half_bits_to_float(uint32_t h) {
    const uint32_t s = (h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e == 0x1Fu) return __uint_as_float(s | 0x7F800000u | (m << 13));
    if (e == 0u) { const float f = (float)m * 0x1p-24f; return s ? -f : f; }   // exact: m < 2^10
    return __uint_as_float(s | ((e + 112u) << 23) | (m << 13));
}
#endif
// (the comparison is false for NaN, so a NaN reaches the conversion unchanged: no fminf / fmaxf, which would make it the bound)
__device__ __forceinline__ uint32_t sh_half(float c) { return half_bits_rn(fabsf(c) > 65504.0f ? copysignf(65504.0f, c) : c); }
__device__ __forceinline__ uint32_t sh_half2(float lo, float hi) { return sh_half(lo) | (sh_half(hi) << 16); }

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
void set_last_error(const char *fmt, ...);

#define GSR_CUDA_TRY(expr)                                                                         \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            ::gsr::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return (_e == cudaErrorMemoryAllocation) ? GSR_ERR_OOM : GSR_ERR_CUDA;                 \
        }                                                                                          \
    } while (0)

// ---------------------------------------------------------------------------------------------
// "gsr deterministic math" (DESIGN.md section 4).  One IEEE binary32 op per operator, no implicit
// contraction (the library is compiled with -fmad=false), explicit __fmaf_rn where the spec says so.
// GLSL min/max/clamp semantics written out (gsplat_projection.glsl uses clamp/max).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float g_max(float x, float y) { return (x < y) ? y : x; }
__device__ __forceinline__ float g_min(float x, float y) { return (y < x) ? y : x; }
__device__ __forceinline__ float g_clamp(float x, float lo, float hi) { return g_min(g_max(x, lo), hi); }

// 2^t: clamp to [-127,128], round-half-even via the 1.5*2^23 magic constant, degree-6 polynomial on
// [-0.5,0.5] (Horner, fma), scale 2^n assembled in the exponent field (n=-127 -> 0, n=128 -> +inf).
__device__ __forceinline__ float det_exp2(float t) {
    const float MAGIC = 12582912.0f;
    float tc = g_min(g_max(t, -127.0f), 128.0f);
    float tm = __fadd_rn(tc, MAGIC);
    float nf = __fsub_rn(tm, MAGIC);
    float f = __fsub_rn(tc, nf);
    float p = 0x1.446c7ep-13f;
    p = __fmaf_rn(p, f, 0x1.5f48c8p-10f);
    p = __fmaf_rn(p, f, 0x1.3b29d8p-7f);
    p = __fmaf_rn(p, f, 0x1.c6aeccp-5f);
    p = __fmaf_rn(p, f, 0x1.ebfbe0p-3f);
    p = __fmaf_rn(p, f, 0x1.62e430p-1f);
    p = __fmaf_rn(p, f, 1.0f);
    uint32_t sbits = (__float_as_uint(tm) << 23) + 0x3F800000u;
    return __fmul_rn(p, __uint_as_float(sbits));
}

// GLSL exp(x) := 2^(x*log2e), log2e rounded to binary32.
__device__ __forceinline__ float det_exp(float x) { return det_exp2(__fmul_rn(x, 0x1.715476p+0f)); }

__device__ __forceinline__ float det_log2(float x) {
    int eadj = 0;
    if (x < 0x1p-126f) { x = __fmul_rn(x, 0x1p+32f); eadj = -32; }
    uint32_t u = __float_as_uint(x);
    int e = (int)(u >> 23) - 127;
    float m = __uint_as_float((u & 0x007FFFFFu) | 0x3F800000u);
    if (m >= 0x1.6a09e6p+0f) { m = __fmul_rn(m, 0.5f); e += 1; }
    float s = __fdiv_rn(__fsub_rn(m, 1.0f), __fadd_rn(m, 1.0f));
    float z = __fmul_rn(s, s);
    float g = 0x1.ba18b8p-2f;
    g = __fmaf_rn(g, z, 0x1.27471ep-1f);
    g = __fmaf_rn(g, z, 0x1.ec70e6p-1f);
    g = __fmaf_rn(g, z, 0x1.715476p+1f);
    return __fadd_rn((float)(e + eadj), __fmul_rn(s, g));
}

// GLSL pow(x,y) := exp2(y*log2(x)), pow(x<=0, y>0) := 0.
__device__ __forceinline__ float det_pow(float x, float y) {
    if (!(x > 0.0f)) return 0.0f;
    return det_exp2(__fmul_rn(y, det_log2(x)));
}

// ---------------------------------------------------------------------------------------------
// per-frame device state (one cudaMemsetAsync clears it; rasterizer.gd:127 clears histogram[0..1024])
// ---------------------------------------------------------------------------------------------
struct FrameState {
    unsigned long long dup_total;  // M, true count (histogram[0] of the reference)
    uint32_t dup_sorted;           // min(M, capacity): what the sort / ranges / compositor see
    uint32_t visible;              // V
    int32_t last_tile_plus1;       // 1 + largest tile id touched (0 = none); atomicMax target
    uint32_t overflow;
    uint32_t proj_ticket;          // dynamic block id for the projection look-back
    uint32_t pad0;
    unsigned long long staged;     // C: instances staged by the compositor (sum of consumed chunk sizes)
    uint32_t comp_head;            // compositor: next tile ticket of the persistent grid
    uint32_t comp_cta_limit;       // compositor: CTAs that may work (0 = all launched); set by tile_order_kernel for sparse frames
    uint32_t pad[4];
};
static_assert(sizeof(FrameState) == 64, "FrameState is one 64-byte slot of the history ring");

// Uniform block exactly as the reference uploads it (rasterizer.gd:126; gsplat_projection.glsl:75-80)
struct Uniforms {
    float camera_pos[3];
    float model_scale;
    int32_t dims[2];
    float time;
    float pad;
};
static_assert(sizeof(Uniforms) == 32, "uniform block must be 32 bytes");

// ---------------------------------------------------------------------------------------------
// radix sorter (radix_sort.cu)
// ---------------------------------------------------------------------------------------------
struct SortWorkspace {
    uint32_t *hist = nullptr;       // [4][256] global digit histograms
    uint32_t *status = nullptr;     // [4][max_tiles][256] decoupled look-back words
    uint32_t *tickets = nullptr;    // [4] dynamic tile counters (same allocation as hist)
    uint32_t *alt_keys = nullptr;   // ping-pong halves
    uint32_t *alt_vals = nullptr;
    uint32_t *n_dev = nullptr;      // device copy of n for the stand-alone sorter
    uint64_t max_n = 0;
    uint32_t max_tiles = 0;
    int grid_hist = 0, grid_sweep_pairs = 0, grid_sweep_keys = 0;
    // depth-order sort (gsr_set_depth_order; sort_workspace_enable_depth): [6][256] histograms + [6] tickets, [6][depth_max_tiles][256]
    // look-back words (depth_max_tiles counts the wide passes' tiles, the smaller ones)
    uint32_t *depth_hist = nullptr, *depth_status = nullptr;
    uint32_t depth_max_tiles = 0;
    int grid_sweep_wide = 0;
    size_t bytes() const;
};
int sort_workspace_create(SortWorkspace &ws, uint64_t max_n, bool need_alt_buffers);
void sort_workspace_destroy(SortWorkspace &ws);
// Sorts n (read on the device from *n_ptr, clamped to ws.max_n) pairs; 4 passes ping-pong between
// keys/vals and alt_keys/alt_vals (the reference's two buffer halves, rasterizer.gd:145), result back in
// keys/vals.  vals/alt_vals may be null (keys only).  *launches += kernels launched.
int sort_pairs_device(SortWorkspace &ws, uint32_t *keys, uint32_t *vals, const uint32_t *n_ptr, uint32_t *alt_keys,
                      uint32_t *alt_vals, cudaStream_t stream, int *launches);
// The depth-order sort's workspace (allocated once; GSR_ERR_OOM leaves ws as it was).
int sort_workspace_enable_depth(SortWorkspace &ws);
// Sorts n pairs stably by (key >> 16, depth word): the frame's (tile, ord(view depth)) order.  6 passes ping-pong between keys / vals /
// depth and the alt buffers; the result is back in keys / vals (depth is scratch: it ends sorted by the word alone).  *launches += 7.
int sort_pairs_depth_device(SortWorkspace &ws, uint32_t *keys, uint32_t *vals, uint32_t *depth, const uint32_t *n_ptr, uint32_t *alt_keys,
                            uint32_t *alt_vals, uint32_t *alt_depth, cudaStream_t stream, int *launches);
uint32_t sort_tile_keys();

// ---------------------------------------------------------------------------------------------
// stage launchers (projection.cu, ranges.cu, compositor.cu, ingest.cu)
// ---------------------------------------------------------------------------------------------
struct ProjectionArgs {
    const float4 *soa;       // 15 planes of `plane_stride` float4 each
    uint64_t plane_stride;
    uint32_t num_splats;
    float vp[32];            // view_matrix, projection_matrix (GLSL column-major)
    Uniforms u;
    float focal_base[2];     // (dims*0.5) * (P00, P11)           gsplat_projection.glsl:127-128
    float lim_lo[2], lim_hi[2];  // -+ (1/(P00,P11)) * 1.3          gsplat_projection.glsl:129,133
    int32_t band_y0, band_y1;  // tile rows [band_y0, band_y1) ...
    int32_t row_mod, row_rem;  // ... of which this context owns those with row % row_mod == row_rem (1, 0 = all)
    int32_t fast_reject;       // sharded fast mode: conservative early reject of splats that cannot touch an owned row;
                               // last_tile is then the LOCAL last emitted tile (global one by all-reduce, gsr_band_fixup)
    int32_t sh_bulk_min;       // warps with at least this many emitting lanes fetch their SH planes with TMA bulk copies
    int32_t fast_mode;         // fast sharded mode (row_mod > 1): last_tile is the LOCAL last emitted tile
    float w_frob2;             // upper bound of |mat3(view_matrix)|_2^2 (for the early reject)
    float4 *records;         // 3 float4 per splat id (RasterizeData layout)
    uint32_t *keys, *values;
    uint32_t capacity;
    float aa_variance;         // gsr_set_antialiasing: the 2D filter's variance (px^2); read only by the anti-aliased kernels.  It fills the
                               // padding after `capacity`: the struct's size, and so the offset of the kernels' second parameter, is unchanged
    unsigned long long *lookback;  // one word per projection CTA (256 splats)
    FrameState *frame;
};
static_assert(sizeof(ProjectionArgs) == 288 && offsetof(ProjectionArgs, lookback) == 272, "ProjectionArgs keeps its layout");
// sh_bands: SH bands the frame evaluates (1..4, at most the store's); the kernel reads planes 0-2 and the first sh_planes(sh_bands) SH planes.
// ortho: the frame's projection is orthographic (GSR_FLAG_ORTHOGRAPHIC; decided on the host at enqueue time, single-context only)
// aa: the frame is anti-aliased with a.aa_variance > 0 (gsr_set_antialiasing; read at enqueue time, single-context only)
// depth_words: non-null = the frame is sorted by view depth (gsr_set_depth_order; single-context only): the projection also stores
// depth_words[g] = depth_order_word(d) beside keys[g] / values[g], d the pair's splat's view depth
// cut: non-null = the frame takes the CUT = true kernels: it draws only the splats the cutout set keeps (gsr_set_cutouts) and, with the
// splat masks in use (gsr_select_*), drops hidden splats and highlights selected ones (single-context only); copied into the launch's
// parameters
struct CutParams;
// sh_half: the store holds binary16 SH planes (GSR_FLAG_SH_HALF; single-context only)
int launch_projection(const ProjectionArgs &a, cudaStream_t stream, int sh_bands = SH_BANDS_MAX, bool ortho = false, bool aa = false,
                      uint32_t *depth_words = nullptr, const CutParams *cut = nullptr, bool sh_half = false);

// gsr_set_cutouts: the active set, split by action on the host so that the kernel runs one loop over the KEEP volumes and one over the
// REMOVE volumes (vol[0, n_keep) then vol[n_keep, n_keep + n_remove)).  It travels by value as the projection's fourth __grid_constant__
// parameter (840 B): no device buffer, no copy, and frames already enqueued keep their set.
struct CutoutVolume {
    float m[12];     // to_local [A | t], column-major 3x4
    int32_t kind;    // shape (GSR_CUTOUT_BOX / _ELLIPSOID) | space << 1 (GSR_CUTOUT_FRAME / _SOURCE)
};
struct CutoutArgs {
    uint32_t n_keep, n_remove;
    CutoutVolume vol[GSR_MAX_CUTOUTS];
};
static_assert(sizeof(CutoutVolume) == 52 && sizeof(CutoutArgs) == 840, "CutoutArgs layout");

// gsr_set_cutouts / gsr_select_volume: is the tested position inside the unit box / sphere of volume v?  u = A p + t (one rounding per
// operation, in the order of include/gsr.h); IEEE comparisons, so a NaN coordinate is outside.  18 FP32 operations.
__device__ __forceinline__ bool cutout_inside(const CutoutVolume &v, float x, float y, float z) {
    const float *C = v.m;
    const float u0 = ((C[0] * x + C[3] * y) + C[6] * z) + C[9];
    const float u1 = ((C[1] * x + C[4] * y) + C[7] * z) + C[10];
    const float u2 = ((C[2] * x + C[5] * y) + C[8] * z) + C[11];
    if (v.kind & 1) return ((u0 * u0 + u1 * u1) + u2 * u2) <= 1.0f;   // GSR_CUTOUT_ELLIPSOID
    return fabsf(u0) <= 1.0f && fabsf(u1) <= 1.0f && fabsf(u2) <= 1.0f;
}

// Splat masks (gsr_select_*, gsr_hide_selection): one bit per SOURCE splat, 32 per word, over [0, max_splats).  hidden == nullptr: the
// masks are not in use.  A hidden splat leaves the projection like a cutout-removed one; a selected one, with `highlight`, has its colour
// replaced by c * keep + add per channel (an FMUL, then an FADD) after the SH clamp and the instance tint.
struct SplatMaskArgs {
    const uint32_t *hidden = nullptr;
    const uint32_t *selected = nullptr;
    float keep = 1.0f;              // 1 - strength
    float add[3] = {0.0f, 0.0f, 0.0f};   // rgb * strength
    uint32_t highlight = 0u;        // strength > 0
};
// The parameter of the CUT = true projection kernels: the cutout set and the splat masks (either may be empty).  It converts from a bare
// cutout set (no masks).
struct CutParams {
    CutoutArgs set;
    SplatMaskArgs masks;
    CutParams() = default;
    __host__ __device__ CutParams(const CutoutArgs &s) : set(s) {}
};
__device__ __forceinline__ bool mask_bit(const uint32_t *m, uint64_t s) { return ((m[s >> 5] >> (uint32_t)(s & 31u)) & 1u) != 0u; }
// One selection operation on a mask word: GSR_SELECT_* of the selected bits and the operation's inside bits (selection.cu, neighbors.cu)
__device__ __forceinline__ uint32_t combine_op(uint32_t op, uint32_t selected, uint32_t inside) {
    switch (op) {
        case GSR_SELECT_SET: return inside;
        case GSR_SELECT_ADD: return selected | inside;
        case GSR_SELECT_SUBTRACT: return selected & ~inside;
        default: return selected ^ inside;   // GSR_SELECT_TOGGLE
    }
}

// ---- selection operations (selection.cu) ----
constexpr int SELECT_MAX_VERTICES = GSR_MAX_SELECT_VERTICES;
// One region operation: inside(s) for the source splats s of [first, first + count) (every other splat is outside), combined into the
// selected mask by `op`, then selected &= ~hidden.  Polygon: q of splat s is sp = plane0[s].xyz * model_scale, or A sp + t with
// `instanced`, and inside = clip3 > 0 and the even-odd test of pix(vp, q) against xy[0, n).  Volume: cutout_inside(vol, sp or q).
struct SelectArgs {
    uint32_t *selected;
    const uint32_t *hidden;
    uint32_t words, op;
    uint64_t max_splats, first, count;
    const float4 *plane0;
    float model_scale;
    int32_t instanced;
    float A[12];
    float vp[32];
    float fw, fh;              // (float)(W - 1), (float)(H - 1)
    CutoutVolume vol;
    uint32_t n;
    float2 xy[SELECT_MAX_VERTICES];
};
enum SelectKind { SELECT_ALL = 0, SELECT_POLYGON = 1, SELECT_VOLUME = 2 };
struct InstanceDesc;
int launch_select_region(const SelectArgs &a, int kind, cudaStream_t stream);
// "select what you see": every pixel of [x0, x1) x [y0, y1) of an ID plane (gsr_set_splat_ids layout) marks the source splat of its
// drawn id in `scratch` (zero on entry), then selected = op(selected, scratch) & ~hidden and scratch is zeroed again.  warp_inst ==
// nullptr: no instances (ids below max_splats are sources); else the layout's `drawn_warps` warps of desc / warp_inst.
int launch_select_ids(const uint32_t *ids, int32_t width, int32_t x0, int32_t y0, int32_t x1, int32_t y1, const uint32_t *warp_inst,
                      const InstanceDesc *desc, uint32_t drawn_warps, uint64_t max_splats, uint32_t *scratch, uint32_t *selected,
                      const uint32_t *hidden, uint32_t words, uint32_t op, cudaStream_t stream);
// hidden |= selected, selected = 0
int launch_hide_selection(uint32_t *hidden, uint32_t *selected, uint32_t words, cudaStream_t stream);
// counts[0] += popcount(selected), counts[1] += popcount(hidden)
int launch_mask_counts(const uint32_t *selected, const uint32_t *hidden, uint32_t words, unsigned long long *counts, cudaStream_t stream);
int preload_selection_kernels();

// ---- selection transform edits (gsr_transform_selection; selection.cu) ----
// The operation's constants: to_source [L | t] (12 floats, column-major 3x4), then the SH band matrices M~_1, M~_2, M~_3 (3x3, 5x5, 7x7,
// row-major): 95 floats, the layout of GSR_BUF_EDIT_TRANSFORM.
__host__ __device__ constexpr int edit_matrix_offset(int l) { return l == 1 ? 12 : l == 2 ? 21 : 46; }   // M~_l, l = 1..3
constexpr int EDIT_TRANSFORM_FLOATS = 95;
// Host, float64: the 95 floats of to_source.  GSR_ERR_INVALID when det(L) is 0 or not finite (entries are checked by the caller).
int edit_transform_matrices(const float to_source[12], float out[EDIT_TRANSFORM_FLOATS]);
struct TransformArgs {
    float4 *dst;               // the store
    const float4 *src;         // the store itself, or a snapshot in its layout
    uint64_t plane_stride;
    const uint32_t *selected;
    uint32_t words;
    float m[EDIT_TRANSFORM_FLOATS];
};
// Rewrites every selected splat of the store from `src` (store bands and format as given).
int launch_transform_selection(const TransformArgs &a, int bands, bool sh_half, cudaStream_t stream);

// ---- selection colour edits (gsr_recolor_selection; selection.cu) ----
// The operation's constants: A (3x3 row-major), d (3), N~_1, N~_2, N~_3 (3x3 row-major each), s, t: 41 floats, the layout of
// GSR_BUF_EDIT_COLOR.
constexpr int EDIT_COLOR_D = 9, EDIT_COLOR_S = 39, EDIT_COLOR_FLOATS = 41;
__host__ __device__ constexpr int edit_color_band_offset(int l) { return 12 + 9 * (l - 1); }   // N~_l, l = 1..3
// Host, float64: the 41 floats of a validated edit (the caller checks the fields).
void edit_color_constants(const gsr_color_edit *e, float out[EDIT_COLOR_FLOATS]);
struct RecolorArgs {
    float4 *dst;               // the store
    const float4 *src;         // the store itself, or a snapshot in its layout
    uint64_t plane_stride;
    const uint32_t *selected;
    uint32_t words;
    float k[EDIT_COLOR_FLOATS];
};
// Rewrites the SH coefficients and opacity of every selected splat of the store from `src` (store bands and format as given).
int launch_recolor_selection(const RecolorArgs &a, int bands, bool sh_half, cudaStream_t stream);

// ---- splat delete and duplicate (gsr_delete_hidden, gsr_duplicate_selection; selection.cu) ----
// One pass of compact_store_kernel moves the planes of the splats of [0, n) whose bit is set (DELETE: hidden clear; DUPLICATE: selected
// set) to prefix (DELETE, in place) or n + prefix (DUPLICATE), in order.  A CTA owns COMPACT_TILE_WORDS mask words (one splat per thread)
// and takes its tile from an atomic ticket; its look-back status word (a 64-bit flag | count) and the ticket live in `lookback`.
enum CompactMode { COMPACT_DELETE = 0, COMPACT_DUPLICATE = 1 };
constexpr int COMPACT_THREADS = 256;
constexpr uint32_t COMPACT_TILE_WORDS = COMPACT_THREADS / 32;
// The look-back scratch of `words` mask words: one status word per tile, then the ticket.
__host__ __device__ constexpr uint64_t compact_lookback_words(uint32_t words) { return (words + COMPACT_TILE_WORDS - 1) / COMPACT_TILE_WORDS + 1; }
struct CompactArgs {
    float4 *soa;
    uint64_t plane_stride;
    uint64_t n;                        // the cloud's size: the kernel reads mask words [0, ceil(n / 32)) and moves splats below n
    const uint32_t *hidden, *selected;
    uint32_t *sel_out;                 // DELETE: the moved splats' selected bits at their destinations, OR-ed into a zeroed scratch mask
    unsigned long long *lookback;      // compact_lookback_words(ceil(n / 32)) words, zeroed before the launch
    unsigned long long *total;         // the tile owning the last word writes the number of moved (DUPLICATE) or kept (DELETE) splats
};
// The launch covers every tile of [0, n); nothing is launched for n == 0.
int launch_compact_store(const CompactArgs &a, int mode, int bands, bool sh_half, cudaStream_t stream);
// After a delete that kept k of n splats: selected = scratch (then zeroed) and hidden = 0 over all `words`, slots [k, n) vacant.
int launch_delete_finish(float4 *soa, uint64_t plane_stride, int planes, uint64_t k, uint64_t n, uint32_t *hidden, uint32_t *selected,
                         uint32_t *scratch, uint32_t words, cudaStream_t stream);
// After a duplicate of S splats behind n: selected = exactly [n, n + S), and hidden cleared there (the copies are not hidden).
int launch_duplicate_finish(uint64_t n, uint64_t S, uint32_t *hidden, uint32_t *selected, uint32_t words, cudaStream_t stream);
// counts[0] = popcount of the selected bits below n
int launch_count_selected(const uint32_t *selected, uint64_t n, unsigned long long *counts, cudaStream_t stream);

// ---- splat export (gsr_export_ply; selection.cu) ----
// The splats of [0, n) that are in scope (hidden == nullptr: the masks are not in use, every splat is kept and none selected) and not
// vacant become 3DGS vertex rows of degree `degree`, in store order.  A counting pass gives their number; the writing pass places a
// CTA's rows (one tile of COMPACT_TILE_WORDS mask words) at its prefix with the look-back of compact_store_kernel.
__host__ __device__ constexpr uint32_t export_row_floats(int degree) { return 17u + 3u * (uint32_t)((degree + 1) * (degree + 1) - 1); }
struct ExportArgs {
    const float4 *soa;
    uint64_t plane_stride;
    uint64_t n;
    const uint32_t *hidden, *selected;
    uint32_t selected_only;            // GSR_EXPORT_SELECTED
    int32_t degree;                    // d, 0 .. the stored degree
    float *dst;                        // device memory: the rows, export_row_floats(degree) floats each
    unsigned long long *lookback;      // compact_lookback_words(ceil(n / 32)) words, zeroed before the writing launch
    unsigned long long *count;         // zeroed before the counting launch: the number of exported splats
};
// The dynamic shared memory of a writing CTA: its rows
__host__ __device__ constexpr size_t export_shared_bytes(int degree) { return sizeof(float) * COMPACT_THREADS * export_row_floats(degree); }
int launch_export_count(const ExportArgs &a, cudaStream_t stream);
int launch_export_rows(const ExportArgs &a, int bands, bool sh_half, cudaStream_t stream);

// The float64 decomposition of the export (export_ply_kernel in selection.cu, compress_chunk_kernel in compressed_ply.cu).
// One cyclic-Jacobi rotation of the symmetric A in the plane (P, Q), accumulated into the columns of V (Numerical Recipes' jacobi):
// A[P][Q] becomes exactly 0.  With `late` (after three sweeps) an element that is negligible beside both diagonal entries is zeroed
// without a rotation.
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&A)[3][3], double (&V)[3][3], bool late) {
    constexpr int R = 3 - P - Q;
    const double apq = A[P][Q];
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq);
    if (late && fabs(A[P][P]) + g == fabs(A[P][P]) && fabs(A[Q][Q]) + g == fabs(A[Q][Q])) {
        A[P][Q] = A[Q][P] = 0.0;
        return;
    }
    const double theta = (A[Q][Q] - A[P][P]) / (2.0 * apq);
    double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));   // theta^2 = inf: t = 0, apq is negligible
    if (theta < 0.0) t = -t;
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
    A[P][P] -= t * apq;
    A[Q][Q] += t * apq;
    A[P][Q] = A[Q][P] = 0.0;
    const double arp = A[R][P], arq = A[R][Q];
    A[R][P] = A[P][R] = arp - s * (arq + arp * tau);
    A[R][Q] = A[Q][R] = arq + s * (arp - arq * tau);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double vp = V[r][P], vq = V[r][Q];
        V[r][P] = vp - s * (vq + vp * tau);
        V[r][Q] = vq + s * (vp - vq * tau);
    }
}

// scale and rot of the covariance words (S00 S01 S02 S11 S12 S22) by the rule of include/gsr.h "Splat export"
__device__ __forceinline__ void export_scale_rot(const float4 &p1, const float4 &p2, float *out) {
    const float w6[6] = {p1.x, p1.y, p1.z, p1.w, p2.x, p2.y};
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 6; ++i) finite = finite && fabsf(w6[i]) <= 3.402823466e38f;
    if (!finite) {
        const float qnan = __uint_as_float(0x7FC00000u);
        out[0] = out[1] = out[2] = qnan;
        out[3] = 1.0f; out[4] = out[5] = out[6] = 0.0f;
        return;
    }
    double A[3][3] = {{w6[0], w6[1], w6[2]}, {w6[1], w6[3], w6[4]}, {w6[2], w6[4], w6[5]}};
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
#pragma unroll 1
    for (int sweep = 0; sweep < 16; ++sweep) {
        if (A[0][1] == 0.0 && A[0][2] == 0.0 && A[1][2] == 0.0) break;
        jacobi_rotate<0, 1>(A, V, sweep >= 3);
        jacobi_rotate<0, 2>(A, V, sweep >= 3);
        jacobi_rotate<1, 2>(A, V, sweep >= 3);
    }
    double l[3] = {A[0][0], A[1][1], A[2][2]};
    // ascending eigenvalues with their columns: compare-exchange (0, 1), (1, 2), (0, 1)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = k == 1 ? 1 : 0, j = i + 1;
        if (l[j] < l[i]) {
            const double t = l[i]; l[i] = l[j]; l[j] = t;
#pragma unroll
            for (int r = 0; r < 3; ++r) { const double v = V[r][i]; V[r][i] = V[r][j]; V[r][j] = v; }
        }
    }
    const double det = V[0][0] * (V[1][1] * V[2][2] - V[1][2] * V[2][1]) - V[0][1] * (V[1][0] * V[2][2] - V[1][2] * V[2][0]) +
                       V[0][2] * (V[1][0] * V[2][1] - V[1][1] * V[2][0]);
    if (det < 0.0) { V[0][0] = -V[0][0]; V[1][0] = -V[1][0]; V[2][0] = -V[2][0]; }
#pragma unroll
    for (int i = 0; i < 3; ++i) out[i] = (float)(0.5 * log(l[i] > 2.2250738585072014e-308 ? l[i] : 2.2250738585072014e-308));
    // Shepperd: the largest of 4w^2 - 1 = tr, and 4x^2 - 1, 4y^2 - 1, 4z^2 - 1 (the diagonal entries), first on a tie
    const double tr = (V[0][0] + V[1][1]) + V[2][2];
    int k = 0;
    double best = tr;
#pragma unroll
    for (int i = 0; i < 3; ++i) if (V[i][i] > best) { best = V[i][i]; k = i + 1; }
    double q[4];
    if (k == 0) {
        const double w = 0.5 * sqrt(1.0 + tr), f = 0.25 / w;
        q[0] = w; q[1] = (V[2][1] - V[1][2]) * f; q[2] = (V[0][2] - V[2][0]) * f; q[3] = (V[1][0] - V[0][1]) * f;
    }
#pragma unroll
    for (int kk = 1; kk <= 3; ++kk) {   // unrolled, so that every index is a constant and V and q stay in registers
        if (k != kk) continue;
        const int a = kk - 1, b = kk % 3, c = (kk + 1) % 3;
        const double v = 0.5 * sqrt(((1.0 + V[a][a]) - V[b][b]) - V[c][c]), f = 0.25 / v;
        q[0] = (V[c][b] - V[b][c]) * f;
        q[1 + a] = v; q[1 + b] = (V[b][a] + V[a][b]) * f; q[1 + c] = (V[c][a] + V[a][c]) * f;
    }
    const double norm = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]), sg = q[0] < 0.0 ? -1.0 : 1.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) out[3 + i] = (float)(sg * (q[i] / norm));
}

// ---- compressed PLY (gsr_export_compressed_ply: compressed_ply.cu; gsr_upload_compressed_ply: ingest.cu) ----
// A file's rows come in chunks of GSR_COMPRESSED_CHUNK; row r of a degree-d file has 4 packed words and cply_sh_bytes(d) SH bytes.
constexpr uint32_t CPLY_CHUNK = GSR_COMPRESSED_CHUNK;
constexpr uint32_t CPLY_CHUNK_FLOATS = 18;                 // what the export writes; 12 (no colour range) is accepted on upload
__host__ __device__ constexpr uint32_t cply_sh_bytes(int degree) { return 3u * (uint32_t)((degree + 1) * (degree + 1) - 1); }
constexpr uint32_t CPLY_NOT_EXPORTED = 0xFFFFFFFFu;        // the sort key of a slot that is not exported: it sorts behind every row
// The bounds pass's result: the order-preserving words (depth_order_word) of the exported positions' least and greatest x, y, z, and
// their count.  Cleared to lo = 0xFFFFFFFF, hi = 0, count = 0 before the pass.
struct CompressBounds {
    uint32_t lo[3], hi[3];
    unsigned long long count;
};
struct CompressArgs {
    const float4 *soa;
    uint64_t plane_stride;
    uint64_t n;                        // slots [0, n) are tested
    const uint32_t *hidden, *selected; // hidden == nullptr: the masks are not in use (every splat kept, none selected)
    uint32_t selected_only;            // GSR_EXPORT_SELECTED
    uint32_t morton;                   // GSR_COMPRESS_MORTON
    int32_t degree;                    // d of the file, 0 .. the stored degree
    CompressBounds *bounds;
    uint32_t *keys, *vals;             // n each: (key, slot) of every slot; sorted, the first `rows` vals are the rows' slots in file order
    uint32_t *sort_n;                  // the sort's device count: the key pass writes n
    uint64_t rows;                     // the exported count (the chunk pass)
    float *chunks;                     // device memory: ceil(rows / 256) x 18 floats
    uint32_t *packed;                  // rows x 4 words
    uint8_t *sh;                       // rows x cply_sh_bytes(degree) bytes (unused for d = 0)
};
int launch_compress_bounds(const CompressArgs &a, cudaStream_t stream);
int launch_compress_keys(const CompressArgs &a, cudaStream_t stream);
int launch_compress_chunks(const CompressArgs &a, int bands, bool sh_half, cudaStream_t stream);
int preload_compressed_kernels();
// The decode: rows [0, rows) of a compressed file (device memory) become splats first + r of the store, by the rule of gsr_upload_ply for
// the decoded float rows with the alpha stored directly.
struct DecompressArgs {
    const float *chunks;               // ceil(rows / 256) x chunk_floats
    const uint32_t *packed;
    const uint8_t *sh;
    uint64_t rows;
    uint32_t chunk_floats;             // 18, or 12 (colours are the unorm8 values themselves)
    int32_t degree;                    // the file's, 0..3
    float creation_time;
    float4 *soa;
    uint64_t plane_stride, first;
};
int launch_compressed_to_soa(const DecompressArgs &a, int bands, bool sh_half, cudaStream_t stream);

// ---- splat property selection (gsr_select_where, gsr_splat_histogram; selection.cu) ----
// The planes a property reads beyond plane 0 (a size, volume or isotropy reads planes 1 and 2).  The kernels are templated on the union
// of a filter set's bits, so each reads only the planes its set needs.
enum PropPlanes : int { PROP_P1 = 1, PROP_P2 = 2, PROP_P3 = 4, PROP_PC = 16 };   // (8: the binary16 bit of the variant tables)
__host__ __device__ constexpr int prop_planes(int32_t p) {
    return p == GSR_PROP_OPACITY ? PROP_P2 : p == GSR_PROP_COLOR_DISTANCE ? PROP_P3 : PROP_P1 | PROP_P2;
}
// The contribution properties (GSR_PROP_CONTRIBUTION ..) read the contribution buffer (PROP_PC) and no plane; the kernels that can
// meet them test for them before prop_planes.
__host__ __device__ constexpr bool prop_is_contrib(int32_t p) { return p >= GSR_PROP_CONTRIBUTION && p <= GSR_PROP_CONTRIBUTING_PIXELS; }
__host__ __device__ constexpr int prop_sources(int32_t p) { return prop_is_contrib(p) ? PROP_PC : prop_planes(p); }
// inside(s) for the splats s of [first, first + count) (the caller bounds it by the cloud's n), combined into the selected mask by `op`
// over every word, then selected &= ~hidden.
struct WhereArgs {
    uint32_t *selected;
    const uint32_t *hidden;
    uint32_t words, op;
    uint64_t first, count;
    const float4 *soa;
    uint64_t plane_stride;
    uint32_t n;                                   // filters
    gsr_splat_filter f[GSR_MAX_SPLAT_FILTERS];
    const gsr_splat_contribution *contrib;        // PROP_PC only: the contribution buffer (gsr_set_splat_contribution)
};
// planes: the union of prop_sources over the set; sh_half: the store's SH format (read only when the set reads plane 3)
int launch_select_where(const WhereArgs &a, int planes, bool sh_half, cudaStream_t stream);
// The histogram's device buffer: the counters, then the min / max keys, then the edges.  The keys are kept as ints so that one
// atomicMax serves both: keys[0] = max of hist_signed_key(~ord(v)) (the least ord(v)), keys[1] = max of hist_signed_key(ord(v)) (the
// greatest), ord the map of gsr_set_depth_order; INT32_MIN, the key of a NaN, means no value.
__host__ __device__ __forceinline__ int32_t hist_signed_key(uint32_t k) { return (int32_t)(k ^ 0x80000000u); }
constexpr uint32_t HIST_COUNTS = GSR_MAX_HISTOGRAM_BINS + 3;
constexpr size_t HIST_KEYS_OFFSET = sizeof(unsigned long long) * HIST_COUNTS, HIST_EDGES_OFFSET = HIST_KEYS_OFFSET + 2 * sizeof(uint32_t);
constexpr size_t HIST_BUFFER_BYTES = HIST_EDGES_OFFSET + sizeof(float) * (GSR_MAX_HISTOGRAM_BINS + 1);
struct HistArgs {
    const float4 *soa;
    uint64_t plane_stride;
    uint64_t first, count;                        // the tested range, bounded by n
    const uint32_t *hidden, *selected;            // hidden == nullptr: the masks are not in use (nothing hidden, nothing selected)
    uint32_t selected_only;                       // GSR_HISTOGRAM_SELECTED
    uint32_t bins, top;                           // top: the largest power of two <= max(bins - 1, 1) (the binary search's first step)
    gsr_splat_filter prop;
    unsigned long long *counts;                   // bins + 3, zeroed
    int32_t *keys;                                // INT32_MIN, INT32_MIN on entry: the least and greatest ord(v), as above
    const float *edges;                           // bins + 1
    const gsr_splat_contribution *contrib;        // PROP_PC only: the contribution buffer (gsr_set_splat_contribution)
};
int launch_splat_histogram(const HistArgs &a, int planes, bool sh_half, int sm_count, cudaStream_t stream);

// ---- splat neighbourhood selection (gsr_select_neighborhood; neighbors.cu) ----
// The grid: a participant's cell is floor(x / h) per axis in float64, clamped to [-2^62, 2^62]; a cell's 32-bit key is a hash of its
// three coordinates, and the key's top p bits are its bucket (2^p buckets).  The pairs (key, slot) of the participants are sorted by key,
// so a bucket is one range of the sorted entries, and within it the cells of different keys are apart.  start[b] is the first entry of
// bucket b (start[2^p] = the participant count), with NB_IMPURE set when the bucket holds entries of more than one cell.
constexpr uint32_t NB_IMPURE = 0x80000000u;
constexpr uint32_t NB_NONE = 0xFFFFFFFFu;   // parent of a slot that does not participate
constexpr uint32_t NB_SEED = 0x80000000u;   // size word of a root: the cluster holds a selected participant
struct NeighborCounters {                   // one device block, read back page-locked
    uint32_t n, pad;                        // participants (the sort's device count)
    unsigned long long candidates, inside, clusters, largest;
};
struct NeighborArgs {
    const float4 *plane0;
    const uint32_t *hidden;
    uint32_t *selected;
    uint32_t words, op;
    uint64_t first, count;                  // the tested range, bounded by the cloud's n
    double h;                               // (double)radius (1 + 2^-20)
    float r2;                               // radius radius
    uint32_t mode, threshold;               // GSR_NEIGHBOR_*, count
    uint32_t shift;                         // 32 - p: bucket = key >> shift
    uint32_t *keys, *vals;                  // max_splats each: the participants' (key, slot), sorted by key
    uint32_t *parent, *size;                // max_splats each, by slot: the union-find (the sort's ping-pong halves once it is done)
    float4 *pos;                            // max_splats: sorted entry e = (x, y, z, slot bits) of slot vals[e]
    uint32_t *start;                        // 2^p + 1
    uint32_t *inside;                       // `words` scratch mask words, zero on entry and left zero: SPARSE / GROW
    NeighborCounters *ctr;                  // zero on entry
};
// The grid's parameters: h, and p for a tested range of `count` slots (the least p >= 1 with 2^p >= 2 count)
double neighbor_cell_size(float radius);
uint32_t neighbor_bucket_bits(uint64_t count);
// Stage launchers, in call order; the entry grids cover the tested range (the participant count is read on the device).  Between keys
// and grid the caller sorts (keys, vals) with sort_pairs_device, parent and size as the ping-pong halves.
int launch_neighbor_keys(const NeighborArgs &a, cudaStream_t stream);
int launch_neighbor_grid(const NeighborArgs &a, uint64_t max_splats, cudaStream_t stream);   // also clears parent and size
int launch_neighbor_budget(const NeighborArgs &a, cudaStream_t stream);
int launch_neighbor_select(const NeighborArgs &a, cudaStream_t stream);   // the mode's queries, then the mask words
int preload_neighbor_kernels();

// gsr_set_depth_order: the order-preserving map of a float's bits to an unsigned word (negative: all bits flipped; positive: the sign
// bit set).  Every finite value orders as its float does, -0 just before +0.
__host__ __device__ __forceinline__ uint32_t depth_order_word(uint32_t bits) { return bits ^ ((bits >> 31) ? 0xFFFFFFFFu : 0x80000000u); }

// ---------------------------------------------------------------------------------------------
// splat instances (gsr_set_instances): ranges of the splat buffer drawn with their own affine transform into frame space
// ---------------------------------------------------------------------------------------------
// Per instance and frame (instance_prepare_kernel): V_k = V * [A|t] (16), cam_k = B * camera_pos + u (3), A (9), t (3), pad.
constexpr int INSTANCE_FRAME_FLOATS = 32;
constexpr int INSTANCE_XFORM_FLOATS = 24;   // what the host hands the prepare kernel per instance: A|t as given, then B|u = its inverse
struct InstanceDesc {                       // static per layout
    uint64_t first;                         // first source splat
    uint32_t count;                         // source splats
    uint32_t warp0;                         // first drawn warp: drawn ids [32 warp0, 32 warp0 + count)
};
// Per instance and frame, the appearance (gsr_set_instance_appearance): tint r g b, opacity, live (uint32 bits: the source splats drawn,
// min(count, draw_count), 0 for opacity 0), pad.
constexpr int INSTANCE_APPEARANCE_FLOATS = 8;
struct InstanceArgs {
    const float *frame;                     // INSTANCE_FRAME_FLOATS per instance: this frame's constants
    const InstanceDesc *desc;
    const uint32_t *warp_inst;              // instance of every drawn warp of the grid; 0xFFFFFFFF = padding warp
    const float *appearance = nullptr;      // INSTANCE_APPEARANCE_FLOATS per instance, this frame's; null: every instance at the default
};
// a.num_splats = D (drawn ids), a.records indexed by drawn id
int launch_projection_instanced(const ProjectionArgs &a, const InstanceArgs &ia, cudaStream_t stream, int sh_bands = SH_BANDS_MAX, bool ortho = false,
                                bool aa = false, uint32_t *depth_words = nullptr, const CutParams *cut = nullptr, bool sh_half = false);
// Per instance and frame with motion vectors (gsr_set_motion_vectors): the previous frame's to_frame [A' | t'] (12).
constexpr int INSTANCE_PREV_FLOATS = 12;
// one CTA: out[k] = the constants of instance k for the frame's view matrix vp[0..15] and camera_pos cam[0..2]; xf = k x 24 floats
// (mapped page-locked host memory on the frame path).  With an appearance (count x 8 floats, same memory) its rows go to appearance_out,
// with previous transforms (count x 12 floats, same memory) they go to prev_out.
int launch_instance_prepare(const float *xf, const float *vp, const float *cam, uint32_t count, float *out, cudaStream_t stream,
                            const float *appearance = nullptr, float *appearance_out = nullptr, const float *prev_xf = nullptr,
                            float *prev_out = nullptr);

// ---------------------------------------------------------------------------------------------
// multi-GPU shard group (group.cu, gsr_group_attach): flag words + receive segments + record tables in every rank's arena
// ---------------------------------------------------------------------------------------------
constexpr int GROUP_MAX = 16;                                   // ranks per group (one NVSwitch domain)
// Receive segments and record tables exist three times (frame seq % 3): a source's scatter projection of frame f+1 runs while the
// destinations still composite frame f (front / back overlap, gsr_api.cu), and frame f-1's consumers are only known to be done
// through the chain  scatter(f+1) after own ranges(f) after all sources' scatter(f) after their ranges(f-1) after their compositor(f-2).
constexpr int GROUP_PHASES = 3;
#define GSR_GROUP_TIMEOUT_NS 2000000000ull                      // every device-side wait gives up after 2 s
struct GroupFlags {                                             // offset 0 of a rank's arena; written by the peers over NVLink
    // [frame phase = seq % 3][source rank][0] = seq << 32 | pairs the source sent to THIS rank's receive segment,
    //                                     [1] = seq << 32 | (largest tile id touched by the source's splats + 1)
    unsigned long long seg_meta[GROUP_PHASES][GROUP_MAX][2];
    uint32_t done[GROUP_MAX];               // presenting rank: done[r] = seq of the newest frame whose rows from rank r have landed
    uint32_t released;                      // set by the presenting rank: frames with seq <= released no longer need their slot
    uint32_t error;                         // local: a wait timed out (1 = segments of a peer, 2 = done / released)
    uint32_t scat_ticket;                   // local: CTAs of the scatter projection that have finished
    int32_t scat_last;                      // local: atomicMax target, last tile + 1 over this rank's slice
    unsigned long long seg_total[GROUP_MAX];  // local: pairs this rank sent to each destination this frame (scan total)
    uint32_t seg_prefix[GROUP_MAX + 1];     // local: exclusive prefix of the received (clamped) segment lengths, [world] = M of this rank
};
constexpr size_t GROUP_FLAGS_BYTES = 4096;                      // the receive segments and record tables follow the flag page
static_assert(sizeof(GroupFlags) <= GROUP_FLAGS_BYTES, "flag page");
struct GroupPeers {                                             // the same pointers on every rank, indexed by rank
    GroupFlags *flags[GROUP_MAX];
    int world, rank;
};
// What the scatter projection of one rank needs to know about the group: every destination's record table and receive segment
// (peer pointers) of the current frame phase (seq % 3; called parity below), and this rank's slice of the splats.
struct ScatterPeers {
    int world, rank, parity;
    uint32_t seq;
    uint32_t first, count;                  // this rank projects splats [first, first + count)
    uint32_t seg_cap;                       // pairs one source may send to one destination per frame
    float4 *records[GROUP_MAX];             // destination d's record table (3 float4 per splat id) of this parity
    uint32_t *keys[GROUP_MAX];              // destination d's receive segment for THIS source: pairs land at [0, seg_cap)
    uint32_t *values[GROUP_MAX];
    GroupFlags *flags[GROUP_MAX];
    unsigned long long *lookback;           // [blocks][world] scan links of this launch (zeroed)
};
// Projection sharded by SPLATS (group mode): rank r projects its slice with the full-frame maths of projection_kernel and emits every
// (key, value) pair and every record straight into the memory of the rank that owns the pair's tile row (row % world), in splat-id
// order per destination -- the all-to-all of SURVEY 8e's "alternative" fused into the kernel as peer stores over NVLink.
int launch_projection_scatter(const ProjectionArgs &a, const ScatterPeers &sp, cudaStream_t stream);
uint32_t projection_scatter_blocks(uint32_t count);
// destination side: wait for every source's segment of this frame, publish M / overflow / the frame-global last tile, then pack the
// world receive segments into the contiguous sort input (source-rank order = splat-id order)
int launch_group_wait_segments(GroupFlags *flags, int parity, int world, uint32_t seq, uint32_t seg_cap, uint32_t capacity, FrameState *frame, cudaStream_t stream);
int launch_gather_segments(const GroupFlags *flags, int world, uint32_t seg_cap, const uint32_t *rx_keys, const uint32_t *rx_vals, uint32_t *keys, uint32_t *vals,
                           int grid, cudaStream_t stream);
// 64-byte FrameState -> mapped pinned host memory with system-scope stores (no copy engine involved)
int launch_publish_frame_state(const FrameState *frame, FrameState *host_mapped, cudaStream_t stream);
int launch_group_wait_released(GroupFlags *flags, uint32_t need, cudaStream_t stream);
int launch_group_wait_done(GroupFlags *flags, int world, uint32_t seq, cudaStream_t stream);
int launch_group_signal_done(const GroupPeers &peers, int root, int rank, uint32_t seq, cudaStream_t stream);
int launch_group_release(const GroupPeers &peers, int world, uint32_t value, cudaStream_t stream);
uint32_t projection_num_blocks(uint32_t num_splats);

// sharded: 0 = full frame, 1 = exact sharded mode (global last tile known from the projection), 2 = fast sharded mode
// (local last tile -> *sync_word = tile + 1; the frame-global quirk is applied later by launch_band_fixup).
int launch_tile_ranges(const uint32_t *sorted_keys, const FrameState *frame, uint2 *bounds, uint32_t num_tiles,
                       int quirks, int sharded, int32_t *sync_word, int grid, cudaStream_t stream);
int launch_band_fixup(const int32_t *global_last_plus1, float4 *out, int32_t width, int32_t height, int32_t tiles_x, int32_t num_tiles_total,
                      int32_t band_y0, int32_t band_y1, int32_t row_mod, int32_t row_rem, cudaStream_t stream);

struct CompositeArgs {
    const float4 *records;
    const uint32_t *values;
    const uint2 *bounds;
    float4 *out;             // W*H RGBA32F
    int32_t width, height, tiles_x;
    int32_t tile_begin;      // first tile id rendered (band_y0 * tiles_x, or the first owned row)
    int32_t row_step;        // distance in tile rows between consecutive owned rows (1 = contiguous band)
    int32_t num_tiles;       // tiles rendered
    float heatmap_factor;
    uint32_t target_tile_id; // 0xFFFFFFFF = none (rasterizer.gd:158)
    float4 *pick;            // tile_splat_pos buffer (gsplat_render.glsl:33-36)
    FrameState *frame;       // ticket counter (comp_head must be 0) + staged-instance counter
    int32_t count_staged;    // add this launch's consumed instances to frame->staged (0 for the pick re-dispatch)
    const uint32_t *order;   // optional: ticket k renders owned tile order[k] (longest chains first, launch_tile_order); nullptr = natural order
    uint32_t *consumed;      // optional [num_tiles]: chunks each owned tile blended before its stop rule fired | 1u << 31 (next frame's order hint)
    int32_t ctas_per_sm;     // resident CTAs per SM of the persistent grid
    int32_t sm_count;
    int32_t contract;        // 1: the gsr spec (explicit fma at the GLSL-legal contraction points); 0: no contraction (GSR_FLAG_UNCONTRACTED_BLEND)
    ulonglong4 *trace;       // optional schedule trace (debug): {tile<<32|smid, t0_ns, t1_ns, consumed<<32|list_chunks<<1|1}
    uint32_t *trace_count;
    uint32_t trace_cap;
    // depth compositing (gsr_set_depth_compositing); depth_out == nullptr: off, the reference's opaque frame
    float view_z[4];           // V[2], V[6], V[10], V[14] of view_proj: the splat's view depth is -(((V2*x + V6*y) + V10*z) + V14)
    const float *scene_depth;  // optional W*H linear scene depth; a pixel stops at the first splat not in front of it (nullptr: +inf)
    float *depth_out;          // W*H: D / (1 - t) of the blended splats, +inf where nothing was blended
};
// Motion vectors (gsr_set_motion_vectors, with depth compositing only): the second __grid_constant__ parameter of the motion variants
// of the compositor.  Per staged splat m = pix(prev_vp, p') - pix(vp, p) (compositor.cu motion_of), accumulated like the depth.
struct MotionArgs {
    float vp[32];               // this frame's view_proj
    float prev_vp[32];          // the previous frame's (this frame's own when there is none)
    float fw, fh;               // (float)(W - 1), (float)(H - 1)
    float *motion_out;          // W*H float2: M / (1 - t), (0, 0) where nothing was blended
    // instances (warp_inst == nullptr: none, p' = p): the source splat s = desc[k].first + (v - 32 desc[k].warp0) of drawn id v and
    // warp instance k = warp_inst[v >> 5], sp = plane0[s].xyz * model_scale, p' = A'_k * sp + t'_k
    const uint32_t *warp_inst;
    const InstanceDesc *desc;
    const float *prev_xf;       // 12 floats per instance: its previous to_frame (this frame's own when there is none)
    const float4 *plane0;       // plane 0 of the store
    float model_scale;
};
// Splat and instance IDs (gsr_set_splat_ids, with depth compositing only): carried in the second __grid_constant__ parameter of the ID
// variants of the compositor, beside the motion constants when both are on.  Per pixel, the drawn id v of the blended splat with the
// largest t - t * (1 - alpha) (the first in sorted order on a tie) and warp_inst[v >> 5].
constexpr uint32_t NO_ID = 0xFFFFFFFFu;
struct SplatIdArgs {
    uint32_t *ids_out;          // W*H uint2 (v, k); (NO_ID, NO_ID) where no splat has t - t' > 0
    const uint32_t *warp_inst;  // instance of every drawn warp; nullptr: no instances, k = NO_ID
};
// Splat contribution (gsr_set_splat_contribution, with depth compositing only, without motion vectors and IDs): the second
// __grid_constant__ parameter of composite_contrib_kernel.  Every (in-image pixel, blended splat) with w = t - t' > 0 adds
// q(w) = __float2uint_rn(w * 2^24), 1, max(peak, w) to the record of the splat's source slot, and the frame once to its views.
struct ContribArgs {
    gsr_splat_contribution *accum;   // max_splats records, indexed by source slot
    const uint32_t *warp_inst;       // instance of every drawn warp; nullptr: no instances, the slot is the drawn id
    const InstanceDesc *desc;        // slot = desc[k].first + (v - 32 desc[k].warp0) for k = warp_inst[v >> 5]
    uint32_t *frames;                // +1 per frame that did not overflow the duplicate capacity
    uint32_t epoch;                  // the frame's: non-zero, the same for gsr_render's re-render of an overflowed frame
};
int launch_composite(const CompositeArgs &a, cudaStream_t stream, const MotionArgs *motion = nullptr, const SplatIdArgs *ids = nullptr,
                     const ContribArgs *contrib = nullptr);
int composite_max_ctas_per_sm(int *out);
// order[0 .. num_tiles) = owned-tile indices sorted by descending expected chain length: the chunk count the tile consumed in the
// previous frame (hint[k] with bit 31 set; the bit is cleared here) or, without a hint, its list length in chunks capped at
// `cap_chunks` (a list is rarely consumed beyond ~20 chunks).  Counting sort, one CTA.  Scheduling only: pixels do not depend on it.
// Sparse frames: when at most `sparse_tiles` owned tiles are occupied, frame->comp_cta_limit = sparse_cta_limit (one CTA per SM:
// a chain that has an SM to itself advances fastest); otherwise 0 = every launched CTA works.
int launch_tile_order(const uint2 *bounds, int32_t tile_begin, int32_t row_step, int32_t tiles_x, int32_t num_tiles, uint32_t *hint, uint32_t *order,
                      FrameState *frame, uint32_t sparse_tiles, uint32_t sparse_cta_limit, cudaStream_t stream);

// The standard 62-property layout of the original 3DGS trainer (x y z nx ny nz f_dc_0..2 f_rest_0..44 opacity scale_0..2 rot_0..3).
constexpr gsr_ply_layout PLY_LAYOUT_3DGS = {62u, 3u, 0, 6, 9, 54, 55, 58};
// PLY vertices of any layout -> the first `planes` (= soa_planes(store bands)) SoA planes
// filter_3d: index of Mip-Splatting's per-splat `filter_3D` property in a vertex (gsr_upload_ply_filtered), -1 = none
// sh_half (GSR_FLAG_SH_HALF): the SH planes are written as packed binary16 values (then planes = soa_planes(store bands, true))
int launch_ply_to_soa(const float *ply, const gsr_ply_layout &layout, uint64_t count, float creation_time, float4 *soa, uint64_t plane_stride,
                      uint64_t first, int planes, cudaStream_t stream, int32_t filter_3d = -1, bool sh_half = false);
// present.cu: RGBA32F frame -> GSR_OUT_* (| GSR_OUT_SRGB_TO_LINEAR)
int launch_present(const float4 *rgba, void *out, uint64_t pixels, int format, cudaStream_t stream);
size_t present_bytes_per_pixel(int format);
int launch_aos_to_soa(const float4 *aos, uint64_t count, float4 *soa, uint64_t plane_stride, uint64_t first, int planes, cudaStream_t stream,
                      bool sh_half = false);

// cudaFuncGetAttributes on every kernel of a file: defeats lazy module loading before the first frame
int preload_group_kernels();
int preload_projection_kernels();
int preload_projection_half_kernels();   // the binary16-store variants (GSR_FLAG_SH_HALF contexts only)
int preload_sort_kernels();
int preload_ranges_kernels();
int launch_frame_clear(FrameState *frame, unsigned long long *links, uint32_t n_links, uint2 *bounds, uint32_t n_bounds, cudaStream_t stream);
int preload_ingest_kernels();
int preload_present_kernels();
int preload_composite_kernels();

}  // namespace gsr
