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
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
