// compositor.cu -- stage 4: per-tile front-to-back alpha blend.  Replaces gsplat_render.glsl:50-111.
//
// One CTA per 16x16 tile like the reference's workgroup, 256-splat chunks staged in shared memory, the same per-pixel
// arithmetic and the same tile-stop vote.  How the blend is issued and scheduled on sm_90:
//   * the blend is almost all FP32 arithmetic, so every thread owns TWO horizontally adjacent pixels: the per-splat shared-memory loads
//     and broadcasts are paid once for two pixels, and the two pixels' dependency chains interleave (Hopper has no packed
//     fp32x2 instructions; each F2 operation below is two scalar IEEE binary32 operations with explicit rounding, so results
//     stay bit-identical to the oracle);
//   * per-splat control flow is gone: dead pixels (t <= 1/255, gsplat_render.glsl:79) keep their state by select, the warp-level
//     "all dead" test runs once per 4 splats on the transmittance of half a group earlier (off the loop-carried path), and the
//     last chunk is padded with null splats (opacity 0);
//   * the transmittance chain is two instructions per splat: alpha and 1 - alpha are formed off the critical path, the update is
//     FMUL + select per pixel (`t = alive ? t * (1 - alpha) : t`, bit-identical to multiplying by 1 - 0);
//   * the conic is pre-scaled at staging time (-0.5*cx, -0.5*cz, -cy: exact power-of-two/sign changes) so the `-0.5 * (...)`
//     multiply of :84 disappears from the inner loop without changing any rounding;
//   * the gather `culled_buffer[sort_buffer[...]]` (:72) for chunk i+1 is issued into registers before the blend loop of chunk i
//     (software prefetch), and the (a, b) words of splat group g+1 are read from shared memory while group g is blended;
//   * the tile-stop vote `atomicAdd(shared_t, uint(t*255))` (:97) is a warp reduction + 4 shared words;
//   * scheduling: a tile is a sequential chain of up to ~19 chunks, a c3 frame has ~1250 such chains of very different length,
//     and the SM's warp scheduler favours its oldest warps -- so the persistent grid takes tiles LONGEST-FIRST (tile_order_kernel:
//     the previous frame's consumed chunk count of the tile, else its list length), keeps few CTAs per SM and never migrates a
//     tile (handing a tile back costs a spill + restore and makes long chains young again).
// Arithmetic contract: "gsr deterministic math" (common.cuh): the GLSL-legal contractions of :84 and :89 are explicit fma
// (CONTRACT = true, the default); CONTRACT = false (GSR_FLAG_UNCONTRACTED_BLEND) evaluates :84-90 with no contraction at all,
// which is bit-identical to the reference's own shader text executed by oracle/glsl_cpu.  exp() is the det_exp() polynomial,
// evaluated here for both pixels side by side.
// Depth compositing (DEPTH = true, gsr_set_depth_compositing): the staged chunk also carries each splat's view depth
// d = -view[2] (the projection's expression on the record's position), a pixel STOPS at the first splat with !(d < Z) for its
// scene depth Z (nothing after it contributes, as if the pixel had died), the depth is accumulated like a fourth colour channel,
// and the outputs are premultiplied rgb, alpha = 1 - t and depth = D / (1 - t) (+inf where nothing was blended).  DEPTH = false
// is the reference's frame and compiles to the same code as before the mode existed.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace gsr {

namespace {

constexpr int CHUNK = 256;    // gsplat_render.glsl:9 WORKGROUP_SIZE: splats per staged chunk / pixels per tile
constexpr int THREADS = 128;  // 2 pixels per thread
constexpr float MIN_ALPHA = 1.0f / 255.0f;

// The two pixels of a thread.  __f*_rn are never contracted (nvcc, and -ffp-contract=off in tests/kernel_emu).
struct F2 { float lo, hi; };
__device__ __forceinline__ F2 pk(float lo, float hi) { F2 r; r.lo = lo; r.hi = hi; return r; }
__device__ __forceinline__ void upk(F2 v, float &lo, float &hi) { lo = v.lo; hi = v.hi; }
__device__ __forceinline__ F2 fma2(F2 a, F2 b, F2 c) { return pk(__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)); }
__device__ __forceinline__ F2 mul2(F2 a, F2 b) { return pk(__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)); }
__device__ __forceinline__ F2 add2(F2 a, F2 b) { return pk(__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)); }
__device__ __forceinline__ F2 sub2(F2 a, F2 b) { return pk(__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)); }
// a*b + c with TWO roundings per lane, for the uncontracted evaluation
__device__ __forceinline__ F2 mul_add2_unfused(F2 a, F2 b, F2 c) { return add2(mul2(a, b), c); }
__device__ __forceinline__ F2 bc(float x) { return pk(x, x); }

struct Staged {  // one gathered record, pre-scaled for the inner loop
    float4 a;    // image_pos.x, image_pos.y, -0.5*conic.x, -0.5*conic.z
    float4 b;    // -conic.y, opacity, color.r, color.g
    float c;     // color.b
    float d;     // DEPTH only: view depth -(((V2*x + V6*y) + V10*z) + V14) of the record's position
};

__device__ __forceinline__ Staged null_splat() {
    Staged s;
    s.a = make_float4(0.f, 0.f, 0.f, 0.f);
    s.b = make_float4(0.f, 0.f, 0.f, 0.f);
    s.c = 0.f;
    s.d = 0.f;   // padding of the last chunk: alpha 0, and a stop it may cause is never seen (the tile ends with that chunk)
    return s;
}

// vz = (V[2], V[6], V[10], V[14]): the view-matrix row of the depth (DEPTH only)
template <bool DEPTH>
__device__ __forceinline__ Staged gather(const float4 *__restrict__ records, const uint32_t *__restrict__ values, uint32_t idx, float4 vz) {
    const uint32_t v = __ldg(values + idx);
    const float4 *r = records + (uint64_t)v * 3u;
    const float4 r0 = __ldg(r + 0), r1 = __ldg(r + 1), r2 = __ldg(r + 2);
    Staged s;
    s.a = make_float4(r0.x, r0.y, -0.5f * r1.x, -0.5f * r1.z);
    s.b = make_float4(-r1.y, r2.w, r2.x, r2.y);
    s.c = r2.z;
    s.d = DEPTH ? -(((vz.x * r0.z + vz.y * r0.w) + vz.z * r1.w) + vz.w * 1.0f) : 0.f;   // == -view[2] of the projection
    return s;
}

#ifndef GSR_COMP_GROUP
#define GSR_COMP_GROUP 4  // splats per software-pipelined group of the blend loop
#endif
constexpr int GU = GSR_COMP_GROUP;
static_assert(CHUNK % GU == 0, "a chunk is a whole number of groups");

#ifndef GSR_CPU_EMU
__device__ __forceinline__ unsigned long long globaltimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint32_t smid() { uint32_t r; asm volatile("mov.u32 %0, %smid;" : "=r"(r)); return r; }
#else
inline unsigned long long globaltimer_ns() { return 0ull; }
inline uint32_t smid() { return 0u; }
#endif

struct BlendK {  // broadcast constants of det_exp() for the two pixels
    F2 L2E2, MAGIC2, ONE2, C6, C5, C4, C3, C2, C1;
};
__device__ __forceinline__ BlendK make_blend_k() {
    BlendK k;
    k.L2E2 = bc(0x1.715476p+0f); k.MAGIC2 = bc(12582912.0f); k.ONE2 = bc(1.0f);
    k.C6 = bc(0x1.446c7ep-13f); k.C5 = bc(0x1.5f48c8p-10f); k.C4 = bc(0x1.3b29d8p-7f); k.C3 = bc(0x1.c6aeccp-5f);
    k.C2 = bc(0x1.ebfbe0p-3f); k.C1 = bc(0x1.62e430p-1f);
    return k;
}

// ---- phase A: alpha = opacity * exp(power) and 1 - alpha of GU splats (their (a, b) words already in registers) for this thread's
//      two pixels, written stage by stage so that the GU dependency chains can be interleaved.  No dependence on the transmittance:
//      this part of gsplat_render.glsl:84-88 runs ahead of the sequential blend.
template <bool CONTRACT>
__device__ __forceinline__ void phase_a(const float4 A[GU], const float4 B[GU], F2 npx2, float fpy, const BlendK &K, F2 al2[GU], F2 om2[GU]) {
    float oy[GU];
    F2 ox2[GU], pw2[GU], tm2[GU], e2[GU];
#pragma unroll
    for (int u = 0; u < GU; ++u) { ox2[u] = add2(bc(A[u].x), npx2); oy[u] = A[u].y - fpy; }
    // power = -0.5*(cx*ox*ox + cz*oy*oy) - cy*ox*oy (:84) on the pre-scaled conic:
    //   CONTRACT:  fma(e, oy, fma((-0.5cz)*oy, oy, ((-0.5cx)*ox)*ox))  with e = (-cy)*ox      (q and power contractions of the gsr spec)
    //   otherwise: (((-0.5cx)*ox)*ox + ((-0.5cz)*oy)*oy) + ((-cy)*ox)*oy                       (one rounding per GLSL operator)
#pragma unroll
    for (int u = 0; u < GU; ++u) pw2[u] = mul2(bc(A[u].z), ox2[u]);
#pragma unroll
    for (int u = 0; u < GU; ++u) {
        const float czoy = A[u].w * oy[u];
        if (CONTRACT) pw2[u] = fma2(bc(czoy), bc(oy[u]), mul2(pw2[u], ox2[u]));
        else pw2[u] = mul_add2_unfused(pw2[u], ox2[u], bc(__fmul_rn(czoy, oy[u])));   // (the second product must not fuse with the sum either)
    }
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = mul2(bc(B[u].x), ox2[u]);
#pragma unroll
    for (int u = 0; u < GU; ++u) pw2[u] = CONTRACT ? fma2(e2[u], bc(oy[u]), pw2[u]) : mul_add2_unfused(e2[u], bc(oy[u]), pw2[u]);
    // exp(power): det_exp() of both pixels
#pragma unroll
    for (int u = 0; u < GU; ++u) pw2[u] = mul2(pw2[u], K.L2E2);
#pragma unroll
    for (int u = 0; u < GU; ++u) {
        float tl, th;
        upk(pw2[u], tl, th);
        tl = g_min(g_max(tl, -127.0f), 128.0f);
        th = g_min(g_max(th, -127.0f), 128.0f);
        pw2[u] = pk(tl, th);
    }
#pragma unroll
    for (int u = 0; u < GU; ++u) tm2[u] = add2(pw2[u], K.MAGIC2);
#pragma unroll
    for (int u = 0; u < GU; ++u) al2[u] = sub2(tm2[u], K.MAGIC2);
#pragma unroll
    for (int u = 0; u < GU; ++u) pw2[u] = sub2(pw2[u], al2[u]);  // f
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(K.C6, pw2[u], K.C5);
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(e2[u], pw2[u], K.C4);
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(e2[u], pw2[u], K.C3);
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(e2[u], pw2[u], K.C2);
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(e2[u], pw2[u], K.C1);
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = fma2(e2[u], pw2[u], K.ONE2);
#pragma unroll
    for (int u = 0; u < GU; ++u) {
        float ml, mh;
        upk(tm2[u], ml, mh);
        tm2[u] = pk(__uint_as_float((__float_as_uint(ml) << 23) + 0x3F800000u), __uint_as_float((__float_as_uint(mh) << 23) + 0x3F800000u));
    }
#pragma unroll
    for (int u = 0; u < GU; ++u) e2[u] = mul2(e2[u], tm2[u]);
#pragma unroll
    for (int u = 0; u < GU; ++u) al2[u] = mul2(bc(B[u].y), e2[u]);
#pragma unroll
    for (int u = 0; u < GU; ++u) om2[u] = sub2(K.ONE2, al2[u]);
}

// ---- phase B: the sequential part (gsplat_render.glsl:89-90).  A dead pixel has left the reference's loop: its colour and
//      transmittance are kept by select.  `alive_mid` = "a pixel of this thread was alive after the first half of the group".
//      DEPTH: o0/o1 = "not stopped by the scene depth" (z0/z1); a live pixel stops at the first splat with !(d < z), before blending
//      it; a stopped pixel is dead from then on.  dd2 accumulates d * alpha * t exactly like a colour channel.
template <bool CONTRACT, bool DEPTH>
__device__ __forceinline__ void phase_b(const float4 B[GU], const float *s_c, const float *s_d, int j, const F2 al2[GU], const F2 om2[GU], F2 &cr2,
                                        F2 &cg2, F2 &cb2, float &t0, float &t1, bool &alive_mid, float z0, float z1, bool &o0, bool &o1, F2 &dd2) {
#pragma unroll
    for (int u = 0; u < GU; ++u) {
        const float cbl = s_c[j + u];
        float dj = 0.f;
        bool a0, a1;
        if constexpr (DEPTH) {
            dj = s_d[j + u];
            if (u == GU / 2) alive_mid = (t0 > MIN_ALPHA && o0) || (t1 > MIN_ALPHA && o1);
            a0 = t0 > MIN_ALPHA && o0; a1 = t1 > MIN_ALPHA && o1;
            const bool v0 = dj < z0, v1 = dj < z1;   // false for NaN: stops
            o0 = a0 ? v0 : o0; o1 = a1 ? v1 : o1;
            a0 = a0 && v0; a1 = a1 && v1;
        } else {
            if (u == GU / 2) alive_mid = (t0 > MIN_ALPHA) || (t1 > MIN_ALPHA);
            a0 = t0 > MIN_ALPHA; a1 = t1 > MIN_ALPHA;
        }
        float al, ah, pl, ph;
        upk(al2[u], al, ah);
        const F2 t2 = pk(t0, t1);
        upk(mul2(t2, om2[u]), pl, ph);
        const F2 m2 = pk(a0 ? al : 0.0f, a1 ? ah : 0.0f);   // alpha = 0: an exact no-op on the colour
        if (CONTRACT) {
            cr2 = fma2(mul2(bc(B[u].z), m2), t2, cr2);
            cg2 = fma2(mul2(bc(B[u].w), m2), t2, cg2);
            cb2 = fma2(mul2(bc(cbl), m2), t2, cb2);
            if constexpr (DEPTH) dd2 = fma2(mul2(bc(dj), m2), t2, dd2);
        } else {
            cr2 = mul_add2_unfused(mul2(bc(B[u].z), m2), t2, cr2);
            cg2 = mul_add2_unfused(mul2(bc(B[u].w), m2), t2, cg2);
            cb2 = mul_add2_unfused(mul2(bc(cbl), m2), t2, cb2);
            if constexpr (DEPTH) dd2 = mul_add2_unfused(mul2(bc(dj), m2), t2, dd2);
        }
        t0 = a0 ? pl : t0;
        t1 = a1 ? ph : t1;
    }
}

#ifndef GSR_COMP_MIN_BLOCKS
#define GSR_COMP_MIN_BLOCKS 3  // resident CTAs per SM the register allocation targets
#endif

// Persistent CTAs.  Ticket k of the launch renders owned tile order[k] (longest chains first) or k itself; every tile is blended
// from its first chunk to its stop by the CTA that took it.
template <bool CONTRACT, bool DEPTH = false>
__global__ void __launch_bounds__(THREADS, GSR_COMP_MIN_BLOCKS) composite_kernel(const __grid_constant__ CompositeArgs p) {
    __shared__ float4 s_a[CHUNK];
    __shared__ float4 s_b[CHUNK];
    __shared__ float s_c[CHUNK];
    __shared__ float s_d[DEPTH ? CHUNK : 1];   // view depth of the staged splats
    __shared__ uint32_t s_vote[THREADS / 32];
    __shared__ uint32_t s_tile;

    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    {   // sparse frame: only the first `comp_cta_limit` CTAs (one per SM: the block scheduler deals a fresh grid breadth-first) work
        const uint32_t limit = p.frame->comp_cta_limit;
        if (limit && blockIdx.x >= limit) return;
    }
    const BlendK K = make_blend_k();
    const float4 vz = DEPTH ? make_float4(p.view_z[0], p.view_z[1], p.view_z[2], p.view_z[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
    uint32_t staged = 0;  // SURVEY 8 symbol C, summed over the tiles this CTA processed (uniform across the CTA)
    unsigned long long t_start = 0;  // trace only

    for (;;) {
        if (tid == 0) {
            const uint32_t ticket = atomicAdd(&p.frame->comp_head, 1u);
            s_tile = ticket < (uint32_t)p.num_tiles ? (p.order ? p.order[ticket] : ticket) : 0xFFFFFFFFu;
            if (p.trace) t_start = globaltimer_ns();
        }
        __syncthreads();
        const uint32_t local_tile = s_tile;   // index among the owned tiles
        if (local_tile == 0xFFFFFFFFu) break;
        // owned tiles: rows tile_begin/tiles_x + k*row_step, all columns (row_step == 1: one contiguous band)
        const uint32_t tile_id = (uint32_t)p.tile_begin + (local_tile / (uint32_t)p.tiles_x) * (uint32_t)(p.row_step * p.tiles_x) + local_tile % (uint32_t)p.tiles_x;

        const uint32_t tx = tile_id % (uint32_t)p.tiles_x, ty = tile_id / (uint32_t)p.tiles_x;
        const int px0 = (int)(tx * TILE + 2u * (tid & 7u)), py = (int)(ty * TILE + (tid >> 3));
        const F2 npx2 = pk(-(float)px0, -(float)(px0 + 1));  // ox = image_pos.x - pixel.x  ==  image_pos.x + (-pixel.x)
        const float fpy = (float)py;

        const uint2 bounds = p.bounds[tile_id];
        const int32_t diff = (int32_t)(bounds.y - bounds.x);
        const int num_splats = diff > 0 ? diff : 0;                              // :61
        const int num_iterations = (int)ceilf((float)num_splats / (float)CHUNK);  // :62

        F2 cr2 = pk(0.f, 0.f), cg2 = cr2, cb2 = cr2;  // blended colour of the two pixels
        float t0 = 1.0f, t1 = 1.0f;                    // transmittance of the two pixels
        bool o0 = true, o1 = true;                     // DEPTH: not stopped by the scene depth
        F2 dd2 = pk(0.f, 0.f);                         // DEPTH: accumulated depth
        float z0 = __uint_as_float(0x7f800000u), z1 = z0; // DEPTH: scene depth (+inf: nothing occludes; also outside the image)
        if (DEPTH && p.scene_depth && py < p.height) {
            const float *zrow = p.scene_depth + (uint64_t)py * (uint64_t)p.width;
            if (px0 < p.width) z0 = zrow[px0];
            if (px0 + 1 < p.width) z1 = zrow[px0 + 1];
        }

        Staged n0 = null_splat(), n1 = null_splat();
        if (num_iterations > 0) {
            if ((int)tid < num_splats) n0 = gather<DEPTH>(p.records, p.values, bounds.x + tid, vz);
            if ((int)tid + THREADS < num_splats) n1 = gather<DEPTH>(p.records, p.values, bounds.x + tid + THREADS, vz);
        }

        int consumed = 0;  // chunks blended before the stop rule fired (next frame's scheduling hint)
        for (int i = 0; i < num_iterations; ++i) {
            const int sort_offset = CHUNK * i;
            const int chunk = (num_splats - sort_offset) < CHUNK ? (num_splats - sort_offset) : CHUNK;
            staged += (uint32_t)chunk;
            consumed = i + 1;
            s_a[tid] = n0.a; s_b[tid] = n0.b; s_c[tid] = n0.c;
            s_a[tid + THREADS] = n1.a; s_b[tid + THREADS] = n1.b; s_c[tid + THREADS] = n1.c;
            if constexpr (DEPTH) { s_d[tid] = n0.d; s_d[tid + THREADS] = n1.d; }
            __syncthreads();
            // prefetch the next chunk's records while this one is blended (slots past the list end become null splats)
            n0 = null_splat(); n1 = null_splat();
            if (i + 1 < num_iterations) {
                const int nb = sort_offset + CHUNK;
                if (nb + (int)tid < num_splats) n0 = gather<DEPTH>(p.records, p.values, bounds.x + (uint32_t)nb + tid, vz);
                if (nb + (int)tid + THREADS < num_splats) n1 = gather<DEPTH>(p.records, p.values, bounds.x + (uint32_t)nb + tid + THREADS, vz);
            }

            // :79-91, GU splats per iteration; `chunk` rounded up to GU reads null splats (opacity 0 => exact no-op).  Software-pipelined:
            // the (a, b) words of group g+1 are loaded while group g is blended, and the warp's "anybody alive?" test uses the
            // transmittance after the first half of the group -- a dead warp may blend one more (fully masked) group before it leaves.
            const int chunkg = (chunk + GU - 1) & ~(GU - 1);
            float4 A[GU], B[GU];
#pragma unroll
            for (int u = 0; u < GU; ++u) { A[u] = s_a[u]; B[u] = s_b[u]; }
            bool go;
            if constexpr (DEPTH) go = __any_sync(0xffffffffu, (t0 > MIN_ALPHA && o0) || (t1 > MIN_ALPHA && o1));
            else go = __any_sync(0xffffffffu, (t0 > MIN_ALPHA) || (t1 > MIN_ALPHA));
            for (int j = 0; j < chunkg && go; j += GU) {
                F2 al2[GU], om2[GU];
                phase_a<CONTRACT>(A, B, npx2, fpy, K, al2, om2);
                float4 Bc[GU];
#pragma unroll
                for (int u = 0; u < GU; ++u) Bc[u] = B[u];
                const int jn = (j + GU < CHUNK) ? j + GU : j;   // the last group re-reads itself instead of running off the array
#pragma unroll
                for (int u = 0; u < GU; ++u) { A[u] = s_a[jn + u]; B[u] = s_b[jn + u]; }
                bool alive_mid = true;
                phase_b<CONTRACT, DEPTH>(Bc, s_c, s_d, j, al2, om2, cr2, cg2, cb2, t0, t1, alive_mid, z0, z1, o0, o1, dd2);
                go = __any_sync(0xffffffffu, alive_mid);
            }

            // :97 tile-stop vote: continue only if the sum over the tile's 256 pixels of uint(t*255) exceeds 255 (a stopped pixel adds 0)
            uint32_t wsum;
            if constexpr (DEPTH) wsum = __reduce_add_sync(0xffffffffu, (o0 ? (uint32_t)(t0 * 255.0f) : 0u) + (o1 ? (uint32_t)(t1 * 255.0f) : 0u));
            else wsum = __reduce_add_sync(0xffffffffu, (uint32_t)(t0 * 255.0f) + (uint32_t)(t1 * 255.0f));
            if (lane == 0) s_vote[warp] = wsum;
            __syncthreads();
            uint32_t shared_t = 0;
#pragma unroll
            for (int w = 0; w < THREADS / 32; ++w) shared_t += s_vote[w];
            if (!(shared_t > 255u)) break;
        }

        // :100-101
        float r0, r1, g0, g1, b0, b1;
        upk(cr2, r0, r1); upk(cg2, g0, g1); upk(cb2, b0, b1);
        const float hx = (float)num_splats * 5e-4f;
        const float h0 = 0.0f * (1.0f - hx) + 1.0f * hx, h1 = 0.0f * (1.0f - hx) + 0.2f * hx, h2c = 1.0f * (1.0f - hx) + 0.2f * hx;
        if (py < p.height) {
            float4 *row = p.out + (uint64_t)py * (uint64_t)p.width;
            const float k0 = 1.0f - t0, k1 = 1.0f - t1;
            const float al0 = DEPTH ? k0 : 1.0f, al1 = DEPTH ? k1 : 1.0f;   // DEPTH: coverage; colour is premultiplied by construction
            if (px0 < p.width)
                row[px0] = make_float4(r0 + h0 * k0 * p.heatmap_factor, g0 + h1 * k0 * p.heatmap_factor, b0 + h2c * k0 * p.heatmap_factor, al0);
            if (px0 + 1 < p.width)
                row[px0 + 1] = make_float4(r1 + h0 * k1 * p.heatmap_factor, g1 + h1 * k1 * p.heatmap_factor, b1 + h2c * k1 * p.heatmap_factor, al1);
            if (DEPTH) {
                float d0, d1;
                upk(dd2, d0, d1);
                const float inf = __uint_as_float(0x7f800000u);
                float *drow = p.depth_out + (uint64_t)py * (uint64_t)p.width;
                if (px0 < p.width) drow[px0] = k0 > 0.0f ? __fdiv_rn(d0, k0) : inf;
                if (px0 + 1 < p.width) drow[px0 + 1] = k1 > 0.0f ? __fdiv_rn(d1, k1) : inf;
            }
        }
        // :105-110 pick: the elected (first) lane of each 32-wide subgroup of the reference's 16x16 workgroup is local
        // index 32*s = pixel (0, 2*s) of the tile = first pixel of thread 16*s here
        if ((tid & 15u) == 0u && tile_id == p.target_tile_id && t0 != 1.0f) {
            const uint32_t v = p.values[bounds.x + (bounds.y - bounds.x) / 10u];
            const float4 q0 = p.records[(uint64_t)v * 3u + 0], q1 = p.records[(uint64_t)v * 3u + 1];
            *p.pick = make_float4(q0.z, q0.w, q1.w, (float)num_splats);
        }
        if (tid == 0) {
            if (p.consumed) p.consumed[local_tile] = (uint32_t)consumed | 0x80000000u;   // bit 31: written this frame
            if (p.trace) {
                const uint32_t k = atomicAdd(p.trace_count, 1u);
                if (k < p.trace_cap) p.trace[k] = make_ulonglong4(((unsigned long long)tile_id << 32) | smid(), t_start, globaltimer_ns(),
                                                                  ((unsigned long long)(uint32_t)consumed << 32) | 1u | ((uint32_t)num_iterations << 1));
            }
        }
        __syncthreads();  // s_tile / staging buffers are reused by the next tile
    }
    if (tid == 0 && staged && p.count_staged) atomicAdd(&p.frame->staged, (unsigned long long)staged);
}

}  // namespace

#ifndef GSR_CPU_EMU
int preload_composite_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, composite_kernel<true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, composite_kernel<false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, composite_kernel<true, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, composite_kernel<false, true>));
    return GSR_OK;
}

int composite_max_ctas_per_sm(int *out) {
    int a = 0, b = 0, c = 0, d = 0;
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, composite_kernel<true>, THREADS, 0));
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, composite_kernel<false>, THREADS, 0));
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, composite_kernel<true, true>, THREADS, 0));
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d, composite_kernel<false, true>, THREADS, 0));
    if (c < a) a = c;
    if (d < b) b = d;
    *out = a < b ? a : b;
    if (*out < 1) *out = 1;
    return GSR_OK;
}

int launch_composite(const CompositeArgs &a, cudaStream_t stream) {
    if (a.num_tiles <= 0) return GSR_OK;
    const int per_sm = a.ctas_per_sm > 0 ? a.ctas_per_sm : 1;
    const int grid = a.num_tiles < a.sm_count * per_sm ? a.num_tiles : a.sm_count * per_sm;
    if (a.depth_out) {   // depth compositing (gsr_set_depth_compositing)
        if (a.contract) composite_kernel<true, true><<<grid, THREADS, 0, stream>>>(a);
        else composite_kernel<false, true><<<grid, THREADS, 0, stream>>>(a);
    } else if (a.contract) {
        composite_kernel<true><<<grid, THREADS, 0, stream>>>(a);
    } else {
        composite_kernel<false><<<grid, THREADS, 0, stream>>>(a);
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
