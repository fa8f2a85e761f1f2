// neighbors.cu -- splat neighbourhood selection (gsr_select_neighborhood; include/gsr.h "Splat neighbourhood selection"; DESIGN.md
// section 5.22).
//
// A spatial hash grid over the participants, built and queried on the GPU in one call:
//   1. neighbor_keys_kernel: one pass over the tested range appends (key, slot) for every participant (a warp-aggregated device counter);
//   2. the pairs are sorted by key with the library's Onesweep sort (the count stays on the device);
//   3. neighbor_grid_kernel gathers the sorted positions as float4 (x, y, z, slot bits) and finds the bucket starts, as ranges.cu finds
//      the tile ranges; neighbor_impure_kernel marks the buckets that hold more than one cell;
//   4. neighbor_budget_kernel sums, over the participants, the occupancy of their 27 cells (the work measure the host checks);
//   5. SPARSE / GROW: neighbor_query_kernel scans the 27 cells of a participant and sets its bit in a scratch mask; CONNECTED /
//      SMALL_CLUSTERS: neighbor_union_kernel joins the two ends of every edge in a lock-free union-find (ECL-CC hooking: the larger root
//      is pointed at the smaller with atomicCAS), neighbor_compress_kernel points every participant at its root and counts the clusters'
//      sizes and seeds on the root;
//   6. neighbor_combine_kernel has the shape of select_region_kernel: a warp per mask word, a ballot, lane 0 combines -- and counts.
// Only plane 0 is read.  Positions are float32 with one rounding per operation (-fmad=false); cells are float64.  Every entry of a cell is
// found by its cell, never by its key alone, so hash collisions cost time, not correctness.
#include "common.cuh"

namespace gsr {

namespace {

constexpr int NB_THREADS = 256;
constexpr int NB_WARPS = NB_THREADS / 32;

struct Cell { long long x, y, z; };

// floor(v / h) in float64, clamped to [-2^62, 2^62]
__device__ __forceinline__ long long nb_axis(float v, double h) {
    const double q = floor((double)v / h);
    return (long long)(q < -0x1p62 ? -0x1p62 : (q > 0x1p62 ? 0x1p62 : q));
}
__device__ __forceinline__ Cell nb_cell(const float4 &p, double h) { return Cell{nb_axis(p.x, h), nb_axis(p.y, h), nb_axis(p.z, h)}; }
__device__ __forceinline__ bool nb_same(const Cell &a, const Cell &b) { return a.x == b.x && a.y == b.y && a.z == b.z; }

// The cell's 32-bit key: a linear form of the coordinates (mod 2^64), then a 64-bit finaliser.  The top p bits are the bucket.
__device__ __forceinline__ uint32_t nb_key(const Cell &c) {
    unsigned long long h = (unsigned long long)c.x * 0x9E3779B97F4A7C15ull + (unsigned long long)c.y * 0xC2B2AE3D27D4EB4Full +
                           (unsigned long long)c.z * 0x165667B19E3779F9ull;
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    return (uint32_t)h;
}

__device__ __forceinline__ bool nb_finite(const float4 &p) {
    return fabsf(p.x) <= 3.402823466e38f && fabsf(p.y) <= 3.402823466e38f && fabsf(p.z) <= 3.402823466e38f;
}

// j = q is a neighbour of i = p: d2 = ((dx dx) + (dy dy)) + (dz dz) <= r2, dx = x_j - x_i
__device__ __forceinline__ bool nb_near(const float4 &p, const float4 &q, float r2) {
    const float dx = __fsub_rn(q.x, p.x), dy = __fsub_rn(q.y, p.y), dz = __fsub_rn(q.z, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) <= r2;
}

__device__ __forceinline__ uint32_t nb_slot(const float4 &q) { return __float_as_uint(q.w); }

// Calls f(q) for every sorted entry q of the 27 cells around c until f returns true (then returns true).  A pure bucket is one cell: one
// cell test for all its entries.  In an impure one, only the entries of the cell's key are tested, each by its own cell.
template <class F>
__device__ __forceinline__ bool nb_visit(const NeighborArgs &a, const Cell &c, F &&f) {
#pragma unroll 1
    for (int o = 0; o < 27; ++o) {
        const Cell d{c.x + (o % 3 - 1), c.y + ((o / 3) % 3 - 1), c.z + (o / 9 - 1)};
        const uint32_t k = nb_key(d), b = k >> a.shift;
        const uint32_t s0 = a.start[b], st = s0 & ~NB_IMPURE, en = a.start[b + 1] & ~NB_IMPURE;
        if (st == en) continue;
        if (!(s0 & NB_IMPURE)) {
            if (!nb_same(nb_cell(a.pos[st], a.h), d)) continue;
#pragma unroll 1
            for (uint32_t e = st; e < en; ++e) if (f(a.pos[e])) return true;
        } else {
#pragma unroll 1
            for (uint32_t e = st; e < en; ++e) {
                if (a.keys[e] != k) continue;
                const float4 q = a.pos[e];
                if (nb_same(nb_cell(q, a.h), d) && f(q)) return true;
            }
        }
    }
    return false;
}

// The participants of cell d (the budget: no position is compared)
__device__ __forceinline__ uint32_t nb_occupancy(const NeighborArgs &a, const Cell &d) {
    const uint32_t k = nb_key(d), b = k >> a.shift;
    const uint32_t s0 = a.start[b], st = s0 & ~NB_IMPURE, en = a.start[b + 1] & ~NB_IMPURE;
    if (st == en) return 0u;
    if (!(s0 & NB_IMPURE)) return nb_same(nb_cell(a.pos[st], a.h), d) ? en - st : 0u;
    uint32_t n = 0u;
#pragma unroll 1
    for (uint32_t e = st; e < en; ++e) n += (a.keys[e] == k && nb_same(nb_cell(a.pos[e], a.h), d)) ? 1u : 0u;
    return n;
}

// ---- union-find over slots: parent[x] <= x always (a root is hooked under a smaller one only), so a root is the least slot of its tree.
// Reads are volatile (another CTA's hook must be seen); the path-halving stores only shorten a path to an ancestor and never touch a root,
// the only words an atomicCAS targets.
__device__ __forceinline__ uint32_t nb_load(const uint32_t *p) { return *(const volatile uint32_t *)p; }

__device__ __forceinline__ uint32_t nb_find(uint32_t *parent, uint32_t x) {
    uint32_t cur = nb_load(parent + x);
    if (cur != x) {
        uint32_t prev = x, next;
#pragma unroll 1
        while (cur > (next = nb_load(parent + cur))) {
            *(volatile uint32_t *)(parent + prev) = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

// The root of x without path halving: once roots are final, a halving store could put a non-root ancestor back into a word another
// thread has just compressed to the root
__device__ __forceinline__ uint32_t nb_root(const uint32_t *parent, uint32_t x) {
    uint32_t next;
#pragma unroll 1
    while ((next = nb_load(parent + x)) != x) x = next;
    return x;
}

// Joins the trees of x and y; returns a slot of the joined tree (its root when the call returned)
__device__ __forceinline__ uint32_t nb_hook(uint32_t *parent, uint32_t x, uint32_t y) {
#pragma unroll 1
    for (;;) {
        x = nb_find(parent, x);
        y = nb_find(parent, y);
        if (x == y) return x;
        const uint32_t lo = x < y ? x : y, hi = x < y ? y : x;
        if (atomicCAS(parent + hi, hi, lo) == hi) return lo;
    }
}

__device__ __forceinline__ uint32_t nb_entries(const NeighborArgs &a) { return *(const volatile uint32_t *)&a.ctr->n; }

// 1. (key, slot) of every participant of the tested range, appended through a warp-aggregated counter (the order within a key is free:
//    no result depends on it)
__global__ void __launch_bounds__(NB_THREADS) neighbor_keys_kernel(const __grid_constant__ NeighborArgs a) {
    const uint64_t i = (uint64_t)blockIdx.x * NB_THREADS + threadIdx.x;
    const uint64_t s = a.first + i;
    bool part = false;
    uint32_t key = 0u;
    if (i < a.count && !mask_bit(a.hidden, s)) {
        const float4 p = __ldg(a.plane0 + s);
        if (nb_finite(p)) {
            part = true;
            key = nb_key(nb_cell(p, a.h));
        }
    }
    const uint32_t lane = threadIdx.x & 31u, ballot = __ballot_sync(0xffffffffu, part);
    uint32_t base = 0u;
    if (lane == 0 && ballot) base = atomicAdd(&a.ctr->n, (uint32_t)__popc(ballot));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (part) {
        const uint32_t e = base + (uint32_t)__popc(ballot & ((1u << lane) - 1u));
        a.keys[e] = key;
        a.vals[e] = (uint32_t)s;
    }
}

// 3a. The sorted positions, every participant its own root, and the bucket starts: entry e writes start[b] = e for the buckets
//     (bucket(e - 1), bucket(e)], the last entry also start[b] = n for the buckets after its own
__global__ void __launch_bounds__(NB_THREADS) neighbor_grid_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    if (e >= n) return;
    const uint32_t s = a.vals[e];
    const float4 p = __ldg(a.plane0 + s);
    a.pos[e] = make_float4(p.x, p.y, p.z, __uint_as_float(s));
    a.parent[s] = s;
    const uint32_t b = a.keys[e] >> a.shift;
#pragma unroll 1
    for (uint32_t x = e ? (a.keys[e - 1] >> a.shift) + 1u : 0u; x <= b; ++x) a.start[x] = e;
    if (e == n - 1u) {
        const uint32_t buckets = 1u << (32u - a.shift);
#pragma unroll 1
        for (uint32_t x = b + 1u; x <= buckets; ++x) a.start[x] = n;
    }
}

// 3b. A bucket holding two neighbouring entries of different keys or cells is impure
__global__ void __launch_bounds__(NB_THREADS) neighbor_impure_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    if (e == 0u || e >= n) return;
    const uint32_t k = a.keys[e], kp = a.keys[e - 1];
    if ((k >> a.shift) != (kp >> a.shift)) return;
    if (k != kp || !nb_same(nb_cell(a.pos[e], a.h), nb_cell(a.pos[e - 1], a.h))) atomicOr(a.start + (k >> a.shift), NB_IMPURE);
}

// 4. candidates += the participants of the 27 cells of every participant (a warp sum, one 64-bit atomic per warp)
__global__ void __launch_bounds__(NB_THREADS) neighbor_budget_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    unsigned long long t = 0ull;
    if (e < n) {
        const Cell c = nb_cell(a.pos[e], a.h);
#pragma unroll 1
        for (int o = 0; o < 27; ++o) t += nb_occupancy(a, Cell{c.x + (o % 3 - 1), c.y + ((o / 3) % 3 - 1), c.z + (o / 9 - 1)});
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31u) == 0u && t) atomicAdd(&a.ctr->candidates, t);
}

// 5a. SPARSE: fewer than `threshold` neighbours (the scan stops at `threshold`); GROW: selected, or a selected neighbour (the scan stops
//     at the first).  Inside sets the participant's bit of the scratch mask.
template <int MODE>
__global__ void __launch_bounds__(NB_THREADS) neighbor_query_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    if (e >= n) return;
    const float4 p = a.pos[e];
    const uint32_t s = nb_slot(p);
    const Cell c = nb_cell(p, a.h);
    bool in;
    if constexpr (MODE == GSR_NEIGHBOR_GROW) {
        in = mask_bit(a.selected, s) ||
             nb_visit(a, c, [&](const float4 &q) { const uint32_t j = nb_slot(q); return j != s && nb_near(p, q, a.r2) && mask_bit(a.selected, j); });
    } else {
        uint32_t found = 0u;
        nb_visit(a, c, [&](const float4 &q) {
            if (nb_slot(q) == s || !nb_near(p, q, a.r2)) return false;
            return ++found >= a.threshold;
        });
        in = found < a.threshold;
    }
    if (in) atomicOr(a.inside + (s >> 5), 1u << (s & 31u));
}

// 5b. Every edge once, from its smaller slot: skipped without the distance test when the other end already hangs on our last known root
__global__ void __launch_bounds__(NB_THREADS) neighbor_union_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    if (e >= n) return;
    const float4 p = a.pos[e];
    const uint32_t s = nb_slot(p);
    uint32_t r = nb_find(a.parent, s);
    nb_visit(a, nb_cell(p, a.h), [&](const float4 &q) {
        const uint32_t j = nb_slot(q);
        if (j > s && nb_load(a.parent + j) != r && nb_near(p, q, a.r2)) r = nb_hook(a.parent, s, j);
        return false;
    });
}

// 5c. After every union: each participant points at its root; the root counts its cluster and marks a selected member (NB_SEED)
__global__ void __launch_bounds__(NB_THREADS) neighbor_compress_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t n = nb_entries(a);
    const uint32_t e = blockIdx.x * NB_THREADS + threadIdx.x;
    if (e >= n) return;
    const uint32_t s = nb_slot(a.pos[e]);
    const uint32_t r = nb_root(a.parent, s);   // every store of this kernel is a root into the thread's own slot
    a.parent[s] = r;
    atomicAdd(a.size + r, 1u);
    if (mask_bit(a.selected, s)) atomicOr(a.size + r, NB_SEED);
}

// 6. One warp per mask word over every word (SET clears outside the tested range): inside from the scratch mask (SPARSE / GROW, which is
//    zeroed again) or from the participant's root (CONNECTED / SMALL_CLUSTERS, which also count the roots and the largest cluster)
template <int MODE>
__global__ void __launch_bounds__(NB_THREADS) neighbor_combine_kernel(const __grid_constant__ NeighborArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t w = blockIdx.x * NB_WARPS + (threadIdx.x >> 5);
    if (w >= a.words) return;   // warp-uniform
    uint32_t inside;
    if constexpr (MODE == GSR_NEIGHBOR_SPARSE || MODE == GSR_NEIGHBOR_GROW) {
        inside = 0u;
        if (lane == 0) {
            inside = a.inside[w];
            if (inside) a.inside[w] = 0u;
        }
    } else {
        const uint64_t s = 32ull * w + lane;
        bool in = false, root = false;
        uint32_t size = 0u;
        if (s >= a.first && s - a.first < a.count) {
            const uint32_t r = a.parent[s];
            if (r != NB_NONE) {
                const uint32_t z = a.size[r];
                in = MODE == GSR_NEIGHBOR_CONNECTED ? (z & NB_SEED) != 0u : (z & ~NB_SEED) < a.threshold;
                root = r == (uint32_t)s;
                size = root ? z & ~NB_SEED : 0u;
            }
        }
        inside = __ballot_sync(0xffffffffu, in);
        const uint32_t roots = __ballot_sync(0xffffffffu, root);
        const int largest = __reduce_max_sync(0xffffffffu, (int)size);
        if (lane == 0 && roots) {
            atomicAdd(&a.ctr->clusters, (unsigned long long)__popc(roots));
            atomicMax(&a.ctr->largest, (unsigned long long)largest);
        }
    }
    if (lane == 0) {
        a.selected[w] = combine_op(a.op, a.selected[w], inside) & ~a.hidden[w];
        if (inside) atomicAdd(&a.ctr->inside, (unsigned long long)__popc(inside));
    }
}

}  // namespace

double neighbor_cell_size(float radius) { return (double)radius * (1.0 + 0x1p-20); }

uint32_t neighbor_bucket_bits(uint64_t count) {
    uint32_t p = 1u;
    while ((1ull << p) < 2ull * count) ++p;
    return p;
}

#ifndef GSR_CPU_EMU  // host side: CUDA only (tests/neighbor_reference drives the kernels above itself)

namespace {
uint32_t nb_blocks(uint64_t items) { return (uint32_t)((items + NB_THREADS - 1) / NB_THREADS); }
}  // namespace

int launch_neighbor_keys(const NeighborArgs &a, cudaStream_t stream) {
    if (a.count == 0) return GSR_OK;
    neighbor_keys_kernel<<<nb_blocks(a.count), NB_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_neighbor_grid(const NeighborArgs &a, uint64_t max_splats, cudaStream_t stream) {
    if (a.count == 0) return GSR_OK;
    GSR_CUDA_TRY(cudaMemsetAsync(a.parent, 0xFF, sizeof(uint32_t) * max_splats, stream));   // NB_NONE: not a participant
    GSR_CUDA_TRY(cudaMemsetAsync(a.size, 0, sizeof(uint32_t) * max_splats, stream));
    neighbor_grid_kernel<<<nb_blocks(a.count), NB_THREADS, 0, stream>>>(a);
    neighbor_impure_kernel<<<nb_blocks(a.count), NB_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_neighbor_budget(const NeighborArgs &a, cudaStream_t stream) {
    if (a.count == 0) return GSR_OK;
    neighbor_budget_kernel<<<nb_blocks(a.count), NB_THREADS, 0, stream>>>(a);
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

int launch_neighbor_select(const NeighborArgs &a, cudaStream_t stream) {
    const uint32_t eb = nb_blocks(a.count), wb = (a.words + NB_WARPS - 1) / NB_WARPS;
    switch (a.mode) {
        case GSR_NEIGHBOR_SPARSE:
            if (eb) neighbor_query_kernel<GSR_NEIGHBOR_SPARSE><<<eb, NB_THREADS, 0, stream>>>(a);
            if (wb) neighbor_combine_kernel<GSR_NEIGHBOR_SPARSE><<<wb, NB_THREADS, 0, stream>>>(a);
            break;
        case GSR_NEIGHBOR_GROW:
            if (eb) neighbor_query_kernel<GSR_NEIGHBOR_GROW><<<eb, NB_THREADS, 0, stream>>>(a);
            if (wb) neighbor_combine_kernel<GSR_NEIGHBOR_GROW><<<wb, NB_THREADS, 0, stream>>>(a);
            break;
        case GSR_NEIGHBOR_CONNECTED:
        case GSR_NEIGHBOR_SMALL_CLUSTERS:
            if (eb) {
                neighbor_union_kernel<<<eb, NB_THREADS, 0, stream>>>(a);
                neighbor_compress_kernel<<<eb, NB_THREADS, 0, stream>>>(a);
            }
            if (wb) {
                if (a.mode == GSR_NEIGHBOR_CONNECTED) neighbor_combine_kernel<GSR_NEIGHBOR_CONNECTED><<<wb, NB_THREADS, 0, stream>>>(a);
                else neighbor_combine_kernel<GSR_NEIGHBOR_SMALL_CLUSTERS><<<wb, NB_THREADS, 0, stream>>>(a);
            }
            break;
        default: set_last_error("neighbour kernels: unknown mode %u", a.mode); return GSR_ERR_INVALID;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    return GSR_OK;
}

// Force-load this file's kernels (the lazy-loading rule of DESIGN.md section 6)
int preload_neighbor_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_keys_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_grid_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_impure_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_budget_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_query_kernel<GSR_NEIGHBOR_SPARSE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_query_kernel<GSR_NEIGHBOR_GROW>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_union_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_compress_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_combine_kernel<GSR_NEIGHBOR_SPARSE>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_combine_kernel<GSR_NEIGHBOR_GROW>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_combine_kernel<GSR_NEIGHBOR_CONNECTED>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, neighbor_combine_kernel<GSR_NEIGHBOR_SMALL_CLUSTERS>));
    return GSR_OK;
}
#endif  // GSR_CPU_EMU

}  // namespace gsr
