// radix_sort.cu -- Onesweep-style stable LSD radix sort of 32-bit keys (+32-bit values), 4 x 8-bit digits.
//
// Replaces radix_sort_upsweep.glsl / radix_sort_spine.glsl / radix_sort_downsweep.glsl x 4 passes
// (12 dispatches with full barriers, rasterizer.gd:143-149; 80 B/pair of traffic) by
//   1 histogram kernel  : reads the keys once, builds all four 256-bin digit histograms (4 B/key) and
//                         clears the look-back status words of the tiles that will be used;
//   4 onesweep kernels  : each reads the pairs once and writes them once (16 B/pair); the per-tile digit
//                         offsets come from a chained scan with decoupled look-back instead of the
//                         separate spine dispatch.  Total 68 B/pair (36 B/key keys-only).
// Semantics = the reference's: stable (ties keep input order), all 32 bits, ascending.
//
// The element count is read from device memory (*n_ptr): like the reference's indirect dispatch
// (rasterizer.gd:146) the host never learns M on the frame path.  Kernels are persistent: a fixed grid
// (a multiple of the SM count) pulls tiles from an atomic ticket, which also gives the look-back its
// forward-progress guarantee.
#include "common.cuh"

// Digit matching inside a warp: 8 ballots (1) or match.any (0).  Ballots cost the same for any digit skew; MATCH.ANY's cost
// grows with the number of distinct digits in the warp.
#ifndef GSR_SORT_BALLOT
#define GSR_SORT_BALLOT 1
#endif
#ifndef GSR_SORT_ATOMIC
#define GSR_SORT_ATOMIC 0  // 1: returning shared atomics, consumed in a second loop; 0: load/add/store per row
#endif

namespace gsr {

namespace {

constexpr int RADIX = 256;
constexpr uint32_t FLAG_AGG = 1u << 30;
constexpr uint32_t FLAG_PREFIX = 1u << 31;
constexpr uint32_t VAL_MASK = (1u << 30) - 1u;
constexpr int HIST_THREADS = 512;

// ------------------------------------------------------------------------------------------------
// histogram of all four digits + status clear
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(HIST_THREADS) sort_hist_kernel(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ n_ptr,
                                                                 uint32_t n_max, uint32_t *__restrict__ hist, uint32_t *__restrict__ status,
                                                                 uint32_t tile_keys, uint32_t max_tiles) {
    __shared__ uint32_t sh[4 * RADIX];
    const uint32_t tid = threadIdx.x;
    const uint32_t gtid = blockIdx.x * HIST_THREADS + tid;
    const uint32_t gsize = gridDim.x * HIST_THREADS;
    uint32_t n = *n_ptr;
    n = n < n_max ? n : n_max;
    for (uint32_t i = tid; i < 4 * RADIX; i += HIST_THREADS) sh[i] = 0;

    // clear the look-back words of the tiles the four passes will touch
    const uint32_t num_tiles = (n + tile_keys - 1) / tile_keys;
    const uint32_t words = num_tiles * RADIX;
    for (uint32_t i = gtid; i < words; i += gsize) {
#pragma unroll
        for (int p = 0; p < 4; ++p) status[(size_t)p * max_tiles * RADIX + i] = 0u;
    }
    __syncthreads();

    const uint32_t n4 = n >> 2;
    const uint4 *k4 = reinterpret_cast<const uint4 *>(keys);
    for (uint32_t i = gtid; i < n4; i += gsize) {
        const uint4 k = __ldg(k4 + i);
        const uint32_t kk[4] = {k.x, k.y, k.z, k.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            atomicAdd(&sh[0 * RADIX + (kk[j] & 255u)], 1u);
            atomicAdd(&sh[1 * RADIX + ((kk[j] >> 8) & 255u)], 1u);
            atomicAdd(&sh[2 * RADIX + ((kk[j] >> 16) & 255u)], 1u);
            atomicAdd(&sh[3 * RADIX + (kk[j] >> 24)], 1u);
        }
    }
    for (uint32_t i = (n4 << 2) + gtid; i < n; i += gsize) {
        const uint32_t k = keys[i];
        atomicAdd(&sh[0 * RADIX + (k & 255u)], 1u);
        atomicAdd(&sh[1 * RADIX + ((k >> 8) & 255u)], 1u);
        atomicAdd(&sh[2 * RADIX + ((k >> 16) & 255u)], 1u);
        atomicAdd(&sh[3 * RADIX + (k >> 24)], 1u);
    }
    __syncthreads();
    for (uint32_t i = tid; i < 4 * RADIX; i += HIST_THREADS) {
        const uint32_t v = sh[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

// ------------------------------------------------------------------------------------------------
// gsr_set_depth_order: histograms of the six passes of the (tile, depth word) sort + status clear.  Reads the keys and the depth
// words once: digits 0-3 of the depth word (the four wide passes) and digits 2-3 of the key (tile = key >> 16, the two narrow passes).
// The wide passes cut the pairs into tiles of `wide_tile` keys, the narrow ones into tiles of `narrow_tile`.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(HIST_THREADS) sort_hist_depth_kernel(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ depth,
                                                                       const uint32_t *__restrict__ n_ptr, uint32_t n_max, uint32_t *__restrict__ hist,
                                                                       uint32_t *__restrict__ status, uint32_t wide_tile, uint32_t narrow_tile,
                                                                       uint32_t max_tiles) {
    __shared__ uint32_t sh[6 * RADIX];
    const uint32_t tid = threadIdx.x;
    const uint32_t gtid = blockIdx.x * HIST_THREADS + tid;
    const uint32_t gsize = gridDim.x * HIST_THREADS;
    uint32_t n = *n_ptr;
    n = n < n_max ? n : n_max;
    for (uint32_t i = tid; i < 6 * RADIX; i += HIST_THREADS) sh[i] = 0;

    const uint32_t wide_words = (n + wide_tile - 1) / wide_tile * RADIX;
    const uint32_t narrow_words = (n + narrow_tile - 1) / narrow_tile * RADIX;
    for (uint32_t i = gtid; i < wide_words; i += gsize) {
#pragma unroll
        for (int p = 0; p < 4; ++p) status[(size_t)p * max_tiles * RADIX + i] = 0u;
        if (i < narrow_words) {
            status[(size_t)4 * max_tiles * RADIX + i] = 0u;
            status[(size_t)5 * max_tiles * RADIX + i] = 0u;
        }
    }
    __syncthreads();

    const uint32_t n4 = n >> 2;
    const uint4 *k4 = reinterpret_cast<const uint4 *>(keys);
    const uint4 *d4 = reinterpret_cast<const uint4 *>(depth);
    for (uint32_t i = gtid; i < n4; i += gsize) {
        const uint4 k = __ldg(k4 + i), d = __ldg(d4 + i);
        const uint32_t kk[4] = {k.x, k.y, k.z, k.w}, dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            atomicAdd(&sh[0 * RADIX + (dd[j] & 255u)], 1u);
            atomicAdd(&sh[1 * RADIX + ((dd[j] >> 8) & 255u)], 1u);
            atomicAdd(&sh[2 * RADIX + ((dd[j] >> 16) & 255u)], 1u);
            atomicAdd(&sh[3 * RADIX + (dd[j] >> 24)], 1u);
            atomicAdd(&sh[4 * RADIX + ((kk[j] >> 16) & 255u)], 1u);
            atomicAdd(&sh[5 * RADIX + (kk[j] >> 24)], 1u);
        }
    }
    for (uint32_t i = (n4 << 2) + gtid; i < n; i += gsize) {
        const uint32_t k = keys[i], d = depth[i];
        atomicAdd(&sh[0 * RADIX + (d & 255u)], 1u);
        atomicAdd(&sh[1 * RADIX + ((d >> 8) & 255u)], 1u);
        atomicAdd(&sh[2 * RADIX + ((d >> 16) & 255u)], 1u);
        atomicAdd(&sh[3 * RADIX + (d >> 24)], 1u);
        atomicAdd(&sh[4 * RADIX + ((k >> 16) & 255u)], 1u);
        atomicAdd(&sh[5 * RADIX + (k >> 24)], 1u);
    }
    __syncthreads();
    for (uint32_t i = tid; i < 6 * RADIX; i += HIST_THREADS) {
        const uint32_t v = sh[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

// ------------------------------------------------------------------------------------------------
// one onesweep pass
// WIDE (gsr_set_depth_order): the sorted word carries two payload words, vals_in / vals_out and vals2_in / vals2_out (PAIRS is then
// true too).  Every wide-only statement is an `if constexpr`: WIDE = false is the pass as it always was.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
    const uint32_t lane = lane_id();
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= (uint32_t)o) v += t;
    }
    return v;
}

template <int THREADS, int ITEMS, bool PAIRS, bool WIDE = false>
__global__ void __launch_bounds__(THREADS, 1024 / THREADS) onesweep_kernel(const uint32_t *__restrict__ keys_in, uint32_t *__restrict__ keys_out,
                                                           const uint32_t *__restrict__ vals_in, uint32_t *__restrict__ vals_out,
                                                           const uint32_t *__restrict__ n_ptr, uint32_t n_max,
                                                           const uint32_t *__restrict__ hist,  // [256], this pass
                                                           uint32_t *status,                   // [tiles][256], this pass
                                                           uint32_t *ticket, int shift,
                                                           const uint32_t *__restrict__ vals2_in = nullptr,  // WIDE: second payload
                                                           uint32_t *__restrict__ vals2_out = nullptr) {
    static_assert(THREADS >= RADIX && THREADS % 32 == 0, "need one thread per digit");
    static_assert(!WIDE || PAIRS, "a wide pass carries pairs");
    constexpr int WARPS = THREADS / 32;
    constexpr uint32_t TILE_KEYS = THREADS * ITEMS;
#ifndef GSR_CPU_EMU
    extern __shared__ uint32_t smem[];
#else  // tests/kernel_emu (CPU logic pre-flight): dynamic shared memory becomes a block-shared array of the same size
    __shared__ uint32_t smem[WARPS * RADIX + (WIDE ? 3 : 2) * TILE_KEYS];
#endif
    uint32_t *s_whist = smem;                    // [WARPS][256] warp-private digit counters
    uint32_t *s_keys = s_whist + WARPS * RADIX;  // [TILE_KEYS]
    uint32_t *s_vals = s_keys + TILE_KEYS;       // [TILE_KEYS] (PAIRS)
    __shared__ uint32_t s_gbase[RADIX];          // exclusive scan of the global histogram
    __shared__ uint32_t s_dstart[RADIX];         // first slot of each digit inside the sorted tile
    __shared__ uint32_t s_base[RADIX];           // global dst = s_base[d] + slot
    __shared__ uint32_t s_wtot[RADIX / 32];
    __shared__ uint32_t s_tile;

    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t n = *n_ptr;
    n = n < n_max ? n : n_max;
    const uint32_t num_tiles = (n + TILE_KEYS - 1) / TILE_KEYS;

    // exclusive prefix of this pass's global histogram (once per CTA)
    {
        uint32_t v = 0, incl = 0;
        if (tid < RADIX) {
            v = hist[tid];
            incl = warp_incl_scan(v);
            if (lane == 31) s_wtot[warp] = incl;
        }
        __syncthreads();
        if (tid < RADIX) {
            uint32_t off = 0;
            for (uint32_t w = 0; w < warp; ++w) off += s_wtot[w];
            s_gbase[tid] = off + incl - v;
        }
    }

    while (true) {
        __syncthreads();  // previous tile fully written; s_wtot free
        if (tid == 0) s_tile = atomicAdd(ticket, 1u);
        for (uint32_t i = tid; i < WARPS * RADIX; i += THREADS) s_whist[i] = 0u;
        __syncthreads();
        const uint32_t tile = s_tile;
        if (tile >= num_tiles) break;

        // ---- load: warp-striped (warp w owns a contiguous slab, row i = 32 consecutive keys) ----
        const uint32_t tile_base = tile * TILE_KEYS;
        const uint32_t my_base = tile_base + warp * (32u * ITEMS) + lane;
        const bool full = (tile_base + TILE_KEYS) <= n;
        uint32_t key[ITEMS], val[ITEMS], rank[ITEMS];
        uint32_t val2[WIDE ? ITEMS : 1];
        if (full) {
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) key[i] = keys_in[my_base + i * 32u];
            if (PAIRS) {
#pragma unroll
                for (int i = 0; i < ITEMS; ++i) val[i] = vals_in[my_base + i * 32u];
            }
            if constexpr (WIDE) {
#pragma unroll
                for (int i = 0; i < ITEMS; ++i) val2[i] = vals2_in[my_base + i * 32u];
            }
        } else {
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) {
                const uint32_t idx = my_base + i * 32u;
                key[i] = idx < n ? keys_in[idx] : 0xFFFFFFFFu;  // pad keys sort last (radix_sort_downsweep.glsl:87)
                if (PAIRS) val[i] = idx < n ? vals_in[idx] : 0u;
                if constexpr (WIDE) val2[i] = idx < n ? vals2_in[idx] : 0u;
            }
        }

        // ---- rank inside the warp: lanes with the same digit are matched, the lowest of them (the leader) bumps the
        //      warp-private counter.  The counter update is a RETURNING shared atomic whose result is not consumed
        //      in this loop, so the ITEMS match + ITEMS atomic operations of a thread pipeline instead of forming a
        //      load->add->store chain per row; __syncwarp() keeps row i's update ordered before row i+1's.
        uint32_t *wh = s_whist + warp * RADIX;
        const uint32_t lt_mask = (1u << lane) - 1u;
#if GSR_SORT_ATOMIC
        uint32_t old[ITEMS];  // counter value before this row (valid in the leader lane)
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const uint32_t d = (key[i] >> shift) & 255u;
#if GSR_SORT_BALLOT
            uint32_t mask = 0xffffffffu;  // 8 ballots -> lanes with the same digit (radix_sort_downsweep.glsl:95-102)
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                const bool bit = (d >> b) & 1u;
                const uint32_t bal = __ballot_sync(0xffffffffu, bit);
                mask &= bit ? bal : ~bal;
            }
#else
            const uint32_t mask = __match_any_sync(0xffffffffu, d);
#endif
            rank[i] = (uint32_t)__popc(mask & lt_mask) | ((uint32_t)(__ffs(mask) - 1) << 8);  // lower | leader << 8
            old[i] = 0u;
            if ((mask & lt_mask) == 0u) old[i] = atomicAdd(&wh[d], (uint32_t)__popc(mask));
            __syncwarp();
        }
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const uint32_t meta = rank[i];
            const uint32_t prev = __shfl_sync(0xffffffffu, old[i], (int)(meta >> 8));
            rank[i] = prev + (meta & 255u);
        }
#else
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const uint32_t d = (key[i] >> shift) & 255u;
            uint32_t mask = 0xffffffffu;
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                const bool bit = (d >> b) & 1u;
                const uint32_t bal = __ballot_sync(0xffffffffu, bit);
                mask &= bit ? bal : ~bal;
            }
            const uint32_t lower = __popc(mask & lt_mask);
            uint32_t prev = 0;
            if (lower == 0) {
                prev = wh[d];
                wh[d] = prev + __popc(mask);
            }
            prev = __shfl_sync(0xffffffffu, prev, __ffs(mask) - 1);
            rank[i] = prev + lower;
            __syncwarp();
        }
#endif
        __syncthreads();  // (A) all warp histograms complete

        // ---- digit totals, cross-warp exclusive offsets, early publication of the tile aggregate ----
        uint32_t agg = 0, incl = 0;
        if (tid < RADIX) {
            uint32_t sum = 0;
#pragma unroll 4
            for (int w = 0; w < WARPS; ++w) {
                const uint32_t c = s_whist[w * RADIX + tid];
                s_whist[w * RADIX + tid] = sum;
                sum += c;
            }
            agg = sum;
            volatile uint32_t *st = status + (size_t)tile * RADIX + tid;
            *st = (tile == 0 ? FLAG_PREFIX : FLAG_AGG) | agg;
            incl = warp_incl_scan(agg);
            if (lane == 31) s_wtot[warp] = incl;
        }
        __syncthreads();  // (B)
        uint32_t dstart = 0;
        if (tid < RADIX) {
            uint32_t off = 0;
            for (uint32_t w = 0; w < warp; ++w) off += s_wtot[w];
            dstart = off + incl - agg;
            s_dstart[tid] = dstart;
        }
        __syncthreads();  // (C)

        // ---- reorder the tile in shared memory (digit runs become contiguous) ----
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const uint32_t d = (key[i] >> shift) & 255u;
            const uint32_t pos = s_dstart[d] + wh[d] + rank[i];
            s_keys[pos] = key[i];
            if (PAIRS) s_vals[pos] = val[i];
            if constexpr (WIDE) s_vals[TILE_KEYS + pos] = val2[i];
        }

        // ---- decoupled look-back: one thread per digit walks the predecessor tiles ----
        if (tid < RADIX) {
            uint32_t excl = 0;
            if (tile > 0) {
                int64_t t = (int64_t)tile - 1;
                while (true) {
                    volatile uint32_t *st = status + (size_t)t * RADIX + tid;
                    uint32_t v;
                    do { v = *st; } while ((v & (FLAG_AGG | FLAG_PREFIX)) == 0u);
                    excl += v & VAL_MASK;
                    if (v & FLAG_PREFIX) break;
                    --t;
                }
                volatile uint32_t *mine = status + (size_t)tile * RADIX + tid;
                *mine = FLAG_PREFIX | ((excl + agg) & VAL_MASK);
            }
            s_base[tid] = s_gbase[tid] + excl - dstart;
        }
        __syncthreads();  // (D)

        // ---- coalesced write-out of the digit runs ----
        const uint32_t tile_n = (n - tile_base) < TILE_KEYS ? (n - tile_base) : TILE_KEYS;
        for (uint32_t idx = tid; idx < tile_n; idx += THREADS) {
            const uint32_t k = s_keys[idx];
            const uint32_t dst = s_base[(k >> shift) & 255u] + idx;
            keys_out[dst] = k;
            if (PAIRS) vals_out[dst] = s_vals[idx];
            if constexpr (WIDE) vals2_out[dst] = s_vals[TILE_KEYS + idx];
        }
    }
}

// configuration table -------------------------------------------------------------------------------
struct SweepConfig { int threads, items; };
#ifndef GSR_SORT_THREADS
#define GSR_SORT_THREADS 512
#endif
#ifndef GSR_SORT_ITEMS
#define GSR_SORT_ITEMS 10  // sm_90a: 12 keys per thread spill the pairs kernel at the 64 registers two CTAs/SM allow
#endif
constexpr int SWEEP_THREADS = GSR_SORT_THREADS;
constexpr int SWEEP_ITEMS = GSR_SORT_ITEMS;
constexpr uint32_t SWEEP_TILE = SWEEP_THREADS * SWEEP_ITEMS;

template <bool PAIRS>
constexpr size_t sweep_smem() {
    return sizeof(uint32_t) * ((SWEEP_THREADS / 32) * RADIX + SWEEP_TILE * (PAIRS ? 2 : 1));
}
// the wide passes of the depth-order sort (three words per key): 8 keys per thread keep them within the 64 registers of two CTAs per SM
constexpr int WIDE_ITEMS = 8;
constexpr uint32_t WIDE_TILE = SWEEP_THREADS * WIDE_ITEMS;
constexpr size_t wide_smem() { return sizeof(uint32_t) * ((SWEEP_THREADS / 32) * RADIX + 3 * WIDE_TILE); }
static_assert(WIDE_TILE <= SWEEP_TILE, "the narrow passes of the depth-order sort use the wide passes' look-back slices");

}  // namespace

#ifndef GSR_CPU_EMU  // host side: CUDA only (tests/kernel_emu drives the kernels above itself)

// Force-load this file's kernels (CUDA loads modules lazily; a first launch that has to load code while another context's
// kernel spins on a flag this launch would satisfy can stall the host: see gsr_group_attach).
int preload_sort_kernels() {
    cudaFuncAttributes fa;
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, sort_hist_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, true>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, false>));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, sort_hist_depth_kernel));
    GSR_CUDA_TRY(cudaFuncGetAttributes(&fa, onesweep_kernel<SWEEP_THREADS, WIDE_ITEMS, true, true>));
    return GSR_OK;
}
size_t SortWorkspace::bytes() const {
    return sizeof(uint32_t) * (4 * RADIX + 8) + sizeof(uint32_t) * 4ull * max_tiles * RADIX + (alt_keys ? 8ull * max_n : 0) +
           (depth_hist ? sizeof(uint32_t) * (6 * RADIX + 8) + sizeof(uint32_t) * 6ull * depth_max_tiles * RADIX : 0);
}

int sort_workspace_enable_depth(SortWorkspace &ws) {
    if (ws.depth_hist) return GSR_OK;
    const uint32_t tiles = (uint32_t)((ws.max_n + WIDE_TILE - 1) / WIDE_TILE);
    uint32_t *h = nullptr, *st = nullptr;
    cudaError_t e = cudaMalloc((void **)&h, sizeof(uint32_t) * (6 * RADIX + 8));
    if (e == cudaSuccess) e = cudaMalloc((void **)&st, sizeof(uint32_t) * 6ull * tiles * RADIX);
    auto kw = onesweep_kernel<SWEEP_THREADS, WIDE_ITEMS, true, true>;
    int occ = 0;
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kw, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wide_smem());
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kw, SWEEP_THREADS, wide_smem());
    if (e != cudaSuccess || occ < 1) {
        cudaFree(h); cudaFree(st);
        set_last_error("sorter: depth-order workspace: %s", e != cudaSuccess ? cudaGetErrorString(e) : "wide onesweep kernel does not fit on an SM");
        return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
    }
    int dev = 0, sm_count = 0;
    GSR_CUDA_TRY(cudaGetDevice(&dev));
    GSR_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    ws.depth_hist = h; ws.depth_status = st; ws.depth_max_tiles = tiles;
    const uint32_t g = (uint32_t)(sm_count * occ);
    ws.grid_sweep_wide = (int)(g < tiles ? g : tiles);
    return GSR_OK;
}

int sort_workspace_create(SortWorkspace &ws, uint64_t max_n, bool need_alt_buffers) {
    if (max_n == 0 || max_n >= (1ull << 30)) {
        set_last_error("sorter: max_n=%llu outside [1, 2^30)", (unsigned long long)max_n);
        return GSR_ERR_INVALID;
    }
    ws.max_n = max_n;
    ws.max_tiles = (uint32_t)((max_n + SWEEP_TILE - 1) / SWEEP_TILE);
    // hist[1024] + tickets[4] + n_dev[1] (+pad) in one small allocation => one memset per sort
    GSR_CUDA_TRY(cudaMalloc(&ws.hist, sizeof(uint32_t) * (4 * RADIX + 8)));
    ws.tickets = ws.hist + 4 * RADIX;
    ws.n_dev = ws.hist + 4 * RADIX + 4;
    GSR_CUDA_TRY(cudaMalloc(&ws.status, sizeof(uint32_t) * 4ull * ws.max_tiles * RADIX));
    if (need_alt_buffers) {
        GSR_CUDA_TRY(cudaMalloc(&ws.alt_keys, sizeof(uint32_t) * max_n));
        GSR_CUDA_TRY(cudaMalloc(&ws.alt_vals, sizeof(uint32_t) * max_n));
    }
    int dev = 0;
    GSR_CUDA_TRY(cudaGetDevice(&dev));
    int sm_count = 0;
    GSR_CUDA_TRY(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    auto kp = onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, true>;
    auto kk = onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, false>;
    GSR_CUDA_TRY(cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sweep_smem<true>()));
    GSR_CUDA_TRY(cudaFuncSetAttribute(kk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sweep_smem<false>()));
    int occ_p = 0, occ_k = 0;
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_p, kp, SWEEP_THREADS, sweep_smem<true>()));
    GSR_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_k, kk, SWEEP_THREADS, sweep_smem<false>()));
    if (occ_p < 1 || occ_k < 1) {
        set_last_error("sorter: onesweep kernel does not fit on an SM");
        return GSR_ERR_CUDA;
    }
    auto cap_grid = [&](int g) { return (int)((uint32_t)g < ws.max_tiles ? (uint32_t)g : ws.max_tiles); };
    ws.grid_sweep_pairs = cap_grid(sm_count * occ_p);
    ws.grid_sweep_keys = cap_grid(sm_count * occ_k);
    ws.grid_hist = sm_count * 4;
    return GSR_OK;
}

void sort_workspace_destroy(SortWorkspace &ws) {
    cudaFree(ws.hist);
    cudaFree(ws.status);
    cudaFree(ws.alt_keys);
    cudaFree(ws.alt_vals);
    cudaFree(ws.depth_hist);
    cudaFree(ws.depth_status);
    ws = SortWorkspace();
}

int sort_pairs_device(SortWorkspace &ws, uint32_t *keys, uint32_t *vals, const uint32_t *n_ptr, uint32_t *alt_keys,
                      uint32_t *alt_vals, cudaStream_t stream, int *launches) {
    const uint32_t n_max = (uint32_t)ws.max_n;
    // zero hist + tickets (n_dev, when used, is written by the caller AFTER this memset region: keep it out)
    GSR_CUDA_TRY(cudaMemsetAsync(ws.hist, 0, sizeof(uint32_t) * (4 * RADIX + 4), stream));
    sort_hist_kernel<<<ws.grid_hist, HIST_THREADS, 0, stream>>>(keys, n_ptr, n_max, ws.hist, ws.status, SWEEP_TILE, ws.max_tiles);
    uint32_t *kin = keys, *kout = alt_keys, *vin = vals, *vout = alt_vals;
    for (int pass = 0; pass < 4; ++pass) {
        uint32_t *st = ws.status + (size_t)pass * ws.max_tiles * RADIX;
        if (vals) {
            onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, true><<<ws.grid_sweep_pairs, SWEEP_THREADS, sweep_smem<true>(), stream>>>(
                kin, kout, vin, vout, n_ptr, n_max, ws.hist + pass * RADIX, st, ws.tickets + pass, 8 * pass);
        } else {
            onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, false><<<ws.grid_sweep_keys, SWEEP_THREADS, sweep_smem<false>(), stream>>>(
                kin, kout, nullptr, nullptr, n_ptr, n_max, ws.hist + pass * RADIX, st, ws.tickets + pass, 8 * pass);
        }
        uint32_t *t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    if (launches) *launches += 5;
    return GSR_OK;
}

// (tile, depth word, input order): four wide passes over the depth word carry (key, value), then two passes of the pairs kernel over
// the tile bits of the key carry the value.  Six passes: the result is back in keys / vals; depth is left sorted by the word alone.
int sort_pairs_depth_device(SortWorkspace &ws, uint32_t *keys, uint32_t *vals, uint32_t *depth, const uint32_t *n_ptr, uint32_t *alt_keys,
                            uint32_t *alt_vals, uint32_t *alt_depth, cudaStream_t stream, int *launches) {
    if (!ws.depth_hist) { set_last_error("sorter: depth-order workspace not allocated"); return GSR_ERR_STATE; }
    const uint32_t n_max = (uint32_t)ws.max_n;
    const size_t slice = (size_t)ws.depth_max_tiles * RADIX;
    GSR_CUDA_TRY(cudaMemsetAsync(ws.depth_hist, 0, sizeof(uint32_t) * (6 * RADIX + 6), stream));
    uint32_t *tickets = ws.depth_hist + 6 * RADIX;
    sort_hist_depth_kernel<<<ws.grid_hist, HIST_THREADS, 0, stream>>>(keys, depth, n_ptr, n_max, ws.depth_hist, ws.depth_status, WIDE_TILE,
                                                                      SWEEP_TILE, ws.depth_max_tiles);
    uint32_t *din = depth, *dout = alt_depth, *kin = keys, *kout = alt_keys, *vin = vals, *vout = alt_vals, *t;
    for (int pass = 0; pass < 4; ++pass) {
        onesweep_kernel<SWEEP_THREADS, WIDE_ITEMS, true, true><<<ws.grid_sweep_wide, SWEEP_THREADS, wide_smem(), stream>>>(
            din, dout, kin, kout, n_ptr, n_max, ws.depth_hist + pass * RADIX, ws.depth_status + pass * slice, tickets + pass, 8 * pass, vin, vout);
        t = din; din = dout; dout = t;
        t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    for (int pass = 4; pass < 6; ++pass) {
        onesweep_kernel<SWEEP_THREADS, SWEEP_ITEMS, true><<<ws.grid_sweep_pairs, SWEEP_THREADS, sweep_smem<true>(), stream>>>(
            kin, kout, vin, vout, n_ptr, n_max, ws.depth_hist + pass * RADIX, ws.depth_status + pass * slice, tickets + pass, 8 * pass - 16);
        t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    GSR_CUDA_TRY(cudaGetLastError());
    if (launches) *launches += 7;
    return GSR_OK;
}

uint32_t sort_tile_keys() { return SWEEP_TILE; }
#endif  // GSR_CPU_EMU

}  // namespace gsr
