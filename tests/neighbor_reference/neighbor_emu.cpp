// neighbor_emu.cpp -- TEST INFRASTRUCTURE, built by tests/neighbor_reference.py.  Two independent things:
//   1. emu_select_neighborhood: the kernels of csrc/neighbors.cu compiled for the CPU on top of tests/kernel_emu, launched in the order of
//      gsr_select_neighborhood with the emulated Onesweep sort of kernel_emu.cpp between the keys and the grid.  The union-find runs
//      several CTAs at once, and every atomicCAS first yields to every other thread, so the hooks of different CTAs interleave.  The
//      bucket count and the candidate limit can be lowered (forced hash collisions, a budget at and over its limit).
//   2. ref_select_neighborhood: the rule of include/gsr.h with a plain serial grid (a hash map of cells) and a serial disjoint-set forest,
//      for the clouds too large for the numpy brute force.  It shares no code with the kernels.
#include <unordered_map>
#include <vector>

#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }
inline unsigned long long atomicMax(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; *p = o < v ? v : o; return o; }
inline unsigned atomicCAS(unsigned *p, unsigned cmp, unsigned v) {
    ::glsl::spin_yield();   // let every other thread run first: hooks of different CTAs interleave here
    const unsigned o = *p;
    if (o == cmp) *p = v;
    return o;
}

// Several CTAs at once (the union-find): one emulated workgroup of ctas x 256 invocations, CTA c = invocations [256 c, 256 c + 256)
namespace nbemu {
constexpr unsigned THREADS = 256, MAX_CTAS = 8;
unsigned g_block_base = 0;
bool g_multi = false;
inline unsigned local() { return ::glsl::sched().cur->local_index; }
inline cuda_emu::dim thread_idx() { return g_multi ? cuda_emu::dim{local() % THREADS, 0, 0} : cuda_emu::thread_idx(); }
inline cuda_emu::dim block_idx() { return g_multi ? cuda_emu::dim{g_block_base + local() / THREADS, 0, 0} : cuda_emu::block_idx(); }
}  // namespace nbemu
#undef threadIdx
#undef blockIdx
#define threadIdx (::nbemu::thread_idx())
#define blockIdx (::nbemu::block_idx())
#include "../../godotgaussiansplatting_b200/csrc/neighbors.cu"

namespace {
template <void (*K)(gsr::NeighborArgs)>
void body(void *p) { K(*static_cast<const gsr::NeighborArgs *>(p)); }

void run_waves(unsigned blocks, void (*f)(void *), gsr::NeighborArgs *a, unsigned ctas) {
    cuda_emu::g_block_dim = cuda_emu::dim{nbemu::THREADS, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{blocks, 1, 1};
    nbemu::g_multi = true;
    for (unsigned b0 = 0; b0 < blocks; b0 += ctas) {
        const unsigned c = blocks - b0 < ctas ? blocks - b0 : ctas;
        nbemu::g_block_base = b0;
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(c * nbemu::THREADS, 1, 1), f, a);
    }
    nbemu::g_multi = false;
    nbemu::g_block_base = 0;
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{1, 1, 1};
}
}  // namespace

// plane0: max_splats float4; hidden / selected: words each (selected is updated).  bucket_bits 0: the library's choice; limit: the
// candidate limit (GSR_MAX_NEIGHBOR_CANDIDATES in the library).  stats[5] = participants, inside, candidates, clusters, largest.
// Returns 0, or 1 when the budget refuses the call (selected untouched).
extern "C" int emu_select_neighborhood(const void *plane0, unsigned long long max_splats, const uint32_t *hidden, uint32_t *selected,
                                       unsigned words, unsigned long long first, unsigned long long count, float radius, int mode,
                                       unsigned threshold, int op, unsigned bucket_bits, unsigned long long limit, unsigned ctas,
                                       unsigned long long *stats) {
    const uint64_t m = max_splats;
    const uint32_t p = bucket_bits ? bucket_bits : gsr::neighbor_bucket_bits(count);
    std::vector<uint32_t> keys(m), vals(m), parent(m), size(m), start((1ull << p) + 1, 0xCDCDCDCDu), inside(words, 0u);
    std::vector<float4> pos(m);
    gsr::NeighborCounters ctr;
    memset(&ctr, 0, sizeof ctr);
    gsr::NeighborArgs a;
    memset(&a, 0, sizeof a);
    a.plane0 = static_cast<const float4 *>(plane0); a.hidden = hidden; a.selected = selected; a.words = words; a.op = (uint32_t)op;
    a.first = first; a.count = count;
    a.h = gsr::neighbor_cell_size(radius);
    a.r2 = radius * radius;
    a.mode = (uint32_t)mode; a.threshold = threshold;
    a.shift = 32u - p;
    a.keys = keys.data(); a.vals = vals.data(); a.parent = parent.data(); a.size = size.data(); a.pos = pos.data(); a.start = start.data();
    a.inside = inside.data(); a.ctr = &ctr;
    const unsigned eb = (unsigned)((count + nbemu::THREADS - 1) / nbemu::THREADS), wb = (words + 7u) / 8u;
    if (count) {
        run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_keys_kernel>, &a);
        emu_sort_pairs(keys.data(), vals.data(), ctr.n, (uint32_t)m, 2);
        memset(parent.data(), 0xFF, sizeof(uint32_t) * m);
        memset(size.data(), 0, sizeof(uint32_t) * m);
        run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_grid_kernel>, &a);
        run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_impure_kernel>, &a);
        run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_budget_kernel>, &a);
        if (ctr.candidates > limit) { stats[2] = ctr.candidates; return 1; }
    }
    switch (mode) {
        case GSR_NEIGHBOR_SPARSE:
            if (eb) run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_query_kernel<GSR_NEIGHBOR_SPARSE>>, &a);
            if (wb) run_blocks(wb, nbemu::THREADS, &body<gsr::neighbor_combine_kernel<GSR_NEIGHBOR_SPARSE>>, &a);
            break;
        case GSR_NEIGHBOR_GROW:
            if (eb) run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_query_kernel<GSR_NEIGHBOR_GROW>>, &a);
            if (wb) run_blocks(wb, nbemu::THREADS, &body<gsr::neighbor_combine_kernel<GSR_NEIGHBOR_GROW>>, &a);
            break;
        default:
            if (eb) {
                run_waves(eb, &body<gsr::neighbor_union_kernel>, &a, ctas < 1 ? 1 : (ctas > nbemu::MAX_CTAS ? nbemu::MAX_CTAS : ctas));
                run_blocks(eb, nbemu::THREADS, &body<gsr::neighbor_compress_kernel>, &a);
            }
            if (wb) {
                if (mode == GSR_NEIGHBOR_CONNECTED) run_blocks(wb, nbemu::THREADS, &body<gsr::neighbor_combine_kernel<GSR_NEIGHBOR_CONNECTED>>, &a);
                else run_blocks(wb, nbemu::THREADS, &body<gsr::neighbor_combine_kernel<GSR_NEIGHBOR_SMALL_CLUSTERS>>, &a);
            }
    }
    for (unsigned w = 0; w < words; ++w) if (inside[w]) return -1;   // the scratch mask must be left zero
    const bool cl = mode >= GSR_NEIGHBOR_CONNECTED;
    stats[0] = ctr.n; stats[1] = ctr.inside; stats[2] = ctr.candidates; stats[3] = cl ? ctr.clusters : 0; stats[4] = cl ? ctr.largest : 0;
    return 0;
}

// ---- the serial reference -------------------------------------------------------------------------------------------------------
namespace {
struct Key { long long x, y, z; bool operator==(const Key &o) const { return x == o.x && y == o.y && z == o.z; } };
struct KeyHash { size_t operator()(const Key &k) const { return (size_t)(k.x * 73856093ll ^ k.y * 19349663ll ^ k.z * 83492791ll); } };
long long ref_axis(float v, double h) {
    const double q = floor((double)v / h);
    return (long long)(q < -0x1p62 ? -0x1p62 : (q > 0x1p62 ? 0x1p62 : q));
}
bool ref_near(const float *p, const float *q, float r2) {
    volatile float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
    volatile float xx = dx * dx, yy = dy * dy, zz = dz * dz;
    volatile float s = xx + yy;
    volatile float d2 = s + zz;
    return d2 <= r2;
}
uint32_t dsu_find(std::vector<uint32_t> &par, uint32_t x) {
    while (par[x] != x) { par[x] = par[par[x]]; x = par[x]; }
    return x;
}
}  // namespace

// xyz: 3 floats per slot, [0, m); part: 1 per participant; sel: the selection (bools) restricted by the caller to participants.
// inside_out: m bytes, stats as above; mode -1: every mode from one pass, inside_out 4 m bytes and stats 4 x 5 in GSR_NEIGHBOR_* order
// (the SPARSE and SMALL_CLUSTERS thresholds both `threshold`).
extern "C" int ref_select_neighborhood(const float *xyz, unsigned long long m, const uint8_t *part, const uint8_t *sel, float radius, int mode,
                                       unsigned threshold, uint8_t *inside_out, unsigned long long *stats) {
    const double h = (double)radius * (1.0 + 0x1p-20);
    const float r2 = radius * radius;
    std::unordered_map<Key, std::vector<uint32_t>, KeyHash> grid;
    std::vector<Key> cell(m);
    unsigned long long participants = 0, candidates = 0;
    for (uint64_t i = 0; i < m; ++i) {
        if (!part[i]) continue;
        cell[i] = Key{ref_axis(xyz[3 * i], h), ref_axis(xyz[3 * i + 1], h), ref_axis(xyz[3 * i + 2], h)};
        grid[cell[i]].push_back((uint32_t)i);
        ++participants;
    }
    std::vector<uint32_t> par(m), nbr(m, 0), size(m, 0);
    std::vector<uint8_t> near_sel(m, 0), seed(m, 0);
    for (uint64_t i = 0; i < m; ++i) par[i] = (uint32_t)i;
    for (uint64_t i = 0; i < m; ++i) {
        if (!part[i]) continue;
        const Key c = cell[i];
        for (int o = 0; o < 27; ++o) {
            auto it = grid.find(Key{c.x + (o % 3 - 1), c.y + ((o / 3) % 3 - 1), c.z + (o / 9 - 1)});
            if (it == grid.end()) continue;
            candidates += it->second.size();
            for (uint32_t j : it->second) {
                if (j == i || !ref_near(xyz + 3 * i, xyz + 3 * j, r2)) continue;
                ++nbr[i];
                if (sel[j]) near_sel[i] = 1;
                const uint32_t a = dsu_find(par, (uint32_t)i), b = dsu_find(par, j);
                if (a != b) par[a > b ? a : b] = a < b ? a : b;
            }
        }
    }
    unsigned long long clusters = 0, largest = 0;
    for (uint64_t i = 0; i < m; ++i) {
        if (!part[i]) continue;
        const uint32_t r = dsu_find(par, (uint32_t)i);
        ++size[r];
        if (sel[i]) seed[r] = 1;
    }
    for (uint64_t i = 0; i < m; ++i) {
        if (part[i] && dsu_find(par, (uint32_t)i) == i) { ++clusters; largest = size[i] > largest ? size[i] : largest; }
    }
    const int m0 = mode < 0 ? 0 : mode, m1 = mode < 0 ? 3 : mode;
    for (int md = m0; md <= m1; ++md) {
        uint8_t *out = inside_out + (mode < 0 ? (size_t)md * m : 0);
        unsigned long long *st = stats + (mode < 0 ? 5 * md : 0), inside = 0;
        for (uint64_t i = 0; i < m; ++i) {
            uint8_t in = 0;
            if (part[i]) {
                const uint32_t r = dsu_find(par, (uint32_t)i);
                switch (md) {
                    case GSR_NEIGHBOR_SPARSE: in = nbr[i] < threshold; break;
                    case GSR_NEIGHBOR_GROW: in = sel[i] || near_sel[i]; break;
                    case GSR_NEIGHBOR_CONNECTED: in = seed[r]; break;
                    default: in = size[r] < threshold; break;
                }
            }
            out[i] = in;
            inside += in;
        }
        const bool cl = md >= GSR_NEIGHBOR_CONNECTED;
        st[0] = participants; st[1] = inside; st[2] = candidates; st[3] = cl ? clusters : 0; st[4] = cl ? largest : 0;
    }
    return 0;
}
