// export_emu.cpp -- the splat export kernels of selection.cu compiled for the CPU on top of tests/kernel_emu: export_count_kernel, then
// export_ply_kernel with several CTAs running at once (they interleave wherever one spins in its look-back or waits at a barrier),
// exactly as gsr_export_ply launches them.  TEST INFRASTRUCTURE: built by tests/export_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // fibers of one thread: sequential

// Several CTAs at once: one emulated workgroup of ctas x 256 invocations, CTA c = invocations [256 c, 256 c + 256).  __syncthreads is a
// per-CTA barrier that spins, and each CTA gets its own shared state and row buffer.  g_slow > 0 makes the first CTA of every wave
// slow where it matters: its second barrier (after its warp counts, before it publishes its count) is released only after g_slow rounds
// of everybody else, so its successors reach their look-backs and wait on it.
namespace expemu {
constexpr unsigned MAX_CTAS = 8, THREADS = 256;
unsigned g_block_base = 0;   // the first block of the running wave (0 outside export_ply_kernel)
unsigned g_slow = 0;
constexpr unsigned COUNT_BARRIER = 1;   // export_ply_kernel's barriers before it: after the ticket
struct Bar { unsigned count, gen; };
Bar g_bars[MAX_CTAS];
inline unsigned local() { return ::glsl::sched().cur->local_index; }
inline cuda_emu::dim tid() { return cuda_emu::dim{local() % THREADS, 0, 0}; }
inline cuda_emu::dim bid() { return cuda_emu::dim{::glsl::sched().cur->group_id.x + g_block_base + local() / THREADS, 0, 0}; }
inline void cta_barrier() {
    const unsigned n = cuda_emu::g_block_dim.x < THREADS ? cuda_emu::g_block_dim.x : THREADS;
    Bar &b = g_bars[local() / THREADS];
    const unsigned g = b.gen;
    if (++b.count == n) {
        if (local() / THREADS == 0 && g == COUNT_BARRIER)
            for (unsigned i = 0; i < g_slow; ++i) ::glsl::spin_yield();
        b.count = 0;
        ++b.gen;
    }
    else while (b.gen == g) ::glsl::spin_yield();
}
template <class T> T &cta_shared() { static T s[MAX_CTAS]; return s[local() / THREADS]; }
inline float *cta_rows() { static float r[MAX_CTAS][THREADS * gsr::export_row_floats(3)]; return r[local() / THREADS]; }
}  // namespace expemu
#undef threadIdx
#undef blockIdx
#define threadIdx (::expemu::tid())
#define blockIdx (::expemu::bid())
#define __syncthreads() ::expemu::cta_barrier()
#define COMPACT_CTA_SHARED(T, name) T &name = ::expemu::cta_shared<T>()
#define EXPORT_CTA_ROWS(name) float *name = ::expemu::cta_rows()
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
template <int B, bool HALF>
void export_body(void *p) { gsr::export_ply_kernel<B, HALF>(*static_cast<gsr::ExportArgs *>(p)); }
void (*pick_export(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &export_body<1, false>;
        case 3: return &export_body<1, true>;
        case 4: return &export_body<2, false>;
        case 5: return &export_body<2, true>;
        case 6: return &export_body<3, false>;
        case 7: return &export_body<3, true>;
        case 8: return &export_body<4, false>;
        case 9: return &export_body<4, true>;
        default: return nullptr;
    }
}
}  // namespace

// gsr_export_ply's kernels on a host store (planes x plane_stride float4) and masks (hidden == NULL: not in use).  Returns the count of
// the counting pass; with dst (dst_rows rows) and a count that fits, the writing pass then fills dst in waves of `ctas` CTAs (a later
// wave starts when the earlier one is done, like CTAs that become resident as others retire; tickets still decide which tile a CTA
// gets).  -1: bad arguments; -2: the writing pass's own total differs from the count.
extern "C" long long emu_export_ply(int bands, int half, const void *soa, unsigned long long plane_stride, unsigned long long n,
                                    const uint32_t *hidden, const uint32_t *selected, int selected_only, int degree, float *dst,
                                    unsigned long long dst_rows, unsigned ctas, unsigned slow) {
    void (*body)(void *) = pick_export(bands, half != 0);
    if (!body || ctas < 1 || ctas > expemu::MAX_CTAS || degree < 0 || degree > bands - 1) return -1;
    gsr::ExportArgs a;
    memset(&a, 0, sizeof a);
    a.soa = static_cast<const float4 *>(soa); a.plane_stride = plane_stride; a.n = n;
    a.hidden = hidden; a.selected = selected; a.selected_only = selected_only ? 1u : 0u; a.degree = degree;
    if (a.selected_only && !hidden) return 0;
    unsigned long long count = 0ull;
    a.count = &count;
    const uint32_t words = (uint32_t)((n + 31ull) >> 5);
    if (words) {
        const unsigned need = (words + gsr::SEL_WARPS - 1) / gsr::SEL_WARPS, blocks = need < 2048u ? need : 2048u;
        run_blocks(blocks, 256, [](void *p) { gsr::export_count_kernel(*static_cast<gsr::ExportArgs *>(p)); }, &a);
    }
    if (!dst || count > dst_rows || count == 0) return (long long)count;
    const uint32_t tiles = (uint32_t)gsr::compact_lookback_words(words) - 1u;
    std::vector<unsigned long long> lookback(tiles + 1, 0ull);
    a.lookback = lookback.data();
    a.dst = dst;
    expemu::g_slow = slow;
    cuda_emu::g_block_dim = cuda_emu::dim{expemu::THREADS, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{tiles, 1, 1};
    for (uint32_t b0 = 0; b0 < tiles; b0 += ctas) {
        const unsigned c = tiles - b0 < ctas ? tiles - b0 : ctas;
        memset(expemu::g_bars, 0, sizeof expemu::g_bars);
        expemu::g_block_base = b0;
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(c * expemu::THREADS, 1, 1), body, &a);
    }
    expemu::g_block_base = 0;
    expemu::g_slow = 0;
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{1, 1, 1};
    // the last tile's PREFIX word is the writing pass's total
    return (lookback[tiles - 1] & gsr::CS_VALUE) == count ? (long long)count : -2;
}
