// property_emu.cpp -- the splat property kernels of selection.cu compiled for the CPU on top of tests/kernel_emu: select_where_kernel
// block by block, and splat_histogram_kernel with several CTAs running at once (they interleave at their barriers and warp collectives,
// each with its own shared histogram, all adding into the same global counters).  TEST INFRASTRUCTURE: built by
// tests/property_reference.py.
#include <type_traits>

#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // fibers of one thread: sequential

// Several CTAs at once: one emulated workgroup of ctas x 512 invocations, CTA c = invocations [512 c, 512 c + 512); __syncthreads is a
// per-CTA barrier that spins, and each CTA gets its own shared state.
namespace propemu {
constexpr unsigned MAX_CTAS = 8, THREADS = 512;
unsigned g_block_base = 0;   // the first block of the running wave
struct Bar { unsigned count, gen; };
Bar g_bars[MAX_CTAS];
inline unsigned local() { return ::glsl::sched().cur->local_index; }
inline cuda_emu::dim tid() { return cuda_emu::dim{local() % THREADS, 0, 0}; }
inline cuda_emu::dim bid() { return cuda_emu::dim{g_block_base + local() / THREADS, 0, 0}; }
inline void cta_barrier() {
    Bar &b = g_bars[local() / THREADS];
    const unsigned g = b.gen;
    if (++b.count == THREADS) { b.count = 0; ++b.gen; }
    else while (b.gen == g) ::glsl::spin_yield();
}
template <class T> T &cta_shared() { static T s[MAX_CTAS]; return s[local() / THREADS]; }
bool g_multi = false;   // inside the histogram's waves
inline cuda_emu::dim thread_idx() { return g_multi ? tid() : cuda_emu::thread_idx(); }
inline cuda_emu::dim block_idx() { return g_multi ? bid() : cuda_emu::block_idx(); }
inline void sync_threads() { if (g_multi) cta_barrier(); else ::glsl::barrier(); }
}  // namespace propemu
#undef threadIdx
#undef blockIdx
#define threadIdx (::propemu::thread_idx())
#define blockIdx (::propemu::block_idx())
#define __syncthreads() ::propemu::sync_threads()
#define HIST_CTA_SHARED(T, name) T &name = ::propemu::cta_shared<T>()
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
struct WhereLaunch { gsr::WhereArgs a; };
struct PropHistLaunch { gsr::HistArgs a; };
template <bool HALF, int PL>
void where_body(void *p) { gsr::select_where_kernel<HALF, PL>(static_cast<WhereLaunch *>(p)->a); }
template <bool HALF, int PL>
void hist_body(void *p) { gsr::splat_histogram_kernel<HALF, PL>(static_cast<PropHistLaunch *>(p)->a); }

// launch_property's variant table
template <class L>
void (*pick(int planes, bool half))(void *) {
    constexpr bool W = std::is_same<L, WhereLaunch>::value;
    switch (planes | (half && (planes & gsr::PROP_P3) ? 8 : 0)) {
        case 2: return W ? &where_body<false, 2> : &hist_body<false, 2>;
        case 3: return W ? &where_body<false, 3> : &hist_body<false, 3>;
        case 4: return W ? &where_body<false, 4> : &hist_body<false, 4>;
        case 6: return W ? &where_body<false, 6> : &hist_body<false, 6>;
        case 7: return W ? &where_body<false, 7> : &hist_body<false, 7>;
        case 8 | 4: return W ? &where_body<true, 4> : &hist_body<true, 4>;
        case 8 | 6: return W ? &where_body<true, 6> : &hist_body<true, 6>;
        case 8 | 7: return W ? &where_body<true, 7> : &hist_body<true, 7>;
        default: return nullptr;
    }
}
}  // namespace

// select_where_kernel over every word of the masks: filters = n gsr_splat_filter structs, [first, first + count) the tested range.
extern "C" int emu_select_where(int half, const void *soa, unsigned long long plane_stride, uint32_t *selected, const uint32_t *hidden,
                                unsigned words, unsigned op, unsigned long long first, unsigned long long count, const void *filters,
                                unsigned n) {
    WhereLaunch l;
    memset(&l, 0, sizeof l);
    gsr::WhereArgs &a = l.a;
    a.selected = selected; a.hidden = hidden; a.words = words; a.op = op;
    a.first = first; a.count = count;
    a.soa = static_cast<const float4 *>(soa); a.plane_stride = plane_stride;
    a.n = n;
    int planes = 0;
    memcpy(a.f, filters, sizeof(gsr_splat_filter) * n);
    for (unsigned i = 0; i < n; ++i) planes |= gsr::prop_planes(a.f[i].property);
    void (*body)(void *) = pick<WhereLaunch>(planes, half != 0);
    if (!body) return -1;
    const unsigned blocks = (words + 7u) / 8u;
    if (blocks) run_blocks(blocks, 256u, body, &l);
    return 0;
}

// splat_histogram_kernel with `blocks` CTAs in waves of `ctas` running at once.  counts (bins + 3) and keys (2, see HistArgs) are the
// global counters, initialised by the caller; hidden == NULL: the masks are not in use.
extern "C" int emu_splat_histogram(int half, const void *soa, unsigned long long plane_stride, unsigned long long first,
                                   unsigned long long count, const uint32_t *hidden, const uint32_t *selected, unsigned selected_only,
                                   const void *prop, const float *edges, unsigned bins, unsigned long long *counts, int32_t *keys,
                                   unsigned blocks, unsigned ctas) {
    if (ctas < 1 || ctas > propemu::MAX_CTAS || bins < 1 || bins > GSR_MAX_HISTOGRAM_BINS) return -1;
    PropHistLaunch l;
    memset(&l, 0, sizeof l);
    gsr::HistArgs &a = l.a;
    a.soa = static_cast<const float4 *>(soa); a.plane_stride = plane_stride;
    a.first = first; a.count = count;
    a.hidden = hidden; a.selected = selected; a.selected_only = selected_only;
    a.bins = bins;
    a.top = 1u;
    while (2u * a.top <= bins - 1u) a.top *= 2u;
    memcpy(&a.prop, prop, sizeof a.prop);
    a.counts = counts; a.keys = keys; a.edges = edges;
    void (*body)(void *) = pick<PropHistLaunch>(gsr::prop_planes(a.prop.property), half != 0);
    if (!body) return -1;
    cuda_emu::g_block_dim = cuda_emu::dim{propemu::THREADS, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{blocks, 1, 1};
    propemu::g_multi = true;
    for (unsigned b0 = 0; b0 < blocks; b0 += ctas) {
        const unsigned c = blocks - b0 < ctas ? blocks - b0 : ctas;
        memset(propemu::g_bars, 0, sizeof propemu::g_bars);
        propemu::g_block_base = b0;
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(c * propemu::THREADS, 1, 1), body, &l);
    }
    propemu::g_multi = false;
    propemu::g_block_base = 0;
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{1, 1, 1};
    return 0;
}
