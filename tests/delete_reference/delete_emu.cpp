// delete_emu.cpp -- the splat delete and duplicate kernels of selection.cu compiled for the CPU on top of tests/kernel_emu:
// compact_store_kernel with several CTAs running at once (they interleave wherever one spins in its look-back or waits at a barrier),
// then the follow-up kernels, exactly as gsr_delete_hidden / gsr_duplicate_selection launch them.  TEST INFRASTRUCTURE: built by
// tests/delete_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // fibers of one thread: sequential

// Several CTAs at once: one emulated workgroup of ctas x 256 invocations, CTA c = invocations [256 c, 256 c + 256).  __syncthreads is a
// per-CTA barrier that spins, and each CTA gets its own shared state.  g_slow > 0 makes the first CTA of every wave slow where it matters:
// its third barrier (the one between the first look-back and the loads of its moved splats) is released only after g_slow rounds of
// everybody else, so its successors run as far as the kernel lets them before its sources are read.
namespace delemu {
constexpr unsigned MAX_CTAS = 8, THREADS = 256;
unsigned g_block_base = 0;   // the first block of the running wave (0 outside compact_store_kernel)
unsigned g_slow = 0;
constexpr unsigned LOAD_BARRIER = 2;   // compact_store_kernel's barriers before it: after the ticket, after the warp counts
struct Bar { unsigned count, gen; };
Bar g_bars[MAX_CTAS];
inline unsigned local() { return ::glsl::sched().cur->local_index; }
inline cuda_emu::dim tid() { return cuda_emu::dim{local() % THREADS, 0, 0}; }
inline cuda_emu::dim bid() { return cuda_emu::dim{::glsl::sched().cur->group_id.x + g_block_base + local() / THREADS, 0, 0}; }
inline void cta_barrier() {
    Bar &b = g_bars[local() / THREADS];
    const unsigned g = b.gen;
    if (++b.count == THREADS) {
        if (local() / THREADS == 0 && g == LOAD_BARRIER)
            for (unsigned i = 0; i < g_slow; ++i) ::glsl::spin_yield();
        b.count = 0;
        ++b.gen;
    }
    else while (b.gen == g) ::glsl::spin_yield();
}
template <class T> T &cta_shared() { static T s[MAX_CTAS]; return s[local() / THREADS]; }
}  // namespace delemu
#undef threadIdx
#undef blockIdx
#define threadIdx (::delemu::tid())
#define blockIdx (::delemu::bid())
#define __syncthreads() ::delemu::cta_barrier()
#define COMPACT_CTA_SHARED(T, name) T &name = ::delemu::cta_shared<T>()
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
struct CompactLaunch { gsr::CompactArgs a; int mode; };
template <int B, bool HALF>
void compact_body(void *p) {
    const CompactLaunch *l = static_cast<CompactLaunch *>(p);
    if (l->mode == gsr::COMPACT_DELETE) gsr::compact_store_kernel<B, HALF, gsr::COMPACT_DELETE>(l->a);
    else gsr::compact_store_kernel<B, HALF, gsr::COMPACT_DUPLICATE>(l->a);
}
void (*pick_compact(int bands, bool half))(void *) {
    switch (bands * 2 + (half ? 1 : 0)) {
        case 2: return &compact_body<1, false>;
        case 3: return &compact_body<1, true>;
        case 4: return &compact_body<2, false>;
        case 5: return &compact_body<2, true>;
        case 6: return &compact_body<3, false>;
        case 7: return &compact_body<3, true>;
        case 8: return &compact_body<4, false>;
        case 9: return &compact_body<4, true>;
        default: return nullptr;
    }
}

// compact_store_kernel over every tile of [0, n), in waves of `ctas` CTAs running at once (a later wave starts when the earlier one is
// done, like CTAs that become resident as others retire; tickets still decide which tile a CTA gets).  Returns *total.
unsigned long long run_compact(CompactLaunch &l, int bands, bool half, unsigned ctas) {
    unsigned long long total = 0ull;
    if (l.a.n == 0) return 0ull;
    const uint32_t words = (uint32_t)((l.a.n + 31ull) >> 5);
    const uint32_t tiles = (uint32_t)gsr::compact_lookback_words(words) - 1u;
    std::vector<unsigned long long> lookback(tiles + 1, 0ull);
    l.a.lookback = lookback.data();
    l.a.total = &total;
    void (*body)(void *) = pick_compact(bands, half);
    cuda_emu::g_block_dim = cuda_emu::dim{delemu::THREADS, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{tiles, 1, 1};
    for (uint32_t b0 = 0; b0 < tiles; b0 += ctas) {
        const unsigned c = tiles - b0 < ctas ? tiles - b0 : ctas;
        memset(delemu::g_bars, 0, sizeof delemu::g_bars);
        delemu::g_block_base = b0;
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(c * delemu::THREADS, 1, 1), body, &l);
    }
    delemu::g_block_base = 0;
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{1, 1, 1};
    return total;
}
}  // namespace

// gsr_delete_hidden's kernels on a host store (planes x plane_stride float4) and masks (words each): returns k.  slow: see g_slow.
extern "C" long long emu_delete_hidden(int bands, int half, void *soa, unsigned long long plane_stride, unsigned long long n, uint32_t *hidden,
                                       uint32_t *selected, uint32_t *scratch, unsigned words, unsigned ctas, unsigned slow) {
    if (!pick_compact(bands, half != 0) || ctas < 1 || ctas > delemu::MAX_CTAS) return -1;
    delemu::g_slow = slow;
    CompactLaunch l;
    memset(&l, 0, sizeof l);
    l.a.soa = static_cast<float4 *>(soa); l.a.plane_stride = plane_stride; l.a.n = n;
    l.a.hidden = hidden; l.a.selected = selected; l.a.sel_out = scratch;
    l.mode = gsr::COMPACT_DELETE;
    const unsigned long long k = run_compact(l, bands, half != 0, ctas);
    delemu::g_slow = 0;
    struct FL { float4 *soa; unsigned long long st; int planes; unsigned long long k, n; uint32_t *h, *s, *x; unsigned words; } fl{
        l.a.soa, plane_stride, gsr::soa_planes(bands, half != 0), k, n, hidden, selected, scratch, words};
    const unsigned long long items = words > n - k ? (unsigned long long)words : n - k;
    if (items)
        run_blocks((unsigned)((items + 255) / 256), 256, [](void *p) {
            FL *f = static_cast<FL *>(p);
            gsr::delete_finish_kernel(f->soa, f->st, f->planes, f->k, f->n, f->h, f->s, f->x, f->words);
        }, &fl);
    return (long long)k;
}

// gsr_duplicate_selection's kernels (the count, then, when the copies fit below max_splats, the copy and the new selection): returns S,
// or -2 - S when they do not fit (nothing written).
extern "C" long long emu_duplicate_selection(int bands, int half, void *soa, unsigned long long plane_stride, unsigned long long n,
                                             unsigned long long max_splats, uint32_t *hidden, uint32_t *selected, unsigned words, unsigned ctas) {
    if (!pick_compact(bands, half != 0) || ctas < 1 || ctas > delemu::MAX_CTAS) return -1;
    unsigned long long S = 0ull;
    struct CL { const uint32_t *s; unsigned long long n, *c; } cl{selected, n, &S};
    const unsigned cw = (unsigned)((n + 31ull) >> 5);
    if (cw) run_blocks((cw + 255) / 256 < 1024 ? (cw + 255) / 256 : 1024, 256, [](void *p) {
            CL *c = static_cast<CL *>(p);
            gsr::count_selected_kernel(c->s, c->n, c->c);
        }, &cl);
    if (S > max_splats - n) return -2 - (long long)S;
    if (S) {
        CompactLaunch l;
        memset(&l, 0, sizeof l);
        l.a.soa = static_cast<float4 *>(soa); l.a.plane_stride = plane_stride; l.a.n = n;
        l.a.hidden = hidden; l.a.selected = selected;
        l.mode = gsr::COMPACT_DUPLICATE;
        if (run_compact(l, bands, half != 0, ctas) != S) return -1;
    }
    struct DL { unsigned long long n, S; uint32_t *h, *s; unsigned words; } dl{n, S, hidden, selected, words};
    if (words) run_blocks((words + 255) / 256, 256, [](void *p) {
            DL *d = static_cast<DL *>(p);
            gsr::duplicate_finish_kernel(d->n, d->S, d->h, d->s, d->words);
        }, &dl);
    return (long long)S;
}
