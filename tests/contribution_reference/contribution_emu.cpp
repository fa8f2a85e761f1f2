// contribution_emu.cpp -- composite_contrib_kernel<CONTRACT> (splat contribution) and the contribution variants of the splat property
// kernels compiled for the CPU on top of tests/kernel_emu (and of tests/property_reference/property_emu.cpp for selection.cu).
// TEST INFRASTRUCTURE: built by tests/contribution_reference.py.
#include "../property_reference/property_emu.cpp"

namespace {
struct ContribLaunch { const gsr::CompositeArgs *args; const gsr::ContribArgs *cb; int variant; };
void contrib_body(void *p) {
    const ContribLaunch *l = static_cast<const ContribLaunch *>(p);
    if (l->variant == 1) gsr::composite_contrib_kernel<false>(*l->args, *l->cb);   // GSR_FLAG_UNCONTRACTED_BLEND
    else gsr::composite_contrib_kernel<true>(*l->args, *l->cb);
}
}  // namespace

// One frame of the full image, its tiles dealt round-robin to `ctas` persistent blocks (CTA c takes tiles c, c + ctas, ...) that run
// one after another and all add into the same records: tiles of different blocks meet on shared slots within one frame.  warp_inst /
// desc: the instance layout, or nullptr.  overflow: the frame's FrameState::overflow.  frames: the device frame counter (block 0 adds
// to it).  Returns 0, or 1 if a tile was left out.
extern "C" int emu_composite_contrib(int variant, const void *records, const uint32_t *values, const uint32_t *bounds, float *out_rgba,
                                     float *depth_out, const float *scene_depth, const float *vp, int width, int height,
                                     const uint32_t *warp_inst, const void *desc, void *accum, uint32_t *frames, uint32_t epoch, int ctas,
                                     int overflow, unsigned long long *staged_out) {
    const int tiles_x = (width + 15) / 16, tiles_y = (height + 15) / 16, T = tiles_x * tiles_y;
    if (ctas < 1) return 1;
    gsr::FrameState frame;
    memset(&frame, 0, sizeof frame);
    frame.overflow = overflow ? 1u : 0u;
    gsr::CompositeArgs a;
    memset(&a, 0, sizeof a);
    a.records = static_cast<const float4 *>(records);
    a.values = values;
    a.bounds = reinterpret_cast<const uint2 *>(bounds);
    a.out = reinterpret_cast<float4 *>(out_rgba);
    a.width = width; a.height = height; a.tiles_x = tiles_x;
    a.tile_begin = 0; a.row_step = 1;
    a.heatmap_factor = 0.0f; a.target_tile_id = 0xFFFFFFFFu;
    float4 pick;
    a.pick = &pick;
    a.frame = &frame; a.count_staged = 1;
    a.ctas_per_sm = 1; a.sm_count = 1; a.contract = variant == 1 ? 0 : 1;
    a.view_z[0] = vp[2]; a.view_z[1] = vp[6]; a.view_z[2] = vp[10]; a.view_z[3] = vp[14];
    a.scene_depth = scene_depth; a.depth_out = depth_out;
    gsr::ContribArgs cb;
    cb.accum = static_cast<gsr_splat_contribution *>(accum);
    cb.warp_inst = warp_inst; cb.desc = static_cast<const gsr::InstanceDesc *>(desc);
    cb.epoch = epoch;
    std::vector<uint32_t> order((size_t)T);
    uint32_t done = 0;
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    for (int c = 0; c < ctas; ++c) {
        uint32_t n = 0;
        for (int k = c; k < T; k += ctas) order[n++] = (uint32_t)k;
        if (!n) continue;
        a.order = order.data(); a.num_tiles = (int32_t)n;
        frame.comp_head = 0;
        cb.frames = c == 0 ? frames : nullptr;   // (the frame's block 0)
        ContribLaunch l{&a, &cb, variant};
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(128, 1, 1), &contrib_body, &l);
        done += frame.comp_head >= n ? n : 0u;
    }
    if (staged_out) *staged_out = frame.staged;
    return done == (uint32_t)T ? 0 : 1;
}

namespace {
template <class L>
void (*pick_contrib(int planes, bool half))(void *) {
    constexpr bool W = std::is_same<L, WhereLaunch>::value;
    constexpr int ALL = gsr::PROP_P1 | gsr::PROP_P2 | gsr::PROP_P3 | gsr::PROP_PC;
    if (!(planes & gsr::PROP_PC)) return pick<L>(planes, half);
    if (planes == gsr::PROP_PC) return W ? &where_body<false, gsr::PROP_PC> : &hist_body<false, gsr::PROP_PC>;
    if (half) return W ? &where_body<true, ALL> : &hist_body<true, ALL>;
    return W ? &where_body<false, ALL> : &hist_body<false, ALL>;
}
}  // namespace

// emu_select_where of property_emu.cpp with the contribution buffer (max_splats records).
extern "C" int emu_select_where_contrib(int half, const void *soa, unsigned long long plane_stride, uint32_t *selected, const uint32_t *hidden,
                                        unsigned words, unsigned op, unsigned long long first, unsigned long long count, const void *filters,
                                        unsigned n, const void *contrib) {
    WhereLaunch l;
    memset(&l, 0, sizeof l);
    gsr::WhereArgs &a = l.a;
    a.selected = selected; a.hidden = hidden; a.words = words; a.op = op;
    a.first = first; a.count = count;
    a.soa = static_cast<const float4 *>(soa); a.plane_stride = plane_stride;
    a.n = n;
    a.contrib = static_cast<const gsr_splat_contribution *>(contrib);
    int planes = 0;
    memcpy(a.f, filters, sizeof(gsr_splat_filter) * n);
    for (unsigned i = 0; i < n; ++i) planes |= gsr::prop_sources(a.f[i].property);
    void (*body)(void *) = pick_contrib<WhereLaunch>(planes, half != 0);
    if (!body) return -1;
    const unsigned blocks = (words + 7u) / 8u;
    if (blocks) run_blocks(blocks, 256u, body, &l);
    return 0;
}

// emu_splat_histogram of property_emu.cpp with the contribution buffer.
extern "C" int emu_splat_histogram_contrib(int half, const void *soa, unsigned long long plane_stride, unsigned long long first,
                                           unsigned long long count, const uint32_t *hidden, const uint32_t *selected, unsigned selected_only,
                                           const void *prop, const float *edges, unsigned bins, unsigned long long *counts, int32_t *keys,
                                           unsigned blocks, unsigned ctas, const void *contrib) {
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
    a.contrib = static_cast<const gsr_splat_contribution *>(contrib);
    void (*body)(void *) = pick_contrib<PropHistLaunch>(gsr::prop_sources(a.prop.property), half != 0);
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
