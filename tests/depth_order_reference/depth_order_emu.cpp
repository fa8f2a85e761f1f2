// depth_order_emu.cpp -- the depth-order kernels of gsr_set_depth_order compiled for the CPU on top of tests/kernel_emu: the projection
// instantiations projection_kernel<INSTANCED, B, ORTHO, AA, true> (every pair's depth word beside its key) and the (tile, depth word)
// sort -- sort_hist_depth_kernel, four wide onesweep passes, two narrow ones.  TEST INFRASTRUCTURE: built by tests/depth_order_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct DepthLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; uint32_t *dw; };
template <bool INST, int B, bool ORTHO, bool AA>
void depth_body(void *p) { DepthLaunch *l = static_cast<DepthLaunch *>(p); gsr::projection_kernel<INST, B, ORTHO, AA, true>(l->a, l->ia, gsr::DepthArgs{l->dw}); }

template <bool INST, bool ORTHO, bool AA>
void (*pick_bands(int bands))(void *) {
    switch (bands) {
        case 1: return &depth_body<INST, 1, ORTHO, AA>;
        case 2: return &depth_body<INST, 2, ORTHO, AA>;
        case 3: return &depth_body<INST, 3, ORTHO, AA>;
        case 4: return &depth_body<INST, 4, ORTHO, AA>;
        default: return nullptr;
    }
}
template <bool INST>
void (*pick_variant(int bands, bool ortho, bool aa))(void *) {
    if (ortho) return aa ? pick_bands<INST, true, true>(bands) : pick_bands<INST, true, false>(bands);
    return aa ? pick_bands<INST, false, true>(bands) : pick_bands<INST, false, false>(bands);
}

struct HistDepthLaunch { const uint32_t *keys, *depth, *n_ptr; uint32_t n_max; uint32_t *hist, *status; uint32_t wide_tile, narrow_tile, max_tiles; };
void hist_depth_body(void *p) {
    const HistDepthLaunch *l = static_cast<const HistDepthLaunch *>(p);
    gsr::sort_hist_depth_kernel(l->keys, l->depth, l->n_ptr, l->n_max, l->hist, l->status, l->wide_tile, l->narrow_tile, l->max_tiles);
}
struct WideLaunch { const uint32_t *din; uint32_t *dout; const uint32_t *kin; uint32_t *kout; const uint32_t *vin; uint32_t *vout;
                    const uint32_t *n_ptr; uint32_t n_max; const uint32_t *hist; uint32_t *status, *ticket; int shift; };
void wide_body(void *p) {
    const WideLaunch *l = static_cast<const WideLaunch *>(p);
    gsr::onesweep_kernel<gsr::SWEEP_THREADS, gsr::WIDE_ITEMS, true, true>(l->din, l->dout, l->kin, l->kout, l->n_ptr, l->n_max, l->hist, l->status,
                                                                         l->ticket, l->shift, l->vin, l->vout);
}
}  // namespace

// projection_kernel<instanced, bands, ortho, v > 0, true> over a store of soa_planes(store) planes, with a.aa_variance = v.  Per-frame
// constants exactly as render_enqueue() derives them; instanced: frame / desc / warp_inst as tests/aa_reference.py builds them.
// depth_words: `capacity` entries beside keys / values.  Returns M, or -1 for an unknown variant.
extern "C" long long emu_depth_projection(int instanced, int bands, int ortho, float v, const void *soa, unsigned long long plane_stride,
                                          unsigned num_splats, const float *vp, const void *uniforms32, int sh_bulk_min, void *records, uint32_t *keys,
                                          uint32_t *values, uint32_t *depth_words, unsigned capacity, unsigned *visible_out, int *last_tile_out,
                                          unsigned *overflow_out, const float *inst_frame, const void *inst_desc, const uint32_t *warp_inst) {
    DepthLaunch l;
    gsr::ProjectionArgs &pa = l.a;
    memset(&pa, 0, sizeof pa);
    pa.soa = static_cast<const float4 *>(soa); pa.plane_stride = plane_stride; pa.num_splats = num_splats;
    memcpy(pa.vp, vp, sizeof pa.vp);
    memcpy(&pa.u, uniforms32, sizeof pa.u);
    {
        const float tfi0 = vp[16 + 0], tfi1 = vp[16 + 5];
        const volatile float hw = (float)pa.u.dims[0] * 0.5f, hh = (float)pa.u.dims[1] * 0.5f;
        const volatile float f0 = hw * tfi0, f1 = hh * tfi1;
        const volatile float t0 = 1.0f / tfi0, t1 = 1.0f / tfi1;
        const volatile float n0 = -t0, n1 = -t1;
        pa.focal_base[0] = f0; pa.focal_base[1] = f1;
        pa.lim_lo[0] = n0 * 1.3f; pa.lim_lo[1] = n1 * 1.3f;
        pa.lim_hi[0] = t0 * 1.3f; pa.lim_hi[1] = t1 * 1.3f;
    }
    pa.band_y0 = 0; pa.band_y1 = (pa.u.dims[1] + gsr::TILE - 1) / gsr::TILE; pa.row_mod = 1; pa.row_rem = 0;
    pa.fast_reject = 0; pa.fast_mode = 0; pa.sh_bulk_min = sh_bulk_min;
    pa.aa_variance = v;
    const unsigned blocks = gsr::projection_num_blocks(num_splats);
    gsr::FrameState fs;
    memset(&fs, 0, sizeof fs);
    std::vector<unsigned long long> lookback(blocks ? blocks : 1, 0ull);
    pa.records = static_cast<float4 *>(records); pa.keys = keys; pa.values = values; pa.capacity = capacity;
    pa.lookback = lookback.data(); pa.frame = &fs;
    l.ia.frame = inst_frame; l.ia.desc = static_cast<const gsr::InstanceDesc *>(inst_desc); l.ia.warp_inst = warp_inst;
    l.dw = depth_words;
    void (*body)(void *) = instanced ? pick_variant<true>(bands, ortho != 0, v > 0.0f) : pick_variant<false>(bands, ortho != 0, v > 0.0f);
    if (!body) return -1;
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    if (overflow_out) *overflow_out = fs.overflow;
    return (long long)fs.dup_total;
}

// sort_pairs_depth_device: the histogram kernel on `hist_grid` blocks, then the four wide passes over the depth word and the two narrow
// passes over the key's tile bits, each by ONE persistent block that pulls every tile in ticket order.  keys / values / depth: n_max
// entries each, sorted in place; n <= n_max is read "from the device".
extern "C" int emu_depth_sort(uint32_t *keys, uint32_t *values, uint32_t *depth, uint32_t n, uint32_t n_max, int hist_grid) {
    const uint32_t max_tiles = (n_max + gsr::WIDE_TILE - 1) / gsr::WIDE_TILE;
    const size_t slice = (size_t)max_tiles * 256;
    uint32_t *hist = static_cast<uint32_t *>(calloc(6 * 256 + 8, sizeof(uint32_t)));
    uint32_t *status = static_cast<uint32_t *>(malloc(sizeof(uint32_t) * 6 * slice));
    memset(status, 0xCD, sizeof(uint32_t) * 6 * slice);   // the histogram kernel must clear what the passes use
    std::vector<uint32_t> alt_k(n_max), alt_v(n_max), alt_d(n_max);
    uint32_t *tickets = hist + 6 * 256;
    const uint32_t n_dev = n;
    HistDepthLaunch h{keys, depth, &n_dev, n_max, hist, status, gsr::WIDE_TILE, gsr::SWEEP_TILE, max_tiles};
    cuda_emu::g_block_dim = cuda_emu::dim{512, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{(unsigned)hist_grid, 1, 1};
    for (int b = 0; b < hist_grid; ++b) glsl::run_workgroup(glsl::uvec3((unsigned)b, 0, 0), glsl::uvec3(512, 1, 1), &hist_depth_body, &h);
    cuda_emu::g_block_dim = cuda_emu::dim{(unsigned)gsr::SWEEP_THREADS, 1, 1};
    cuda_emu::g_grid_dim = cuda_emu::dim{1, 1, 1};
    uint32_t *din = depth, *dout = alt_d.data(), *kin = keys, *kout = alt_k.data(), *vin = values, *vout = alt_v.data(), *t;
    for (int pass = 0; pass < 4; ++pass) {
        WideLaunch l{din, dout, kin, kout, vin, vout, &n_dev, n_max, hist + pass * 256, status + pass * slice, tickets + pass, 8 * pass};
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3((unsigned)gsr::SWEEP_THREADS, 1, 1), &wide_body, &l);
        t = din; din = dout; dout = t;
        t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    for (int pass = 4; pass < 6; ++pass) {
        SweepLaunch l{kin, kout, vin, vout, &n_dev, n_max, hist + pass * 256, status + pass * slice, tickets + pass, 8 * pass - 16};
        glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3((unsigned)gsr::SWEEP_THREADS, 1, 1), &sweep_pairs_body, &l);
        t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    free(hist); free(status);
    return 0;
}
