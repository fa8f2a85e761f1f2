// cutout_emu.cpp -- the cutout projection kernels of gsr_set_cutouts compiled for the CPU on top of tests/kernel_emu: every instantiation
// projection_kernel<INSTANCED, B, ORTHO, AA, DEPTH, true>, and the matching CUT = false kernel for comparisons.  TEST INFRASTRUCTURE: built
// by tests/cutout_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct CutLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; uint32_t *dw; gsr::CutoutArgs ct; };
template <bool INST, int B, bool ORTHO, bool AA, bool DEPTH, bool CUT>
void cut_body(void *p) {
    CutLaunch *l = static_cast<CutLaunch *>(p);
    if constexpr (CUT) gsr::projection_kernel<INST, B, ORTHO, AA, DEPTH, true>(l->a, l->ia, gsr::DepthArgs{l->dw}, l->ct);
    else gsr::projection_kernel<INST, B, ORTHO, AA, DEPTH, false>(l->a, l->ia, gsr::DepthArgs{l->dw});
}

template <bool INST, bool ORTHO, bool AA, bool DEPTH, bool CUT>
void (*pick_bands(int bands))(void *) {
    switch (bands) {
        case 1: return &cut_body<INST, 1, ORTHO, AA, DEPTH, CUT>;
        case 2: return &cut_body<INST, 2, ORTHO, AA, DEPTH, CUT>;
        case 3: return &cut_body<INST, 3, ORTHO, AA, DEPTH, CUT>;
        case 4: return &cut_body<INST, 4, ORTHO, AA, DEPTH, CUT>;
        default: return nullptr;
    }
}
template <bool INST, bool DEPTH, bool CUT>
void (*pick_modes(int bands, bool ortho, bool aa))(void *) {
    if (ortho) return aa ? pick_bands<INST, true, true, DEPTH, CUT>(bands) : pick_bands<INST, true, false, DEPTH, CUT>(bands);
    return aa ? pick_bands<INST, false, true, DEPTH, CUT>(bands) : pick_bands<INST, false, false, DEPTH, CUT>(bands);
}
template <bool INST, bool CUT>
void (*pick_depth(int bands, bool ortho, bool aa, bool depth))(void *) {
    return depth ? pick_modes<INST, true, CUT>(bands, ortho, aa) : pick_modes<INST, false, CUT>(bands, ortho, aa);
}
template <bool INST>
void (*pick_variant(int bands, bool ortho, bool aa, bool depth, bool cut))(void *) {
    return cut ? pick_depth<INST, true>(bands, ortho, aa, depth) : pick_depth<INST, false>(bands, ortho, aa, depth);
}
}  // namespace

extern "C" unsigned emu_cutout_args_bytes() { return (unsigned)sizeof(gsr::CutoutArgs); }

// projection_kernel<instanced, bands, ortho, v > 0, depth_words != null, cutouts != null> over a store of soa_planes(store) planes, with
// a.aa_variance = v.  Per-frame constants exactly as render_enqueue() derives them; instanced: frame / desc / warp_inst as
// tests/depth_order_reference.py builds them.  cutouts: a CutoutArgs (KEEP volumes first), or null for the CUT = false kernel.
// Returns M, or -1 for an unknown variant.
extern "C" long long emu_cutout_projection(int instanced, int bands, int ortho, float v, const void *soa, unsigned long long plane_stride,
                                           unsigned num_splats, const float *vp, const void *uniforms32, int sh_bulk_min, void *records,
                                           uint32_t *keys, uint32_t *values, uint32_t *depth_words, unsigned capacity, unsigned *visible_out,
                                           int *last_tile_out, unsigned *overflow_out, const float *inst_frame, const void *inst_desc,
                                           const uint32_t *warp_inst, const void *cutouts) {
    CutLaunch l;
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
    memset(&l.ct, 0, sizeof l.ct);
    if (cutouts) memcpy(&l.ct, cutouts, sizeof l.ct);
    void (*body)(void *) = instanced ? pick_variant<true>(bands, ortho != 0, v > 0.0f, depth_words != nullptr, cutouts != nullptr)
                                     : pick_variant<false>(bands, ortho != 0, v > 0.0f, depth_words != nullptr, cutouts != nullptr);
    if (!body) return -1;
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    if (overflow_out) *overflow_out = fs.overflow;
    return (long long)fs.dup_total;
}
