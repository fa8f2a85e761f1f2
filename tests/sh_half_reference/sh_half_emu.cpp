// sh_half_emu.cpp -- the binary16 SH store (GSR_FLAG_SH_HALF) on the CPU, on top of tests/kernel_emu: the two conversions, the HALF
// ingest kernels aos_to_soa_kernel<true> / ply_to_soa_kernel<FILTER3D, true>, and every projection_kernel<INSTANCED, B, ORTHO, AA, DEPTH,
// CUT, true> (with instance_prepare_kernel and an optional appearance table for the instanced ones).  TEST INFRASTRUCTURE: built by
// tests/test_sh_half.py.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct HalfAosLaunch { const float4 *aos; uint64_t count; float4 *soa; uint64_t stride, first; int planes; };
void half_aos_body(void *p) {
    const HalfAosLaunch *l = static_cast<const HalfAosLaunch *>(p);
    gsr::aos_to_soa_kernel<true>(l->aos, l->count, l->soa, l->stride, l->first, l->planes);
}
struct HalfPlyLaunch { const float *ply; gsr_ply_layout lay; uint64_t count; float creation; float4 *soa; uint64_t stride, first; int planes; int32_t f3d; };
template <bool FILTER3D>
void half_ply_body(void *p) {
    const HalfPlyLaunch *l = static_cast<const HalfPlyLaunch *>(p);
    gsr::ply_to_soa_kernel<FILTER3D, true>(l->ply, l->lay.nprops, l->count, l->creation, l->soa, l->stride, l->first, l->lay, l->planes, l->f3d);
}

struct PrepLaunch { gsr::InstancePrepareArgs p; };
void prep_body(void *p) { gsr::instance_prepare_kernel(static_cast<PrepLaunch *>(p)->p); }

struct HalfLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; uint32_t *dw; gsr::CutoutArgs ct; };
template <bool INST, int B, bool ORTHO, bool AA, bool DEPTH, bool CUT>
void half_body(void *p) {
    HalfLaunch *l = static_cast<HalfLaunch *>(p);
    if constexpr (CUT) gsr::projection_kernel<INST, B, ORTHO, AA, DEPTH, true, true>(l->a, l->ia, gsr::DepthArgs{l->dw}, l->ct);
    else gsr::projection_kernel<INST, B, ORTHO, AA, DEPTH, false, true>(l->a, l->ia, gsr::DepthArgs{l->dw});
}
template <bool INST, bool ORTHO, bool AA, bool DEPTH, bool CUT>
void (*pick_bands(int bands))(void *) {
    switch (bands) {
        case 1: return &half_body<INST, 1, ORTHO, AA, DEPTH, CUT>;
        case 2: return &half_body<INST, 2, ORTHO, AA, DEPTH, CUT>;
        case 3: return &half_body<INST, 3, ORTHO, AA, DEPTH, CUT>;
        case 4: return &half_body<INST, 4, ORTHO, AA, DEPTH, CUT>;
        default: return nullptr;
    }
}
template <bool INST, bool DEPTH, bool CUT>
void (*pick_modes(int bands, bool ortho, bool aa))(void *) {
    if (ortho) return aa ? pick_bands<INST, true, true, DEPTH, CUT>(bands) : pick_bands<INST, true, false, DEPTH, CUT>(bands);
    return aa ? pick_bands<INST, false, true, DEPTH, CUT>(bands) : pick_bands<INST, false, false, DEPTH, CUT>(bands);
}
template <bool INST>
void (*pick_variant(int bands, bool ortho, bool aa, bool depth, bool cut))(void *) {
    if (cut) return depth ? pick_modes<INST, true, true>(bands, ortho, aa) : pick_modes<INST, false, true>(bands, ortho, aa);
    return depth ? pick_modes<INST, true, false>(bands, ortho, aa) : pick_modes<INST, false, false>(bands, ortho, aa);
}
}  // namespace

// h(c) as the ingest kernels store it (gsr::sh_half), and the exact decode
extern "C" void emu_sh_half_encode(const float *in, uint16_t *out, unsigned long long n) {
    for (unsigned long long i = 0; i < n; ++i) out[i] = (uint16_t)gsr::sh_half(in[i]);
}
extern "C" void emu_sh_half_decode(const uint16_t *in, float *out, unsigned long long n) {
    for (unsigned long long i = 0; i < n; ++i) out[i] = gsr::half_bits_to_float(in[i]);
}

// planes = soa_planes(store bands, true)
extern "C" int emu_sh_half_aos_to_soa(const void *aos60, unsigned long long count, void *soa, unsigned long long plane_stride, unsigned long long first,
                                      int planes) {
    HalfAosLaunch l{static_cast<const float4 *>(aos60), count, static_cast<float4 *>(soa), plane_stride, first, planes};
    run_blocks((unsigned)((count + gsr::SPLATS_PER_BLOCK - 1) / gsr::SPLATS_PER_BLOCK), 256, &half_aos_body, &l);
    return 0;
}

// layout: 8 ints in gsr_ply_layout order; filter_3d >= 0: the filtered upload (gsr_upload_ply_filtered)
extern "C" int emu_sh_half_ply_to_soa(const float *ply, const int *layout8, unsigned long long count, float creation_time, void *soa,
                                      unsigned long long plane_stride, unsigned long long first, int planes, int filter_3d) {
    HalfPlyLaunch l;
    memcpy(&l.lay, layout8, sizeof l.lay);
    if (l.lay.nprops < 1 || l.lay.nprops > 256) return 1;
    l.ply = ply; l.count = count; l.creation = creation_time; l.soa = static_cast<float4 *>(soa); l.stride = plane_stride; l.first = first;
    l.planes = planes; l.f3d = filter_3d;
    run_blocks((unsigned)((count + gsr::INGEST_SPLATS - 1) / gsr::INGEST_SPLATS), (unsigned)gsr::INGEST_SPLATS,
               filter_3d >= 0 ? &half_ply_body<true> : &half_ply_body<false>, &l);
    return 0;
}

// projection_kernel<n > 0, bands, ortho, v > 0, depth_words != null, cutouts != null, true> over a binary16 store (soa_planes(store bands,
// true) planes x plane_stride float4), per-frame constants exactly as render_enqueue() derives them.  n = 0: the plain kernel over
// num_splats splats.  n > 0: the instanced front part like emu_appearance_projection (xf = n x 24 floats, ranges = n x (first, count),
// rows = n x 8 appearance floats or null).  Returns M, or -1 for an argument out of range.
extern "C" long long emu_sh_half_projection(int bands, int ortho, float v, const void *soa, unsigned long long plane_stride, unsigned num_splats,
                                            const float *vp, const void *uniforms32, int sh_bulk_min, unsigned n, const float *xf,
                                            const unsigned long long *ranges, const float *rows, void *records, uint32_t *keys, uint32_t *values,
                                            uint32_t *depth_words, unsigned capacity, unsigned *visible_out, int *last_tile_out, unsigned *overflow_out,
                                            const void *cutouts) {
    HalfLaunch l;
    gsr::ProjectionArgs &pa = l.a;
    memset(&pa, 0, sizeof pa);
    memcpy(&pa.u, uniforms32, sizeof pa.u);
    std::vector<gsr::InstanceDesc> desc(n ? n : 1);
    std::vector<uint32_t> warp_inst;
    std::vector<float> frame((size_t)(n ? n : 1) * gsr::INSTANCE_FRAME_FLOATS, 0.0f);
    std::vector<float> table((size_t)(n ? n : 1) * gsr::INSTANCE_APPEARANCE_FLOATS, -1.0f);
    uint32_t drawn = num_splats;
    if (n) {   // the layout, exactly like gsr_set_instances, and the prepare kernel
        uint64_t warps = 0;
        for (unsigned k = 0; k < n; ++k) {
            if (ranges[2 * k] + ranges[2 * k + 1] > plane_stride) return -1;
            desc[k].first = ranges[2 * k]; desc[k].count = (uint32_t)ranges[2 * k + 1]; desc[k].warp0 = (uint32_t)warps;
            warps += (ranges[2 * k + 1] + 31) / 32;
        }
        drawn = (uint32_t)(32 * warps);
        warp_inst.assign((size_t)gsr::projection_num_blocks(drawn) * (gsr::PROJ_THREADS / 32) + 1, 0xFFFFFFFFu);
        for (unsigned k = 0; k < n; ++k)
            for (uint32_t j = 0; j < (ranges[2 * k + 1] + 31) / 32; ++j) warp_inst[desc[k].warp0 + j] = k;
        PrepLaunch pl;
        pl.p.xf = xf;
        memcpy(pl.p.v, vp, sizeof pl.p.v);
        memcpy(pl.p.cam, pa.u.camera_pos, sizeof pl.p.cam);
        pl.p.count = n; pl.p.out = frame.data();
        pl.p.appearance = rows; pl.p.appearance_out = table.data();
        run_blocks(1, 256, &prep_body, &pl);
    } else if (num_splats > plane_stride) {
        return -1;
    }
    const unsigned blocks = gsr::projection_num_blocks(drawn);
    pa.soa = static_cast<const float4 *>(soa); pa.plane_stride = plane_stride; pa.num_splats = drawn;
    memcpy(pa.vp, vp, sizeof pa.vp);
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
    gsr::FrameState fs;
    memset(&fs, 0, sizeof fs);
    std::vector<unsigned long long> lookback(blocks ? blocks : 1, 0ull);
    pa.records = static_cast<float4 *>(records); pa.keys = keys; pa.values = values; pa.capacity = capacity;
    pa.lookback = lookback.data(); pa.frame = &fs;
    l.ia.frame = frame.data(); l.ia.desc = desc.data(); l.ia.warp_inst = n ? warp_inst.data() : nullptr;
    l.ia.appearance = (n && rows) ? table.data() : nullptr;
    l.dw = depth_words;
    memset(&l.ct, 0, sizeof l.ct);
    if (cutouts) memcpy(&l.ct, cutouts, sizeof l.ct);
    const bool aa = v > 0.0f, depth = depth_words != nullptr, cut = cutouts != nullptr;
    void (*body)(void *) = n ? pick_variant<true>(bands, ortho != 0, aa, depth, cut) : pick_variant<false>(bands, ortho != 0, aa, depth, cut);
    if (!body) return -1;
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    if (overflow_out) *overflow_out = fs.overflow;
    return (long long)fs.dup_total;
}
