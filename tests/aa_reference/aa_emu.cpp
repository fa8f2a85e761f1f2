// aa_emu.cpp -- the anti-aliased projection instantiations projection_kernel<INSTANCED, B, ORTHO, true> (gsr_set_antialiasing) and the
// filtered ingest ply_to_soa_kernel<true> (gsr_upload_ply_filtered) compiled for the CPU on top of tests/kernel_emu.  TEST
// INFRASTRUCTURE: built by tests/aa_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct AaLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; };
template <bool INST, int B, bool ORTHO>
void aa_body(void *p) { AaLaunch *l = static_cast<AaLaunch *>(p); gsr::projection_kernel<INST, B, ORTHO, true>(l->a, l->ia); }
struct AaPlyLaunch { const float *ply; gsr_ply_layout lay; uint64_t count; float creation; float4 *soa; uint64_t stride, first; int planes, filter_3d; };
void aa_ply_body(void *p) {
    const AaPlyLaunch *l = static_cast<const AaPlyLaunch *>(p);
    gsr::ply_to_soa_kernel<true>(l->ply, l->lay.nprops, l->count, l->creation, l->soa, l->stride, l->first, l->lay, l->planes, l->filter_3d);
}
}  // namespace

// projection_kernel<instanced, bands, ortho, true> with a.aa_variance = v over a store of soa_planes(store) planes (the kernel reads
// planes 0-2 and the first sh_planes(bands)).  Per-frame constants exactly as render_enqueue() derives them.  Instanced: frame = n x 32
// constants of instance_prepare_kernel, desc / warp_inst the drawn-id layout (tests/aa_reference.py builds them).  Returns M, or -1 for
// an unknown variant.
extern "C" long long emu_aa_projection(int instanced, int bands, int ortho, float v, const void *soa, unsigned long long plane_stride,
                                       unsigned num_splats, const float *vp, const void *uniforms32, int sh_bulk_min, void *records, uint32_t *keys,
                                       uint32_t *values, unsigned capacity, unsigned *visible_out, int *last_tile_out, const float *inst_frame,
                                       const void *inst_desc, const uint32_t *warp_inst) {
    AaLaunch l;
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
    void (*body)(void *) = nullptr;
    switch (bands + (instanced ? 10 : 0) + (ortho ? 100 : 0)) {
        case 1: body = &aa_body<false, 1, false>; break;
        case 2: body = &aa_body<false, 2, false>; break;
        case 3: body = &aa_body<false, 3, false>; break;
        case 4: body = &aa_body<false, 4, false>; break;
        case 11: body = &aa_body<true, 1, false>; break;
        case 12: body = &aa_body<true, 2, false>; break;
        case 13: body = &aa_body<true, 3, false>; break;
        case 14: body = &aa_body<true, 4, false>; break;
        case 101: body = &aa_body<false, 1, true>; break;
        case 102: body = &aa_body<false, 2, true>; break;
        case 103: body = &aa_body<false, 3, true>; break;
        case 104: body = &aa_body<false, 4, true>; break;
        case 111: body = &aa_body<true, 1, true>; break;
        case 112: body = &aa_body<true, 2, true>; break;
        case 113: body = &aa_body<true, 3, true>; break;
        case 114: body = &aa_body<true, 4, true>; break;
        default: return -1;
    }
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    return (long long)fs.dup_total;
}

// ply_to_soa_kernel<true> (gsr_upload_ply_filtered).  layout: 8 ints in gsr_ply_layout order; planes = soa_planes(store bands).
extern "C" int emu_aa_ply_to_soa(const float *ply, const int *layout8, int filter_3d, unsigned long long count, float creation_time, void *soa,
                                 unsigned long long plane_stride, unsigned long long first, int planes) {
    AaPlyLaunch l;
    memcpy(&l.lay, layout8, sizeof l.lay);
    if (l.lay.nprops < 1 || l.lay.nprops > 256 || filter_3d < 0 || filter_3d >= (int)l.lay.nprops) return 1;
    l.ply = ply; l.count = count; l.creation = creation_time; l.soa = static_cast<float4 *>(soa); l.stride = plane_stride; l.first = first;
    l.planes = planes; l.filter_3d = filter_3d;
    run_blocks((unsigned)((count + gsr::INGEST_SPLATS - 1) / gsr::INGEST_SPLATS), (unsigned)gsr::INGEST_SPLATS, &aa_ply_body, &l);
    return 0;
}
