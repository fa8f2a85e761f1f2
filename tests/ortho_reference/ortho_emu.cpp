// ortho_emu.cpp -- the orthographic projection instantiations projection_kernel<INSTANCED, B, true> (GSR_FLAG_ORTHOGRAPHIC) compiled for
// the CPU on top of tests/kernel_emu.  TEST INFRASTRUCTURE: built by tests/ortho_reference.py.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct OrthoLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; };
template <bool INST, int B>
void ortho_body(void *p) { OrthoLaunch *l = static_cast<OrthoLaunch *>(p); gsr::projection_kernel<INST, B, true>(l->a, l->ia); }
}  // namespace

// projection_kernel<instanced, bands, true> over a store of soa_planes(store) planes (the kernel reads planes 0-2 and the first
// sh_planes(bands)).  Per-frame constants exactly as render_enqueue() derives them.  Instanced: frame = n x 32 constants of
// instance_prepare_kernel, desc / warp_inst the drawn-id layout (tests/ortho_reference.py builds them).  Returns M, or -1 for an unknown
// variant.
extern "C" long long emu_ortho_projection(int instanced, int bands, const void *soa, unsigned long long plane_stride, unsigned num_splats,
                                          const float *vp, const void *uniforms32, int sh_bulk_min, void *records, uint32_t *keys, uint32_t *values,
                                          unsigned capacity, unsigned *visible_out, int *last_tile_out, const float *inst_frame,
                                          const void *inst_desc, const uint32_t *warp_inst) {
    OrthoLaunch l;
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
    const unsigned blocks = gsr::projection_num_blocks(num_splats);
    gsr::FrameState fs;
    memset(&fs, 0, sizeof fs);
    std::vector<unsigned long long> lookback(blocks ? blocks : 1, 0ull);
    pa.records = static_cast<float4 *>(records); pa.keys = keys; pa.values = values; pa.capacity = capacity;
    pa.lookback = lookback.data(); pa.frame = &fs;
    l.ia.frame = inst_frame; l.ia.desc = static_cast<const gsr::InstanceDesc *>(inst_desc); l.ia.warp_inst = warp_inst;
    void (*body)(void *) = nullptr;
    switch (bands + (instanced ? 10 : 0)) {
        case 1: body = &ortho_body<false, 1>; break;
        case 2: body = &ortho_body<false, 2>; break;
        case 3: body = &ortho_body<false, 3>; break;
        case 4: body = &ortho_body<false, 4>; break;
        case 11: body = &ortho_body<true, 1>; break;
        case 12: body = &ortho_body<true, 2>; break;
        case 13: body = &ortho_body<true, 3>; break;
        case 14: body = &ortho_body<true, 4>; break;
        default: return -1;
    }
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    return (long long)fs.dup_total;
}
