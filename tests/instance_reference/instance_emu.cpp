// instance_emu.cpp -- instance_prepare_kernel + projection_kernel<true> (splat instances) compiled for the CPU on top of tests/kernel_emu.
// TEST INFRASTRUCTURE: built by tests/instance_reference.py.  kernel_emu.cpp brings every kernel file of csrc/ and the CUDA shim.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct PrepLaunch { gsr::InstancePrepareArgs p; };
void prep_body(void *p) { gsr::instance_prepare_kernel(static_cast<PrepLaunch *>(p)->p); }
struct InstLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; };
void inst_body(void *p) { InstLaunch *l = static_cast<InstLaunch *>(p); gsr::projection_kernel<true>(l->a, l->ia); }
}  // namespace

// The library's instanced front part for one frame: `xf` = n x 24 floats (A|t, B|u per instance), `ranges` = n x (first, count).
// Per-frame constants are derived exactly like render_enqueue() in gsr_api.cu; the drawn-id layout exactly like gsr_set_instances.
// soa: 15 planes x plane_stride float4.  records: D entries of 48 B.  frame_out (nullable): n x 32 floats of the prepare kernel.
// Returns M, or -1 if an argument is out of range.
extern "C" long long emu_projection_instanced(const void *soa, unsigned long long plane_stride, const float *vp, const void *uniforms32,
                                              unsigned n, const float *xf, const unsigned long long *ranges, void *records, uint32_t *keys,
                                              uint32_t *values, unsigned capacity, unsigned *visible_out, int *last_tile_out,
                                              unsigned *overflow_out, float *frame_out) {
    // the layout
    std::vector<gsr::InstanceDesc> desc(n ? n : 1);
    uint64_t warps = 0;
    for (unsigned k = 0; k < n; ++k) {
        if (ranges[2 * k] + ranges[2 * k + 1] > plane_stride) return -1;
        desc[k].first = ranges[2 * k]; desc[k].count = (uint32_t)ranges[2 * k + 1]; desc[k].warp0 = (uint32_t)warps;
        warps += (ranges[2 * k + 1] + 31) / 32;
    }
    const uint32_t drawn = (uint32_t)(32 * warps);
    const unsigned blocks = gsr::projection_num_blocks(drawn);
    std::vector<uint32_t> warp_inst((size_t)blocks * (gsr::PROJ_THREADS / 32) + 1, 0xFFFFFFFFu);
    for (unsigned k = 0; k < n; ++k)
        for (uint32_t j = 0; j < (ranges[2 * k + 1] + 31) / 32; ++j) warp_inst[desc[k].warp0 + j] = k;
    // the prepare kernel: one block
    std::vector<float> frame((size_t)(n ? n : 1) * gsr::INSTANCE_FRAME_FLOATS, 0.0f);
    gsr::Uniforms u;
    memcpy(&u, uniforms32, sizeof u);
    PrepLaunch pl;
    pl.p.xf = xf;
    memcpy(pl.p.v, vp, sizeof pl.p.v);
    memcpy(pl.p.cam, u.camera_pos, sizeof pl.p.cam);
    pl.p.count = n; pl.p.out = frame.data();
    run_blocks(1, 256, &prep_body, &pl);
    if (frame_out) memcpy(frame_out, frame.data(), sizeof(float) * gsr::INSTANCE_FRAME_FLOATS * n);
    // the projection over the drawn ids
    InstLaunch il;
    gsr::ProjectionArgs &pa = il.a;
    memset(&pa, 0, sizeof pa);
    pa.soa = static_cast<const float4 *>(soa); pa.plane_stride = plane_stride; pa.num_splats = drawn;
    memcpy(pa.vp, vp, sizeof pa.vp);
    pa.u = u;
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
    pa.fast_reject = 0; pa.fast_mode = 0; pa.sh_bulk_min = 12;
    gsr::FrameState fs;
    memset(&fs, 0, sizeof fs);
    std::vector<unsigned long long> lookback(blocks ? blocks : 1, 0ull);
    pa.records = static_cast<float4 *>(records); pa.keys = keys; pa.values = values; pa.capacity = capacity;
    pa.lookback = lookback.data(); pa.frame = &fs;
    il.ia.frame = frame.data(); il.ia.desc = desc.data(); il.ia.warp_inst = warp_inst.data();
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, &inst_body, &il);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    if (overflow_out) *overflow_out = fs.overflow;
    return (long long)fs.dup_total;
}
