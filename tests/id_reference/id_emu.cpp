// id_emu.cpp -- composite_ids_kernel<CONTRACT, MOTION> (splat IDs, with or without motion vectors) compiled for the CPU on top
// of tests/kernel_emu.
// TEST INFRASTRUCTURE: built by tests/id_reference.py.  kernel_emu.cpp brings every kernel file of csrc/ and the CUDA shim.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct IdLaunch { const gsr::CompositeArgs *args; const gsr::MotionArgs *mo; const gsr::SplatIdArgs *ids; int variant, motion; };
void id_body(void *p) {
    const IdLaunch *l = static_cast<const IdLaunch *>(p);
    if (l->motion) {
        gsr::WithIds<true> x;
        static_cast<gsr::MotionArgs &>(x) = *l->mo;
        x.ids = *l->ids;
        if (l->variant == 1) gsr::composite_ids_kernel<false, true>(*l->args, x);   // GSR_FLAG_UNCONTRACTED_BLEND
        else gsr::composite_ids_kernel<true, true>(*l->args, x);
    } else {
        gsr::WithIds<false> x;
        x.ids = *l->ids;
        if (l->variant == 1) gsr::composite_ids_kernel<false, false>(*l->args, x);
        else gsr::composite_ids_kernel<true, false>(*l->args, x);
    }
}
}  // namespace

// One persistent block renders every tile of the full frame in natural ticket order.  variant 1: uncontracted.  motion: also run the
// motion variant (vp / prev_vp and the instance tables as in tests/motion_reference/motion_emu.cpp; motion_out W*H*2).  ids_out: W*H*2.
// warp_inst: the instance of every drawn warp, or nullptr without instances.  Returns 0, or 1 if a tile was left out.
extern "C" int emu_composite_ids(int variant, int motion, const void *records, const uint32_t *values, const uint32_t *bounds, float *out_rgba,
                                 float *depth_out, float *motion_out, uint32_t *ids_out, const float *scene_depth, const float *vp,
                                 const float *prev_vp, int width, int height, float heatmap_factor, const uint32_t *warp_inst, const void *desc,
                                 const float *prev_xf, const float *plane0, float model_scale, unsigned long long *staged_out) {
    const int tiles_x = (width + 15) / 16, tiles_y = (height + 15) / 16;
    gsr::FrameState frame;
    memset(&frame, 0, sizeof frame);
    gsr::CompositeArgs a;
    memset(&a, 0, sizeof a);
    a.records = static_cast<const float4 *>(records);
    a.values = values;
    a.bounds = reinterpret_cast<const uint2 *>(bounds);
    a.out = reinterpret_cast<float4 *>(out_rgba);
    a.width = width; a.height = height; a.tiles_x = tiles_x;
    a.tile_begin = 0; a.row_step = 1; a.num_tiles = tiles_x * tiles_y;
    a.heatmap_factor = heatmap_factor; a.target_tile_id = 0xFFFFFFFFu;
    float4 pick;
    a.pick = &pick;
    a.frame = &frame; a.count_staged = 1;
    a.ctas_per_sm = 1; a.sm_count = 1; a.contract = variant == 1 ? 0 : 1;
    a.view_z[0] = vp[2]; a.view_z[1] = vp[6]; a.view_z[2] = vp[10]; a.view_z[3] = vp[14];
    a.scene_depth = scene_depth; a.depth_out = depth_out;
    gsr::MotionArgs mo;
    memset(&mo, 0, sizeof mo);
    if (motion) {
        memcpy(mo.vp, vp, sizeof mo.vp);
        memcpy(mo.prev_vp, prev_vp, sizeof mo.prev_vp);
        mo.fw = (float)(width - 1); mo.fh = (float)(height - 1);
        mo.motion_out = motion_out;
        mo.warp_inst = warp_inst; mo.desc = static_cast<const gsr::InstanceDesc *>(desc); mo.prev_xf = prev_xf;
        mo.plane0 = reinterpret_cast<const float4 *>(plane0); mo.model_scale = model_scale;
    }
    gsr::SplatIdArgs ids;
    ids.ids_out = ids_out; ids.warp_inst = warp_inst;
    IdLaunch l{&a, &mo, &ids, variant, motion};
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(128, 1, 1), &id_body, &l);
    if (staged_out) *staged_out = frame.staged;
    return frame.comp_head >= (uint32_t)a.num_tiles ? 0 : 1;
}
