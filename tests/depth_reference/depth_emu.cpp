// depth_emu.cpp -- composite_kernel<CONTRACT, true> (depth compositing) compiled for the CPU on top of tests/kernel_emu.
// TEST INFRASTRUCTURE: built by tests/depth_reference.py.  kernel_emu.cpp brings every kernel file of csrc/ and the CUDA shim.
#include "../kernel_emu/kernel_emu.cpp"

namespace {
struct DepthLaunch { const gsr::CompositeArgs *args; int variant; };
void depth_body(void *p) {
    const DepthLaunch *l = static_cast<const DepthLaunch *>(p);
    if (l->variant == 1) gsr::composite_kernel<false, true>(*l->args);   // GSR_FLAG_UNCONTRACTED_BLEND
    else gsr::composite_kernel<true, true>(*l->args);
}
}  // namespace

// One persistent block renders every tile of the full frame in natural ticket order.  vp: the 32-float view_proj (its view row gives
// the splats' depth); scene_depth: nullable W*H; depth_out: W*H.  Returns 0, or 1 if a tile was left out.
extern "C" int emu_composite_depth(int variant, const void *records, const uint32_t *values, const uint32_t *bounds, float *out_rgba, float *depth_out,
                                   const float *scene_depth, const float *vp, int width, int height, float heatmap_factor,
                                   unsigned long long *staged_out) {
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
    DepthLaunch l{&a, variant};
    cuda_emu::g_block_dim = cuda_emu::dim{128, 1, 1};
    glsl::run_workgroup(glsl::uvec3(0, 0, 0), glsl::uvec3(128, 1, 1), &depth_body, &l);
    if (staged_out) *staged_out = frame.staged;
    return frame.comp_head >= (uint32_t)a.num_tiles ? 0 : 1;
}
