// selection_emu.cpp -- the splat-selection kernels compiled for the CPU on top of tests/kernel_emu: the CUT = true projection kernels with
// splat masks, and the selection kernels of selection.cu.  TEST INFRASTRUCTURE: built by tests/test_splat_selection.py.
#include "../kernel_emu/kernel_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }   // blocks run one at a time
#include "../../godotgaussiansplatting_b200/csrc/selection.cu"

namespace {
struct SelLaunch { gsr::ProjectionArgs a; gsr::InstanceArgs ia; gsr::CutParams ct; };
template <bool INST, int B, bool ORTHO, bool AA>
void sel_body(void *p) {
    SelLaunch *l = static_cast<SelLaunch *>(p);
    gsr::projection_kernel<INST, B, ORTHO, AA, false, true>(l->a, l->ia, gsr::DepthArgs{nullptr}, l->ct);
}
template <bool INST, bool ORTHO, bool AA>
void (*pick_bands(int bands))(void *) {
    switch (bands) {
        case 1: return &sel_body<INST, 1, ORTHO, AA>;
        case 2: return &sel_body<INST, 2, ORTHO, AA>;
        case 3: return &sel_body<INST, 3, ORTHO, AA>;
        case 4: return &sel_body<INST, 4, ORTHO, AA>;
        default: return nullptr;
    }
}
template <bool INST>
void (*pick_variant(int bands, bool ortho, bool aa))(void *) {
    if (ortho) return aa ? pick_bands<INST, true, true>(bands) : pick_bands<INST, true, false>(bands);
    return aa ? pick_bands<INST, false, true>(bands) : pick_bands<INST, false, false>(bands);
}
struct RegionLaunch { gsr::SelectArgs a; };
template <int KIND>
void region_body(void *p) { gsr::select_region_kernel<KIND>(static_cast<RegionLaunch *>(p)->a); }
}  // namespace

// projection_kernel<instanced, bands, ortho, v > 0, false, true> with the cutout set `cutouts` (a CutoutArgs or null) and the masks.
extern "C" long long emu_selection_projection(int instanced, int bands, int ortho, float v, const void *soa, unsigned long long plane_stride,
                                              unsigned num_splats, const float *vp, const void *uniforms32, int sh_bulk_min, void *records,
                                              uint32_t *keys, uint32_t *values, unsigned capacity, unsigned *visible_out, int *last_tile_out,
                                              const float *inst_frame, const void *inst_desc, const uint32_t *warp_inst, const void *cutouts,
                                              const uint32_t *hidden, const uint32_t *selected, float keep, const float *add, int highlight) {
    SelLaunch l;
    gsr::ProjectionArgs &pa = l.a;
    memset(&pa, 0, sizeof pa);
    pa.soa = static_cast<const float4 *>(soa); pa.plane_stride = plane_stride; pa.num_splats = num_splats;
    memcpy(pa.vp, vp, sizeof pa.vp);
    memcpy(&pa.u, uniforms32, sizeof pa.u);
    {   // render_enqueue's frame constants
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
    pa.sh_bulk_min = sh_bulk_min;
    pa.aa_variance = v;
    const unsigned blocks = gsr::projection_num_blocks(num_splats);
    gsr::FrameState fs;
    memset(&fs, 0, sizeof fs);
    std::vector<unsigned long long> lookback(blocks ? blocks : 1, 0ull);
    pa.records = static_cast<float4 *>(records); pa.keys = keys; pa.values = values; pa.capacity = capacity;
    pa.lookback = lookback.data(); pa.frame = &fs;
    l.ia.frame = inst_frame; l.ia.desc = static_cast<const gsr::InstanceDesc *>(inst_desc); l.ia.warp_inst = warp_inst;
    memset(&l.ct.set, 0, sizeof l.ct.set);
    if (cutouts) memcpy(&l.ct.set, cutouts, sizeof l.ct.set);
    l.ct.masks.hidden = hidden; l.ct.masks.selected = selected;
    l.ct.masks.keep = keep;
    for (int i = 0; i < 3; ++i) l.ct.masks.add[i] = add[i];
    l.ct.masks.highlight = highlight ? 1u : 0u;
    void (*body)(void *) = instanced ? pick_variant<true>(bands, ortho != 0, v > 0.0f) : pick_variant<false>(bands, ortho != 0, v > 0.0f);
    if (!body) return -1;
    if (blocks) run_blocks(blocks, (unsigned)gsr::PROJ_THREADS, body, &l);
    if (visible_out) *visible_out = fs.visible;
    if (last_tile_out) *last_tile_out = fs.last_tile_plus1 - 1;
    return (long long)fs.dup_total;
}

// select_region_kernel<kind> over every word: first / count the tested range, A (12) its transform or null, vp (32), fw / fh, the volume
// (12 + kind) and the polygon (n vertices).
extern "C" int emu_select_region(int kind, uint32_t *selected, const uint32_t *hidden, unsigned words, unsigned op, unsigned long long max_splats,
                                 unsigned long long first, unsigned long long count, const void *plane0, float model_scale, const float *A,
                                 const float *vp, float fw, float fh, const float *vol12, int vol_kind, unsigned n, const float *xy) {
    RegionLaunch l;
    memset(&l, 0, sizeof l);
    gsr::SelectArgs &a = l.a;
    a.selected = selected; a.hidden = hidden; a.words = words; a.op = op;
    a.max_splats = max_splats; a.first = first; a.count = count;
    a.plane0 = static_cast<const float4 *>(plane0); a.model_scale = model_scale;
    a.instanced = A != nullptr;
    if (A) memcpy(a.A, A, sizeof a.A);
    if (vp) memcpy(a.vp, vp, sizeof a.vp);
    a.fw = fw; a.fh = fh;
    if (vol12) memcpy(a.vol.m, vol12, sizeof a.vol.m);
    a.vol.kind = vol_kind;
    a.n = n;
    for (unsigned i = 0; i < n && i < (unsigned)gsr::SELECT_MAX_VERTICES; ++i) a.xy[i] = make_float2(xy[2 * i], xy[2 * i + 1]);
    const unsigned blocks = (words + 7u) / 8u;
    void (*body)(void *) = kind == 0 ? &region_body<0> : kind == 1 ? &region_body<1> : &region_body<2>;
    if (blocks) run_blocks(blocks, 256u, body, &l);
    return 0;
}
