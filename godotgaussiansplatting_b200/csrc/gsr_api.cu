// gsr_api.cu -- the C-ABI of libgsr.so (include/gsr.h): context, buffers, per-frame sequencing.
//
// Host-side counterpart of GaussianSplattingRasterizer.init_gpu / rasterize / get_splat_position /
// cleanup_gpu (util/gaussian_splatting_rasterizer.gd:65-171) and of RenderingContext
// (util/render_context.gd).  Fifteen compute dispatches with full barriers per frame in the reference
// become 1 + 5 + 1 + 1 kernel launches on one CUDA stream, with no host synchronisation on the frame path.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <stddef.h>
#include <string.h>
#include <unistd.h>

#include <new>
#include <vector>

#include "common.cuh"

namespace gsr {

static thread_local char g_last_error[512] = "";

void set_last_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof g_last_error, fmt, ap);
    va_end(ap);
}

}  // namespace gsr

using namespace gsr;

constexpr int EV_PER_FRAME = 7;

struct gsr_ctx {
    int device = 0;
    uint32_t flags = 0;
    uint64_t max_splats = 0, capacity = 0, plane_stride = 0, num_splats = 0;
    uint64_t cap_stride = 0;     // capacity rounded up to 1024 pairs: distance between the three pair buffers (keeps each 16-byte aligned)
    cudaStream_t stream = nullptr, own_stream = nullptr;
    float4 *soa = nullptr;       // soa_planes(sh_bands, sh_half) planes x plane_stride (15 for a degree-3 float store)
    int sh_bands = SH_BANDS_MAX; // SH bands the store keeps (gsr_config.sh_bands)
    int sh_degree = -1;          // render degree (gsr_set_sh_degree); -1 = the stored degree
    float aa_variance = 0.0f;    // anti-aliasing filter of the next frames (gsr_set_antialiasing); 0 = off
    int32_t depth_order = GSR_DEPTH_ORDER_KEY16;   // sort order of the next frames (gsr_set_depth_order)
    CutoutArgs cutouts = {};     // cutout set of the next frames (gsr_set_cutouts), KEEP volumes first; none = off
    // splat masks (gsr_select_*): one device allocation of [hidden | selected | scratch] words, then two 64-bit counters (and the
    // look-back words of delete / duplicate); allocated by the first call that can set a bit and kept until gsr_destroy.  on == false: not in use (the frames take their usual kernels).
    struct Masks {
        bool on = false;
        uint32_t words = 0;               // ceil(max_splats / 32)
        uint32_t *hidden = nullptr, *selected = nullptr, *scratch = nullptr;
        unsigned long long *counts = nullptr;
        unsigned long long *lookback = nullptr;   // gsr_delete_hidden / gsr_duplicate_selection: tile status words and ticket
        cudaEvent_t ids_ready = nullptr;  // gsr_select_ids with front / back overlap: the render stream's work that wrote the ID plane
        float rgb[3] = {1.0f, 0.5f, 0.0f};
        float strength = 0.5f;
    } masks;
    // store edits and snapshots (gsr_transform_selection, gsr_recolor_selection, gsr_copy_splat_store, gsr_restore_splat_store)
    float edit_last[EDIT_TRANSFORM_FLOATS] = {};   // GSR_BUF_EDIT_TRANSFORM: the constants of the last accepted transform
    float color_last[EDIT_COLOR_FLOATS] = {};      // GSR_BUF_EDIT_COLOR: the constants of the last accepted colour edit
    cudaEvent_t store_ready = nullptr;             // with front / back overlap: the render stream's work enqueued before the operation
    void *hist = nullptr;                          // gsr_splat_histogram: HIST_BUFFER_BYTES (counters, min / max keys, edges), first call
    unsigned char *hist_host = nullptr;            // its page-locked image (upload and read-back)
    // gsr_select_neighborhood: the grid's scratch (GSR_NEIGHBOR_SCRATCH_BYTES_PER_SLOT per slot, the bucket starts, a sort workspace of
    // max_splats pairs and the counters with their page-locked image), allocated by the first call and kept until gsr_destroy
    struct Neighbors {
        SortWorkspace ws;
        uint32_t *keys = nullptr, *vals = nullptr, *parent = nullptr, *size = nullptr, *start = nullptr;
        float4 *pos = nullptr;
        NeighborCounters *ctr = nullptr, *ctr_host = nullptr;
    } nb;
    // gsr_export_ply: the exported count, then the look-back words of ceil(max_splats / 256) tiles and the ticket; first call
    unsigned long long *export_words = nullptr;
    // gsr_export_compressed_ply: a sort workspace of max_splats pairs, the pairs and their ping-pong halves (16 B per slot), and the
    // bounds pass's result with its page-locked image; allocated by the first call and kept until gsr_destroy
    struct Compressed {
        SortWorkspace ws;
        uint32_t *pairs = nullptr;   // keys | vals | alt keys | alt vals, max_splats each
        CompressBounds *bounds = nullptr, *bounds_host = nullptr;
    } cply;
    float4 *records = nullptr;  // 3 float4 per splat id; two tables (consecutive frames alternate: front / back overlap)
    float4 *records2 = nullptr;
    uint32_t *keys = nullptr;    // 3 * capacity: sort input of even frames | of odd frames | ping-pong partner (rasterizer.gd:88 has two halves)
    uint32_t *vals = nullptr;    // 3 * capacity
    uint32_t *depth_words = nullptr;   // 3 * capacity like keys, allocated by the first switch to GSR_DEPTH_ORDER_VIEW_DEPTH
    uint32_t *keys_cur = nullptr, *vals_cur = nullptr;   // sorted pairs of the most recent frame
    float4 *records_cur = nullptr;                       // record table the most recent frame composited from
    // front / back overlap: the projection of frame f+1 (front: HBM-bound) runs on its own stream beside the compositor of frame f
    // (back: FMA-pipe / chain bound) when the host enqueues frames back to back (gsr_render_async).  gsr_debug_pipeline(ctx, 0) = serial.
    cudaStream_t front_stream = nullptr;
    cudaEvent_t front_gate = nullptr;    // recorded after the tile ranges of the most recent frame (nullptr: nothing to wait for)
    int overlap = -1;                    // -1 = default = off (DESIGN.md section 6)
    SortWorkspace sort;
    FrameState *ring = nullptr;  // GSR_HISTORY_FRAMES slots; slot = frame_counter % GSR_HISTORY_FRAMES
    FrameState *frame = nullptr; // slot of the most recent frame
    unsigned long long *lookback = nullptr;  // one word per projection block, cleared every frame
    uint32_t lookback_blocks = 0;
    uint64_t frame_counter = 0;
    uint2 *bounds = nullptr;     // followed in the same allocation by the compositor queue (one memset per frame)
    uint32_t *comp_order = nullptr, *comp_hint = nullptr;   // longest-chain-first ticket order of the compositor + last frame's consumed chunks
    int comp_ctas_per_sm = 2, comp_order_mode = 1, comp_max_ctas = 1, comp_sparse_per_sm = 5;   // scheduling of the compositor's persistent grid (gsr_debug_compositor_config)
    uint64_t comp_hint_key = 0;   // ownership (band, rows) the hints were recorded under: a change invalidates them
    FrameState *pick_frame = nullptr;  // queue counters of the single-tile pick launch
    ulonglong4 *trace = nullptr;       // GSR_BUF_COMPOSITOR_TRACE (debug; allocated by gsr_debug_enable_trace)
    uint32_t *trace_count = nullptr;
    uint32_t trace_cap = 0;
    float4 *fb = nullptr, *fb_ext = nullptr;
    // depth compositing (gsr_set_depth_compositing): caller-owned W*H float planes; depth_out == nullptr = off
    const float *scene_depth = nullptr;
    float *depth_out = nullptr;
    // motion vectors (gsr_set_motion_vectors, with depth compositing): caller-owned W*H float2 plane; nullptr = off
    float *motion_out = nullptr;
    // splat IDs (gsr_set_splat_ids, with depth compositing): caller-owned W*H uint32 pair plane; nullptr = off
    uint32_t *ids_out = nullptr;
    // splat contribution (gsr_set_splat_contribution, with depth compositing): caller-owned max_splats records; nullptr = off.  The
    // device frame counter is allocated by the first set; contrib_epoch is the epoch of the last frame enqueued (0: none yet).
    gsr_splat_contribution *contrib = nullptr;
    uint32_t *contrib_frames = nullptr;
    uint32_t contrib_epoch = 0;
    // The camera and instance transforms of a frame, recorded for every frame enqueued by gsr_render* (motion on or off): `mot_last` is
    // the last enqueued frame's, the previous state of the next frame; `mot_used` is the previous state the last frame was enqueued
    // with (gsr_render's re-render of an overflowed frame uses it again).  valid == false: no previous frame (first frame, gsr_resize,
    // gsr_reset_motion), the frame is its own previous state.
    struct MotionState {
        bool valid = false;
        float vp[32] = {};
        std::vector<uint64_t> range;   // the instance layout, 2 per instance (empty: no instances)
        std::vector<float> to_frame;   // INSTANCE_PREV_FLOATS per instance
    };
    MotionState mot_last, mot_used;
    float4 *pick_strip = nullptr;   // 16 pixel rows: where gsr_pick's default-path re-dispatch writes while depth compositing is on
    float4 *fb2 = nullptr;                       // second frame for pipelined read-back (gsr_render_async)
    void *stage[2] = {nullptr, nullptr};         // converted copies of the two frames (GSR_OUT_* other than RGBA32F), lazily allocated (16 B/pixel)
    float4 *fb_last = nullptr;                   // frame written by the most recent render
    cudaStream_t copy_stream = nullptr;          // D2H read-back overlaps the next frame's kernels
    cudaEvent_t ev_done[2] = {nullptr, nullptr}, ev_copied[2] = {nullptr, nullptr};
    bool copied_valid[2] = {false, false};
    uint64_t async_counter = 0;
    // multi-GPU peer mode: every rank's compositor stores its band straight into the presenting rank's two frames
    bool peer_mode = false, peer_opened = false;
    float4 *peer_fb[2] = {nullptr, nullptr};
    uint64_t peer_counter = 0;
    float4 *pick = nullptr;
    float4 *staging = nullptr;
    uint64_t staging_splats = 0;
    uint64_t staging_bytes = 0;  // 16 B x stored planes x staging_splats (at least one 240-byte AoS struct)
    uint32_t *unsorted_keys = nullptr, *unsorted_vals = nullptr;
    uint32_t *unsorted_depth = nullptr;   // GSR_BUF_DEPTH_WORDS_UNSORTED: with keep_unsorted once depth_words exist
    bool keep_unsorted = false;
    int width = 0, height = 0, tiles_x = 0, tiles_y = 0, band_y0 = 0, band_y1 = 0;
    bool band_set = false;
    int row_mod = 1, row_rem = 0;   // cyclic tile-row ownership (gsr_set_row_interleave): fast sharded mode when row_mod > 1
    int32_t *sync_word = nullptr;   // local (then all-reduced) last occupied tile + 1
    // multi-GPU shard group (gsr_group_export / gsr_group_attach): NCCL-free frame path, see group.cu
    struct Group {
        void *arena = nullptr;            // this rank's arena: flag page | receive segments (2 parities x keys, values) | records (2 parities)
        uint64_t rx_capacity = 0;         // pairs per receive buffer (all sources together); seg_cap = rx_capacity / world
        int rank = 0, world = 0;          // world > 1 <=> attached
        char *peer_arena[GROUP_MAX] = {};    // every rank's arena (peer pointers)
        GroupFlags *flags[GROUP_MAX] = {};   // every rank's flag page
        float4 *root_fb[2] = {nullptr, nullptr};  // the presenting rank's two frames
        void *opened[3 * GROUP_MAX] = {};    // IPC mappings to close
        int n_opened = 0;
        int present_rows = 0;             // 1: every rank keeps its rows in its own frames and reads them back itself (gsr_group_set_present)
        uint32_t seq = 0;                 // frames rendered by the group so far (lockstep on all ranks)
        uint64_t slice = 0;               // splats per rank (256-aligned)
        uint32_t seg_cap = 0;             // pairs one source may send to one destination per frame
    } grp;
    cudaEvent_t *ev = nullptr;   // [GSR_HISTORY_FRAMES][EV_PER_FRAME]: front start, front end | back start, received, sorted, ranges, rendered
    // dynamic duplicate capacity (replaces the reference's static 10 x N, rasterizer.gd:79 "FIXME: This should not be a static
    // value!"): every frame's M travels to a pinned host mirror without a host sync; the capacity grows ahead of need
    FrameState *host_ring = nullptr;       // pinned mirror of `ring`
    cudaEvent_t *ev_stat = nullptr;        // [GSR_HISTORY_FRAMES] recorded after the slot's copy
    uint64_t stats_polled = 0;             // frames whose mirror has been examined
    uint64_t m_high = 0;                   // high-water mark of M over the examined frames
    uint64_t capacity_max = 0;
    bool ev_valid = false;
    uint32_t last_launches = 0;
    int sm_count = 0;
    uint64_t dup_factor = 10;
    uint64_t rec_entries = 0;    // ids each record table holds: max(max_splats, D of the largest instance layout so far)
    uint32_t lookback_cap = 0;   // projection links the look-back words cover (scatter links come on top)
    // splat instances (gsr_set_instances); inst_n == 0: off
    struct Instances {
        uint32_t n = 0;                  // instances of the current layout
        uint64_t drawn = 0;              // D
        uint64_t *range = nullptr;       // [2n] first, count (the layout)
        float *xf = nullptr;             // [24n] A|t as given, B|u = the inverse (host copy; GSR_BUF_INSTANCES)
        gsr_instance_appearance *app = nullptr;   // [n] gsr_set_instance_appearance as given; null: every instance at the default
        InstanceDesc *desc = nullptr;    // device [n]
        uint32_t *warps = nullptr;       // device: instance of every drawn warp of the projection grid
        float *frame = nullptr;          // device [2][cap][INSTANCE_FRAME_FLOATS]: this frame's constants, by frame parity; then
                                         // [2][cap][INSTANCE_APPEARANCE_FLOATS]: this frame's appearance rows, by frame parity; then
                                         // [2][cap][INSTANCE_PREV_FLOATS]: the previous transforms of its motion vectors, by parity
        uint32_t cap = 0;                // instances the device tables and the ring are sized for
        float *ring = nullptr;           // mapped page-locked [GSR_INSTANCE_RING][cap][24 + 8 + 12]: per slot the transforms of one
                                         // frame ([cap][24]), then its appearance rows ([cap][8]), then its previous transforms ([cap][12])
        float *ring_dev = nullptr;
        cudaEvent_t ev[GSR_INSTANCE_RING] = {};   // recorded after the prepare kernel that read the slot
        bool ev_used[GSR_INSTANCE_RING] = {};
        uint64_t seq = 0;                // instanced frames enqueued
    } inst;
};

struct gsr_sorter {
    int device = 0;
    SortWorkspace ws;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool timed = false;
};

namespace {

// one slot of the instance ring, per instance of the capacity: the transforms, the appearance rows, the previous transforms
constexpr size_t INSTANCE_SLOT_FLOATS = INSTANCE_XFORM_FLOATS + INSTANCE_APPEARANCE_FLOATS + INSTANCE_PREV_FLOATS;

// the device appearance rows of the frames of parity `half` (they follow the two tables of per-frame constants)
float *instance_appearance_table(const gsr_ctx::Instances &I, int half) {
    return I.frame + 2ull * I.cap * INSTANCE_FRAME_FLOATS + (size_t)half * I.cap * INSTANCE_APPEARANCE_FLOATS;
}

// the device previous transforms of the frames of parity `half` (motion vectors; they follow the appearance rows)
float *instance_prev_table(const gsr_ctx::Instances &I, int half) {
    return I.frame + 2ull * I.cap * (INSTANCE_FRAME_FLOATS + INSTANCE_APPEARANCE_FLOATS) + (size_t)half * I.cap * INSTANCE_PREV_FLOATS;
}

// The stored appearance as the kernels read it (common.cuh): tint, opacity, live_k = min(count_k, draw_count) or 0 at opacity 0, pad.
void instance_appearance_rows(const gsr_ctx::Instances &I, float *rows) {
    for (uint32_t k = 0; k < I.n; ++k) {
        const gsr_instance_appearance &p = I.app[k];
        const uint64_t count = I.range[2 * k + 1];
        const uint32_t live = p.opacity == 0.0f ? 0u : (uint32_t)(p.draw_count < count ? p.draw_count : count);
        float *r = rows + (size_t)k * INSTANCE_APPEARANCE_FLOATS;
        r[0] = p.tint[0]; r[1] = p.tint[1]; r[2] = p.tint[2]; r[3] = p.opacity;
        memcpy(r + 4, &live, sizeof live);
        r[5] = r[6] = r[7] = 0.0f;
    }
}

int use_device(int device) {
    GSR_CUDA_TRY(cudaSetDevice(device));
    return GSR_OK;
}

int check_device(int device) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_last_error("no CUDA device available (%s); libgsr has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "count=0");
        return GSR_ERR_CUDA;
    }
    if (device < 0 || device >= count) {
        set_last_error("device ordinal %d out of range [0,%d)", device, count);
        return GSR_ERR_INVALID;
    }
    cudaDeviceProp prop;
    GSR_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_last_error("device %d is sm_%d%d; libgsr is built for sm_90a only", device, prop.major, prop.minor);
        return GSR_ERR_CUDA;
    }
    return GSR_OK;
}

void group_detach(gsr_ctx *c) {
    if (c->front_stream) cudaStreamSynchronize(c->front_stream);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    for (int i = 0; i < c->grp.n_opened; ++i) cudaIpcCloseMemHandle(c->grp.opened[i]);
    c->grp.n_opened = 0;
    if (c->grp.world > 1) { c->row_mod = 1; c->row_rem = 0; }
    c->grp.world = 0; c->grp.rank = 0; c->grp.seq = 0; c->grp.present_rows = 0;
    c->grp.root_fb[0] = c->grp.root_fb[1] = nullptr;
}

float4 *framebuffer(gsr_ctx *c) { return c->fb_ext ? c->fb_ext : (c->fb_last ? c->fb_last : c->fb); }

// SH bands the next frame evaluates, and whether the context stores or renders fewer than 4 (single-context only, like depth compositing)
// (GSR_FLAG_SH_HALF: a binary16 store is single-context only too -- the sharded, scatter and band kernels read float stores)
int render_bands(const gsr_ctx *c) { return c->sh_degree < 0 ? c->sh_bands : c->sh_degree + 1; }
bool sh_half(const gsr_ctx *c) { return (c->flags & GSR_FLAG_SH_HALF) != 0u; }
bool reduced_sh(const gsr_ctx *c) { return c->sh_bands < SH_BANDS_MAX || render_bands(c) < SH_BANDS_MAX || sh_half(c); }
bool view_depth_order(const gsr_ctx *c) { return c->depth_order == GSR_DEPTH_ORDER_VIEW_DEPTH; }
bool cutouts_on(const gsr_ctx *c) { return c->cutouts.n_keep + c->cutouts.n_remove != 0u; }

// The single-context rule (gsr.h, "Single-context features") is decided by these two functions only: a call that would shard the
// context refuses while single_context_feature() names a feature, and a call that would turn a feature on refuses while sharded().
// So no frame of a shard group, of peer framebuffers, of a partial band or of row interleave has any of these features.
//
// The reason text of the first feature that is on, or nullptr.  for_group_export skips depth compositing and instances:
// gsr_group_export accepts them, and only gsr_group_attach with world > 1 refuses them.
const char *single_context_feature(const gsr_ctx *c, bool for_group_export) {
    if (!for_group_export && c->depth_out) return "depth compositing is on";
    if (!for_group_export && c->inst.n) return "instances are set";
    if (reduced_sh(c)) return "SH stored as binary16, or stored or rendered below degree 3";
    if (c->aa_variance > 0.0f) return "anti-aliasing is on";
    if (view_depth_order(c)) return "depth order is on";
    if (cutouts_on(c)) return "cutouts are set";
    if (c->masks.on) return "splat masks are in use";
    return nullptr;
}

// Whether the context is sharded: an attached shard group, exported or imported peer framebuffers, row interleave, or a band short of
// the full frame (there is no band before gsr_resize).
bool sharded(const gsr_ctx *c) {
    const bool partial = c->tiles_y != 0 && !(c->band_y0 == 0 && c->band_y1 == c->tiles_y);
    return c->grp.world > 1 || c->peer_mode || c->row_mod > 1 || partial;
}

constexpr char SINGLE_CONTEXT_ONLY[] = "single-context only (no group, peer framebuffers, partial band or row interleave)";

// The depth-order buffers at the current capacity: the depth words (3 * cap_stride), GSR_BUF_DEPTH_WORDS_UNSORTED while unsorted pairs
// are kept, and the sorter's depth-order workspace.  On failure nothing is left half allocated.
int alloc_depth_order(gsr_ctx *c) {
    if (!c->depth_words) {
        uint32_t *dw = nullptr;
        GSR_CUDA_TRY(cudaMalloc((void **)&dw, sizeof(uint32_t) * 3ull * c->cap_stride));
        int rc = sort_workspace_enable_depth(c->sort);
        if (rc) { cudaFree(dw); return rc; }
        c->depth_words = dw;
    }
    if (c->unsorted_keys && !c->unsorted_depth) GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_depth, sizeof(uint32_t) * c->capacity));
    return GSR_OK;
}

void free_neighbors(gsr_ctx::Neighbors &nb) {
    sort_workspace_destroy(nb.ws);
    cudaFree(nb.keys); cudaFree(nb.vals); cudaFree(nb.parent); cudaFree(nb.size); cudaFree(nb.start); cudaFree(nb.pos); cudaFree(nb.ctr);
    if (nb.ctr_host) cudaFreeHost(nb.ctr_host);
    nb = gsr_ctx::Neighbors();
}

// gsr_select_neighborhood's scratch for max_splats slots; on failure nothing is left allocated
int alloc_neighbors(gsr_ctx *c, const char *where) {
    gsr_ctx::Neighbors &nb = c->nb;
    if (nb.ctr) return GSR_OK;
    const uint64_t m = c->max_splats, buckets = 1ull << neighbor_bucket_bits(m);
    int rc = sort_workspace_create(nb.ws, m, /*need_alt_buffers=*/false);
    cudaError_t e = cudaSuccess;
    if (!rc) {
        e = cudaMalloc((void **)&nb.keys, sizeof(uint32_t) * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.vals, sizeof(uint32_t) * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.parent, sizeof(uint32_t) * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.size, sizeof(uint32_t) * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.pos, sizeof(float4) * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.start, sizeof(uint32_t) * (buckets + 1));
        if (e == cudaSuccess) e = cudaMalloc((void **)&nb.ctr, sizeof(NeighborCounters));
        if (e == cudaSuccess) e = cudaMallocHost((void **)&nb.ctr_host, sizeof(NeighborCounters));
    }
    if (rc || e != cudaSuccess) {
        free_neighbors(nb);
        if (e != cudaSuccess) {
            set_last_error("%s: grid scratch for %llu slots -> %s", where, (unsigned long long)m, cudaGetErrorString(e));
            rc = e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
        return rc;
    }
    return GSR_OK;
}

void free_compressed(gsr_ctx::Compressed &cp) {
    sort_workspace_destroy(cp.ws);
    cudaFree(cp.pairs); cudaFree(cp.bounds);
    if (cp.bounds_host) cudaFreeHost(cp.bounds_host);
    cp = gsr_ctx::Compressed();
}

// gsr_export_compressed_ply's scratch for max_splats slots; on failure nothing is left allocated
int alloc_compressed(gsr_ctx *c, const char *where) {
    gsr_ctx::Compressed &cp = c->cply;
    if (cp.bounds_host) return GSR_OK;
    const uint64_t m = c->max_splats;
    int rc = sort_workspace_create(cp.ws, m, /*need_alt_buffers=*/false);
    cudaError_t e = cudaSuccess;
    if (!rc) {
        e = cudaMalloc((void **)&cp.pairs, sizeof(uint32_t) * 4ull * m);
        if (e == cudaSuccess) e = cudaMalloc((void **)&cp.bounds, sizeof(CompressBounds));
        if (e == cudaSuccess) e = cudaMallocHost((void **)&cp.bounds_host, sizeof(CompressBounds));
    }
    if (rc || e != cudaSuccess) {
        free_compressed(cp);
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_last_error("%s: sort scratch for %llu slots -> %s", where, (unsigned long long)m, cudaGetErrorString(e));
            rc = e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
        return rc;
    }
    return GSR_OK;
}

void free_ctx(gsr_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->front_stream) { cudaStreamSynchronize(c->front_stream); cudaStreamDestroy(c->front_stream); }
    cudaFree(c->soa); cudaFree(c->records); cudaFree(c->records2); cudaFree(c->keys); cudaFree(c->vals);
    sort_workspace_destroy(c->sort);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    if (c->peer_opened) { cudaIpcCloseMemHandle(c->peer_fb[0]); cudaIpcCloseMemHandle(c->peer_fb[1]); }
    cudaFree(c->stage[0]); cudaFree(c->stage[1]);
    cudaFree(c->ring); cudaFree(c->lookback); cudaFree(c->bounds); cudaFree(c->comp_order); cudaFree(c->comp_hint); cudaFree(c->pick_frame); cudaFree(c->fb); cudaFree(c->fb2); cudaFree(c->pick); cudaFree(c->staging); cudaFree(c->pick_strip);
    for (int i = 0; i < 2; ++i) { if (c->ev_done[i]) cudaEventDestroy(c->ev_done[i]); if (c->ev_copied[i]) cudaEventDestroy(c->ev_copied[i]); }
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    cudaFree(c->sync_word);
    for (int i = 0; i < c->grp.n_opened; ++i) cudaIpcCloseMemHandle(c->grp.opened[i]);
    cudaFree(c->grp.arena);
    cudaFree(c->unsorted_keys); cudaFree(c->unsorted_vals); cudaFree(c->trace); cudaFree(c->trace_count);
    cudaFree(c->depth_words); cudaFree(c->unsorted_depth);
    cudaFree(c->inst.desc); cudaFree(c->inst.warps); cudaFree(c->inst.frame);
    cudaFree(c->masks.counts);   // the base of the mask allocation
    if (c->masks.ids_ready) cudaEventDestroy(c->masks.ids_ready);
    if (c->store_ready) cudaEventDestroy(c->store_ready);
    cudaFree(c->hist);
    cudaFree(c->export_words);
    cudaFree(c->contrib_frames);
    free_compressed(c->cply);
    free_neighbors(c->nb);
    if (c->hist_host) cudaFreeHost(c->hist_host);
    if (c->inst.ring) cudaFreeHost(c->inst.ring);
    for (int i = 0; i < GSR_INSTANCE_RING; ++i) if (c->inst.ev[i]) cudaEventDestroy(c->inst.ev[i]);
    delete[] c->inst.range; delete[] c->inst.xf; delete[] c->inst.app;
    if (c->ev) {
        for (int i = 0; i < GSR_HISTORY_FRAMES * EV_PER_FRAME; ++i) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
        delete[] c->ev;
    }
    if (c->ev_stat) {
        for (int i = 0; i < GSR_HISTORY_FRAMES; ++i) if (c->ev_stat[i]) cudaEventDestroy(c->ev_stat[i]);
        delete[] c->ev_stat;
    }
    if (c->host_ring) cudaFreeHost(c->host_ring);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

}  // namespace

extern "C" {

GSR_API const char *gsr_error_string(int code) {
    switch (code) {
        case GSR_OK: return "ok";
        case GSR_ERR_INVALID: return "invalid argument";
        case GSR_ERR_CUDA: return "CUDA failure or no usable sm_90 device (no CPU fallback exists)";
        case GSR_ERR_OOM: return "device out of memory";
        case GSR_ERR_STATE: return "call order violated";
        case GSR_ERR_OVERFLOW: return "duplicate list exceeded capacity";
        default: return "unknown error";
    }
}
GSR_API const char *gsr_last_error(void) { return g_last_error; }
GSR_API const char *gsr_version(void) { return "gsr 0.1.0 (sm_90a)"; }
GSR_API int gsr_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

GSR_API int gsr_create(const gsr_config *cfg, gsr_ctx **out) {
    if (!cfg || !out || cfg->max_splats == 0) { set_last_error("gsr_create: null config/out or max_splats == 0"); return GSR_ERR_INVALID; }
    *out = nullptr;
    int rc = check_device(cfg->device);
    if (rc) return rc;
    if ((rc = use_device(cfg->device))) return rc;
    if (cfg->max_splats >= (1ull << 32) - 256ull) { set_last_error("max_splats must be < 2^32-256"); return GSR_ERR_INVALID; }
    if (cfg->sh_bands > (uint32_t)SH_BANDS_MAX) { set_last_error("gsr_create: sh_bands %u > %d (degree 3)", cfg->sh_bands, SH_BANDS_MAX); return GSR_ERR_INVALID; }
    gsr_ctx *c = new (std::nothrow) gsr_ctx();
    if (!c) return GSR_ERR_OOM;
    c->device = cfg->device;
    c->flags = cfg->flags;
    if (!(c->flags & (GSR_FLAG_REFERENCE_QUIRKS | GSR_FLAG_FIXED_RANGES))) c->flags |= GSR_FLAG_REFERENCE_QUIRKS;
    c->max_splats = cfg->max_splats;
    c->sh_bands = cfg->sh_bands ? (int)cfg->sh_bands : SH_BANDS_MAX;
    const uint64_t planes = (uint64_t)soa_planes(c->sh_bands, sh_half(c));
    const uint64_t factor = cfg->dup_capacity_factor ? cfg->dup_capacity_factor : 10;  // rasterizer.gd:79
    c->dup_factor = factor;
    c->capacity_max = (1ull << 30) - 1;  // look-back words carry 30-bit counts
    c->capacity = c->max_splats * factor;
    if (c->capacity > c->capacity_max) c->capacity = c->capacity_max;
    c->plane_stride = (c->max_splats + 255ull) & ~255ull;
    cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, c->device);
    if ((rc = composite_max_ctas_per_sm(&c->comp_max_ctas))) { delete c; return rc; }

#define TRY_ALLOC(ptr, bytes)                                                                      \
    do {                                                                                           \
        cudaError_t _e = cudaMalloc((void **)&(ptr), (bytes));                                     \
        if (_e != cudaSuccess) {                                                                   \
            set_last_error("cudaMalloc(%s, %llu B) -> %s", #ptr, (unsigned long long)(bytes), cudaGetErrorString(_e)); \
            free_ctx(c);                                                                           \
            return _e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;                   \
        }                                                                                          \
    } while (0)

    cudaError_t se;
    {
        int least = 0, greatest = 0;
        cudaDeviceGetStreamPriorityRange(&least, &greatest);
        se = cudaStreamCreateWithPriority(&c->own_stream, cudaStreamNonBlocking, greatest);
    }
    if (se != cudaSuccess) { set_last_error("cudaStreamCreate -> %s", cudaGetErrorString(se)); free_ctx(c); return GSR_ERR_CUDA; }
    c->stream = c->own_stream;
    se = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
    if (se == cudaSuccess) {   // the front stream yields to the render stream wherever the host gave that one a higher priority
        int least = 0, greatest = 0;
        cudaDeviceGetStreamPriorityRange(&least, &greatest);
        se = cudaStreamCreateWithPriority(&c->front_stream, cudaStreamNonBlocking, least);
    }
    for (int i = 0; i < 2 && se == cudaSuccess; ++i) {
        se = cudaEventCreateWithFlags(&c->ev_done[i], cudaEventDisableTiming);
        if (se == cudaSuccess) se = cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming);
    }
    if (se != cudaSuccess) { set_last_error("copy stream/events -> %s", cudaGetErrorString(se)); free_ctx(c); return GSR_ERR_CUDA; }
    TRY_ALLOC(c->soa, sizeof(float4) * planes * c->plane_stride);
    TRY_ALLOC(c->records, sizeof(float4) * 3ull * c->max_splats);
    TRY_ALLOC(c->records2, sizeof(float4) * 3ull * c->max_splats);
    c->cap_stride = (c->capacity + 1023ull) & ~1023ull;
    TRY_ALLOC(c->keys, sizeof(uint32_t) * 3ull * c->cap_stride);
    TRY_ALLOC(c->vals, sizeof(uint32_t) * 3ull * c->cap_stride);
    c->keys_cur = c->keys; c->vals_cur = c->vals; c->records_cur = c->records;
    c->rec_entries = c->max_splats;
    c->lookback_blocks = projection_num_blocks((uint32_t)c->max_splats);  // one scan link per CTA
    c->lookback_cap = c->lookback_blocks;
    TRY_ALLOC(c->ring, sizeof(FrameState) * GSR_HISTORY_FRAMES);
    TRY_ALLOC(c->lookback, sizeof(unsigned long long) * ((size_t)c->lookback_blocks + 2u * GROUP_MAX * GROUP_MAX));  // scatter mode: (N/G/256 + 1) x G links
    c->frame = c->ring;
    TRY_ALLOC(c->pick, sizeof(float4));
    TRY_ALLOC(c->sync_word, sizeof(int32_t));
    c->staging_splats = c->max_splats < (1ull << 18) ? c->max_splats : (1ull << 18);
    c->staging_bytes = sizeof(float4) * planes * c->staging_splats;
    if (c->staging_bytes < 240ull) c->staging_bytes = 240ull;
    TRY_ALLOC(c->staging, c->staging_bytes);
#undef TRY_ALLOC
    rc = sort_workspace_create(c->sort, c->capacity, /*need_alt_buffers=*/false);
    if (rc) { free_ctx(c); return rc; }
    c->ev = new (std::nothrow) cudaEvent_t[GSR_HISTORY_FRAMES * EV_PER_FRAME]();
    if (!c->ev) { free_ctx(c); return GSR_ERR_OOM; }
    for (int i = 0; i < GSR_HISTORY_FRAMES * EV_PER_FRAME; ++i) {
        if (cudaEventCreate(&c->ev[i]) != cudaSuccess) { set_last_error("cudaEventCreate failed"); free_ctx(c); return GSR_ERR_CUDA; }
    }
    c->ev_stat = new (std::nothrow) cudaEvent_t[GSR_HISTORY_FRAMES]();
    if (!c->ev_stat) { free_ctx(c); return GSR_ERR_OOM; }
    for (int i = 0; i < GSR_HISTORY_FRAMES; ++i) {
        if (cudaEventCreateWithFlags(&c->ev_stat[i], cudaEventDisableTiming) != cudaSuccess) { set_last_error("cudaEventCreate failed"); free_ctx(c); return GSR_ERR_CUDA; }
    }
    if (cudaHostAlloc((void **)&c->host_ring, sizeof(FrameState) * GSR_HISTORY_FRAMES, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
        set_last_error("cudaHostAlloc(frame mirror) failed"); c->host_ring = nullptr; free_ctx(c); return GSR_ERR_OOM;
    }
    memset(c->host_ring, 0, sizeof(FrameState) * GSR_HISTORY_FRAMES);
    cudaMemsetAsync(c->soa, 0, sizeof(float4) * planes * c->plane_stride, c->stream);
    cudaMemsetAsync(c->records, 0, sizeof(float4) * 3ull * c->max_splats, c->stream);
    cudaMemsetAsync(c->records2, 0, sizeof(float4) * 3ull * c->max_splats, c->stream);
    cudaMemsetAsync(c->pick, 0, sizeof(float4), c->stream);
    cudaMemsetAsync(c->sync_word, 0, sizeof(int32_t), c->stream);
    cudaMemsetAsync(c->ring, 0, sizeof(FrameState) * GSR_HISTORY_FRAMES, c->stream);
    // load every kernel now: with lazy module loading a FIRST launch may have to synchronise with the device, which must not
    // happen on the frame path (and would deadlock a group whose ranks share one process: a wait kernel spins meanwhile)
    if ((rc = preload_group_kernels()) || (rc = preload_projection_kernels()) || (rc = preload_sort_kernels()) || (rc = preload_ranges_kernels()) ||
        (rc = preload_ingest_kernels()) || (rc = preload_present_kernels()) || (rc = preload_composite_kernels()) || (rc = preload_selection_kernels()) ||
        (rc = preload_neighbor_kernels()) || (rc = preload_compressed_kernels()) || (sh_half(c) && (rc = preload_projection_half_kernels()))) { free_ctx(c); return rc; }
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_last_error("init sync -> %s", cudaGetErrorString(e)); free_ctx(c); return GSR_ERR_CUDA; }
    *out = c;
    return GSR_OK;
}

GSR_API int gsr_destroy(gsr_ctx *ctx) {
    free_ctx(ctx);
    return GSR_OK;
}

GSR_API int gsr_set_stream(gsr_ctx *c, void *cuda_stream) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
    c->ev_valid = false; c->front_gate = nullptr;
    return GSR_OK;
}

GSR_API int gsr_upload_splats_aos(gsr_ctx *c, const float *splat60, uint64_t first, uint64_t count) {
    if (!c || (!splat60 && count)) return GSR_ERR_INVALID;
    if (count > c->max_splats || first > c->max_splats - count) { set_last_error("upload range [%llu,%llu) exceeds max_splats %llu", (unsigned long long)first, (unsigned long long)(first + count), (unsigned long long)c->max_splats); return GSR_ERR_INVALID; }
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));   // a projection in flight reads the planes this call rewrites
    const uint64_t per = c->staging_bytes / 240ull;           // 60-float structs per chunk (staging_splats for a degree-3 store)
    uint64_t done = 0;
    while (done < count) {
        const uint64_t m = (count - done) < per ? (count - done) : per;
        GSR_CUDA_TRY(cudaMemcpyAsync(c->staging, splat60 + (done * 60ull), m * 240ull, cudaMemcpyHostToDevice, c->stream));
        if ((rc = launch_aos_to_soa(c->staging, m, c->soa, c->plane_stride, first + done, soa_planes(c->sh_bands, sh_half(c)), c->stream, sh_half(c)))) return rc;
        done += m;
    }
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));  // the caller may free/reuse splat60 (buffer_update semantics)
    if (first + count > c->num_splats) c->num_splats = first + count;
    return GSR_OK;
}

static int upload_ply(gsr_ctx *c, const float *ply, const gsr_ply_layout &lay, uint64_t first, uint64_t count, float creation_time,
                      int32_t filter_3d = -1) {
    if (count > c->max_splats || first > c->max_splats - count) { set_last_error("upload range [%llu,%llu) exceeds max_splats %llu", (unsigned long long)first, (unsigned long long)(first + count), (unsigned long long)c->max_splats); return GSR_ERR_INVALID; }
    int rc = use_device(c->device);
    if (rc) return rc;
    const uint32_t nprops = lay.nprops;
    const uint64_t staging_floats = c->staging_bytes / sizeof(float);  // the AoS staging buffer, reused for raw vertices
    const uint64_t per = staging_floats / nprops;
    if (per == 0) { set_last_error("gsr_upload_ply: staging buffer too small"); return GSR_ERR_INVALID; }
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));   // a projection in flight reads the planes this call rewrites
    uint64_t done = 0;
    while (done < count) {
        const uint64_t m = (count - done) < per ? (count - done) : per;
        GSR_CUDA_TRY(cudaMemcpyAsync(c->staging, ply + done * nprops, m * nprops * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if ((rc = launch_ply_to_soa(reinterpret_cast<const float *>(c->staging), lay, m, creation_time, c->soa, c->plane_stride, first + done,
                                    soa_planes(c->sh_bands, sh_half(c)), c->stream, filter_3d, sh_half(c)))) return rc;
        done += m;
    }
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (first + count > c->num_splats) c->num_splats = first + count;
    return GSR_OK;
}

GSR_API int gsr_upload_ply_raw(gsr_ctx *c, const float *ply, uint32_t nprops, uint64_t first, uint64_t count, float creation_time) {
    if (!c || (!ply && count)) return GSR_ERR_INVALID;
    if (nprops < 62 || nprops > 256) { set_last_error("gsr_upload_ply_raw: %u properties; need the 62 standard 3DGS floats (x..rot_3) first", nprops); return GSR_ERR_INVALID; }
    gsr_ply_layout lay = PLY_LAYOUT_3DGS;
    lay.nprops = nprops;
    return upload_ply(c, ply, lay, first, count, creation_time);
}

static int check_ply_layout(const gsr_ply_layout *layout) {
    if (!layout) { set_last_error("gsr_upload_ply: NULL layout"); return GSR_ERR_INVALID; }
    const gsr_ply_layout &L = *layout;
    if (L.nprops < 1 || L.nprops > 256) { set_last_error("gsr_upload_ply: nprops %u outside 1..256", L.nprops); return GSR_ERR_INVALID; }
    if (L.sh_degree > 3) { set_last_error("gsr_upload_ply: sh_degree %u > 3", L.sh_degree); return GSR_ERR_INVALID; }
    if ((L.sh_degree == 0) != (L.f_rest < 0)) { set_last_error("gsr_upload_ply: f_rest %d does not match sh_degree %u (-1 iff degree 0)", L.f_rest, L.sh_degree); return GSR_ERR_INVALID; }
    const int64_t rest = 3ll * ((int64_t)(L.sh_degree + 1) * (L.sh_degree + 1) - 1);
    const struct { const char *name; int32_t at; int64_t len; } groups[] = {
        {"x", L.x, 3}, {"f_dc", L.f_dc, 3}, {"f_rest", L.f_rest, rest}, {"opacity", L.opacity, 1}, {"scale", L.scale, 3}, {"rot", L.rot, 4}};
    for (const auto &g : groups) {
        if (g.len == 0) continue;   // f_rest of a degree-0 file
        if (g.at < 0 || (int64_t)g.at + g.len > (int64_t)L.nprops) {
            set_last_error("gsr_upload_ply: %s at %d (+%lld floats) does not fit %u properties", g.name, g.at, (long long)g.len, L.nprops);
            return GSR_ERR_INVALID;
        }
    }
    return GSR_OK;
}

GSR_API int gsr_upload_ply(gsr_ctx *c, const float *ply, const gsr_ply_layout *layout, uint64_t first, uint64_t count, float creation_time) {
    if (!c || (!ply && count)) return GSR_ERR_INVALID;
    const int rc = check_ply_layout(layout);
    if (rc) return rc;
    return upload_ply(c, ply, *layout, first, count, creation_time);
}

GSR_API int gsr_upload_ply_filtered(gsr_ctx *c, const float *ply, const gsr_ply_layout *layout, int32_t filter_3d, uint64_t first, uint64_t count,
                                    float creation_time) {
    if (!c || (!ply && count)) return GSR_ERR_INVALID;
    const int rc = check_ply_layout(layout);
    if (rc) return rc;
    if (filter_3d < -1 || filter_3d >= (int32_t)layout->nprops) {
        set_last_error("gsr_upload_ply_filtered: filter_3d %d outside -1..%u", filter_3d, layout->nprops - 1);
        return GSR_ERR_INVALID;
    }
    return upload_ply(c, ply, *layout, first, count, creation_time, filter_3d);
}

GSR_API int gsr_resize(gsr_ctx *c, int32_t width, int32_t height) {
    if (!c || width < 1 || height < 1) { set_last_error("gsr_resize: bad size %dx%d", width, height); return GSR_ERR_INVALID; }
    const int tx = (width + TILE - 1) / TILE, ty = (height + TILE - 1) / TILE;
    if ((int64_t)tx * ty > 65536) {  // tile id must fit the 16 key bits above the depth code (gsplat_projection.glsl:222)
        set_last_error("gsr_resize: %d tiles exceed the 16-bit tile id of the sort key", tx * ty);
        return GSR_ERR_INVALID;
    }
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->front_gate = nullptr;
    c->width = c->height = c->tiles_x = c->tiles_y = 0;  // a failure below leaves the context in the "before gsr_resize" state
    cudaFree(c->bounds); c->bounds = nullptr;
    cudaFree(c->comp_order); c->comp_order = nullptr;
    cudaFree(c->comp_hint); c->comp_hint = nullptr;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->copy_stream));
    cudaFree(c->fb); c->fb = nullptr;
    cudaFree(c->fb2); c->fb2 = nullptr;
    cudaFree(c->stage[0]); cudaFree(c->stage[1]); c->stage[0] = c->stage[1] = nullptr;
    c->fb_last = nullptr; c->copied_valid[0] = c->copied_valid[1] = false;
    // peer mode refers to the frames freed above (exported) or to another process's frames of the old size (imported): drop it.
    // The host must export / import again after a resize (every rank resizes, then the presenting rank re-exports).
    if (c->peer_opened) { cudaIpcCloseMemHandle(c->peer_fb[0]); cudaIpcCloseMemHandle(c->peer_fb[1]); c->peer_opened = false; }
    c->peer_mode = false; c->peer_fb[0] = c->peer_fb[1] = nullptr; c->peer_counter = 0; c->async_counter = 0;
    group_detach(c);   // same for a shard group: every rank resizes, exports and attaches again
    c->scene_depth = nullptr; c->depth_out = nullptr;   // the caller's depth planes have the old size: depth compositing is off
    c->motion_out = nullptr; c->mot_last.valid = false;   // so are motion vectors, and the next frame has no previous one
    c->ids_out = nullptr;                                  // and splat IDs
    c->contrib = nullptr;                                  // and splat contribution
    cudaFree(c->pick_strip); c->pick_strip = nullptr;
    GSR_CUDA_TRY(cudaMalloc((void **)&c->bounds, sizeof(uint2) * (size_t)tx * ty));
    GSR_CUDA_TRY(cudaMalloc((void **)&c->comp_order, sizeof(uint32_t) * (size_t)tx * ty));
    GSR_CUDA_TRY(cudaMalloc((void **)&c->comp_hint, sizeof(uint32_t) * (size_t)tx * ty));
    GSR_CUDA_TRY(cudaMemsetAsync(c->comp_hint, 0, sizeof(uint32_t) * (size_t)tx * ty, c->stream));
    c->comp_hint_key = 0;
    if (!c->pick_frame) GSR_CUDA_TRY(cudaMalloc((void **)&c->pick_frame, sizeof(FrameState)));
    GSR_CUDA_TRY(cudaMalloc((void **)&c->fb, sizeof(float4) * (size_t)width * height));
    GSR_CUDA_TRY(cudaMalloc((void **)&c->fb2, sizeof(float4) * (size_t)width * height));
    GSR_CUDA_TRY(cudaMemsetAsync(c->fb, 0, sizeof(float4) * (size_t)width * height, c->stream));
    GSR_CUDA_TRY(cudaMemsetAsync(c->fb2, 0, sizeof(float4) * (size_t)width * height, c->stream));
    c->width = width; c->height = height; c->tiles_x = tx; c->tiles_y = ty;
    if (!c->band_set) { c->band_y0 = 0; c->band_y1 = ty; }
    if (c->band_y1 > ty) c->band_y1 = ty;
    if (c->band_y0 > c->band_y1) c->band_y0 = c->band_y1;
    return GSR_OK;
}

GSR_API int gsr_set_row_interleave(gsr_ctx *c, int32_t row_rem, int32_t row_mod) {
    if (!c || row_mod < 1 || row_rem < 0 || row_rem >= row_mod) { set_last_error("gsr_set_row_interleave: need 0 <= rem < mod"); return GSR_ERR_INVALID; }
    const char *why = row_mod > 1 ? single_context_feature(c, false) : nullptr;
    if (why) { set_last_error("gsr_set_row_interleave: %s (single-context only)", why); return GSR_ERR_STATE; }
    c->row_mod = row_mod; c->row_rem = row_rem;
    return GSR_OK;
}

GSR_API void *gsr_band_sync_word(gsr_ctx *c) { return c ? (void *)c->sync_word : nullptr; }

GSR_API int gsr_band_fixup(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    if (c->row_mod <= 1 || !c->fb_last) return GSR_OK;  // exact modes resolve the quirk inside tile_ranges_kernel
    if (c->flags & GSR_FLAG_FIXED_RANGES) return GSR_OK;
    int rc = use_device(c->device);
    if (rc) return rc;
    return launch_band_fixup(c->sync_word, c->fb_last, c->width, c->height, c->tiles_x, c->tiles_x * c->tiles_y, c->band_y0, c->band_y1,
                             c->row_mod, c->row_rem, c->stream);
}

GSR_API int gsr_set_band(gsr_ctx *c, int32_t row_begin, int32_t row_end) {
    if (!c || c->tiles_y == 0) { set_last_error("gsr_set_band before gsr_resize"); return GSR_ERR_STATE; }
    if (row_begin < 0 || row_end > c->tiles_y || row_begin > row_end) { set_last_error("band [%d,%d) outside [0,%d]", row_begin, row_end, c->tiles_y); return GSR_ERR_INVALID; }
    const bool partial = !(row_begin == 0 && row_end == c->tiles_y);
    const char *why = partial ? single_context_feature(c, false) : nullptr;
    if (why) { set_last_error("gsr_set_band: %s (single-context only)", why); return GSR_ERR_STATE; }
    c->band_y0 = row_begin; c->band_y1 = row_end;
    c->band_set = partial;
    return GSR_OK;
}

// Per-frame constants of the projection: project_covariance's focal / limit terms and the norm bound of the conservative reject.
static void frame_constants(const float *view_proj, const Uniforms &u, ProjectionArgs &pa) {
    {   // per-frame constants of project_covariance, same IEEE binary32 operations as gsplat_projection.glsl:127-133
        const float tfi0 = view_proj[16 + 0], tfi1 = view_proj[16 + 5];
        const volatile float hw = (float)u.dims[0] * 0.5f, hh = (float)u.dims[1] * 0.5f;
        const volatile float f0 = hw * tfi0, f1 = hh * tfi1;
        const volatile float t0 = 1.0f / tfi0, t1 = 1.0f / tfi1;
        const volatile float n0 = -t0, n1 = -t1;
        pa.focal_base[0] = f0; pa.focal_base[1] = f1;
        pa.lim_lo[0] = n0 * 1.3f; pa.lim_lo[1] = n1 * 1.3f;
        pa.lim_hi[0] = t0 * 1.3f; pa.lim_hi[1] = t1 * 1.3f;
    }
    {   // |W|_2^2 <= |W^T W|_inf (largest absolute row sum of the Gram matrix); exactly 1 for a rigid camera
        float g[3][3];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                g[i][j] = 0.0f;
                for (int r = 0; r < 3; ++r) g[i][j] += view_proj[4 * i + r] * view_proj[4 * j + r];
            }
        float nrm = 0.0f;
        for (int i = 0; i < 3; ++i) {
            float row = 0.0f;
            for (int j = 0; j < 3; ++j) row += g[i][j] < 0.0f ? -g[i][j] : g[i][j];
            nrm = row > nrm ? row : nrm;
        }
        pa.w_frob2 = nrm * 1.0001f;
    }
}

// ---- dynamic duplicate capacity ------------------------------------------------------------------------------------------
static int grow_capacity(gsr_ctx *c, uint64_t want) {
    if (want > c->capacity_max) want = c->capacity_max;
    if (want <= c->capacity) return GSR_OK;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->copy_stream));
    c->front_gate = nullptr;
    cudaFree(c->keys); cudaFree(c->vals); c->keys = c->vals = c->keys_cur = c->vals_cur = nullptr;
    sort_workspace_destroy(c->sort);
    const bool unsorted = c->unsorted_keys != nullptr;
    cudaFree(c->unsorted_keys); cudaFree(c->unsorted_vals); c->unsorted_keys = c->unsorted_vals = nullptr;
    c->capacity = want;
    c->cap_stride = (c->capacity + 1023ull) & ~1023ull;
    GSR_CUDA_TRY(cudaMalloc((void **)&c->keys, sizeof(uint32_t) * 3ull * c->cap_stride));
    GSR_CUDA_TRY(cudaMalloc((void **)&c->vals, sizeof(uint32_t) * 3ull * c->cap_stride));
    c->keys_cur = c->keys; c->vals_cur = c->vals;
    if (unsorted) {
        GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_keys, sizeof(uint32_t) * c->capacity));
        GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_vals, sizeof(uint32_t) * c->capacity));
    }
    int rc = sort_workspace_create(c->sort, c->capacity, /*need_alt_buffers=*/false);
    if (rc || !c->depth_words) return rc;
    // the depth-order buffers grow with the pairs once they exist
    cudaFree(c->depth_words); cudaFree(c->unsorted_depth); c->depth_words = c->unsorted_depth = nullptr;
    return alloc_depth_order(c);
}

// Examine the mirrors of the frames that have completed since the last call (no host sync: event queries) and grow the
// capacity once M has used more than half of it -- an overflow then needs M to more than double from one frame to the next.
static int track_capacity(gsr_ctx *c) {
    if (c->flags & GSR_FLAG_STATIC_CAPACITY) return GSR_OK;
    while (c->stats_polled < c->frame_counter) {
        if (c->frame_counter - c->stats_polled > GSR_HISTORY_FRAMES) { c->stats_polled = c->frame_counter - GSR_HISTORY_FRAMES; continue; }
        const uint32_t slot = (uint32_t)(c->stats_polled % GSR_HISTORY_FRAMES);
        if (cudaEventQuery(c->ev_stat[slot]) != cudaSuccess) { cudaGetLastError(); break; }
        const uint64_t m = c->host_ring[slot].dup_total;
        if (m > c->m_high) c->m_high = m;
        c->stats_polled += 1;
    }
    if (c->m_high * 2ull > c->capacity && c->capacity < c->capacity_max) return grow_capacity(c, c->m_high * 3ull);
    return GSR_OK;
}

struct GroupFrame { uint32_t seq; int parity; int rows_local; };

// GPU time of one frame's stages from its events: 'Projection' = front part (clear + projection kernel, on the front stream when frames
// overlap) + receive (group mode: segment wait + gather); total = the sum of the stages = GPU time attributable to the frame (with
// overlap the frame PERIOD is shorter than that: the front part runs beside the previous frame's compositor).
static int stage_times(gsr_ctx *c, uint32_t slot, float out[5], float *front_ms) {
    cudaEvent_t *ev = c->ev + EV_PER_FRAME * slot;
    float front = 0.f, recv = 0.f;
    GSR_CUDA_TRY(cudaEventElapsedTime(&front, ev[0], ev[1]));
    GSR_CUDA_TRY(cudaEventElapsedTime(&recv, ev[2], ev[3]));
    out[0] = front + recv;
    for (int i = 1; i < 4; ++i) GSR_CUDA_TRY(cudaEventElapsedTime(&out[i], ev[2 + i], ev[3 + i]));
    out[4] = out[0] + out[1] + out[2] + out[3];
    if (front_ms) *front_ms = front;
    return GSR_OK;
}

// arena layout (identical on every rank of a group: same max_splats, same rx_capacity)
// (`parity` = frame phase seq % GROUP_PHASES)
static size_t arena_rx_keys_off(uint64_t cap, int parity) { return GROUP_FLAGS_BYTES + sizeof(uint32_t) * cap * (size_t)parity; }
static size_t arena_rx_vals_off(uint64_t cap, int parity) { return GROUP_FLAGS_BYTES + sizeof(uint32_t) * cap * (size_t)(GROUP_PHASES + parity); }
static size_t arena_records_off(uint64_t cap, uint64_t max_splats, int parity) { return GROUP_FLAGS_BYTES + sizeof(uint32_t) * cap * 2 * GROUP_PHASES + sizeof(float4) * 3ull * max_splats * (size_t)parity; }
static size_t arena_bytes(uint64_t cap, uint64_t max_splats) { return arena_records_off(cap, max_splats, GROUP_PHASES); }

static GroupPeers group_peers(const gsr_ctx *c, int parity) {
    (void)parity;
    GroupPeers p;
    memset(&p, 0, sizeof p);
    p.world = c->grp.world; p.rank = c->grp.rank;
    for (int r = 0; r < c->grp.world; ++r) p.flags[r] = c->grp.flags[r];
    return p;
}

// GSR_FLAG_ORTHOGRAPHIC: whether the frame takes the orthographic projection path (its projection's w row is exactly (0, 0, 0, 1)), and
// GSR_ERR_STATE when it does on a sharded context (checked before anything of the frame is enqueued).
static int frame_is_orthographic(const gsr_ctx *c, const float *view_proj, bool *ortho) {
    *ortho = (c->flags & GSR_FLAG_ORTHOGRAPHIC) && view_proj[19] == 0.0f && view_proj[23] == 0.0f && view_proj[27] == 0.0f && view_proj[31] == 1.0f;
    if (*ortho && sharded(c)) { set_last_error("orthographic frame: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    return GSR_OK;
}

// same_frame: gsr_render's re-render of a frame that overflowed -- the same frame again, with the same previous state (motion vectors),
// and the history does not advance
static int render_enqueue(gsr_ctx *c, const float *view_proj, const void *uniforms32, float heatmap_factor, float4 *target = nullptr,
                          const GroupFrame *gf = nullptr, bool same_frame = false) {
    if (!c || !view_proj || !uniforms32) return GSR_ERR_INVALID;
    if (c->width == 0) { set_last_error("gsr_render before gsr_resize"); return GSR_ERR_STATE; }
    bool ortho = false;
    int rc = frame_is_orthographic(c, view_proj, &ortho);
    if (rc) return rc;
    Uniforms u;
    memcpy(&u, uniforms32, sizeof u);
    if (u.dims[0] != c->width || u.dims[1] != c->height) {
        set_last_error("uniform dims %dx%d differ from gsr_resize %dx%d", u.dims[0], u.dims[1], c->width, c->height);
        return GSR_ERR_INVALID;
    }
    if ((rc = use_device(c->device))) return rc;
    if ((rc = track_capacity(c))) return rc;
    cudaStream_t s = c->stream;
    // Front / back overlap.  The front part of a frame (clear + projection: HBM-bound) needs nothing from the frame before it, the back
    // part (sort, ranges, compositor) nothing from the frame after it.  With overlap on, the front part runs on its own stream and
    // is released when the PREVIOUS frame's tile ranges are done: it then shares the GPU with that frame's compositor (FMA-pipe /
    // chain bound, 1-2 small CTAs per SM), which leaves the memory system idle.  Consecutive frames alternate between two sort
    // inputs and two record tables; the back part waits for its own front part.  A host that renders one frame at a time
    // (gsr_render) sees the same kernels in the same order.
    const bool overlap = c->overlap > 0 && c->front_stream != nullptr;
    cudaStream_t fs = overlap ? c->front_stream : s;
    int launches = 0;
    const uint32_t slot = (uint32_t)(c->frame_counter % GSR_HISTORY_FRAMES);
    c->frame = c->ring + slot;
    cudaEvent_t *ev = c->ev + EV_PER_FRAME * slot;
    const int half = (int)(c->frame_counter & 1u);
    uint32_t *keys_in = c->keys + (size_t)half * c->cap_stride, *vals_in = c->vals + (size_t)half * c->cap_stride;
    uint32_t *keys_alt = c->keys + 2ull * c->cap_stride, *vals_alt = c->vals + 2ull * c->cap_stride;
    float4 *records = half ? c->records2 : c->records;
    const uint32_t n_tiles = (uint32_t)(c->tiles_x * c->tiles_y);

    // ---- front: rasterizer.gd:127-128 (clear M = this frame's history slot + the scan links), then the projection ----
    if (overlap && c->front_gate) GSR_CUDA_TRY(cudaStreamWaitEvent(fs, c->front_gate, 0));
    // A group frame (gf) has none of the single-context features read below: single_context_feature() and sharded() keep them apart.
    const bool inst = c->inst.n > 0;
    // motion vectors (gsr_set_motion_vectors, read here: frames already enqueued keep their plane): the previous state of this frame
    const bool motion = c->motion_out && c->depth_out;
    const gsr_ctx::MotionState &prev = same_frame ? c->mot_used : c->mot_last;
    // splat IDs (gsr_set_splat_ids), read here as well
    const bool ids = c->ids_out && c->depth_out;
    // splat contribution (gsr_set_splat_contribution), and the frame's epoch (a re-render keeps its frame's)
    const bool contrib = c->contrib && c->depth_out;
    if (contrib && !same_frame) c->contrib_epoch = c->contrib_epoch + 1u ? c->contrib_epoch + 1u : 1u;
    {
        uint32_t links = projection_num_blocks((uint32_t)(inst ? c->inst.drawn : c->max_splats));
        if (gf) {
            const uint64_t first = (uint64_t)c->grp.rank * c->grp.slice;
            const uint64_t count = first < c->max_splats ? ((c->max_splats - first) < c->grp.slice ? (c->max_splats - first) : c->grp.slice) : 0;
            links = projection_scatter_blocks((uint32_t)count) * (uint32_t)c->grp.world;
        }
        // serial: one kernel clears the tile bounds as well; overlapped: the bounds belong to the back part (the previous frame's
        // compositor may still read them)
        if ((rc = launch_frame_clear(c->frame, c->lookback, links, overlap ? nullptr : c->bounds, overlap ? 0u : n_tiles, fs))) return rc;
        launches += 1;
    }
    GSR_CUDA_TRY(cudaEventRecord(ev[0], fs));  // 'Start'
    if (inst) {
        // this frame's transforms -> a slot of the mapped ring (no copy engine, no host sync while the host is fewer than
        // GSR_INSTANCE_RING frames ahead), then one small kernel composes every instance's V_k / cam_k into this parity's table
        const uint32_t rs = (uint32_t)(c->inst.seq % GSR_INSTANCE_RING);
        if (c->inst.ev_used[rs] && cudaEventQuery(c->inst.ev[rs]) != cudaSuccess) {
            cudaGetLastError();
            GSR_CUDA_TRY(cudaEventSynchronize(c->inst.ev[rs]));
        }
        const size_t per = (size_t)c->inst.cap * INSTANCE_SLOT_FLOATS, app_off = (size_t)c->inst.cap * INSTANCE_XFORM_FLOATS;
        memcpy(c->inst.ring + rs * per, c->inst.xf, sizeof(float) * INSTANCE_XFORM_FLOATS * c->inst.n);
        // the appearance travels in the same slot (read here: frames already enqueued keep theirs); none set: no table this frame
        if (c->inst.app) instance_appearance_rows(c->inst, c->inst.ring + rs * per + app_off);
        // motion vectors: every instance's previous to_frame travels in the same slot -- the previous frame's where it had the same
        // layout, else the instance's own (no instance motion, camera motion only)
        const size_t prev_off = app_off + (size_t)c->inst.cap * INSTANCE_APPEARANCE_FLOATS;
        if (motion) {
            const bool same_layout = prev.valid && prev.range.size() == 2ull * c->inst.n &&
                                     memcmp(prev.range.data(), c->inst.range, sizeof(uint64_t) * 2ull * c->inst.n) == 0;
            float *pr = c->inst.ring + rs * per + prev_off;
            for (uint32_t k = 0; k < c->inst.n; ++k)
                memcpy(pr + (size_t)k * INSTANCE_PREV_FLOATS, same_layout ? prev.to_frame.data() + (size_t)k * INSTANCE_PREV_FLOATS
                                                                          : c->inst.xf + (size_t)k * INSTANCE_XFORM_FLOATS,
                       sizeof(float) * INSTANCE_PREV_FLOATS);
        }
        if ((rc = launch_instance_prepare(c->inst.ring_dev + rs * per, view_proj, u.camera_pos, c->inst.n,
                                          c->inst.frame + (size_t)half * c->inst.cap * INSTANCE_FRAME_FLOATS, fs,
                                          c->inst.app ? c->inst.ring_dev + rs * per + app_off : nullptr, instance_appearance_table(c->inst, half),
                                          motion ? c->inst.ring_dev + rs * per + prev_off : nullptr, instance_prev_table(c->inst, half)))) return rc;
        GSR_CUDA_TRY(cudaEventRecord(c->inst.ev[rs], fs));
        c->inst.ev_used[rs] = true;
        c->inst.seq += 1;
        launches += 1;
    }

    ProjectionArgs pa;
    // the reference dispatches over splat_buffer.length() = point_cloud.size every frame (rasterizer.gd:83,134), i.e. also over the
    // zero-initialised structs of splats the loader has not delivered yet: so does libgsr (the SoA planes start zeroed)
    pa.soa = c->soa; pa.plane_stride = c->plane_stride; pa.num_splats = (uint32_t)(inst ? c->inst.drawn : c->max_splats);
    memcpy(pa.vp, view_proj, sizeof pa.vp);
    pa.u = u;
    frame_constants(view_proj, u, pa);
    const bool fast = c->row_mod > 1 && !gf;   // group mode is exact: the frame-global last tile travels with the pairs
    pa.band_y0 = c->band_y0; pa.band_y1 = c->band_y1;
    pa.row_mod = c->row_mod; pa.row_rem = c->row_rem;
    // Conservative early reject + compaction of the survivors over 1024-splat CTAs (projection_sharded_kernel): exact, but it only
    // pays when a rank owns a small share of the rows (with two ranks nearly every splat's conservative extent touches both).
    // So: on by default from 6 ranks, or on request (GSR_FLAG_FAST_REJECT).
    const bool want_reject = (c->flags & GSR_FLAG_FAST_REJECT) != 0 || c->row_mod >= 6;
    pa.fast_reject = (want_reject && fast) ? 1 : 0;
    pa.fast_mode = fast ? 1 : 0;
    // full frame: 12 of 32 lanes (below that, per-lane 128-bit gathers move fewer bytes); sharded: few lanes of a warp land in
    // this rank's rows and the latency-bound gather path is slower than fetching the whole 6 KB slice
    pa.sh_bulk_min = (fast || c->row_mod > 1) ? 1 : 12;
    pa.records = records; pa.keys = keys_in; pa.values = vals_in; pa.capacity = (uint32_t)c->capacity;
    pa.lookback = c->lookback; pa.frame = c->frame;
    pa.aa_variance = c->aa_variance;   // read here: frames already enqueued keep their filter
    const bool aa = c->aa_variance > 0.0f;
    // gsr_set_depth_order, read here like the filter: the projection stores every pair's depth word beside its key, and the sort orders
    // the pairs by (tile, depth word) instead of by the key
    uint32_t *depth_in = nullptr, *depth_alt = nullptr;
    if (view_depth_order(c)) {
        depth_in = c->depth_words + (size_t)half * c->cap_stride;
        depth_alt = c->depth_words + 2ull * c->cap_stride;
    }
    // gsr_set_cutouts and the splat masks (gsr_select_*, gsr_set_selection_style), read here too: the set, the mask pointers and the
    // highlight are copied into the projection's launch parameters
    CutParams cut_params(c->cutouts);
    if (c->masks.on) {
        SplatMaskArgs &m = cut_params.masks;
        m.hidden = c->masks.hidden; m.selected = c->masks.selected;
        const volatile float sh = c->masks.strength;   // float32 on the host, once per frame
        m.keep = 1.0f - sh;
        for (int i = 0; i < 3; ++i) { const volatile float h = c->masks.rgb[i] * sh; m.add[i] = h; }
        m.highlight = sh > 0.0f ? 1u : 0u;
    }
    const CutParams *cut = (cutouts_on(c) || c->masks.on) ? &cut_params : nullptr;
    if (gf) {
        // group mode: the projection is sharded by SPLATS.  This rank projects its slice and stores every pair and record into the
        // memory of the rank that owns it (peer stores over NVLink); the back part then waits for the other sources' flags and packs
        // what it received -- its own rows' pairs of ALL splats, in splat-id order -- into the sort input.
        const int G = c->grp.world;
        ScatterPeers sp;
        memset(&sp, 0, sizeof sp);
        sp.world = G; sp.rank = c->grp.rank; sp.parity = gf->parity; sp.seq = gf->seq;
        const uint64_t first = (uint64_t)c->grp.rank * c->grp.slice;
        sp.first = (uint32_t)(first < c->max_splats ? first : c->max_splats);
        sp.count = (uint32_t)(first < c->max_splats ? ((c->max_splats - first) < c->grp.slice ? (c->max_splats - first) : c->grp.slice) : 0);
        sp.seg_cap = c->grp.seg_cap;
        for (int d = 0; d < G; ++d) {
            char *ar = c->grp.peer_arena[d];
            sp.records[d] = reinterpret_cast<float4 *>(ar + arena_records_off(c->grp.rx_capacity, c->max_splats, gf->parity));
            sp.keys[d] = reinterpret_cast<uint32_t *>(ar + arena_rx_keys_off(c->grp.rx_capacity, gf->parity)) + (size_t)c->grp.rank * c->grp.seg_cap;
            sp.values[d] = reinterpret_cast<uint32_t *>(ar + arena_rx_vals_off(c->grp.rx_capacity, gf->parity)) + (size_t)c->grp.rank * c->grp.seg_cap;
            sp.flags[d] = c->grp.flags[d];
        }
        sp.lookback = c->lookback;
        if ((rc = launch_projection_scatter(pa, sp, fs))) return rc;
        launches += 1;
    } else if (inst) {
        InstanceArgs ia;
        ia.frame = c->inst.frame + (size_t)half * c->inst.cap * INSTANCE_FRAME_FLOATS;
        ia.desc = c->inst.desc; ia.warp_inst = c->inst.warps;
        ia.appearance = c->inst.app ? instance_appearance_table(c->inst, half) : nullptr;
        if ((rc = launch_projection_instanced(pa, ia, fs, render_bands(c), ortho, aa, depth_in, cut, sh_half(c)))) return rc;
        launches += pa.num_splats ? 1 : 0;
    } else {
        if ((rc = launch_projection(pa, fs, render_bands(c), ortho, aa, depth_in, cut, sh_half(c)))) return rc;
        launches += pa.num_splats ? 1 : 0;
    }
    GSR_CUDA_TRY(cudaEventRecord(ev[1], fs));  // end of the front part

    // ---- back ----
    if (overlap) {
        GSR_CUDA_TRY(cudaStreamWaitEvent(s, ev[1], 0));
        if ((rc = launch_frame_clear(nullptr, nullptr, 0u, c->bounds, n_tiles, s))) return rc;
        launches += 1;
    }
    GSR_CUDA_TRY(cudaEventRecord(ev[2], s));
    if (gf) {
        const int G = c->grp.world;
        char *mine = c->grp.peer_arena[c->grp.rank];
        if ((rc = launch_group_wait_segments(c->grp.flags[c->grp.rank], gf->parity, G, gf->seq, c->grp.seg_cap, (uint32_t)c->capacity, c->frame, s))) return rc;
        if ((rc = launch_gather_segments(c->grp.flags[c->grp.rank], G, c->grp.seg_cap,
                                         reinterpret_cast<const uint32_t *>(mine + arena_rx_keys_off(c->grp.rx_capacity, gf->parity)),
                                         reinterpret_cast<const uint32_t *>(mine + arena_rx_vals_off(c->grp.rx_capacity, gf->parity)), keys_in, vals_in,
                                         c->sm_count * 8, s))) return rc;
        records = reinterpret_cast<float4 *>(mine + arena_records_off(c->grp.rx_capacity, c->max_splats, gf->parity));
        launches += 2;
    }
    c->keys_cur = keys_in; c->vals_cur = vals_in; c->records_cur = records;
    GSR_CUDA_TRY(cudaEventRecord(ev[3], s));  // 'Projection' = front + receive

    if (c->keep_unsorted) {
        GSR_CUDA_TRY(cudaMemcpyAsync(c->unsorted_keys, keys_in, sizeof(uint32_t) * c->capacity, cudaMemcpyDeviceToDevice, s));
        GSR_CUDA_TRY(cudaMemcpyAsync(c->unsorted_vals, vals_in, sizeof(uint32_t) * c->capacity, cudaMemcpyDeviceToDevice, s));
        if (depth_in) GSR_CUDA_TRY(cudaMemcpyAsync(c->unsorted_depth, depth_in, sizeof(uint32_t) * c->capacity, cudaMemcpyDeviceToDevice, s));
    }
    const uint32_t *m_ptr = reinterpret_cast<const uint32_t *>(reinterpret_cast<const char *>(c->frame) + offsetof(FrameState, dup_sorted));
    if (depth_in) {
        if ((rc = sort_pairs_depth_device(c->sort, keys_in, vals_in, depth_in, m_ptr, keys_alt, vals_alt, depth_alt, s, &launches))) return rc;
    } else {
        if ((rc = sort_pairs_device(c->sort, keys_in, vals_in, m_ptr, keys_alt, vals_alt, s, &launches))) return rc;
    }
    GSR_CUDA_TRY(cudaEventRecord(ev[4], s));  // 'Sort'

    const int sharded = fast ? 2 : ((!(c->band_y0 == 0 && c->band_y1 == c->tiles_y) || c->row_mod > 1) ? 1 : 0);
    if (fast) GSR_CUDA_TRY(cudaMemsetAsync(c->sync_word, 0, sizeof(int32_t), s));
    const int quirks = (c->flags & GSR_FLAG_FIXED_RANGES) ? 0 : 1;
    if ((rc = launch_tile_ranges(keys_in, c->frame, c->bounds, n_tiles, quirks, sharded, fast ? c->sync_word : nullptr, c->sm_count * 8, s))) return rc;
    launches += 1;
    GSR_CUDA_TRY(cudaEventRecord(ev[5], s));  // 'Boundaries'
    c->front_gate = ev[5];   // the next frame's front part may start here, beside this frame's compositor

    CompositeArgs ca;
    float4 *out_fb = c->fb_ext ? c->fb_ext : (target ? target : c->fb);
    // a pipelined read-back of this buffer may still be in flight on the copy stream (gsr_render_async followed by gsr_render)
    for (int i = 0; i < 2; ++i) {
        const float4 *owned = c->peer_mode ? c->peer_fb[i] : (i ? c->fb2 : c->fb);
        if (c->copied_valid[i] && owned == out_fb) GSR_CUDA_TRY(cudaStreamWaitEvent(s, c->ev_copied[i], 0));
    }
    c->fb_last = out_fb;
    ca.records = records; ca.values = vals_in; ca.bounds = c->bounds; ca.out = out_fb;
    ca.width = c->width; ca.height = c->height; ca.tiles_x = c->tiles_x;
    {   // owned tile rows: band rows with row % row_mod == row_rem
        int first = c->band_y0 + ((c->row_rem - c->band_y0 % c->row_mod) + c->row_mod) % c->row_mod;
        int nrows = first < c->band_y1 ? (c->band_y1 - 1 - first) / c->row_mod + 1 : 0;
        ca.tile_begin = first * c->tiles_x;
        ca.row_step = c->row_mod;
        ca.num_tiles = nrows * c->tiles_x;
    }
    ca.heatmap_factor = heatmap_factor;
    ca.target_tile_id = 0xFFFFFFFFu;  // rasterizer.gd:158
    ca.pick = c->pick;
    ca.frame = c->frame; ca.count_staged = 1;
    ca.order = nullptr; ca.consumed = c->comp_hint;
    ca.ctas_per_sm = c->comp_ctas_per_sm < c->comp_max_ctas ? c->comp_ctas_per_sm : c->comp_max_ctas; ca.sm_count = c->sm_count;
    ca.contract = (c->flags & GSR_FLAG_UNCONTRACTED_BLEND) ? 0 : 1;
    {   // the hints describe the owned-tile indexing of the frame that wrote them: drop them when the ownership changes
        const uint64_t key = ((uint64_t)(uint32_t)ca.tile_begin << 32) ^ ((uint64_t)(uint32_t)ca.row_step << 24) ^ (uint64_t)(uint32_t)ca.num_tiles;
        if (key != c->comp_hint_key) { GSR_CUDA_TRY(cudaMemsetAsync(c->comp_hint, 0, sizeof(uint32_t) * (size_t)c->tiles_x * c->tiles_y, s)); c->comp_hint_key = key; }
    }
    if (c->comp_order_mode && ca.num_tiles > 0) {   // longest chains first: the long sequential chains start at once instead of in the tail
        if ((rc = launch_tile_order(c->bounds, ca.tile_begin, ca.row_step, ca.tiles_x, ca.num_tiles, c->comp_hint, c->comp_order, c->frame,
                                    (uint32_t)(c->comp_sparse_per_sm * c->sm_count), (uint32_t)c->sm_count, s))) return rc;
        ca.order = c->comp_order;
        launches += 1;
    }
    ca.trace = c->trace; ca.trace_count = c->trace_count; ca.trace_cap = c->trace_cap;
    ca.view_z[0] = view_proj[2]; ca.view_z[1] = view_proj[6]; ca.view_z[2] = view_proj[10]; ca.view_z[3] = view_proj[14];
    ca.scene_depth = c->scene_depth; ca.depth_out = c->depth_out;
    if (c->trace) GSR_CUDA_TRY(cudaMemsetAsync(c->trace_count, 0, sizeof(uint32_t), s));
    if (gf && !gf->rows_local && c->grp.rank != 0 && gf->seq >= 3u) {   // the presenting rank must have consumed the frame that used this slot
        if ((rc = launch_group_wait_released(c->grp.flags[c->grp.rank], gf->seq - 2u, s))) return rc;
        launches += 1;
    }
    MotionArgs ma;
    if (motion) {
        memcpy(ma.vp, view_proj, sizeof ma.vp);
        memcpy(ma.prev_vp, prev.valid ? prev.vp : view_proj, sizeof ma.prev_vp);
        ma.fw = (float)(c->width - 1); ma.fh = (float)(c->height - 1);
        ma.motion_out = c->motion_out;
        ma.warp_inst = inst ? c->inst.warps : nullptr; ma.desc = c->inst.desc;
        ma.prev_xf = inst ? instance_prev_table(c->inst, half) : nullptr;
        ma.plane0 = c->soa; ma.model_scale = u.model_scale;
    }
    SplatIdArgs sa;
    sa.ids_out = c->ids_out;
    sa.warp_inst = inst ? c->inst.warps : nullptr;
    ContribArgs cb;
    cb.accum = c->contrib;
    cb.warp_inst = inst ? c->inst.warps : nullptr; cb.desc = c->inst.desc;
    cb.frames = c->contrib_frames;
    cb.epoch = c->contrib_epoch;
    if ((rc = launch_composite(ca, s, motion ? &ma : nullptr, ids ? &sa : nullptr, contrib ? &cb : nullptr))) return rc;
    launches += ca.num_tiles > 0 ? 1 : 0;
    if (gf && !gf->rows_local) {   // rows have landed in the presenting rank's frame: tell it (system-scope flag store after the kernel boundary)
        if ((rc = launch_group_signal_done(group_peers(c, gf->parity), 0, c->grp.rank, gf->seq, s))) return rc;
        launches += 1;
    }
    GSR_CUDA_TRY(cudaEventRecord(ev[6], s));  // 'Render'
    // this frame's counters (M, overflow, C) to the pinned mirror: what track_capacity() reads without ever syncing
    // (a 16-byte-store kernel into mapped pinned memory, NOT a cudaMemcpyAsync: a D2H copy on the render stream would queue behind the
    // frame read-back on the copy engine and serialise the two streams)
    if ((rc = launch_publish_frame_state(c->frame, c->host_ring + slot, s))) return rc;
    GSR_CUDA_TRY(cudaEventRecord(c->ev_stat[slot], s));
    c->ev_valid = true;
    c->frame_counter += 1;
    c->last_launches = (uint32_t)launches;
    if (!same_frame) {   // the history: this frame is the next frame's previous one
        std::swap(c->mot_used, c->mot_last);
        gsr_ctx::MotionState &h = c->mot_last;
        h.valid = true;
        memcpy(h.vp, view_proj, sizeof h.vp);
        h.range.assign(inst ? c->inst.range : nullptr, inst ? c->inst.range + 2ull * c->inst.n : nullptr);
        h.to_frame.resize(inst ? (size_t)INSTANCE_PREV_FLOATS * c->inst.n : 0u);
        for (uint32_t k = 0; inst && k < c->inst.n; ++k)
            memcpy(h.to_frame.data() + (size_t)k * INSTANCE_PREV_FLOATS, c->inst.xf + (size_t)k * INSTANCE_XFORM_FLOATS, sizeof(float) * INSTANCE_PREV_FLOATS);
    }
    return GSR_OK;
}

GSR_API int gsr_render(gsr_ctx *c, const float view_proj[32], const void *uniforms32, float heatmap_factor, float *out_host) {
    if (c && c->grp.world > 1) { set_last_error("gsr_render: a context attached to a group renders with gsr_render_async (all ranks, same frame)"); return GSR_ERR_STATE; }
    int rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor);
    if (rc) return rc;
    if (out_host) {
        // synchronous path: a frame that overflowed the duplicate capacity is never returned -- grow and render it again
        // (the reference truncates silently: rasterizer.gd:79, main.gd:100; GSR_FLAG_STATIC_CAPACITY keeps that behaviour)
        for (int attempt = 0; attempt < 8 && !(c->flags & GSR_FLAG_STATIC_CAPACITY); ++attempt) {
            const uint32_t slot = (uint32_t)((c->frame_counter - 1) % GSR_HISTORY_FRAMES);
            GSR_CUDA_TRY(cudaEventSynchronize(c->ev_stat[slot]));
            const FrameState &fs = c->host_ring[slot];
            if (!fs.overflow || c->capacity >= c->capacity_max) break;
            if ((rc = grow_capacity(c, fs.dup_total + fs.dup_total / 4ull + 1024ull))) return rc;
            if ((rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor, nullptr, nullptr, true))) return rc;
        }
        GSR_CUDA_TRY(cudaMemcpyAsync(out_host, framebuffer(c), sizeof(float4) * (size_t)c->width * c->height, cudaMemcpyDeviceToHost, c->stream));
        GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    return GSR_OK;
}

static int readback_enqueue(gsr_ctx *c, float4 *frame, int slot, void *pinned_host, int format, uint32_t group_seq = 0) {
    const size_t pixels = (size_t)c->width * c->height;
    const size_t bpp = present_bytes_per_pixel(format);
    if (!bpp) { set_last_error("unknown output format 0x%x", format); return GSR_ERR_INVALID; }
    int rc;
    const bool convert = format != GSR_OUT_RGBA32F;
    if (convert && !c->stage[slot]) GSR_CUDA_TRY(cudaMalloc(&c->stage[slot], sizeof(float4) * pixels + 64));
    GSR_CUDA_TRY(cudaEventRecord(c->ev_done[slot], c->stream));
    GSR_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->ev_done[slot], 0));
    // group mode: the other ranks' rows arrive over NVLink; their done flags gate the copy (device-side wait on the copy stream)
    if (group_seq && (rc = launch_group_wait_done(c->grp.flags[c->grp.rank], c->grp.world, group_seq, c->copy_stream))) return rc;
    if (convert) {
        if ((rc = launch_present(frame, c->stage[slot], pixels, format, c->copy_stream))) return rc;
        GSR_CUDA_TRY(cudaMemcpyAsync(pinned_host, c->stage[slot], bpp * pixels, cudaMemcpyDeviceToHost, c->copy_stream));
    } else {
        GSR_CUDA_TRY(cudaMemcpyAsync(pinned_host, frame, sizeof(float4) * pixels, cudaMemcpyDeviceToHost, c->copy_stream));
    }
    GSR_CUDA_TRY(cudaEventRecord(c->ev_copied[slot], c->copy_stream));
    c->copied_valid[slot] = true;
    return GSR_OK;
}

static int render_async_impl(gsr_ctx *c, const float *view_proj, const void *uniforms32, float heatmap_factor, void *pinned_host, int format) {
    if (!c) return GSR_ERR_INVALID;
    if (view_proj) {   // an orthographic frame on a sharded context enqueues nothing (the group and peer paths below enqueue waits before the frame)
        bool ortho = false;
        const int rc = frame_is_orthographic(c, view_proj, &ortho);
        if (rc) return rc;
    }
    if (c->grp.world > 1) {   // shard group: every rank enqueues the same frame; rows land in the presenting rank's frames
        if (pinned_host) { set_last_error("group mode: render with a NULL host pointer on every rank, then gsr_readback_async on rank 0"); return GSR_ERR_STATE; }
        int rc = use_device(c->device);
        if (rc) return rc;
        GroupFrame gf;
        gf.seq = c->grp.seq + 1u; gf.parity = (int)(gf.seq % (uint32_t)GROUP_PHASES);
        const int slot = (int)((gf.seq - 1u) & 1u);
        gf.rows_local = c->grp.present_rows;
        float4 *target = c->grp.root_fb[slot];
        if (gf.rows_local) {   // every rank presents its own rows (host consumer, one PCIe link per GPU): only its own read-back gates the slot
            target = slot ? c->fb2 : c->fb;   // (render_enqueue orders the compositor after the slot's read-back)
        } else if (c->grp.rank == 0) {
            if (c->copied_valid[slot]) GSR_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_copied[slot], 0));
            if (gf.seq >= 3u && (rc = launch_group_release(group_peers(c, gf.parity), c->grp.world, gf.seq - 2u, c->stream))) return rc;
        }
        if ((rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor, target, &gf))) return rc;
        c->grp.seq = gf.seq;
        return GSR_OK;
    }
    if (c->peer_mode) {  // frames alternate between the presenting rank's two frames; read-back is a separate call
        if (pinned_host) { set_last_error("peer mode: render with a NULL host pointer, then gsr_readback_async on the presenting rank"); return GSR_ERR_STATE; }
        int rc = use_device(c->device);
        if (rc) return rc;
        const int slot = (int)(c->peer_counter & 1u);
        if (c->copied_valid[slot]) GSR_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_copied[slot], 0));
        if ((rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor, c->peer_fb[slot]))) return rc;
        c->peer_counter += 1;
        return GSR_OK;
    }
    if (!pinned_host || c->fb_ext) {  // nothing to read back, or the caller owns the frame memory: plain enqueue
        if (format != GSR_OUT_RGBA32F && pinned_host) { set_last_error("converted read-back is unavailable with an external framebuffer"); return GSR_ERR_STATE; }
        int rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor);
        if (rc) return rc;
        if (pinned_host)
            GSR_CUDA_TRY(cudaMemcpyAsync(pinned_host, framebuffer(c), sizeof(float4) * (size_t)c->width * c->height, cudaMemcpyDeviceToHost, c->stream));
        return GSR_OK;
    }
    // Pipelined read-back: frames alternate between two device framebuffers; the D2H copy of frame i runs on the
    // copy stream while the render stream already works on frame i+1.  Frame i+2 waits for copy i before it
    // overwrites the same buffer.
    int rc = use_device(c->device);
    if (rc) return rc;
    const int slot = (int)(c->async_counter & 1u);
    float4 *target = slot ? c->fb2 : c->fb;   // (render_enqueue orders the compositor after the slot's read-back; sort and ranges need not wait)
    if ((rc = render_enqueue(c, view_proj, uniforms32, heatmap_factor, target))) return rc;
    if ((rc = readback_enqueue(c, target, slot, pinned_host, format))) return rc;
    c->async_counter += 1;
    return GSR_OK;
}

GSR_API int gsr_render_async(gsr_ctx *c, const float view_proj[32], const void *uniforms32, float heatmap_factor, float *pinned_host) {
    return render_async_impl(c, view_proj, uniforms32, heatmap_factor, pinned_host, GSR_OUT_RGBA32F);
}

GSR_API int gsr_render_async_rgb(gsr_ctx *c, const float view_proj[32], const void *uniforms32, float heatmap_factor, float *pinned_host_rgb) {
    return render_async_impl(c, view_proj, uniforms32, heatmap_factor, pinned_host_rgb, GSR_OUT_RGB32F);
}

GSR_API int gsr_render_async_fmt(gsr_ctx *c, const float view_proj[32], const void *uniforms32, float heatmap_factor, void *pinned_host, int32_t format) {
    if (!present_bytes_per_pixel(format)) { set_last_error("unknown output format 0x%x", format); return GSR_ERR_INVALID; }
    return render_async_impl(c, view_proj, uniforms32, heatmap_factor, pinned_host, format);
}

GSR_API size_t gsr_output_bytes(int32_t format, int32_t width, int32_t height) {
    return (width > 0 && height > 0) ? present_bytes_per_pixel(format) * (size_t)width * (size_t)height : 0;
}

// Converted copy of the most recent frame into CALLER-OWNED DEVICE memory on the render stream: the hand-off to an imported
// external image / buffer (Vulkan VK_KHR_external_memory via cudaImportExternalMemory, done by the embedder) without touching the host.
GSR_API int gsr_present_device(gsr_ctx *c, void *dst_device, int32_t format) {
    if (!c || !dst_device) return GSR_ERR_INVALID;
    if (!c->fb_last && !c->fb_ext) { set_last_error("gsr_present_device: no frame rendered yet"); return GSR_ERR_STATE; }
    if (!present_bytes_per_pixel(format)) { set_last_error("unknown output format 0x%x", format); return GSR_ERR_INVALID; }
    int rc = use_device(c->device);
    if (rc) return rc;
    if (c->grp.world > 1) {   // the other ranks' rows must have landed (device-side wait, same stream)
        if (c->grp.rank != 0) { set_last_error("gsr_present_device: only rank 0 of a group presents the frame"); return GSR_ERR_STATE; }
        if ((rc = launch_group_wait_done(c->grp.flags[0], c->grp.world, c->grp.seq, c->stream))) return rc;
    }
    return launch_present(framebuffer(c), dst_device, (uint64_t)c->width * c->height, format, c->stream);
}

GSR_API int gsr_readback_async(gsr_ctx *c, void *pinned_host, int32_t format) {
    if (!c || !pinned_host) return GSR_ERR_INVALID;
    if (!c->fb_last || c->fb_ext) { set_last_error("gsr_readback_async: no library-owned frame rendered yet"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    if (c->grp.world > 1) {
        if (c->grp.rank != 0) { set_last_error("gsr_readback_async: only rank 0 of a group presents the frame"); return GSR_ERR_STATE; }
        return readback_enqueue(c, c->fb_last, (int)((c->grp.seq - 1u) & 1u), pinned_host, format, c->grp.seq);
    }
    const int slot = (c->fb_last == c->fb2 || (c->peer_mode && c->fb_last == c->peer_fb[1])) ? 1 : 0;
    return readback_enqueue(c, c->fb_last, slot, pinned_host, format);
}

GSR_API int gsr_group_set_present(gsr_ctx *c, int32_t rows_local) {
    if (!c) return GSR_ERR_INVALID;
    if (c->grp.world <= 1) { set_last_error("gsr_group_set_present: attach the group first"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->copy_stream));
    c->grp.present_rows = rows_local != 0;
    c->copied_valid[0] = c->copied_valid[1] = false;
    return GSR_OK;
}

// Rows-local presentation: this rank's tile rows (row % world == rank) of the most recent frame -> the same rows of a full-frame
// RGBA32F host image (`host_frame` = address of pixel (0,0); page-locked in THIS process), on this rank's copy stream and PCIe link.
GSR_API int gsr_readback_rows_async(gsr_ctx *c, void *host_frame) {
    if (!c || !host_frame) return GSR_ERR_INVALID;
    if (c->grp.world <= 1 || !c->grp.present_rows || !c->fb_last) { set_last_error("gsr_readback_rows_async: needs an attached group in rows-local presentation and a rendered frame"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    const int slot = (int)((c->grp.seq - 1u) & 1u);
    const size_t row_bytes = sizeof(float4) * (size_t)c->width, slab = row_bytes * TILE;
    const int G = c->grp.world, r = c->grp.rank;
    GSR_CUDA_TRY(cudaEventRecord(c->ev_done[slot], c->stream));
    GSR_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->ev_done[slot], 0));
    const int full_rows = c->height / TILE;                        // tile rows that are 16 pixel rows high
    const int n_full = r < full_rows ? (full_rows - 1 - r) / G + 1 : 0;
    const char *src = reinterpret_cast<const char *>(c->fb_last);
    char *dst = static_cast<char *>(host_frame);
    if (n_full) GSR_CUDA_TRY(cudaMemcpy2DAsync(dst + (size_t)r * slab, (size_t)G * slab, src + (size_t)r * slab, (size_t)G * slab, slab, (size_t)n_full,
                                               cudaMemcpyDeviceToHost, c->copy_stream));
    if (c->height % TILE && full_rows % G == r)                    // the ragged last tile row, if this rank owns it
        GSR_CUDA_TRY(cudaMemcpyAsync(dst + (size_t)full_rows * slab, src + (size_t)full_rows * slab, row_bytes * (size_t)(c->height % TILE), cudaMemcpyDeviceToHost, c->copy_stream));
    GSR_CUDA_TRY(cudaEventRecord(c->ev_copied[slot], c->copy_stream));
    c->copied_valid[slot] = true;
    return GSR_OK;
}

GSR_API int gsr_peer_export_framebuffers(gsr_ctx *c, void *handles128) {
    if (!c || !handles128) return GSR_ERR_INVALID;
    const char *why = single_context_feature(c, false);
    if (why) { set_last_error("gsr_peer_export_framebuffers: %s (single-context only)", why); return GSR_ERR_STATE; }
    if (!c->fb || !c->fb2 || c->fb_ext) { set_last_error("gsr_peer_export_framebuffers: call gsr_resize first (library-owned frames only)"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaIpcMemHandle_t h[2];
    GSR_CUDA_TRY(cudaIpcGetMemHandle(&h[0], c->fb));
    GSR_CUDA_TRY(cudaIpcGetMemHandle(&h[1], c->fb2));
    memcpy(handles128, h, sizeof h);
    c->peer_fb[0] = c->fb; c->peer_fb[1] = c->fb2;
    c->peer_mode = true;
    return GSR_OK;
}

GSR_API int gsr_peer_import_framebuffers(gsr_ctx *c, const void *handles128) {
    if (!c || !handles128) return GSR_ERR_INVALID;
    const char *why = single_context_feature(c, false);
    if (why) { set_last_error("gsr_peer_import_framebuffers: %s (single-context only)", why); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaIpcMemHandle_t h[2];
    memcpy(h, handles128, sizeof h);
    GSR_CUDA_TRY(cudaIpcOpenMemHandle((void **)&c->peer_fb[0], h[0], cudaIpcMemLazyEnablePeerAccess));
    GSR_CUDA_TRY(cudaIpcOpenMemHandle((void **)&c->peer_fb[1], h[1], cudaIpcMemLazyEnablePeerAccess));
    c->peer_mode = true; c->peer_opened = true;
    return GSR_OK;
}

// ---- multi-GPU shard group: one context per GPU (processes or threads), NCCL-free frame path (group.cu) ----
namespace {
struct GroupBlob {   // what gsr_group_export hands to the other ranks (any transport; 320 bytes)
    uint32_t magic, version;
    uint64_t pid;
    int32_t device, width, height, pad;
    uint64_t max_splats, rx_capacity;
    void *arena, *fb[2];
    cudaIpcMemHandle_t h_arena, h_fb[2];
    unsigned char reserved[GSR_GROUP_BLOB_BYTES - 264];
};
static_assert(sizeof(GroupBlob) == GSR_GROUP_BLOB_BYTES, "blob layout");
constexpr uint32_t GROUP_MAGIC = 0x47535247u;  // "GRSG"

}  // namespace

GSR_API int gsr_group_export(gsr_ctx *c, void *blob) {
    if (!c || !blob) return GSR_ERR_INVALID;
    if (!c->fb || !c->fb2 || c->fb_ext) { set_last_error("gsr_group_export: call gsr_resize first (library-owned frames only)"); return GSR_ERR_STATE; }
    const char *why = single_context_feature(c, true);
    if (why) { set_last_error("gsr_group_export: %s (single-context only)", why); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    if (!c->grp.arena) {
        c->grp.rx_capacity = (c->capacity + 1023ull) & ~1023ull;   // the receive segments of all sources together hold as many pairs as one sort input
        const size_t bytes = arena_bytes(c->grp.rx_capacity, c->max_splats);
        cudaError_t e = cudaMalloc(&c->grp.arena, bytes);
        if (e != cudaSuccess) { set_last_error("cudaMalloc(group arena, %zu B) -> %s", bytes, cudaGetErrorString(e)); c->grp.arena = nullptr; return GSR_ERR_OOM; }
        GSR_CUDA_TRY(cudaMemset(c->grp.arena, 0, bytes));
    }
    GroupBlob b;
    memset(&b, 0, sizeof b);
    b.magic = GROUP_MAGIC; b.version = 1; b.pid = (uint64_t)getpid();
    b.device = c->device; b.width = c->width; b.height = c->height;
    b.max_splats = c->max_splats; b.rx_capacity = c->grp.rx_capacity;
    b.arena = c->grp.arena; b.fb[0] = c->fb; b.fb[1] = c->fb2;
    // IPC handles are needed only by ranks living in other processes; a failure here surfaces there (zero handle)
    if (cudaIpcGetMemHandle(&b.h_arena, c->grp.arena) != cudaSuccess || cudaIpcGetMemHandle(&b.h_fb[0], c->fb) != cudaSuccess ||
        cudaIpcGetMemHandle(&b.h_fb[1], c->fb2) != cudaSuccess) {
        cudaGetLastError();
        memset(&b.h_arena, 0, sizeof b.h_arena); memset(b.h_fb, 0, sizeof b.h_fb);
    }
    memcpy(blob, &b, sizeof b);
    return GSR_OK;
}

GSR_API int gsr_group_attach(gsr_ctx *c, int32_t rank, int32_t world, const void *blobs) {
    if (!c || !blobs || world < 1 || world > GROUP_MAX || rank < 0 || rank >= world) { set_last_error("gsr_group_attach: need 0 <= rank < world <= %d", GROUP_MAX); return GSR_ERR_INVALID; }
    if (!c->grp.arena || !c->fb) { set_last_error("gsr_group_attach before gsr_group_export"); return GSR_ERR_STATE; }
    const char *why = world > 1 ? single_context_feature(c, false) : nullptr;
    if (why) { set_last_error("gsr_group_attach: %s (single-context only)", why); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    group_detach(c);
    if (world == 1) return GSR_OK;
    const GroupBlob *B = reinterpret_cast<const GroupBlob *>(blobs);
    const uint64_t slice = (((c->max_splats + (uint64_t)world - 1) / (uint64_t)world) + 255ull) & ~255ull;
    for (int r = 0; r < world; ++r) {
        if (B[r].magic != GROUP_MAGIC || B[r].version != 1) { set_last_error("gsr_group_attach: blob %d is not a gsr_group_export blob", r); return GSR_ERR_INVALID; }
        if (B[r].max_splats != c->max_splats || B[r].width != c->width || B[r].height != c->height || B[r].rx_capacity != c->grp.rx_capacity) {
            set_last_error("gsr_group_attach: rank %d was created with a different scene / frame size", r);
            return GSR_ERR_INVALID;
        }
    }
    if (B[rank].arena != c->grp.arena || B[rank].pid != (uint64_t)getpid()) { set_last_error("gsr_group_attach: blob %d is not this context's export", rank); return GSR_ERR_INVALID; }
    auto fail = [&](const char *what, int r, cudaError_t e) {
        set_last_error("gsr_group_attach: %s of rank %d -> %s", what, r, cudaGetErrorString(e));
        group_detach(c);
        return GSR_ERR_CUDA;
    };
    for (int r = 0; r < world; ++r) {
        char *arena = nullptr;
        float4 *fb[2] = {nullptr, nullptr};
        if (r == rank) {
            arena = (char *)c->grp.arena; fb[0] = c->fb; fb[1] = c->fb2;
        } else if (B[r].pid == (uint64_t)getpid()) {   // same process (one thread per GPU, the GDExtension case): plain peer pointers
            if (B[r].device != c->device) {
                int can = 0;
                cudaDeviceCanAccessPeer(&can, c->device, B[r].device);
                if (!can) return fail("no peer access to the device", r, cudaErrorPeerAccessUnsupported);
                cudaError_t e = cudaDeviceEnablePeerAccess(B[r].device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail("cudaDeviceEnablePeerAccess", r, e);
                cudaGetLastError();
            }
            arena = (char *)B[r].arena; fb[0] = (float4 *)B[r].fb[0]; fb[1] = (float4 *)B[r].fb[1];
        } else {                                       // another process: CUDA IPC mappings
            cudaError_t e = cudaIpcOpenMemHandle((void **)&arena, B[r].h_arena, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) return fail("cudaIpcOpenMemHandle(arena)", r, e);
            c->grp.opened[c->grp.n_opened++] = arena;
            if (r == 0) {
                for (int k = 0; k < 2; ++k) {
                    e = cudaIpcOpenMemHandle((void **)&fb[k], B[r].h_fb[k], cudaIpcMemLazyEnablePeerAccess);
                    if (e != cudaSuccess) return fail("cudaIpcOpenMemHandle(frame)", r, e);
                    c->grp.opened[c->grp.n_opened++] = fb[k];
                }
            }
        }
        c->grp.flags[r] = reinterpret_cast<GroupFlags *>(arena);
        c->grp.peer_arena[r] = arena;
        if (r == 0) { c->grp.root_fb[0] = fb[0]; c->grp.root_fb[1] = fb[1]; }
    }
    GSR_CUDA_TRY(cudaMemsetAsync(c->grp.arena, 0, GROUP_FLAGS_BYTES, c->stream));   // flags start at seq 0 (all ranks attach, then barrier)
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->grp.rank = rank; c->grp.world = world; c->grp.slice = slice; c->grp.seq = 0;
    c->grp.seg_cap = (uint32_t)(c->grp.rx_capacity / (uint64_t)world) & ~3u;   // segments start 16-byte aligned
    c->row_mod = world; c->row_rem = rank;   // cyclic tile rows: balanced by construction
    c->band_y0 = 0; c->band_y1 = c->tiles_y; c->band_set = false;
    c->copied_valid[0] = c->copied_valid[1] = false;
    return GSR_OK;
}

GSR_API int gsr_group_detach(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    group_detach(c);
    return GSR_OK;
}

GSR_API int gsr_stream_join(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    for (int i = 0; i < 2; ++i)
        if (c->copied_valid[i]) GSR_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_copied[i], 0));
    return GSR_OK;
}

GSR_API int gsr_sync(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->copy_stream));
    if (c->grp.world > 1) {   // a device-side wait of the group protocol gave up (peer lost / frames enqueued out of lockstep)
        uint32_t err = 0;
        GSR_CUDA_TRY(cudaMemcpy(&err, &c->grp.flags[c->grp.rank]->error, sizeof err, cudaMemcpyDeviceToHost));
        if (err) {
            cudaMemset(&c->grp.flags[c->grp.rank]->error, 0, sizeof err);
            set_last_error("group: a device-side wait timed out (%s)", err == 1 ? "segments of a peer" : "done / released flag");
            return GSR_ERR_STATE;
        }
    }
    return GSR_OK;
}

GSR_API void *gsr_framebuffer_device_ptr(gsr_ctx *c) { return c ? (void *)framebuffer(c) : nullptr; }

GSR_API int gsr_set_framebuffer_external(gsr_ctx *c, void *device_ptr) {
    if (!c) return GSR_ERR_INVALID;
    c->fb_ext = (float4 *)device_ptr;
    return GSR_OK;
}

GSR_API int gsr_set_depth_compositing(gsr_ctx *c, const float *scene_depth_device, float *depth_out_device) {
    if (!c) return GSR_ERR_INVALID;
    if (!depth_out_device) {
        if (scene_depth_device) { set_last_error("gsr_set_depth_compositing: a scene depth needs a depth output"); return GSR_ERR_INVALID; }
        c->scene_depth = nullptr; c->depth_out = nullptr;
        c->motion_out = nullptr;   // motion vectors are a companion of the mode
        c->ids_out = nullptr;      // and so are splat IDs
        c->contrib = nullptr;      // and splat contribution
        return GSR_OK;
    }
    if (c->width == 0) { set_last_error("gsr_set_depth_compositing before gsr_resize"); return GSR_ERR_STATE; }
    if (sharded(c)) { set_last_error("gsr_set_depth_compositing: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    c->scene_depth = scene_depth_device; c->depth_out = depth_out_device;
    return GSR_OK;
}

GSR_API int gsr_set_motion_vectors(gsr_ctx *c, float *motion_out_device) {
    if (!c) return GSR_ERR_INVALID;
    if (!motion_out_device) { c->motion_out = nullptr; return GSR_OK; }
    if (!c->depth_out) { set_last_error("gsr_set_motion_vectors: depth compositing is off"); return GSR_ERR_STATE; }
    if (c->contrib) { set_last_error("gsr_set_motion_vectors: splat contribution is on"); return GSR_ERR_STATE; }
    if (motion_out_device == c->depth_out || motion_out_device == c->scene_depth) {
        set_last_error("gsr_set_motion_vectors: the motion plane is the depth output or the scene depth");
        return GSR_ERR_INVALID;
    }
    if (c->ids_out && (const void *)motion_out_device == (const void *)c->ids_out) {
        set_last_error("gsr_set_motion_vectors: the motion plane is the splat ID plane");
        return GSR_ERR_INVALID;
    }
    c->motion_out = motion_out_device;   // read by the next render_enqueue: frames already enqueued keep their plane
    return GSR_OK;
}

GSR_API int gsr_set_splat_ids(gsr_ctx *c, uint32_t *ids_out_device) {
    if (!c) return GSR_ERR_INVALID;
    if (!ids_out_device) { c->ids_out = nullptr; return GSR_OK; }
    if (!c->depth_out) { set_last_error("gsr_set_splat_ids: depth compositing is off"); return GSR_ERR_STATE; }
    if (c->contrib) { set_last_error("gsr_set_splat_ids: splat contribution is on"); return GSR_ERR_STATE; }
    const void *p = ids_out_device;
    if (p == (const void *)c->depth_out || p == (const void *)c->scene_depth || p == (const void *)c->motion_out) {
        set_last_error("gsr_set_splat_ids: the ID plane is the depth output, the scene depth or the motion plane");
        return GSR_ERR_INVALID;
    }
    c->ids_out = ids_out_device;   // read by the next render_enqueue: frames already enqueued keep their plane
    return GSR_OK;
}

// ---- splat contribution (gsr_set_splat_contribution): the buffer is read when a frame is enqueued; the reset and the frame counter
// are ordered on the render stream, where every frame's compositor runs
static bool bytes_overlap(const void *a, size_t na, const void *b, size_t nb) {
    const char *x = static_cast<const char *>(a), *y = static_cast<const char *>(b);
    return a && b && x < y + nb && y < x + na;
}

GSR_API int gsr_set_splat_contribution(gsr_ctx *c, gsr_splat_contribution *accum_device, uint64_t slots) {
    if (!c) return GSR_ERR_INVALID;
    if (!accum_device) { c->contrib = nullptr; return GSR_OK; }
    if (slots != c->max_splats) {
        set_last_error("gsr_set_splat_contribution: %llu slots, the context has max_splats %llu", (unsigned long long)slots,
                       (unsigned long long)c->max_splats);
        return GSR_ERR_INVALID;
    }
    if (!c->depth_out) { set_last_error("gsr_set_splat_contribution: depth compositing is off"); return GSR_ERR_STATE; }
    const size_t bytes = sizeof(gsr_splat_contribution) * slots, pixels = (size_t)c->width * c->height;
    if (bytes_overlap(accum_device, bytes, c->depth_out, sizeof(float) * pixels) ||
        bytes_overlap(accum_device, bytes, c->scene_depth, sizeof(float) * pixels) ||
        bytes_overlap(accum_device, bytes, c->motion_out, 2 * sizeof(float) * pixels) ||
        bytes_overlap(accum_device, bytes, c->ids_out, 2 * sizeof(uint32_t) * pixels)) {
        set_last_error("gsr_set_splat_contribution: the buffer overlaps the depth output, the scene depth, the motion or the ID plane");
        return GSR_ERR_INVALID;
    }
    if (c->motion_out || c->ids_out) {
        set_last_error("gsr_set_splat_contribution: motion vectors or splat IDs are on");
        return GSR_ERR_STATE;
    }
    int rc = use_device(c->device);
    if (rc) return rc;
    if (!c->contrib_frames) {
        cudaError_t e = cudaMalloc((void **)&c->contrib_frames, sizeof(uint32_t));
        if (e != cudaSuccess) {
            c->contrib_frames = nullptr;
            set_last_error("gsr_set_splat_contribution: frame counter -> %s", cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
    }
    GSR_CUDA_TRY(cudaMemsetAsync(c->contrib_frames, 0, sizeof(uint32_t), c->stream));
    c->contrib = accum_device;   // read by the next render_enqueue: frames already enqueued keep their buffer
    return GSR_OK;
}

GSR_API int gsr_reset_splat_contribution(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    if (!c->contrib) { set_last_error("gsr_reset_splat_contribution: no contribution buffer is set"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaMemsetAsync(c->contrib, 0, sizeof(gsr_splat_contribution) * c->max_splats, c->stream));
    GSR_CUDA_TRY(cudaMemsetAsync(c->contrib_frames, 0, sizeof(uint32_t), c->stream));
    return GSR_OK;
}

GSR_API int gsr_splat_contribution_frames(gsr_ctx *c, uint32_t *frames) {
    if (!c || !frames) { set_last_error("gsr_splat_contribution_frames: NULL argument"); return GSR_ERR_INVALID; }
    if (!c->contrib) { set_last_error("gsr_splat_contribution_frames: no contribution buffer is set"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaMemcpyAsync(frames, c->contrib_frames, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return GSR_OK;
}

GSR_API int gsr_reset_motion(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    c->mot_last.valid = false;   // the next frame is its own previous state
    return GSR_OK;
}

// [A | t] -> [A | t, B | u] with B = A^-1, u = -A^-1 t in double precision, rounded to float.  False: non-finite or singular.
static bool instance_inverse(const float m[12], float out[24]) {
    double A[3][3], t[3];   // A[c][r]
    for (int e = 0; e < 12; ++e) if (!isfinite(m[e])) return false;
    for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) A[c][r] = m[3 * c + r];
    for (int r = 0; r < 3; ++r) t[r] = m[9 + r];
    auto a = [&](int r, int col) { return A[col][r]; };   // row r, column col
    const double c00 = a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1), c01 = a(1, 2) * a(2, 0) - a(1, 0) * a(2, 2), c02 = a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0);
    const double det = a(0, 0) * c00 + a(0, 1) * c01 + a(0, 2) * c02;
    if (!(det != 0.0) || !isfinite(det)) return false;
    double inv[3][3];   // inv[r][col] = (A^-1) row r, column col = adj / det
    inv[0][0] = c00 / det; inv[0][1] = (a(0, 2) * a(2, 1) - a(0, 1) * a(2, 2)) / det; inv[0][2] = (a(0, 1) * a(1, 2) - a(0, 2) * a(1, 1)) / det;
    inv[1][0] = c01 / det; inv[1][1] = (a(0, 0) * a(2, 2) - a(0, 2) * a(2, 0)) / det; inv[1][2] = (a(0, 2) * a(1, 0) - a(0, 0) * a(1, 2)) / det;
    inv[2][0] = c02 / det; inv[2][1] = (a(0, 1) * a(2, 0) - a(0, 0) * a(2, 1)) / det; inv[2][2] = (a(0, 0) * a(1, 1) - a(0, 1) * a(1, 0)) / det;
    memcpy(out, m, sizeof(float) * 12);
    for (int col = 0; col < 3; ++col)
        for (int r = 0; r < 3; ++r) out[12 + 3 * col + r] = (float)inv[r][col];
    for (int r = 0; r < 3; ++r) out[21 + r] = (float)-(inv[r][0] * t[0] + inv[r][1] * t[1] + inv[r][2] * t[2]);
    for (int e = 12; e < 24; ++e) if (!isfinite(out[e])) return false;
    return true;
}

// New drawn-id layout: device tables, ring and record / look-back / sort capacity for n instances drawing D ids.  The caller synchronised.
static int instance_layout(gsr_ctx *c, const uint64_t *range, uint32_t n, uint64_t drawn) {
    auto &I = c->inst;
    const uint32_t blocks = projection_num_blocks((uint32_t)drawn);
    if (drawn > c->rec_entries) {   // record tables for max(max_splats, D) drawn ids
        float4 *r1 = nullptr, *r2 = nullptr;
        GSR_CUDA_TRY(cudaMalloc((void **)&r1, sizeof(float4) * 3ull * drawn));
        cudaError_t e = cudaMalloc((void **)&r2, sizeof(float4) * 3ull * drawn);
        if (e != cudaSuccess) { cudaFree(r1); set_last_error("cudaMalloc(records, D = %llu) -> %s", (unsigned long long)drawn, cudaGetErrorString(e)); return GSR_ERR_OOM; }
        GSR_CUDA_TRY(cudaMemset(r1, 0, sizeof(float4) * 3ull * drawn));
        GSR_CUDA_TRY(cudaMemset(r2, 0, sizeof(float4) * 3ull * drawn));
        cudaFree(c->records); cudaFree(c->records2);
        c->records = r1; c->records2 = r2; c->records_cur = r1; c->rec_entries = drawn;
    }
    if (blocks > c->lookback_cap) {
        unsigned long long *lb = nullptr;
        GSR_CUDA_TRY(cudaMalloc((void **)&lb, sizeof(unsigned long long) * ((size_t)blocks + 2u * GROUP_MAX * GROUP_MAX)));
        cudaFree(c->lookback);
        c->lookback = lb; c->lookback_cap = blocks;
    }
    if (n > I.cap) {
        cudaFree(I.desc); cudaFree(I.frame); I.desc = nullptr; I.frame = nullptr;
        if (I.ring) cudaFreeHost(I.ring);
        I.ring = I.ring_dev = nullptr; I.cap = 0;
        GSR_CUDA_TRY(cudaMalloc((void **)&I.desc, sizeof(InstanceDesc) * n));
        GSR_CUDA_TRY(cudaMalloc((void **)&I.frame, sizeof(float) * 2ull * (INSTANCE_FRAME_FLOATS + INSTANCE_APPEARANCE_FLOATS + INSTANCE_PREV_FLOATS) * n));
        if (cudaHostAlloc((void **)&I.ring, sizeof(float) * GSR_INSTANCE_RING * INSTANCE_SLOT_FLOATS * (size_t)n, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError(); I.ring = nullptr; set_last_error("cudaHostAlloc(instance ring) failed"); return GSR_ERR_OOM;
        }
        GSR_CUDA_TRY(cudaHostGetDevicePointer((void **)&I.ring_dev, I.ring, 0));
        I.cap = n;
    }
    for (int i = 0; i < GSR_INSTANCE_RING; ++i) {
        if (!I.ev[i]) GSR_CUDA_TRY(cudaEventCreateWithFlags(&I.ev[i], cudaEventDisableTiming));
        I.ev_used[i] = false;
    }
    // static tables: descriptors and the instance of every warp of the grid (padding warps of the last CTA: none)
    InstanceDesc *desc = new (std::nothrow) InstanceDesc[n ? n : 1];
    const size_t nwarps = (size_t)blocks * (PROJ_THREADS / 32);
    uint32_t *warps = new (std::nothrow) uint32_t[nwarps ? nwarps : 1];
    if (!desc || !warps) { delete[] desc; delete[] warps; return GSR_ERR_OOM; }
    uint32_t w = 0;
    for (uint32_t k = 0; k < n; ++k) {
        desc[k].first = range[2 * k]; desc[k].count = (uint32_t)range[2 * k + 1]; desc[k].warp0 = w;
        const uint32_t nw = (uint32_t)((range[2 * k + 1] + 31ull) / 32ull);
        for (uint32_t j = 0; j < nw; ++j) warps[w + j] = k;
        w += nw;
    }
    for (size_t j = w; j < nwarps; ++j) warps[j] = 0xFFFFFFFFu;
    cudaFree(I.warps); I.warps = nullptr;
    cudaError_t e = cudaMalloc((void **)&I.warps, sizeof(uint32_t) * (nwarps ? nwarps : 1));
    if (e == cudaSuccess && n) e = cudaMemcpy(I.desc, desc, sizeof(InstanceDesc) * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && nwarps) e = cudaMemcpy(I.warps, warps, sizeof(uint32_t) * nwarps, cudaMemcpyHostToDevice);
    delete[] desc; delete[] warps;
    if (e != cudaSuccess) { set_last_error("instance tables -> %s", cudaGetErrorString(e)); return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA; }
    // the first instanced frame must not overflow: the initial capacity rule (factor x splats) applied to the drawn ids
    if (drawn > c->max_splats) {
        int rc = grow_capacity(c, c->dup_factor * drawn);
        if (rc) return rc;
    }
    return GSR_OK;
}

GSR_API int gsr_set_instances(gsr_ctx *c, const gsr_instance *instances, uint32_t n) {
    if (!c) return GSR_ERR_INVALID;
    if (n == 0) {   // tables stay allocated; frames in flight keep reading them
        c->inst.n = 0; c->inst.drawn = 0;
        delete[] c->inst.app; c->inst.app = nullptr;
        return GSR_OK;
    }
    if (!instances) { set_last_error("gsr_set_instances: NULL array with n = %u", n); return GSR_ERR_INVALID; }
    if (n > GSR_MAX_INSTANCES) { set_last_error("gsr_set_instances: %u instances exceed GSR_MAX_INSTANCES (%d)", n, GSR_MAX_INSTANCES); return GSR_ERR_INVALID; }
    if (sharded(c)) { set_last_error("gsr_set_instances: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    float *xf = new (std::nothrow) float[(size_t)INSTANCE_XFORM_FLOATS * n];
    uint64_t *range = new (std::nothrow) uint64_t[2ull * n];
    if (!xf || !range) { delete[] xf; delete[] range; return GSR_ERR_OOM; }
    uint64_t warps = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const gsr_instance &g = instances[k];
        const char *bad = nullptr;
        if (g.count > c->max_splats || g.first > c->max_splats - g.count) bad = "range beyond max_splats";
        else if (!instance_inverse(g.to_frame, xf + (size_t)INSTANCE_XFORM_FLOATS * k)) bad = "non-finite or singular transform";
        if (bad) {
            set_last_error("gsr_set_instances: instance %u [%llu, +%llu): %s", k, (unsigned long long)g.first, (unsigned long long)g.count, bad);
            delete[] xf; delete[] range;
            return GSR_ERR_INVALID;
        }
        range[2 * k] = g.first; range[2 * k + 1] = g.count;
        warps += (g.count + 31ull) / 32ull;
    }
    const uint64_t drawn = 32ull * warps;
    if (drawn >= (1ull << 32) - 256ull) {
        set_last_error("gsr_set_instances: %llu drawn ids (padded to whole warps) must be < 2^32 - 256", (unsigned long long)drawn);
        delete[] xf; delete[] range;
        return GSR_ERR_INVALID;
    }
    auto &I = c->inst;
    const bool same_layout = I.n == n && I.range && memcmp(I.range, range, sizeof(uint64_t) * 2ull * n) == 0;
    if (!same_layout) {   // new drawn-id layout: may synchronise and reallocate
        int rc = use_device(c->device);
        if (!rc) {
            cudaError_t e = cudaStreamSynchronize(c->front_stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c->copy_stream);
            if (e != cudaSuccess) { set_last_error("gsr_set_instances: sync -> %s", cudaGetErrorString(e)); rc = GSR_ERR_CUDA; }
        }
        c->front_gate = nullptr;
        I.n = 0; I.drawn = 0;   // a failure below leaves instancing off
        delete[] I.app; I.app = nullptr;   // a new layout starts at the default appearance
        if (!rc) rc = instance_layout(c, range, n, drawn);
        if (rc) { delete[] xf; delete[] range; return rc; }
        delete[] I.range;
        I.range = range;
    } else {
        delete[] range;
    }
    // transforms: the host copy the next frames hand to the ring
    delete[] I.xf;
    I.xf = xf;
    I.n = n; I.drawn = drawn;
    return GSR_OK;
}

GSR_API int gsr_set_instance_appearance(gsr_ctx *c, const gsr_instance_appearance *appearance, uint32_t n) {
    if (!c) return GSR_ERR_INVALID;
    auto &I = c->inst;
    if (n == 0 && (!appearance || I.n == 0)) {   // the default for every instance
        delete[] I.app; I.app = nullptr;
        return GSR_OK;
    }
    if (!appearance) { set_last_error("gsr_set_instance_appearance: NULL array with n = %u", n); return GSR_ERR_INVALID; }
    if (n != I.n) { set_last_error("gsr_set_instance_appearance: n = %u, but %u instances are set", n, I.n); return GSR_ERR_INVALID; }
    for (uint32_t k = 0; k < n; ++k) {
        const gsr_instance_appearance &p = appearance[k];
        const char *bad = nullptr;
        for (int i = 0; i < 3; ++i)
            if (!(p.tint[i] >= 0.0f && p.tint[i] <= GSR_TINT_MAX)) bad = "tint outside [0, GSR_TINT_MAX] or not a number";
        if (!(p.opacity >= 0.0f && p.opacity <= 1.0f)) bad = "opacity outside [0, 1] or not a number";
        if (bad) { set_last_error("gsr_set_instance_appearance: instance %u: %s", k, bad); return GSR_ERR_INVALID; }
    }
    if (!I.app) {   // (an existing array holds I.n = n entries: every layout change drops it)
        I.app = new (std::nothrow) gsr_instance_appearance[n];
        if (!I.app) return GSR_ERR_OOM;
    }
    memcpy(I.app, appearance, sizeof(gsr_instance_appearance) * n);
    return GSR_OK;
}

GSR_API int gsr_set_sh_degree(gsr_ctx *c, int32_t degree) {
    if (!c) return GSR_ERR_INVALID;
    if (degree < -1 || degree > c->sh_bands - 1) {
        set_last_error("gsr_set_sh_degree: degree %d outside -1..%d (the stored degree)", degree, c->sh_bands - 1);
        return GSR_ERR_INVALID;
    }
    if (degree >= 0 && degree < SH_BANDS_MAX - 1 && sharded(c)) { set_last_error("gsr_set_sh_degree: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    c->sh_degree = degree;   // read by the next render_enqueue: frames already enqueued keep their degree
    return GSR_OK;
}

GSR_API int gsr_set_antialiasing(gsr_ctx *c, float filter_variance) {
    if (!c) return GSR_ERR_INVALID;
    if (!(filter_variance >= 0.0f && filter_variance <= 64.0f)) {   // NaN fails both
        set_last_error("gsr_set_antialiasing: filter variance %g outside 0..64 px^2", (double)filter_variance);
        return GSR_ERR_INVALID;
    }
    if (filter_variance > 0.0f && sharded(c)) { set_last_error("gsr_set_antialiasing: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    c->aa_variance = filter_variance;   // read by the next render_enqueue: frames already enqueued keep their filter
    return GSR_OK;
}

GSR_API int gsr_set_depth_order(gsr_ctx *c, int32_t mode) {
    if (!c) return GSR_ERR_INVALID;
    if (mode != GSR_DEPTH_ORDER_KEY16 && mode != GSR_DEPTH_ORDER_VIEW_DEPTH) {
        set_last_error("gsr_set_depth_order: mode %d is neither GSR_DEPTH_ORDER_KEY16 nor GSR_DEPTH_ORDER_VIEW_DEPTH", mode);
        return GSR_ERR_INVALID;
    }
    if (mode == GSR_DEPTH_ORDER_VIEW_DEPTH) {
        if (sharded(c)) { set_last_error("gsr_set_depth_order: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
        int rc = use_device(c->device);
        if (rc) return rc;
        if ((rc = alloc_depth_order(c))) return rc;   // the first switch only (cudaMalloc may synchronise)
    }
    c->depth_order = mode;   // read by the next render_enqueue: frames already enqueued keep their order
    return GSR_OK;
}

GSR_API int gsr_set_cutouts(gsr_ctx *c, const gsr_cutout *cutouts, uint32_t n) {
    if (!c) return GSR_ERR_INVALID;
    if (n > GSR_MAX_CUTOUTS) { set_last_error("gsr_set_cutouts: %u volumes, at most GSR_MAX_CUTOUTS = %d", n, GSR_MAX_CUTOUTS); return GSR_ERR_INVALID; }
    if (n > 0 && !cutouts) { set_last_error("gsr_set_cutouts: cutouts == NULL with n = %u", n); return GSR_ERR_INVALID; }
    for (uint32_t i = 0; i < n; ++i) {
        const gsr_cutout &v = cutouts[i];
        for (int e = 0; e < 12; ++e) {
            if (!(fabsf(v.to_local[e]) <= 3.402823466e38f)) { set_last_error("gsr_set_cutouts: volume %u has a non-finite to_local[%d]", i, e); return GSR_ERR_INVALID; }
        }
        if (v.shape != GSR_CUTOUT_BOX && v.shape != GSR_CUTOUT_ELLIPSOID) { set_last_error("gsr_set_cutouts: volume %u: unknown shape %d", i, v.shape); return GSR_ERR_INVALID; }
        if (v.action != GSR_CUTOUT_KEEP && v.action != GSR_CUTOUT_REMOVE) { set_last_error("gsr_set_cutouts: volume %u: unknown action %d", i, v.action); return GSR_ERR_INVALID; }
        if (v.space != GSR_CUTOUT_FRAME && v.space != GSR_CUTOUT_SOURCE) { set_last_error("gsr_set_cutouts: volume %u: unknown space %d", i, v.space); return GSR_ERR_INVALID; }
    }
    if (n > 0 && sharded(c)) { set_last_error("gsr_set_cutouts: %s", SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    // split by action, KEEP volumes first (the rule does not depend on the order): the kernel runs one loop over each list
    CutoutArgs s = {};
    for (int pass = 0; pass < 2; ++pass) {
        for (uint32_t i = 0; i < n; ++i) {
            const gsr_cutout &v = cutouts[i];
            if (v.action != (pass ? GSR_CUTOUT_REMOVE : GSR_CUTOUT_KEEP)) continue;
            CutoutVolume &d = s.vol[s.n_keep + s.n_remove];
            memcpy(d.m, v.to_local, sizeof d.m);
            d.kind = v.shape | (v.space << 1);
            if (pass) s.n_remove += 1;
            else s.n_keep += 1;
        }
    }
    c->cutouts = s;   // read by the next render_enqueue: frames already enqueued keep their set
    return GSR_OK;
}

// ---- splat selection (gsr_select_*): the masks live on the device; every operation is enqueued on the projections' stream ----------
// The stream the projections run on (the front stream with front / back overlap): every mask operation is enqueued there, so it is
// ordered after the projections of the frames enqueued before it and before those of the frames after it.  The sort and the
// compositor never read the masks, so an operation does not hold the next frame's projection behind the previous frame's compositor.
// (gsr_debug_pipeline synchronises both streams, so a switch of the overlap mode never leaves an operation behind.)
static cudaStream_t mask_stream(const gsr_ctx *c) { return (c->overlap > 0 && c->front_stream) ? c->front_stream : c->stream; }

static bool select_op_valid(int32_t op) { return op >= GSR_SELECT_SET && op <= GSR_SELECT_TOGGLE; }

// The first call that can set a bit puts the masks in use: allocated and zeroed once (GSR_ERR_OOM / GSR_ERR_CUDA keep the state as it
// was), zeroed again by gsr_clear_splat_masks, so a later first call only switches them on.
static int masks_use(gsr_ctx *c, const char *where) {
    if (sharded(c)) { set_last_error("%s: %s", where, SINGLE_CONTEXT_ONLY); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    gsr_ctx::Masks &m = c->masks;
    if (!m.hidden) {
        const uint32_t words = (uint32_t)((c->max_splats + 31ull) / 32ull);
        const size_t mask_bytes = (2 * sizeof(unsigned long long) + sizeof(uint32_t) * 3ull * words + 7ull) & ~7ull;
        const size_t bytes = mask_bytes + sizeof(unsigned long long) * compact_lookback_words(words);
        void *buf = nullptr;
        cudaEvent_t ev = nullptr;
        cudaError_t e = cudaMalloc(&buf, bytes);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaMemsetAsync(buf, 0, bytes, mask_stream(c));
        if (e != cudaSuccess) {
            cudaFree(buf);
            if (ev) cudaEventDestroy(ev);
            set_last_error("%s: splat masks of %llu B -> %s", where, (unsigned long long)bytes, cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
        m.counts = static_cast<unsigned long long *>(buf);
        m.hidden = reinterpret_cast<uint32_t *>(m.counts + 2);
        m.selected = m.hidden + words;
        m.scratch = m.selected + words;
        m.lookback = reinterpret_cast<unsigned long long *>(static_cast<char *>(buf) + mask_bytes);
        m.words = words;
        m.ids_ready = ev;
    }
    m.on = true;
    return GSR_OK;
}

// The tested range and transform of instance `instance` (-1: every splat, no transform)
static int select_range(const gsr_ctx *c, const char *where, int32_t instance, SelectArgs &a) {
    if (instance < -1 || instance >= (int32_t)c->inst.n) {
        set_last_error("%s: instance %d outside the current layout (-1 or 0..%u)", where, instance, c->inst.n ? c->inst.n - 1u : 0u);
        return GSR_ERR_INVALID;
    }
    if (instance < 0) { a.first = 0; a.count = c->max_splats; a.instanced = 0; return GSR_OK; }
    a.first = c->inst.range[2 * instance]; a.count = c->inst.range[2 * instance + 1]; a.instanced = 1;
    memcpy(a.A, c->inst.xf + (size_t)instance * INSTANCE_XFORM_FLOATS, sizeof a.A);
    return GSR_OK;
}

static int select_region(gsr_ctx *c, const char *where, SelectArgs &a, int kind, int32_t op) {
    int rc = masks_use(c, where);
    if (rc) return rc;
    a.selected = c->masks.selected; a.hidden = c->masks.hidden; a.words = c->masks.words; a.op = (uint32_t)op;
    a.max_splats = c->max_splats; a.plane0 = c->soa;
    return launch_select_region(a, kind, mask_stream(c));
}

GSR_API int gsr_select_all(gsr_ctx *c, int32_t op) {
    if (!c) return GSR_ERR_INVALID;
    if (!select_op_valid(op)) { set_last_error("gsr_select_all: unknown op %d", op); return GSR_ERR_INVALID; }
    SelectArgs a;
    memset(&a, 0, sizeof a);
    a.first = 0; a.count = c->max_splats;
    return select_region(c, "gsr_select_all", a, SELECT_ALL, op);
}

GSR_API int gsr_select_polygon(gsr_ctx *c, const float view_proj[32], float model_scale, int32_t instance, const float *xy, uint32_t n,
                               int32_t op) {
    if (!c || !view_proj || !xy) { set_last_error("gsr_select_polygon: NULL argument"); return GSR_ERR_INVALID; }
    if (!select_op_valid(op)) { set_last_error("gsr_select_polygon: unknown op %d", op); return GSR_ERR_INVALID; }
    if (n < 3 || n > GSR_MAX_SELECT_VERTICES) { set_last_error("gsr_select_polygon: %u vertices, need 3..%d", n, GSR_MAX_SELECT_VERTICES); return GSR_ERR_INVALID; }
    for (uint32_t i = 0; i < 2 * n; ++i) {
        if (!(fabsf(xy[i]) <= 3.402823466e38f)) { set_last_error("gsr_select_polygon: vertex %u is not finite", i / 2); return GSR_ERR_INVALID; }
    }
    if (c->width == 0) { set_last_error("gsr_select_polygon before gsr_resize"); return GSR_ERR_STATE; }
    SelectArgs a;
    memset(&a, 0, sizeof a);
    int rc = select_range(c, "gsr_select_polygon", instance, a);
    if (rc) return rc;
    a.model_scale = model_scale;
    memcpy(a.vp, view_proj, sizeof a.vp);
    a.fw = (float)(c->width - 1); a.fh = (float)(c->height - 1);
    a.n = n;
    for (uint32_t i = 0; i < n; ++i) a.xy[i] = make_float2(xy[2 * i], xy[2 * i + 1]);
    return select_region(c, "gsr_select_polygon", a, SELECT_POLYGON, op);
}

GSR_API int gsr_select_volume(gsr_ctx *c, const gsr_cutout *volume, float model_scale, int32_t instance, int32_t op) {
    if (!c || !volume) { set_last_error("gsr_select_volume: NULL argument"); return GSR_ERR_INVALID; }
    if (!select_op_valid(op)) { set_last_error("gsr_select_volume: unknown op %d", op); return GSR_ERR_INVALID; }
    for (int e = 0; e < 12; ++e) {
        if (!(fabsf(volume->to_local[e]) <= 3.402823466e38f)) { set_last_error("gsr_select_volume: non-finite to_local[%d]", e); return GSR_ERR_INVALID; }
    }
    if (volume->shape != GSR_CUTOUT_BOX && volume->shape != GSR_CUTOUT_ELLIPSOID) { set_last_error("gsr_select_volume: unknown shape %d", volume->shape); return GSR_ERR_INVALID; }
    if (volume->space != GSR_CUTOUT_FRAME && volume->space != GSR_CUTOUT_SOURCE) { set_last_error("gsr_select_volume: unknown space %d", volume->space); return GSR_ERR_INVALID; }
    SelectArgs a;
    memset(&a, 0, sizeof a);
    int rc = select_range(c, "gsr_select_volume", instance, a);
    if (rc) return rc;
    a.model_scale = model_scale;
    memcpy(a.vol.m, volume->to_local, sizeof a.vol.m);
    a.vol.kind = volume->shape | (volume->space << 1);
    return select_region(c, "gsr_select_volume", a, SELECT_VOLUME, op);
}

GSR_API int gsr_select_ids(gsr_ctx *c, const uint32_t *ids_device, int32_t x0, int32_t y0, int32_t x1, int32_t y1, int32_t op) {
    if (!c || !ids_device) { set_last_error("gsr_select_ids: NULL argument"); return GSR_ERR_INVALID; }
    if (!select_op_valid(op)) { set_last_error("gsr_select_ids: unknown op %d", op); return GSR_ERR_INVALID; }
    if (c->width == 0) { set_last_error("gsr_select_ids before gsr_resize"); return GSR_ERR_STATE; }
    if (x0 < 0 || y0 < 0 || x1 < x0 || y1 < y0 || x1 > c->width || y1 > c->height) {
        set_last_error("gsr_select_ids: rectangle [%d,%d) x [%d,%d) outside the %dx%d image", x0, x1, y0, y1, c->width, c->height);
        return GSR_ERR_INVALID;
    }
    int rc = masks_use(c, "gsr_select_ids");
    if (rc) return rc;
    cudaStream_t ms = mask_stream(c);
    if (ms != c->stream) {   // the ID plane is written by the compositor of an earlier frame, on the render stream
        GSR_CUDA_TRY(cudaEventRecord(c->masks.ids_ready, c->stream));
        GSR_CUDA_TRY(cudaStreamWaitEvent(ms, c->masks.ids_ready, 0));
    }
    const bool inst = c->inst.n > 0;
    if ((rc = launch_select_ids(ids_device, c->width, x0, y0, x1, y1, inst ? c->inst.warps : nullptr, c->inst.desc,
                                inst ? (uint32_t)(c->inst.drawn / 32ull) : 0u, c->max_splats, c->masks.scratch, c->masks.selected,
                                c->masks.hidden, c->masks.words, (uint32_t)op, ms))) return rc;
    return GSR_OK;
}

GSR_API int gsr_hide_selection(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    if (!c->masks.on) return GSR_OK;   // nothing is selected
    int rc = use_device(c->device);
    if (rc) return rc;
    return launch_hide_selection(c->masks.hidden, c->masks.selected, c->masks.words, mask_stream(c));
}

GSR_API int gsr_unhide_all(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    if (!c->masks.on) return GSR_OK;   // nothing is hidden
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaMemsetAsync(c->masks.hidden, 0, sizeof(uint32_t) * c->masks.words, mask_stream(c)));
    return GSR_OK;
}

GSR_API int gsr_clear_splat_masks(gsr_ctx *c) {
    if (!c) return GSR_ERR_INVALID;
    if (!c->masks.on) return GSR_OK;
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaMemsetAsync(c->masks.hidden, 0, sizeof(uint32_t) * 2ull * c->masks.words, mask_stream(c)));   // hidden | selected
    c->masks.on = false;
    return GSR_OK;
}

static int check_mask_words(const gsr_ctx *c, const char *where, const void *hidden, const void *selected, uint64_t words) {
    if (!hidden || !selected) { set_last_error("%s: NULL array", where); return GSR_ERR_INVALID; }
    const uint64_t want = (c->max_splats + 31ull) / 32ull;
    if (words != want) { set_last_error("%s: %llu words, need ceil(max_splats / 32) = %llu", where, (unsigned long long)words, (unsigned long long)want); return GSR_ERR_INVALID; }
    return GSR_OK;
}

GSR_API int gsr_get_splat_masks(gsr_ctx *c, uint32_t *hidden, uint32_t *selected, uint64_t words) {
    if (!c) return GSR_ERR_INVALID;
    int rc = check_mask_words(c, "gsr_get_splat_masks", hidden, selected, words);
    if (rc) return rc;
    if (!c->masks.on) {
        memset(hidden, 0, sizeof(uint32_t) * words);
        memset(selected, 0, sizeof(uint32_t) * words);
        return GSR_OK;
    }
    if ((rc = use_device(c->device))) return rc;
    cudaStream_t ms = mask_stream(c);
    GSR_CUDA_TRY(cudaMemcpyAsync(hidden, c->masks.hidden, sizeof(uint32_t) * words, cudaMemcpyDeviceToHost, ms));
    GSR_CUDA_TRY(cudaMemcpyAsync(selected, c->masks.selected, sizeof(uint32_t) * words, cudaMemcpyDeviceToHost, ms));
    GSR_CUDA_TRY(cudaStreamSynchronize(ms));
    return GSR_OK;
}

GSR_API int gsr_set_splat_masks(gsr_ctx *c, const uint32_t *hidden, const uint32_t *selected, uint64_t words) {
    if (!c) return GSR_ERR_INVALID;
    int rc = check_mask_words(c, "gsr_set_splat_masks", hidden, selected, words);
    if (rc) return rc;
    const uint32_t tail = (uint32_t)(c->max_splats & 31ull), past = tail ? ~((1u << tail) - 1u) : 0u;   // bits past max_splats
    for (uint64_t w = 0; w < words; ++w) {
        if (hidden[w] & selected[w]) { set_last_error("gsr_set_splat_masks: word %llu has splats both hidden and selected", (unsigned long long)w); return GSR_ERR_INVALID; }
    }
    if ((hidden[words - 1] | selected[words - 1]) & past) { set_last_error("gsr_set_splat_masks: bits past max_splats"); return GSR_ERR_INVALID; }
    if ((rc = masks_use(c, "gsr_set_splat_masks"))) return rc;
    // pageable host memory: each copy has read its source when it returns
    GSR_CUDA_TRY(cudaMemcpyAsync(c->masks.hidden, hidden, sizeof(uint32_t) * words, cudaMemcpyHostToDevice, mask_stream(c)));
    GSR_CUDA_TRY(cudaMemcpyAsync(c->masks.selected, selected, sizeof(uint32_t) * words, cudaMemcpyHostToDevice, mask_stream(c)));
    return GSR_OK;
}

GSR_API int gsr_splat_mask_counts(gsr_ctx *c, uint64_t *selected, uint64_t *hidden) {
    if (!c || !selected || !hidden) { set_last_error("gsr_splat_mask_counts: NULL argument"); return GSR_ERR_INVALID; }
    *selected = 0; *hidden = 0;
    if (!c->masks.on) return GSR_OK;
    int rc = use_device(c->device);
    cudaStream_t ms = mask_stream(c);
    if (rc || (rc = launch_mask_counts(c->masks.selected, c->masks.hidden, c->masks.words, c->masks.counts, ms))) return rc;
    unsigned long long n[2] = {0ull, 0ull};
    GSR_CUDA_TRY(cudaMemcpyAsync(n, c->masks.counts, sizeof n, cudaMemcpyDeviceToHost, ms));
    GSR_CUDA_TRY(cudaStreamSynchronize(ms));
    *selected = n[0]; *hidden = n[1];
    return GSR_OK;
}

GSR_API int gsr_set_selection_style(gsr_ctx *c, const float rgb[3], float strength) {
    if (!c || !rgb) { set_last_error("gsr_set_selection_style: NULL argument"); return GSR_ERR_INVALID; }
    for (int i = 0; i < 3; ++i) {
        if (!(rgb[i] >= 0.0f && rgb[i] <= GSR_TINT_MAX)) { set_last_error("gsr_set_selection_style: rgb[%d] = %g outside [0, GSR_TINT_MAX]", i, (double)rgb[i]); return GSR_ERR_INVALID; }
    }
    if (!(strength >= 0.0f && strength <= 1.0f)) { set_last_error("gsr_set_selection_style: strength %g outside [0, 1]", (double)strength); return GSR_ERR_INVALID; }
    memcpy(c->masks.rgb, rgb, sizeof c->masks.rgb);
    c->masks.strength = strength;   // read by the next render_enqueue
    return GSR_OK;
}

// ---- splat transform and colour edits, store snapshots ---------------------------------------------------------------------------
// Enqueued on the projections' stream (mask_stream) like the mask operations, so they come before the projections of later frames.
// Unlike them they also wait for the render stream's work: the previous frame's compositor reads plane 0 for the motion vectors of
// instanced frames.
static int store_stream(gsr_ctx *c, cudaStream_t *out) {
    const cudaStream_t ms = mask_stream(c);
    if (ms != c->stream) {
        if (!c->store_ready) GSR_CUDA_TRY(cudaEventCreateWithFlags(&c->store_ready, cudaEventDisableTiming));
        GSR_CUDA_TRY(cudaEventRecord(c->store_ready, c->stream));
        GSR_CUDA_TRY(cudaStreamWaitEvent(ms, c->store_ready, 0));
    }
    *out = ms;
    return GSR_OK;
}

static uint64_t store_bytes(const gsr_ctx *c) { return sizeof(float4) * (uint64_t)soa_planes(c->sh_bands, sh_half(c)) * c->plane_stride; }

GSR_API int gsr_transform_selection(gsr_ctx *c, const float to_source[12], const void *src_store) {
    if (!c || !to_source) { set_last_error("gsr_transform_selection: NULL argument"); return GSR_ERR_INVALID; }
    for (int e = 0; e < 12; ++e) {
        if (!(fabsf(to_source[e]) <= 3.402823466e38f)) { set_last_error("gsr_transform_selection: non-finite to_source[%d]", e); return GSR_ERR_INVALID; }
    }
    TransformArgs a;
    if (edit_transform_matrices(to_source, a.m)) { set_last_error("gsr_transform_selection: det(L) is 0 or not finite"); return GSR_ERR_INVALID; }
    if (!c->masks.on) { set_last_error("gsr_transform_selection: the splat masks are not in use"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    a.dst = c->soa;
    a.src = src_store ? static_cast<const float4 *>(src_store) : c->soa;
    a.plane_stride = c->plane_stride;
    a.selected = c->masks.selected;
    a.words = c->masks.words;
    if ((rc = launch_transform_selection(a, c->sh_bands, sh_half(c), s))) return rc;
    memcpy(c->edit_last, a.m, sizeof c->edit_last);
    return GSR_OK;
}

GSR_API int gsr_recolor_selection(gsr_ctx *c, const gsr_color_edit *e, const void *src_store) {
    if (!c || !e) { set_last_error("gsr_recolor_selection: NULL argument"); return GSR_ERR_INVALID; }
    for (int i = 0; i < 12; ++i) {
        if (!(fabsf(e->matrix[i]) <= GSR_TINT_MAX)) { set_last_error("gsr_recolor_selection: matrix[%d] = %g not finite or beyond GSR_TINT_MAX", i, (double)e->matrix[i]); return GSR_ERR_INVALID; }
    }
    for (int l = 0; l < 3; ++l) {
        if (!(e->band_scale[l] >= 0.0f && e->band_scale[l] <= GSR_TINT_MAX)) { set_last_error("gsr_recolor_selection: band_scale[%d] = %g outside [0, GSR_TINT_MAX]", l, (double)e->band_scale[l]); return GSR_ERR_INVALID; }
    }
    if (!(e->opacity_scale >= 0.0f && e->opacity_scale <= GSR_TINT_MAX)) { set_last_error("gsr_recolor_selection: opacity_scale = %g outside [0, GSR_TINT_MAX]", (double)e->opacity_scale); return GSR_ERR_INVALID; }
    if (!(e->opacity_offset >= -1.0f && e->opacity_offset <= 1.0f)) { set_last_error("gsr_recolor_selection: opacity_offset = %g outside [-1, 1]", (double)e->opacity_offset); return GSR_ERR_INVALID; }
    if (!c->masks.on) { set_last_error("gsr_recolor_selection: the splat masks are not in use"); return GSR_ERR_STATE; }
    RecolorArgs a;
    edit_color_constants(e, a.k);
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    a.dst = c->soa;
    a.src = src_store ? static_cast<const float4 *>(src_store) : c->soa;
    a.plane_stride = c->plane_stride;
    a.selected = c->masks.selected;
    a.words = c->masks.words;
    if ((rc = launch_recolor_selection(a, c->sh_bands, sh_half(c), s))) return rc;
    memcpy(c->color_last, a.k, sizeof c->color_last);
    return GSR_OK;
}

// ---- splat delete and duplicate: structural edits of the store, enqueued like the edits above; each synchronises the host once ----
GSR_API int gsr_delete_hidden(gsr_ctx *c, uint64_t *kept_out) {
    if (!c || !kept_out) { set_last_error("gsr_delete_hidden: NULL argument"); return GSR_ERR_INVALID; }
    if (!c->masks.on) { set_last_error("gsr_delete_hidden: the splat masks are not in use"); return GSR_ERR_STATE; }
    if (c->inst.n > 0) { set_last_error("gsr_delete_hidden: instances are set (their ranges would point at other splats)"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    const uint64_t n = c->num_splats;
    CompactArgs a;
    a.soa = c->soa; a.plane_stride = c->plane_stride; a.n = n;
    a.hidden = c->masks.hidden; a.selected = c->masks.selected; a.sel_out = c->masks.scratch;
    a.lookback = c->masks.lookback; a.total = c->masks.counts;
    GSR_CUDA_TRY(cudaMemsetAsync(c->masks.counts, 0, sizeof(unsigned long long), s));
    if ((rc = launch_compact_store(a, COMPACT_DELETE, c->sh_bands, sh_half(c), s))) return rc;
    unsigned long long k = 0ull;
    GSR_CUDA_TRY(cudaMemcpyAsync(&k, c->masks.counts, sizeof k, cudaMemcpyDeviceToHost, s));
    GSR_CUDA_TRY(cudaStreamSynchronize(s));
    if ((rc = launch_delete_finish(c->soa, c->plane_stride, soa_planes(c->sh_bands, sh_half(c)), k, n, c->masks.hidden, c->masks.selected,
                                   c->masks.scratch, c->masks.words, s))) return rc;
    c->num_splats = k;
    *kept_out = k;
    return GSR_OK;
}

GSR_API int gsr_duplicate_selection(gsr_ctx *c, uint64_t *copies_out) {
    if (!c || !copies_out) { set_last_error("gsr_duplicate_selection: NULL argument"); return GSR_ERR_INVALID; }
    if (!c->masks.on) { set_last_error("gsr_duplicate_selection: the splat masks are not in use"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    const uint64_t n = c->num_splats;
    if ((rc = launch_count_selected(c->masks.selected, n, c->masks.counts, s))) return rc;
    unsigned long long S = 0ull;
    GSR_CUDA_TRY(cudaMemcpyAsync(&S, c->masks.counts, sizeof S, cudaMemcpyDeviceToHost, s));
    GSR_CUDA_TRY(cudaStreamSynchronize(s));
    if (S > c->max_splats - n) {
        set_last_error("gsr_duplicate_selection: %llu selected splats, room for %llu behind the cloud's %llu", S,
                       (unsigned long long)(c->max_splats - n), (unsigned long long)n);
        return GSR_ERR_INVALID;
    }
    if (S) {
        CompactArgs a;
        a.soa = c->soa; a.plane_stride = c->plane_stride; a.n = n;
        a.hidden = c->masks.hidden; a.selected = c->masks.selected; a.sel_out = nullptr;
        a.lookback = c->masks.lookback; a.total = c->masks.counts;
        if ((rc = launch_compact_store(a, COMPACT_DUPLICATE, c->sh_bands, sh_half(c), s))) return rc;
    }
    if ((rc = launch_duplicate_finish(n, S, c->masks.hidden, c->masks.selected, c->masks.words, s))) return rc;
    c->num_splats = n + S;
    *copies_out = S;
    return GSR_OK;
}

GSR_API int gsr_set_splat_count(gsr_ctx *c, uint64_t n) {
    if (!c) return GSR_ERR_INVALID;
    if (n > c->max_splats) { set_last_error("gsr_set_splat_count: %llu > max_splats %llu", (unsigned long long)n, (unsigned long long)c->max_splats); return GSR_ERR_INVALID; }
    c->num_splats = n;
    return GSR_OK;
}

// ---- splat property selection: gsr_select_where is enqueued like the selections, gsr_splat_histogram like the store edits ----------
static int check_property(const gsr_splat_filter &f, const char *where, uint32_t i) {
    if ((f.property < GSR_PROP_OPACITY || f.property > GSR_PROP_COLOR_DISTANCE) && !prop_is_contrib(f.property)) {
        set_last_error("%s: filter %u: unknown property %d", where, i, f.property);
        return GSR_ERR_INVALID;
    }
    if (f.property != GSR_PROP_COLOR_DISTANCE) return GSR_OK;   // rgb is ignored
    for (int k = 0; k < 3; ++k) {
        if (!(fabsf(f.rgb[k]) <= 3.402823466e38f)) { set_last_error("%s: filter %u: non-finite rgb[%d]", where, i, k); return GSR_ERR_INVALID; }
    }
    return GSR_OK;
}

// The tested range of select_range (instance -1: the store, k: instance k's source range) intersected with the cloud [0, n)
static int property_range(const gsr_ctx *c, const char *where, int32_t instance, uint64_t &first, uint64_t &count) {
    SelectArgs a;
    int rc = select_range(c, where, instance, a);
    if (rc) return rc;
    const uint64_t n = c->num_splats;
    first = a.first;
    count = a.first >= n ? 0ull : (a.count < n - a.first ? a.count : n - a.first);
    return GSR_OK;
}

GSR_API int gsr_select_where(gsr_ctx *c, const gsr_splat_filter *filters, uint32_t n, int32_t instance, int32_t op) {
    if (!c || !filters) { set_last_error("gsr_select_where: NULL argument"); return GSR_ERR_INVALID; }
    if (n < 1 || n > GSR_MAX_SPLAT_FILTERS) { set_last_error("gsr_select_where: %u filters, need 1..%d", n, GSR_MAX_SPLAT_FILTERS); return GSR_ERR_INVALID; }
    int planes = 0, rc;
    for (uint32_t i = 0; i < n; ++i) {
        if ((rc = check_property(filters[i], "gsr_select_where", i))) return rc;
        if (filters[i].lo != filters[i].lo || filters[i].hi != filters[i].hi) { set_last_error("gsr_select_where: filter %u: NaN bound", i); return GSR_ERR_INVALID; }
        planes |= prop_sources(filters[i].property);
    }
    if (!select_op_valid(op)) { set_last_error("gsr_select_where: unknown op %d", op); return GSR_ERR_INVALID; }
    if ((planes & PROP_PC) && !c->contrib) { set_last_error("gsr_select_where: a contribution property, and no contribution buffer is set"); return GSR_ERR_STATE; }
    WhereArgs a;
    memset(&a, 0, sizeof a);
    if ((rc = property_range(c, "gsr_select_where", instance, a.first, a.count))) return rc;
    if ((rc = masks_use(c, "gsr_select_where"))) return rc;
    a.selected = c->masks.selected; a.hidden = c->masks.hidden; a.words = c->masks.words; a.op = (uint32_t)op;
    a.soa = c->soa; a.plane_stride = c->plane_stride;
    a.n = n;
    memcpy(a.f, filters, sizeof(gsr_splat_filter) * n);
    a.contrib = c->contrib;
    cudaStream_t s = mask_stream(c);
    // the contribution buffer is written by the compositor of every earlier frame, on the render stream
    if ((planes & PROP_PC) && (rc = store_stream(c, &s))) return rc;
    return launch_select_where(a, planes, sh_half(c), s);
}

// ord (gsr_set_depth_order) back to the float
static float ord_float(uint32_t key) { const uint32_t b = (key >> 31) ? key ^ 0x80000000u : ~key; float f; memcpy(&f, &b, 4); return f; }

GSR_API int gsr_splat_histogram(gsr_ctx *c, const gsr_splat_filter *property, int32_t instance, int32_t scope, const float *edges,
                                uint32_t bins, uint64_t *counts, float minmax[2]) {
    if (!c || !property || !edges || !counts) { set_last_error("gsr_splat_histogram: NULL argument"); return GSR_ERR_INVALID; }
    if (bins < 1 || bins > GSR_MAX_HISTOGRAM_BINS) { set_last_error("gsr_splat_histogram: %u bins, need 1..%d", bins, GSR_MAX_HISTOGRAM_BINS); return GSR_ERR_INVALID; }
    for (uint32_t i = 0; i <= bins; ++i) {
        if (!(fabsf(edges[i]) <= 3.402823466e38f)) { set_last_error("gsr_splat_histogram: edge %u is not finite", i); return GSR_ERR_INVALID; }
        if (i && !(edges[i] > edges[i - 1])) { set_last_error("gsr_splat_histogram: edge %u does not increase", i); return GSR_ERR_INVALID; }
    }
    int rc = check_property(*property, "gsr_splat_histogram", 0);
    if (rc) return rc;
    if (scope != GSR_HISTOGRAM_KEPT && scope != GSR_HISTOGRAM_SELECTED) { set_last_error("gsr_splat_histogram: unknown scope %d", scope); return GSR_ERR_INVALID; }
    if (prop_is_contrib(property->property) && !c->contrib) {
        set_last_error("gsr_splat_histogram: a contribution property, and no contribution buffer is set");
        return GSR_ERR_STATE;
    }
    HistArgs a;
    memset(&a, 0, sizeof a);
    if ((rc = property_range(c, "gsr_splat_histogram", instance, a.first, a.count))) return rc;
    const bool none = scope == GSR_HISTOGRAM_SELECTED && !c->masks.on;   // nothing is selected
    unsigned long long *got = nullptr;
    int32_t keys[2] = {INT32_MIN, INT32_MIN};
    if (a.count && !none) {
        if ((rc = use_device(c->device))) return rc;
        if (!c->hist) {   // the device buffer and its page-locked image, so both copies are asynchronous
            void *d = nullptr, *h = nullptr;
            cudaError_t e = cudaMalloc(&d, HIST_BUFFER_BYTES);
            if (e == cudaSuccess) e = cudaMallocHost(&h, HIST_BUFFER_BYTES);
            if (e != cudaSuccess) {
                cudaFree(d);
                set_last_error("gsr_splat_histogram: %zu B -> %s", HIST_BUFFER_BYTES, cudaGetErrorString(e));
                return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
            }
            c->hist = d;
            c->hist_host = static_cast<unsigned char *>(h);
        }
        cudaStream_t s;
        if ((rc = store_stream(c, &s))) return rc;
        // the image: zeroed counters, the initial keys, the edges
        unsigned char *img = c->hist_host;
        memset(img, 0, HIST_EDGES_OFFSET);
        memcpy(img + HIST_KEYS_OFFSET, keys, sizeof keys);
        memcpy(img + HIST_EDGES_OFFSET, edges, sizeof(float) * (bins + 1));
        char *buf = static_cast<char *>(c->hist);
        GSR_CUDA_TRY(cudaMemcpyAsync(buf, img, HIST_EDGES_OFFSET + sizeof(float) * (bins + 1), cudaMemcpyHostToDevice, s));
        a.soa = c->soa; a.plane_stride = c->plane_stride;
        a.hidden = c->masks.on ? c->masks.hidden : nullptr; a.selected = c->masks.on ? c->masks.selected : nullptr;
        a.selected_only = scope == GSR_HISTOGRAM_SELECTED;
        a.bins = bins;
        a.top = 1u;
        while (2u * a.top <= bins - 1u) a.top *= 2u;
        a.prop = *property;
        a.counts = reinterpret_cast<unsigned long long *>(buf);
        a.keys = reinterpret_cast<int32_t *>(buf + HIST_KEYS_OFFSET);
        a.edges = reinterpret_cast<const float *>(buf + HIST_EDGES_OFFSET);
        a.contrib = c->contrib;
        if ((rc = launch_splat_histogram(a, prop_sources(property->property), sh_half(c), c->sm_count, s))) return rc;
        GSR_CUDA_TRY(cudaMemcpyAsync(img, buf, HIST_EDGES_OFFSET, cudaMemcpyDeviceToHost, s));
        GSR_CUDA_TRY(cudaStreamSynchronize(s));
        got = reinterpret_cast<unsigned long long *>(img);
        memcpy(keys, img + HIST_KEYS_OFFSET, sizeof keys);
    }
    for (uint32_t i = 0; i < bins + 3; ++i) counts[i] = got ? got[i] : 0ull;
    if (minmax) {
        const bool any = keys[1] != INT32_MIN;
        minmax[0] = any ? ord_float(~((uint32_t)keys[0] ^ 0x80000000u)) : INFINITY;
        minmax[1] = any ? ord_float((uint32_t)keys[1] ^ 0x80000000u) : -INFINITY;
    }
    return GSR_OK;
}

// ---- splat neighbourhood selection: enqueued like gsr_splat_histogram; synchronises the host for the budget and for the stats --------
GSR_API int gsr_select_neighborhood(gsr_ctx *c, const gsr_neighborhood *q, int32_t op, gsr_neighborhood_stats *stats) {
    static const char *where = "gsr_select_neighborhood";
    if (!c || !q) { set_last_error("%s: NULL argument", where); return GSR_ERR_INVALID; }
    if (q->mode < GSR_NEIGHBOR_SPARSE || q->mode > GSR_NEIGHBOR_SMALL_CLUSTERS) { set_last_error("%s: unknown mode %d", where, q->mode); return GSR_ERR_INVALID; }
    if (!(q->radius >= GSR_NEIGHBOR_MIN_RADIUS && q->radius <= GSR_NEIGHBOR_MAX_RADIUS)) {
        set_last_error("%s: radius %g is not finite or outside [2^-60, 2^60]", where, (double)q->radius);
        return GSR_ERR_INVALID;
    }
    if (q->count == 0 && (q->mode == GSR_NEIGHBOR_SPARSE || q->mode == GSR_NEIGHBOR_SMALL_CLUSTERS)) {
        set_last_error("%s: count 0 (need >= 1)", where);
        return GSR_ERR_INVALID;
    }
    if (!select_op_valid(op)) { set_last_error("%s: unknown op %d", where, op); return GSR_ERR_INVALID; }
    NeighborArgs a;
    memset(&a, 0, sizeof a);
    int rc = property_range(c, where, q->instance, a.first, a.count);
    if (rc || (rc = masks_use(c, where)) || (rc = alloc_neighbors(c, where))) return rc;
    gsr_ctx::Neighbors &nb = c->nb;
    a.plane0 = c->soa; a.hidden = c->masks.hidden; a.selected = c->masks.selected; a.words = c->masks.words; a.op = (uint32_t)op;
    a.h = neighbor_cell_size(q->radius);
    a.r2 = q->radius * q->radius;
    a.mode = (uint32_t)q->mode; a.threshold = q->count;
    a.shift = 32u - neighbor_bucket_bits(a.count);
    a.keys = nb.keys; a.vals = nb.vals; a.parent = nb.parent; a.size = nb.size; a.pos = nb.pos; a.start = nb.start;
    a.inside = c->masks.scratch;
    a.ctr = nb.ctr;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    GSR_CUDA_TRY(cudaMemsetAsync(nb.ctr, 0, sizeof(NeighborCounters), s));
    if (a.count) {
        if ((rc = launch_neighbor_keys(a, s))) return rc;
        // the participants' pairs sorted by key; parent and size are the sort's ping-pong halves until launch_neighbor_grid clears them
        if ((rc = sort_pairs_device(nb.ws, nb.keys, nb.vals, &nb.ctr->n, nb.parent, nb.size, s, nullptr))) return rc;
        if ((rc = launch_neighbor_grid(a, c->max_splats, s)) || (rc = launch_neighbor_budget(a, s))) return rc;
        GSR_CUDA_TRY(cudaMemcpyAsync(nb.ctr_host, nb.ctr, sizeof(NeighborCounters), cudaMemcpyDeviceToHost, s));
        GSR_CUDA_TRY(cudaStreamSynchronize(s));
        if (nb.ctr_host->candidates > GSR_MAX_NEIGHBOR_CANDIDATES) {
            set_last_error("%s: %llu candidates at radius %g, more than GSR_MAX_NEIGHBOR_CANDIDATES (%llu)", where, nb.ctr_host->candidates,
                           (double)q->radius, (unsigned long long)GSR_MAX_NEIGHBOR_CANDIDATES);
            return GSR_ERR_INVALID;
        }
    }
    if ((rc = launch_neighbor_select(a, s))) return rc;
    if (stats) {
        GSR_CUDA_TRY(cudaMemcpyAsync(nb.ctr_host, nb.ctr, sizeof(NeighborCounters), cudaMemcpyDeviceToHost, s));
        GSR_CUDA_TRY(cudaStreamSynchronize(s));
        const NeighborCounters &k = *nb.ctr_host;
        const bool clusters = q->mode == GSR_NEIGHBOR_CONNECTED || q->mode == GSR_NEIGHBOR_SMALL_CLUSTERS;
        stats->participants = k.n; stats->inside = k.inside; stats->candidates = k.candidates;
        stats->clusters = clusters ? k.clusters : 0ull; stats->largest_cluster = clusters ? k.largest : 0ull;
    }
    return GSR_OK;
}

// ---- splat export: enqueued like gsr_splat_histogram; synchronises the host for the count, and once more for rows into host memory ----
GSR_API int gsr_export_ply(gsr_ctx *c, int32_t scope, int32_t sh_degree, void *dst, uint64_t dst_rows, uint64_t *rows_out) {
    static const char *where = "gsr_export_ply";
    if (!c || !rows_out) { set_last_error("%s: NULL argument", where); return GSR_ERR_INVALID; }
    if (scope != GSR_EXPORT_KEPT && scope != GSR_EXPORT_SELECTED) { set_last_error("%s: unknown scope %d", where, scope); return GSR_ERR_INVALID; }
    if (sh_degree < -1 || sh_degree > c->sh_bands - 1) {
        set_last_error("%s: sh_degree %d, need -1 .. the stored degree %d", where, sh_degree, c->sh_bands - 1);
        return GSR_ERR_INVALID;
    }
    const int degree = sh_degree < 0 ? c->sh_bands - 1 : sh_degree;
    const uint64_t row_bytes = sizeof(float) * export_row_floats(degree);
    int rc = use_device(c->device);
    if (rc) return rc;
    ExportArgs a;
    memset(&a, 0, sizeof a);
    a.soa = c->soa; a.plane_stride = c->plane_stride; a.n = c->num_splats;
    a.hidden = c->masks.on ? c->masks.hidden : nullptr; a.selected = c->masks.on ? c->masks.selected : nullptr;
    a.selected_only = scope == GSR_EXPORT_SELECTED;
    a.degree = degree;
    unsigned long long rows = 0ull;
    cudaStream_t s = nullptr;
    if (a.n && !(a.selected_only && !a.hidden)) {   // while the masks are not in use nothing is selected
        if (!c->export_words) {
            const size_t bytes = sizeof(unsigned long long) * (1ull + compact_lookback_words((uint32_t)((c->max_splats + 31ull) / 32ull)));
            cudaError_t e = cudaMalloc((void **)&c->export_words, bytes);
            if (e != cudaSuccess) {
                c->export_words = nullptr;
                set_last_error("%s: look-back words of %zu B -> %s", where, bytes, cudaGetErrorString(e));
                return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
            }
        }
        a.count = c->export_words; a.lookback = c->export_words + 1;
        if ((rc = store_stream(c, &s)) || (rc = launch_export_count(a, s))) return rc;
        GSR_CUDA_TRY(cudaMemcpyAsync(&rows, a.count, sizeof rows, cudaMemcpyDeviceToHost, s));
        GSR_CUDA_TRY(cudaStreamSynchronize(s));
    }
    *rows_out = rows;
    if (!dst) return GSR_OK;
    if (dst_rows < rows) {
        set_last_error("%s: %llu exported rows, dst holds %llu", where, rows, (unsigned long long)dst_rows);
        return GSR_ERR_INVALID;
    }
    if (!rows) return GSR_OK;
    cudaPointerAttributes pa;
    GSR_CUDA_TRY(cudaPointerGetAttributes(&pa, dst));
    const bool device = pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged;
    float *out = static_cast<float *>(dst);
    if (!device) {   // host memory: rows x row_bytes of device staging, freed before the call returns
        cudaError_t e = cudaMalloc((void **)&out, rows * row_bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_last_error("%s: staging of %llu B for host memory -> %s (export into device memory instead)", where,
                           (unsigned long long)(rows * row_bytes), cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
    }
    a.dst = out;
    rc = launch_export_rows(a, c->sh_bands, sh_half(c), s);
    cudaError_t e = cudaSuccess;
    if (!rc && !device) e = cudaMemcpyAsync(dst, out, rows * row_bytes, cudaMemcpyDeviceToHost, s);
    if (!rc && e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (!device) cudaFree(out);
    if (rc) return rc;
    GSR_CUDA_TRY(e);
    return GSR_OK;
}

// ---- compressed PLY ----------------------------------------------------------------------------------------------------------------
// The three element bodies of a compressed file of `rows` rows and SH degree d, and where each lives
struct CplyBuffers {
    void *ptr[3];
    uint64_t bytes[3];
    bool device[3];
    uint64_t staged;   // bytes of device staging the host-memory buffers need (each part 16-byte aligned)
};
static int cply_buffers(CplyBuffers &b, const void *chunks, const void *packed, const void *sh, uint64_t rows, uint32_t chunk_floats,
                        int degree) {
    b.ptr[0] = const_cast<void *>(chunks); b.ptr[1] = const_cast<void *>(packed); b.ptr[2] = const_cast<void *>(sh);
    b.bytes[0] = sizeof(float) * chunk_floats * ((rows + CPLY_CHUNK - 1) / CPLY_CHUNK);
    b.bytes[1] = sizeof(uint32_t) * 4ull * rows;
    b.bytes[2] = (uint64_t)cply_sh_bytes(degree) * rows;
    b.staged = 0;
    for (int i = 0; i < 3; ++i) {
        b.device[i] = true;
        if (!b.bytes[i]) continue;
        cudaPointerAttributes pa;
        GSR_CUDA_TRY(cudaPointerGetAttributes(&pa, b.ptr[i]));
        b.device[i] = pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged;
        if (!b.device[i]) b.staged += (b.bytes[i] + 15ull) & ~15ull;
    }
    return GSR_OK;
}
// Device staging for the host-memory buffers of b: dev[i] is where the kernels read or write part i.  GSR_ERR_OOM when it cannot be
// allocated (*stage stays nullptr).
static int cply_stage(CplyBuffers &b, void **stage, void *dev[3], const char *where) {
    *stage = nullptr;
    if (b.staged) {
        cudaError_t e = cudaMalloc(stage, b.staged);
        if (e != cudaSuccess) {
            cudaGetLastError();
            *stage = nullptr;
            set_last_error("%s: staging of %llu B for host memory -> %s (use device memory instead)", where, (unsigned long long)b.staged,
                           cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA;
        }
    }
    uint64_t off = 0;
    for (int i = 0; i < 3; ++i) {
        dev[i] = b.ptr[i];
        if (!b.device[i]) { dev[i] = static_cast<char *>(*stage) + off; off += (b.bytes[i] + 15ull) & ~15ull; }
    }
    return GSR_OK;
}

// Enqueued like gsr_export_ply: synchronises the host for the count, and once more for the file
GSR_API int gsr_export_compressed_ply(gsr_ctx *c, int32_t scope, int32_t sh_degree, int32_t order, gsr_compressed_ply *dst, uint64_t *rows_out) {
    static const char *where = "gsr_export_compressed_ply";
    if (!c || !rows_out) { set_last_error("%s: NULL argument", where); return GSR_ERR_INVALID; }
    if (scope != GSR_EXPORT_KEPT && scope != GSR_EXPORT_SELECTED) { set_last_error("%s: unknown scope %d", where, scope); return GSR_ERR_INVALID; }
    if (order != GSR_COMPRESS_STORE_ORDER && order != GSR_COMPRESS_MORTON) { set_last_error("%s: unknown order %d", where, order); return GSR_ERR_INVALID; }
    if (sh_degree < -1 || sh_degree > c->sh_bands - 1) {
        set_last_error("%s: sh_degree %d, need -1 .. the stored degree %d", where, sh_degree, c->sh_bands - 1);
        return GSR_ERR_INVALID;
    }
    if (c->max_splats >= (1ull << 32)) { set_last_error("%s: the store index is 32-bit; max_splats %llu", where, (unsigned long long)c->max_splats); return GSR_ERR_INVALID; }
    const int degree = sh_degree < 0 ? c->sh_bands - 1 : sh_degree;
    if (dst && (!dst->chunks || !dst->packed || (degree > 0 && !dst->sh))) { set_last_error("%s: NULL buffer in dst", where); return GSR_ERR_INVALID; }
    int rc = use_device(c->device);
    if (rc) return rc;
    CompressArgs a;
    memset(&a, 0, sizeof a);
    a.soa = c->soa; a.plane_stride = c->plane_stride; a.n = c->num_splats;
    a.hidden = c->masks.on ? c->masks.hidden : nullptr; a.selected = c->masks.on ? c->masks.selected : nullptr;
    a.selected_only = scope == GSR_EXPORT_SELECTED;
    a.morton = order == GSR_COMPRESS_MORTON;
    a.degree = degree;
    uint64_t rows = 0;
    cudaStream_t s = nullptr;
    gsr_ctx::Compressed &cp = c->cply;
    if (a.n && !(a.selected_only && !a.hidden)) {   // while the masks are not in use nothing is selected
        if ((rc = alloc_compressed(c, where))) return rc;
        a.bounds = cp.bounds;
        if ((rc = store_stream(c, &s)) || (rc = launch_compress_bounds(a, s))) return rc;
        GSR_CUDA_TRY(cudaMemcpyAsync(cp.bounds_host, cp.bounds, sizeof(CompressBounds), cudaMemcpyDeviceToHost, s));
        GSR_CUDA_TRY(cudaStreamSynchronize(s));
        rows = cp.bounds_host->count;
    }
    *rows_out = rows;
    if (!dst) return GSR_OK;
    if (dst->rows < rows) {
        set_last_error("%s: %llu exported rows, dst holds %llu", where, (unsigned long long)rows, (unsigned long long)dst->rows);
        return GSR_ERR_INVALID;
    }
    if (rows) {
        CplyBuffers b;
        if ((rc = cply_buffers(b, dst->chunks, dst->packed, dst->sh, rows, CPLY_CHUNK_FLOATS, degree))) return rc;
        void *stage = nullptr, *dev[3];
        if ((rc = cply_stage(b, &stage, dev, where))) return rc;
        const uint64_t m = c->max_splats;
        a.keys = cp.pairs; a.vals = cp.pairs + m; a.sort_n = cp.ws.n_dev; a.rows = rows;
        a.chunks = static_cast<float *>(dev[0]); a.packed = static_cast<uint32_t *>(dev[1]); a.sh = static_cast<uint8_t *>(dev[2]);
        rc = launch_compress_keys(a, s);
        if (!rc) rc = sort_pairs_device(cp.ws, a.keys, a.vals, a.sort_n, cp.pairs + 2 * m, cp.pairs + 3 * m, s, nullptr);
        if (!rc) rc = launch_compress_chunks(a, c->sh_bands, sh_half(c), s);
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < 3 && !rc && e == cudaSuccess; ++i)
            if (!b.device[i] && b.bytes[i]) e = cudaMemcpyAsync(b.ptr[i], dev[i], b.bytes[i], cudaMemcpyDeviceToHost, s);
        if (!rc && e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (stage) cudaFree(stage);
        if (rc) return rc;
        GSR_CUDA_TRY(e);
    }
    dst->rows = rows;
    dst->chunk_count = (rows + CPLY_CHUNK - 1) / CPLY_CHUNK;
    dst->sh_degree = (uint32_t)degree;
    dst->chunk_floats = CPLY_CHUNK_FLOATS;
    return GSR_OK;
}

// Synchronises like gsr_upload_ply: the caller may free or reuse src's buffers when it returns
GSR_API int gsr_upload_compressed_ply(gsr_ctx *c, const gsr_compressed_ply *src, uint64_t first, float creation_time) {
    static const char *where = "gsr_upload_compressed_ply";
    if (!c || !src) { set_last_error("%s: NULL argument", where); return GSR_ERR_INVALID; }
    if (src->chunk_floats != 12u && src->chunk_floats != 18u) { set_last_error("%s: chunk_floats %u, need 12 or 18", where, src->chunk_floats); return GSR_ERR_INVALID; }
    if (src->sh_degree > 3u) { set_last_error("%s: sh_degree %u > 3", where, src->sh_degree); return GSR_ERR_INVALID; }
    if (!src->chunks || !src->packed || (src->sh_degree > 0u && !src->sh)) { set_last_error("%s: NULL buffer in src", where); return GSR_ERR_INVALID; }
    const uint64_t rows = src->rows;
    if (src->chunk_count != (rows + CPLY_CHUNK - 1) / CPLY_CHUNK) {
        set_last_error("%s: %llu chunks for %llu rows, need %llu", where, (unsigned long long)src->chunk_count, (unsigned long long)rows,
                       (unsigned long long)((rows + CPLY_CHUNK - 1) / CPLY_CHUNK));
        return GSR_ERR_INVALID;
    }
    if (rows > c->max_splats || first > c->max_splats - rows) {
        set_last_error("%s: upload range [%llu,%llu) exceeds max_splats %llu", where, (unsigned long long)first, (unsigned long long)(first + rows),
                       (unsigned long long)c->max_splats);
        return GSR_ERR_INVALID;
    }
    int rc = use_device(c->device);
    if (rc || !rows) return rc;
    CplyBuffers b;
    if ((rc = cply_buffers(b, src->chunks, src->packed, src->sh, rows, src->chunk_floats, (int)src->sh_degree))) return rc;
    void *stage = nullptr, *dev[3];
    if ((rc = cply_stage(b, &stage, dev, where))) return rc;
    DecompressArgs a;
    memset(&a, 0, sizeof a);
    a.chunks = static_cast<const float *>(dev[0]); a.packed = static_cast<const uint32_t *>(dev[1]); a.sh = static_cast<const uint8_t *>(dev[2]);
    a.rows = rows; a.chunk_floats = src->chunk_floats; a.degree = (int32_t)src->sh_degree; a.creation_time = creation_time;
    a.soa = c->soa; a.plane_stride = c->plane_stride; a.first = first;
    cudaError_t e = cudaStreamSynchronize(c->front_stream);   // a projection in flight reads the planes this call rewrites
    for (int i = 0; i < 3 && e == cudaSuccess; ++i)
        if (!b.device[i] && b.bytes[i]) e = cudaMemcpyAsync(dev[i], b.ptr[i], b.bytes[i], cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) rc = launch_compressed_to_soa(a, c->sh_bands, sh_half(c), c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (stage) cudaFree(stage);
    if (rc) return rc;
    GSR_CUDA_TRY(e);
    if (first + rows > c->num_splats) c->num_splats = first + rows;
    return GSR_OK;
}

GSR_API uint64_t gsr_splat_store_bytes(gsr_ctx *c) { return c ? store_bytes(c) : 0ull; }

static int store_copy(gsr_ctx *c, void *dst, const void *src, const char *where) {
    if (!c || !dst || !src) { set_last_error("%s: NULL argument", where); return GSR_ERR_INVALID; }
    int rc = use_device(c->device);
    if (rc) return rc;
    cudaStream_t s;
    if ((rc = store_stream(c, &s))) return rc;
    GSR_CUDA_TRY(cudaMemcpyAsync(dst, src, store_bytes(c), cudaMemcpyDefault, s));
    return GSR_OK;
}

GSR_API int gsr_copy_splat_store(gsr_ctx *c, void *dst) { return store_copy(c, dst, c ? c->soa : nullptr, "gsr_copy_splat_store"); }

GSR_API int gsr_restore_splat_store(gsr_ctx *c, const void *src) { return store_copy(c, c ? c->soa : nullptr, src, "gsr_restore_splat_store"); }

GSR_API int gsr_pick(gsr_ctx *c, uint32_t tile_id, float heatmap_factor, float out_xyzn[4]) {
    if (!c || !out_xyzn) return GSR_ERR_INVALID;
    if (c->width == 0) { set_last_error("gsr_pick before gsr_resize"); return GSR_ERR_STATE; }
    if (c->frame_counter == 0 || !c->fb_last) { set_last_error("gsr_pick before the first gsr_render at this size"); return GSR_ERR_STATE; }
    int rc = use_device(c->device);
    if (rc) return rc;
    const uint32_t T = (uint32_t)(c->tiles_x * c->tiles_y);
    const uint32_t t0 = (uint32_t)(c->band_y0 * c->tiles_x), t1 = (uint32_t)(c->band_y1 * c->tiles_x);
    if (tile_id < T && tile_id >= t0 && tile_id < t1 && (int)(tile_id / (uint32_t)c->tiles_x) % c->row_mod == c->row_rem) {
        CompositeArgs ca;
        ca.records = c->records_cur; ca.values = c->vals_cur; ca.bounds = c->bounds; ca.out = framebuffer(c);
        ca.width = c->width; ca.height = c->height; ca.tiles_x = c->tiles_x;
        ca.tile_begin = (int32_t)tile_id; ca.num_tiles = 1; ca.row_step = 1;
        ca.heatmap_factor = heatmap_factor; ca.target_tile_id = tile_id; ca.pick = c->pick;
        ca.frame = c->pick_frame; ca.count_staged = 0;  // own queue counters; slot 0 of the queue, state slot 0
        ca.order = nullptr; ca.consumed = nullptr; ca.ctas_per_sm = 1; ca.sm_count = c->sm_count;
        ca.contract = (c->flags & GSR_FLAG_UNCONTRACTED_BLEND) ? 0 : 1;
        ca.trace = nullptr; ca.trace_count = nullptr; ca.trace_cap = 0;
        ca.view_z[0] = ca.view_z[1] = ca.view_z[2] = ca.view_z[3] = 0.0f;
        ca.scene_depth = nullptr; ca.depth_out = nullptr;   // the pick re-dispatch is always the default compositor
        if (c->depth_out) {
            // ... whose opaque pixels must not replace the depth-composited tile: they go to a 16-row strip instead (the kernel
            // stores pixel (x, y) at out[y * width + x], y in the tile's 16 rows)
            if (!c->pick_strip) GSR_CUDA_TRY(cudaMalloc((void **)&c->pick_strip, sizeof(float4) * (size_t)TILE * c->width));
            ca.out = c->pick_strip - (size_t)(tile_id / (uint32_t)c->tiles_x) * TILE * (size_t)c->width;
        }
        for (int i = 0; i < 2; ++i)   // the re-dispatch rewrites the tile's pixels: not under a read-back in flight
            if (c->copied_valid[i]) GSR_CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_copied[i], 0));
        GSR_CUDA_TRY(cudaMemsetAsync(c->pick_frame, 0, sizeof(FrameState), c->stream));
        if ((rc = launch_composite(ca, c->stream))) return rc;
    }
    GSR_CUDA_TRY(cudaMemcpyAsync(out_xyzn, c->pick, sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return GSR_OK;
}

GSR_API int gsr_get_stats(gsr_ctx *c, gsr_stats *out) {
    if (!c || !out) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    memset(out, 0, sizeof *out);
    FrameState fs;
    GSR_CUDA_TRY(cudaMemcpyAsync(&fs, c->frame, sizeof fs, cudaMemcpyDeviceToHost, c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    out->num_splats = c->num_splats;
    out->duplicates = fs.dup_total;
    out->visible = fs.visible;
    out->capacity = c->capacity;
    out->last_tile = (int64_t)fs.last_tile_plus1 - 1;
    out->overflow = fs.overflow;
    out->width = (uint32_t)c->width; out->height = (uint32_t)c->height;
    out->tiles_x = (uint32_t)c->tiles_x; out->tiles_y = (uint32_t)c->tiles_y;
    out->band_y0 = (uint32_t)c->band_y0; out->band_y1 = (uint32_t)c->band_y1;
    out->kernel_launches = c->last_launches;
    out->staged = fs.staged;
    if (c->ev_valid && c->frame_counter > 0) {
        if ((rc = stage_times(c, (uint32_t)((c->frame_counter - 1) % GSR_HISTORY_FRAMES), out->stage_ms, nullptr))) return rc;
    }
    return GSR_OK;
}

GSR_API int gsr_get_frame_history(gsr_ctx *c, uint32_t max_frames, gsr_frame_record *out, uint32_t *n_out) {
    if (!c || !out || !n_out) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    *n_out = 0;
    if (!c->ev_valid || c->frame_counter == 0) return GSR_OK;
    uint64_t n = c->frame_counter < GSR_HISTORY_FRAMES ? c->frame_counter : GSR_HISTORY_FRAMES;
    if (n > max_frames) n = max_frames;
    static thread_local FrameState host_ring[GSR_HISTORY_FRAMES];
    GSR_CUDA_TRY(cudaMemcpyAsync(host_ring, c->ring, sizeof(FrameState) * GSR_HISTORY_FRAMES, cudaMemcpyDeviceToHost, c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (uint64_t k = 0; k < n; ++k) {
        const uint64_t fi = c->frame_counter - n + k;
        const uint32_t slot = (uint32_t)(fi % GSR_HISTORY_FRAMES);
        const FrameState &fs = host_ring[slot];
        gsr_frame_record &r = out[k];
        memset(&r, 0, sizeof r);
        r.frame_index = fi; r.duplicates = fs.dup_total; r.visible = fs.visible; r.staged = fs.staged; r.overflow = fs.overflow;
        if ((rc = stage_times(c, slot, r.stage_ms, &r.front_ms))) return rc;
    }
    *n_out = (uint32_t)n;
    return GSR_OK;
}

GSR_API int gsr_debug_keep_unsorted(gsr_ctx *c, int enable) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    if (enable && !c->unsorted_keys) {
        GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_keys, sizeof(uint32_t) * c->capacity));
        GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_vals, sizeof(uint32_t) * c->capacity));
    }
    if (enable && c->depth_words && !c->unsorted_depth) GSR_CUDA_TRY(cudaMalloc((void **)&c->unsorted_depth, sizeof(uint32_t) * c->capacity));
    c->keep_unsorted = enable != 0;
    return GSR_OK;
}

GSR_API int gsr_debug_compositor_config(gsr_ctx *c, int32_t ctas_per_sm, int32_t longest_first, int32_t sparse_tiles_per_sm) {
    if (!c || ctas_per_sm < 0 || sparse_tiles_per_sm < 0) return GSR_ERR_INVALID;
    c->comp_ctas_per_sm = ctas_per_sm ? ctas_per_sm : c->comp_max_ctas; c->comp_order_mode = longest_first != 0; c->comp_sparse_per_sm = sparse_tiles_per_sm;
    return GSR_OK;
}

GSR_API int gsr_debug_pipeline(gsr_ctx *c, int32_t overlap) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->front_stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->overlap = overlap < 0 ? -1 : (overlap != 0); c->front_gate = nullptr;
    return GSR_OK;
}

GSR_API int gsr_debug_enable_trace(gsr_ctx *c, uint32_t max_items) {
    if (!c) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    cudaFree(c->trace); cudaFree(c->trace_count);
    c->trace = nullptr; c->trace_count = nullptr; c->trace_cap = 0;
    if (max_items) {
        GSR_CUDA_TRY(cudaMalloc((void **)&c->trace, sizeof(ulonglong4) * (size_t)max_items + 32));
        GSR_CUDA_TRY(cudaMalloc((void **)&c->trace_count, sizeof(uint32_t)));
        GSR_CUDA_TRY(cudaMemset(c->trace_count, 0, sizeof(uint32_t)));
        c->trace_cap = max_items;
    }
    return GSR_OK;
}

GSR_API int gsr_debug_copy(gsr_ctx *c, int which, void *dst, size_t bytes) {
    if (!c || !dst) return GSR_ERR_INVALID;
    int rc = use_device(c->device);
    if (rc) return rc;
    const void *src = nullptr;
    size_t avail = 0;
    switch (which) {
        case GSR_BUF_RECORDS: src = c->records_cur; avail = sizeof(float4) * 3ull * (c->inst.n ? c->inst.drawn : c->max_splats); break;
        case GSR_BUF_KEYS: src = c->keys_cur; avail = sizeof(uint32_t) * c->capacity; break;
        case GSR_BUF_VALUES: src = c->vals_cur; avail = sizeof(uint32_t) * c->capacity; break;
        case GSR_BUF_BOUNDS: src = c->bounds; avail = sizeof(uint2) * (size_t)c->tiles_x * c->tiles_y; break;
        case GSR_BUF_KEYS_UNSORTED: src = c->unsorted_keys; avail = c->unsorted_keys ? sizeof(uint32_t) * c->capacity : 0; break;
        case GSR_BUF_VALUES_UNSORTED: src = c->unsorted_vals; avail = c->unsorted_vals ? sizeof(uint32_t) * c->capacity : 0; break;
        case GSR_BUF_DEPTH_WORDS_UNSORTED: src = c->unsorted_depth; avail = c->unsorted_depth ? sizeof(uint32_t) * c->capacity : 0; break;
        case GSR_BUF_FRAMEBUFFER: src = framebuffer(c); avail = sizeof(float4) * (size_t)c->width * c->height; break;
        case GSR_BUF_COMPOSITOR_TRACE: src = c->trace; avail = c->trace ? sizeof(ulonglong4) * (size_t)c->trace_cap : 0; break;
        case GSR_BUF_COMPOSITOR_TRACE_COUNT: src = c->trace_count; avail = c->trace_count ? sizeof(uint32_t) : 0; break;
        case GSR_BUF_SPLATS: src = c->soa; avail = sizeof(float4) * (size_t)soa_planes(c->sh_bands, sh_half(c)) * c->plane_stride; break;
        case GSR_BUF_INSTANCES: {   // host copy: no device involved
            avail = sizeof(float) * INSTANCE_XFORM_FLOATS * c->inst.n;
            if (bytes > avail) { set_last_error("gsr_debug_copy(%d): %zu bytes requested, %zu available", which, bytes, avail); return GSR_ERR_INVALID; }
            memcpy(dst, c->inst.xf, bytes);
            return GSR_OK;
        }
        case GSR_BUF_EDIT_TRANSFORM: {   // host copy: no device involved
            avail = sizeof c->edit_last;
            if (bytes > avail) { set_last_error("gsr_debug_copy(%d): %zu bytes requested, %zu available", which, bytes, avail); return GSR_ERR_INVALID; }
            memcpy(dst, c->edit_last, bytes);
            return GSR_OK;
        }
        case GSR_BUF_EDIT_COLOR: {   // host copy: no device involved
            avail = sizeof c->color_last;
            if (bytes > avail) { set_last_error("gsr_debug_copy(%d): %zu bytes requested, %zu available", which, bytes, avail); return GSR_ERR_INVALID; }
            memcpy(dst, c->color_last, bytes);
            return GSR_OK;
        }
        case GSR_BUF_INSTANCE_APPEARANCE: {   // host copy: no device involved
            avail = sizeof(gsr_instance_appearance) * c->inst.n;
            if (bytes > avail) { set_last_error("gsr_debug_copy(%d): %zu bytes requested, %zu available", which, bytes, avail); return GSR_ERR_INVALID; }
            if (c->inst.app) { memcpy(dst, c->inst.app, bytes); return GSR_OK; }
            const gsr_instance_appearance def = {{1.0f, 1.0f, 1.0f}, 1.0f, UINT64_MAX};
            for (size_t o = 0; o < bytes; o += sizeof def) memcpy((char *)dst + o, &def, bytes - o < sizeof def ? bytes - o : sizeof def);
            return GSR_OK;
        }
        default: set_last_error("gsr_debug_copy: unknown buffer %d", which); return GSR_ERR_INVALID;
    }
    if (!src || bytes > avail) { set_last_error("gsr_debug_copy(%d): %zu bytes requested, %zu available", which, bytes, avail); return GSR_ERR_INVALID; }
    GSR_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    GSR_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return GSR_OK;
}

// ---------------------------------------------------------------------------------------------------
// stand-alone sorter
// ---------------------------------------------------------------------------------------------------
GSR_API int gsr_sorter_create(int32_t device, uint64_t max_n, gsr_sorter **out) {
    if (!out || max_n == 0) return GSR_ERR_INVALID;
    *out = nullptr;
    int rc = check_device(device);
    if (rc) return rc;
    if ((rc = use_device(device))) return rc;
    gsr_sorter *s = new (std::nothrow) gsr_sorter();
    if (!s) return GSR_ERR_OOM;
    s->device = device;
    rc = sort_workspace_create(s->ws, max_n, /*need_alt_buffers=*/true);
    if (rc == GSR_OK && (cudaEventCreate(&s->e0) != cudaSuccess || cudaEventCreate(&s->e1) != cudaSuccess)) rc = GSR_ERR_CUDA;
    if (rc) { sort_workspace_destroy(s->ws); delete s; return rc; }
    *out = s;
    return GSR_OK;
}

GSR_API int gsr_sorter_destroy(gsr_sorter *s) {
    if (!s) return GSR_OK;
    cudaSetDevice(s->device);
    cudaDeviceSynchronize();
    sort_workspace_destroy(s->ws);
    if (s->e0) cudaEventDestroy(s->e0);
    if (s->e1) cudaEventDestroy(s->e1);
    delete s;
    return GSR_OK;
}

GSR_API int gsr_sorter_sort_device(gsr_sorter *s, void *d_keys, void *d_values, uint64_t n, void *cuda_stream) {
    if (!s || (!d_keys && n)) return GSR_ERR_INVALID;
    if (n > s->ws.max_n) { set_last_error("sort of %llu exceeds sorter capacity %llu", (unsigned long long)n, (unsigned long long)s->ws.max_n); return GSR_ERR_INVALID; }
    int rc = use_device(s->device);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const uint32_t n32 = (uint32_t)n;
    GSR_CUDA_TRY(cudaMemcpyAsync(s->ws.n_dev, &n32, sizeof n32, cudaMemcpyHostToDevice, st));
    GSR_CUDA_TRY(cudaEventRecord(s->e0, st));
    int launches = 0;
    rc = sort_pairs_device(s->ws, (uint32_t *)d_keys, (uint32_t *)d_values, s->ws.n_dev, s->ws.alt_keys, d_values ? s->ws.alt_vals : nullptr, st, &launches);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaEventRecord(s->e1, st));
    s->timed = true;
    return GSR_OK;
}

GSR_API int gsr_sorter_last_ms(gsr_sorter *s, float *ms) {
    if (!s || !ms || !s->timed) return GSR_ERR_STATE;
    int rc = use_device(s->device);
    if (rc) return rc;
    GSR_CUDA_TRY(cudaEventSynchronize(s->e1));
    GSR_CUDA_TRY(cudaEventElapsedTime(ms, s->e0, s->e1));
    return GSR_OK;
}

GSR_API int gsr_sort_pairs_host(int32_t device, uint32_t *keys, uint32_t *values, uint64_t n) {
    if (n == 0) return GSR_OK;
    if (!keys) return GSR_ERR_INVALID;
    gsr_sorter *s = nullptr;
    int rc = gsr_sorter_create(device, n, &s);
    if (rc) return rc;
    uint32_t *dk = nullptr, *dv = nullptr;
    cudaError_t e = cudaMalloc((void **)&dk, 4 * n);
    if (e == cudaSuccess && values) e = cudaMalloc((void **)&dv, 4 * n);
    if (e == cudaSuccess) e = cudaMemcpy(dk, keys, 4 * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && values) e = cudaMemcpy(dv, values, 4 * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        rc = gsr_sorter_sort_device(s, dk, dv, n, nullptr);
        if (rc == GSR_OK) e = cudaDeviceSynchronize();
    }
    if (e == cudaSuccess && rc == GSR_OK) e = cudaMemcpy(keys, dk, 4 * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && rc == GSR_OK && values) e = cudaMemcpy(values, dv, 4 * n, cudaMemcpyDeviceToHost);
    cudaFree(dk); cudaFree(dv);
    gsr_sorter_destroy(s);
    if (e != cudaSuccess) { set_last_error("gsr_sort_pairs_host: %s", cudaGetErrorString(e)); return e == cudaErrorMemoryAllocation ? GSR_ERR_OOM : GSR_ERR_CUDA; }
    return rc;
}

}  // extern "C"
