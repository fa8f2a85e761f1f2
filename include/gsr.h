/*
 * gsr.h -- C-ABI of libgsr.so: the H100-native (sm_90a) forward 3D-Gaussian-splatting rasterizer that
 * replaces the body of 2Retr0/GodotGaussianSplatting's `GaussianSplattingRasterizer`
 * (util/gaussian_splatting_rasterizer.gd) plus the six compute shaders it dispatches
 * (the .glsl files of resources/shaders/compute) and the RenderingDevice wrapper (util/render_context.gd).
 *
 * The reference has no native/FFI boundary of its own: its "plugin API" is the GDScript class.  Each
 * entry point below cites the reference interface it replaces (paths relative to the reference root).
 * A Godot host binds these through a GDExtension shim or C# P/Invoke (see INTEGRATION.md); this repo's
 * tests and bench bind them with Python ctypes (godotgaussiansplatting_b200/_lib.py).
 *
 * Conventions: plain C, opaque handle, `int` status returns (0 = GSR_OK), no exceptions cross the
 * boundary, no torch/CUDA types in signatures (device pointers and streams travel as void*).
 * All calls on one handle must be serialised by the caller (the reference calls everything from the
 * render thread: main.gd:122,152,156).  There is NO CPU fallback: every entry point fails with
 * GSR_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef GSR_H_
#define GSR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_API __attribute__((visibility("default")))

/* ---- status codes ---- */
enum {
    GSR_OK = 0,
    GSR_ERR_INVALID = 1,  /* bad argument / out-of-range size */
    GSR_ERR_CUDA = 2,     /* CUDA runtime failure, or no usable device (see gsr_last_error) */
    GSR_ERR_OOM = 3,      /* device allocation failed */
    GSR_ERR_STATE = 4,    /* call order violated (e.g. render before resize) */
    GSR_ERR_OVERFLOW = 5  /* duplicate list exceeded capacity (main.gd:100 "(buffer overflow!)") */
};

/* ---- gsr_config.flags ---- */
#define GSR_FLAG_REFERENCE_QUIRKS 0x1u /* reproduce gsplat_boundaries.glsl:47-49 tile-range quirks (Q10); default */
#define GSR_FLAG_FIXED_RANGES     0x2u /* corrected tile ranges instead (every occupied tile gets [start,end)) */
#define GSR_FLAG_FAST_REJECT      0x4u /* sharded (row-interleaved) contexts: force the conservative early reject + CTA-level compaction
                                          in the projection (exact; selected automatically from 6 ranks, where it is faster) */

#define GSR_FLAG_STATIC_CAPACITY  0x8u /* keep the reference's fixed duplicate capacity factor*N and truncate on overflow (rasterizer.gd:79,
                                          main.gd:100).  Default: the capacity starts at factor*N and GROWS -- every frame's M reaches a
                                          pinned host mirror without a host sync and the buffers are enlarged once M passes half of them;
                                          gsr_render with a host pointer re-renders a frame that still overflowed, so it never returns a
                                          truncated frame; an asynchronous frame that overflowed is flagged (gsr_stats.overflow /
                                          gsr_frame_record.overflow) and the next one has room */

#define GSR_FLAG_UNCONTRACTED_BLEND 0x10u /* debug: evaluate gsplat_render.glsl:84-90 with one rounding per GLSL operator (no fma anywhere).
                                            The default contracts at the five GLSL-legal points of the gsr spec (DESIGN.md section 4); without
                                            contraction the frame is bit-identical to the reference's own shader text executed on the CPU
                                            (oracle/_ref; oracle.set_blend_contraction(False)). */

#define GSR_FLAG_ORTHOGRAPHIC 0x20u /* render orthographic cameras (Godot Camera3D.PROJECTION_ORTHOGONAL).  On a context created with this
                                      flag, a frame whose projection's w row is exactly (0, 0, 0, 1) -- view_proj[19] == 0, [23] == 0,
                                      [27] == 0, [31] == 1, what Godot's Projection::set_orthogonal gives -- takes the orthographic
                                      projection path: the cull keeps the whole [near, far] slab, the EWA Jacobian has no depth divide,
                                      the SH view direction is the camera's forward axis, and the 16-bit depth key is linear in view
                                      depth, t = clamp(ndc.z * 0.5 + 0.5, 0, 1), key = uint(t * 65535).  It resolves depth to
                                      (far - near) / 65536: set near / far around the content.  Every other frame (perspective and
                                      frustum matrices, anything the reference's packing produces: it writes (0, 0, -1, 0)) takes the
                                      perspective path unchanged.  The choice is made per frame when it is enqueued, without a sync.
                                      A single-context feature (see "Single-context features"): an orthographic frame on a sharded
                                      context returns GSR_ERR_STATE and enqueues nothing. */

#define GSR_FLAG_SH_HALF 0x40u /* store the SH coefficients of the gsr_config.sh_bands bands as IEEE binary16 (no reference counterpart):
                                   a degree-3 splat takes 144 instead of 240 bytes.  Planes 0-2 (position / time, covariance, opacity)
                                   stay float32.  Every upload rounds each coefficient once, on the device: h(c) = c rounded to
                                   binary16 to nearest even, subnormal halves and signed zeros kept, finite or infinite values beyond
                                   +-65504 saturated to +-65504, NaN kept a NaN (payload and sign unspecified).  Layout: after planes
                                   0-2 come P_h = ceil(3K / 8) planes of 16 bytes per splat (K = B^2; B = 1..4 gives 1, 2, 4, 6 planes:
                                   64 / 80 / 112 / 144 B per splat); value i = 3k + channel sits in plane 3 + (i >> 3), slot i & 7 of its
                                   8 halves (slot 0 = the low half of the plane's first 32-bit word), slots past 3K are +0.  Every frame
                                   is bit for bit the frame of the same context without the flag holding the cloud whose coefficients
                                   are float(h(c)), with every frame feature and every rendered degree (gsr_set_sh_degree reads the
                                   first ceil(3 (d+1)^2 / 8) half planes).  Fixed at creation.  A single-context feature, like a
                                   reduced store (see "Single-context features"; DESIGN.md section 5.14). */

/* ---- gsr_debug_copy selectors (parity taps; not on the frame path) ---- */
enum {
    GSR_BUF_RECORDS = 0, /* 48 B RasterizeData per splat id (gsplat_projection.glsl:42-48), max_splats entries */
    GSR_BUF_KEYS = 1,    /* sorted keys, M entries (descriptors['sort_keys'] half 0) */
    GSR_BUF_VALUES = 2,  /* sorted values, M entries (descriptors['sort_values'] half 0) */
    GSR_BUF_BOUNDS = 3,  /* uvec2 per tile (descriptors['tile_bounds']) */
    GSR_BUF_KEYS_UNSORTED = 4,  /* keys in emission order (only valid if flags keep them; see gsr_debug_keep_unsorted) */
    GSR_BUF_VALUES_UNSORTED = 5,
    GSR_BUF_FRAMEBUFFER = 6,  /* RGBA32F W*H (descriptors['render_texture']) */
    GSR_BUF_COMPOSITOR_TRACE = 7,       /* schedule trace of the last frame's compositor (gsr_debug_enable_trace) */
    GSR_BUF_COMPOSITOR_TRACE_COUNT = 8, /* number of trace items written (uint32) */
    GSR_BUF_INSTANCES = 9,              /* gsr_set_instances: 24 floats per instance, to_frame as given then the library's inverse
                                           [A^-1 | -A^-1 t] rounded to float (both 3x4, column-major) */
    GSR_BUF_SPLATS = 10,                /* the stored splat planes, plane-major: (3 + P) x plane_stride float4, plane_stride = max_splats
                                           rounded up to 256 (gsr_config.sh_bands; 3 + P_h planes of binary16 SH with GSR_FLAG_SH_HALF) */
    GSR_BUF_DEPTH_WORDS_UNSORTED = 11,  /* gsr_set_depth_order: the last mode-1 frame's ord(d) per pair in emission order, M entries
                                           (kept with gsr_debug_keep_unsorted once mode 1 has been switched on) */
    GSR_BUF_INSTANCE_APPEARANCE = 12,   /* gsr_set_instance_appearance: one gsr_instance_appearance per instance as stored (the default
                                           when none was set) */
    GSR_BUF_EDIT_TRANSFORM = 13,        /* gsr_transform_selection: the last accepted call's to_source (12 floats), then M~_1, M~_2, M~_3
                                           row-major (9 + 25 + 49): 95 floats, zeros before the first call */
    GSR_BUF_EDIT_COLOR = 14             /* gsr_recolor_selection: the last accepted call's A (9 floats, row-major), d (3), N~_1, N~_2, N~_3
                                           (27, row-major), s and t: 41 floats, zeros before the first call */
};

typedef struct gsr_ctx gsr_ctx;       /* one rasterizer = one GaussianSplattingRasterizer instance */
typedef struct gsr_sorter gsr_sorter; /* stand-alone radix sorter (config c5 microbench) */

typedef struct gsr_config {
    int32_t device;               /* CUDA ordinal (RenderingServer.get_rendering_device(), rasterizer.gd:70) */
    uint32_t flags;               /* GSR_FLAG_*; 0 = GSR_FLAG_REFERENCE_QUIRKS */
    uint64_t max_splats;          /* point_cloud.size (rasterizer.gd:79,83) */
    uint32_t dup_capacity_factor; /* initial sort capacity = factor * max_splats; 0 -> 10 (rasterizer.gd:79); grows on demand */
    uint32_t sh_bands;            /* SH bands the context stores = SH degree + 1: 1 (DC only) .. 4 (degree 3); 0 -> 4.  The splat buffer holds
                                     3 + P float4 planes per splat, P = ceil(3 B^2 / 4) = 1, 3, 7, 12: 64 / 96 / 160 / 240 bytes.  Uploads drop
                                     the coefficients the store does not keep.  > 4: GSR_ERR_INVALID.  A store of fewer than 4 bands is a
                                     single-context feature (see "Single-context features"). */
} gsr_config;

typedef struct gsr_stats {
    uint64_t num_splats;  /* the cloud's size n: uploads raise it to first + count when that is larger; gsr_delete_hidden,
                             gsr_duplicate_selection and gsr_set_splat_count set it (see "Splat delete and duplicate") */
    uint64_t duplicates;  /* M = histogram[0] of the reference (main.gd:98) -- true count, may exceed capacity */
    uint64_t visible;     /* V: splats that passed the cull and touch >= 1 tile */
    uint64_t capacity;    /* sort capacity in pairs */
    int64_t last_tile;    /* largest tile id touched by any visible splat (-1 if none) */
    uint32_t overflow;    /* 1 if duplicates > capacity in the last frame */
    uint32_t width, height, tiles_x, tiles_y;
    uint32_t band_y0, band_y1;  /* tile-row band rendered by this context */
    uint32_t kernel_launches;   /* kernels launched by the last gsr_render */
    float stage_ms[5];    /* 'Projection','Sort','Boundaries','Render' (rasterizer.gd:139,150,155,160) + total */
    uint64_t staged;      /* C: instances actually staged by the compositor (sum of consumed chunk sizes) */
} gsr_stats;

/* One entry of the per-frame history ring (the last GSR_HISTORY_FRAMES frames rendered by a context). */
#define GSR_HISTORY_FRAMES 512
typedef struct gsr_frame_record {
    uint64_t frame_index; /* 0-based count of gsr_render calls on this context */
    uint64_t duplicates;  /* M */
    uint64_t visible;     /* V */
    uint64_t staged;      /* C */
    uint32_t overflow;
    uint32_t reserved;
    float stage_ms[5];    /* Projection, Sort, Boundaries, Render, total (= their sum) -- GPU time between CUDA events around every stage */
    float front_ms;       /* the part of Projection that ran on the front stream (clear + projection kernel): overlapped with the previous
                             frame's compositor when frames are enqueued back to back, so the frame period is shorter than `total` */
} gsr_frame_record;

/* ---- lifecycle: replaces _init/init_gpu/cleanup_gpu (rasterizer.gd:59-120) and RenderingContext
 *      (render_context.gd:35-51).  Allocates every buffer of rasterizer.gd:83-92 (SoA instead of AoS). ---- */
GSR_API int gsr_create(const gsr_config *cfg, gsr_ctx **out);
GSR_API int gsr_destroy(gsr_ctx *ctx);

/* Use an existing CUDA stream (cudaStream_t as void*; NULL = the context's own stream).  The host that
 * owns the GPU work queue (Godot's render thread; torch's current stream in bench.py) passes its stream. */
GSR_API int gsr_set_stream(gsr_ctx *ctx, void *cuda_stream);

/* ---- splat upload: replaces device.buffer_update(buffer, i*STRUCT_SIZE*stride*4, ...) of
 *      PlyFile.load_gaussian_splats (util/ply_file.gd:71).  `splat60` = `count` std430 Splat structs of
 *      60 floats (gsplat_projection.glsl:33-40) in host memory; converted to SoA planes on the device.
 *      May be called repeatedly with disjoint or overlapping ranges (chunked async load). ---- */
GSR_API int gsr_upload_splats_aos(gsr_ctx *ctx, const float *splat60, uint64_t first, uint64_t count);

/* Same, but from RAW PLY vertices (scope row f1): `ply` = `count` vertices of `nprops` float32 each in the standard 3DGS
 * order (x,y,z,nx,ny,nz,f_dc_0..2,f_rest_0..44,opacity,scale_0..2,rot_0..3,...).  The per-splat preprocessing of
 * PlyFile.load_gaussian_splats (util/ply_file.gd:44-69: exp(scale), quaternion -> R, Sigma = R S^2 R^T, sigmoid(opacity),
 * SH re-interleave) runs on the device and writes the SoA planes directly; `creation_time` stamps the chunk (:40,47). */
GSR_API int gsr_upload_ply_raw(gsr_ctx *ctx, const float *ply, uint32_t nprops, uint64_t first, uint64_t count, float creation_time);

/* Same, for PLY vertices of any SH degree and property order (DC-only exports, degree-1 and degree-2 trainings, files without the
 * nx ny nz normals, extra properties): `layout` names where each group sits in a vertex of `nprops` floats.  f_rest holds
 * 3 * ((sh_degree + 1)^2 - 1) floats, channel-major (R.., G.., B..) as the 3DGS trainer writes them.  Coefficients above the file's
 * degree are stored as zero, those above the store's (gsr_config.sh_bands) are dropped.  The preprocessing is that of
 * gsr_upload_ply_raw, which is this call with the standard layout {62, 3, 0, 6, 9, 54, 55, 58}.  GSR_ERR_INVALID: a NULL layout,
 * nprops outside 1..256, sh_degree > 3, a group that does not fit inside nprops, f_rest >= 0 with sh_degree 0 or < 0 with
 * sh_degree > 0, or an upload range beyond max_splats. */
typedef struct gsr_ply_layout {
    uint32_t nprops;     /* floats per vertex, 1..256 */
    uint32_t sh_degree;  /* of the file, 0..3 */
    int32_t x, f_dc, f_rest, opacity, scale, rot;  /* index of x (y, z follow), f_dc_0, f_rest_0 (-1 iff degree 0), opacity, scale_0, rot_0 */
} gsr_ply_layout;
GSR_API int gsr_upload_ply(gsr_ctx *ctx, const float *ply, const gsr_ply_layout *layout, uint64_t first, uint64_t count, float creation_time);

/* gsr_upload_ply, plus the per-splat 3D filter of Mip-Splatting: filter_3d = index of the `filter_3D` property, -1 = none
 * (then exactly gsr_upload_ply).  Mip-Splatting's trainer writes filter_3D to point_cloud.ply and its renderer folds it into scale and
 * opacity; gsr_upload_ply ignores the property, so such a cloud renders too thin.  Here, for a splat with f = filter_3D > 0, in float64
 * and narrowed to float once: q_i = exp(scale_i)^2, q'_i = q_i + f*f, the covariance is built from the scales sqrt(q'_i) and the opacity
 * is sigmoid(opacity) * sqrt((q_0 q_1 q_2) / (q'_0 q'_1 q'_2)).  A splat with f <= 0 or NaN is stored exactly as gsr_upload_ply stores
 * it.  Load-time data preparation: any context may use it.  GSR_ERR_INVALID: what gsr_upload_ply rejects, or filter_3d outside
 * -1..nprops-1.  Such clouds are trained with the 2D filter of gsr_set_antialiasing at 0.1. */
GSR_API int gsr_upload_ply_filtered(gsr_ctx *ctx, const float *ply, const gsr_ply_layout *layout, int32_t filter_3d,
                                    uint64_t first, uint64_t count, float creation_time);

/* ---- texture_size setter (rasterizer.gd:26-48): reallocates tile_bounds + render_texture ---- */
GSR_API int gsr_resize(gsr_ctx *ctx, int32_t width, int32_t height);

/* Multi-GPU tile-row sharding (no counterpart in the single-device reference): this context renders tile
 * rows [row_begin, row_end) only; keys keep the global tile id.  (0, tiles_y) restores the full frame. */
GSR_API int gsr_set_band(gsr_ctx *ctx, int32_t row_begin, int32_t row_end);

/* Cyclic tile-row ownership for balanced multi-GPU sharding: this context owns the tile rows with
 * row % row_mod == row_rem (inside its band).  row_mod > 1 selects the FAST sharded mode: the projection rejects, with a
 * conservative radius bound, splats that cannot touch an owned row, so it no longer knows the frame-global last
 * occupied tile that the reference's tile-range quirk (gsplat_boundaries.glsl:47-49) depends on.  Instead every rank
 * leaves its local last occupied tile + 1 in the int32 at gsr_band_sync_word(); the host all-reduces that word (MAX,
 * in place, on the render stream) after the frame and calls gsr_band_fixup, which blanks the one affected tile on the
 * rank that owns it.  (1, 0) restores the exact single-context behaviour. */
GSR_API int gsr_set_row_interleave(gsr_ctx *ctx, int32_t row_rem, int32_t row_mod);
GSR_API void *gsr_band_sync_word(gsr_ctx *ctx);
GSR_API int gsr_band_fixup(gsr_ctx *ctx);

/* Fused compositor + framebuffer gather over NVLink peer memory (replaces the NCCL gather of SURVEY 8e): the presenting
 * rank exports CUDA-IPC handles of its two frames (2 x 64 bytes); every other rank imports them, after which its
 * compositor stores its tile-row band straight into the presenting rank's memory.  In this mode gsr_render_async is
 * called with a NULL host pointer on every rank (frames alternate between the two buffers in lockstep), the ranks
 * synchronise per frame with any 4-byte collective, and the presenting rank calls gsr_readback_async. */
GSR_API int gsr_peer_export_framebuffers(gsr_ctx *ctx, void *handles128);
GSR_API int gsr_peer_import_framebuffers(gsr_ctx *ctx, const void *handles128);

/* ---- Single-context features: frame features that work only on a context that renders the whole frame by itself.
 *        - depth compositing (gsr_set_depth_compositing), with its companions motion vectors and splat IDs;
 *        - instances (gsr_set_instances with n > 0);
 *        - a store of fewer than 4 SH bands (gsr_config.sh_bands), a binary16 store (GSR_FLAG_SH_HALF), and a rendered SH degree
 *          below 3 (gsr_set_sh_degree 0..2);
 *        - anti-aliasing (gsr_set_antialiasing > 0);
 *        - view-depth order (gsr_set_depth_order GSR_DEPTH_ORDER_VIEW_DEPTH);
 *        - cutouts (gsr_set_cutouts with n > 0);
 *        - splat masks in use (gsr_select_*, gsr_set_splat_masks; until gsr_clear_splat_masks);
 *        - orthographic frames (GSR_FLAG_ORTHOGRAPHIC; the flag alone is no feature, each orthographic frame is).
 *      A context is sharded while any of these holds:
 *        - a shard group is attached (gsr_group_attach with world > 1);
 *        - it exported or imported peer framebuffers (gsr_peer_export_framebuffers / gsr_peer_import_framebuffers);
 *        - its band is not the full frame (gsr_set_band other than (0, tiles_y));
 *        - row_mod > 1 (gsr_set_row_interleave).
 *      gsr_resize detaches the group and drops the peer framebuffers.  The rule holds in both directions, with GSR_ERR_STATE and
 *      the context left as it was:
 *        - on a sharded context, every call that would turn a feature on is refused, and an orthographic frame enqueues nothing;
 *        - while a feature is on, every call that would shard the context is refused: gsr_set_band with a partial band,
 *          gsr_set_row_interleave with row_mod > 1, gsr_group_attach with world > 1, and both gsr_peer_* calls.
 *      The calls that turn a feature off, gsr_set_band(0, tiles_y) and gsr_set_row_interleave(0, 1) are never refused by the rule.
 *      gsr_group_export is refused as well while a feature is on, except for depth compositing and instances: a context with
 *      those may export, but not attach with world > 1. ---- */

/* ---- rasterize() (rasterizer.gd:122-160).
 *      view_proj: the 128-byte push constant of update_camera_matrices (rasterizer.gd:181-193):
 *                 view_matrix then projection_matrix, GLSL column-major.
 *      uniforms:  the 32-byte uniform block of rasterizer.gd:126, byte-identical:
 *                 float camera_pos[3], float model_scale, int32 width, int32 height, float time, pad.
 *                 (width/height must equal the gsr_resize values.)
 *      heatmap_factor: float(should_enable_heatmap) (rasterizer.gd:158).
 *      out_rgba32f_host: NULL (frame stays on the device, like the reference's Texture2DRD) or a host
 *                 buffer of width*height*4 floats that receives the frame (synchronous).
 *      Enqueues on the context's stream and returns without a host sync when out_rgba32f_host is NULL. */
GSR_API int gsr_render(gsr_ctx *ctx, const float view_proj[32], const void *uniforms32, float heatmap_factor,
                       float *out_rgba32f_host);

/* Pipelined host read-back: enqueue the frame and an asynchronous device->host copy into `pinned_host` (page-locked
 * memory; with pageable memory the copy degrades to a synchronous one).  Frames alternate between two internal
 * framebuffers and the copy runs on a separate stream, so the read-back of frame i overlaps the kernels of frame i+1.
 * gsr_stream_join makes the render stream wait for all copies enqueued so far (so that an event recorded on the
 * render stream afterwards covers them); gsr_sync blocks the host until renders and copies are complete. */
GSR_API int gsr_render_async(gsr_ctx *ctx, const float view_proj[32], const void *uniforms32, float heatmap_factor,
                             float *pinned_host);
/* Same, but the host frame is RGB32F (width*height*3 floats): the alpha channel of the reference's output is the
 * constant 1.0 (gsplat_render.glsl:101), so it is packed away on the device before the PCIe transfer (-25 % bytes). */
GSR_API int gsr_render_async_rgb(gsr_ctx *ctx, const float view_proj[32], const void *uniforms32, float heatmap_factor,
                                 float *pinned_host_rgb);
/* ---- presentation hand-off (scope row f3; resources/shaders/spatial/main.gdshader:7-19, rasterizer.gd:41,48,92,101).
 *      The reference keeps an RGBA32F image and converts sRGB -> linear in the fragment shader that samples it.  A consumer that
 *      wants fewer bytes (PCIe read-back, the gather message) or the converted values asks for them here; the conversion is fused
 *      into the copy-out kernel.  format = GSR_OUT_* optionally OR-ed with GSR_OUT_SRGB_TO_LINEAR (rgb channels only). ---- */
enum {
    GSR_OUT_RGBA32F = 0, /* 16 B/pixel: the reference's texture, bit for bit */
    GSR_OUT_RGB32F = 1,  /* 12 B/pixel: alpha is the constant 1.0 (gsplat_render.glsl:101) */
    GSR_OUT_RGBA16F = 2, /*  8 B/pixel: IEEE binary16, round to nearest even */
    GSR_OUT_RGBA8 = 3    /*  4 B/pixel: UNORM8 = rint(clamp(x, 0, 1) * 255) */
};
#define GSR_OUT_SRGB_TO_LINEAR 0x100 /* apply main.gdshader:7-11 srgb_to_linear() to r,g,b first (pow = the library's deterministic pow) */
GSR_API size_t gsr_output_bytes(int32_t format, int32_t width, int32_t height);
/* gsr_render_async with a converted host frame (gsr_output_bytes(format, w, h) bytes of page-locked memory). */
GSR_API int gsr_render_async_fmt(gsr_ctx *ctx, const float view_proj[32], const void *uniforms32, float heatmap_factor,
                                 void *pinned_host, int32_t format);
/* Read the most recently rendered library-owned frame back to page-locked host memory on the copy stream, ordered
 * after everything enqueued on the render stream so far (shard group: after every rank's rows have landed).
 * format: GSR_OUT_* (0 = RGBA32F, 1 = RGB32F -- the former `rgb_only` argument). */
GSR_API int gsr_readback_async(gsr_ctx *ctx, void *pinned_host, int32_t format);
/* Converted copy of the most recent frame into caller-owned DEVICE memory, on the render stream, no host involvement: the
 * zero-copy hand-off to an image the embedder imported from its graphics API (Vulkan VK_KHR_external_memory_fd ->
 * cudaImportExternalMemory -> cudaExternalMemoryGetMappedBuffer; see INTEGRATION.md). */
GSR_API int gsr_present_device(gsr_ctx *ctx, void *dst_device, int32_t format);
GSR_API int gsr_stream_join(gsr_ctx *ctx);

/* ---- Multi-GPU shard group (no reference counterpart -- the reference is single-device; SURVEY 8e).  One context per GPU,
 *      in one process (a thread per GPU) or in one process per GPU.  The frame path of an attached group uses neither the
 *      host nor NCCL: per frame every rank (1) projects ITS slice of the splats (cull, EWA, SH: once per splat in the whole group) and
 *      stores every (key, value) pair and every 48-byte record into the memory of the rank that owns the pair's tile row
 *      (cyclic rows: row % world == rank) with peer stores over NVLink/NVSwitch, in splat-id order per destination, (2) packs,
 *      sorts and scans the pairs it received, (3) composites its rows straight into the presenting rank's (rank 0) frame, or
 *      keeps them (gsr_group_set_present); sequence-numbered flag words behind one system-scope fence per kernel order all of
 *      it on the devices.
 *      Results are bit-identical to the single-GPU frame (same rects, same emission order, exact Q10 bookkeeping).
 *        every rank:  gsr_resize; gsr_group_export(ctx, blob)            -> exchange the blobs (any transport)
 *                     gsr_group_attach(ctx, rank, world, all_blobs)       -> barrier once (any transport)
 *        per frame:   gsr_render_async(ctx, vp, uniforms, heat, NULL) on every rank (same frame order everywhere);
 *                     rank 0: gsr_readback_async(ctx, pinned, format) and/or gsr_present_device / gsr_framebuffer_device_ptr
 *      gsr_resize detaches (export / attach again).  A lost peer makes the bounded device-side waits expire: gsr_sync then
 *      returns GSR_ERR_STATE instead of the GPU hanging. ---- */
#define GSR_GROUP_BLOB_BYTES 320
#define GSR_GROUP_MAX_RANKS 16
GSR_API int gsr_group_export(gsr_ctx *ctx, void *blob /* GSR_GROUP_BLOB_BYTES */);
GSR_API int gsr_group_attach(gsr_ctx *ctx, int32_t rank, int32_t world, const void *blobs /* world x GSR_GROUP_BLOB_BYTES, rank order */);
GSR_API int gsr_group_detach(gsr_ctx *ctx);
/* Where an attached group presents (same value on every rank; default 0):
 *   0  rows are composited into rank 0's frames over NVLink -- the frame is complete on ONE device (display GPU, gsr_present_device,
 *      gsr_readback_async on rank 0);
 *   1  every rank keeps its rows in its own frames and reads them back itself with gsr_readback_rows_async into one full-frame
 *      RGBA32F host image that is page-locked in every rank's process (shared memory): a host consumer gets the frame over
 *      world PCIe links instead of one, and no frame data crosses NVLink at all. */
GSR_API int gsr_group_set_present(gsr_ctx *ctx, int32_t rows_local);
GSR_API int gsr_readback_rows_async(gsr_ctx *ctx, void *host_frame_rgba32f);
GSR_API int gsr_sync(gsr_ctx *ctx);

/* Device pointer of the RGBA32F frame (render_texture.texture_rd_rid, rasterizer.gd:48,101); row-major W*H. */
GSR_API void *gsr_framebuffer_device_ptr(gsr_ctx *ctx);
/* Render into caller-owned device memory instead (>= width*height*16 bytes; NULL restores the internal one). */
GSR_API int gsr_set_framebuffer_external(gsr_ctx *ctx, void *device_ptr);

/* ---- Depth compositing: splats composited into the host's 3D scene (no reference counterpart: the reference shows an opaque
 *      frame on a full-screen quad).  Both pointers are caller-owned device float[width*height], row-major like the frame.
 *      depth_out_device != NULL switches the mode on, NULL switches it off (scene_depth_device must then be NULL too).
 *      scene_depth_device (optional, NULL = nothing occludes) holds the scene's LINEAR view depth per pixel: the distance along
 *      the camera's viewing axis, positive in front of the camera (Godot: -(VIEW_MATRIX * world position).z), in the world units
 *      of view_proj; +inf = nothing.  Per pixel, in the tile's sorted order, the compositor stops before the first splat whose
 *      view depth d = -(view_matrix * splat position).z is not in front of the scene depth (!(d < Z), NaN included): that splat and
 *      every later one contribute nothing.  The frame then carries:
 *        rgb   = the same blend as the default frame (bit-identical to it without a scene depth), i.e. premultiplied colour;
 *        alpha = 1 - t, the splats' coverage (the default frame's alpha is the constant 1.0);
 *      and depth_out the coverage-weighted linear view depth of the blended splats, +inf where nothing was blended.
 *      depth_out is written by every frame's compositor on the render stream; the caller orders its reads like those of an
 *      external framebuffer.  GSR_OUT_RGB32F drops the coverage; GSR_OUT_SRGB_TO_LINEAR converts the premultiplied values as
 *      they are.  A single-context feature (see "Single-context features").  gsr_resize switches the mode off;
 *      gsr_pick keeps the default path (and leaves the depth-composited frame as it is).  GSR_ERR_STATE before gsr_resize. ---- */
GSR_API int gsr_set_depth_compositing(gsr_ctx *ctx, const float *scene_depth_device, float *depth_out_device);

/* ---- Motion vectors: the per-pixel screen motion of the splats since the previous frame, for a host's temporal anti-aliasing,
 *      upscaler or motion blur (no reference counterpart).  motion_out_device: caller-owned device float[2*width*height], (x, y) per
 *      pixel, row-major like the frame; NULL switches the mode off.  A companion of depth compositing: GSR_ERR_STATE while depth
 *      compositing is off (a NULL scene depth is enough), and gsr_set_depth_compositing(ctx, NULL, NULL) and gsr_resize switch it off;
 *      its single-context rules are those of depth compositing.  GSR_ERR_INVALID, previous state kept: a pointer equal to depth_out or
 *      scene_depth.  The pointer is read when a frame is enqueued (frames already enqueued keep theirs: a host may double-buffer its
 *      velocity textures).  The call never synchronises, allocates or copies.
 *      Motion of one staged splat (float32, one rounding per operation, no contraction):
 *        - p is the record's frame-space position, the one gsr_pick returns and depth compositing uses; p' its position in the previous
 *          frame: p' = p without instances (uploads and the load-in animation are not motion); for drawn id v of instance k the source
 *          splat is s = first_k + (v - 32 w_k), sp = (x_s ms, y_s ms, z_s ms) with this frame's model_scale ms, and
 *          p'[r] = ((A'[r] sp0 + A'[3+r] sp1) + A'[6+r] sp2) + A'[9+r] with A' instance k's previous to_frame (an unchanged transform
 *          gives p' == p bit for bit);
 *        - pix(M, q) for a view_proj M = (V, P): view[r] = ((V[r] q0 + V[4+r] q1) + V[8+r] q2) + V[12+r],
 *          clip[r] = ((P[r] view0 + P[4+r] view1) + P[8+r] view2) + P[12+r] view3 (r = 0, 1, 3), and
 *          pix = (((clip0/clip3 + 1) 0.5) (W-1), ((clip1/clip3 + 1) 0.5) (H-1)): the projection's image_pos without the load-in term;
 *        - m = pix(M', p') - pix(M, p), previous minus current, in the frame's pixel axes (column, row; y grows downwards); (0, 0) unless
 *          clip3' > 0 and both components are finite.
 *      Per pixel m.x and m.y accumulate exactly like depth_out (same stop rule and transmittance: fma(m alpha, t, M), unfused under
 *      GSR_FLAG_UNCONTRACTED_BLEND), and motion_out = (Mx / (1 - t), My / (1 - t)), (0, 0) where 1 - t == 0.  rgba and depth_out are
 *      bit-identical to the frame without motion vectors.
 *      Previous state: the context records the view_proj and the instance transforms of every frame enqueued by gsr_render* (motion on
 *      or off); a frame's previous state is the last enqueued frame's, except that it is the frame's own for the context's first frame,
 *      the first frame after gsr_resize and the first after gsr_reset_motion (a camera cut), and, per instance, when the previous frame
 *      had a different instance layout (another (first, count) sequence, or no instances).  gsr_render's re-render of a frame that
 *      overflowed is the same frame with the same previous state; gsr_pick neither reads nor updates the history and leaves
 *      motion_out as it is. ---- */
GSR_API int gsr_set_motion_vectors(gsr_ctx *ctx, float *motion_out_device);
GSR_API int gsr_reset_motion(gsr_ctx *ctx);

/* ---- Splat and instance IDs: per pixel, which splat and which instance dominate the depth-composited blend, for click picking,
 *      selection outlines and any post effect that needs to know which object owns a pixel (no reference counterpart).
 *      ids_out_device: caller-owned device uint32_t[2*width*height], (v, k) per pixel, row-major like the frame; NULL switches the
 *      mode off.  A companion of depth compositing: GSR_ERR_STATE while depth compositing is off (a NULL scene depth is enough), and
 *      gsr_set_depth_compositing(ctx, NULL, NULL) and gsr_resize switch it off; its single-context rules are those of depth
 *      compositing.  GSR_ERR_INVALID, previous state kept: a pointer equal to depth_out, scene_depth or motion_out
 *      (gsr_set_motion_vectors likewise refuses the ID plane while IDs are on).  The pointer is read when a frame is enqueued (frames
 *      already enqueued keep theirs: a host may double-buffer).  The call never synchronises, allocates or copies.
 *      Rule: a pixel's splats are those its depth-composited blend blends (same stop rule at the scene depth, same dead-pixel rule
 *      t > 1/255, same sorted order).  For each, w = t - t' in float32 (one subtraction), with t the pixel's transmittance before the
 *      splat and t' = t * (1 - alpha) the value the blend stores after it; alpha is that of the context's blend (contracted, or
 *      GSR_FLAG_UNCONTRACTED_BLEND).  The pixel's splat is the first in sorted order with the largest w: a later splat replaces it
 *      only when its w is strictly greater.
 *        v = its drawn id, the sort value: the splat index without instances; with instances, drawn id v of instance k maps to source
 *            splat first_k + (v - 32 w_k) (see gsr_set_instances);
 *        k = the instance that owns drawn warp v >> 5, GSR_NO_ID without instances.
 *      A pixel where no splat has w > 0 (exactly where the coverage alpha 1 - t is 0) holds (GSR_NO_ID, GSR_NO_ID).  Hidden
 *      instances and splats beyond an instance's draw_count are never blended, so they never appear.  rgba, depth_out and motion_out
 *      are bit-identical to the frame without IDs; pixels outside the image are not written.  gsr_render's re-render of a frame
 *      that overflowed writes the same IDs; gsr_pick keeps the default path and leaves the ID plane as it is. ---- */
#define GSR_NO_ID 0xFFFFFFFFu
GSR_API int gsr_set_splat_ids(gsr_ctx *ctx, uint32_t *ids_out_device);

/* ---- Splat instances (no reference counterpart: the reference draws one cloud at the origin).  An instance draws the source range
 *      [first, first + count) of the uploaded splats with its own affine transform `to_frame` = [A | t] (3x4, column-major: columns
 *      a0, a1, a2, t) from the range's splat coordinates (position * model_scale) into FRAME space, the space the uploaded splats, the
 *      view matrix of view_proj and uniforms.camera_pos live in.  With n > 0 instances set, every later gsr_render* draws exactly the
 *      instances' splats, all of them in ONE sorted frame, so overlapping clouds blend in the correct order:
 *        - ranges may overlap and the same range may be drawn any number of times (one asset stored once, drawn many times);
 *          splats outside every range are not drawn;
 *        - instance k is projected with V_k = V * [A|t] in place of the view matrix and cam_k = A^-1 (camera_pos - t) in place of the
 *          camera position: cull, EWA covariance, depth key and the SH view direction (evaluated in the object's own frame) follow
 *          the default projection exactly; the records' position words hold the frame-space position A * sp + t, so gsr_pick returns
 *          frame-space positions and depth compositing works unchanged.  For rigid and uniformly scaled transforms this is the
 *          transformed cloud; with a non-uniform scale positions and covariances are still exact, but the SH colour is evaluated
 *          in the object's frame (the coefficients are not rotated);
 *        - drawn ids: instance k owns [32 w_k, 32 w_k + count_k), w_k = sum over j < k of ceil(count_j / 32); D = 32 * sum ceil(count/32).
 *          Pairs of equal keys keep instance order, then source order.  GSR_BUF_RECORDS returns D records.
 *      The array is copied; frames already enqueued keep the transforms they were enqueued with.  A call with the same (first, count)
 *      sequence as the current instances only replaces the transforms: the per-frame path, it never synchronises the host (the
 *      transforms reach the device through a mapped page-locked ring consumed by a kernel on the frame's stream; only a host more than
 *      GSR_INSTANCE_RING frames ahead of the GPU waits for a slot).  Any other call re-lays out the drawn ids: it synchronises and may
 *      reallocate (record tables for max(max_splats, D) ids; the sort capacity is raised to factor * D when D > max_splats).
 *      n == 0 switches instancing off: the default frame.  GSR_ERR_INVALID, previous state kept: n > GSR_MAX_INSTANCES, a range beyond
 *      max_splats, a non-finite entry, a singular A, D >= 2^32 - 256.  A single-context feature (see "Single-context features").
 *      gsr_resize keeps the instances. ---- */
#define GSR_MAX_INSTANCES 4096
#define GSR_INSTANCE_RING 8
typedef struct gsr_instance {
    uint64_t first, count;  /* source range of the uploaded splats */
    float to_frame[12];     /* [A | t], column-major 3x4 */
} gsr_instance;
GSR_API int gsr_set_instances(gsr_ctx *ctx, const gsr_instance *instances, uint32_t n);

/* ---- Per-instance appearance: show and hide, fade, tint, and draw a prefix of every instance, changed per frame.  appearance[k]
 *      belongs to instance k of the current gsr_set_instances layout.  For instance k, in float32 with one rounding per operation:
 *        - drawn splats: live_k = min(count_k, draw_count), and 0 when opacity == 0 (-0.0f counts as 0).  Only the source splats
 *          [first_k, first_k + live_k) are drawn.  The drawn-id layout does NOT change: instance k keeps the ids
 *          [32 w_k, 32 w_k + count_k), so values, records and gsr_pick keep their ids; records of ids that are not drawn are
 *          unspecified, like those of culled splats.  A hidden instance, and every warp of 32 ids past live_k, reads no splat data;
 *        - opacity multiplies the STORED opacity of every splat before anything else reads it: the frame is exactly the frame of a
 *          cloud whose stored opacities were multiplied in float32 (load-in animation, anti-aliasing compensation, the splat's
 *          radius -- a faded splat's rect shrinks -- and the record's opacity word all follow from it);
 *        - tint multiplies the splat's colour channel-wise after the SH evaluation and its clamp at 0 (it cannot revive a clamped
 *          channel; it may exceed 1, the frame is float).
 *      With every instance at the default ({1, 1, 1}, 1, UINT64_MAX) the frame is bit for bit the frame without an appearance.
 *      n must equal the number of instances set; (NULL, 0) restores the default for every instance (valid with no instances too).
 *      The array is copied and read when a frame is enqueued: frames already enqueued keep theirs.  The call never synchronises,
 *      allocates device memory or copies to the device: the values travel with the transforms through the instance ring.
 *      gsr_set_instances with the same layout (the per-frame transform update) keeps the appearance; with a new layout, or n == 0, it
 *      resets every instance to the default.  gsr_resize keeps it.  GSR_ERR_INVALID, previous state kept: n differs from the instance
 *      count, a NULL array with n > 0, a NaN, infinite or out-of-range field (the message names the instance). ---- */
#define GSR_TINT_MAX 16.0f
typedef struct gsr_instance_appearance {
    float    tint[3];     /* multiplies the splat colour (r, g, b); finite, 0 <= tint <= GSR_TINT_MAX */
    float    opacity;     /* multiplies the stored splat opacity; 0 <= opacity <= 1; 0 = the instance is not drawn */
    uint64_t draw_count;  /* draw only the source splats [first, first + min(draw_count, count)); UINT64_MAX = all */
} gsr_instance_appearance;    /* 24 bytes; the default is {1, 1, 1}, 1, UINT64_MAX */
GSR_API int gsr_set_instance_appearance(gsr_ctx *ctx, const gsr_instance_appearance *appearance, uint32_t n);

/* ---- SH degree of the rendered colour (no reference counterpart: the reference always evaluates degree 3).  Frames enqueued after
 *      the call evaluate the view-dependent colour up to `degree` (0 = the DC colour only) from the first P = ceil(3 (degree+1)^2 / 4)
 *      SH planes, so a lower degree also reads fewer bytes.  -1 = the stored degree (gsr_config.sh_bands - 1), the default.  The degree
 *      is read when a frame is enqueued: frames already enqueued keep theirs, and the call never synchronises.  A frame drawn at
 *      degree d is bit for bit the frame of the same cloud with every coefficient above degree d set to zero (DESIGN.md section 5.9).
 *      GSR_ERR_INVALID: a degree below -1 or above the stored one.  A degree below 3, like a store of fewer than 4 bands, is a
 *      single-context feature (see "Single-context features"). ---- */
GSR_API int gsr_set_sh_degree(gsr_ctx *ctx, int32_t degree);

/* ---- Anti-aliased trainings (no reference counterpart: the reference dilates the 2D covariance by a fixed 0.3 px^2 and keeps the
 *      opacity as stored).  The original 3DGS trainer with --antialiasing, gsplat / nerfstudio with rasterize_mode="antialiased" and
 *      Mip-Splatting dilate by a variance v and also scale the opacity by sqrt(det(cov_2d) / det(cov_2d + v I)); their opacities are
 *      trained for that factor, so drawn the reference's way every sub-pixel splat is too opaque, more so as the camera zooms out.
 *      filter_variance: 0 = off (the reference: +0.3 dilation, opacity as stored; the default).
 *      > 0: frames enqueued afterwards dilate the 2D covariance by filter_variance (px^2) and multiply the opacity by the
 *      compensation factor coef = sqrt(max(0.000025, det(cov_2d) / det(cov_2d + v I))) (GLSL max: NaN gives the floor); that
 *      opacity also sets the splat's radius.  0.3 = 3DGS --antialiasing / gsplat "antialiased"; 0.1 = Mip-Splatting's 2D filter.
 *      The value is read when a frame is enqueued: frames already enqueued keep theirs, and the call never synchronises.  Back at 0
 *      the frame is bit for bit that of a context that never used the filter.  gsr_resize keeps the setting.  GSR_ERR_INVALID,
 *      previous state kept: a negative, NaN or infinite variance, or one above 64.  A single-context feature while the filter is on
 *      (see "Single-context features"). ---- */
GSR_API int gsr_set_antialiasing(gsr_ctx *ctx, float filter_variance);

/* ---- Order splats by exact view depth (no reference counterpart: the reference sorts each frame's pairs by tile << 16 | a 16-bit
 *      depth, so splats whose depths share a 16-bit bin -- 0.5 units wide at depth 100 with near = 0.05 -- keep splat-id order, which
 *      pops as the camera moves and can end a depth-composited pixel on a tied splat behind the scene).
 *      GSR_DEPTH_ORDER_KEY16 (0): the reference's order, the default.
 *      GSR_DEPTH_ORDER_VIEW_DEPTH (1): frames enqueued afterwards sort their pairs by (tile id, ord(d), emission order), d =
 *      -(((V[2] x + V[6] y) + V[10] z) + V[14]) in float32 with x, y, z the record's (frame-space) position and V the frame's view
 *      matrix (view_proj[0..15]) -- the d of depth compositing -- and ord the order-preserving map of a float's bits (every finite d,
 *      negative ones included; -0 just before +0).  Ties keep emission order (drawn-id order, tile order inside a splat's rect).  The
 *      keys, records, M, V, C, overflow and tile bounds are those of the default frame; only the order inside each tile's range
 *      changes, and GSR_BUF_KEYS / GSR_BUF_VALUES return it.  Works with instances, orthographic frames, anti-aliasing, reduced SH,
 *      depth compositing, the heat map, GSR_FLAG_STATIC_CAPACITY and front / back overlap.
 *      Cost: the projection writes 4 more bytes per pair and the sort takes six passes over 48 bits instead of four over 32 (about
 *      twice the sort's traffic; DESIGN.md section 5.12).  The first switch to mode 1 allocates 12 bytes per pair of capacity (and may
 *      synchronise once: GSR_ERR_OOM keeps the previous state); later switches never synchronise.  The mode is read when a frame is
 *      enqueued: frames already enqueued keep theirs, and gsr_resize keeps the setting.  GSR_ERR_INVALID: any other mode.
 *      Mode 1 is a single-context feature (see "Single-context features"). ---- */
#define GSR_DEPTH_ORDER_KEY16 0
#define GSR_DEPTH_ORDER_VIEW_DEPTH 1
GSR_API int gsr_set_depth_order(gsr_ctx *ctx, int32_t mode);

/* ---- Splat cutouts (no reference counterpart: the reference draws every splat of the cloud).  Up to GSR_MAX_CUTOUTS boxes and
 *      ellipsoids that crop the cloud (KEEP) or cut splats away (REMOVE) -- backgrounds, floaters, the ground a capture stood on,
 *      runtime cutaways -- without touching the uploaded data.  A splat is drawn iff
 *        - no KEEP volume is set, or its tested position is inside at least one KEEP volume, and
 *        - its tested position is inside no REMOVE volume.
 *      The order of the volumes does not matter.  The test is on the splat's CENTRE: a splat is kept or removed whole, its footprint
 *      is not clipped at the volume's boundary.  A removed splat is treated exactly like a frustum-culled one: no record, no pairs,
 *      no share of M, V or the last tile: the sort and the compositor see fewer pairs (DESIGN.md section 5.7 has measured costs).
 *      Tested position, in float32 with one rounding per operation: u[r] = ((C[r] x + C[3+r] y) + C[6+r] z) + C[9+r] with C =
 *      to_local ([A | t], column-major 3x4 like gsr_instance.to_frame: the tested position -> the unit shape's space) and
 *        - GSR_CUTOUT_SOURCE: (x, y, z) = the splat's source coordinates, position * model_scale (before any instance transform);
 *        - GSR_CUTOUT_FRAME: (x, y, z) = the record's position words: the source coordinates without instances, A * sp + t with them
 *          (the position gsr_pick returns and depth compositing uses).
 *      Without instances the two spaces coincide; with instances a SOURCE volume is an asset-space crop that travels with every copy
 *      of the asset, a FRAME volume a world-space cutaway.  Inside a box: |u0| <= 1 && |u1| <= 1 && |u2| <= 1 (the faces included);
 *      inside an ellipsoid: ((u0 u0 + u1 u1) + u2 u2) <= 1.  Comparisons are IEEE: a NaN coordinate is outside every volume.  A
 *      singular to_local is allowed (a flat slab, an infinite prism).
 *      The array is copied and read when a frame is enqueued: frames already enqueued keep their set.  The call never synchronises,
 *      allocates nothing and copies nothing to the device (the set travels with the projection's launch parameters).  n == 0 switches
 *      cutouts off: the default frame, bit for bit.  gsr_resize keeps the set.  GSR_ERR_INVALID, previous set kept: n >
 *      GSR_MAX_CUTOUTS, cutouts == NULL with n > 0, a non-finite to_local entry, an unknown shape, action or space.  A non-empty set
 *      is a single-context feature (see "Single-context features"). ---- */
#define GSR_MAX_CUTOUTS 16
#define GSR_CUTOUT_BOX 0        /* inside: |u0| <= 1 && |u1| <= 1 && |u2| <= 1 */
#define GSR_CUTOUT_ELLIPSOID 1  /* inside: ((u0*u0 + u1*u1) + u2*u2) <= 1 */
#define GSR_CUTOUT_KEEP 0       /* action: with any KEEP volume set, only splats inside one are drawn */
#define GSR_CUTOUT_REMOVE 1     /* action: splats inside are not drawn */
#define GSR_CUTOUT_FRAME 0      /* space: the record's frame-space position */
#define GSR_CUTOUT_SOURCE 1     /* space: the splat's source coordinates (before an instance transform) */
typedef struct gsr_cutout {
    float to_local[12];         /* [A | t], column-major 3x4: tested position -> the unit shape's space */
    int32_t shape, action, space;
} gsr_cutout;
GSR_API int gsr_set_cutouts(gsr_ctx *ctx, const gsr_cutout *cutouts, uint32_t n);

/* ---- Splat selection: select, highlight and hide individual splats (no reference counterpart).  The cleaning loop of a splat editor
 *      -- select floaters with a screen lasso, a volume or a click on what is visible, look at the highlighted selection, hide it, undo,
 *      export what is left -- without touching the uploaded data.
 *      State: two bitmasks over the SOURCE splats [0, max_splats), `hidden` and `selected`, one bit per splat, 32 splats per uint32 word
 *      (splat s is bit s & 31 of word s >> 5); bits at or past max_splats are always 0.  With instances, a source splat's bits apply to
 *      every instance that draws it (an edit of the asset, like a GSR_CUTOUT_SOURCE volume).  A hidden splat is never selected: every
 *      operation ends with selected &= ~hidden.
 *      The masks are IN USE from the first call that can set a bit (any gsr_select_*, gsr_set_splat_masks) until gsr_clear_splat_masks.
 *      The first such call allocates the masks zeroed (it may synchronise once; GSR_ERR_OOM keeps the previous state); later calls never
 *      synchronise and never allocate.  Uploads, gsr_resize, gsr_set_instances and appearance changes keep the masks.
 *      Frame rule, while the masks are in use: the source splat of a drawn id v is s = v without instances and s = first_k + (v - 32 w_k)
 *      with them (see gsr_set_instances).
 *        - hidden: the splat is removed after the frustum cull and the cutouts, exactly like a cutout-removed splat: no record, no
 *          pairs, no share of M, V or the last tile;
 *        - selected, with highlight strength s_h > 0: after the SH clamp and the instance tint, each colour channel becomes
 *          c' = (c * k) + h, an FMUL then an FADD (not fused), with k = 1 - s_h and h = rgb * s_h computed once in float32;
 *        - everything else is bit for bit the frame without masks, including masks in use but empty, and s_h = 0.
 *      Depth compositing, motion vectors and splat IDs follow from the records: IDs never report a hidden splat, and gsr_pick sees none.
 *      Masks in use are a single-context feature (see "Single-context features"); gsr_clear_splat_masks is never refused.
 *      Operations: each is enqueued on the stream the frames' projections run on (the render stream; with gsr_debug_pipeline(ctx, 1)
 *      the front stream, so an operation does not wait for the previous frame's compositor, except gsr_select_ids, which reads an ID
 *      plane a compositor wrote), does not synchronise the host, and is ordered after every frame enqueued before it and before every
 *      frame enqueued after it.  `op` combines the operation's `inside` set with the selection:
 *        GSR_SELECT_SET       selected = inside (splats outside the tested range count as outside)
 *        GSR_SELECT_ADD       selected | inside
 *        GSR_SELECT_SUBTRACT  selected & ~inside
 *        GSR_SELECT_TOGGLE    selected ^ inside
 *      gsr_select_all: inside = every splat (SET: select all; SUBTRACT: select none; TOGGLE: invert).
 *      gsr_select_polygon: a screen lasso or rectangle of 3 <= n <= GSR_MAX_SELECT_VERTICES vertices xy (x0, y0, x1, y1, ...) in the
 *        frame's pixel axes (column, row; y grows downwards) at the current gsr_resize size.  Tested position q: instance = -1 tests every
 *        splat with q = sp = position * model_scale; instance = k tests only instance k's source range with
 *        q[r] = ((A[r] sp0 + A[3+r] sp1) + A[6+r] sp2) + A[9+r], A = instance k's current to_frame.  (px, py) = pix(view_proj, q), the
 *        rule of gsr_set_motion_vectors.  Inside requires clip3 > 0 and the even-odd test in float32 (one rounding per operation, no
 *        contraction): for every edge a -> b (the last vertex connects to the first) with (a.y > py) != (b.y > py),
 *        x = (((b.x - a.x) (py - a.y)) / (b.y - a.y)) + a.x, and px < x toggles inside.  A NaN position is outside.
 *      gsr_select_volume: the cutout shape test of gsr_set_cutouts on the same tested range, on sp (GSR_CUTOUT_SOURCE) or q
 *        (GSR_CUTOUT_FRAME); `action` is ignored.
 *      gsr_select_ids: "select what you see".  Every pixel of [x0, x1) x [y0, y1) of a device ID plane in the layout of gsr_set_splat_ids
 *        whose v != GSR_NO_ID marks the source splat of v under the current instance layout; a v past the layout's drawn ids is ignored.
 *        An ID plane written before a gsr_delete_hidden or gsr_duplicate_selection names the splats by their indices before it.
 *      gsr_select_polygon and gsr_select_ids return GSR_ERR_STATE before gsr_resize.
 *      gsr_hide_selection: hidden |= selected, then selected = 0.  gsr_unhide_all: hidden = 0.
 *      gsr_clear_splat_masks: both masks 0 and no longer in use: frames take exactly the kernels they took before.
 *      gsr_get_splat_masks / gsr_splat_mask_counts synchronise and return the masks (zeros while not in use) / their population counts.
 *      gsr_set_splat_masks (undo, restore) has read the host arrays when it returns: a copy from pageable memory, it may wait for the
 *      work already enqueued on that stream.
 *      gsr_set_selection_style: rgb finite in [0, GSR_TINT_MAX], strength in [0, 1]; default {1, 0.5, 0} at 0.5; read when a frame is
 *        enqueued.
 *      GSR_ERR_INVALID, previous state kept: an unknown op, an instance outside the current layout, n out of range, a non-finite vertex
 *      or to_local, an unknown shape or space, a rectangle outside the image, a NULL array, words != ceil(max_splats / 32), bits past
 *      max_splats, hidden and selected bits that overlap (gsr_set_splat_masks).  Export of the kept cloud: the stored splats whose hidden
 *      bit is 0, read from the device with gsr_copy_splat_store (after gsr_transform_selection or gsr_recolor_selection the host's
 *      source table is stale; see "Splat transform edits" and "Splat colour edits"). ---- */
#define GSR_MAX_SELECT_VERTICES 64
#define GSR_SELECT_SET 0
#define GSR_SELECT_ADD 1
#define GSR_SELECT_SUBTRACT 2
#define GSR_SELECT_TOGGLE 3
GSR_API int gsr_select_all(gsr_ctx *ctx, int32_t op);
GSR_API int gsr_select_polygon(gsr_ctx *ctx, const float view_proj[32], float model_scale, int32_t instance, const float *xy, uint32_t n,
                               int32_t op);
GSR_API int gsr_select_volume(gsr_ctx *ctx, const gsr_cutout *volume, float model_scale, int32_t instance, int32_t op);
GSR_API int gsr_select_ids(gsr_ctx *ctx, const uint32_t *ids_device, int32_t x0, int32_t y0, int32_t x1, int32_t y1, int32_t op);
GSR_API int gsr_hide_selection(gsr_ctx *ctx);
GSR_API int gsr_unhide_all(gsr_ctx *ctx);
GSR_API int gsr_clear_splat_masks(gsr_ctx *ctx);
GSR_API int gsr_get_splat_masks(gsr_ctx *ctx, uint32_t *hidden, uint32_t *selected, uint64_t words);
GSR_API int gsr_set_splat_masks(gsr_ctx *ctx, const uint32_t *hidden, const uint32_t *selected, uint64_t words);
GSR_API int gsr_splat_mask_counts(gsr_ctx *ctx, uint64_t *selected, uint64_t *hidden);
GSR_API int gsr_set_selection_style(gsr_ctx *ctx, const float rgb[3], float strength);

/* ---- Splat transform edits: move, rotate, scale or mirror the selected splats in the store (no reference counterpart).
 *      gsr_transform_selection rewrites, for every source splat whose `selected` bit is set when the operation runs, its stored planes
 *      from `src_store`: NULL = the store itself, or a caller-owned device snapshot in the layout of gsr_copy_splat_store (a gizmo drag
 *      re-applies a growing transform to the snapshot taken at mouse-down, so no rounding accumulates).  Unselected (and so hidden)
 *      splats are never written, also with a snapshot.  to_source = [L | t], column-major 3x4, acts on the stored position (plane 0
 *      xyz, before model_scale).  Per selected splat, in float32 with one rounding per operation and no contraction:
 *        - position: x'[r] = ((L[r] x + L[3+r] y) + L[6+r] z) + L[9+r] (the instance formula: at model_scale 1 a whole-cloud edit
 *          gives exactly the positions an instance with to_frame = [L | t] writes into its records);
 *        - covariance: with S the symmetric matrix of the six stored words, G[r][c] = ((L[r] S[0][c] + L[3+r] S[1][c]) + L[6+r] S[2][c])
 *          and S'[r][c] = ((G[r][0] L[c] + G[r][1] L[3+c]) + G[r][2] L[6+c]) for the six stored entries (r <= c);
 *        - SH bands 1 .. B-1 of the store: Q = the orthogonal polar factor of L (U V^T of its SVD), in float64 on the host: the
 *          rotation of a rigid or similarity L (improper for a reflection), and for other L the same approximation gsr_set_instances
 *          makes for non-uniform scales.  P_l(d) = the 2l+1 polynomials that multiply coefficients l^2 .. l^2 + 2l in the projection's
 *          SH evaluation, M_l the float64 matrix with P_l(Q^T d) = M_l P_l(d) for every d, and M~_l = M_l with entries below 1e-9 in
 *          magnitude set to +0, rounded to float32 (the identity gives exactly I).  Per channel c'_j = (..((c_0 M~[0][j] + c_1 M~[1][j])
 *          + c_2 M~[2][j]) ..), left to right over i.  With GSR_FLAG_SH_HALF c is the stored half widened (exact) and c' is stored as
 *          h(c') (round to nearest even, +-65504 saturation, as at upload);
 *        - copied bit for bit: plane-0 w (creation time), opacity, the plane-2 pad and the DC coefficients; the floats or half slots
 *          past 3K stay +0.
 *      A frame after an edit is the default frame of the edited cloud; an edit is not motion (like an upload): with a static camera and
 *      unchanged instance transforms the frame after it has motion (0, 0).  GSR_ERR_INVALID, store unchanged: a NULL to_source, a
 *      non-finite entry, det(L) (float64) 0 or not finite.  GSR_ERR_STATE while the splat masks are not in use (so never on a sharded
 *      context).
 *      gsr_splat_store_bytes: the byte size of GSR_BUF_SPLATS, (3 + P) planes x plane_stride x 16.  gsr_copy_splat_store copies the
 *      whole store to dst in that layout, gsr_restore_splat_store writes it back from src; both use cudaMemcpyDefault, so dst / src may
 *      be device or page-locked host memory (pageable memory makes the copy synchronous), and both are allowed on any context.
 *      Ordering of all three: after everything enqueued before on the context's streams (the render stream, and the front stream under
 *      gsr_debug_pipeline(ctx, 1), including the previous frame's compositor), before the projection of every frame enqueued after
 *      it; none synchronises the host.  Undo of an edit is exact: restore the snapshot taken before it, and the masks with
 *      gsr_set_splat_masks. ---- */
GSR_API int gsr_transform_selection(gsr_ctx *ctx, const float to_source[12], const void *src_store);
GSR_API uint64_t gsr_splat_store_bytes(gsr_ctx *ctx);
GSR_API int gsr_copy_splat_store(gsr_ctx *ctx, void *dst);
GSR_API int gsr_restore_splat_store(gsr_ctx *ctx, const void *src);

/* ---- Splat colour edits: recolour, fade or flatten the selected splats in the store (no reference counterpart).
 *      gsr_recolor_selection rewrites, for every source splat whose `selected` bit is set when the operation runs, its SH coefficients
 *      and opacity from `src_store`: NULL = the store itself, or a caller-owned device snapshot in the layout of gsr_copy_splat_store
 *      (a colour-slider drag re-applies a growing edit to the snapshot taken at mouse-down, so no rounding accumulates).  Unselected
 *      (and so hidden) splats are never written, also with a snapshot.  The edit covers all B stored bands, whatever gsr_set_sh_degree
 *      renders.
 *      Meaning: for every view direction, the selected splat's colour before the projection's clamp at 0 (0.5 + C0 c_0 + the
 *      view-dependent terms) becomes A colour + b, up to float32 rounding, with the view-dependent share of band l scaled by
 *      band_scale[l-1].  A channel that was clamped at 0 before the edit is edited from its unclamped value.
 *      Constants, each computed in float64 from the float fields and rounded to float32 once: A[i][j] = matrix[3j + i];
 *      d_i = ((((A[i][0] 0.5 + A[i][1] 0.5) + A[i][2] 0.5) + b_i) - 0.5) / C0 with C0 the projection's float SH_C0;
 *      N~_l[i][j] = band_scale[l-1] A[i][j] (l = 1, 2, 3); s = opacity_scale, t = opacity_offset.
 *      Per selected splat, in float32 with one rounding per operation and no contraction, for each stored coefficient k < K = B^2 with
 *      c = (c_r, c_g, c_b) = values 3k .. 3k+2 (with GSR_FLAG_SH_HALF the stored halves widened, exact):
 *        - k = 0: c'_i = (((A[i][0] c_r + A[i][1] c_g) + A[i][2] c_b) + d_i);
 *        - k in band l >= 1: c'_i = ((N~_l[i][0] c_r + N~_l[i][1] c_g) + N~_l[i][2] c_b);
 *        - with GSR_FLAG_SH_HALF c' is stored as h(c') (round to nearest even, +-65504 saturation, NaN stays NaN, as at upload);
 *        - opacity (plane-2 z): u = (o s) + t, o' = u > 1 ? 1 : (u > 0 ? u : +0), so NaN, +-0 and negative values give +0;
 *        - copied bit for bit: planes 0 and 1 (position, creation time, covariance), plane-2 x, y and w; the floats or half slots past
 *          3K stay +0.
 *      The identity edit ({I | 0}, {1, 1, 1}, 1, 0) leaves every stored word of finite coefficients unchanged, except that a -0
 *      coefficient may become +0, so its frame is bit for bit the unedited frame (an infinite coefficient turns the other channels of
 *      its triple NaN: 0 * inf).  A frame after an edit is the default frame of the edited cloud; an edit is not
 *      motion.  Ordering as gsr_transform_selection: on the projections' stream after an event on the render stream, after everything
 *      enqueued before and before the projection of every frame enqueued after it; it never synchronises the host.  Undo of an edit is
 *      exact: restore the snapshot taken before it, then the masks with gsr_set_splat_masks.
 *      GSR_ERR_INVALID, store unchanged: a NULL edit, a non-finite field, |A[i][j]| or |b_i| > GSR_TINT_MAX, a band_scale or
 *      opacity_scale outside [0, GSR_TINT_MAX], opacity_offset outside [-1, 1].  The arguments are checked first; then GSR_ERR_STATE
 *      while the splat masks are not in use (so never on a sharded context). ---- */
typedef struct gsr_color_edit {
    float matrix[12];       /* [A | b], column-major 3x4 like gsr_instance.to_frame: colour' = A colour + b, on the colour the
                               projection evaluates before its clamp at 0 */
    float band_scale[3];    /* further multiplies A for SH bands 1, 2, 3 (the view-dependent colour): 1 keeps it, 0 removes it */
    float opacity_scale, opacity_offset;   /* stored opacity o' = clamp(o * scale + offset, 0, 1), rule above */
} gsr_color_edit;           /* 68 bytes; identity = {I | 0}, {1, 1, 1}, 1, 0 */
GSR_API int gsr_recolor_selection(gsr_ctx *ctx, const gsr_color_edit *edit, const void *src_store);

/* ---- Splat delete and duplicate: change how many splats the cloud has (no reference counterpart).
 *      The cloud is the splats of [0, n), n = gsr_stats.num_splats.  A slot that stops holding a splat is left vacant: plane-0 x, y and
 *      z the quiet NaN 0x7FC00000, every other float word of every plane +0 (with GSR_FLAG_SH_HALF every half slot +0), its hidden and
 *      selected bits 0.  Every projection variant culls a vacant slot like a frustum-culled splat (no record, no pairs, no share of M, V
 *      or the last tile) by its rule that a splat whose projected centre or radius is not finite is culled; a NaN position is also
 *      outside every polygon and volume selection.
 *      gsr_delete_hidden: the kept splats are those of [0, n) whose hidden bit is 0.  They move to [0, k) in their order, every word of
 *      every plane bit for bit, each with its selected bit; then [k, n) is vacant, every hidden bit is cleared, every selected bit at or
 *      above k is cleared, n = k and *kept_out = k.  Slots at or above the old n are not touched.  The new index of the splat at s is
 *      the number of kept splats below s, so the host can remap from masks read before the call (no device index map is returned).
 *      A frame after a delete is bit for bit the frame before it with the deleted splats hidden (RGBA, depth, motion, M, V, last tile,
 *      keys, tile ranges and the selection highlight): only sort values, record indices and IDs change, by the rank rule above.
 *      GSR_ERR_INVALID: a NULL kept_out.  GSR_ERR_STATE while the splat masks are not in use, or while instances are set (their ranges
 *      would silently point at other splats).  Nothing changes on an error.
 *      gsr_duplicate_selection: the S selected splats of [0, n) are copied in order, bit for bit, to [n, n + S); then n = n + S and
 *      *copies_out = S.  The selection is then exactly the copies (the originals are deselected and selected bits at or above the old n
 *      dropped); hidden bits are unchanged except that the copies are not hidden.  Paste-and-move is gsr_duplicate_selection followed by
 *      gsr_transform_selection.  With instances set the copies lie outside every instance range (so are not drawn) until the host
 *      changes the ranges.  GSR_ERR_INVALID, nothing written and the state kept: a NULL copies_out, or n + S > max_splats (the message
 *      gives S and the room left).  The arguments are checked first; then GSR_ERR_STATE while the splat masks are not in use.
 *      gsr_set_splat_count: sets n and writes nothing else, for undo.  GSR_ERR_INVALID: n > max_splats.  Undo of a delete or duplicate
 *      is exact: gsr_restore_splat_store of the snapshot taken before it, then gsr_set_splat_masks, then gsr_set_splat_count.
 *      Ordering as gsr_transform_selection: on the projections' stream after an event on the render stream, after every frame enqueued
 *      before it and before every frame enqueued after it.  Unlike the other edits each synchronises the host once (a delete must learn
 *      k, a duplicate must know S before it writes anything): they are click-time operations, not per-frame ones.  Neither is motion
 *      (like an upload).  Masks in use are single-context, so neither applies to a sharded context. ---- */
GSR_API int gsr_delete_hidden(gsr_ctx *ctx, uint64_t *kept_out);
GSR_API int gsr_duplicate_selection(gsr_ctx *ctx, uint64_t *copies_out);
GSR_API int gsr_set_splat_count(gsr_ctx *ctx, uint64_t n);

/* ---- Splat property selection: select splats by what they are -- opacity, size, shape, colour -- and histogram those properties
 *      (no reference counterpart).  The cleanup of a capture: floaters and haze are nearly transparent, "spikes" are needle-shaped,
 *      a trainer's sky or fog is huge, a colour cast is a colour.  A UI places a threshold on a histogram and selects by it.
 *      Properties: a float32 value per stored splat from its stored words (source units, before model_scale and any instance
 *      transform), in float32 with one rounding per operation, no contraction, in the order written.  S00 S01 S02 S11 = plane 1 x y z w,
 *      S12 S22 = plane 2 x y, o = plane-2 z, f_r f_g f_b = SH values 0..2 (plane 3 x y z; with GSR_FLAG_SH_HALF half slots 0..2 of
 *      plane 3 widened, which is exact):
 *        GSR_PROP_OPACITY         o
 *        GSR_PROP_SIZE            t = (S00 + S11) + S22, the sum of the squared principal scales
 *        GSR_PROP_VOLUME          det = ((S00 ((S11 S22) - (S12 S12))) - (S01 ((S01 S22) - (S12 S02)))) + (S02 ((S01 S12) - (S11 S02))),
 *                                 the product of the squared scales
 *        GSR_PROP_ISOTROPY        (27 det) / ((t t) t): 1 for a sphere, towards 0 for needles and discs
 *        GSR_PROP_COLOR_DISTANCE  c_i = 0.5 + (f_i SH_C0) (the projection's DC colour before its clamp, view-dependent terms excluded),
 *                                 d_i = c_i - rgb_i, value ((d_r d_r) + (d_g d_g)) + (d_b d_b)
 *      No eigen-decomposition and no transcendental function: the values are exact functions of the stored words.  A value can be
 *      negative (det under cancellation), infinite or NaN; it is still the value.  A NaN value is outside every range.
 *      Tested range: instance = -1 the splats of [0, n), n = gsr_stats.num_splats; instance = k instance k's source range intersected
 *      with [0, n).  A tested splat counts only if none of its plane-0 x, y, z is NaN (so a vacant slot never counts).
 *      gsr_select_where: inside = the tested splat passes ALL n filters, 1 <= n <= GSR_MAX_SPLAT_FILTERS; filter f passes iff
 *        f.lo <= v && v <= f.hi (IEEE: lo > hi is empty, +-inf bounds are allowed).  `op` combines inside with the selection as every
 *        gsr_select_* (GSR_SELECT_SET clears the splats outside the tested range), then selected &= ~hidden.  The call puts the masks
 *        in use (so it is refused with GSR_ERR_STATE on a sharded context), is enqueued like the other selections and never
 *        synchronises the host.  GSR_ERR_INVALID, state kept: a NULL array, n out of range, an unknown property, a NaN lo or hi, a
 *        non-finite rgb of a GSR_PROP_COLOR_DISTANCE filter (rgb is ignored otherwise), an unknown op, an instance outside the layout.
 *      gsr_splat_histogram: counts the property `property->property` (with `property->rgb`; lo and hi are ignored) over the tested
 *        splats that are not hidden and, with GSR_HISTOGRAM_SELECTED, selected.  edges = bins + 1 finite, strictly increasing floats,
 *        1 <= bins <= GSR_MAX_HISTOGRAM_BINS (linear, log-spaced or quantile edges: the rule is comparisons only).  counts has bins + 3
 *        entries: counts[i] = #(e_i <= v < e_{i+1}), the last bin also takes v == e_bins (numpy's convention); counts[bins] = #(v < e_0),
 *        counts[bins + 1] = #(v > e_bins), counts[bins + 2] = #NaN.  minmax (may be NULL) receives the least and the greatest non-NaN
 *        v of the counted splats in the order of gsr_set_depth_order's ord (-0 before +0), or (+inf, -inf) when there is none.  While
 *        the masks are not in use nothing is hidden and nothing is selected.  The call reads only: it does not put the masks in use and
 *        is allowed on any context, sharded ones included.  It is enqueued like the store edits (on the projections' stream after an
 *        event on the render stream, so after every upload, selection and edit enqueued before it) and synchronises the host once.
 *        GSR_ERR_INVALID, nothing written: a NULL property, edges or counts, bins out of range, non-finite or non-increasing edges, an
 *        unknown property, scope or instance, a non-finite rgb of a GSR_PROP_COLOR_DISTANCE property. ---- */
#define GSR_PROP_OPACITY 0
#define GSR_PROP_SIZE 1
#define GSR_PROP_VOLUME 2
#define GSR_PROP_ISOTROPY 3
#define GSR_PROP_COLOR_DISTANCE 4
/* read from the contribution buffer, not from the stored words: see "Splat contribution" below (5 .. 15 stay unknown) */
#define GSR_PROP_CONTRIBUTION 16
#define GSR_PROP_PEAK_CONTRIBUTION 17
#define GSR_PROP_VIEWS 18
#define GSR_PROP_CONTRIBUTING_PIXELS 19
#define GSR_MAX_SPLAT_FILTERS 8
typedef struct gsr_splat_filter {
    int32_t property;   /* GSR_PROP_* */
    float lo, hi;       /* passes iff lo <= v && v <= hi (a NaN v never passes); +-inf allowed, NaN not */
    float rgb[3];       /* GSR_PROP_COLOR_DISTANCE: the reference colour; ignored otherwise */
} gsr_splat_filter;     /* 24 bytes */
GSR_API int gsr_select_where(gsr_ctx *ctx, const gsr_splat_filter *filters, uint32_t n, int32_t instance, int32_t op);
#define GSR_MAX_HISTOGRAM_BINS 1024
#define GSR_HISTOGRAM_KEPT 0       /* every tested splat that is not hidden */
#define GSR_HISTOGRAM_SELECTED 1   /* only the selected ones */
GSR_API int gsr_splat_histogram(gsr_ctx *ctx, const gsr_splat_filter *property, int32_t instance, int32_t scope, const float *edges,
                                uint32_t bins, uint64_t *counts, float minmax[2]);

/* ---- Splat contribution: how much every stored splat shows up in the rendered views, accumulated on the GPU over any number of
 *      depth-composited frames, so a host can select and prune the splats that contribute least (no reference counterpart).
 *      accum_device: caller-owned device array of `slots` records, one per source slot [0, max_splats); `slots` must equal max_splats
 *      (GSR_ERR_INVALID otherwise).  NULL switches the mode off.  The call does not zero the buffer: the host zeroes it, or calls
 *      gsr_reset_splat_contribution.  The mode rules are those of gsr_set_splat_ids: GSR_ERR_STATE while depth compositing is off (a
 *      NULL scene depth is enough); gsr_set_depth_compositing(ctx, NULL, NULL) and gsr_resize switch it off; its single-context rules
 *      are those of depth compositing; the pointer is read when a frame is enqueued; gsr_pick does not accumulate.
 *      GSR_ERR_INVALID, previous state kept: a buffer that aliases depth_out, scene_depth, motion_out or the ID plane.  GSR_ERR_STATE,
 *      previous state kept: motion vectors or splat IDs are on (gsr_set_motion_vectors and gsr_set_splat_ids likewise refuse while the
 * mode is on).  The call never synchronises; the first one allocates a 4-byte frame counter.
 *      Rule: a frame enqueued with the mode on adds, for every pixel inside the image and every splat that the pixel's depth-composited
 *      blend blends (the splats of the ID rule of gsr_set_splat_ids: same scene-depth stop, dead-pixel rule t > 1/255, sorted order and
 *      tile-stop vote), with w = t - t' exactly the float32 w of the ID rule (the context's contraction mode), to the record of the
 *      splat's SOURCE slot (the drawn id v without instances, first_k + (v - 32 w_k) with them) if w > 0:
 *        weight += q(w) = __float2uint_rn(w * 2^24);  pixels += 1;  peak = max(peak, w);
 *        views += 1 once per frame and slot, however many tiles, pixels and instances touch it.
 *      Integer sums, a max and a once-per-frame count: every field is order-independent and bit-exact.  weight cannot overflow before
 *      2^40 full-weight pixel hits.  Hidden splats, hidden instances and splats past an instance's draw_count are never blended.
 *      A frame whose pairs overflowed the duplicate capacity adds nothing: gsr_render's re-render of an overflowed frame adds that frame
 *      exactly once, and an asynchronous overflowed frame, or an overflowed frame under GSR_FLAG_STATIC_CAPACITY, adds nothing.  rgba
 *      and depth_out are bit-identical to the same frame without the mode.
 *      gsr_reset_splat_contribution: enqueues a zeroing of the buffer and of the frame counter, ordered after every frame enqueued before
 *      it and before every later one; it never synchronises.  GSR_ERR_STATE if no buffer is set.
 *      gsr_splat_contribution_frames: synchronises the context and returns the frames added since the last set or reset (the overflowed
 *      ones are not).  GSR_ERR_STATE if no buffer is set.
 *      Store edits do not touch the buffer, which is indexed by slot: after gsr_delete_hidden or gsr_duplicate_selection its
 *      statistics are stale until a reset (the rank rule of gsr_delete_hidden lets a host remap them).
 *      Properties for gsr_select_where and gsr_splat_histogram, read from the buffer, combinable with the others in one filter set:
 *        GSR_PROP_CONTRIBUTION         (float)weight * 2^-24 (a round to nearest, then an exact scale)
 *        GSR_PROP_PEAK_CONTRIBUTION    peak
 *        GSR_PROP_VIEWS                (float)views
 *        GSR_PROP_CONTRIBUTING_PIXELS  (float)pixels
 *      They refuse with GSR_ERR_STATE while no buffer is set, and are ordered after the compositor of every frame enqueued before the
 *      call. ---- */
typedef struct gsr_splat_contribution {
    uint64_t weight;      /* sum of q(w) over every blended (pixel, frame, drawn copy) with w > 0 */
    uint64_t pixels;      /* number of those (pixel, frame, drawn copy) triples */
    float peak;           /* the largest w, +0 if none */
    uint32_t views;       /* accumulated frames in which the splat had some w > 0 */
    uint32_t last_frame;  /* library-owned (the views rule); hosts do not interpret it */
    uint32_t pad;
} gsr_splat_contribution; /* 32 bytes */
GSR_API int gsr_set_splat_contribution(gsr_ctx *ctx, gsr_splat_contribution *accum_device, uint64_t slots);
GSR_API int gsr_reset_splat_contribution(gsr_ctx *ctx);
GSR_API int gsr_splat_contribution_frames(gsr_ctx *ctx, uint32_t *frames);

/* ---- Splat neighbourhood selection: select splats by the splats around them -- isolated floaters, one step of "select more", the
 *      object under a clicked splat, every small clump (no reference counterpart).  Queries run on a spatial grid on the GPU.
 *      Participants: the splats of the tested range (the rule of gsr_select_where: instance = -1 [0, n), instance = k instance k's
 *        source range intersected with [0, n)) whose hidden bit is 0 and whose plane-0 x, y and z are all finite.  Vacant slots, NaN
 *        and infinite positions and hidden splats never participate and are never inside.
 *      Neighbours: for participants i != j, dx = x_j - x_i (dy, dz the same way) and d2 = ((dx dx) + (dy dy)) + (dz dz), all float32,
 *        one rounding per operation, no contraction; j is a neighbour of i iff d2 <= r2, r2 = radius radius in float32.  The relation is
 *        symmetric (fl(a - b) = -fl(b - a)); coincident splats (a duplicate and its copy) are neighbours.  A cluster is a connected
 *        component of the graph of participants with these edges (single linkage at `radius`).  radius is in source units (the stored
 *        position, before model_scale and any instance transform).
 *      Modes (`selected` = the selection when the call runs, restricted to participants):
 *        GSR_NEIGHBOR_SPARSE          inside = participants with fewer than `count` neighbours (count >= 1; 1 = no neighbour at all)
 *        GSR_NEIGHBOR_GROW            inside = participants that are selected or have a selected neighbour (one step, not a fixed point)
 *        GSR_NEIGHBOR_CONNECTED       inside = the participants of every cluster that holds a selected participant
 *        GSR_NEIGHBOR_SMALL_CLUSTERS  inside = the participants of clusters of fewer than `count` participants ("keep the main object":
 *                                     count = largest_cluster of an earlier call)
 *      `op` combines inside with the selection as every gsr_select_* (GSR_SELECT_SET clears everything outside the tested range), then
 *      selected &= ~hidden.  The call puts the masks in use (so it is refused with GSR_ERR_STATE on a sharded context).
 *      Grid and work measure (part of the contract, so that a refusal is deterministic): h = (double)radius (1 + 2^-20); a splat's cell
 *        is floor(x / h), floor(y / h), floor(z / h) in float64, each clamped to [-2^62, 2^62]; candidates = the sum over participants
 *        of the number of participants in the 27 cells around its own cell.  candidates > GSR_MAX_NEIGHBOR_CANDIDATES returns
 *        GSR_ERR_INVALID with the masks unchanged (the message gives the count): a radius far too large for the cloud is a refused call,
 *        not a kernel that runs for minutes.
 *      Ordering: enqueued like gsr_splat_histogram (after every upload, edit and selection enqueued before it, before every frame
 *        enqueued after it); it synchronises the host at most twice (the budget check and the stats): a click-time call.
 *      Memory: scratch of GSR_NEIGHBOR_SCRATCH_BYTES_PER_SLOT bytes per slot of max_splats, plus 4 B per hash bucket (the least power
 *        of two >= 2 max_splats: 8 to 16 B per slot) and the sort's look-back words, allocated by the first call and kept until
 *        gsr_destroy; separate from the frame's buffers.  GSR_ERR_OOM keeps the state.
 *      stats (may be NULL): participants, inside (participants inside), candidates; clusters and largest_cluster for CONNECTED and
 *        SMALL_CLUSTERS, 0 otherwise.  Written only when the call succeeds.
 *      GSR_ERR_INVALID, state kept, checked in this order: a NULL q; an unknown mode; a radius that is not finite or outside
 *        [GSR_NEIGHBOR_MIN_RADIUS, GSR_NEIGHBOR_MAX_RADIUS] (so that r2 is a normal float: the grid's argument needs it); count = 0 for
 *        SPARSE and SMALL_CLUSTERS; an unknown op; an instance outside the layout. ---- */
#define GSR_NEIGHBOR_SPARSE 0           /* inside: fewer than `count` other participants within `radius` */
#define GSR_NEIGHBOR_GROW 1             /* inside: selected, or a selected participant within `radius` */
#define GSR_NEIGHBOR_CONNECTED 2        /* inside: in a cluster that holds a selected participant */
#define GSR_NEIGHBOR_SMALL_CLUSTERS 3   /* inside: in a cluster of fewer than `count` participants */
#define GSR_MAX_NEIGHBOR_CANDIDATES (1ull << 34)
#define GSR_NEIGHBOR_MIN_RADIUS 0x1p-60f
#define GSR_NEIGHBOR_MAX_RADIUS 0x1p+60f
#define GSR_NEIGHBOR_SCRATCH_BYTES_PER_SLOT 32
typedef struct gsr_neighborhood {
    int32_t mode;       /* GSR_NEIGHBOR_* */
    float radius;       /* source units; finite, in [GSR_NEIGHBOR_MIN_RADIUS, GSR_NEIGHBOR_MAX_RADIUS] */
    uint32_t count;     /* SPARSE, SMALL_CLUSTERS: the threshold (>= 1); ignored otherwise */
    int32_t instance;   /* -1: [0, n); k: instance k's source range intersected with [0, n) */
} gsr_neighborhood;     /* 16 bytes */
typedef struct gsr_neighborhood_stats {
    uint64_t participants, inside, candidates;   /* candidates: the work measure above */
    uint64_t clusters, largest_cluster;           /* CONNECTED / SMALL_CLUSTERS; 0 otherwise */
} gsr_neighborhood_stats;                         /* 40 bytes */
GSR_API int gsr_select_neighborhood(gsr_ctx *ctx, const gsr_neighborhood *q, int32_t op, gsr_neighborhood_stats *stats /* may be NULL */);

/* ---- Splat export: the edited cloud written back out as the vertex rows of a standard 3DGS PLY, on the GPU (the inverse of
 *      gsr_upload_ply's ingest; no reference counterpart).  "Save" of an editor: the cleaned capture, or one object picked out of it.
 *      Exported splats: every s of [0, n), n = gsr_stats.num_splats, none of whose plane-0 x, y, z is NaN (a vacant slot is never
 *        exported: the rule of gsr_select_where) and that is in scope: GSR_EXPORT_KEPT its hidden bit is 0, GSR_EXPORT_SELECTED its
 *        selected bit is 1.  While the masks are not in use KEPT is every splat and SELECTED none.  One row per exported splat, in
 *        ascending store index.
 *      Row: the vertex of a binary little-endian 3DGS PLY of SH degree d, in the trainer's property order
 *        x y z nx ny nz f_dc_0..2 f_rest_0..(3((d+1)^2 - 1) - 1) opacity scale_0..2 rot_0..3: 17 + 3((d+1)^2 - 1) float32 values (17, 26,
 *        41 or 62 for d = 0..3).  sh_degree = -1 exports the stored degree (sh_bands - 1); 0 .. the stored degree drops the bands above d.
 *        The file a host writes is the header
 *          ply / format binary_little_endian 1.0 / element vertex <rows> / property float <name>, one per column in the order above /
 *          end_header
 *        (one line each, '\n'-terminated), then the rows as they are.
 *      Fields, per exported splat (source units: the stored position, before model_scale):
 *        x y z      plane-0 x, y, z, bit for bit;  nx ny nz  +0
 *        f_dc, f_rest  the stored coefficients bit for bit (a GSR_FLAG_SH_HALF half widened, which is exact); f_rest is channel-major as
 *                   the trainer writes it: with K = (d+1)^2, column c (K - 1) + (k - 1) holds stored value 3k + c
 *        opacity    the logit of o = plane-2 z in float64, log(o) - log1p(-o), clamped to [-104, 104], NaN replaced by +0, rounded to
 *                   float32 once (within 1 float32 ulp of that value): o = 0 gives -104, o = 1 gives 104, o < 0, o > 1 or NaN give 0
 *        scale, rot from S, the symmetric float64 matrix of the six covariance words: when any word is not finite the scales are the quiet
 *                   NaN and rot = (1, 0, 0, 0).  Else float64 eigenvalues l0 <= l1 <= l2 and orthonormal eigenvectors V (cyclic Jacobi,
 *                   |S - V diag(l) V^T|max <= 1e-12 max|S|), column 0 of V negated when det V < 0; scale_i = 0.5 log(max(l_i, DBL_MIN));
 *                   rot = (w, x, y, z), the unit quaternion of V (Shepperd's method), normalised in float64, negated when w < 0.  Each
 *                   value is rounded to float32 once.
 *        A row depends only on the splat's stored words and on d: the same splat at another index, in another scope or call gives the
 *        same bits.
 *      dst: device memory, page-locked or pageable host memory of dst_rows rows.  Host memory is written through a temporary device
 *        buffer of rows x row bytes, freed before the call returns; when it cannot be allocated the call returns GSR_ERR_OOM and writes
 *        nothing (retry into device memory).  dst = NULL counts only.  *rows_out = the number of exported splats, also when dst_rows is
 *        below it: then the call returns GSR_ERR_INVALID, writes nothing and names the count in gsr_last_error().
 *      Ordering: enqueued like gsr_splat_histogram (after every upload, selection and edit enqueued before it, before every frame
 *        enqueued after it); it synchronises the host (it returns the count): a save-time call.  It only reads: it does not put the
 *        masks in use and is allowed on any context, sharded ones included.  Look-back words for ceil(max_splats / 256) tiles are
 *        allocated by the first call and kept until gsr_destroy.
 *      GSR_ERR_INVALID, nothing written: a NULL ctx or rows_out, an unknown scope, sh_degree < -1 or above the stored degree, the
 *        capacity refusal above. ---- */
#define GSR_EXPORT_KEPT 0       /* the splats whose hidden bit is 0 */
#define GSR_EXPORT_SELECTED 1   /* the splats whose selected bit is 1 */
GSR_API int gsr_export_ply(gsr_ctx *ctx, int32_t scope, int32_t sh_degree, void *dst, uint64_t dst_rows, uint64_t *rows_out);

/* ---- Compressed PLY: the SuperSplat / PlayCanvas `compressed.ply` layout, written and read on the GPU.  About 61 B per degree-3 splat
 *      (16 B at degree 0) instead of the 248 B of a float 3DGS PLY.  The library fills or reads the three element bodies; the host writes
 *      or parses the header:
 *        ply / format binary_little_endian 1.0 /
 *        element chunk <ceil(rows / 256)> / property float <name>, one line each for min_x min_y min_z max_x max_y max_z min_scale_x
 *          min_scale_y min_scale_z max_scale_x max_scale_y max_scale_z min_r min_g min_b max_r max_g max_b /
 *        element vertex <rows> / property uint packed_position / property uint packed_rotation / property uint packed_scale /
 *          property uint packed_color /
 *        element sh <rows> / property uchar f_rest_0 .. f_rest_<3((d+1)^2 - 1) - 1>   (only for d > 0) /
 *        end_header
 *      ('\n'-terminated lines; `comment` lines may appear anywhere in the header), then the chunk floats, the packed words and the SH
 *      bytes as they are.  Row r belongs to chunk r / 256; the last chunk may be partial.  Older files have 12-float chunks (no colour
 *      range); they are accepted on upload.  The layout and the quantisation follow the public description of SuperSplat's format; no
 *      file written by another tool has been checked against this library, and other decoders may reconstruct bin edges slightly
 *      differently.  Bit-exactness is a property of this library's own rule below.
 *
 *      Export rule.  Every value in float64 from float32 inputs, one rounding per operation (the library is built with -fmad=false).
 *        Exported splats: those of gsr_export_ply's rule (scope, vacant slots skipped) whose plane-0 x, y, z are also finite (an infinite
 *          position cannot be quantised and is not exported).
 *        Per row: position = plane-0 x, y, z; log-scales s0..s2 and quaternion (w x y z) = the scale and rot gsr_export_ply writes for
 *          the splat, bit for bit; colour c_k = (float)(f_dc_k * 0.28209479177387814 + 0.5); alpha o = plane-2 z (the stored sigmoid);
 *          SH = the stored coefficients 1 .. (d+1)^2 - 1, channel-major as in a degree-d 3DGS PLY.
 *        Sanitised before the chunk statistics: log-scales clamped to [-20, 20], NaN -> -20; colours clamped to [-64, 64], NaN -> 0.5;
 *          alpha clamped to [0, 1], NaN -> 0.
 *        Chunk: the exact float32 minimum and maximum over the chunk's rows of x, y, z, s0..s2 and c0..c2 (18 floats, ordered as in the
 *          header; -0 orders below +0).
 *        norm(x, lo, hi) = 0 if x <= lo, 1 if x >= hi, 0 if hi - lo < 1e-5, else (x - lo) / (hi - lo).
 *        unorm(v, b) = min(t, max(0, floor(v t + 0.5))), t = 2^b - 1.
 *        packed_position, packed_scale = unorm(nx, 11) << 21 | unorm(ny, 10) << 11 | unorm(nz, 11) (n = norm over the chunk's range).
 *        packed_color = unorm(nr, 8) << 24 | unorm(ng, 8) << 16 | unorm(nb, 8) << 8 | unorm(o, 8).
 *        packed_rotation: i = the index of the largest |q_k| (the first on a tie); q negated when q_i < 0; the other three components in
 *          ascending index, each unorm(q_k sqrt(0.5) + 0.5, 10); i << 30 | a << 20 | b << 10 | c.
 *        SH byte = min(255, max(0, trunc((v / 8 + 0.5) 256))), NaN -> 128.
 *        Row order: GSR_COMPRESS_STORE_ORDER ascending store index (the rows and order of gsr_export_ply).  GSR_COMPRESS_MORTON: lo, hi =
 *          the float32 bounds of the exported positions; per axis cell = min(1023, floor((p - lo) / (hi - lo) 1024)), 0 when hi == lo;
 *          key = part1by2(z) << 2 | part1by2(y) << 1 | part1by2(x) (30 bits); ascending key, ties in ascending store index.
 *      Decode rule (upload).  float32, one IEEE operation at a time.  u(v, b) = v / (2^b - 1); lerp(lo, hi, u) = lo + (hi - lo) u.
 *        Position and log-scale: lerp over the chunk's range.  Colour: lerp over the chunk's range (a 12-float chunk: u(v, 8) itself),
 *          f_dc = (c - 0.5f) / 0.28209479177387814f.  Quaternion: a, b, c = (u(field, 10) - 0.5f) 1.41421356f,
 *          m = sqrt(max(0, 1 - ((a a + b b) + c c))) at index i, a, b, c at the other indices in ascending order.  SH: (q + 0.5f) 0.03125f
 *          - 4.0f (the bin's midpoint).
 *        The store then holds what gsr_upload_ply stores for the decoded float rows (x y z f_dc f_rest opacity scale rot), except plane-2
 *          z = u(alpha, 8) itself (no logit and sigmoid).  Coefficients above the file's degree are stored as 0, those above the store's
 *          bands are dropped.
 *
 *      gsr_export_compressed_ply(ctx, scope, sh_degree, order, dst, rows_out): scope GSR_EXPORT_KEPT / _SELECTED, sh_degree -1 (the
 *        stored degree) or 0 .. the stored degree, order GSR_COMPRESS_*.  dst->rows is the capacity in rows: dst->chunks holds
 *        ceil(dst->rows / 256) x 18 floats, dst->packed dst->rows x 4 words, dst->sh dst->rows x 3((d+1)^2 - 1) bytes (unused for d = 0).
 *        The three may be device, page-locked or pageable memory (host memory goes through temporary device staging, freed before the
 *        call returns).  dst = NULL counts only.  *rows_out = the exported count, also when it exceeds dst->rows: then GSR_ERR_INVALID and
 *        nothing is written.  On success dst->rows, dst->chunk_count, dst->sh_degree and dst->chunk_floats (18) describe the file written,
 *        so dst can be passed to gsr_upload_compressed_ply as it is.  Ordered like gsr_export_ply; it only reads the store, does not put
 *        the masks in use and is allowed on sharded contexts.  Scratch of 16 B per slot plus a sort workspace is allocated by the first
 *        call and kept until gsr_destroy (GSR_ERR_OOM, nothing kept, when it cannot be).  GSR_ERR_INVALID: a NULL ctx or rows_out, an
 *        unknown scope or order, a bad sh_degree, a NULL buffer in dst (sh only with d > 0), the capacity refusal, max_splats >= 2^32.
 *      gsr_upload_compressed_ply(ctx, src, first, creation_time): rows [0, src->rows) become splats [first, first + rows).  src's buffers
 *        may be device or host memory.  A chunk-aligned piece of a file (rows from a multiple of 256, its chunks from that chunk on) is a
 *        file itself, so a load may be split into pieces.  Synchronises like gsr_upload_ply.  GSR_ERR_INVALID, nothing written: NULL ctx,
 *        src or buffer (sh == NULL with d > 0), chunk_floats not 12 or 18, sh_degree > 3, chunk_count != ceil(rows / 256),
 *        [first, first + rows) beyond max_splats. ---- */
#define GSR_COMPRESSED_CHUNK 256
#define GSR_COMPRESS_STORE_ORDER 0   /* ascending store index: the rows of gsr_export_ply */
#define GSR_COMPRESS_MORTON 1        /* 30-bit Morton order over the exported bounds (SuperSplat's; the smaller chunk ranges) */
typedef struct gsr_compressed_ply {
    float *chunks;          /* chunk_count x chunk_floats */
    uint32_t *packed;       /* rows x 4: position, rotation, scale, color */
    uint8_t *sh;            /* rows x 3((d+1)^2 - 1); may be NULL iff sh_degree 0 */
    uint64_t rows;
    uint64_t chunk_count;   /* ceil(rows / 256) */
    uint32_t sh_degree;     /* 0..3 */
    uint32_t chunk_floats;  /* 18; 12 accepted on upload */
} gsr_compressed_ply;       /* 48 bytes */
GSR_API int gsr_export_compressed_ply(gsr_ctx *ctx, int32_t scope, int32_t sh_degree, int32_t order, gsr_compressed_ply *dst /* NULL: count */,
                                      uint64_t *rows_out);
GSR_API int gsr_upload_compressed_ply(gsr_ctx *ctx, const gsr_compressed_ply *src, uint64_t first, float creation_time);

/* ---- get_splat_position() (rasterizer.gd:162-171): re-dispatches the compositor for `tile_id` and reads the
 *      16-byte tile_splat_pos buffer (gsplat_render.glsl:33-36,105-110).  out_xyzn = splat_pos.xyz,
 *      num_tile_splats -- persistent across calls exactly like the reference's storage buffer.
 *      GSR_ERR_STATE before the first gsr_render at the current size (no tile ranges exist yet). ---- */
GSR_API int gsr_pick(gsr_ctx *ctx, uint32_t tile_id, float heatmap_factor, float out_xyzn[4]);

/* ---- update_debug_info() (main.gd:93-119): M, overflow, per-stage GPU ms.  Synchronises the stream. ---- */
GSR_API int gsr_get_stats(gsr_ctx *ctx, gsr_stats *out);

/* Per-frame GPU timestamps + counters of the most recent frames, oldest first (capture_timestamp/
 * get_captured_timestamp_gpu_time, rasterizer.gd:135-160, main.gd:106-119).  Synchronises the stream once. */
GSR_API int gsr_get_frame_history(gsr_ctx *ctx, uint32_t max_frames, gsr_frame_record *out, uint32_t *n_out);

/* ---- parity taps: copy an internal buffer to host (synchronises).  bytes = size of dst. ---- */
GSR_API int gsr_debug_copy(gsr_ctx *ctx, int which, void *dst, size_t bytes);
/* Record, for every work item of the compositor, {tile<<32|SM id, start ns, end ns, first_chunk<<32|chunks<<1|finished}
 * (4 x uint64 per item, %globaltimer).  max_items = 0 disables.  Profiling aid; not on the frame path by default. */
GSR_API int gsr_debug_enable_trace(gsr_ctx *ctx, uint32_t max_items);
/* Scheduling of the compositor's persistent grid (results never depend on it): resident CTAs per SM (0 = as many as fit; default 2),
 * longest-chain-first ticket order (default on), and the sparse-frame rule of that order pass: with at most
 * sparse_tiles_per_sm * SMs occupied tiles only one CTA per SM works (default 5; 0 = never). */
GSR_API int gsr_debug_compositor_config(gsr_ctx *ctx, int32_t ctas_per_sm, int32_t longest_first, int32_t sparse_tiles_per_sm);
/* Front / back overlap of consecutive frames (results never depend on it): 1 = a frame's clear + projection run on a second
 * stream, released when the previous frame's tile ranges are done, i.e. beside that frame's compositor; 0 or -1 (default) = every
 * kernel of a frame on the render stream, frames strictly one after the other.  Off by default: on one GPU the projection and
 * the compositor compete for the same issue slots, and beside a rows-local read-back the overlap can slow a shard group down
 * (DESIGN.md section 6). */
GSR_API int gsr_debug_pipeline(gsr_ctx *ctx, int32_t overlap);
/* Keep an unsorted copy of the emitted pairs each frame (costs 8*M bytes of traffic; off by default). */
GSR_API int gsr_debug_keep_unsorted(gsr_ctx *ctx, int enable);

/* ---- stand-alone radix sort (config c5; replaces radix_sort_{upsweep,spine,downsweep}.glsl x 4 passes,
 *      rasterizer.gd:143-149).  Stable LSD sort of 32-bit keys (+ optional 32-bit values), 4 x 8-bit digits. ---- */
GSR_API int gsr_sorter_create(int32_t device, uint64_t max_n, gsr_sorter **out);
GSR_API int gsr_sorter_destroy(gsr_sorter *s);
/* Device-resident sort: keys/values are device pointers (values may be NULL); result in place.
 * cuda_stream: cudaStream_t as void* (NULL = default stream).  No host sync. */
GSR_API int gsr_sorter_sort_device(gsr_sorter *s, void *d_keys, void *d_values, uint64_t n, void *cuda_stream);
/* Host convenience: copies in, sorts on the GPU, copies out (values may be NULL). */
GSR_API int gsr_sort_pairs_host(int32_t device, uint32_t *keys, uint32_t *values, uint64_t n);
/* ms of the last gsr_sorter_sort_device call measured with CUDA events on its stream (synchronises). */
GSR_API int gsr_sorter_last_ms(gsr_sorter *s, float *ms);

/* ---- misc ---- */
GSR_API const char *gsr_error_string(int code);
GSR_API const char *gsr_last_error(void); /* thread-local detail of the last failure */
GSR_API int gsr_device_count(void);
GSR_API const char *gsr_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GSR_H_ */
