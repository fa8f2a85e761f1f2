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
                                      Single-context only: an orthographic frame on a context with a shard group, peer framebuffers, a
                                      partial band or row interleave returns GSR_ERR_STATE and enqueues nothing. */

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
                                           rounded up to 256 (gsr_config.sh_bands) */
    GSR_BUF_DEPTH_WORDS_UNSORTED = 11   /* gsr_set_depth_order: the last mode-1 frame's ord(d) per pair in emission order, M entries
                                           (kept with gsr_debug_keep_unsorted once mode 1 has been switched on) */
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
                                     the coefficients the store does not keep.  > 4: GSR_ERR_INVALID.  A store of fewer than 4 bands is
                                     single-context only (see gsr_set_sh_degree). */
} gsr_config;

typedef struct gsr_stats {
    uint64_t num_splats;  /* highest uploaded splat index + 1 */
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
 *      they are.  Single-context only: GSR_ERR_STATE on a context with an attached group, peer framebuffers, a partial band
 *      or row_mod > 1, and those calls fail with GSR_ERR_STATE while the mode is on.  gsr_resize switches the mode off;
 *      gsr_pick keeps the default path (and leaves the depth-composited frame as it is).  GSR_ERR_STATE before gsr_resize. ---- */
GSR_API int gsr_set_depth_compositing(gsr_ctx *ctx, const float *scene_depth_device, float *depth_out_device);

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
 *      max_splats, a non-finite entry, a singular A, D >= 2^32 - 256.  Single-context only: GSR_ERR_STATE with an attached group, peer
 *      framebuffers, a partial band or row_mod > 1, and those calls fail with GSR_ERR_STATE while instances are set.  gsr_resize
 *      keeps the instances. ---- */
#define GSR_MAX_INSTANCES 4096
#define GSR_INSTANCE_RING 8
typedef struct gsr_instance {
    uint64_t first, count;  /* source range of the uploaded splats */
    float to_frame[12];     /* [A | t], column-major 3x4 */
} gsr_instance;
GSR_API int gsr_set_instances(gsr_ctx *ctx, const gsr_instance *instances, uint32_t n);

/* ---- SH degree of the rendered colour (no reference counterpart: the reference always evaluates degree 3).  Frames enqueued after
 *      the call evaluate the view-dependent colour up to `degree` (0 = the DC colour only) from the first P = ceil(3 (degree+1)^2 / 4)
 *      SH planes, so a lower degree also reads fewer bytes.  -1 = the stored degree (gsr_config.sh_bands - 1), the default.  The degree
 *      is read when a frame is enqueued: frames already enqueued keep theirs, and the call never synchronises.  A frame drawn at
 *      degree d is bit for bit the frame of the same cloud with every coefficient above degree d set to zero (DESIGN.md section 5.9).
 *      GSR_ERR_INVALID: a degree below -1 or above the stored one.  A degree below 3, like a store of fewer than 4 bands, is
 *      single-context only: GSR_ERR_STATE with an attached group, peer framebuffers, a partial band or row_mod > 1, and those calls
 *      (and gsr_group_export) fail with GSR_ERR_STATE on such a store or while a degree below 3 is set. ---- */
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
 *      previous state kept: a negative, NaN or infinite variance, or one above 64.  Single-context only: turning the filter on returns
 *      GSR_ERR_STATE with an attached group, peer framebuffers, a partial band or row_mod > 1, and those calls (and gsr_group_export)
 *      fail with GSR_ERR_STATE while it is on. ---- */
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
 *      Single-context only: switching mode 1 on returns GSR_ERR_STATE with an attached group, peer framebuffers, a partial band or
 *      row_mod > 1, and those calls (and gsr_group_export) fail with GSR_ERR_STATE while it is on. ---- */
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
 *      GSR_MAX_CUTOUTS, cutouts == NULL with n > 0, a non-finite to_local entry, an unknown shape, action or space.  Single-context
 *      only: a non-empty set returns GSR_ERR_STATE with an attached group, peer framebuffers, a partial band or row_mod > 1, and those
 *      calls (and gsr_group_export) fail with GSR_ERR_STATE while a set is active. ---- */
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
