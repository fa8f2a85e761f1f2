/*
 * gsr_host.c -- a minimal C99 host of the C-ABI (include/gsr.h): the smallest program a maintainer of the reference
 * could link against libgsr.so.  It plays the role of GaussianSplattingRasterizer.rasterize()
 * (util/gaussian_splatting_rasterizer.gd:122-160) for ONE frame described by a request file:
 *
 *   request  := header | splats | camera | uniforms
 *   header   := uint32 magic 'GSRQ', uint32 n_splats, uint32 width, uint32 height, float heatmap, uint32 flags
 *   splats   := n_splats * 60 floats   (the std430 Splat of gsplat_projection.glsl:33-40, what ply_file.gd:71 uploads)
 *   camera   := 32 floats              (the push constant of update_camera_matrices(), rasterizer.gd:175-195)
 *   uniforms := 32 bytes               (the std140 block rasterizer.gd:126 writes)
 *
 *   gsr_host <request> <out.rgba>      writes width*height*4 floats (the rgba32f render texture) and prints the
 *                                      frame statistics main.gd:93-119 shows (M, overflow flag, stage times).
 *
 * Exit codes: 0 ok; 2 usage / unreadable request; 3 a libgsr call failed (message on stderr) -- in particular
 * GSR_ERR_CUDA without an sm_90 device: there is no CPU fallback.
 *
 * Build: gcc -std=c99 -O2 -Iinclude examples/gsr_host.c -Lgodotgaussiansplatting_b200 -lgsr -Wl,-rpath,... -o gsr_host
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gsr.h"

#define GSRQ_MAGIC 0x51525347u /* 'G','S','R','Q' little endian */

typedef struct {
    uint32_t magic, n_splats, width, height;
    float heatmap;
    uint32_t flags;
} request_header;

static int fail(const char *what, int rc) {
    fprintf(stderr, "gsr_host: %s failed: %s (%s)\n", what, gsr_error_string(rc), gsr_last_error());
    return 3;
}

int main(int argc, char **argv) {
    if (argc != 3) {
        fprintf(stderr, "usage: %s <request> <out.rgba>   (libgsr %s, %d CUDA device(s))\n", argv[0], gsr_version(), gsr_device_count());
        return 2;
    }
    FILE *f = fopen(argv[1], "rb");
    request_header h;
    if (!f || fread(&h, sizeof h, 1, f) != 1 || h.magic != GSRQ_MAGIC) {
        fprintf(stderr, "gsr_host: cannot read request %s\n", argv[1]);
        return 2;
    }
    float *splats = (float *)malloc((size_t)h.n_splats * 60 * sizeof(float) + 4);
    float camera[32];
    unsigned char uniforms[32];
    if (!splats || fread(splats, sizeof(float) * 60, h.n_splats, f) != h.n_splats || fread(camera, sizeof camera, 1, f) != 1 ||
        fread(uniforms, sizeof uniforms, 1, f) != 1) {
        fprintf(stderr, "gsr_host: truncated request %s\n", argv[1]);
        return 2;
    }
    fclose(f);

    /* _init / init_gpu (rasterizer.gd:59-113) */
    gsr_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.device = 0;
    cfg.flags = h.flags;
    cfg.max_splats = h.n_splats;
    cfg.dup_capacity_factor = 10; /* rasterizer.gd:79 */
    gsr_ctx *ctx = NULL;
    int rc = gsr_create(&cfg, &ctx);
    if (rc != GSR_OK) return fail("gsr_create", rc);
    if ((rc = gsr_resize(ctx, (int32_t)h.width, (int32_t)h.height)) != GSR_OK) return fail("gsr_resize", rc);
    /* PlyFile.load_gaussian_splats uploads in chunks of size/1000 (ply_file.gd:36-71): do the same */
    uint64_t chunk = h.n_splats / 1000 ? h.n_splats / 1000 : 1;
    for (uint64_t first = 0; first < h.n_splats; first += chunk) {
        uint64_t count = (h.n_splats - first < chunk) ? h.n_splats - first : chunk;
        if ((rc = gsr_upload_splats_aos(ctx, splats + first * 60, first, count)) != GSR_OK) return fail("gsr_upload_splats_aos", rc);
    }

    /* rasterize() (rasterizer.gd:122-160) */
    float *frame = (float *)malloc((size_t)h.width * h.height * 4 * sizeof(float));
    if (!frame) return 2;
    if ((rc = gsr_render(ctx, camera, uniforms, h.heatmap, frame)) != GSR_OK) return fail("gsr_render", rc);

    gsr_stats st;
    if ((rc = gsr_get_stats(ctx, &st)) != GSR_OK) return fail("gsr_get_stats", rc);
    printf("splats %llu visible %llu duplicates %llu%s staged %llu launches %u\n", (unsigned long long)st.num_splats,
           (unsigned long long)st.visible, (unsigned long long)st.duplicates, st.overflow ? " (buffer overflow!)" : "",
           (unsigned long long)st.staged, st.kernel_launches);
    printf("Projection %.3f ms  Sort %.3f ms  Boundaries %.3f ms  Render %.3f ms  total %.3f ms\n", st.stage_ms[0], st.stage_ms[1],
           st.stage_ms[2], st.stage_ms[3], st.stage_ms[4]);

    FILE *o = fopen(argv[2], "wb");
    if (!o || fwrite(frame, sizeof(float) * 4, (size_t)h.width * h.height, o) != (size_t)h.width * h.height) {
        fprintf(stderr, "gsr_host: cannot write %s\n", argv[2]);
        return 2;
    }
    fclose(o);
    gsr_destroy(ctx); /* cleanup_gpu (rasterizer.gd:116-120) */
    free(frame);
    free(splats);
    return 0;
}
