/*
 * id_oracle.c -- the CPU oracle of splat IDs (include/gsr.h gsr_set_splat_ids).
 *
 * TEST INFRASTRUCTURE.  Built by tests/id_reference.py into its own shared library.  It compiles tests/depth_reference/depth_oracle.c
 * (and with it oracle/gsr_oracle.c) into the same translation unit and adds the (best, id) walk to the depth-compositing blend;
 * neither of those files changes.
 *
 * Per pixel, for every splat the depth blend blends (same stop rule, dead-pixel rule and order): t' = t * (1 - alpha), the value the
 * blend stores, and w = t - t'.  The pixel's splat is the first with the largest w (a later one replaces it only when its w is strictly
 * greater); ids_out holds its drawn id (the sorted value), NO_ID where no w was > 0.  rgba and depth are dco_render_depth's.
 */
#include "../depth_reference/depth_oracle.c"

#define IDO_NO_ID 0xFFFFFFFFu

void ido_set_blend_contraction(int on) { orc_set_blend_contraction(on); }

static void ido_blend_pixel(const orc_record *records, const uint32_t *vals, int chunk, float px, float py, const float *vz, float z,
                            float *t, float col[3], float *dacc, float *best, uint32_t *id, int *stopped) {
    const float MIN_ALPHA = 1.0f / 255.0f;
    float tt = *t, r = col[0], g = col[1], b = col[2], D = *dacc, bw = *best;
    uint32_t v = *id;
    for (int j = 0; j < chunk && tt > MIN_ALPHA && !*stopped; ++j) {
        const orc_record *s = &records[vals[j]];
        const float d = -(((vz[0] * s->pos_xy[0] + vz[1] * s->pos_xy[1]) + vz[2] * s->pos_z) + vz[3] * 1.0f);
        if (!(d < z)) { *stopped = 1; break; }
        float ox = s->image_pos[0] - px, oy = s->image_pos[1] - py;
        float alpha;
        if (!g_blend_contraction) {
            float power = -0.5f * (s->conic[0] * ox * ox + s->conic[2] * oy * oy) - s->conic[1] * ox * oy;
            alpha = s->color[3] * orc_exp(power);
            r = r + s->color[0] * alpha * tt;
            g = g + s->color[1] * alpha * tt;
            b = b + s->color[2] * alpha * tt;
            D = D + d * alpha * tt;
        } else {
            float q = fmaf(s->conic[2] * oy, oy, s->conic[0] * ox * ox);
            float power = fmaf(-(s->conic[1] * ox), oy, -0.5f * q);
            alpha = s->color[3] * orc_exp(power);
            r = fmaf(s->color[0] * alpha, tt, r);
            g = fmaf(s->color[1] * alpha, tt, g);
            b = fmaf(s->color[2] * alpha, tt, b);
            D = fmaf(d * alpha, tt, D);
        }
        const float tn = tt * (1.0f - alpha);
        const float w = tt - tn;
        if (w > bw) { bw = w; v = vals[j]; }
        tt = tn;
    }
    *t = tt; col[0] = r; col[1] = g; col[2] = b; *dacc = D; *best = bw; *id = v;
}

/* The full frame: dco_render_depth plus ids_out (W*H drawn ids, IDO_NO_ID where no splat had w > 0). */
void ido_render_ids(const orc_record *records, const uint32_t *values, const uint32_t *bounds, int W, int H, float heatmap_factor,
                    const float *vp, const float *scene_depth, float *out, float *depth_out, uint32_t *ids_out, int64_t *staged_out) {
    const int gx = (W + ORC_TILE - 1) / ORC_TILE, gy = (H + ORC_TILE - 1) / ORC_TILE;
    const float vz[4] = {vp[2], vp[6], vp[10], vp[14]};
    int64_t staged_total = 0;
#pragma omp parallel for schedule(dynamic, 1) collapse(2) reduction(+ : staged_total)
    for (int ty = 0; ty < gy; ++ty)
        for (int tx = 0; tx < gx; ++tx) {
            const uint32_t tile_id = (uint32_t)(ty * gx + tx);
            const uint32_t bx = bounds[2 * tile_id], by = bounds[2 * tile_id + 1];
            const int32_t diff = (int32_t)(by - bx);
            const int num_splats = diff > 0 ? diff : 0;
            const int num_iterations = (int)ceilf((float)num_splats / 256.0f);
            float col[ORC_WG][3], t[ORC_WG], dacc[ORC_WG], best[ORC_WG], z[ORC_WG];
            uint32_t id[ORC_WG];
            int stopped[ORC_WG];
            for (int l = 0; l < ORC_WG; ++l) {
                const int px = tx * ORC_TILE + (l & 15), py = ty * ORC_TILE + (l >> 4);
                col[l][0] = col[l][1] = col[l][2] = 0.0f; t[l] = 1.0f; dacc[l] = 0.0f; best[l] = 0.0f; id[l] = IDO_NO_ID; stopped[l] = 0;
                z[l] = (scene_depth && px < W && py < H) ? scene_depth[(size_t)py * W + px] : INFINITY;
            }
            uint32_t shared_t = 0xFFFFFFFFu;
            for (int i = 0; i < num_iterations && shared_t > 255u; ++i) {
                const int sort_offset = ORC_WG * i;
                const int chunk = (num_splats - sort_offset) < ORC_WG ? (num_splats - sort_offset) : ORC_WG;
                staged_total += chunk;
                shared_t = 0;
                for (int l = 0; l < ORC_WG; ++l) {
                    const float px = (float)(tx * ORC_TILE + (l & 15)), py = (float)(ty * ORC_TILE + (l >> 4));
                    ido_blend_pixel(records, values + bx + (uint32_t)sort_offset, chunk, px, py, vz, z[l], &t[l], col[l], &dacc[l], &best[l],
                                    &id[l], &stopped[l]);
                    if (!stopped[l]) shared_t += (uint32_t)(t[l] * 255.0f);
                }
            }
            const float hx = (float)num_splats * 5e-4f;
            const float h0 = 0.0f * (1.0f - hx) + 1.0f * hx, h1 = 0.0f * (1.0f - hx) + 0.2f * hx, h2 = 1.0f * (1.0f - hx) + 0.2f * hx;
            for (int l = 0; l < ORC_WG; ++l) {
                const int px = tx * ORC_TILE + (l & 15), py = ty * ORC_TILE + (l >> 4);
                if (px >= W || py >= H) continue;
                float *o = out + ((size_t)py * W + px) * 4;
                const float k = 1.0f - t[l];
                o[0] = col[l][0] + h0 * k * heatmap_factor;
                o[1] = col[l][1] + h1 * k * heatmap_factor;
                o[2] = col[l][2] + h2 * k * heatmap_factor;
                o[3] = k;
                depth_out[(size_t)py * W + px] = k > 0.0f ? dacc[l] / k : INFINITY;
                ids_out[(size_t)py * W + px] = best[l] > 0.0f ? id[l] : IDO_NO_ID;
            }
        }
    if (staged_out) *staged_out = staged_total;
}
