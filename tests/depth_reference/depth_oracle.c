/*
 * depth_oracle.c -- the CPU oracle of depth compositing (include/gsr.h gsr_set_depth_compositing).
 *
 * TEST INFRASTRUCTURE.  Built by tests/depth_reference.py into its own shared library.  It compiles oracle/gsr_oracle.c into the
 * same translation unit, so the blend below uses the oracle's own deterministic exp (orc_exp), record layout and contraction
 * switch, and the default frame of that library stays exactly what oracle/ computes.
 *
 * The rules, per pixel p of a tile with scene depth Z(p) (+inf without a plane and for the tile's pixels outside the image):
 *   - the splat's view depth is d = -(((V[2]*x + V[6]*y) + V[10]*z) + V[14]*1.0f) on the record's position (-view[2] of project_one);
 *   - before splat j is blended into p: if !(d_j < Z(p)) (NaN included), p stops -- splat j and every later splat contribute nothing,
 *     t is kept, and p adds 0 to the tile-stop vote;
 *   - colour and t follow orc_render; the depth accumulates like a fourth colour channel: D = fma(d*alpha, t, D) (contracted) or
 *     D = D + d*alpha*t (uncontracted);
 *   - rgb is orc_render's expression, alpha = 1 - t, depth = (1 - t) > 0 ? D / (1 - t) : +inf.
 */
#include "../../oracle/gsr_oracle.c"

void dco_set_blend_contraction(int on) { orc_set_blend_contraction(on); }

/* One pixel's walk over one staged chunk; vals = the chunk's sorted values. */
static void dco_blend_pixel(const orc_record *records, const uint32_t *vals, int chunk, float px, float py, const float *vz, float z,
                            float *t, float col[3], float *dacc, int *stopped) {
    const float MIN_ALPHA = 1.0f / 255.0f;
    float tt = *t, r = col[0], g = col[1], b = col[2], D = *dacc;
    for (int j = 0; j < chunk && tt > MIN_ALPHA && !*stopped; ++j) {
        const orc_record *s = &records[vals[j]];
        const float d = -(((vz[0] * s->pos_xy[0] + vz[1] * s->pos_xy[1]) + vz[2] * s->pos_z) + vz[3] * 1.0f);
        if (!(d < z)) { *stopped = 1; break; }
        float ox = s->image_pos[0] - px, oy = s->image_pos[1] - py;
        float alpha;
        if (!g_blend_contraction) {   /* orc_render's uncontracted evaluation */
            float power = -0.5f * (s->conic[0] * ox * ox + s->conic[2] * oy * oy) - s->conic[1] * ox * oy;
            alpha = s->color[3] * orc_exp(power);
            r = r + s->color[0] * alpha * tt;
            g = g + s->color[1] * alpha * tt;
            b = b + s->color[2] * alpha * tt;
            D = D + d * alpha * tt;
        } else {                      /* orc_render's gsr spec: the explicit contractions */
            float q = fmaf(s->conic[2] * oy, oy, s->conic[0] * ox * ox);
            float power = fmaf(-(s->conic[1] * ox), oy, -0.5f * q);
            alpha = s->color[3] * orc_exp(power);
            r = fmaf(s->color[0] * alpha, tt, r);
            g = fmaf(s->color[1] * alpha, tt, g);
            b = fmaf(s->color[2] * alpha, tt, b);
            D = fmaf(d * alpha, tt, D);
        }
        tt = tt * (1.0f - alpha);
    }
    *t = tt; col[0] = r; col[1] = g; col[2] = b; *dacc = D;
}

/* The full frame.  vp: the 32-float view_proj; scene_depth: nullable W*H; out: W*H*4; depth_out: W*H;
 * staged_out (nullable): instances staged (sum over tiles and consumed chunks of the chunk size). */
void dco_render_depth(const orc_record *records, const uint32_t *values, const uint32_t *bounds, int W, int H, float heatmap_factor,
                      const float *vp, const float *scene_depth, float *out, float *depth_out, int64_t *staged_out) {
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
            float col[ORC_WG][3], t[ORC_WG], dacc[ORC_WG], z[ORC_WG];
            int stopped[ORC_WG];
            for (int l = 0; l < ORC_WG; ++l) {
                const int px = tx * ORC_TILE + (l & 15), py = ty * ORC_TILE + (l >> 4);
                col[l][0] = col[l][1] = col[l][2] = 0.0f; t[l] = 1.0f; dacc[l] = 0.0f; stopped[l] = 0;
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
                    dco_blend_pixel(records, values + bx + (uint32_t)sort_offset, chunk, px, py, vz, z[l], &t[l], col[l], &dacc[l], &stopped[l]);
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
            }
        }
    if (staged_out) *staged_out = staged_total;
}
