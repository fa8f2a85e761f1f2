/*
 * contribution_oracle.c -- the CPU oracle of splat contribution (include/gsr.h gsr_set_splat_contribution).
 *
 * TEST INFRASTRUCTURE.  Built by tests/contribution_reference.py into its own shared library.  It compiles
 * tests/depth_reference/depth_oracle.c (and with it oracle/gsr_oracle.c) into the same translation unit; neither changes.
 *
 * The per-pixel walk of tests/id_reference/id_oracle.c: for every pixel of every tile, every splat the depth-composited blend blends
 * (same stop rule at the scene depth, dead-pixel rule, sorted order and tile-stop vote), t' = t * (1 - alpha) and w = t - t'.  Every
 * in-image pixel and splat with w > 0 adds q(w) = rn(w * 2^24), 1 and max(peak, w) to the record of the splat's slot, and the frame
 * adds 1 to the views of every slot it touched.
 */
#include "../depth_reference/depth_oracle.c"

void cto_set_blend_contraction(int on) { orc_set_blend_contraction(on); }

/* One frame.  slot_of: the source slot of every drawn id (NULL: the drawn id itself); seen: n_slots zero bytes of scratch. */
void cto_accumulate(const orc_record *records, const uint32_t *values, const uint32_t *bounds, int W, int H, const float *vp,
                    const float *scene_depth, const uint32_t *slot_of, uint64_t *weight, uint64_t *pixels, float *peak, uint32_t *views,
                    uint8_t *seen, int64_t n_slots) {
    const float MIN_ALPHA = 1.0f / 255.0f;
    const int gx = (W + ORC_TILE - 1) / ORC_TILE, gy = (H + ORC_TILE - 1) / ORC_TILE;
    const float vz[4] = {vp[2], vp[6], vp[10], vp[14]};
    for (int ty = 0; ty < gy; ++ty)
        for (int tx = 0; tx < gx; ++tx) {
            const uint32_t tile_id = (uint32_t)(ty * gx + tx);
            const uint32_t bx = bounds[2 * tile_id], by = bounds[2 * tile_id + 1];
            const int32_t diff = (int32_t)(by - bx);
            const int num_splats = diff > 0 ? diff : 0;
            const int num_iterations = (int)ceilf((float)num_splats / 256.0f);
            float t[ORC_WG], z[ORC_WG];
            int stopped[ORC_WG];
            for (int l = 0; l < ORC_WG; ++l) {
                const int px = tx * ORC_TILE + (l & 15), py = ty * ORC_TILE + (l >> 4);
                t[l] = 1.0f; stopped[l] = 0;
                z[l] = (scene_depth && px < W && py < H) ? scene_depth[(size_t)py * W + px] : INFINITY;
            }
            uint32_t shared_t = 0xFFFFFFFFu;
            for (int i = 0; i < num_iterations && shared_t > 255u; ++i) {
                const int sort_offset = ORC_WG * i;
                const int chunk = (num_splats - sort_offset) < ORC_WG ? (num_splats - sort_offset) : ORC_WG;
                const uint32_t *vals = values + bx + (uint32_t)sort_offset;
                shared_t = 0;
                for (int l = 0; l < ORC_WG; ++l) {
                    const int ipx = tx * ORC_TILE + (l & 15), ipy = ty * ORC_TILE + (l >> 4);
                    const int inside = ipx < W && ipy < H;
                    const float px = (float)ipx, py = (float)ipy;
                    float tt = t[l];
                    for (int j = 0; j < chunk && tt > MIN_ALPHA && !stopped[l]; ++j) {
                        const orc_record *s = &records[vals[j]];
                        const float d = -(((vz[0] * s->pos_xy[0] + vz[1] * s->pos_xy[1]) + vz[2] * s->pos_z) + vz[3] * 1.0f);
                        if (!(d < z[l])) { stopped[l] = 1; break; }
                        const float ox = s->image_pos[0] - px, oy = s->image_pos[1] - py;
                        float alpha;
                        if (!g_blend_contraction) {
                            const float power = -0.5f * (s->conic[0] * ox * ox + s->conic[2] * oy * oy) - s->conic[1] * ox * oy;
                            alpha = s->color[3] * orc_exp(power);
                        } else {
                            const float q = fmaf(s->conic[2] * oy, oy, s->conic[0] * ox * ox);
                            const float power = fmaf(-(s->conic[1] * ox), oy, -0.5f * q);
                            alpha = s->color[3] * orc_exp(power);
                        }
                        const float tn = tt * (1.0f - alpha);
                        const float w = tt - tn;
                        if (inside && w > 0.0f) {
                            const uint32_t slot = slot_of ? slot_of[vals[j]] : vals[j];
                            if ((int64_t)slot < n_slots) {
                                weight[slot] += (uint64_t)nearbyintf(w * 16777216.0f);
                                pixels[slot] += 1u;
                                if (w > peak[slot]) peak[slot] = w;
                                seen[slot] = 1;
                            }
                        }
                        tt = tn;
                    }
                    t[l] = tt;
                    if (!stopped[l]) shared_t += (uint32_t)(t[l] * 255.0f);
                }
            }
        }
    for (int64_t s = 0; s < n_slots; ++s) { views[s] += seen[s]; seen[s] = 0; }
}
