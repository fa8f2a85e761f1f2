/*
 * aa_oracle.c -- the CPU oracle of anti-aliased frames (include/gsr.h gsr_set_antialiasing).
 *
 * TEST INFRASTRUCTURE.  Built by tests/aa_reference.py into its own shared library.  It compiles oracle/gsr_oracle.c into the same
 * translation unit, so the frame below uses the oracle's own deterministic pow / exp, record layout, sort, tile ranges and compositor,
 * and the default frame of that library stays exactly what oracle/ computes.
 *
 * aao_project_one is project_one of gsr_oracle.c, operation for operation, except for the lines marked AA (v = the filter variance):
 *   - cx = c2_00 + v, cz = c2_11 + v instead of + 0.3;
 *   - after the det == 0 and eigenvalue culls: det0 = c2_00*c2_11 - c2_01*c2_01, coef = sqrtf(max(0.000025, det0 / det)) (GLSL max:
 *     NaN gives the floor), opacity = splat_opacity * coef -- the radius (pow(opacity, 0.2)) and the record's opacity use it.
 * ortho != 0 applies the orthographic lines of tests/ortho_reference/ortho_oracle.c (GSR_FLAG_ORTHOGRAPHIC) as well, marked ORTHO.
 * Instances need no function of their own: instance k is this projection with vp = (V_k, P) (tests/aa_reference.py).
 */
#include "../../oracle/gsr_oracle.c"

static void aao_project_one(const float *s, const float *vp, const orc_uniforms *u, float v, int ortho, orc_record *rec, orc_proj *out) {
    const float *V = vp, *P = vp + 16; /* X[c][r] = X[4*c + r] */
    const int W = u->dims[0], H = u->dims[1];
    const uint32_t gx = (uint32_t)((W + ORC_TILE - 1) / ORC_TILE), gy = (uint32_t)((H + ORC_TILE - 1) / ORC_TILE);
    const float ms = u->model_scale;
    out->ntiles = 0;

    /* :158-166 frustum cull */
    float sp[3] = {s[0] * ms, s[1] * ms, s[2] * ms};
    float view[4], clip[4];
    for (int r = 0; r < 4; ++r) view[r] = ((V[0 + r] * sp[0] + V[4 + r] * sp[1]) + V[8 + r] * sp[2]) + V[12 + r] * 1.0f;
    for (int r = 0; r < 4; ++r) clip[r] = ((P[0 + r] * view[0] + P[4 + r] * view[1]) + P[8 + r] * view[2]) + P[12 + r] * view[3];
    float vb = clip[3] * 1.2f;
    float zlo = ortho ? -clip[3] : 0.0f; /* ORTHO: the whole [near, far] slab */
    if (clip[0] < -vb || clip[1] < -vb || clip[2] < zlo || clip[0] > vb || clip[1] > vb || clip[2] > clip[3]) return;

    /* :169-174 load-in animation */
    float splat_time = u->time - s[3];
    float tf = ease_out_cubic(orc_clamp(splat_time, 0.0f, 1.0f));
    float tfl = ease_out_cubic(orc_clamp(splat_time - 0.35f, 0.0f, 1.0f));
    float splat_opacity = s[10] * tfl * tfl;
    float splat_scale = ms * (2.0f * (1.0f - tfl) + 1.0f * tfl); /* mix(2.0, 1.0, tfl) */

    /* :124-142 project_covariance */
    const float *c = s + 4;
    mat3 cov3 = {{{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}}};
    for (int cc = 0; cc < 3; ++cc) for (int r = 0; r < 3; ++r) cov3.m[cc][r] = cov3.m[cc][r] * splat_scale * splat_scale;
    float tfi[2] = {P[0], P[5]};
    float focal[2] = {((float)W * 0.5f) * tfi[0], ((float)H * 0.5f) * tfi[1]};
    float B0[3], B1[3], T0[3], T1[3];
    if (ortho) { /* ORTHO: no z_inv, no mean clamp; the Jacobian is diag(focal.x, focal.y, 0) */
        for (int r = 0; r < 3; ++r) {
            B0[r] = V[4 * r + 0] * focal[0];
            B1[r] = V[4 * r + 1] * focal[1];
        }
    } else {
        float tanfov[2] = {1.0f / tfi[0], 1.0f / tfi[1]};
        float z_inv = 1.0f / view[2];
        focal[0] *= z_inv; focal[1] *= z_inv;
        float mx = orc_clamp(view[0] * z_inv, -tanfov[0] * 1.3f, tanfov[0] * 1.3f);
        float my = orc_clamp(view[1] * z_inv, -tanfov[1] * 1.3f, tanfov[1] * 1.3f);
        float j02 = -focal[1] * mx, j12 = -focal[1] * my;
        for (int r = 0; r < 3; ++r) {
            B0[r] = V[4 * r + 0] * focal[0] + V[4 * r + 2] * j02;
            B1[r] = V[4 * r + 1] * focal[1] + V[4 * r + 2] * j12;
        }
    }
    for (int cc = 0; cc < 3; ++cc) { /* t1 = transpose(b) * cov_3d: T0[c] = t1[c][0], T1[c] = t1[c][1] */
        T0[cc] = (B0[0] * cov3.m[cc][0] + B0[1] * cov3.m[cc][1]) + B0[2] * cov3.m[cc][2];
        T1[cc] = (B1[0] * cov3.m[cc][0] + B1[1] * cov3.m[cc][1]) + B1[2] * cov3.m[cc][2];
    }
    float c2_00 = (T0[0] * B0[0] + T0[1] * B0[1]) + T0[2] * B0[2];
    float c2_01 = (T1[0] * B0[0] + T1[1] * B0[1]) + T1[2] * B0[2];
    float c2_11 = (T1[0] * B1[0] + T1[1] * B1[1]) + T1[2] * B1[2];
    float cx = c2_00 + v, cy = c2_01, cz = c2_11 + v; /* AA */

    /* :177-182 */
    float det = cx * cz - cy * cy;
    if (det == 0.0f) return;
    float mid = 0.5f * (cx + cz);
    float sq = sqrtf(orc_max(0.1f, mid * mid - det));
    float e1 = mid + 1.0f * sq, e2 = mid + -1.0f * sq;
    if (e1 < 0.0f || e2 < 0.0f) return;
    float det0 = c2_00 * c2_11 - c2_01 * c2_01;           /* AA: the undilated determinant */
    float coef = sqrtf(orc_max(0.000025f, det0 / det));   /* AA */
    float opacity = splat_opacity * coef;                  /* AA: the splat's opacity from here on */

    /* :184-185 */
    float ndc[3] = {clip[0] / clip[3], clip[1] / clip[3], clip[2] / clip[3]};
    float ipx = ((ndc[0] + 1.0f) * 0.5f - 1.0f * (1.0f - tf)) * (float)(W - 1);
    float ipy = ((ndc[1] + 1.0f) * 0.5f - 0.75f * (1.0f - tf)) * (float)(H - 1);

    /* :190-194 */
    float radius = orc_pow(opacity, 0.2f) * 2.5f * sqrtf(orc_max(e1, e2)); /* AA: the compensated opacity */
    if (!(fabsf(ipx) <= 3.0e38f) || !(fabsf(ipy) <= 3.0e38f) || !(radius <= 3.0e38f)) return;
    float fgx = (float)gx, fgy = (float)gy;
    int32_t x0 = (int32_t)orc_clamp((ipx - radius) / 16.0f, 0.0f, fgx);
    int32_t y0 = (int32_t)orc_clamp((ipy - radius) / 16.0f, 0.0f, fgy);
    int32_t x1 = (int32_t)orc_clamp(ceilf((ipx + radius) / 16.0f), 0.0f, fgx);
    int32_t y1 = (int32_t)orc_clamp(ceilf((ipy + radius) / 16.0f), 0.0f, fgy);
    uint32_t n = (uint32_t)(x1 - x0) * (uint32_t)(y1 - y0);
    if (n == 0) return;

    /* :198-206 */
    float d[3];
    if (ortho) { d[0] = -V[2]; d[1] = -V[6]; d[2] = -V[10]; } /* ORTHO: the camera's forward axis */
    else { d[0] = sp[0] - u->camera_pos[0]; d[1] = sp[1] - u->camera_pos[1]; d[2] = sp[2] - u->camera_pos[2]; }
    float inv_len = 1.0f / sqrtf((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    float dx = d[0] * inv_len, dy = d[1] * inv_len, dz = d[2] * inv_len;
    rec->image_pos[0] = ipx; rec->image_pos[1] = ipy;
    rec->conic[0] = cz / det; rec->conic[1] = -cy / det; rec->conic[2] = cx / det;
    const float *sh = s + 12;
    rec->color[0] = sh_channel(sh, 0, dx, dy, dz);
    rec->color[1] = sh_channel(sh, 1, dx, dy, dz);
    rec->color[2] = sh_channel(sh, 2, dx, dy, dz);
    rec->color[3] = opacity; /* AA */
    rec->pos_xy[0] = sp[0]; rec->pos_xy[1] = sp[1]; rec->pos_z = sp[2];

    if (ortho) out->depth = ((uint32_t)(orc_clamp(ndc[2] * 0.5f + 0.5f, 0.0f, 1.0f) * 65535.0f)) & 0xFFFFu; /* ORTHO */
    else out->depth = ((uint32_t)(ndc[2] * ndc[2] * ndc[2] * 65535.0f)) & 0xFFFFu;                        /* :218 */
    out->rect[0] = (uint32_t)x0; out->rect[1] = (uint32_t)y0; out->rect[2] = (uint32_t)x1; out->rect[3] = (uint32_t)y1;
    out->ntiles = n;
}

/* orc_project (full frame) with aao_project_one: records at splat id, pairs in splat-id order, row-major within a rect.
 * Returns M; visible_out / last_tile_out (nullable) as in orc_project. */
int64_t aao_project(const float *splat60, int64_t n, const float *vp, const orc_uniforms *u, float v, int ortho, orc_record *records,
                    uint32_t *keys, uint32_t *values, int64_t cap, int64_t *visible_out, int64_t *last_tile_out) {
    const uint32_t gx = (uint32_t)((u->dims[0] + ORC_TILE - 1) / ORC_TILE);
    orc_proj *pr = (orc_proj *)malloc(sizeof(orc_proj) * (size_t)(n > 0 ? n : 1));
    int64_t m = 0, vis = 0, last = -1;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) aao_project_one(splat60 + (size_t)i * 60, vp, u, v, ortho, records + i, pr + i);
    for (int64_t i = 0; i < n; ++i) {
        if (!pr[i].ntiles) continue;
        vis += 1;
        for (uint32_t y = pr[i].rect[1]; y < pr[i].rect[3]; ++y)
            for (uint32_t x = pr[i].rect[0]; x < pr[i].rect[2]; ++x) {
                if (m < cap) { keys[m] = ((y * gx + x) << 16) | pr[i].depth; values[m] = (uint32_t)i; }
                ++m;
            }
        const int64_t t = (int64_t)(pr[i].rect[3] - 1) * gx + (pr[i].rect[2] - 1);
        if (t > last) last = t;
    }
    if (visible_out) *visible_out = vis;
    if (last_tile_out) *last_tile_out = last;
    free(pr);
    return m;
}

/* One anti-aliased frame: aao_project, then the oracle's own sort, tile ranges and compositor (orc_frame without a band).
 * Returns 0, or 1 if M > cap (frame not rendered). */
int aao_frame(const float *splat60, int64_t n, const float *vp, const orc_uniforms *u, float v, int ortho, float heatmap_factor, int quirks,
              orc_record *records, uint32_t *keys, uint32_t *values, int64_t cap, uint32_t *bounds, float *out, orc_frame_stats *st) {
    const int gx = (u->dims[0] + ORC_TILE - 1) / ORC_TILE, gy = (u->dims[1] + ORC_TILE - 1) / ORC_TILE;
    int64_t vis = 0, last = -1;
    const int64_t m = aao_project(splat60, n, vp, u, v, ortho, records, keys, values, cap, &vis, &last);
    if (st) { memset(st, 0, sizeof *st); st->visible = vis; st->duplicates = m; st->last_tile = last; }
    if (m > cap) return 1;
    orc_sort_pairs(keys, values, m);
    orc_boundaries(keys, m, (int64_t)gx * gy, bounds, quirks, -1);
    int64_t staged = 0;
    orc_render(records, values, bounds, u->dims[0], u->dims[1], heatmap_factor, 0xFFFFFFFFu, 0, gy, out, NULL, &staged, NULL);
    if (st) st->staged = staged;
    return 0;
}

void aao_set_blend_contraction(int on) { orc_set_blend_contraction(on); }
