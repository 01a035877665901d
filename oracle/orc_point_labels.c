/* orc_point_labels.c -- TEST INFRASTRUCTURE (CPU oracle): the per-point label records of a scan (sb_point_label,
 * DESIGN.md section 13), from the oracle's own K1 projection and depth test, its current frame, the integrated flags of
 * its map update and its current model frame. No counterpart in the reference. Built on its own against liborc.so and
 * the deskewing library (oracle/point_labels.py), which it does not change. */
#include "orc_deskew.h"
#include "orc_internal.h"

#include <stdlib.h>

typedef struct orc_point_label {
  int32_t pixel;
  uint32_t flags;
  uint32_t frame_label;
  float frame_prob;
  int32_t map_pixel;
  uint32_t map_label;
  float map_prob;
  float map_range;
} orc_point_label;
enum { ORC_POINT_WON = 1, ORC_POINT_VERTEX = 2, ORC_POINT_INTEGRATED = 4, ORC_POINT_MAP = 8 };

/* The leading members of struct orc_slam (orc_slam.c), which holds the current model frame the public interface does not
 * hand out; orc_slam_point_labels checks the view against orc_slam_map and orc_slam_current_frame before it reads it. */
typedef struct { float *v, *n, *s; } orc_pl_frame;
typedef struct {
  orc_params p;
  orc_map* map;
  orc_pl_frame cur, last, cur_model, last_model;
} orc_pl_slam_head;

/* gen_vertexmap.vert:83-89 as orc_k1_project computes it: the pixel of pos at range d; 0 when clipped */
static int pl_pixel(orc_v3 pos, float d, int W, int H, float fov_up, float fov, int* ix, int* iy) {
  float yaw = orc_atan2f(pos.y, pos.x);
  float pitch = -orc_asinf(pos.z / d);
  float x = -yaw * ORC_INV_PI_F;
  float y = 1.0f - (2.0f * (ORC_RAD2DEG_F * pitch + fov_up)) / fov;
  float fx = floorf((0.5f * (x + 1.0f)) * (float)W);
  float fy = floorf((0.5f * (y + 1.0f)) * (float)H);
  if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) return 0;
  *ix = (int)fx;
  *iy = (int)fy;
  return 1;
}

/* rintf(255 x) as an unsigned id: NaN and negatives 0, values past the range saturate */
static uint32_t pl_label_id(float x) {
  const float f = rintf(x * 255.0f);
  return f > 0.0f ? (f < 4294967296.0f ? (uint32_t)f : 0xffffffffu) : 0u;
}

/* the records of the scan the slam has just processed; pts4: its points as projected (deskewed when deskewing is on).
 * Returns 0, or -1 when the view of orc_slam does not match the library. */
int orc_slam_point_labels(orc_slam* s, const float* pts4, uint32_t n, orc_point_label* out) {
  const orc_pl_slam_head* h = (const orc_pl_slam_head*)s;
  float *cv, *cn, *cs;
  orc_slam_current_frame(s, &cv, &cn, &cs);
  if (h->map != orc_slam_map(s) || h->cur.v != cv || h->cur.n != cn || h->cur.s != cs) return -1;
  const orc_params* p = &h->p;
  const int W = p->data_width, H = p->data_height, Wm = p->model_width, Hm = p->model_height;
  const float fov_up = fabsf(p->data_fov_up), fov = fov_up + fabsf(p->data_fov_down);
  const float m_fov_up = fabsf(p->model_fov_up), m_fov = m_fov_up + fabsf(p->model_fov_down);
  const size_t P = (size_t)W * H;
  uint8_t* integrated = (uint8_t*)malloc(P);
  uint64_t* best = (uint64_t*)malloc(P * sizeof(uint64_t));
  uint64_t* key = (uint64_t*)malloc((size_t)(n ? n : 1) * sizeof(uint64_t));
  orc_map_get_update_debug(h->map, NULL, NULL, integrated, NULL, NULL);
  for (size_t i = 0; i < P; ++i) best[i] = ~0ull;
  /* K1 and its depth test (GL_LESS in buffer order: the lowest index wins a tie) */
  for (uint32_t i = 0; i < n; ++i) {
    orc_point_label* r = out + i;
    memset(r, 0, sizeof(*r));
    r->pixel = r->map_pixel = -1;
    key[i] = ~0ull;
    const orc_v3 pos = orc_mk3(pts4[4 * (size_t)i + 0], pts4[4 * (size_t)i + 1], pts4[4 * (size_t)i + 2]);
    const float d = orc_len3(pos);
    int ix, iy;
    if (!pl_pixel(pos, d, W, H, fov_up, fov, &ix, &iy)) continue;
    const float z = 2.0f * ((d - p->min_depth) / (p->max_depth - p->min_depth)) - 1.0f;
    if (!(z >= -1.0f && z <= 1.0f)) continue;
    const uint32_t d24 = orc_depth24(0.5f * z + 0.5f);
    if (d24 >= ORC_DEPTH_CLEAR) continue;
    r->pixel = iy * W + ix;
    key[i] = ((uint64_t)d24 << 32) | i;
    if (key[i] < best[r->pixel]) best[r->pixel] = key[i];
  }
  for (uint32_t i = 0; i < n; ++i) {
    orc_point_label* r = out + i;
    if (r->pixel < 0) continue;
    const size_t pix = (size_t)r->pixel;
    if (best[pix] == key[i]) r->flags |= ORC_POINT_WON;
    if (h->cur.v[4 * pix + 3] > 0.0f) r->flags |= ORC_POINT_VERTEX;
    if (integrated[pix]) r->flags |= ORC_POINT_INTEGRATED;
    r->frame_label = pl_label_id(h->cur.s[4 * pix + 0]);
    r->frame_prob = h->cur.s[4 * pix + 3];
    const orc_v3 pos = orc_mk3(pts4[4 * (size_t)i + 0], pts4[4 * (size_t)i + 1], pts4[4 * (size_t)i + 2]);
    int mx, my;
    if (!pl_pixel(pos, orc_len3(pos), Wm, Hm, m_fov_up, m_fov, &mx, &my)) continue;
    r->map_pixel = my * Wm + mx;
    if (!p->render_after_update) continue; /* no model frame of this scan */
    const float* mv = h->cur_model.v + 4 * (size_t)r->map_pixel;
    if (!(mv[3] > 0.0f)) continue;
    const float* ms = h->cur_model.s + 4 * (size_t)r->map_pixel;
    r->flags |= ORC_POINT_MAP;
    r->map_label = pl_label_id(ms[0]);
    r->map_prob = ms[3];
    r->map_range = orc_len3(orc_mk3(mv[0], mv[1], mv[2]));
  }
  free(integrated);
  free(best);
  free(key);
  return 0;
}

/* orc_slam_process_scan_timed (orc_deskew.c) and the records of the scan: out[n] */
int orc_slam_process_scan_labels(orc_slam* s, const float* pts4, const float* labels, const float* probs,
                                 const float* times, uint32_t n, int32_t mode, float ref_time, float start_azimuth,
                                 int32_t clockwise, orc_point_label* out) {
  float* moved = (float*)malloc((size_t)(n ? n : 1) * 16);
  /* lastIncrement_ as the previous scan left it, as orc_slam_process_scan_timed moves the points */
  orc_deskew_points(pts4, times, n, mode, ref_time, start_azimuth, clockwise, orc_slam_pose_member(s, 6), moved);
  orc_slam_process_scan(s, moved, labels, probs, n);
  const int r = orc_slam_point_labels(s, moved, n, out);
  free(moved);
  return r;
}
