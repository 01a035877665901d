/* orc_deskew.c -- TEST INFRASTRUCTURE (CPU oracle): per-point deskewing before the projection (DESIGN.md section 11).
 * No counterpart in the reference. The motion over the sweep goes through the same host function as the library's
 * (include/suma_b200_deskew.h); the per-point formula is restated here in fp32 with the oracle's pinned arithmetic, in
 * the order of sb_math.cuh deskew_sweep_time / deskew_point. Built on its own against liborc.so (oracle/deskew.py):
 * it moves the points and hands them to the oracle's unchanged preprocessing and processScan. */
#include "orc_deskew.h"
#include "orc_internal.h"

#include <stdlib.h>

#include "../include/suma_b200_deskew.h"

/* sweep time in [0, 1]: mode 1 the caller's time (clamped, non-finite -> ref), mode 2 frac(dir (a0 - yaw) / 2pi) */
static float orc_sweep_time(int32_t mode, float t, float yaw, float ref, float a0, int32_t clockwise) {
  if (mode == 1) {
    if (!(fabsf(t) <= 3.402823466e38f)) return ref;
    return t < 0.0f ? 0.0f : (t > 1.0f ? 1.0f : t);
  }
  const float u = clockwise ? a0 - yaw : yaw - a0;
  const float q = u / 6.28318530717958647692f;
  return q - floorf(q);
}

/* p' = Exp(tau w) p + tau t; tau == 0: the bits of p */
static orc_v3 orc_deskew_point(orc_v3 p, float tau, orc_v3 w, orc_v3 t) {
  if (tau == 0.0f) return p;
  const orc_v3 wt = orc_scale3(tau, w);
  const float th2 = orc_dot3(wt, wt);
  float a = 1.0f, b = 0.5f;
  if (th2 > 1e-30f) {
    const float th = sqrtf(th2);
    const float h = orc_sinf(0.5f * th);
    a = orc_sinf(th) / th;
    b = (2.0f * (h * h)) / th2;
  }
  const orc_v3 c1 = orc_cross3(wt, p);
  const orc_v3 c2 = orc_cross3(wt, c1);
  return orc_mk3(((p.x + a * c1.x) + b * c2.x) + tau * t.x, ((p.y + a * c1.y) + b * c2.y) + tau * t.y,
                 ((p.z + a * c1.z) + b * c2.z) + tau * t.z);
}

int orc_deskew_points(const float* pts4, const float* times, uint32_t n, int32_t mode, float ref_time,
                      float start_azimuth, int32_t clockwise, const double motion[16], float* out4) {
  float w[3] = {0, 0, 0}, t[3] = {0, 0, 0};
  const int still = mode == 0 || motion == NULL || sb_deskew_motion(motion, w, t);
  if (still) {
    if (out4 != pts4) memcpy(out4, pts4, (size_t)n * 16);
    return 0;
  }
  const orc_v3 W = orc_mk3(w[0], w[1], w[2]), T = orc_mk3(t[0], t[1], t[2]);
  for (uint32_t i = 0; i < n; ++i) {
    const float* p = pts4 + 4 * (size_t)i;
    const float s = orc_sweep_time(mode, mode == 1 ? times[i] : 0.0f, mode == 2 ? orc_atan2f(p[1], p[0]) : 0.0f,
                                   ref_time, start_azimuth, clockwise != 0);
    const orc_v3 q = orc_deskew_point(orc_mk3(p[0], p[1], p[2]), s - ref_time, W, T);
    const float pw = p[3];
    out4[4 * (size_t)i + 0] = q.x;
    out4[4 * (size_t)i + 1] = q.y;
    out4[4 * (size_t)i + 2] = q.z;
    out4[4 * (size_t)i + 3] = pw;
  }
  return 1;
}

void orc_preprocess_deskew(const orc_params* p, const float* pts4, const float* labels, const float* probs,
                           const float* times, uint32_t n, uint32_t timestamp, int32_t mode, float ref_time,
                           float start_azimuth, int32_t clockwise, const double motion[16], float* vertex_map,
                           float* normal_map, float* semantic_map) {
  float* moved = (float*)malloc((size_t)(n ? n : 1) * 16);
  orc_deskew_points(pts4, times, n, mode, ref_time, start_azimuth, clockwise, motion, moved);
  orc_preprocess(p, moved, labels, probs, n, timestamp, vertex_map, normal_map, semantic_map);
  free(moved);
}

void orc_slam_process_scan_timed(orc_slam* s, const float* pts4, const float* labels, const float* probs,
                                 const float* times, uint32_t n, int32_t mode, float ref_time, float start_azimuth,
                                 int32_t clockwise) {
  if (mode == 0) {
    orc_slam_process_scan(s, pts4, labels, probs, n);
    return;
  }
  float* moved = (float*)malloc((size_t)(n ? n : 1) * 16);
  /* lastIncrement_ as the previous scan left it: the increment the next Gauss-Newton run starts from */
  orc_deskew_points(pts4, times, n, mode, ref_time, start_azimuth, clockwise, orc_slam_pose_member(s, 6), moved);
  orc_slam_process_scan(s, moved, labels, probs, n);
  free(moved);
}
