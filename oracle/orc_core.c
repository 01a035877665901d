/* orc_core.c -- TEST INFRASTRUCTURE (CPU oracle): params, K1-K3 preprocessing, K5 Jacobian, Gauss-Newton, SE3.
 * See orc.h for the status of this code. Citations are relative to /root/reference/src. */
#include "orc.h"
#include "orc_internal.h"

#include <stdio.h>
#include <stdlib.h>

/* config/default.xml:7-83 */
#ifdef _OPENMP
#include <omp.h>
#endif
static int g_orc_threads = 0; /* 0 = not chosen yet */
int orc_threads(void) {
  if (g_orc_threads <= 0) orc_set_threads(0);
  return g_orc_threads;
}
int orc_set_threads(int n) {
#ifdef _OPENMP
  if (n <= 0) {
    const char* e = getenv("ORC_THREADS");
    n = e ? atoi(e) : omp_get_num_procs();
  }
  if (n < 1) n = 1;
  if (n > 64) n = 64;
#else
  n = 1;
#endif
  g_orc_threads = n;
  return n;
}

void orc_default_params(orc_params* p) {
  memset(p, 0, sizeof(*p));
  p->data_width = 900; p->data_height = 64;
  p->data_fov_up = 3.0f; p->data_fov_down = -25.0f;
  p->min_depth = 2.0f; p->max_depth = 75.0f;
  p->model_width = 900; p->model_height = 64;
  p->model_fov_up = 3.0f; p->model_fov_down = -25.0f;
  p->model_min_depth = 2.0f; p->model_max_depth = 75.0f;
  p->max_iterations = 33; p->stopping_threshold = 0.0001f; p->delta = 0.0001f;
  p->icp_max_distance = 2.0f; p->icp_max_angle = 30.0f;
  p->weighting = 1; p->factor = 0.5f;
  p->initialize_identity = 0; p->bilinear_sampling = 1;
  p->fallback_mode = 1; p->fallback_max_distance = 0.5f; p->fallback_max_angle = 30.0f;
  p->compose_rendering = 1; p->max_loop_closure_distance = 8.0f;
  p->min_radius = 0.03f; p->max_radius = 1.0f; p->max_angle = 90.0f;
  p->map_max_distance = 0.2f; p->map_max_angle = 45.0f;
  p->unstable_age = 3; p->confidence_mode = 3; p->confidence_threshold = 0.0f;
  p->p_stable = 0.6f; p->p_prior = 0.5f; p->sigma_angle = 1.0f; p->sigma_distance = 1.0f;
  p->use_stability = 1; p->active_timestamps = 100; p->max_weight = 20.0f;
  p->weighting_scheme = 0; p->averaging_scheme = 0; p->update_always = 0;
  p->submap_dimension = 4; p->submap_extent = 10.0f; p->partial_extraction = 1;
  p->label_offset_quirk = 1; p->render_after_update = 1;
}

/* the rule of sb_create: image sizes, and the Q33.30 head-room of the exact ICP sums -- data pixels x (the longer of the
 * two depth ranges + 25 m for the pose's translation)^2 x 2^30 must stay within int64 (DESIGN.md section 2) */
const char* orc_check_params(const orc_params* p) {
  if (p->data_width <= 0 || p->data_height <= 0 || p->model_width <= 0 || p->model_height <= 0) return "image size <= 0";
  if ((size_t)p->data_width * p->data_height > (1u << 24)) return "more than 2^24 data pixels";
  if (p->data_width < 2) return "data width < 2";
  if (p->model_width > 65536 || p->model_height > 65536)
    return "model image side > 65536 (the render pass packs pixel boxes in 16 bits)";
  if (!(p->max_depth > p->min_depth) || !(p->model_max_depth > p->model_min_depth)) return "max depth <= min depth";
  const double range = (p->max_depth > p->model_max_depth ? p->max_depth : p->model_max_depth) + 25.0;
  if ((double)p->data_width * p->data_height * range * range * 1073741824.0 > 9223372036854775807.0)
    return "data pixels x (max depth + 25 m)^2 x 2^30 exceeds the int64 range of the exact ICP sums";
  return NULL;
}

float orc_t_atan2f(float y, float x) { return orc_atan2f(y, x); }
float orc_t_asinf(float x) { return orc_asinf(x); }
float orc_t_acosf(float x) { return orc_acosf(x); }
float orc_t_sinf(float x) { return orc_sinf(x); }
float orc_t_expf(float x) { return orc_expf(x); }
float orc_t_logf(float x) { return orc_logf(x); }
void orc_t_sincos(double x, double* s, double* c) { orc_sincos(x, s, c); }

/* ===================================================================================================
 * K1: gen_vertexmap.vert:73-103 + .frag:16-23, drawn with depth test GL_LESS (Preprocessing.cpp:158-184)
 * =================================================================================================== */
static void orc_k1_project(const orc_params* p, const float* pts4, const float* labels, const float* probs,
                           uint32_t n, uint32_t timestamp, float* vertex_map, float* semantic_map) {
  const int W = p->data_width, H = p->data_height;
  const size_t P = (size_t)W * H;
  const float fov_up = fabsf(p->data_fov_up), fov_down = fabsf(p->data_fov_down); /* Preprocessing.cpp:94-95 */
  const float fov = fov_up + fov_down;
  const float min_depth = p->min_depth, max_depth = p->max_depth;
  const int isfirst = timestamp < 10; /* Preprocessing.cpp:176 */
  uint32_t* depth = (uint32_t*)malloc(P * sizeof(uint32_t));
  for (size_t i = 0; i < P; ++i) depth[i] = ORC_DEPTH_CLEAR;
  memset(vertex_map, 0, P * 4 * sizeof(float));
  memset(semantic_map, 0, P * 4 * sizeof(float));

  /* phase 1 (all host threads): the per-point projection; phase 2 (buffer order): the depth test and the writes */
  int32_t* ppix = (int32_t*)malloc((size_t)(n ? n : 1) * sizeof(int32_t));
  uint32_t* pd24 = (uint32_t*)malloc((size_t)(n ? n : 1) * sizeof(uint32_t));
#pragma omp parallel for schedule(static) num_threads(orc_threads())
  for (uint32_t i = 0; i < n; ++i) {
    orc_v3 pos = orc_mk3(pts4[4 * i + 0], pts4[4 * i + 1], pts4[4 * i + 2]);
    ppix[i] = -1;
    float d = orc_len3(pos);
    float yaw = orc_atan2f(pos.y, pos.x);
    float pitch = -orc_asinf(pos.z / d);
    float x = -yaw * ORC_INV_PI_F;                                           /* .vert:83 */
    float y = 1.0f - (2.0f * (ORC_RAD2DEG_F * pitch + fov_up)) / fov;        /* .vert:84 */
    float z = 2.0f * ((d - min_depth) / (max_depth - min_depth)) - 1.0f;     /* .vert:85 */
    float fx = floorf((0.5f * (x + 1.0f)) * (float)W);                       /* .vert:88 */
    float fy = floorf((0.5f * (y + 1.0f)) * (float)H);                       /* .vert:89 */
    if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) continue; /* clipped */
    if (!(z >= -1.0f && z <= 1.0f)) continue;
    pd24[i] = orc_depth24(0.5f * z + 0.5f);
    ppix[i] = (int32_t)((size_t)(int)fy * W + (size_t)(int)fx);
  }
  for (uint32_t i = 0; i < n; ++i) {
    if (ppix[i] < 0) continue;
    const size_t pix = (size_t)ppix[i];
    const uint32_t d24 = pd24[i];
    if (d24 < depth[pix]) { /* GL_LESS, primitives in buffer order */
      depth[pix] = d24;
      /* Q1: attribute pointers start 16 / 20 bytes into the stride-4 label / prob buffers (Preprocessing.cpp:142-145);
       * reads past the end return 0 (robust buffer access). */
      float label = 0.0f, prob = 0.0f;
      if (labels) {
        uint32_t li = p->label_offset_quirk ? i + 4 : i;
        if (li < n) label = labels[li];
      }
      if (probs) {
        uint32_t pi = p->label_offset_quirk ? i + 5 : i;
        if (pi < n) prob = probs[pi];
      }
      float* v = vertex_map + 4 * pix;
      if (isfirst && orc_is_movable(label)) { /* .vert:95-102 */
        v[0] = v[1] = v[2] = v[3] = 0.0f;
      } else {
        v[0] = pts4[4 * i + 0]; v[1] = pts4[4 * i + 1]; v[2] = pts4[4 * i + 2]; v[3] = 1.0f;
      }
      float* sm = semantic_map + 4 * pix;
      float l = label / 255.0f; /* .frag:20 */
      sm[0] = l; sm[1] = l; sm[2] = l; sm[3] = prob;
    }
  }
  free(ppix);
  free(pd24);
  free(depth);
}

/* texel fetch with CLAMP_TO_BORDER (border = 0) in y and the shader's own wrap() in x */
static inline const float* orc_tex_wrapx(const float* img, int W, int H, int x, int y) {
  static const float zero[4] = {0, 0, 0, 0};
  if (y < 0 || y >= H) return zero;
  if (x >= W) x -= W;
  if (x < 0) x += W;
  return img + 4 * ((size_t)y * W + x);
}

/* K2: gen_normalmap.frag:41-99 */
static void orc_k2_normals(const orc_params* p, const float* vertex_map, const float* sem_in, float* normal_map,
                           float* eroded) {
  const int W = p->data_width, H = p->data_height;
#pragma omp parallel for collapse(2) schedule(static) num_threads(orc_threads())
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      size_t pix = (size_t)y * W + x;
      float* nrm = normal_map + 4 * pix;
      float* ero = eroded + 4 * pix;
      const float* P = vertex_map + 4 * pix;
      nrm[0] = nrm[1] = nrm[2] = 0.0f; nrm[3] = 1.0f; /* invalid = (0,0,0,1), .frag:39,45 (Q2) */
      ero[0] = ero[1] = ero[2] = 0.0f; ero[3] = 1.0f;
      if (!(P[3] > 0.0f)) continue;
      float nw = 1.0f;
      const float* U = orc_tex_wrapx(vertex_map, W, H, x + 1, y);
      const float* V = orc_tex_wrapx(vertex_map, W, H, x, y + 1);
      const float* S = orc_tex_wrapx(vertex_map, W, H, x - 1, y);
      const float* T = orc_tex_wrapx(vertex_map, W, H, x, y - 1);
      if (U[3] < 1.0f && V[3] < 1.0f) nw = 0.0f;       /* .frag:63 */
      if (S[3] < 1.0f && T[3] < 1.0f) nw = 0.0f;       /* .frag:64 */
      if (!(U[3] > 0.5f) || !(V[3] > 0.5f)) nw = 0.0f; /* .frag:66 */
      /* erosion, kernel_size = 2 -> offset 1 only (.frag:69-85) */
      const float* sp = sem_in + 4 * pix;
      ero[0] = sp[0]; ero[1] = sp[1]; ero[2] = sp[2]; ero[3] = sp[3];
      float pl = sp[0];
      float ul = orc_tex_wrapx(sem_in, W, H, x + 1, y)[0];
      float vl = orc_tex_wrapx(sem_in, W, H, x, y + 1)[0];
      float sl = orc_tex_wrapx(sem_in, W, H, x - 1, y)[0];
      float tl = orc_tex_wrapx(sem_in, W, H, x, y - 1)[0];
      if ((pl != ul && ul != 0.0f) || (pl != vl && vl != 0.0f) || (pl != sl && sl != 0.0f) ||
          (pl != tl && tl != 0.0f)) {
        ero[0] = ero[1] = ero[2] = 0.0f; ero[3] = 1.0f;
      }
      if (nw > 0.0f) { /* .frag:91-97 */
        orc_v3 pp = orc_mk3(P[0], P[1], P[2]);
        orc_v3 u = orc_normalize3(orc_sub3(orc_mk3(U[0], U[1], U[2]), pp));
        orc_v3 v = orc_normalize3(orc_sub3(orc_mk3(V[0], V[1], V[2]), pp));
        orc_v3 w = orc_cross3(u, v);
        float len = orc_len3(w);
        nrm[0] = w.x / len; nrm[1] = w.y / len; nrm[2] = w.z / len;
        nrm[3] = (len > 0.0000001f) ? 1.0f : 0.0f;
      } else {
        nrm[3] = 0.0f;
      }
    }
}

/* K3: floodfill.frag:34-84 */
static void orc_k3_floodfill(const orc_params* p, const float* vertex_map, const float* eroded, float* semantic_map) {
  const int W = p->data_width, H = p->data_height;
  static const int dx[4] = {1, 0, -1, 0}, dy[4] = {0, 1, 0, -1};
#pragma omp parallel for collapse(2) schedule(static) num_threads(orc_threads())
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      size_t pix = (size_t)y * W + x;
      float* out = semantic_map + 4 * pix;
      const float* pl = eroded + 4 * pix;
      out[0] = pl[0]; out[1] = pl[1]; out[2] = pl[2]; out[3] = pl[3];
      if (pl[0] != 0.0f) continue;
      const float* P = vertex_map + 4 * pix;
      float lp = orc_len3(orc_mk3(P[0], P[1], P[2]));
      int done = 0;
      for (int offset = 1; offset < 3 && !done; ++offset)
        for (int k = 0; k < 4; ++k) {
          int qx = x + dx[k] * offset, qy = y + dy[k] * offset;
          const float* ql = orc_tex_wrapx(eroded, W, H, qx, qy);
          const float* Q = orc_tex_wrapx(vertex_map, W, H, qx, qy);
          float lq = orc_len3(orc_mk3(Q[0], Q[1], Q[2]));
          if (ql[0] != 0.0f && fabsf(lp - lq) < 0.007f * lp) {
            out[0] = ql[0]; out[1] = ql[1]; out[2] = ql[2];
            out[3] = ql[3] / (float)(offset + 1);
            done = 1;
            break;
          }
        }
    }
}

void orc_preprocess(const orc_params* p, const float* pts4, const float* labels, const float* probs, uint32_t n,
                    uint32_t timestamp, float* vertex_map, float* normal_map, float* semantic_map) {
  const size_t P = (size_t)p->data_width * p->data_height;
  float* sem_raw = (float*)malloc(P * 4 * sizeof(float));
  float* eroded = (float*)malloc(P * 4 * sizeof(float));
  orc_k1_project(p, pts4, labels, probs, n, timestamp, vertex_map, sem_raw);
  orc_k2_normals(p, vertex_map, sem_raw, normal_map, eroded);
  orc_k3_floodfill(p, vertex_map, eroded, semantic_map);
  free(sem_raw);
  free(eroded);
}

/* ===================================================================================================
 * K5: Frame2Model_jacobians.geom:67-247, host side Frame2Model.cpp:65-110, 136-261
 * =================================================================================================== */
static inline void orc_tex_border(const float* img, int W, int H, int x, int y, float out[4]) {
  if (x < 0 || x >= W || y < 0 || y >= H) {
    out[0] = out[1] = out[2] = out[3] = 0.0f;
  } else {
    const float* t = img + 4 * ((size_t)y * W + x);
    out[0] = t[0]; out[1] = t[1]; out[2] = t[2]; out[3] = t[3];
  }
}

/* GL_LINEAR on a rectangle texture, CLAMP_TO_BORDER with border (0,0,0,0) (Frame2Model.cpp:102-105):
 * full-precision fp32 weights in the order of the GL spec formula (eq. 8.x): the oracle fixes this rule;
 * hardware uses 8-bit weights. */
static void orc_sample(const float* img, int W, int H, float u, float v, int bilinear, float out[4]) {
  if (!bilinear) {
    orc_tex_border(img, W, H, (int)floorf(u), (int)floorf(v), out);
    return;
  }
  float a = u - 0.5f, b = v - 0.5f;
  float fa = floorf(a), fb = floorf(b);
  int i0 = (int)fa, j0 = (int)fb;
  float al = a - fa, be = b - fb;
  float t00[4], t10[4], t01[4], t11[4];
  orc_tex_border(img, W, H, i0, j0, t00);
  orc_tex_border(img, W, H, i0 + 1, j0, t10);
  orc_tex_border(img, W, H, i0, j0 + 1, t01);
  orc_tex_border(img, W, H, i0 + 1, j0 + 1, t11);
  float w00 = (1.0f - al) * (1.0f - be), w10 = al * (1.0f - be), w01 = (1.0f - al) * be, w11 = al * be;
  for (int c = 0; c < 4; ++c) out[c] = ((w00 * t00[c] + w10 * t10[c]) + w01 * t01[c]) + w11 * t11[c];
}

typedef struct {
  int valid;   /* contributes to n_valid */
  int inlier;
  float t[29]; /* 21 lower-tri JtJ (col-major walk c<=r), 6 Jtf, F, F_inlier */
} orc_k5_terms;

/* one data pixel; returns 0 = invalid, 1 = valid */
static int orc_k5_pixel(const orc_params* p, const float* Mf, const float* data_v, const float* data_n,
                        const float* data_s, const float* model_v, const float* model_n, const float* model_s,
                        int x, int y, int iteration, float distance_thresh, float angle_thresh, orc_k5_terms* o) {
  const int W = p->data_width, Wm = p->model_width, Hm = p->model_height;
  const float fov_up = fabsf(p->data_fov_up), fov_down = fabsf(p->data_fov_down); /* Frame2Model.cpp:82-83 */
  const float fov = fov_up + fov_down;
  size_t pix = (size_t)y * W + x;
  const float* Vd = data_v + 4 * pix;
  const float* Nd = data_n + 4 * pix;
  float e_d = Vd[3] + Nd[3];                                   /* .geom:88 */
  orc_v3 v_d = orc_xform_point(Mf, orc_mk3(Vd[0], Vd[1], Vd[2])); /* :89 */
  orc_v3 n_d = orc_xform_dir(Mf, orc_mk3(Nd[0], Nd[1], Nd[2]));   /* :90 */
  o->valid = 0; o->inlier = 0;
  if (!(e_d > 1.5f)) return 0; /* an invalid data pixel can never pass :105; skip the (NaN) projection */
  /* project2model, .geom:53-65 */
  float depth = orc_len3(v_d);
  float yaw = orc_atan2f(v_d.y, v_d.x);
  float pitch = -orc_asinf(v_d.z / depth);
  float px = 0.5f * ((-yaw * ORC_INV_PI_F) + 1.0f);
  float py = 1.0f - (ORC_RAD2DEG_F * pitch + fov_up) / fov;
  float ix = px * (float)Wm, iy = py * (float)Hm;
  if (!(ix >= 0.0f && ix < (float)Wm && iy >= 0.0f && iy < (float)Hm)) return 0; /* :95-98 (NaN -> invalid) */
  float Vm[4], Nm[4], Sm[4];
  orc_sample(model_v, Wm, Hm, ix, iy, p->bilinear_sampling, Vm);
  orc_sample(model_n, Wm, Hm, ix, iy, p->bilinear_sampling, Nm);
  float e_m = Vm[3] + Nm[3];
  if (!(e_m > 1.5f)) return 0; /* :105 */
  orc_v3 v_m = orc_mk3(Vm[0], Vm[1], Vm[2]), n_m = orc_mk3(Nm[0], Nm[1], Nm[2]);
  int inlier = 1;
  if (orc_len3(orc_sub3(v_m, v_d)) > distance_thresh) inlier = 0; /* :111 */
  if (orc_dot3(n_m, n_d) < angle_thresh) inlier = 0;              /* :112 */
  float residual = orc_dot3(n_m, orc_sub3(v_d, v_m));             /* :114 */
  orc_v3 cp = orc_cross3(v_d, n_m);                               /* :116 */
  float weight = 1.0f;
  if (p->weighting == 4 || p->weighting == 1) { /* huber :120-127 */
    if (fabsf(residual) > p->factor) weight = p->factor / fabsf(residual);
  } else if (p->weighting == 2 && iteration > 0) { /* turkey :128-141 */
    if (fabsf(residual) > p->factor) {
      weight = 0.0f;
    } else {
      float alpha = residual / p->factor;
      weight = 1.0f - alpha * alpha;
      weight = weight * weight;
    }
  }
  /* semantic weighting :144-158 */
  if (data_s && model_s) {
    orc_sample(model_s, Wm, Hm, ix, iy, p->bilinear_sampling, Sm);
    const float* Sd = data_s + 4 * pix;
    float data_label = Sd[0] * 255.0f, data_prob = Sd[3], model_label = Sm[0] * 255.0f;
    if (orc_is_movable(model_label)) {
      if (orc_roundf(data_label) != orc_roundf(model_label))
        weight = weight * (1.0f - data_prob);
      else
        weight = weight * data_prob;
    }
  }
  float J[6] = {n_m.x, n_m.y, n_m.z, cp.x, cp.y, cp.z};
  int k = 0;
  /* temp[c] += weight * J_c * J  (:163-175): entry (r,c) = (weight*J_c)*J_r ; lower triangle r >= c */
  for (int c = 0; c < 6; ++c) {
    float wc = weight * J[c];
    for (int r = c; r < 6; ++r) o->t[k++] = wc * J[r];
  }
  float wr = weight * residual;
  for (int r = 0; r < 6; ++r) o->t[k++] = wr * J[r]; /* :179-181 */
  o->t[27] = wr * residual;                          /* :184 / :193 */
  o->t[28] = inlier ? wr * residual : 0.0f;          /* :186 */
  o->valid = 1;
  o->inlier = inlier;
  return 1;
}

static void orc_k5_thresholds(float max_distance, float max_angle_deg, float* dthr, float* athr) {
  *athr = (float)cos((double)max_angle_deg * 3.14159265358979323846 / 180.0); /* Frame2Model.cpp:66, Math.h:44-47 */
  *dthr = max_distance;
}

void orc_icp_unpack(const int64_t raw[32], double out48[48]) {
  const double s = 1.0 / 1073741824.0;
  int k = 0;
  for (int c = 0; c < 6; ++c)
    for (int r = c; r < 6; ++r) {
      double v = (double)raw[k++] * s;
      out48[c * 6 + r] = v;
      out48[r * 6 + c] = v;
    }
  for (int r = 0; r < 6; ++r) out48[36 + r] = (double)raw[k++] * s;
  out48[42] = (double)raw[29];     /* n_valid */
  out48[43] = (double)raw[27] * s; /* F */
  out48[44] = (double)raw[30];     /* n_outlier */
  out48[45] = (double)raw[28] * s; /* F inlier */
  out48[46] = (double)raw[31];     /* n_invalid */
  out48[47] = 0.0;
}

/* Summation mode of the 48 values. 0 (default): exact Q33.30 fixed-point sums -- the contract of the CUDA path.
 * 1: the reference's own accumulation (fp32 partial sums of 64 pixels in the geometry shader, fp32 ROP adds in primitive
 * order = orc_icp_jacobian_fp32gl), so that whole runs can be compared bit for bit with the reference's classes running
 * on the software GL (oracle/_ref/libsuma_ref_full.so). Test infrastructure only. */
static int orc_gl_sums_ = 0;
int orc_set_gl_sums(int on) {
  int old = orc_gl_sums_;
  orc_gl_sums_ = on ? 1 : 0;
  return old;
}

void orc_icp_jacobian(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                      const float* model_v, const float* model_n, const float* model_s, const double pose[16],
                      int32_t iteration, float max_distance, float max_angle_deg, int32_t row_begin,
                      int32_t row_end, double out48[48], int64_t raw32[32]) {
  if (orc_gl_sums_ && row_begin == 0 && row_end == p->data_height) {
    float f48[48];
    orc_icp_jacobian_fp32gl(p, data_v, data_n, data_s, model_v, model_n, model_s, pose, iteration, max_distance,
                            max_angle_deg, f48);
    if (out48)
      for (int i = 0; i < 48; ++i) out48[i] = (double)f48[i];
    if (raw32) memset(raw32, 0, 32 * sizeof(int64_t));
    return;
  }
  float Mf[16];
  for (int i = 0; i < 16; ++i) Mf[i] = (float)pose[i]; /* pose_.cast<float>(), Frame2Model.cpp:194 */
  float dthr, athr;
  orc_k5_thresholds(max_distance, max_angle_deg, &dthr, &athr);
  int64_t acc[32];
  memset(acc, 0, sizeof(acc));
  const int W = p->data_width;
  /* integer (Q33.30) sums: the reduction order does not matter */
#pragma omp parallel for collapse(2) schedule(static) reduction(+ : acc[:32]) num_threads(orc_threads())
  for (int y = row_begin; y < row_end; ++y)
    for (int x = 0; x < W; ++x) {
      orc_k5_terms t;
      if (!orc_k5_pixel(p, Mf, data_v, data_n, data_s, model_v, model_n, model_s, x, y, iteration, dthr, athr, &t)) {
        acc[31] += 1; /* invalid, .geom:198 */
        continue;
      }
      acc[29] += 1; /* n_valid */
      if (t.inlier) {
        for (int k = 0; k < 27; ++k) acc[k] += orc_fix30(t.t[k]);
        acc[28] += orc_fix30(t.t[28]);
      } else {
        acc[30] += 1; /* outlier */
      }
      acc[27] += orc_fix30(t.t[27]);
    }
  if (raw32) memcpy(raw32, acc, sizeof(acc));
  if (out48) orc_icp_unpack(acc, out48);
}

/* The reference's own accumulation: the geometry shader sums entries_per_kernel = 64 pixels of one row in fp32
 * (Frame2Model.cpp:26-30, .geom:81) and the ROP adds those partial sums in an unspecified order; here: row-major
 * over the vertex buffer order (x-block outer, row inner). */
void orc_icp_jacobian_fp32gl(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                             const float* model_v, const float* model_n, const float* model_s,
                             const double pose[16], int32_t iteration, float max_distance, float max_angle_deg,
                             float out48[48]) {
  float Mf[16];
  for (int i = 0; i < 16; ++i) Mf[i] = (float)pose[i];
  float dthr, athr;
  orc_k5_thresholds(max_distance, max_angle_deg, &dthr, &athr);
  const int W = p->data_width, H = p->data_height;
  float tot[32];
  memset(tot, 0, sizeof(tot));
  orc_k5_terms t;
  for (int xb = 0; xb < W; xb += 64)
    for (int y = 0; y < H; ++y) {
      float part[32];
      memset(part, 0, sizeof(part));
      for (int e = 0; e < 64; ++e) {
        int x = xb + e;
        if (x >= W) continue;
        if (!orc_k5_pixel(p, Mf, data_v, data_n, data_s, model_v, model_n, model_s, x, y, iteration, dthr, athr,
                          &t)) {
          part[31] += 1.0f;
          continue;
        }
        part[29] += 1.0f;
        if (t.inlier) {
          for (int k = 0; k < 27; ++k) part[k] += t.t[k];
          part[28] += t.t[28];
        } else {
          part[30] += 1.0f;
        }
        part[27] += t.t[27];
      }
      for (int k = 0; k < 32; ++k) tot[k] += part[k];
    }
  int k = 0;
  for (int c = 0; c < 6; ++c)
    for (int r = c; r < 6; ++r) {
      out48[c * 6 + r] = tot[k];
      out48[r * 6 + c] = tot[k];
      ++k;
    }
  for (int r = 0; r < 6; ++r) out48[36 + r] = tot[k++];
  out48[42] = tot[29]; out48[43] = tot[27]; out48[44] = tot[30]; out48[45] = tot[28]; out48[46] = tot[31];
  out48[47] = 0.0f;
}

/* ===================================================================================================
 * SE3 exp/log (lie_algebra.cpp:4-71), 6x6 LDLT, Gauss-Newton step (LieGaussNewton.cpp:53-79)
 * =================================================================================================== */
void orc_se3_exp(const double x[6], double T[16]) {
  for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  const double v[3] = {x[0], x[1], x[2]}, w[3] = {x[3], x[4], x[5]};
  double theta = sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]);
  if (theta > 1e-10) {
    /* K = skew(w) (row-major here), K2 = K*K */
    double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    double K2[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) K2[r * 3 + c] = (K[r * 3 + 0] * K[0 * 3 + c] + K[r * 3 + 1] * K[1 * 3 + c]) + K[r * 3 + 2] * K[2 * 3 + c];
    double s, c;
    orc_sincos(theta, &s, &c);
    double alpha = s / theta;
    double beta = (1.0 - c) / (theta * theta);
    double gamma = beta; /* lie_algebra.cpp:24: (1.0f - cos)/theta^2 */
    double delta = (theta - s) / ((theta * theta) * theta);
    double V[9];
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc) {
        double I = (r == cc) ? 1.0 : 0.0;
        T[cc * 4 + r] = (I + alpha * K[r * 3 + cc]) + beta * K2[r * 3 + cc];
        V[r * 3 + cc] = (I + gamma * K[r * 3 + cc]) + delta * K2[r * 3 + cc];
      }
    for (int r = 0; r < 3; ++r) T[12 + r] = (V[r * 3 + 0] * v[0] + V[r * 3 + 1] * v[1]) + V[r * 3 + 2] * v[2];
  } else {
    T[12] = v[0]; T[13] = v[1]; T[14] = v[2];
  }
}

void orc_se3_log(const double M[16], double x[6]) {
  for (int i = 0; i < 6; ++i) x[i] = 0.0;
  double d = 0.5 * (((M[0] + M[5]) + M[10]) - 1.0);
  double K[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; /* row-major omega_skew */
  if (d < 1 - 1e-10) {
    double theta = acos(d);
    double f = theta / (2 * sin(theta));
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) K[r * 3 + c] = f * (M[c * 4 + r] - M[r * 4 + c]);
    x[3] = K[2 * 3 + 1]; x[4] = K[0 * 3 + 2]; x[5] = K[1 * 3 + 0];
  }
  double theta = sqrt((x[3] * x[3] + x[4] * x[4]) + x[5] * x[5]);
  x[0] = M[12]; x[1] = M[13]; x[2] = M[14];
  if (fabs(theta) > 1e-10) {
    double half = 0.5 * theta;
    double beta = 1 / (theta * theta) * (1 - theta * cos(half) / (2 * sin(half)));
    double K2[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) K2[r * 3 + c] = (K[r * 3 + 0] * K[0 * 3 + c] + K[r * 3 + 1] * K[1 * 3 + c]) + K[r * 3 + 2] * K[2 * 3 + c];
    double t[3] = {M[12], M[13], M[14]};
    for (int r = 0; r < 3; ++r) {
      double acc = 0;
      for (int c = 0; c < 3; ++c) {
        double Vi = ((r == c ? 1.0 : 0.0) + (-0.5) * K[r * 3 + c]) + beta * K2[r * 3 + c];
        acc += Vi * t[c];
      }
      x[r] = acc;
    }
  }
}

/* LDL^T with symmetric (diagonal) pivoting, reading the lower triangle -- the algorithm family of
 * Eigen::LDLT used at LieGaussNewton.cpp:60; evaluation order fixed here. A is column-major 6x6. */
int orc_ldlt_solve6(const double Ain[36], const double bin[6], double x[6]) {
  double A[36];
  int perm[6];
  for (int c = 0; c < 6; ++c)
    for (int r = 0; r < 6; ++r) A[c * 6 + r] = (r >= c) ? Ain[c * 6 + r] : Ain[r * 6 + c]; /* symmetrize from lower */
  for (int i = 0; i < 6; ++i) perm[i] = i;
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double best = fabs(A[k * 6 + k]);
    for (int i = k + 1; i < 6; ++i) {
      double v = fabs(A[i * 6 + i]);
      if (v > best) { best = v; piv = i; }
    }
    if (piv != k) { /* symmetric row/column swap of the full matrix */
      for (int i = 0; i < 6; ++i) { double t = A[k * 6 + i]; A[k * 6 + i] = A[piv * 6 + i]; A[piv * 6 + i] = t; }
      for (int i = 0; i < 6; ++i) { double t = A[i * 6 + k]; A[i * 6 + k] = A[i * 6 + piv]; A[i * 6 + piv] = t; }
      int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
    }
    double dk = A[k * 6 + k];
    if (dk == 0.0) continue; /* leaves zeros: solution component becomes 0 (Eigen does the same for exact 0 pivots) */
    for (int i = k + 1; i < 6; ++i) A[k * 6 + i] = A[k * 6 + i] / dk; /* L(i,k) stored at column k, row i */
    for (int j = k + 1; j < 6; ++j)
      for (int i = j; i < 6; ++i) {
        A[j * 6 + i] = A[j * 6 + i] - (A[k * 6 + i] * dk) * A[k * 6 + j];
        A[i * 6 + j] = A[j * 6 + i];
      }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) y[i] = bin[perm[i]];
  for (int i = 0; i < 6; ++i)
    for (int k = 0; k < i; ++k) y[i] = y[i] - A[k * 6 + i] * y[k];
  for (int i = 0; i < 6; ++i) y[i] = (A[i * 6 + i] == 0.0) ? 0.0 : y[i] / A[i * 6 + i];
  for (int i = 5; i >= 0; --i)
    for (int k = i + 1; k < 6; ++k) y[i] = y[i] - A[i * 6 + k] * y[k];
  for (int i = 0; i < 6; ++i) x[perm[i]] = y[i];
  return 0;
}

int orc_gn_step(const double out48[48], double last_error, double eps, double delta_thr, double pose[16],
                double dx[6]) {
  int result = 1;
  double current_error = out48[43];
  double nb[6];
  for (int i = 0; i < 6; ++i) nb[i] = -out48[36 + i];
  orc_ldlt_solve6(out48, nb, dx);
  double linf = 0.0, maxc = out48[36];
  for (int i = 0; i < 6; ++i) {
    if (fabs(dx[i]) > linf) linf = fabs(dx[i]);
    if (out48[36 + i] > maxc) maxc = out48[36 + i];
  }
  if (linf < delta_thr) result = 0;                                                     /* LieGaussNewton.cpp:64 */
  if (fabs(maxc) < eps) result = 0;                                                     /* :65 */
  if (current_error < last_error && fabs(current_error - last_error) < eps) result = 0; /* :66 */
  double E[16], Pn[16];
  orc_se3_exp(dx, E);
  orc_mat4_mul_d(E, pose, Pn); /* Objective.h:46 */
  memcpy(pose, Pn, sizeof(Pn));
  return result;
}

int orc_icp_minimize(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                     const float* model_v, const float* model_n, const float* model_s, const double T0[16],
                     float max_distance, float max_angle_deg, double pose_out[16], double out48[48],
                     double* history, int32_t* history_len) {
  double pose[16], o48[48], dx[6];
  memcpy(pose, T0, sizeof(pose));
  memset(o48, 0, sizeof(o48));
  double last_error = (double)3.402823466e+38f; /* numeric_limits<float>::max(), LieGaussNewton.cpp:48 */
  int k = 0, hl = 0;
  const int maxIter = p->max_iterations;
  for (;;) {
    if (history) memcpy(history + 16 * hl, pose, sizeof(pose));
    ++hl;
    if (maxIter > 0 && k >= maxIter) break; /* LieGaussNewton.cpp:27 */
    orc_icp_jacobian(p, data_v, data_n, data_s, model_v, model_n, model_s, pose, k, max_distance, max_angle_deg, 0,
                     p->data_height, o48, NULL);
    int result = orc_gn_step(o48, last_error, p->stopping_threshold, p->delta, pose, dx);
    last_error = o48[43];
    if (result == 0) break;
    ++k;
  }
  memcpy(pose_out, pose, sizeof(pose));
  if (out48) memcpy(out48, o48, sizeof(o48));
  if (history_len) *history_len = hl;
  return k;
}
