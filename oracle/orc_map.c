/* orc_map.c -- TEST INFRASTRUCTURE (CPU oracle): SurfelMap render (K4/K4b), update (K6a-e), submap paging.
 * Follows core/SurfelMap.cpp and shader/{render_surfels,render_compose,gen_indexmap,init_radiusConf,
 * update_surfels,gen_surfels,copy_surfels,extract_surfels}.*  (paths relative to /root/reference/src). */
#include "orc.h"
#include "orc_internal.h"

#include <stdio.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_MAX_SURFELS (2048u * 2048u) /* SurfelMap.h:87 */
#define ORC_MAX_POSES 10000u            /* SurfelMap.h:205 */
#define ORC_EXTRACT_CAP 500000u         /* SurfelMap.cpp:279 */
#define ORC_COMPOSE_AGE 100u            /* SurfelMap.h:144 */

typedef struct { float *v, *n, *s; } orc_frame;

typedef struct { int32_t i, j; orc_surfel* surfels; uint32_t n; } orc_tile;

struct orc_map {
  orc_params p;
  uint32_t timestamp;
  orc_surfel* surfels; /* surfels_ */
  uint32_t n;
  orc_surfel* scratch; /* updated_surfels_ | data_surfels_ */
  float* poses;        /* poseBuffer_, MAX_POSES x 16 col-major */
  float* poses_inv;
  orc_frame oldf, newf, compf;
  uint32_t* rdepth; /* render depth buffer (model size) */
  /* update intermediates */
  uint32_t* idepth;
  uint32_t* index_map; /* id+1, 0 = empty (gen_indexmap.vert:79) */
  float* radius_map;   /* (radius, 0, 0, valid) */
  uint8_t* integrated;
  uint32_t n_updated, n_new;
  /* submaps (SurfelMap.h:186-203) */
  int32_t origin_i, origin_j;
  int32_t* extraction; /* pairs */
  uint32_t n_extraction, cap_extraction;
  orc_tile* tiles;
  uint32_t n_tiles, cap_tiles;
  /* per-thread raster targets + chunk bookkeeping of the multi-threaded passes (see render_pass / chunked_compact) */
  int mt_threads;
  size_t mt_pixels;
  uint32_t** mt_depth;
  uint32_t** mt_index;
  orc_frame* mt_frame;
  orc_surfel* scratch2;
  /* derived parameters (SurfelMap.cpp:336-457) */
  float pixel_size, p_unstable, log_prior, log_unstable, radconf_angle_thresh, update_angle_thresh;
};

static void frame_alloc(orc_frame* f, size_t P) {
  f->v = (float*)calloc(P * 4, sizeof(float));
  f->n = (float*)calloc(P * 4, sizeof(float));
  f->s = (float*)calloc(P * 4, sizeof(float));
}
static void frame_free(orc_frame* f) { free(f->v); free(f->n); free(f->s); }
static void frame_clear(orc_frame* f, size_t P) {
#pragma omp parallel for schedule(static) num_threads(orc_threads())
  for (size_t r = 0; r < 64; ++r) {
    size_t b = P * 16 * r / 64, e = P * 16 * (r + 1) / 64;
    memset((char*)f->v + b, 0, e - b); memset((char*)f->n + b, 0, e - b); memset((char*)f->s + b, 0, e - b);
  }
}

static float deg2rad_f(float d) { return d * (float)(3.14159265358979323846 / 180.0); }

static void orc_map_derive(orc_map* m) {
  const orc_params* p = &m->p;
  /* SurfelMap.cpp:339-344 */
  float vfov = fabsf(p->data_fov_up) + fabsf(p->data_fov_down);
  float hfov = 360.0f;
  float vpix = (float)tan(0.5f * ((double)vfov * 3.14159265358979323846 / 180.0) / (uint32_t)p->data_height);
  float hpix = (float)tan(0.5f * ((double)hfov * 3.14159265358979323846 / 180.0) / (uint32_t)p->data_width);
  m->pixel_size = vpix > hpix ? vpix : hpix;
  m->p_unstable = 1.0f - p->p_stable;                                    /* :347 */
  m->log_prior = (float)log(p->p_prior / (1.0 - p->p_prior));            /* :349 */
  m->log_unstable = (float)log(m->p_unstable / (1.0 - m->p_unstable));   /* :350 */
  m->radconf_angle_thresh = (float)cos((double)deg2rad_f(p->max_angle)); /* :395 */
  m->update_angle_thresh = (float)sin((double)deg2rad_f(p->map_max_angle)); /* :407 */
}

orc_map* orc_map_create(const orc_params* p) {
  if (orc_check_params(p)) return NULL;
  orc_map* m = (orc_map*)calloc(1, sizeof(orc_map));
  m->p = *p;
  size_t Pm = (size_t)p->model_width * p->model_height, Pd = (size_t)p->data_width * p->data_height;
  m->surfels = (orc_surfel*)malloc(sizeof(orc_surfel) * ORC_MAX_SURFELS);
  m->scratch = (orc_surfel*)malloc(sizeof(orc_surfel) * ORC_MAX_SURFELS);
  m->poses = (float*)malloc(sizeof(float) * 16 * ORC_MAX_POSES);
  m->poses_inv = (float*)malloc(sizeof(float) * 16 * ORC_MAX_POSES);
  frame_alloc(&m->oldf, Pm); frame_alloc(&m->newf, Pm); frame_alloc(&m->compf, Pm);
  m->rdepth = (uint32_t*)malloc(Pm * 4);
  m->idepth = (uint32_t*)malloc(Pd * 4);
  m->index_map = (uint32_t*)calloc(Pd, 4);
  m->radius_map = (float*)calloc(Pd * 4, 4);
  m->integrated = (uint8_t*)calloc(Pd, 1);
  orc_map_derive(m);
  orc_map_reset(m);
  return m;
}

static void tiles_clear(orc_map* m) {
  for (uint32_t t = 0; t < m->n_tiles; ++t) free(m->tiles[t].surfels);
  m->n_tiles = 0;
}

void orc_map_destroy(orc_map* m) {
  if (!m) return;
  tiles_clear(m);
  free(m->tiles); free(m->extraction);
  free(m->surfels); free(m->scratch); free(m->poses); free(m->poses_inv);
  frame_free(&m->oldf); frame_free(&m->newf); frame_free(&m->compf);
  free(m->rdepth); free(m->idepth); free(m->index_map); free(m->radius_map); free(m->integrated);
  for (int t = 0; t < m->mt_threads; ++t) { free(m->mt_depth[t]); free(m->mt_index[t]); frame_free(&m->mt_frame[t]); }
  free(m->mt_depth); free(m->mt_index); free(m->mt_frame); free(m->scratch2);
  free(m);
}

/* SurfelMap::reset, SurfelMap.cpp:473-482 */
void orc_map_reset(orc_map* m) {
  m->n = 0;
  m->timestamp = 0;
  m->origin_i = m->origin_j = 0;
  m->n_extraction = 0;
  tiles_clear(m);
  for (uint32_t t = 0; t < ORC_MAX_POSES; ++t)
    for (int i = 0; i < 16; ++i) {
      m->poses[16 * t + i] = (i % 5 == 0) ? 1.0f : 0.0f;
      m->poses_inv[16 * t + i] = (i % 5 == 0) ? 1.0f : 0.0f;
    }
}

uint32_t orc_map_size(const orc_map* m) { return m->n; }
uint32_t orc_map_timestamp(const orc_map* m) { return m->timestamp; }
uint32_t orc_map_download(const orc_map* m, orc_surfel* dst, uint32_t cap) {
  uint32_t k = m->n < cap ? m->n : cap;
  memcpy(dst, m->surfels, sizeof(orc_surfel) * k);
  return k;
}
void orc_map_upload(orc_map* m, const orc_surfel* src, uint32_t n, uint32_t timestamp) {
  if (n > ORC_MAX_SURFELS) n = ORC_MAX_SURFELS;
  memcpy(m->surfels, src, sizeof(orc_surfel) * n);
  m->n = n;
  m->timestamp = timestamp;
}
void orc_map_set_pose(orc_map* m, uint32_t t, const float pose[16]) {
  if (t >= ORC_MAX_POSES) return;
  memcpy(m->poses + 16 * t, pose, 64);
  orc_rigid_inverse_f(pose, m->poses_inv + 16 * t);
}
void orc_map_update_poses(orc_map* m, const float* poses16, uint32_t count) {
  for (uint32_t t = 0; t < count && t < ORC_MAX_POSES; ++t) orc_map_set_pose(m, t, poses16 + 16 * t);
}
void orc_map_get_frame(const orc_map* m, int which, float* v, float* n, float* s) {
  const orc_frame* f = which == 0 ? &m->oldf : (which == 1 ? &m->newf : &m->compf);
  size_t B = (size_t)m->p.model_width * m->p.model_height * 16;
  if (v) memcpy(v, f->v, B);
  if (n) memcpy(n, f->n, B);
  if (s) memcpy(s, f->s, B);
}
void orc_map_get_update_debug(const orc_map* m, uint32_t* index_map, float* radius_map, uint8_t* integrated,
                              uint32_t* n_updated, uint32_t* n_new) {
  size_t Pd = (size_t)m->p.data_width * m->p.data_height;
  if (index_map) memcpy(index_map, m->index_map, Pd * 4);
  if (radius_map) memcpy(radius_map, m->radius_map, Pd * 16);
  if (integrated) memcpy(integrated, m->integrated, Pd);
  if (n_updated) *n_updated = m->n_updated;
  if (n_new) *n_new = m->n_new;
}
void orc_map_get_submap_origin(const orc_map* m, int32_t* i, int32_t* j, uint32_t* pending) {
  if (i) *i = m->origin_i;
  if (j) *j = m->origin_j;
  if (pending) *pending = m->n_extraction;
}

static inline int surfel_pose_index(const orc_surfel* s) {
  int c = (int)s->count;
  if (c < 0) c = 0;
  if (c >= (int)ORC_MAX_POSES) c = ORC_MAX_POSES - 1;
  return c;
}

/* ===================================================================================================
 * K4: render_surfels.{vert,geom,frag}. GL rules fixed by the oracle: vertices snapped to 1/256 pixel, pixel-centre
 * sampling, exact integer edge functions with a consistent tie rule, barycentric attribute interpolation in fp32,
 * primitive clipped to 0 <= z_window <= 1, 24-bit depth, GL_LESS (or GL_LEQUAL), primitives in buffer order.
 * =================================================================================================== */
typedef struct { int64_t X, Y; float z, tx, ty; } orc_rvert;

static inline int64_t floor_div(int64_t a, int64_t b) { int64_t q = a / b, r = a % b; return (r != 0 && ((r < 0) != (b < 0))) ? q - 1 : q; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return -floor_div(-a, b); }
static inline int64_t edge_fn(const orc_rvert* P, const orc_rvert* Q, int64_t X, int64_t Y) {
  return (Q->X - P->X) * (Y - P->Y) - (Q->Y - P->Y) * (X - P->X);
}
static inline int edge_in(int64_t w, const orc_rvert* P, const orc_rvert* Q) {
  if (w > 0) return 1;
  if (w < 0) return 0;
  int64_t dx = Q->X - P->X, dy = Q->Y - P->Y;
  return dy > 0 || (dy == 0 && dx > 0);
}

typedef struct {
  orc_map* m;
  uint32_t* depth;
  orc_frame* out;
  int lequal;
  orc_v3 p, n;       /* flat attributes (.geom:95-99): surfel centre, normal */
  const float* sem;  /* surfel semantic vec4 */
} orc_rctx;

static void raster_tri(orc_rctx* rc, orc_rvert A, orc_rvert B, orc_rvert C) {
  const int W = rc->m->p.model_width, H = rc->m->p.model_height;
  int64_t area = (B.X - A.X) * (C.Y - A.Y) - (B.Y - A.Y) * (C.X - A.X);
  if (area == 0) return;
  if (area < 0) { orc_rvert t = B; B = C; C = t; area = -area; }
  int64_t minX = A.X < B.X ? A.X : B.X; if (C.X < minX) minX = C.X;
  int64_t maxX = A.X > B.X ? A.X : B.X; if (C.X > maxX) maxX = C.X;
  int64_t minY = A.Y < B.Y ? A.Y : B.Y; if (C.Y < minY) minY = C.Y;
  int64_t maxY = A.Y > B.Y ? A.Y : B.Y; if (C.Y > maxY) maxY = C.Y;
  int64_t i0 = ceil_div(minX - 128, 256), i1 = floor_div(maxX - 128, 256);
  int64_t j0 = ceil_div(minY - 128, 256), j1 = floor_div(maxY - 128, 256);
  if (i0 < 0) i0 = 0; if (j0 < 0) j0 = 0;
  if (i1 > W - 1) i1 = W - 1; if (j1 > H - 1) j1 = H - 1;
  float farea = (float)area;
  for (int64_t j = j0; j <= j1; ++j)
    for (int64_t i = i0; i <= i1; ++i) {
      int64_t X = i * 256 + 128, Y = j * 256 + 128;
      int64_t wA = edge_fn(&B, &C, X, Y), wB = edge_fn(&C, &A, X, Y), wC = edge_fn(&A, &B, X, Y);
      if (!edge_in(wA, &B, &C) || !edge_in(wB, &C, &A) || !edge_in(wC, &A, &B)) continue;
      float fB = (float)wB / farea, fC = (float)wC / farea;
      float fA = (1.0f - fB) - fC;
      float tx = (fA * A.tx + fB * B.tx) + fC * C.tx;
      float ty = (fA * A.ty + fB * B.ty) + fC * C.ty;
      if (tx * tx + ty * ty > 1.0f) continue; /* render_surfels.frag:22-28 */
      float z = (fA * A.z + fB * B.z) + fC * C.z;
      if (!(z >= 0.0f && z <= 1.0f)) continue; /* near/far clip */
      uint32_t d24 = orc_depth24(z);
      size_t pix = (size_t)j * W + (size_t)i;
      if (rc->lequal ? (d24 <= rc->depth[pix]) : (d24 < rc->depth[pix])) {
        rc->depth[pix] = d24;
        float* v = rc->out->v + 4 * pix; float* n = rc->out->n + 4 * pix; float* s = rc->out->s + 4 * pix;
        v[0] = rc->p.x; v[1] = rc->p.y; v[2] = rc->p.z; v[3] = 1.0f; /* .frag:30 */
        n[0] = rc->n.x; n[1] = rc->n.y; n[2] = rc->n.z; n[3] = 1.0f; /* .geom:97 */
        s[0] = rc->sem[0]; s[1] = rc->sem[1]; s[2] = rc->sem[2]; s[3] = rc->sem[3];
      }
    }
}

/* one glDrawArrays(GL_POINTS, surfels_) with the render program */
static void render_range(orc_map* m, uint32_t k_begin, uint32_t k_end, const float inv_pose[16], float conf_thr,
                         int t_thr, int render_old, int lequal, uint32_t* depth, orc_frame* out) {
  const orc_params* p = &m->p;
  const int W = p->model_width, H = p->model_height;
  const float fov_up = fabsf(p->model_fov_up), fov = fabsf(p->model_fov_up) + fabsf(p->model_fov_down);
  const float mind = p->model_min_depth, maxd = p->model_max_depth;
  orc_rctx rc;
  rc.m = m; rc.depth = depth; rc.out = out; rc.lequal = lequal;
  for (uint32_t k = k_begin; k < k_end; ++k) {
    const orc_surfel* s = &m->surfels[k];
    int c = surfel_pose_index(s);
    float T[16];
    orc_mat4_mul_f(inv_pose, m->poses + 16 * c, T); /* render_surfels.vert:46: (inv_pose * surfelPose) * v */
    orc_v3 pp = orc_xform_point(T, orc_mk3(s->x, s->y, s->z));
    orc_v3 nn = orc_xform_dir(T, orc_mk3(s->nx, s->ny, s->nz));
    float r = s->radius;
    int visible = orc_dot3(nn, orc_divs3(orc_neg3(pp), orc_len3(pp))) > 0.01f; /* .geom:84 */
    float cx, cy, cz;
    orc_project01(pp, fov_up, fov, mind, maxd, &cx, &cy, &cz);
    if (!(visible && cx >= 0.0f && cy >= 0.0f && cz >= 0.0f && cx < 1.0f && cy < 1.0f && cz < 1.0f)) continue;
    if (!(!p->use_stability || s->confidence > conf_thr)) continue; /* .geom:87 */
    int creation = (int)s->count, ts = (int)s->timestamp;
    int valid = render_old && (creation < t_thr);
    valid = valid || (!render_old && (creation >= t_thr || ts >= t_thr)); /* .geom:90-91 */
    if (!valid) continue;
    orc_v3 u = orc_normalize3(orc_mk3(nn.y - nn.z, -nn.x, nn.x)); /* .geom:80 */
    orc_v3 v = orc_normalize3(orc_cross3(nn, u));                 /* .geom:81 */
    orc_v3 ru = orc_scale3(r, u), rv = orc_scale3(r, v);
    orc_v3 corner[4];
    corner[0] = orc_sub3(orc_sub3(pp, ru), rv);
    corner[1] = orc_sub3(orc_add3(pp, ru), rv);
    corner[2] = orc_add3(orc_sub3(pp, ru), rv);
    corner[3] = orc_add3(orc_add3(pp, ru), rv);
    static const float tcx[4] = {-1.0f, 1.0f, -1.0f, 1.0f}, tcy[4] = {-1.0f, -1.0f, 1.0f, 1.0f};
    orc_rvert q[4];
    for (int i = 0; i < 4; ++i) {
      float x, y, z;
      orc_project01(corner[i], fov_up, fov, mind, maxd, &x, &y, &z);
      if (cx - x > 0.5f) x += 1.0f; /* .geom:68 */
      if (x - cx > 0.5f) x -= 1.0f; /* .geom:69 */
      /* gl_Position = 2*proj - 1; viewport: window = (ndc*0.5 + 0.5) * size */
      float xw = (0.5f * (2.0f * x - 1.0f) + 0.5f) * (float)W;
      float yw = (0.5f * (2.0f * y - 1.0f) + 0.5f) * (float)H;
      q[i].z = 0.5f * (2.0f * z - 1.0f) + 0.5f;
      q[i].X = (int64_t)llrintf(xw * 256.0f);
      q[i].Y = (int64_t)llrintf(yw * 256.0f);
      q[i].tx = tcx[i]; q[i].ty = tcy[i];
    }
    rc.p = pp; rc.n = nn; rc.sem = &s->r;
    raster_tri(&rc, q[0], q[1], q[2]);
    raster_tri(&rc, q[1], q[2], q[3]);
  }
}

static void depth_clear(uint32_t* d, size_t P) { for (size_t i = 0; i < P; ++i) d[i] = ORC_DEPTH_CLEAR; }

/* per-thread raster targets, (re)allocated for the larger of the two image sizes */
static void mt_prepare(orc_map* m, int T) {
  size_t Pm = (size_t)m->p.model_width * m->p.model_height, Pd = (size_t)m->p.data_width * m->p.data_height;
  size_t P = Pm > Pd ? Pm : Pd;
  if (m->mt_threads >= T && m->mt_pixels >= P) return;
  for (int t = 0; t < m->mt_threads; ++t) { free(m->mt_depth[t]); free(m->mt_index[t]); frame_free(&m->mt_frame[t]); }
  free(m->mt_depth); free(m->mt_index); free(m->mt_frame);
  m->mt_depth = (uint32_t**)calloc((size_t)T, sizeof(uint32_t*));
  m->mt_index = (uint32_t**)calloc((size_t)T, sizeof(uint32_t*));
  m->mt_frame = (orc_frame*)calloc((size_t)T, sizeof(orc_frame));
  for (int t = 0; t < T; ++t) {
    m->mt_depth[t] = (uint32_t*)malloc(P * 4);
    m->mt_index[t] = (uint32_t*)malloc(P * 4);
    frame_alloc(&m->mt_frame[t], P);
  }
  m->mt_threads = T;
  m->mt_pixels = P;
}
static inline void chunk_of(uint32_t n, int T, int t, uint32_t* b, uint32_t* e) {
  *b = (uint32_t)(((uint64_t)n * (uint64_t)t) / (uint64_t)T);
  *e = (uint32_t)(((uint64_t)n * (uint64_t)(t + 1)) / (uint64_t)T);
}

/* One draw call. With T host threads the surfel buffer is cut into T contiguous chunks; every chunk is rasterised in
 * buffer order into its own depth/attribute target (cleared above every 24-bit depth), and the targets are merged into
 * the real one in chunk order with the SAME depth comparison. Because "first (GL_LESS) / last (GL_LEQUAL) fragment of
 * minimal depth in buffer order" is associative over contiguous chunks, the result is the sequential one bit for bit. */
static void render_pass(orc_map* m, const float inv_pose[16], float conf_thr, int t_thr, int render_old, int lequal,
                        uint32_t* depth, orc_frame* out) {
  const int T = orc_threads();
  if (T <= 1 || m->n < 4096u) {
    render_range(m, 0, m->n, inv_pose, conf_thr, t_thr, render_old, lequal, depth, out);
    return;
  }
  const size_t P = (size_t)m->p.model_width * m->p.model_height;
  mt_prepare(m, T);
#pragma omp parallel num_threads(T)
  {
#ifdef _OPENMP
    const int t = omp_get_thread_num();
#else
    const int t = 0;
#endif
    uint32_t b, e;
    chunk_of(m->n, T, t, &b, &e);
    memset(m->mt_depth[t], 0xFF, P * 4); /* 0xFFFFFFFF: above every depth24, so "untouched" is recognisable */
    render_range(m, b, e, inv_pose, conf_thr, t_thr, render_old, lequal, m->mt_depth[t], &m->mt_frame[t]);
#pragma omp barrier
#pragma omp for schedule(static)
    for (size_t pix = 0; pix < P; ++pix) {
      for (int c = 0; c < T; ++c) {
        uint32_t d = m->mt_depth[c][pix];
        if (d == 0xFFFFFFFFu) continue;
        if (lequal ? (d <= depth[pix]) : (d < depth[pix])) {
          depth[pix] = d;
          memcpy(out->v + 4 * pix, m->mt_frame[c].v + 4 * pix, 16);
          memcpy(out->n + 4 * pix, m->mt_frame[c].n + 4 * pix, 16);
          memcpy(out->s + 4 * pix, m->mt_frame[c].s + 4 * pix, 16);
        }
      }
    }
  }
}

static int t_threshold(const orc_map* m) { return (int)(m->timestamp - ORC_COMPOSE_AGE); } /* SurfelMap.cpp:873 (Q9) */

/* render_compose.frag:26-48 */
static void compose(const orc_map* m, float* fv, float* fn, float* fs) {
  size_t P = (size_t)m->p.model_width * m->p.model_height;
  const float maxdist = m->p.max_loop_closure_distance;
#pragma omp parallel for schedule(static) num_threads(orc_threads())
  for (size_t i = 0; i < P; ++i) {
    const float* nv = m->newf.v + 4 * i; const float* nn = m->newf.n + 4 * i; const float* ns = m->newf.s + 4 * i;
    const float* ov = m->oldf.v + 4 * i; const float* on = m->oldf.n + 4 * i; const float* os = m->oldf.s + 4 * i;
    int valid = ov[3] > 0.5f && on[3] > 0.5f;
    int new_valid = nv[3] > 0.5f && nn[3] > 0.5f;
    const float *sv = nv, *sn = nn, *ss = ns;
    if (!new_valid && valid &&
        (nv[3] < 0.5f || orc_len3(orc_sub3(orc_mk3(nv[0], nv[1], nv[2]), orc_mk3(ov[0], ov[1], ov[2]))) < maxdist)) {
      sv = ov; sn = on; ss = os;
    }
    memcpy(fv + 4 * i, sv, 16); memcpy(fn + 4 * i, sn, 16); memcpy(fs + 4 * i, ss, 16);
  }
}

void orc_map_render(orc_map* m, const float pose_old[16], const float pose_new[16], float conf_thr, float* fv,
                    float* fn, float* fs) {
  size_t P = (size_t)m->p.model_width * m->p.model_height;
  float inv_old[16], inv_new[16];
  orc_rigid_inverse_f(pose_old, inv_old);
  orc_rigid_inverse_f(pose_new, inv_new);
  if (m->p.compose_rendering) {
    int thr = t_threshold(m);
    frame_clear(&m->oldf, P); depth_clear(m->rdepth, P);
    render_pass(m, inv_old, conf_thr, thr, 1, 0, m->rdepth, &m->oldf); /* SurfelMap.cpp:875-882 */
    frame_clear(&m->newf, P); depth_clear(m->rdepth, P);
    render_pass(m, inv_new, conf_thr, thr, 0, 0, m->rdepth, &m->newf); /* :884-891 */
    frame_clear(&m->compf, P); depth_clear(m->rdepth, P);
    render_pass(m, inv_old, conf_thr, thr, 1, 0, m->rdepth, &m->compf); /* :893-901 */
    render_pass(m, inv_new, conf_thr, thr, 0, 0, m->rdepth, &m->compf); /* :903-906, not cleared */
    compose(m, fv, fn, fs);                                             /* :911-940 */
  } else {
    orc_frame f = {fv, fn, fs};
    frame_clear(&f, P); depth_clear(m->rdepth, P);
    render_pass(m, inv_old, conf_thr, 0, 0, 0, m->rdepth, &f); /* :980-1002 */
    memcpy(m->newf.v, fv, P * 16); memcpy(m->newf.n, fn, P * 16); memcpy(m->newf.s, fs, P * 16); /* :1016-1017 */
    memcpy(m->oldf.v, fv, P * 16); memcpy(m->oldf.n, fn, P * 16); memcpy(m->oldf.s, fs, P * 16);
  }
}

/* Q4: render_active / _inactive / _composed attach COLOR0/1 only; the semantic image keeps its previous content. */
void orc_map_render_active(orc_map* m, const float pose[16], float conf_thr) {
  size_t P = (size_t)m->p.model_width * m->p.model_height;
  float inv[16];
  orc_rigid_inverse_f(pose, inv);
  float* tmp_s = (float*)malloc(P * 16);
  memcpy(tmp_s, m->newf.s, P * 16);
  frame_clear(&m->newf, P); depth_clear(m->rdepth, P);
  render_pass(m, inv, conf_thr, t_threshold(m), 0, 0, m->rdepth, &m->newf);
  memcpy(m->newf.s, tmp_s, P * 16);
  free(tmp_s);
}
void orc_map_render_inactive(orc_map* m, const float pose[16], float conf_thr) {
  size_t P = (size_t)m->p.model_width * m->p.model_height;
  float inv[16];
  orc_rigid_inverse_f(pose, inv);
  float* tmp_s = (float*)malloc(P * 16);
  memcpy(tmp_s, m->oldf.s, P * 16);
  frame_clear(&m->oldf, P); depth_clear(m->rdepth, P);
  render_pass(m, inv, conf_thr, t_threshold(m), 1, 0, m->rdepth, &m->oldf);
  memcpy(m->oldf.s, tmp_s, P * 16);
  free(tmp_s);
}
void orc_map_render_composed(orc_map* m, const float pose_old[16], const float pose_new[16], float conf_thr) {
  size_t P = (size_t)m->p.model_width * m->p.model_height;
  float inv_old[16], inv_new[16];
  orc_rigid_inverse_f(pose_old, inv_old);
  orc_rigid_inverse_f(pose_new, inv_new);
  float* tmp_s = (float*)malloc(P * 16);
  memcpy(tmp_s, m->compf.s, P * 16);
  frame_clear(&m->compf, P); depth_clear(m->rdepth, P);
  render_pass(m, inv_old, conf_thr, t_threshold(m), 1, 1, m->rdepth, &m->compf); /* GL_LEQUAL, SurfelMap.cpp:1126 */
  render_pass(m, inv_new, conf_thr, t_threshold(m), 0, 1, m->rdepth, &m->compf);
  memcpy(m->compf.s, tmp_s, P * 16);
  free(tmp_s);
}

/* ===================================================================================================
 * K6: SurfelMap::update, SurfelMap.cpp:492-584
 * =================================================================================================== */
static inline void data_tex(const float* img, int W, int H, float fx, float fy, float out[4]) {
  /* rectangle texture fetch at a texel centre, CLAMP_TO_BORDER (SurfelMap.cpp:170) */
  if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) {
    out[0] = out[1] = out[2] = out[3] = 0.0f;
    return;
  }
  const float* t = img + 4 * ((size_t)(int)fy * W + (size_t)(int)fx);
  out[0] = t[0]; out[1] = t[1]; out[2] = t[2]; out[3] = t[3];
}

/* K6a gen_indexmap.vert:62-81 */
static void k6a_range(orc_map* m, uint32_t k_begin, uint32_t k_end, const float inv_pose[16], uint32_t* idepth,
                      uint32_t* index_map) {
  const orc_params* p = &m->p;
  const int W = p->data_width, H = p->data_height;
  const float fov_up = fabsf(p->data_fov_up), fov = fabsf(p->data_fov_up) + fabsf(p->data_fov_down);
  for (uint32_t k = k_begin; k < k_end; ++k) {
    const orc_surfel* s = &m->surfels[k];
    float T[16];
    orc_mat4_mul_f(inv_pose, m->poses + 16 * surfel_pose_index(s), T);
    orc_v3 v = orc_xform_point(T, orc_mk3(s->x, s->y, s->z));
    orc_v3 n = orc_xform_dir(T, orc_mk3(s->nx, s->ny, s->nz));
    if (!(orc_dot3(n, orc_divs3(orc_neg3(v), orc_len3(v))) > 0.01f)) continue; /* :75 */
    float x, y, z;
    orc_project01(v, fov_up, fov, p->min_depth, p->max_depth, &x, &y, &z);
    float fx = floorf(x * (float)W), fy = floorf(y * (float)H); /* :47-48 */
    if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) continue;
    float zn = 2.0f * z - 1.0f;
    if (!(zn >= -1.0f && zn <= 1.0f)) continue;
    uint32_t d24 = orc_depth24(0.5f * zn + 0.5f);
    size_t pix = (size_t)(int)fy * W + (size_t)(int)fx;
    if (d24 < idepth[pix]) {
      idepth[pix] = d24;
      index_map[pix] = k + 1;
    }
  }
}
static void k6a_indexmap(orc_map* m, const float inv_pose[16]) {
  const size_t P = (size_t)m->p.data_width * m->p.data_height;
  const int T = orc_threads();
  depth_clear(m->idepth, P);
  memset(m->index_map, 0, P * 4);
  if (T <= 1 || m->n < 4096u) {
    k6a_range(m, 0, m->n, inv_pose, m->idepth, m->index_map);
    return;
  }
  mt_prepare(m, T); /* chunks in buffer order, merged with GL_LESS in chunk order: see render_pass */
#pragma omp parallel num_threads(T)
  {
#ifdef _OPENMP
    const int t = omp_get_thread_num();
#else
    const int t = 0;
#endif
    uint32_t b, e;
    chunk_of(m->n, T, t, &b, &e);
    memset(m->mt_depth[t], 0xFF, P * 4);
    k6a_range(m, b, e, inv_pose, m->mt_depth[t], m->mt_index[t]);
#pragma omp barrier
#pragma omp for schedule(static)
    for (size_t pix = 0; pix < P; ++pix)
      for (int c = 0; c < T; ++c) {
        uint32_t d = m->mt_depth[c][pix];
        if (d != 0xFFFFFFFFu && d < m->idepth[pix]) {
          m->idepth[pix] = d;
          m->index_map[pix] = m->mt_index[c][pix];
        }
      }
  }
}

/* K6b init_radiusConf.vert:41-68 */
static void k6b_radius(orc_map* m, const float* fv, const float* fn) {
  const orc_params* p = &m->p;
  const size_t P = (size_t)p->data_width * p->data_height;
#pragma omp parallel for schedule(static) num_threads(orc_threads())
  for (size_t i = 0; i < P; ++i) {
    const float* V = fv + 4 * i; const float* N = fn + 4 * i;
    float* o = m->radius_map + 4 * i;
    o[0] = o[1] = o[2] = o[3] = 0.0f;
    orc_v3 v = orc_mk3(V[0], V[1], V[2]), n = orc_mk3(N[0], N[1], N[2]);
    float d = orc_len3(v);
    orc_v3 view_dir = orc_divs3(orc_neg3(v), d);
    float angle = orc_dot3(n, view_dir);
    if (V[3] > 0.5f && N[3] > 0.5f && angle > m->radconf_angle_thresh) {
      float c = angle < 0.5f ? 0.5f : (angle > 1.0f ? 1.0f : angle); /* clamp(.,0.5,1) = min(max(x,.5),1) */
      float radius = ((1.41f * d) * m->pixel_size) / c;              /* :38 */
      float lo = radius > p->min_radius ? radius : p->min_radius;
      radius = lo < p->max_radius ? lo : p->max_radius;              /* :66 */
      o[0] = radius; o[3] = 1.0f;                                    /* Q3: confidence stays 0 */
    }
  }
}

static orc_v3 slerp(orc_v3 v0, orc_v3 v1, float weight) { /* update_surfels.vert:113-124 */
  float omega = orc_acosf(orc_dot3(orc_normalize3(v0), orc_normalize3(v1)));
  float eta = 1.0f / orc_sinf(omega);
  float w0 = eta * orc_sinf(weight * omega);
  float w1 = eta * orc_sinf((1.0f - weight) * omega);
  return orc_add3(orc_scale3(w0, v0), orc_scale3(w1, v1));
}

/* K6c update_surfels.vert:140-333 ; returns keep flag */
static int k6c_surfel(orc_map* m, uint32_t k, const float pose[16], const float inv_pose[16], const float* fv,
                      const float* fn, const float* fs, orc_surfel* out) {
  const orc_params* p = &m->p;
  const int W = p->data_width, H = p->data_height;
  const float fov_up = fabsf(p->data_fov_up), fov = fabsf(p->data_fov_up) + fabsf(p->data_fov_down);
  const orc_surfel* s = &m->surfels[k];
  const int timestamp = (int)m->timestamp;
  int surfel_age = timestamp - (int)s->timestamp;
  int creation = (int)s->count;
  int ci = surfel_pose_index(s);
  const float* sp = m->poses + 16 * ci;
  orc_v3 old_position = orc_xform_point(sp, orc_mk3(s->x, s->y, s->z));
  orc_v3 old_normal = orc_xform_dir(sp, orc_mk3(s->nx, s->ny, s->nz));
  float old_radius = s->radius, old_conf = s->confidence, old_weight = s->weight;
  int valid_out = 1;
  if (old_conf < p->confidence_threshold && p->use_stability) valid_out = surfel_age < p->unstable_age; /* :157 */
  *out = *s;
  out->color = orc_pack_rgb(0.3f, 0.3f, 0.3f);
  orc_v3 vertex = orc_xform_point(inv_pose, old_position);
  orc_v3 normal = orc_normalize3(orc_xform_dir(inv_pose, old_normal));
  int visible = orc_dot3(normal, orc_divs3(orc_neg3(vertex), orc_len3(vertex))) > 0.0f; /* :169 */
  float x, y, z;
  orc_project01(vertex, fov_up, fov, p->min_depth, p->max_depth, &x, &y, &z);
  float ix = floorf(x * (float)W) + 0.5f, iy = floorf(y * (float)H) + 0.5f; /* :89-90 */
  float Vt[4], Nt[4];
  data_tex(fv, W, H, ix, iy, Vt);
  data_tex(fn, W, H, ix, iy, Nt);
  int valid = (Vt[3] > 0.5f) && (Nt[3] > 0.5f);
  int inside = (ix < (float)W && iy < (float)H && z < 1.0f) && !(ix < 0.0f && iy < 0.0f && z < 0.0f); /* :174 (Q7) */
  float penalty = 0.0f;
  float update_conf = m->log_prior;
  int64_t integrated_pix = -1;
  if (valid && inside && visible) {
    float St[4], Rt[4];
    data_tex(fs, W, H, ix, iy, St);
    data_tex(m->radius_map, W, H, ix, iy, Rt);
    float data_label = St[0] * 255.0f, data_prob = St[3];
    float model_label = s->r * 255.0f, model_prob = s->w;
    int label_diff = orc_roundf(data_label) != orc_roundf(model_label);
    if (label_diff && orc_is_movable(model_label)) penalty = 1.0f; /* :187-195 */
    orc_v3 v = orc_mk3(Vt[0], Vt[1], Vt[2]), n = orc_mk3(Nt[0], Nt[1], Nt[2]);
    orc_v3 v_global = orc_xform_point(pose, v);
    orc_v3 n_global = orc_normalize3(orc_xform_dir(pose, n));
    float depth = orc_len3(v);
    orc_v3 view_dir = orc_divs3(orc_neg3(v), orc_len3(v));
    float distance = fabsf(orc_dot3(old_normal, orc_sub3(v_global, old_position))); /* :210 */
    float angle = orc_len3(orc_cross3(n_global, old_normal));                       /* :211 */
    float new_radius = Rt[0], new_conf = Rt[1];
    if (distance < p->map_max_distance && angle < m->update_angle_thresh) { /* :217 */
      /* :219 integrated flag: a point at (pixel, 2z-1) through clipping + depth test GL_LESS -- drawn only if the
       * geometry shader emits the surfel, i.e. if it is still valid at the end (update_surfels.geom:35-48); see below */
      float zn = 2.0f * z - 1.0f;
      if (zn >= -1.0f && zn <= 1.0f && orc_depth24(0.5f * zn + 0.5f) < ORC_DEPTH_CLEAR)
        integrated_pix = (int64_t)((size_t)(int)iy * W + (size_t)(int)ix);
      float confidence = old_conf + new_conf;
      out->confidence = confidence;
      out->timestamp = (uint32_t)timestamp;
      float avg_radius = new_radius < old_radius ? new_radius : old_radius; /* :224 */
      avg_radius = avg_radius > 0.0f ? avg_radius : 0.0f; /* max(avg_radius, min_radius uniform = 0.0, SurfelMap.cpp:422) */
      out->radius = avg_radius;
      valid_out = 1; /* :227 */
      out->color = orc_pack_rgb(0.0f, 0.7f, 0.0f);
      out->count = (float)creation;
      float a = angle, d = distance;
      float pr = p->p_stable;
      if (p->confidence_mode == 1 || p->confidence_mode == 3) pr = pr * orc_expf(((-a) * a) / (p->sigma_angle * p->sigma_angle));
      if (p->confidence_mode == 2 || p->confidence_mode == 3) pr = pr * orc_expf(((-d) * d) / (p->sigma_distance * p->sigma_distance));
      pr = pr > m->p_unstable ? pr : m->p_unstable; /* clamp(p, p_unstable, 1.0) */
      pr = pr < 1.0f ? pr : 1.0f;
      update_conf = orc_logf(pr / (1.0f - pr)); /* :243 */
      (void)depth;
      if ((new_radius < old_radius && timestamp - creation < p->active_timestamps) || p->update_always) { /* :245 */
        float w1 = 0.9f, w2 = 0.1f;
        if (p->weighting_scheme > 0) {
          w1 = old_weight;
          w2 = 1.0f;
          if (p->weighting_scheme == 2) w2 = orc_dot3(n, view_dir);
          float sw = w1 + w2;
          out->weight = p->max_weight < sw ? p->max_weight : sw;
          float sum = w1 + w2;
          w1 = w1 / sum;
          w2 = w2 / sum;
        }
        orc_v3 avg_position = orc_add3(orc_scale3(w1, old_position), orc_scale3(w2, v_global)); /* :263 */
        orc_v3 avg_normal = slerp(old_normal, n_global, w1);                                    /* :265 */
        float avg_prob;
        if (label_diff)
          avg_prob = w1 * model_prob + w2 * (1.0f - data_prob);
        else
          avg_prob = w1 * model_prob + w2 * data_prob;
        out->w = avg_prob; /* :273 */
        if (p->averaging_scheme == 1) {
          avg_position = orc_add3(old_position, orc_scale3(w2 * distance, old_normal)); /* :286 */
          avg_normal = slerp(old_normal, n_global, w1);
        }
        avg_normal = orc_normalize3(avg_normal);
        const float* spi = m->poses_inv + 16 * ci; /* inverse(surfelPose), :197 -- rigid inverse (see orc_math.h) */
        avg_position = orc_xform_point(spi, avg_position);
        avg_normal = orc_xform_dir(spi, avg_normal);
        out->x = avg_position.x; out->y = avg_position.y; out->z = avg_position.z; out->radius = avg_radius;
        out->nx = avg_normal.x; out->ny = avg_normal.y; out->nz = avg_normal.z; out->confidence = confidence;
        out->color = orc_pack_rgb(1.0f, 0.0f, 1.0f);
      }
    } else {
      uint32_t idx1 = 0;
      if (ix >= 0.0f && ix < (float)W && iy >= 0.0f && iy < (float)H) idx1 = m->index_map[(size_t)(int)iy * W + (size_t)(int)ix];
      if ((int)idx1 - 1 == (int)k) { /* :302-308 */
        update_conf = orc_logf(m->p_unstable / (1.0f - m->p_unstable));
        out->color = orc_pack_rgb(0.0f, 1.0f, 1.0f);
      }
    }
  }
  update_conf = update_conf - penalty; /* :324 */
  if (p->use_stability) {
    float c = (old_conf + update_conf) - m->log_prior;
    out->confidence = c < 20.0f ? c : 20.0f; /* :328 */
  } else {
    out->confidence = old_conf;
  }
  if (out->confidence < m->log_unstable && p->use_stability) valid_out = 0; /* :332 */
  /* update_surfels.geom:35: `if(gs_in[0].valid)` -- a surfel that matched its measurement but is removed in the same
   * pass (penalty / negative confidence) emits no vertex, so its pixel is NOT marked integrated and gen_surfels creates
   * a new surfel there. (Found by oracle/_ref, the transpiled reference shaders; round 1 set the flag unconditionally.) */
  if (valid_out && integrated_pix >= 0)
    __atomic_store_n(&m->integrated[(size_t)integrated_pix], (uint8_t)1, __ATOMIC_RELAXED);
  return valid_out;
}

/* copy_surfels.vert:38-56 */
static int k6e_keep(const orc_map* m, const orc_surfel* s, float cx, float cy, float extent) {
  orc_v3 w = orc_xform_point(m->poses + 16 * surfel_pose_index(s), orc_mk3(s->x, s->y, s->z));
  if ((int)s->timestamp < 0 || fabsf(w.x - cx) > extent || fabsf(w.y - cy) > extent) return 0;
  return 1;
}

static orc_tile* tile_get(orc_map* m, int32_t i, int32_t j) { /* submapCache_[idx] (creates an empty entry) */
  for (uint32_t t = 0; t < m->n_tiles; ++t)
    if (m->tiles[t].i == i && m->tiles[t].j == j) return &m->tiles[t];
  if (m->n_tiles == m->cap_tiles) {
    m->cap_tiles = m->cap_tiles ? 2 * m->cap_tiles : 64;
    m->tiles = (orc_tile*)realloc(m->tiles, sizeof(orc_tile) * m->cap_tiles);
  }
  orc_tile* t = &m->tiles[m->n_tiles++];
  t->i = i; t->j = j; t->surfels = NULL; t->n = 0;
  return t;
}
static void extraction_push(orc_map* m, int32_t i, int32_t j) {
  if (m->n_extraction == m->cap_extraction) {
    m->cap_extraction = m->cap_extraction ? 2 * m->cap_extraction : 64;
    m->extraction = (int32_t*)realloc(m->extraction, sizeof(int32_t) * 2 * m->cap_extraction);
  }
  m->extraction[2 * m->n_extraction] = i; m->extraction[2 * m->n_extraction + 1] = j;
  m->n_extraction++;
}
static void append_tiles(orc_map* m, int32_t i0, int32_t j0, int di, int dj) { /* SurfelMap.cpp:770-780 */
  const int dim = m->p.submap_dimension;
  for (int32_t c = -dim; c <= dim; ++c) {
    orc_tile* t = tile_get(m, i0 + di * c, j0 + dj * c);
    uint32_t room = ORC_MAX_SURFELS - m->n;
    uint32_t k = t->n < room ? t->n : room;
    if (k) memcpy(m->surfels + m->n, t->surfels, sizeof(orc_surfel) * k);
    m->n += k;
  }
}
/* extract_surfels.vert:44-62, SurfelMap.cpp:708-742 */
static void extract_surfels(orc_map* m, int partially) {
  const float ext = m->p.submap_extent;
  while (m->n_extraction > 0) {
    m->n_extraction--;
    int32_t i = m->extraction[2 * m->n_extraction], j = m->extraction[2 * m->n_extraction + 1];
    float cx = (float)(2.0 * i * ext), cy = (float)(2.0 * j * ext);
    orc_tile* t = tile_get(m, i, j);
    free(t->surfels);
    t->surfels = NULL; t->n = 0;
    uint32_t cnt = 0;
    for (int pass = 0; pass < 2; ++pass) { /* pass 0 counts, pass 1 copies (capacity ORC_EXTRACT_CAP, TF drops the rest) */
      uint32_t w_i = 0;
      for (uint32_t k = 0; k < m->n; ++k) {
        const orc_surfel* s = &m->surfels[k];
        orc_v3 w = orc_xform_point(m->poses + 16 * surfel_pose_index(s), orc_mk3(s->x, s->y, s->z));
        if (fabsf(w.x - cx) > ext || fabsf(w.y - cy) > ext) continue;
        if (pass == 0) { ++cnt; continue; }
        if (w_i < cnt) t->surfels[w_i++] = *s;
      }
      if (pass == 0) {
        if (cnt > ORC_EXTRACT_CAP) cnt = ORC_EXTRACT_CAP;
        t->surfels = cnt ? (orc_surfel*)malloc(sizeof(orc_surfel) * cnt) : NULL;
      }
    }
    t->n = cnt;
    if (partially) break;
  }
}

/* SurfelMap.cpp:744-824 */
static void update_active_submaps(orc_map* m, const float pose[16]) {
  const int dim = m->p.submap_dimension;
  const float ext = m->p.submap_extent;
  float cx = (float)(2.0 * m->origin_i * ext), cy = (float)(2.0 * m->origin_j * ext);
  float changex = pose[12] - cx, changey = pose[13] - cy;
  float factor = 1.1f;
  if (fabsf(changex) > factor * ext || fabsf(changey) > factor * ext) {
    if (fabsf(changex) > factor * ext) {
      int dir = changex < 0 ? -1 : 1;
      for (int32_t c = -dim; c <= dim; ++c) extraction_push(m, m->origin_i - dir * dim, m->origin_j + c);
      m->origin_i += dir;
      append_tiles(m, m->origin_i + dir * dim, m->origin_j, 0, 1);
    }
    if (fabsf(changey) > factor * ext) {
      int dir = changey < 0 ? -1 : 1;
      for (int32_t r = -dim; r <= dim; ++r) extraction_push(m, m->origin_i + r, m->origin_j - dir * dim);
      m->origin_j += dir;
      append_tiles(m, m->origin_i, m->origin_j + dir * dim, 1, 0);
    }
  }
  if (m->n_extraction > 0) extract_surfels(m, m->p.partial_extraction);
}

void orc_map_update(orc_map* m, const float pose[16], const float* fv, const float* fn, const float* fs) {
  const orc_params* p = &m->p;
  const int W = p->data_width, H = p->data_height;
  const size_t P = (size_t)W * H;
  if (m->timestamp < ORC_MAX_POSES) orc_map_set_pose(m, m->timestamp, pose); /* SurfelMap.cpp:494-495 */
  float inv_pose[16];
  orc_rigid_inverse_f(pose, inv_pose); /* :497 */
  k6a_indexmap(m, inv_pose);
  k6b_radius(m, fv, fn);
  /* K6c */
  memset(m->integrated, 0, P);
  uint32_t nu = 0;
  const int T = orc_threads();
  if (T <= 1 || m->n < 4096u) {
    for (uint32_t k = 0; k < m->n; ++k) {
      orc_surfel o;
      if (k6c_surfel(m, k, pose, inv_pose, fv, fn, fs, &o)) m->scratch[nu++] = o;
    }
  } else {
    /* ordered stream compaction (transform feedback order): every thread packs its contiguous chunk in place in a
     * second buffer, the chunk counts are prefix-summed, the chunks are copied behind one another */
    uint32_t cnt[64], off[65];
    if (!m->scratch2) m->scratch2 = (orc_surfel*)malloc(sizeof(orc_surfel) * ORC_MAX_SURFELS);
#pragma omp parallel num_threads(T)
    {
#ifdef _OPENMP
      const int t = omp_get_thread_num();
#else
      const int t = 0;
#endif
      uint32_t b, e, c = 0;
      chunk_of(m->n, T, t, &b, &e);
      for (uint32_t k = b; k < e; ++k) {
        orc_surfel o;
        if (k6c_surfel(m, k, pose, inv_pose, fv, fn, fs, &o)) m->scratch2[b + c++] = o;
      }
      cnt[t] = c;
#pragma omp barrier
#pragma omp single
      {
        off[0] = 0;
        for (int i = 0; i < T; ++i) off[i + 1] = off[i] + cnt[i];
      }
      memcpy(m->scratch + off[t], m->scratch2 + b, sizeof(orc_surfel) * (size_t)c);
    }
    nu = off[T];
  }
  m->n_updated = nu;
  /* K6d gen_surfels.vert:38-52 + .geom:109-145, pixels in x-major order (SurfelMap.cpp:88-92) */
  uint32_t nn = 0;
  const int timestamp = (int)m->timestamp;
  /* phase 1 (all host threads): which pixels emit a surfel; phase 2: emission in x-major order */
  uint8_t* emit = (uint8_t*)malloc(P);
#pragma omp parallel for schedule(static) num_threads(orc_threads())
  for (size_t pix = 0; pix < P; ++pix) {
    const float* V = fv + 4 * pix; const float* N = fn + 4 * pix; const float* R = m->radius_map + 4 * pix;
    int invalid = (V[3] < 1.0f) || (N[3] < 1.0f);
    invalid = invalid || (R[3] < 0.5f);
    int integrated = m->integrated[pix] != 0;
    orc_v3 v = orc_mk3(V[0], V[1], V[2]), n = orc_mk3(N[0], N[1], N[2]);
    orc_v3 view_dir = orc_divs3(orc_neg3(v), orc_len3(v));
    emit[pix] = (uint8_t)(!invalid && !integrated && (orc_dot3(n, view_dir) > 0.01f));
  }
  for (int x = 0; x < W; ++x)
    for (int y = 0; y < H; ++y) {
      size_t pix = (size_t)y * W + x;
      if (!emit[pix]) continue;
      if (nu + nn >= ORC_MAX_SURFELS) continue;
      const float* V = fv + 4 * pix; const float* N = fn + 4 * pix; const float* R = m->radius_map + 4 * pix;
      orc_v3 v = orc_mk3(V[0], V[1], V[2]), n = orc_mk3(N[0], N[1], N[2]);
      orc_surfel* o = &m->scratch[nu + nn];
      orc_v3 ng = orc_normalize3(n);
      o->x = v.x; o->y = v.y; o->z = v.z; o->radius = R[0];
      o->nx = ng.x; o->ny = ng.y; o->nz = ng.z; o->confidence = m->log_prior;
      o->timestamp = (uint32_t)timestamp;
      o->color = orc_pack_rgb(0.0f, 0.0f, 1.0f); o->weight = 1.0f; o->count = (float)timestamp;
      const float* S = fs + 4 * pix;
      o->r = S[0]; o->g = S[1]; o->b = S[2]; o->w = S[3];
      if (orc_is_movable(S[0] * 255.0f)) o->confidence = m->log_prior - 0.5f; /* .geom:135-140 */
      ++nn;
    }
  free(emit);
  m->n_new = nn;
  /* K6e copySurfels, SurfelMap.cpp:667-698 */
  float cx = (float)(2.0 * m->origin_i * p->submap_extent), cy = (float)(2.0 * m->origin_j * p->submap_extent);
  float extent = 2.0f * p->submap_dimension * p->submap_extent + p->submap_extent;
  if (p->partial_extraction && m->n_extraction > 0) extent += 2.0f * p->submap_extent;
  uint32_t no = 0;
  if (T <= 1 || nu + nn < 4096u) {
    for (uint32_t k = 0; k < nu + nn; ++k)
      if (k6e_keep(m, &m->scratch[k], cx, cy, extent)) m->surfels[no++] = m->scratch[k];
  } else {
    uint32_t cnt[64], off[65];
    const uint32_t total = nu + nn;
    if (!m->scratch2) m->scratch2 = (orc_surfel*)malloc(sizeof(orc_surfel) * ORC_MAX_SURFELS);
#pragma omp parallel num_threads(T)
    {
#ifdef _OPENMP
      const int t = omp_get_thread_num();
#else
      const int t = 0;
#endif
      uint32_t b, e, c = 0;
      chunk_of(total, T, t, &b, &e);
      for (uint32_t k = b; k < e; ++k)
        if (k6e_keep(m, &m->scratch[k], cx, cy, extent)) m->scratch2[b + c++] = m->scratch[k];
      cnt[t] = c;
#pragma omp barrier
#pragma omp single
      {
        off[0] = 0;
        for (int i = 0; i < T; ++i) off[i + 1] = off[i] + cnt[i];
      }
      memcpy(m->surfels + off[t], m->scratch2 + b, sizeof(orc_surfel) * (size_t)c);
    }
    no = off[T];
  }
  m->n = no;
  update_active_submaps(m, pose);
  m->timestamp += 1;
}
