/* orc_slam.c -- TEST INFRASTRUCTURE (CPU oracle): SurfelMapping::processScan with loop closure disabled.
 * Follows core/SurfelMapping.cpp:175-210 (processScan), 323-358 (initialize/preprocess), 372-476 (updatePose),
 * 797-804 (updateMap). */
#include "orc.h"
#include "orc_internal.h"

#include <stdlib.h>
#include <time.h>

typedef struct { float *v, *n, *s; } sframe;

struct orc_slam {
  orc_params p;
  orc_map* map;
  sframe cur, last;          /* currentFrame_, lastFrame_ (data size) */
  sframe cur_model, last_model; /* currentModelFrame_, lastModelFrame_ (model size) */
  float *tmp_v, *tmp_n, *tmp_s; /* newMapFrame download */
  uint32_t timestamp;
  double currentPose[16], lastPose[16], currentPose_old[16], currentPose_new[16], lastIncrement[16];
  double lastPose_old[16], increment[16], prevIncrement[16]; /* lastPose_old_ (:454), this scan's increment, lastIncrement_ before it */
  orc_slam_hook hook;        /* called between updatePose() and updateMap(): where checkLoopClosure() runs (:196-200) */
  void* hook_user;
  float confidence_threshold, log_unstable;
  double stats[16];
  uint32_t trackLoss;
};

static void sframe_alloc(sframe* f, size_t P) {
  f->v = (float*)calloc(P * 4, 4); f->n = (float*)calloc(P * 4, 4); f->s = (float*)calloc(P * 4, 4);
}
static void sframe_free(sframe* f) { free(f->v); free(f->n); free(f->s); }
static void ident_d(double* M) { for (int i = 0; i < 16; ++i) M[i] = (i % 5 == 0) ? 1.0 : 0.0; }
static void cast_f(const double* M, float* F) { for (int i = 0; i < 16; ++i) F[i] = (float)M[i]; }
static double now_s(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }

orc_slam* orc_slam_create(const orc_params* p) {
  if (orc_check_params(p)) return NULL;
  orc_slam* s = (orc_slam*)calloc(1, sizeof(orc_slam));
  s->p = *p;
  s->map = orc_map_create(p);
  size_t Pd = (size_t)p->data_width * p->data_height, Pm = (size_t)p->model_width * p->model_height;
  sframe_alloc(&s->cur, Pd); sframe_alloc(&s->last, Pd);
  sframe_alloc(&s->cur_model, Pm); sframe_alloc(&s->last_model, Pm);
  s->tmp_v = (float*)calloc(Pm * 4, 4); s->tmp_n = (float*)calloc(Pm * 4, 4); s->tmp_s = (float*)calloc(Pm * 4, 4);
  ident_d(s->currentPose); ident_d(s->lastPose); ident_d(s->currentPose_old); ident_d(s->currentPose_new);
  ident_d(s->lastIncrement); ident_d(s->lastPose_old); ident_d(s->increment); ident_d(s->prevIncrement);
  s->confidence_threshold = p->confidence_threshold;        /* SurfelMapping.cpp:111-113 */
  { float pu = 0.1f; s->log_unstable = logf(pu / (1.0f - pu)); } /* :108-109 */
  return s;
}
void orc_slam_destroy(orc_slam* s) {
  if (!s) return;
  orc_map_destroy(s->map);
  sframe_free(&s->cur); sframe_free(&s->last); sframe_free(&s->cur_model); sframe_free(&s->last_model);
  free(s->tmp_v); free(s->tmp_n); free(s->tmp_s);
  free(s);
}

/* SurfelMapping.cpp:333-340, time_init = 10 (SurfelMapping.h:192) */
static float conf_threshold(const orc_slam* s) {
  float ct = s->confidence_threshold;
  if (s->timestamp < 10) {
    float alpha = (float)s->timestamp / 10.0f;
    ct = (float)((1.0 - (double)alpha) * (double)s->log_unstable + (double)(alpha * s->confidence_threshold));
  }
  return ct;
}

static void update_pose(orc_slam* s) {
  const orc_params* p = &s->p;
  double T0[16];
  if (!p->initialize_identity) memcpy(T0, s->lastIncrement, sizeof(T0)); else ident_d(T0);
  size_t Pm = (size_t)p->model_width * p->model_height;
  /* objective_->setData(currentFrame_, map_->newMapFrame()), :384 */
  orc_map_get_frame(s->map, 1, s->tmp_v, s->tmp_n, s->tmp_s);
  double increment[16], o48[48];
  int iters = orc_icp_minimize(p, s->cur.v, s->cur.n, s->cur.s, s->tmp_v, s->tmp_n, s->tmp_s, T0,
                               p->icp_max_distance, p->icp_max_angle, increment, o48, NULL, NULL);
  s->stats[0] = iters;
  double inv_last[16], delta[16];
  orc_rigid_inverse_d(s->lastIncrement, inv_last);
  orc_mat4_mul_d(inv_last, increment, delta); /* :397 */
  /* :405-413 */
  double Pn[16];
  float Pf[16];
  orc_mat4_mul_d(s->currentPose_new, increment, Pn);
  cast_f(Pn, Pf);
  orc_map_render_active(s->map, Pf, conf_threshold(s));
  orc_map_get_frame(s->map, 1, s->tmp_v, s->tmp_n, s->tmp_s);
  memcpy(s->last_model.v, s->tmp_v, Pm * 16); memcpy(s->last_model.n, s->tmp_n, Pm * 16);
  memcpy(s->last_model.s, s->tmp_s, Pm * 16); /* lastModelFrame_->copy(newMapFrame) */
  double I[16], r48[48];
  ident_d(I);
  orc_icp_jacobian(p, s->cur.v, s->cur.n, s->cur.s, s->tmp_v, s->tmp_n, s->tmp_s, I, 0, p->icp_max_distance,
                   p->icp_max_angle, 0, p->data_height, r48, NULL);
  s->stats[1] = r48[43];
  s->stats[3] = r48[44];
  s->stats[2] = (double)((uint32_t)r48[42] - (uint32_t)r48[44]); /* Frame2Model.cpp:222-226 */
  s->stats[4] = r48[46];
  s->stats[5] = (float)r48[45];
  /* :430-449 track-loss test */
  float t_err = (float)sqrt((delta[12] * delta[12] + delta[13] * delta[13]) + delta[14] * delta[14]);
  float angle = (float)(0.5 * (((delta[0] + delta[5]) + delta[10]) - 1.0));
  float ca = angle < 1.0f ? angle : 1.0f;
  ca = ca > -1.0f ? ca : -1.0f;
  float r_err = orc_acosf(ca); /* fixed polynomial (orc_math.h): the device-side pose bookkeeping must take the same branch */
  if (s->timestamp > 1 && (t_err > 0.4 || r_err > 0.1) && p->fallback_mode) {
    s->trackLoss += 1;
    /* recovery_->setData(currentFrame_, lastFrame_): frame-to-frame with the fallback thresholds, :89-96, 438-449 */
    orc_icp_minimize(p, s->cur.v, s->cur.n, s->cur.s, s->last.v, s->last.n, s->last.s, T0, p->fallback_max_distance,
                     p->fallback_max_angle, increment, o48, NULL, NULL);
  }
  s->stats[6] = s->trackLoss;
  memcpy(s->lastPose, s->currentPose, sizeof(s->lastPose));
  double np[16];
  orc_mat4_mul_d(s->currentPose, increment, np); /* :452 */
  memcpy(s->currentPose, np, sizeof(np));
  memcpy(s->lastPose_old, s->currentPose_old, sizeof(np)); /* :454 */
  memcpy(s->prevIncrement, s->lastIncrement, sizeof(np));
  memcpy(s->increment, increment, sizeof(np));
  memcpy(s->currentPose_old, np, sizeof(np));
  memcpy(s->currentPose_new, np, sizeof(np));
  memcpy(s->lastIncrement, increment, sizeof(increment)); /* :473 */
}

void orc_slam_process_scan(orc_slam* s, const float* pts4, const float* labels, const float* probs, uint32_t n) {
  const orc_params* p = &s->p;
  double t_all = now_s();
  /* initialize(), :323-331 */
  { sframe t = s->last; s->last = s->cur; s->cur = t; }
  { sframe t = s->last_model; s->last_model = s->cur_model; s->cur_model = t; }
  /* preprocess(), :342-358 */
  double t0 = now_s();
  orc_preprocess(p, pts4, labels, probs, n, s->timestamp, s->cur.v, s->cur.n, s->cur.s);
  float ct = conf_threshold(s);
  float Pold[16], Pnew[16];
  cast_f(s->currentPose_old, Pold);
  cast_f(s->currentPose_new, Pnew);
  orc_map_render(s->map, Pold, Pnew, ct, s->last_model.v, s->last_model.n, s->last_model.s);
  s->stats[8] = now_s() - t0;
  t0 = now_s();
  if (s->timestamp > 0) {
    update_pose(s);
    if (s->hook) s->hook(s, s->hook_user); /* checkLoopClosure(), :198 */
  }
  s->stats[9] = now_s() - t0;
  /* updateMap(), :797-804 */
  t0 = now_s();
  float Pc[16];
  cast_f(s->currentPose, Pc);
  orc_map_update(s->map, Pc, s->cur.v, s->cur.n, s->cur.s);
  if (p->render_after_update) {
    ct = conf_threshold(s);
    orc_map_render(s->map, Pc, Pc, ct, s->cur_model.v, s->cur_model.n, s->cur_model.s);
  }
  s->stats[10] = now_s() - t0;
  s->stats[7] = orc_map_size(s->map);
  s->stats[11] = now_s() - t_all;
  s->timestamp += 1;
}

void orc_slam_get_pose(const orc_slam* s, double pose[16]) { memcpy(pose, s->currentPose, sizeof(s->currentPose)); }
uint32_t orc_slam_timestamp(const orc_slam* s) { return s->timestamp; }
orc_map* orc_slam_map(orc_slam* s) { return s->map; }
void orc_slam_get_stats(const orc_slam* s, double stats[16]) { memcpy(stats, s->stats, sizeof(s->stats)); }
void orc_slam_get_frame(const orc_slam* s, int which, float* v, float* n, float* sem) {
  const sframe* f = which == 0 ? &s->cur : &s->last_model;
  size_t P = which == 0 ? (size_t)s->p.data_width * s->p.data_height : (size_t)s->p.model_width * s->p.model_height;
  if (v) memcpy(v, f->v, P * 16);
  if (n) memcpy(n, f->n, P * 16);
  if (sem) memcpy(sem, f->s, P * 16);
}

/* ---- hooks for the loop-closure twin (oracle/orc_loop.cpp) ---- */
void orc_slam_set_hook(orc_slam* s, orc_slam_hook hook, void* user) { s->hook = hook; s->hook_user = user; }
double* orc_slam_pose_member(orc_slam* s, int which) {
  switch (which) {
    case 0: return s->currentPose;
    case 1: return s->currentPose_old;
    case 2: return s->currentPose_new;
    case 3: return s->lastPose_old;
    case 4: return s->prevIncrement;  /* lastIncrement_ as checkLoopClosure reads it?  NO: see orc_loop.cpp -- it reads the NEW lastIncrement_ */
    case 5: return s->increment;
    case 6: return s->lastIncrement;
    default: return NULL;
  }
}
void orc_slam_current_frame(orc_slam* s, float** v, float** n, float** sem) { *v = s->cur.v; *n = s->cur.n; *sem = s->cur.s; }
float orc_slam_conf_threshold(const orc_slam* s) { return conf_threshold(s); }
const orc_params* orc_slam_params(const orc_slam* s) { return &s->p; }
