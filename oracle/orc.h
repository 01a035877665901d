/* orc.h -- TEST INFRASTRUCTURE: CPU oracle for the SuMa++ per-scan hot path.
 *
 * A plain-C restatement of the reference's GLSL passes and their C++ drivers (PRBonn/semantic_suma @ 531954dd;
 * every function cites the file:line it follows, relative to /root/reference/src). It exists to CHECK the CUDA
 * path; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 *
 * PARITY STATUS: pinned to THE REFERENCE ITSELF, run here. The reference ships no tests, golden vectors or fixtures for
 * this path (SURVEY.md section 4) and its GPU build (OpenGL + un-vendored glow/gtsam/rangenet_lib + Qt) cannot run in
 * this environment, but its sources compile from where they lie under /root/reference (oracle/ref_harness/Makefile ->
 * oracle/_ref/, git-ignored):
 *   libsuma_ref_full.so    the core classes themselves (Preprocessing, Frame2Model, LieGaussNewton, SurfelMap,
 *                          SurfelMapping::processScan ...) driving the reference's own transpiled shaders on a stand-in
 *                          glow over a generic software GL. With what GL / Eigen / libm leave open pinned to the rules
 *                          of orc_math.h / DESIGN.md section 2, and this oracle adding the 48 ICP values the way the GL
 *                          path does (orc_set_gl_sums), oracle and reference agree BIT FOR BIT over whole runs -- poses,
 *                          iteration counts, frames, every surfel record -- incl. the track-loss fallback, submap paging,
 *                          loop-closure detection, 24 parameter variants, 64x900 / 64x2048 / 128x4096
 *                          (tests/test_ref_full.py); tests/golden/reference_golden.json holds digests of its outputs. An UNPINNED build of the same
 *                          library (libsuma_ref_full_precise.so) agrees with this oracle within 2e-3 m / 0.2 %.
 *   libsuma_ref_pinned.so / _precise.so   the shaders per operator, also on adversarial random inputs
 *                          (tests/test_ref_shaders.py); _host.so: the host sources unpinned (tests/test_ref_host.py).
 * The default mode of this oracle (exact Q33.30 sums of the 48 values) is the contract of the CUDA path; it differs from
 * the reference's fp32 blending by < 1e-5 of the matrix scale per evaluation (test_jacobian_sums_equal_reference_shader).
 * Deviations found by running the reference, all documented in DESIGN.md section 2: update_surfels.geom:35 (fixed), the
 * stale attribute tail of quirk Q1 (kept: the reference reads the previous upload's data there, we read 0).
 * Still "by construction": the fixed-function GL rules themselves (no GL implementation exists here to test them against).
 *
 * Conventions: images are [H][W][4] float32, row 0 = lowest beam; 4x4 matrices are column-major (Eigen/GL).
 */
#ifndef ORC_H_
#define ORC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_params {
  /* data / model image geometry (config/default.xml:7-12, 30-35) */
  int32_t data_width, data_height;
  float data_fov_up, data_fov_down; /* degrees, signed as in the XML */
  float min_depth, max_depth;
  int32_t model_width, model_height;
  float model_fov_up, model_fov_down;
  float model_min_depth, model_max_depth;
  /* ICP (default.xml:16-26) */
  int32_t max_iterations;
  double stopping_threshold, delta;
  float icp_max_distance, icp_max_angle; /* m, degrees */
  int32_t weighting;                     /* 0 none, 1 huber, 2 turkey, 3 stability (Frame2Model.cpp:69-80) */
  float factor;
  int32_t initialize_identity;
  int32_t bilinear_sampling;
  int32_t fallback_mode;
  float fallback_max_distance, fallback_max_angle;
  /* surfel map (default.xml:37-67) */
  int32_t compose_rendering;
  float max_loop_closure_distance;
  float min_radius, max_radius, max_angle;
  float map_max_distance, map_max_angle;
  int32_t unstable_age, confidence_mode;
  float confidence_threshold;
  float p_stable, p_prior, sigma_angle, sigma_distance;
  int32_t use_stability, active_timestamps;
  float max_weight;
  int32_t weighting_scheme, averaging_scheme, update_always;
  int32_t submap_dimension;
  float submap_extent;
  int32_t partial_extraction;
  /* quirk switches (1 = behave exactly like the reference) */
  int32_t label_offset_quirk; /* Q1: point i reads labels[i+4], probs[i+5] (Preprocessing.cpp:142-145) */
  int32_t render_after_update; /* SurfelMapping.cpp:803 re-renders the model after the map update */
} orc_params;

/* 64-byte surfel record, Surfel.h:5-15 */
typedef struct orc_surfel {
  float x, y, z, radius;
  float nx, ny, nz, confidence;
  uint32_t timestamp;
  float color, weight, count;
  float r, g, b, w;
} orc_surfel;

void orc_default_params(orc_params* p); /* config/default.xml */
/* the parameters the CUDA library's sb_create accepts: NULL, or the reason they are refused. orc_map_create and
 * orc_slam_create return NULL on refused parameters. */
const char* orc_check_params(const orc_params* p);
/* host threads used by the oracle's loops (OpenMP); 0 = all the machine offers (capped at 64). Results are
 * bit-identical for every thread count. Returns the count now in effect. */
int orc_set_threads(int n);

/* ---- scalar functions exported for unit tests ---- */
float orc_t_atan2f(float y, float x);
float orc_t_asinf(float x);
float orc_t_acosf(float x);
float orc_t_sinf(float x);
float orc_t_expf(float x);
float orc_t_logf(float x);
void orc_t_sincos(double x, double* s, double* c);

/* ---- K1-K3: Preprocessing::process (Preprocessing.cpp:120-339) ---- */
void orc_preprocess(const orc_params* p, const float* pts4, const float* labels, const float* probs, uint32_t n,
                    uint32_t timestamp, float* vertex_map, float* normal_map, float* semantic_map);

/* ---- K5: Frame2Model::jacobianProducts (Frame2Model.cpp:136-261) ----
 * out48 has the reference's 48-float layout (JtJ col-major 6x6 | Jtf | n_valid, F, n_outlier, F_inlier, n_invalid, 0)
 * as doubles; raw32 (optional) are the exact Q33.30 fixed-point sums (21 lower-tri + 6 + F + F_inlier) and the
 * three integer counters. row_begin/row_end restrict the data rows (multi-GPU striping); use 0, data_height. */
void orc_icp_jacobian(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                      const float* model_v, const float* model_n, const float* model_s, const double pose[16],
                      int32_t iteration, float max_distance, float max_angle_deg, int32_t row_begin,
                      int32_t row_end, double out48[48], int64_t raw32[32]);
void orc_icp_unpack(const int64_t raw32[32], double out48[48]);
/* 1: sum the way the reference's GL path does (see orc_core.c); returns the previous mode. Test infrastructure. */
int orc_set_gl_sums(int on);
/* same sums, accumulated the way the GL path does (fp32 partial sums of 64 pixels, then fp32 adds): used only to
 * show that the reference's own arithmetic lies within the 1e-5 band around the exact sums. */
void orc_icp_jacobian_fp32gl(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                             const float* model_v, const float* model_n, const float* model_s,
                             const double pose[16], int32_t iteration, float max_distance, float max_angle_deg,
                             float out48[48]);

/* ---- LieGaussNewton / SE3 (LieGaussNewton.cpp:13-79, lie_algebra.cpp:4-71) ---- */
void orc_se3_exp(const double x[6], double T[16]);
void orc_se3_log(const double T[16], double x[6]);
int orc_ldlt_solve6(const double A[36], const double b[6], double x[6]); /* x = A^-1 b, A sym. (lower used) */
/* GN step given the 48 values: delta, stop flag, new pose. Returns 0 if converged (LieGaussNewton.cpp:53-79). */
int orc_gn_step(const double out48[48], double last_error, double eps, double delta_thr, double pose[16],
                double dx[6]);
/* full minimize (LieGaussNewton.cpp:13-37). history: (max_iter+1)*16 doubles or NULL. returns iterations k_. */
int orc_icp_minimize(const orc_params* p, const float* data_v, const float* data_n, const float* data_s,
                     const float* model_v, const float* model_n, const float* model_s, const double T0[16],
                     float max_distance, float max_angle_deg, double pose_out[16], double out48[48],
                     double* history, int32_t* history_len);

/* ---- surfel map (SurfelMap.cpp) ---- */
typedef struct orc_map orc_map;
orc_map* orc_map_create(const orc_params* p);
void orc_map_destroy(orc_map* m);
void orc_map_reset(orc_map* m);
uint32_t orc_map_size(const orc_map* m);
uint32_t orc_map_timestamp(const orc_map* m);
uint32_t orc_map_download(const orc_map* m, orc_surfel* dst, uint32_t cap);
void orc_map_upload(orc_map* m, const orc_surfel* src, uint32_t n, uint32_t timestamp); /* test hook */
void orc_map_set_pose(orc_map* m, uint32_t t, const float pose[16]);                    /* test hook */
void orc_map_update_poses(orc_map* m, const float* poses16, uint32_t count);            /* SurfelMap.cpp:485-490 */
/* SurfelMap::render (847-1021): fills the internal old/new/composed frames and writes `frame` */
void orc_map_render(orc_map* m, const float pose_old[16], const float pose_new[16], float conf_thr, float* frame_v,
                    float* frame_n, float* frame_s);
void orc_map_render_active(orc_map* m, const float pose[16], float conf_thr);   /* 1023-1069 */
void orc_map_render_inactive(orc_map* m, const float pose[16], float conf_thr); /* 1071-1114 */
void orc_map_render_composed(orc_map* m, const float pose_old[16], const float pose_new[16], float conf_thr);
/* which: 0 old, 1 new, 2 composed */
void orc_map_get_frame(const orc_map* m, int which, float* v, float* n, float* s);
/* SurfelMap::update (492-584) */
void orc_map_update(orc_map* m, const float pose[16], const float* frame_v, const float* frame_n,
                    const float* frame_s);
/* intermediate products of the last update, for stage-wise parity tests */
void orc_map_get_update_debug(const orc_map* m, uint32_t* index_map, float* radius_map, uint8_t* integrated,
                              uint32_t* n_updated, uint32_t* n_new);
void orc_map_get_submap_origin(const orc_map* m, int32_t* i, int32_t* j, uint32_t* pending);

/* ---- SurfelMapping::processScan (SurfelMapping.cpp:175-210) with loop closure off ---- */
typedef struct orc_slam orc_slam;
orc_slam* orc_slam_create(const orc_params* p);
void orc_slam_destroy(orc_slam* s);
void orc_slam_process_scan(orc_slam* s, const float* pts4, const float* labels, const float* probs, uint32_t n);
void orc_slam_get_pose(const orc_slam* s, double pose[16]);
uint32_t orc_slam_timestamp(const orc_slam* s);
orc_map* orc_slam_map(orc_slam* s);
/* stats: [0] icp iterations, [1] F (result_new_.error), [2] inlier, [3] outlier, [4] invalid, [5] inlier_residual,
 * [6] track losses, [7] n surfels; times (s): [8] preprocess [9] icp [10] mapping [11] complete */
void orc_slam_get_stats(const orc_slam* s, double stats[16]);
void orc_slam_get_frame(const orc_slam* s, int which /*0 current data, 1 last model frame*/, float* v, float* n,
                        float* sem);
/* hooks for the loop-closure twin (orc_loop.cpp): a callback between updatePose() and updateMap() and the members it uses */
typedef void (*orc_slam_hook)(orc_slam* s, void* user);
void orc_slam_set_hook(orc_slam* s, orc_slam_hook hook, void* user);
double* orc_slam_pose_member(orc_slam* s, int which /*0 current 1 current_old 2 current_new 3 last_old 5 increment 6 lastIncrement*/);
void orc_slam_current_frame(orc_slam* s, float** v, float** n, float** sem);
float orc_slam_conf_threshold(const orc_slam* s);
const orc_params* orc_slam_params(const orc_slam* s);

#ifdef __cplusplus
}
#endif
#endif /* ORC_H_ */
