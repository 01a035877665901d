/* suma_b200.h -- C ABI of libsuma_b200.so: a Hopper (sm_90a) projective-ICP + surfel-fusion core that replaces
 * the OpenGL/GLSL hot path of PRBonn/semantic_suma (SuMa++) behind the reference's own operator surface.
 *
 * The reference has no FFI layer: its boundary is four C++ classes (SurfelMapping, Frame2Model, SurfelMap,
 * Preprocessing). Each entry point below names the reference method (file:line under /root/reference/src) it
 * replaces; include/suma_b200.hpp re-creates those classes on top of this ABI.
 *
 * Conventions
 *   - every function returns 0 (SB_OK) or a negative sb_status; nothing throws across the boundary
 *   - 4x4 matrices are 16 values in COLUMN-MAJOR order (what Eigen's .data() hands out)
 *   - images are [H][W][4] float32, row 0 = lowest beam, column 0 = yaw +pi (gen_vertexmap.vert:83-89)
 *   - one sb_ctx = one CUDA device + one stream; externally synchronised (like the GL context it replaces)
 *   - host pointers unless a parameter says "device"; transfers are issued on the context's stream
 */
#ifndef SUMA_B200_H_
#define SUMA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_VERSION 100

typedef enum sb_status {
  SB_OK = 0,
  SB_ERR_INVALID = -1,  /* bad argument */
  SB_ERR_CUDA = -2,     /* CUDA runtime error (see sb_last_error) */
  SB_ERR_NOMEM = -3,
  SB_ERR_CAPACITY = -4, /* surfel / pose capacity exceeded */
  SB_ERR_STATE = -5,    /* call not valid in the current state */
  SB_ERR_NOGPU = -6     /* no CUDA device: there is no CPU fallback */
} sb_status;

/* The parameters the hot path reads; names follow the XML keys of config/default.xml
 * (Preprocessing.cpp:76-117, Frame2Model.cpp:20-23,65-110, SurfelMap.cpp:265-273,336-457,
 *  SurfelMapping.cpp:68-129, LieGaussNewton.cpp:8-10,81-91). */
typedef struct sb_params {
  int32_t data_width, data_height;
  float data_fov_up, data_fov_down;
  float min_depth, max_depth;
  int32_t model_width, model_height;
  float model_fov_up, model_fov_down;
  float model_min_depth, model_max_depth;
  int32_t max_iterations;            /* "max iterations" */
  double stopping_threshold, delta;  /* "stopping threshold", "delta" */
  float icp_max_distance, icp_max_angle;
  int32_t weighting; /* 0 none, 1 huber, 2 turkey, 3 stability */
  float factor;
  int32_t initialize_identity;
  int32_t bilinear_sampling;
  int32_t fallback_mode;
  float fallback_max_distance, fallback_max_angle;
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
  /* behaviour switches; 1 = exactly what the reference does */
  int32_t label_offset_quirk;  /* Preprocessing.cpp:142-145: point i is paired with labels[i+4], probs[i+5] */
  int32_t render_after_update; /* SurfelMapping.cpp:803: re-render the model after the map update */
} sb_params;

/* Surfel.h:5-15 (64 bytes) */
typedef struct sb_surfel {
  float x, y, z, radius;
  float nx, ny, nz, confidence;
  uint32_t timestamp;
  float color, weight, count;
  float r, g, b, w;
} sb_surfel;

typedef struct sb_ctx sb_ctx;
typedef struct sb_frame sb_frame; /* Frame.h:21-79: vertex / normal / semantic maps on the device */

enum { SB_MAP_VERTEX = 0, SB_MAP_NORMAL = 1, SB_MAP_SEMANTIC = 2 };
enum { SB_FRAME_OLD = 0, SB_FRAME_NEW = 1, SB_FRAME_COMPOSED = 2 };          /* SurfelMap.h:59-61 */
enum { SB_SLAM_CURRENT = 0, SB_SLAM_LAST = 1, SB_SLAM_CURRENT_MODEL = 2, SB_SLAM_LAST_MODEL = 3 };

/* ---- context ---------------------------------------------------------------------------------------------- */
int sb_default_params(sb_params* p);                               /* config/default.xml */
/* sb_create and sb_set_params return SB_ERR_INVALID (reason on stderr / in sb_last_error) for:
 *  - image sizes <= 0, more than 2^24 data pixels, or a data width of 1 (the preprocessing stencils reach two columns
 *    around the azimuth seam, which one column cannot provide);
 *  - a model image side over 65536 pixels (the render pass packs a quad's pixel box origin in 16 bits per axis);
 *  - depth ranges with max <= min;
 *  - parameters whose exact ICP sums could leave the int64 range: data pixels x (max(max_depth, model_max_depth) + 25 m)^2
 *    x 2^30 > 2^63 - 1. The 25 m allow for the translation of the pose. 128x4096 at 75 m is accepted; the largest image
 *    at 75 m has 858 993 pixels. */
int sb_create(const sb_params* p, int device, sb_ctx** out);       /* SurfelMapping::SurfelMapping, SurfelMapping.cpp:19 */
int sb_destroy(sb_ctx* ctx);
int sb_reset(sb_ctx* ctx);                                         /* SurfelMapping::reset / SurfelMap::reset, SurfelMap.cpp:473 */
int sb_set_params(sb_ctx* ctx, const sb_params* p);                /* SurfelMapping::setParameters, SurfelMapping.cpp:68 */
int sb_get_params(const sb_ctx* ctx, sb_params* p);               /* the parameters in effect (e.g. after sb_state_load) */
const char* sb_last_error(const sb_ctx* ctx);
int sb_synchronize(sb_ctx* ctx);
int sb_device_count(void);
/* CUDA stream (cudaStream_t) the context launches on, for callers that time or order work themselves */
void* sb_stream(sb_ctx* ctx);
/* number of kernels this library has launched on the context so far */
uint64_t sb_launch_count(const sb_ctx* ctx);

/* ---- frames ----------------------------------------------------------------------------------------------- */
int sb_frame_create(sb_ctx* ctx, int width, int height, sb_frame** out); /* Frame::Frame, Frame.h:25 */
int sb_frame_destroy(sb_frame* f);
int sb_frame_copy(sb_frame* dst, const sb_frame* src);                   /* Frame::copy, Frame.h:49-61 */
int sb_frame_download(const sb_frame* f, int which, float* dst /* H*W*4 */);
int sb_frame_upload(sb_frame* f, int which, const float* src /* H*W*4 */);
int sb_frame_size(const sb_frame* f, int* width, int* height);

/* ---- K1-K3: Preprocessing::process, Preprocessing.cpp:120-339 ---------------------------------------------------
 * labels / probs may be NULL (geometric SuMa: every label 0, prob 0). pts_on_device != 0: the three arrays are
 * device pointers already resident in HBM. */
int sb_preprocess(sb_ctx* ctx, const float* pts4, const float* labels, const float* probs, uint32_t n,
                  uint32_t timestamp, int pts_on_device, sb_frame* out);

/* ---- K4: SurfelMap::render*, SurfelMap.cpp:847-1165 ------------------------------------------------------------ */
int sb_map_render(sb_ctx* ctx, const float pose_old[16], const float pose_new[16], float conf_thr, sb_frame* out);
int sb_map_render_active(sb_ctx* ctx, const float pose[16], float conf_thr);   /* SurfelMap.cpp:1023 */
int sb_map_render_inactive(sb_ctx* ctx, const float pose[16], float conf_thr); /* SurfelMap.cpp:1071 */
int sb_map_render_composed(sb_ctx* ctx, const float pose_old[16], const float pose_new[16], float conf_thr);
int sb_map_frame(sb_ctx* ctx, int which, sb_frame** out); /* oldMapFrame/newMapFrame/composedFrame (borrowed) */

/* ---- K5: Frame2Model::jacobianProducts, Frame2Model.cpp:136-261 -------------------------------------------------
 * out48: [0..35] JtWJ (column-major 6x6), [36..41] JtWr, [42] n_valid, [43] F, [44] n_outlier, [45] F_inlier,
 * [46] n_invalid, [47] 0 -- the layout of the reference's 2x8 RGB32F blend target, as doubles.
 * raw32 (optional): the exact Q33.30 fixed-point sums behind out48 (21 lower-triangle + 6 + F + F_inlier) and the
 * three counters; summing raw32 over row stripes / GPUs and calling sb_icp_unpack is bit-identical to one pass. */
int sb_icp_jacobian(sb_ctx* ctx, const sb_frame* data, const sb_frame* model, const double pose[16], int iteration,
                    float max_distance, float max_angle_deg, int row_begin, int row_end, double out48[48],
                    int64_t raw32[32]);
void sb_icp_unpack(const int64_t raw32[32], double out48[48]);

/* ---- LieGaussNewton::minimize, LieGaussNewton.cpp:13-37 (+ step :53-79, Objective::increment Objective.h:45) ----
 * The whole Gauss-Newton loop runs on the device (K5 + 6x6 LDLT + SE3 exp per iteration, no host round trip).
 * history (optional): (max_iter+1)*16 doubles; history_len receives the number of poses pushed. max_iter <= 0 (the
 * reference's "no limit") or > 256 runs at most 256 iterations and is only accepted with history == NULL
 * (SB_ERR_INVALID otherwise).
 * Returns the iteration count k_ in *iters. */
int sb_icp_minimize(sb_ctx* ctx, const sb_frame* data, const sb_frame* model, const double T0[16], int max_iter,
                    double eps, double delta, float max_distance, float max_angle_deg, double pose_out[16],
                    double out48[48], int* iters, double* history, int* history_len);
/* host-side helpers with the library's arithmetic (lie_algebra.cpp:4-71, LieGaussNewton.cpp:60) */
void sb_se3_exp(const double x[6], double T[16]);
void sb_se3_log(const double T[16], double x[6]);
int sb_ldlt_solve6(const double A[36], const double b[6], double x[6]);
int sb_gn_step(const double out48[48], double last_error, double eps, double delta, double pose[16], double dx[6]);

/* ---- K6: SurfelMap::update, SurfelMap.cpp:492-584 (+ paging :708-824) ------------------------------------------ */
/* ---- pose table (DESIGN.md section 12). Each surfel refers to the pose-table entry of the scan that created it. The
 * table starts at the reference's 10 000 entries (SurfelMap.h:205) and doubles, at a call boundary, before any entry at
 * or beyond it is written or referenced: by sb_process_scan / sb_process_scan_timed / sb_map_update (entry
 * sb_map_timestamp), sb_map_set_pose (entry t), sb_map_update_poses / sb_integrate_loop_closures (entries [0, count)),
 * sb_map_upload (the largest entry its surfels refer to) and sb_state_load (the checkpoint's size). The last entry is
 * 16 777 215 (2^24 - 1: the float count field holds larger integers inexactly); a call that needs more returns
 * SB_ERR_CAPACITY, and one whose allocation fails SB_ERR_NOMEM, both before anything changes. sb_reset returns to 10 000.
 * The per-scan product tables inv(P) * poses[t] cover only the entries the active map can refer to: none of this changes
 * a result bit. */
int sb_map_update(sb_ctx* ctx, const float pose[16], const sb_frame* frame);
int sb_map_update_poses(sb_ctx* ctx, const float* poses16, uint32_t count); /* SurfelMap::updatePoses :485 */
int sb_map_size(sb_ctx* ctx, uint32_t* n);                                  /* SurfelMap::size */
int sb_map_timestamp(sb_ctx* ctx, uint32_t* t);
int sb_map_download(sb_ctx* ctx, sb_surfel* dst, uint32_t cap, uint32_t* n); /* SurfelMap::getAllSurfels */
/* test / restore hook: replaces the active map and sets its timestamp; SB_ERR_CAPACITY for a surfel whose count is
   2^24 or more */
int sb_map_upload(sb_ctx* ctx, const sb_surfel* src, uint32_t n, uint32_t timestamp);
int sb_map_set_pose(sb_ctx* ctx, uint32_t t, const float pose[16]); /* any t < 2^24: the table grows to hold it */
/* the pose table's size (capacity) and the window [begin, end) over which the product tables are computed: begin is a
   lower bound on the smallest entry a live surfel of the active map refers to (any pointer may be NULL) */
int sb_pose_table_info(sb_ctx* ctx, uint32_t* capacity, uint32_t* begin, uint32_t* end);
/* intermediates of the last update (any pointer may be NULL): index map (id+1), radius map, integrated flags.
   After sb_map_update the ids index the surfels in order (as sb_map_download returns them); after sb_process_scan they
   are the map's physical slots, which may include slots of surfels removed by in-place updates (same relative order). */
int sb_map_update_debug(sb_ctx* ctx, uint32_t* index_map, float* radius_map4, uint8_t* integrated,
                        uint32_t* n_updated, uint32_t* n_new);
int sb_map_submap_origin(sb_ctx* ctx, int32_t* i, int32_t* j, uint32_t* pending);
/* ---- managed submap tile cache (no counterpart in the reference, whose submapCache_ is host RAM without a bound) ----
 * By default the tiles that leave the active window go into an append-only HBM pool of 16 M surfels: every extraction
 * takes new pool space and a record slot (16384 in all), and a surfel that finds the pool full is dropped (stats[12]).
 * sb_set_tile_cache makes the cache of this context managed: abandoned pool ranges are reclaimed on the device, cold
 * tiles move to pinned host memory and come back from it, and record slots are reused, so that a surfel is dropped only
 * when both tiers are full (counted in stats[12] with the same message). The map's bits do not depend on the tier a tile
 * lived in. pool_surfels: the HBM share, 500 000 <= pool_surfels <= 16 M; host_surfels: surfels that may live in host
 * memory (UINT64_MAX = no bound, as in the reference). Valid while the cache is empty (after sb_create / sb_reset,
 * before the first extraction): SB_ERR_STATE otherwise. Kept across sb_reset; saved and restored by sb_state_save /
 * sb_state_load (a checkpoint of a default context makes the loading context default again). */
int sb_set_tile_cache(sb_ctx* ctx, uint32_t pool_surfels, uint64_t host_surfels);
typedef struct sb_tile_cache_info {
  uint32_t managed, tiles_in_pool, tiles_on_host, pad;
  uint64_t pool_capacity, pool_used, pool_referenced; /* surfels: capacity, used range, held by cached tiles */
  uint64_t host_capacity, host_used;
  uint64_t reclaims, reclaim_moved, evictions, host_fills, dropped; /* pool compactions and the surfels they moved,
                                                                       tiles moved to / re-inserted from the host,
                                                                       surfels dropped (stats[12]) */
} sb_tile_cache_info;
int sb_get_tile_cache_info(sb_ctx* ctx, sb_tile_cache_info* out);

/* ---- SurfelMapping::processScan, SurfelMapping.cpp:175-210 (loop closure off) ---------------------------------- */
int sb_process_scan(sb_ctx* ctx, const float* pts4, const float* labels, const float* probs, uint32_t n,
                    int pts_on_device);
/* ---- per-point deskewing (no counterpart in the reference; DESIGN.md section 11) ----------------------------------
 * A spinning LiDAR measures its points over a whole sweep. With deskewing on, preprocessing first moves every point to
 * the scan's reference time with the motion the next Gauss-Newton run starts from (M = lastIncrement_: identity at
 * timestamp 0, after sb_reset and after a reset load; after sb_state_load what the checkpoint holds; the same with
 * initialize_identity on or off; after a track-loss recovery the recovery's increment, as for the initial guess):
 *   p' = Exp((s - s_ref) w) p + (s - s_ref) t,   w = log_SO3(R_M), t = t_M (fp64 once per scan, rounded to fp32)
 * with s in [0, 1] the point's sweep time: mode 1 the caller's per-point time (clamped; non-finite -> s_ref), mode 2
 * frac(dir (a0 - yaw) / 2pi) of the point's azimuth, dir = +1 for a clockwise spin (the defaults a0 = +pi, clockwise give
 * the range image's column fraction). Everything after the projection sees p'. When s == s_ref or M rounds to the
 * identity, the point's bits pass through: with zero motion deskewing on gives the bits of deskewing off. */
typedef struct sb_deskew_params {
  int32_t mode;        /* 0 off, 1 per-point times, 2 azimuth */
  float ref_time;      /* s_ref in [0, 1]: the sweep time the scan's pose refers to */
  float start_azimuth; /* a0, radians (mode 2) */
  int32_t clockwise;   /* mode 2 */
} sb_deskew_params;
void sb_default_deskew(sb_deskew_params* p); /* off, 0.5, +pi, clockwise */
/* SB_ERR_INVALID for a mode outside {0, 1, 2}, a ref_time outside [0, 1] or not finite, a non-finite start_azimuth.
 * Valid at any time; kept across sb_reset; saved by sb_state_save when on (a checkpoint without it loads with it off). */
int sb_set_deskew(sb_ctx* ctx, const sb_deskew_params* p);
int sb_get_deskew(sb_ctx* ctx, sb_deskew_params* p);
/* sb_process_scan with per-point times (float, one per point). times follow pts_on_device: device memory when it is set,
 * host memory otherwise; sb_prefetch_scan does not stage them (this call uploads them itself). SB_ERR_INVALID, before
 * anything changes, for mode 1 without times and for times while the mode is not 1. sb_process_scan is this call with
 * times = NULL. */
int sb_process_scan_timed(sb_ctx* ctx, const float* pts4, const float* labels, const float* probs, const float* times,
                          uint32_t n, int pts_on_device);
/* sb_preprocess with deskewing by an explicit motion (column-major, NULL = identity) and setting, for tests and tools */
int sb_preprocess_deskew(sb_ctx* ctx, const float* pts4, const float* labels, const float* probs, const float* times,
                         uint32_t n, uint32_t timestamp, const sb_deskew_params* d, const double motion[16],
                         int pts_on_device, sb_frame* out);
/* Optional input double buffering (no counterpart in the reference, which uploads inside processScan,
 * SurfelMapping.cpp:325-331): start the host-to-device copy of the NEXT scan on a separate copy stream; a following
 * sb_process_scan with the same host pointers / count (on_device = 0) uses the staged copy. At most two scans staged. */
int sb_prefetch_scan(sb_ctx* ctx, const float* pts4, const float* labels, const float* probs, uint32_t n);
/* ---- per-point labels (no counterpart in the reference; DESIGN.md section 13) -------------------------------------
 * With the mode on, every sb_process_scan / sb_process_scan_timed leaves one 32-byte record per input point, in input
 * order, for SemanticKITTI-style tools that want one label per point. Every field is an exact function of the point and
 * of what the scan computed:
 *   pixel        y * data_width + x of the data pixel the projection gives the point (the deskewed point p' when
 *                deskewing is on); -1 when the point enters no pixel: non-finite, the origin, clipped by the field of view
 *                or the seam, z outside [-1, 1], or at the clear depth
 *   flags        SB_POINT_WON: the pixel's depth test kept this point (ties: the lowest index, GL_LESS in buffer order);
 *                SB_POINT_VERTEX: the frame's vertex at pixel has w > 0 (clear for the movable winner of a scan before
 *                timestamp 10); SB_POINT_INTEGRATED: this scan's map update fused the pixel into an existing surfel (the
 *                flag of sb_map_update_debug); SB_POINT_MAP: the model vertex at map_pixel has w > 0
 *   frame_label / frame_prob  rintf(255 sem.x) and sem.w of the current frame's semantic image at pixel: the pixel's
 *                label after the Q1 pairing, erosion and flood fill, not the point's own input label
 *   map_pixel    y * model_width + x of p' under the model image's projection (no depth range); -1 when pixel is -1
 *   map_label / map_prob / map_range  label and probability of the current model frame at map_pixel and |v| of its
 *                vertex ((x*x + y*y) + z*z in fp32), when SB_POINT_MAP is set, else 0. That frame is the map after the
 *                scan's update rendered at the scan's pose; with render_after_update = 0 there is none and the flag is
 *                never set.
 * Labels decode with one fp32 expression, so ids up to 65535 round-trip. */
enum { SB_POINT_WON = 1, SB_POINT_VERTEX = 2, SB_POINT_INTEGRATED = 4, SB_POINT_MAP = 8 };
typedef struct sb_point_label {
  int32_t pixel;
  uint32_t flags; /* SB_POINT_* */
  uint32_t frame_label;
  float frame_prob;
  int32_t map_pixel;
  uint32_t map_label;
  float map_prob;
  float map_range;
} sb_point_label; /* 32 bytes */
/* Valid at any time; kept across sb_reset; not part of a checkpoint (its bytes do not depend on the mode). With the mode
 * off the scan pipeline launches exactly what it launches without this feature. Records exist from the first scan after
 * the mode is turned on; sb_reset, sb_state_load, sb_set_params and turning the mode off drop them. The record buffer
 * grows with the scan: a scan whose allocation fails returns SB_ERR_NOMEM before it changes anything. */
int sb_set_point_labels(sb_ctx* ctx, int on);
/* The records of the last scan. *n is always set (0 while none exist); SB_ERR_STATE while none exist, SB_ERR_INVALID
 * (nothing written) when cap < *n. dst_on_device != 0: dst is device memory (a device-to-device copy). */
int sb_get_point_labels(sb_ctx* ctx, sb_point_label* dst, uint32_t cap, uint32_t* n, int dst_on_device);
/* ---- loop closure: SurfelMapping::checkLoopClosure, core/SurfelMapping.cpp:478-795 ("close-loops", default.xml:70-76) ----
 * When enabled, sb_process_scan runs the reference's detection / verification between updatePose() and updateMap()
 * (:196-200): render_inactive at a candidate pose, three Gauss-Newton runs against the old map frame, render_composed,
 * residual comparison, verification over consecutive scans, and the chained "old" pose (currentPose_old_) that the next
 * scan's composed rendering uses. The pose-graph OPTIMISATION (gtsam, core/Posegraph.cpp) stays with the host application:
 * the library records what the reference feeds into gtsam (sb_get_loop_edges: odometry + loop edges; initial poses =
 * the odometry chain) and raises optimisation_requested; optimised poses come back through
 * sb_integrate_loop_closures (integrateLoopClosures, :212-258). */
typedef struct sb_loop_params {
  float search_distance;         /* loop-search-distance (default.xml: 50) */
  float min_trajectory_distance; /* loop-min-trajectory-distance (SurfelMapping.h:224: 200) */
  int32_t min_verifications;     /* loop-min-verifications (5) */
  float residual_threshold;      /* loop-residual-threshold (1.15) */
  float outlier_threshold;       /* loop-outlier-threshold (1.1) */
  float valid_threshold;         /* loop-valid-threshold (0.95) */
} sb_loop_params;
typedef struct sb_loop_info {
  uint32_t enabled, loop_count, time_without_loop_closure, candidates_tested, loop_edges_added, unverified;
  uint32_t already_verified, found_candidate, use_candidate, optimisation_requested;
  int32_t last_added_candidate;
  uint32_t n_edges, n_poses;
  float valid_ratio, outlier_ratio, rel_error; /* statistics_["loop_valid_ratio" / "loop_outlier_ratio" / "loop_relative_error_all"] */
  double residual_old, residual_new;
  double current_pose_old[16];                 /* currentPose_old_ after the check */
} sb_loop_info;
typedef struct sb_loop_edge {
  int32_t from, to;
  double rel_pose[16];
} sb_loop_edge;
void sb_default_loop_params(sb_loop_params* p);
int sb_set_loop_closure(sb_ctx* ctx, int enabled, const sb_loop_params* p /* NULL = defaults */);
int sb_get_loop_info(sb_ctx* ctx, sb_loop_info* out);
int sb_get_loop_edges(sb_ctx* ctx, sb_loop_edge* dst, uint32_t cap, uint32_t* n_total);
/* SurfelMapping::integrateLoopClosures, core/SurfelMapping.cpp:212-258, called by the reference at the top of processScan
 * once its asynchronous gtsam run has finished: poses16 = the optimised poses of scans 0 .. n-1 (column-major doubles; n >=
 * the scan the request was raised at + 1; NULL = leave the graph's poses as they are). Later poses and the current pose are
 * carried along, loop_count and the trajectory distances are updated, the map's pose table is rewritten
 * (SurfelMap::updatePoses). *integrated = number of poses written, 0 if no request was pending. */
int sb_integrate_loop_closures(sb_ctx* ctx, const double* poses16, uint32_t n, uint32_t* integrated);
int sb_set_current_pose(sb_ctx* ctx, const double pose[16]); /* SurfelMapping::setCurrentPose, core/SurfelMapping.h:66 */

int sb_get_pose(sb_ctx* ctx, double pose[16]);     /* getCurrentPose */
int sb_get_last_pose(sb_ctx* ctx, double pose[16]); /* getLastPose, core/SurfelMapping.h:63 (pose before the last processScan) */
int sb_timestamp(sb_ctx* ctx, uint32_t* t);        /* timestamp() */
int sb_slam_frame(sb_ctx* ctx, int which, sb_frame** out); /* getCurrentFrame / LastFrame / *ModelFrame (borrowed) */
/* stats[16]: [0] icp iterations [1] F [2] inlier [3] outlier [4] invalid [5] inlier_residual [6] track losses
 * [7] surfels; wall seconds: [11] complete (getStatistics key "complete-time"); the reference's three stage timers have
 * no counterpart -- the stages overlap on the stream -- so their slots [8] [9] [10] carry the host-side split of the
 * call: enqueue / wait for the device / bookkeeping after the wait;
 * [12] surfels dropped because the HBM cache of extracted submap tiles (16 M surfels) was full -- the reference's
 * host-side submapCache_ is unbounded; sb_last_error carries the message (with sb_set_tile_cache: both tiers full) */
int sb_get_statistics(sb_ctx* ctx, double stats[16]);

/* ---- checkpoint / resume (no counterpart in the reference: its Posegraph::save/load are empty stubs) --------------
 * A checkpoint holds everything the next scan depends on: the live surfels in order, the used part of the HBM tile pool
 * with its records and bookkeeping, both pose tables, the device pose block, the SLAM poses, statistics, the seven frames,
 * the loop-closure state, the sb_params and the loop parameters. N scans, save, load into a fresh context, M scans give
 * the bits of N + M scans without a break. Format (DESIGN.md section 9): little-endian header (magic, format version,
 * SB_VERSION, sizeof(sb_surfel), pose capacity, image sizes, total size, sb_params, loop parameters), length-prefixed
 * sections, a 64-bit digest of everything before it. save(load(save(x))) == save(x) byte for byte.
 *  - sb_state_save does not change the context; sb_state_size is the exact size of a checkpoint taken now.
 *  - sb_state_load restores into any context created with the same image sizes, applies the saved sb_params (validated as
 *    sb_set_params does) and drops the render memo. A bad header, a size mismatch or a truncated buffer returns
 *    SB_ERR_INVALID before anything changes; a digest mismatch returns SB_ERR_INVALID with the context reset (sb_reset).
 *  - a save or a load that goes ahead drops the scans staged by sb_prefetch_scan (a checkpoint neither carries nor consumes
 *    them); a call refused for its arguments, a too small buffer or a bad header leaves them staged; a load refused for
 *    its digest has dropped them with the rest of the context's state.
 *  - both return SB_ERR_STATE while a multi-GPU exchange is set up.
 *  - a map with surfels removed in place is restored dense: only the physical slot ids that sb_map_update_debug reports
 *    after the next sb_process_scan can differ
 *  - the header's pose capacity is the context's pose-table size (10 000 unless the table grew). A load accepts sizes
 *    from 10 000 to 2^24 and gives the loading context the checkpoint's size (SB_ERR_NOMEM, nothing changed, when that
 *    allocation fails); libraries without a growing table refuse a checkpoint of a grown one. */
int sb_state_size(sb_ctx* ctx, uint64_t* bytes);
int sb_state_save(sb_ctx* ctx, void* dst, uint64_t cap, uint64_t* written);
int sb_state_load(sb_ctx* ctx, const void* src, uint64_t n);

/* ---- per-kernel device time (CUDA events on the context's stream around every launch; off by default) ------------ */
int sb_profile_enable(sb_ctx* ctx, int on);
int sb_profile_kernels(void);              /* number of kernel classes */
const char* sb_profile_name(int id);
/* sums since the last collect: total_ms[id], count[id]; cap >= sb_profile_kernels(). Synchronises the stream. */
int sb_profile_collect(sb_ctx* ctx, double* total_ms, uint64_t* count, int cap);

/* ---- multi-GPU: row-striped K5 with a one-shot peer-memory all-reduce of the 32 fixed-point sums ---------------
 * Every rank calls sb_comm_export to obtain an opaque 64-byte handle of its mailbox (each call clears the mailbox and
 * starts a new session: export again before every sb_comm_init, and only after all ranks have left the previous
 * session), exchanges the handles out of band (e.g. torch.distributed.all_gather) and passes all of them to
 * sb_comm_init; a barrier between the ranks must follow before the first striped call. Waiting inside the kernel is
 * bounded (10 s): a rank that never arrives makes the call fail with SB_ERR_STATE instead of hanging. Afterwards sb_icp_minimize /
 * sb_process_scan reduce the sums over ranks inside the Jacobian kernel. rows [row_begin,row_end) of the data image
 * belong to this rank. */
int sb_comm_export(sb_ctx* ctx, uint8_t handle[64]);
int sb_comm_init(sb_ctx* ctx, int rank, int nranks, const uint8_t* handles /* nranks*64 */, int row_begin,
                 int row_end);
int sb_comm_shutdown(sb_ctx* ctx);
/* Baseline exchange: the library calls `fn(user, sums32)` once per Gauss-Newton iteration with this rank's 32 int64
 * partial sums; the callback all-reduces them in place (e.g. torch.distributed / NCCL / MPI on the host side). The
 * loop then runs on the host (one K5 launch + read-back per iteration). fn == NULL switches the mode off. */
typedef int (*sb_allreduce_fn)(void* user, int64_t* sums32);
int sb_comm_set_callback(sb_ctx* ctx, sb_allreduce_fn fn, void* user, int row_begin, int row_end);

#ifdef __cplusplus
}
#endif
#endif /* SUMA_B200_H_ */
