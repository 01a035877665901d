// sb_api.cu -- the C ABI of libsuma_b200 (include/suma_b200.h): context, frames, the operator-level entry points
// (Preprocessing::process, SurfelMap::render*/update, Frame2Model::jacobianProducts, LieGaussNewton::minimize) and the
// per-scan orchestration of SurfelMapping::processScan (core/SurfelMapping.cpp:175-210, 323-358, 372-476, 797-804).
// There is no CPU fallback: without a CUDA device sb_create fails with SB_ERR_NOGPU.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "sb_gn.cuh"
#include "sb_internal.cuh"
#include "../../include/suma_b200_loop.hpp"

using namespace sb;

struct sb_frame {
  sb_ctx* ctx;
  uint64_t id;  // unique within the context, never reused (keys the render memo)
  FrameDev d;   // views into base
  DevPtr<float4> base;
};
using FramePtr = Owned<sb_frame, std::default_delete<sb_frame>>;

struct DevTile {  // SubmapCache, SurfelMap.h:179-181 -- kept in HBM (tile pool) instead of host RAM
  uint32_t slot = 0;
  bool known = false;  // base / count read back from the device record
  uint32_t base = 0, count = 0;
};

struct sb_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  sb_params p;
  KParams kp;
  std::string err;
  uint64_t launches = 0;
  Profiler prof;

  // ---- preprocessing scratch
  PrepKeys prep;            // two alternating z-buffer key images of the scan projection (+ TMA maps)
  bool prepped_for_update = false;  // radius map / index keys / integrated flags of c->cur are ready (pipeline mode)
  DevPtr<float4> d_pts;
  DevPtr<float> d_labels;
  DevPtr<float> d_probs;
  size_t pts_cap = 0;
  // optional input prefetch (sb_prefetch_scan): a ring of staging buffers filled on a copy stream while the previous
  // scan is being processed; created on first use, the default path never touches it
  struct PrefetchSlot {
    DevPtr<float4> pts;
    DevPtr<float> labels;
    DevPtr<float> probs;
    const float* host_pts = nullptr;
    uint32_t n = 0;
    bool has_labels = false, has_probs = false, valid = false, in_use = false;
    cudaEvent_t done = nullptr;      // copy finished (recorded on the copy stream)
    cudaEvent_t released = nullptr;  // every kernel that read the slot has been enqueued before this (compute stream)
    bool has_released = false;
  };
  PrefetchSlot prefetch[3];
  cudaStream_t copy_stream = nullptr;

  // ---- ICP
  DevPtr<GnState> gn;
  DevPtr<GnState> gn2;  // state of the frame-to-frame fallback minimisation
  DevPtr<long long> acc_slots;  // per-block partial sums of the Jacobian kernels (1024 x 32 int64)
  DevPtr<unsigned int> ticket;
  // pinned staging of the small read-backs and uploads; one member per transfer, so none overlaps another
  struct Staging {
    ResultBlock result;                      // mirror of the per-scan result block (also stages the initial pose block)
    GnHead gn;                               // head of a Gauss-Newton state
    long long sums[32];                      // raw sums of one Jacobian pass
    double history[(kMaxGnIter + 1) * 16];   // poses of a host-driven Gauss-Newton run
  };
  PinnedPtr<Staging> host;
  int icp_blocks = 296;
  int icp_coop_blocks = 0;  // grid of the persistent cooperative Gauss-Newton kernel
  unsigned int epoch_base = 1;  // epoch words of the persistent GN kernel: each launch owns a fresh range of values
  DevPtr<unsigned long long> gn_pub;  // 32 (half pose value, epoch tag) words published by every Gauss-Newton step
  // loop closure (SurfelMapping::checkLoopClosure; include/suma_b200_loop.hpp): off unless sb_set_loop_closure enables it
  bool close_loops = false;
  suma_b200::loop::State loop;
  double lastPose_old[16];

  // ---- map
  // current surfels, updated (same index), generated (per pixel), extraction buffer: views into the *_mem allocations
  SurfelPlanes A{}, T{}, G{}, X{};
  DevPtr<float4> A_mem, T_mem, G_mem, X_mem;
  // liveness byte per slot of A, valid below the physical end: set by every writer of a slot, cleared only by the
  // in-place map update (a surfel it removes stays where it is, dead, until the next compaction)
  DevPtr<uint8_t> live;
  DevPtr<uint8_t> keep;
  DevPtr<uint32_t> block_counts;
  DevPtr<unsigned long long> lb_desc;  // look-back descriptors of the single-pass compactions
  DevPtr<uint32_t> lb_ticket;
  uint32_t lb_gen = 0;
  DevPtr<ResultBlock> res;  // pose block, statistics sums and surfel counts of the scan
  DevPtr<float> poses;      // device pose table, kMaxPoses x 16
  DevPtr<float> poses_inv;
  std::vector<float> h_poses, h_poses_inv;
  DevPtr<float> Mtab_old;
  DevPtr<float> Mtab_new;
  DevPtr<unsigned long long> key_old;  // three model-size key images, contiguous
  unsigned long long* key_new = nullptr;
  unsigned long long* key_comp = nullptr;
  DevPtr<unsigned long long> key_index;
  DevPtr<float4> radius_map;
  DevPtr<uint8_t> integrated;
  DevPtr<uint32_t> group_counts;  // kGroupCounts totals of the update pass / a tile extraction (64 blocks each)
  FramePtr f_old, f_new, f_comp;
  uint64_t frames_created = 0;
  uint32_t n_host = 0;   // physical end of the surfel slots (exact; refreshed after every update)
  uint32_t n_holes = 0;  // dead slots below n_host: the map holds n_host - n_holes surfels
  bool lazy_update = false;  // the map update in flight is the in-place one (its counts[5] is the new n_holes)
  uint32_t n_upper = 0;  // upper bound used for grid sizing while the exact count is still in flight
  uint32_t n_updated = 0, n_new = 0;
  uint32_t map_timestamp = 0;
  // one past the largest pose-table entry a surfel of the map or of a cached tile can refer to (creation timestamp,
  // clamped as pose_index() does): while it is <= map_timestamp, no surfel reads the entry the scan's pose goes into
  uint32_t pose_ref_end = 0;
  int32_t origin_i = 0, origin_j = 0;
  std::vector<std::pair<int32_t, int32_t>> extraction;
  std::map<std::pair<int32_t, int32_t>, DevTile> tiles;
  SurfelPlanes pool{};            // tile cache lanes
  DevPtr<float4> pool_mem;
  DevPtr<uint2> d_tile_rec;       // {end in the pool, surfels of the tile} per extraction; slot s starts at the end of s - 1
  uint32_t n_slots = 0;
  bool tiles_pending = false;     // some records have not been read back yet

  // Full-render memo: SurfelMapping re-renders the unchanged map at the unchanged pose at the start of the next scan
  // (SurfelMapping.cpp:351 after :803); identical arguments on an unmodified map reproduce identical images. The memo
  // holds while nothing but that render has written the frames it covers (old, new, composed and `out`: see
  // frame_written) and nothing the render reads has changed (map_version, sb_set_params, sb_set_current_pose).
  struct RenderMemo {
    struct Key {
      float pose_old[16], pose_new[16];
      float conf_thr;
      uint32_t map_timestamp;
      uint64_t map_version;
      uint64_t out;  // sb_frame::id
      int compose;
      int pad;       // no padding bytes: keys are compared with memcmp
    };
    static_assert(sizeof(Key) == 160, "RenderMemo::Key has padding");
    Key key{};
    bool valid = false;
    bool matches(const Key& k) const { return valid && memcmp(&key, &k, sizeof(k)) == 0; }
    void store(const Key& k) {
      key = k;
      valid = true;
    }
    void clear() { valid = false; }
  } memo;
  uint64_t map_version = 0;
  uint64_t renders_skipped = 0;

  // ---- SurfelMapping state
  FramePtr cur, last, cur_model, last_model;
  uint32_t timestamp = 0;
  double currentPose[16], lastPose[16], currentPose_old[16], currentPose_new[16], lastIncrement[16];
  float confidence_threshold = 0.f, log_unstable_slam = 0.f;
  double stats[16];
  uint32_t trackLoss = 0;
  bool cur_has_semantics = false, last_has_semantics = false;

  // ---- multi-GPU
  DevPtr<long long> mailbox;
  DevPtr<unsigned int> comm_epoch;
  CommDev comm{};
  bool comm_on = false;
  sb_allreduce_fn comm_cb = nullptr;  // host-side exchange (baseline); exclusive with the fused peer-memory mode
  void* comm_cb_user = nullptr;
  int row_begin = 0, row_end = 0;
  std::vector<void*> peer_ptrs;

  // ---- checkpoints (sb_state_save / sb_state_load): a pinned double buffer for the chunked copies, its two events and the
  // device digest accumulator; created on first use, so contexts that never checkpoint pay nothing
  PinnedPtr<uint8_t> state_stage;
  cudaEvent_t state_ev[2] = {nullptr, nullptr};
  DevPtr<unsigned long long> state_acc;
};

namespace {

int fail(sb_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}

#define SB_CUDA(ctx, call)                                                                              \
  do {                                                                                                  \
    cudaError_t e__ = (call);                                                                           \
    if (e__ != cudaSuccess)                                                                             \
      return fail(ctx, SB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));               \
  } while (0)

Launch L_(sb_ctx* c) { return Launch{c->stream, &c->launches, &c->prof}; }

void ident_d(double* M) {
  for (int i = 0; i < 16; ++i) M[i] = (i % 5 == 0) ? 1.0 : 0.0;
}
Mat4 mat4_from(const float* m) {
  Mat4 r;
  memcpy(r.m, m, 64);
  return r;
}
void cast_f(const double* M, float* F) {
  for (int i = 0; i < 16; ++i) F[i] = (float)M[i];
}
double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
float deg2rad_f(float d) { return d * (float)(3.14159265358979323846 / 180.0); }

// host-side derived constants: SurfelMap.cpp:336-457, Preprocessing.cpp:76-117, Frame2Model.cpp:65-110
void derive(sb_ctx* c) {
  const sb_params& p = c->p;
  KParams& k = c->kp;
  memset(&k, 0, sizeof(k));
  k.W = p.data_width; k.H = p.data_height; k.Wm = p.model_width; k.Hm = p.model_height;
  k.fov_up = fabsf(p.data_fov_up); k.fov = fabsf(p.data_fov_up) + fabsf(p.data_fov_down);
  k.min_depth = p.min_depth; k.max_depth = p.max_depth;
  k.m_fov_up = fabsf(p.model_fov_up); k.m_fov = fabsf(p.model_fov_up) + fabsf(p.model_fov_down);
  k.m_min_depth = p.model_min_depth; k.m_max_depth = p.model_max_depth;
  k.weighting = p.weighting; k.bilinear = p.bilinear_sampling; k.factor = p.factor;
  k.use_stability = p.use_stability; k.unstable_age = p.unstable_age; k.confidence_mode = p.confidence_mode;
  k.active_timestamps = p.active_timestamps; k.weighting_scheme = p.weighting_scheme;
  k.averaging_scheme = p.averaging_scheme; k.update_always = p.update_always;
  k.confidence_threshold = p.confidence_threshold; k.p_stable = p.p_stable;
  k.p_unstable = 1.0f - p.p_stable;                                   // SurfelMap.cpp:347
  k.log_prior = (float)log(p.p_prior / (1.0 - p.p_prior));            // :349
  k.log_unstable = (float)log(k.p_unstable / (1.0 - k.p_unstable));   // :350
  k.sigma_angle = p.sigma_angle; k.sigma_distance = p.sigma_distance; k.max_weight = p.max_weight;
  float vfov = fabsf(p.data_fov_up) + fabsf(p.data_fov_down);         // :339-344
  float vpix = (float)tan(0.5f * ((double)vfov * 3.14159265358979323846 / 180.0) / (uint32_t)p.data_height);
  float hpix = (float)tan(0.5f * ((double)360.0f * 3.14159265358979323846 / 180.0) / (uint32_t)p.data_width);
  k.pixel_size = vpix > hpix ? vpix : hpix;
  k.min_radius = p.min_radius; k.max_radius = p.max_radius;
  k.radconf_angle_thresh = (float)cos((double)deg2rad_f(p.max_angle));     // :395
  k.update_angle_thresh = (float)sin((double)deg2rad_f(p.map_max_angle));  // :407
  k.map_max_distance = p.map_max_distance;
  k.max_loop_closure_distance = p.max_loop_closure_distance;
  k.label_offset_quirk = p.label_offset_quirk;
  c->confidence_threshold = p.confidence_threshold;  // SurfelMapping.cpp:111-113
  float pu = 0.1f;
  c->log_unstable_slam = logf(pu / (1.0f - pu));     // SurfelMapping.cpp:108-109
}

int alloc_planes(sb_ctx* c, DevPtr<float4>& mem, SurfelPlanes* s, size_t n) {
  SB_CUDA(c, dev_alloc(mem, n * 4 * sizeof(float4)));
  s->p0 = mem; s->p1 = mem + n; s->p2 = mem + 2 * n; s->p3 = mem + 3 * n;
  return SB_OK;
}

int frame_create(sb_ctx* c, int w, int h, FramePtr& out) {
  if (!c || w <= 0 || h <= 0) return fail(c, SB_ERR_INVALID, "frame_create: bad arguments");
  FramePtr f(new sb_frame());
  f->ctx = c;
  f->id = ++c->frames_created;
  size_t P = (size_t)w * h;
  cudaError_t e = dev_alloc(f->base, P * 3 * sizeof(float4));
  if (e != cudaSuccess) return fail(c, SB_ERR_NOMEM, std::string("frame alloc: ") + cudaGetErrorString(e));
  cudaMemsetAsync(f->base, 0, P * 3 * sizeof(float4), c->stream);
  f->d.W = w; f->d.H = h;
  f->d.vertex = f->base; f->d.normal = f->base + P; f->d.semantic = f->base + 2 * P;
  out = std::move(f);
  return SB_OK;
}

// Every write to a frame other than the memoised render itself goes through here: the memo is dropped when it covers
// the frame (the map's old / new / composed frames, or the `out` frame of the memoised render).
void frame_written(sb_ctx* c, const sb_frame* f) {
  if (f == c->f_old || f == c->f_new || f == c->f_comp || f->id == c->memo.key.out) c->memo.clear();
}

int reset_state(sb_ctx* c) {
  // SurfelMap::reset (SurfelMap.cpp:473-482) + the SurfelMapping members set up in its constructor
  c->map_version += 1;
  c->n_host = 0; c->n_holes = 0; c->lazy_update = false;
  c->n_updated = 0; c->n_new = 0; c->map_timestamp = 0; c->pose_ref_end = 0;
  c->origin_i = c->origin_j = 0;
  c->extraction.clear();
  c->tiles.clear();
  c->n_slots = 0;
  c->tiles_pending = false;
  c->stats[12] = 0.0;
  c->loop.reset();  // posegraph_->clear(); trajectory_distances_ ... (SurfelMapping.cpp:158-163)
  for (int i = 0; i < 16; ++i) c->lastPose_old[i] = (i % 5 == 0) ? 1.0 : 0.0;
  c->h_poses.assign((size_t)kMaxPoses * 16, 0.0f);
  for (uint32_t t = 0; t < kMaxPoses; ++t)
    for (int i = 0; i < 4; ++i) c->h_poses[16 * (size_t)t + 5 * i] = 1.0f;
  c->h_poses_inv = c->h_poses;
  SB_CUDA(c, cudaMemcpyAsync(c->poses, c->h_poses.data(), (size_t)kMaxPoses * 64, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemcpyAsync(c->poses_inv, c->h_poses.data(), (size_t)kMaxPoses * 64, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemsetAsync(c->res->counts, 0, sizeof(c->res->counts), c->stream));
  c->timestamp = 0;
  ident_d(c->currentPose); ident_d(c->lastPose); ident_d(c->currentPose_old); ident_d(c->currentPose_new);
  ident_d(c->lastIncrement);
  memset(c->stats, 0, sizeof(c->stats));
  c->trackLoss = 0;
  c->n_upper = 0;
  {
    // staged in the context's own pinned buffer (read by the async copy until the synchronize at the end of this
    // function; no other transfer of this context is in flight here): contexts reset concurrently share nothing
    PoseDev& h = c->host->result.pose;
    memset(&h, 0, sizeof(h));
    ident_d(h.currentPose); ident_d(h.lastPose); ident_d(h.lastIncrement); ident_d(h.increment); ident_d(h.T0);
    for (int i = 0; i < 4; ++i) h.P_active.m[5 * i] = h.invP_active.m[5 * i] = h.P_cur.m[5 * i] = h.invP_cur.m[5 * i] = 1.0f;
    SB_CUDA(c, cudaMemcpyAsync(&c->res->pose, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  }
  c->cur_has_semantics = c->last_has_semantics = false;
  for (const sb_frame* f : {c->f_old.get(), c->f_new.get(), c->f_comp.get(), c->cur.get(), c->last.get(),
                           c->cur_model.get(), c->last_model.get()})
    SB_CUDA(c, cudaMemsetAsync(f->base, 0, (size_t)f->d.W * f->d.H * 3 * sizeof(float4), c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}

int alloc_buffers(sb_ctx* c) {
  const sb_params& p = c->p;
  size_t Pd = (size_t)p.data_width * p.data_height, Pm = (size_t)p.model_width * p.model_height;
  SB_CUDA(c, dev_alloc(c->res, sizeof(ResultBlock)));
  SB_CUDA(c, cudaMemsetAsync(c->res, 0, sizeof(ResultBlock), c->stream));
  const size_t Pk = preprocess_key_elems(p.data_width, p.data_height);
  for (int i = 0; i < 2; ++i) {
    SB_CUDA(c, dev_alloc(c->prep.img[i], Pk * 8));
    // TMA staging of the key tiles wherever the device has a TMA unit: measured 2 % (64x2048) / 1.5 % (128x4096)
    // faster than plain loads (DESIGN.md section 4)
    c->prep.tmap_ok[i] = make_key_tensor_map(&c->prep.tmap[i], c->prep.img[i], p.data_width, p.data_height);
  }
  c->pts_cap = Pd * 2 + 1024;
  SB_CUDA(c, dev_alloc(c->d_pts, c->pts_cap * 16));
  SB_CUDA(c, dev_alloc(c->d_labels, c->pts_cap * 4));
  SB_CUDA(c, dev_alloc(c->d_probs, c->pts_cap * 4));
  SB_CUDA(c, dev_alloc(c->gn, sizeof(GnState)));
  SB_CUDA(c, dev_alloc(c->gn2, sizeof(GnState)));
  SB_CUDA(c, cudaMemsetAsync(c->gn2, 0, sizeof(GnState), c->stream));
  SB_CUDA(c, dev_alloc(c->acc_slots, 1024 * 32 * sizeof(long long)));
  SB_CUDA(c, cudaMemsetAsync(c->acc_slots, 0, 1024 * 32 * sizeof(long long), c->stream));
  SB_CUDA(c, dev_alloc(c->ticket, 128));
  SB_CUDA(c, dev_alloc(c->gn_pub, 64 * 8));
  SB_CUDA(c, cudaMemsetAsync(c->gn_pub, 0, 64 * 8, c->stream));
  SB_CUDA(c, cudaMemsetAsync(c->ticket, 0, 128, c->stream));
  {
    void* h = nullptr;
    SB_CUDA(c, cudaMallocHost(&h, sizeof(sb_ctx::Staging)));
    c->host.reset(static_cast<sb_ctx::Staging*>(h));
  }
  int r;
  if ((r = alloc_planes(c, c->A_mem, &c->A, kMaxSurfels))) return r;
  if ((r = alloc_planes(c, c->T_mem, &c->T, kMaxSurfels))) return r;
  if ((r = alloc_planes(c, c->G_mem, &c->G, Pd))) return r;
  if ((r = alloc_planes(c, c->X_mem, &c->X, 16))) return r;
  if ((r = alloc_planes(c, c->pool_mem, &c->pool, kTilePoolCap))) return r;
  SB_CUDA(c, dev_alloc(c->d_tile_rec, (size_t)kMaxTileSlots * sizeof(uint2)));
  SB_CUDA(c, dev_alloc(c->live, kMaxSurfels));
  SB_CUDA(c, dev_alloc(c->keep, kMaxSurfels));
  size_t nb = (kMaxSurfels + 127) / 128 + 16;  // blocks of the finest-grained surfel kernel
  SB_CUDA(c, dev_alloc(c->block_counts, nb * 4));
  SB_CUDA(c, dev_alloc(c->lb_desc, (nb + 16) * 8));
  SB_CUDA(c, cudaMemsetAsync(c->lb_desc, 0, (nb + 16) * 8, c->stream));
  SB_CUDA(c, dev_alloc(c->lb_ticket, 64));
  SB_CUDA(c, cudaMemsetAsync(c->lb_ticket, 0, 64, c->stream));
  SB_CUDA(c, dev_alloc(c->poses, (size_t)kMaxPoses * 64));
  SB_CUDA(c, dev_alloc(c->poses_inv, (size_t)kMaxPoses * 64));
  SB_CUDA(c, dev_alloc(c->Mtab_old, (size_t)kMaxPoses * 64));
  SB_CUDA(c, dev_alloc(c->Mtab_new, (size_t)kMaxPoses * 64));
  SB_CUDA(c, dev_alloc(c->key_old, Pm * 8 * 3));
  c->key_new = c->key_old + Pm;
  c->key_comp = c->key_old + 2 * Pm;
  SB_CUDA(c, cudaMemsetAsync(c->key_old, 0xff, Pm * 8 * 3, c->stream));
  for (int i = 0; i < 2; ++i) SB_CUDA(c, cudaMemsetAsync(c->prep.img[i], 0xff, Pk * 8, c->stream));
  c->prep.cur = 0;
  SB_CUDA(c, dev_alloc(c->key_index, Pd * 8));
  SB_CUDA(c, dev_alloc(c->radius_map, Pd * 16));
  SB_CUDA(c, dev_alloc(c->integrated, Pd));
  SB_CUDA(c, dev_alloc(c->group_counts, kGroupCounts * 4));
  SB_CUDA(c, cudaMemsetAsync(c->group_counts, 0, kGroupCounts * 4, c->stream));
  SB_CUDA(c, dev_alloc(c->comm_epoch, 64));
  SB_CUDA(c, cudaMemsetAsync(c->comm_epoch, 0, 64, c->stream));
  if ((r = frame_create(c, p.model_width, p.model_height, c->f_old))) return r;
  if ((r = frame_create(c, p.model_width, p.model_height, c->f_new))) return r;
  if ((r = frame_create(c, p.model_width, p.model_height, c->f_comp))) return r;
  if ((r = frame_create(c, p.data_width, p.data_height, c->cur))) return r;
  if ((r = frame_create(c, p.data_width, p.data_height, c->last))) return r;
  if ((r = frame_create(c, p.model_width, p.model_height, c->cur_model))) return r;
  if ((r = frame_create(c, p.model_width, p.model_height, c->last_model))) return r;
  return reset_state(c);
}

uint32_t n_grid(const sb_ctx* c) { return c->n_upper > c->n_host ? c->n_upper : c->n_host; }

uint32_t n_live(const sb_ctx* c) { return c->n_host - c->n_holes; }

int t_threshold(const sb_ctx* c) { return (int)(c->map_timestamp - kComposeAge); }  // SurfelMap.cpp:873 (Q9)

uint32_t pose_table_count(const sb_ctx* c) {
  uint32_t n = c->map_timestamp + 1;
  return n < kMaxPoses ? n : kMaxPoses;
}

int set_pose_entry(sb_ctx* c, uint32_t t, const float* pose) {
  c->map_version += 1;
  if (t >= kMaxPoses) return fail(c, SB_ERR_CAPACITY, "pose table full (10000 poses, SurfelMap.h:205)");
  memcpy(&c->h_poses[16 * (size_t)t], pose, 64);
  sbg::rigid_inverse_f(pose, &c->h_poses_inv[16 * (size_t)t]);
  SB_CUDA(c, cudaMemcpyAsync(c->poses + 16 * (size_t)t, &c->h_poses[16 * (size_t)t], 64, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemcpyAsync(c->poses_inv + 16 * (size_t)t, &c->h_poses_inv[16 * (size_t)t], 64, cudaMemcpyHostToDevice,
                             c->stream));
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// rendering
// ---------------------------------------------------------------------------------------------------------
FrameDev null_frame() {
  FrameDev f;
  f.W = f.H = 0;
  f.vertex = f.normal = f.semantic = nullptr;
  return f;
}

sb_ctx::RenderMemo::Key memo_key(const sb_ctx* c, const float* pose_old, const float* pose_new, float conf_thr,
                                 const sb_frame* out) {
  sb_ctx::RenderMemo::Key k{};
  memcpy(k.pose_old, pose_old, 64);
  memcpy(k.pose_new, pose_new, 64);
  k.conf_thr = conf_thr;
  k.map_timestamp = c->map_timestamp;
  k.map_version = c->map_version;
  k.out = out->id;
  k.compose = c->p.compose_rendering;
  return k;
}

int render_full(sb_ctx* c, const float* pose_old, const float* pose_new, float conf_thr, sb_frame* out,
                const Mat4* inv_dev = nullptr, bool table_ready = false) {
  if (!inv_dev && c->memo.matches(memo_key(c, pose_old, pose_new, conf_thr, out))) {
    c->renders_skipped += 1;  // old / new / composed frames and `out` already hold exactly this rendering
    return SB_OK;
  }
  const KParams& kp = c->kp;
  Launch L = L_(c);
  size_t Pm = (size_t)kp.Wm * kp.Hm;
  float inv_old[16] = {0}, inv_new[16] = {0};
  if (!inv_dev) {
    sbg::rigid_inverse_f(pose_old, inv_old);
    sbg::rigid_inverse_f(pose_new, inv_new);
  }
  const bool same = inv_dev != nullptr || memcmp(pose_old, pose_new, 64) == 0;
  uint32_t np = pose_table_count(c);
  // table_ready: Mtab_old already holds inv(pose) * poseTable from the map update of this scan (same pose)
  if (!table_ready) launch_pose_products(L, mat4_from(inv_old), inv_dev, c->poses, c->Mtab_old, np);
  float* Mnew = c->Mtab_old;
  if (!same) {
    launch_pose_products(L, mat4_from(inv_new), nullptr, c->poses, c->Mtab_new, np);
    Mnew = c->Mtab_new;
  }
  if (c->p.compose_rendering) {
    // the composed view needs no atomics of its own: it is derived from the old / new key images in the resolve pass
    // (key images are cleared by the resolve pass that consumes them)
    RenderTargets t{c->key_old, c->key_new, nullptr};
    int thr = t_threshold(c);
    if (same) {
      launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, conf_thr, thr, 1, 1, 0, t);
    } else {
      RenderTargets to{c->key_old, nullptr, nullptr}, tn{nullptr, c->key_new, nullptr};
      launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, conf_thr, thr, 1, 0, 0, to);
      launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), Mnew, conf_thr, thr, 0, 1, 0, tn);
    }
    launch_render_resolve(L, kp, c->A, c->Mtab_old, Mnew, t, c->f_old->d, c->f_new->d, c->f_comp->d, out->d, null_frame(), 0, 0);
  } else {
    // SurfelMap.cpp:977-1017: one view with render_old_surfels = false, timestamp_threshold = 0, copied to old and new
    RenderTargets t{nullptr, c->key_new, nullptr};
    launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, conf_thr, 0, 0, 1, 0, t);
    launch_render_resolve(L, kp, c->A, c->Mtab_old, c->Mtab_old, t, null_frame(), c->f_new->d, null_frame(), null_frame(),
                          null_frame(), 0, 0);
    SB_CUDA(c, cudaMemcpyAsync(c->f_old->base, c->f_new->base, Pm * 48, cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(c, cudaMemcpyAsync(out->base, c->f_new->base, Pm * 48, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (inv_dev)  // pose still on the device: the caller stores the memo once it has read the pose back
    c->memo.clear();
  else
    c->memo.store(memo_key(c, pose_old, pose_new, conf_thr, out));
  return SB_OK;
}

// which: 1 = active (new surfels into newMapFrame), 0 = inactive (old surfels into oldMapFrame); Q4: semantic map kept
int render_single(sb_ctx* c, const float* pose, float conf_thr, int which, const Mat4* inv_dev = nullptr,
                  bool table_ready = false, sb_frame* copy_to = nullptr, const IndexFuse* index = nullptr) {
  frame_written(c, which ? c->f_new : c->f_old);
  if (copy_to) frame_written(c, copy_to);
  const KParams& kp = c->kp;
  Launch L = L_(c);
  size_t Pm = (size_t)kp.Wm * kp.Hm;
  float inv[16] = {0};
  if (pose) sbg::rigid_inverse_f(pose, inv);
  if (!table_ready) launch_pose_products(L, mat4_from(inv), inv_dev, c->poses, c->Mtab_old, pose_table_count(c));
  unsigned long long* key = which ? c->key_new : c->key_old;
  RenderTargets t{which ? nullptr : key, which ? key : nullptr, nullptr};
  launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, conf_thr, t_threshold(c), which ? 0 : 1,
                        which ? 1 : 0, 0, t, index);
  // copy_to: lastModelFrame_->copy(*map_->newMapFrame()), SurfelMapping.cpp:407 (the semantic image is the stale one, Q4),
  // written by the same resolve pass
  launch_render_resolve(L, kp, c->A, c->Mtab_old, c->Mtab_old, t, c->f_old->d, c->f_new->d, null_frame(), null_frame(),
                        (copy_to && which) ? copy_to->d : null_frame(), 1, 0);
  if (copy_to && !which)
    SB_CUDA(c, cudaMemcpyAsync(copy_to->base, c->f_old->base, Pm * 48, cudaMemcpyDeviceToDevice, c->stream));
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// ICP
// ---------------------------------------------------------------------------------------------------------
// every launch of the persistent Gauss-Newton kernel publishes epoch values base+1 .. base+max_iter+2: hand out disjoint
// ranges so that the epoch word never has to be reset between launches
// A Gauss-Newton launch that gave up (bounded spin: a block or a peer GPU never arrived) leaves its arrival ticket and
// accumulator replicas mid-pass: return them to the state every launch starts from, so that the context stays usable.
int gn_fail(sb_ctx* c) {
  cudaMemsetAsync(c->ticket, 0, 128, c->stream);
  cudaMemsetAsync(c->acc_slots, 0, 1024 * 32 * sizeof(long long), c->stream);
  cudaMemsetAsync(&c->res->pose.gn_error, 0, sizeof(int), c->stream);
  cudaStreamSynchronize(c->stream);
  return fail(c, SB_ERR_STATE, "Gauss-Newton kernel timed out waiting for a block or a peer GPU");
}

unsigned int next_epoch_base(sb_ctx* c, int max_iter) {
  unsigned int b = c->epoch_base;
  c->epoch_base += (unsigned int)max_iter + 8u;
  return b;
}

IcpArgs icp_args(sb_ctx* c, const sb_frame* data, const sb_frame* model, float max_distance, float max_angle_deg,
                 int row_begin, int row_end, bool semantics) {
  IcpArgs a;
  a.data_v = data->d.vertex; a.data_n = data->d.normal; a.data_s = data->d.semantic;
  a.model_v = model->d.vertex; a.model_n = model->d.normal; a.model_s = model->d.semantic;
  a.distance_thresh = max_distance;
  a.angle_thresh = (float)cos((double)max_angle_deg * 3.14159265358979323846 / 180.0);  // Frame2Model.cpp:66
  a.row_begin = row_begin; a.row_end = row_end;
  a.has_semantics = semantics ? 1 : 0;
  a.Wm = model->d.W; a.Hm = model->d.H;
  return a;
}

int icp_check(sb_ctx* c, const sb_frame* data, const sb_frame* model) {
  if (!c || !data || !model) return fail(c, SB_ERR_INVALID, "icp: null argument");
  // the model may be a rendered model frame or another data frame (frame-to-frame objective, SurfelMapping.cpp:442):
  // its own size is what the kernel samples with (textureSize(vertex_model))
  const bool model_ok = (model->d.W == c->kp.Wm && model->d.H == c->kp.Hm) || (model->d.W == c->kp.W && model->d.H == c->kp.H);
  if (data->d.W != c->kp.W || data->d.H != c->kp.H || !model_ok)
    return fail(c, SB_ERR_INVALID, "icp: frame size does not match data_/model_ width/height");
  return SB_OK;
}

int icp_jacobian_raw(sb_ctx* c, const sb_frame* data, const sb_frame* model, const double* pose, int iteration,
                     float max_distance, float max_angle_deg, int r0, int r1, bool semantics, long long* raw) {
  IcpArgs a = icp_args(c, data, model, max_distance, max_angle_deg, r0, r1, semantics);
  Mat4 P;
  for (int i = 0; i < 16; ++i) P.m[i] = (float)pose[i];  // pose_.cast<float>(), Frame2Model.cpp:194
  launch_icp_jacobian(L_(c), c->kp, a, P, iteration, c->res->sums, c->acc_slots, c->ticket + 16, c->icp_blocks);
  SB_CUDA(c, cudaMemcpyAsync(c->host->sums, c->res->sums, sizeof(c->host->sums), cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  memcpy(raw, c->host->sums, sizeof(c->host->sums));
  return SB_OK;
}

// Row-striped minimisation with a host-side all-reduce callback (sb_comm_set_callback): LieGaussNewton::minimize driven
// from the host, one striped K5 launch + 256-byte read-back + callback per iteration; the result is written into the
// device GN state st so that the rest of the pipeline proceeds as after the device-resident loop.
int icp_minimize_callback(sb_ctx* c, GnState* st, const sb_frame* data, const sb_frame* model, const double* T0,
                          int max_iter, double eps, double delta, float max_distance, float max_angle_deg, bool semantics) {
  IcpArgs a = icp_args(c, data, model, max_distance, max_angle_deg, c->row_begin, c->row_end, semantics);
  GnHead& h = c->host->gn;
  memset(&h, 0, sizeof(h));
  memcpy(h.pose, T0, sizeof(h.pose));
  h.last_error = (double)3.402823466e+38f;
  int k = 0;
  for (;;) {
    memcpy(c->host->history + 16 * h.history_len++, h.pose, sizeof(h.pose));  // at most max_iter + 1 <= 257 poses
    if (k >= max_iter) break;
    Mat4 P;
    for (int i = 0; i < 16; ++i) P.m[i] = (float)h.pose[i];
    launch_icp_jacobian(L_(c), c->kp, a, P, k, c->res->sums, c->acc_slots, c->ticket + 16, c->icp_blocks);
    long long* raw = c->host->sums;
    SB_CUDA(c, cudaMemcpyAsync(raw, c->res->sums, sizeof(c->host->sums), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(c, cudaStreamSynchronize(c->stream));
    if (c->comm_cb(c->comm_cb_user, (int64_t*)raw) != 0) return fail(c, SB_ERR_STATE, "all-reduce callback failed");
    sbg::unpack48(raw, h.out48);
    double dx[6];
    int result = sbg::gn_step(h.out48, h.last_error, eps, delta, h.pose, dx);
    h.last_error = h.out48[43];
    if (result == 0) break;
    ++k;
  }
  h.k = k;
  h.done = 1;
  SB_CUDA(c, cudaMemcpyAsync(static_cast<GnHead*>(st), &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemcpyAsync(st->history, c->host->history, (size_t)h.history_len * 16 * sizeof(double),
                             cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}

// LieGaussNewton::minimize; the result stays in c->gn. One cooperative launch for the whole minimisation, or the
// host-driven loop when a host all-reduce callback is set.
int icp_minimize_enqueue(sb_ctx* c, const sb_frame* data, const sb_frame* model, const double* T0, int max_iter,
                         double eps, double delta, float max_distance, float max_angle_deg, bool semantics) {
  if (max_iter <= 0 || max_iter > kMaxGnIter) max_iter = kMaxGnIter;
  if (c->comm_cb)
    return icp_minimize_callback(c, c->gn, data, model, T0, max_iter, eps, delta, max_distance, max_angle_deg, semantics);
  IcpArgs a = icp_args(c, data, model, max_distance, max_angle_deg, c->comm_on ? c->row_begin : 0,
                       c->comm_on ? c->row_end : c->kp.H, semantics);
  Mat4d T;
  memcpy(T.m, T0, sizeof(T.m));
  Launch L = L_(c);
  launch_gn_init(L, c->gn, T, c->res->sums);
  GnJob job;
  memset(&job, 0, sizeof(job));
  job.mode = GN_PLAIN;
  job.a = a;
  job.st = c->gn;
  job.max_iter = max_iter;
  job.eps = eps;
  job.delta = delta;
  job.epoch_base = next_epoch_base(c, max_iter);
  if (launch_gn_persistent(L, c->kp, job, c->acc_slots, c->ticket, c->gn_pub, c->comm_on ? &c->comm : nullptr,
                           c->icp_coop_blocks) != 0) {
    cudaGetLastError();
    return fail(c, SB_ERR_CUDA, "cooperative launch of the Gauss-Newton kernel failed");
  }
  return SB_OK;
}

int icp_minimize_fetch(sb_ctx* c, double* pose_out, double* out48, int* iters, double* history, int* history_len) {
  GnHead& h = c->host->gn;
  SB_CUDA(c, cudaMemcpyAsync(&h, static_cast<GnHead*>(c->gn), sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (h.error) return gn_fail(c);
  if (pose_out) memcpy(pose_out, h.pose, sizeof(h.pose));
  if (out48) memcpy(out48, h.out48, sizeof(h.out48));
  if (iters) *iters = h.k;
  if (history_len) *history_len = h.history_len;
  if (history && h.history_len > 0) {
    SB_CUDA(c, cudaMemcpy(history, c->gn->history, (size_t)h.history_len * 16 * sizeof(double), cudaMemcpyDeviceToHost));
  }
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// map update: SurfelMap::update, SurfelMap.cpp:492-584
// ---------------------------------------------------------------------------------------------------------
// The per-scan map update runs dense (update into T + compaction back into A) once the dead slots left by the in-place
// updates reach this fraction of the physical end (1 / kDenseHoleFraction); DESIGN.md section 7 gives the measurements.
constexpr uint32_t kDenseHoleFraction = 8;

float2 submap_center(const sb_ctx* c, int32_t i, int32_t j) {  // submapIndex2center, SurfelMap.cpp:704-706
  return make_float2((float)(2.0 * i * c->p.submap_extent), (float)(2.0 * j * c->p.submap_extent));
}

int fetch_counts(sb_ctx* c, uint32_t* dst, int n) {
  SB_CUDA(c, cudaMemcpyAsync(c->host->result.counts, c->res->counts, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  memcpy(dst, c->host->result.counts, n * sizeof(uint32_t));
  return SB_OK;
}

int refresh_tile_records(sb_ctx* c) {  // read back the records of the tiles extracted so far
  if (!c->tiles_pending || c->n_slots == 0) return SB_OK;
  std::vector<uint2> rec(c->n_slots);
  SB_CUDA(c, cudaMemcpyAsync(rec.data(), c->d_tile_rec, (size_t)c->n_slots * sizeof(uint2), cudaMemcpyDeviceToHost,
                             c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  auto base = [&](uint32_t s) { return s ? rec[s - 1].x : 0u; };
  {  // surfels that did not fit the 16 M-surfel HBM tile pool (the reference's host-side cache is unbounded); slots are
     // never reused, so the sum over all slots counts every drop since the last reset
    uint64_t dropped = 0;
    for (uint32_t s = 0; s < c->n_slots; ++s) dropped += std::min(rec[s].y, kExtractCap) - (rec[s].x - base(s));
    if ((double)dropped != c->stats[12]) {
      c->stats[12] = (double)dropped;
      c->err = "submap tile pool exhausted: " + std::to_string(dropped) + " surfels of leaving tiles were dropped";
    }
  }
  for (auto& kv : c->tiles) {
    DevTile& t = kv.second;
    if (!t.known) {
      t.base = base(t.slot);
      t.count = rec[t.slot].x - t.base;
      t.known = true;
    }
  }
  c->tiles_pending = false;
  return SB_OK;
}

// Moves the live surfels of a map with dead slots to the front, in order (A -> T, then the two sets swap roles): what
// observers of the map and the operator-level update see, and what a tile that needs the room finds.
int compact_map(sb_ctx* c) {
  if (c->n_holes == 0) return SB_OK;
  // the host's physical end is the one to compact: tile re-insertion raises it ahead of counts[0]
  SB_CUDA(c, cudaMemcpyAsync(c->res->counts, &c->n_host, 4, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemsetAsync(c->group_counts, 0, kGroupCounts * 4, c->stream));
  launch_compact_live(L_(c), c->A, c->res->counts, c->n_host, c->live, c->keep, c->block_counts, c->group_counts, c->T,
                      c->res->counts + 6);
  SB_CUDA(c, cudaStreamSynchronize(c->stream));  // (the copy above reads the member changed below)
  std::swap(c->A, c->T);  // both are kMaxSurfels sets with the same lane pitch
  std::swap(c->A_mem, c->T_mem);
  c->n_host = n_live(c);
  c->n_holes = 0;
  c->n_upper = c->n_host;
  SB_CUDA(c, cudaMemcpyAsync(c->res->counts, &c->n_host, 4, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));  // the copy reads a member of the context: keep it ordered
  return SB_OK;
}

int append_tiles(sb_ctx* c, int32_t i0, int32_t j0, int di, int dj) {  // SurfelMap.cpp:769-780
  const int dim = c->p.submap_dimension;
  int r;
  bool appended = false;
  for (int32_t k = -dim; k <= dim; ++k) {
    auto it = c->tiles.find(std::make_pair(i0 + di * k, j0 + dj * k));
    if (it == c->tiles.end()) continue;  // submapCache_[idx] of a tile never extracted: empty
    if (!it->second.known && (r = refresh_tile_records(c))) return r;
    const DevTile& t = it->second;
    // the reference's map has no dead slots: a tile that does not fit behind them fits (or is cut) after compaction
    if (t.count > kMaxSurfels - c->n_host && (r = compact_map(c))) return r;
    uint32_t room = kMaxSurfels - c->n_host;
    uint32_t n = t.count < room ? t.count : room;
    if (n == 0) continue;
    // the four lanes of A and of the pool lie at fixed pitches (kMaxSurfels, kTilePoolCap) in one allocation each
    for (size_t lane = 0; lane < 4; ++lane)
      SB_CUDA(c, cudaMemcpyAsync(c->A.p0 + lane * kMaxSurfels + c->n_host, c->pool.p0 + lane * kTilePoolCap + t.base,
                                 (size_t)n * 16, cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(c, cudaMemsetAsync(c->live + c->n_host, 1, n, c->stream));
    c->n_host += n;
    c->n_upper = c->n_host;
    appended = true;
  }
  if (appended) {
    c->map_version += 1;
    SB_CUDA(c, cudaMemcpyAsync(c->res->counts, &c->n_host, 4, cudaMemcpyHostToDevice, c->stream));
    SB_CUDA(c, cudaStreamSynchronize(c->stream));  // the copy reads a member of the context: keep it ordered
  }
  return SB_OK;
}

// SurfelMap.cpp:708-742 + extract_surfels.vert: the tile is compacted into the HBM pool; nothing is read back here
int extract_surfels(sb_ctx* c, bool partially) {
  Launch L = L_(c);
  while (!c->extraction.empty()) {
    std::pair<int32_t, int32_t> idx = c->extraction.back();
    c->extraction.pop_back();
    if (c->n_slots >= kMaxTileSlots) return fail(c, SB_ERR_CAPACITY, "tile cache: out of record slots");
    float2 ctr = submap_center(c, idx.first, idx.second);
    uint32_t slot = c->n_slots++;
    // extractions can follow each other with no per-pixel prologue in between to clear the group totals
    SB_CUDA(c, cudaMemsetAsync(c->group_counts, 0, kGroupCounts * 4, c->stream));
    launch_extract_to_pool(L, c->A, c->res->counts, c->live, c->n_host, c->poses, ctr, c->p.submap_extent, c->keep,
                           c->block_counts, c->group_counts, c->pool, kTilePoolCap, c->d_tile_rec, slot, kExtractCap);
    DevTile t;
    t.slot = slot;
    t.known = false;
    c->tiles[idx] = t;  // a tile extracted again replaces its cache entry (the old pool range is abandoned)
    c->tiles_pending = true;
    if (partially) break;
  }
  return SB_OK;
}

int update_active_submaps(sb_ctx* c, const float* pose) {  // SurfelMap.cpp:744-824
  const int dim = c->p.submap_dimension;
  const float ext = c->p.submap_extent;
  float2 ctr = submap_center(c, c->origin_i, c->origin_j);
  float changex = pose[12] - ctr.x, changey = pose[13] - ctr.y;
  float factor = 1.1f;
  int r;
  if (fabsf(changex) > factor * ext || fabsf(changey) > factor * ext) {
    if (fabsf(changex) > factor * ext) {
      int dir = changex < 0 ? -1 : 1;
      for (int32_t k = -dim; k <= dim; ++k) c->extraction.push_back(std::make_pair(c->origin_i - dir * dim, c->origin_j + k));
      c->origin_i += dir;
      if ((r = append_tiles(c, c->origin_i + dir * dim, c->origin_j, 0, 1))) return r;
    }
    if (fabsf(changey) > factor * ext) {
      int dir = changey < 0 ? -1 : 1;
      for (int32_t k = -dim; k <= dim; ++k) c->extraction.push_back(std::make_pair(c->origin_i + k, c->origin_j - dir * dim));
      c->origin_j += dir;
      if ((r = append_tiles(c, c->origin_i, c->origin_j + dir * dim, 1, 0))) return r;
    }
  }
  if (!c->extraction.empty()) return extract_surfels(c, c->p.partial_extraction != 0);
  return SB_OK;
}

// pose_dev / inv_dev != nullptr: pipeline mode -- the pose (and its pose-table entry) already lives on the device,
// nothing is read back here; the caller finishes with map_update_finish() after its end-of-scan synchronisation.
// index_fused: the post-ICP render of this scan has written the index keys unless the track-loss recovery ran (IndexFuse)
int map_update(sb_ctx* c, const float* pose, const sb_frame* frame, const Mat4* pose_dev = nullptr,
               const Mat4* inv_dev = nullptr, bool table_ready = false, bool index_fused = false) {
  c->map_version += 1;
  const KParams& kp = c->kp;
  Launch L = L_(c);
  const size_t Pd = (size_t)kp.W * kp.H;
  const bool deferred = pose_dev != nullptr;
  int r;
  float inv_pose[16] = {0}, pose_h[16] = {0};
  // the operator-level update works on the compacted map: its index map (sb_map_update_debug) indexes the surfels in order
  if (!deferred && (r = compact_map(c))) return r;
  if (!deferred) {
    if (c->map_timestamp < kMaxPoses) {
      if ((r = set_pose_entry(c, c->map_timestamp, pose))) return r;  // SurfelMap.cpp:494-495
    }
    sbg::rigid_inverse_f(pose, inv_pose);  // :497
    memcpy(pose_h, pose, 64);
  }
  // K6a (table_ready: the Gauss-Newton kernel of this scan has already filled inv(pose) * poses[t])
  if (!table_ready) launch_pose_products(L, mat4_from(inv_pose), inv_dev, c->poses, c->Mtab_old, pose_table_count(c));
  // K6b (+ index keys re-armed, integrated flags cleared) -- already done by the tiled preprocessing pass of this scan
  // when the frame is the one it produced
  if (!(c->prepped_for_update && frame == c->cur)) launch_radius(L, kp, frame->d, c->radius_map, c->key_index, c->integrated, c->group_counts);
  c->prepped_for_update = false;
  // K6a: nearest visible surfel per data pixel. After a fused post-ICP render only a scan with track-loss recovery needs
  // the pass (P_cur then differs from the render's pose); the launch is gated on that flag on the device.
  launch_index_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, c->key_index,
                       index_fused ? &c->res->pose.fallback : nullptr);
  // K6c + K6e predicate
  float2 ctr = submap_center(c, c->origin_i, c->origin_j);
  float extent = 2.0f * c->p.submap_dimension * c->p.submap_extent + c->p.submap_extent;  // :674
  if (c->p.partial_extraction && !c->extraction.empty()) extent += 2.0f * c->p.submap_extent;  // :677
  // In place (lazy) or dense, decided from what the host already knows (no extra synchronisation); DESIGN.md section 7.
  // Dense when the dead slots reach 1 / kDenseHoleFraction of the physical end, when the new surfels could hit the capacity
  // behind the dead slots (k_gen_compact must cut exactly where the compacted map would), and at the operator level.
  const uint32_t n = n_grid(c);
  const bool lazy = deferred && n > 0 && (uint64_t)c->n_holes * kDenseHoleFraction < n &&
                    (uint64_t)n + Pd <= kMaxSurfels;
  c->lazy_update = lazy;
  // Dense: K6c + K6e predicate into T, then ordered compaction back into the map lanes: counts[1] = S', counts[2] = kept.
  // (A single-pass variant with decoupled look-back was measured twice and loses: round 1 with a 32-wide chain, round 2
  // with 256-wide windows that stop at the nearest inclusive prefix -- 80.2 us against 48.8 + 23.8 us for the two
  // passes at S = 1.2 M: the ~400 resident blocks finish their heavy per-surfel work together, hold their SM slots
  // through several dependent L2 round trips and only then issue their writes.)
  // Lazy: the changed lanes are stored in place and removed surfels marked dead; counts[1] = physical end, and the
  // generation pass below writes [2] = kept and [5] = dead slots from the update's group totals.
  launch_update_surfels(L, kp, lazy, c->A, c->T, c->res->counts, n, mat4_from(pose_h), mat4_from(inv_pose), pose_dev,
                        inv_dev, c->poses, c->poses_inv, c->key_index, c->radius_map, frame->d, (int)c->map_timestamp,
                        ctr, extent, c->integrated, c->live, c->keep, c->block_counts, c->group_counts);
  if (!lazy)
    launch_compact(L, c->T, c->keep, c->block_counts, c->group_counts, c->res->counts, n, c->A, c->live, nullptr,
                   kMaxSurfels, kMaxSurfels, c->res->counts + 1);
  // K6d + K6e: new surfels appended behind counts[1]; counts[0] = new physical end, counts[3] = new surfels
  c->lb_gen = (c->lb_gen + 1) & 0x3fffffffu;
  if (c->lb_gen == 0) c->lb_gen = 1;
  launch_gen_compact(L, kp, frame->d, c->radius_map, c->integrated, c->poses, (int)c->map_timestamp, ctr, extent, c->A,
                     c->live, lazy ? c->group_counts.get() : nullptr, c->lb_desc, c->lb_ticket, c->lb_gen, kMaxSurfels,
                     c->res->counts);
  uint64_t up = (uint64_t)n_grid(c) + Pd;  // the map can grow by at most one surfel per pixel
  c->n_upper = up > kMaxSurfels ? kMaxSurfels : (uint32_t)up;
  const uint32_t entry = c->map_timestamp < kMaxPoses ? c->map_timestamp : kMaxPoses - 1;  // of the new surfels
  if (entry + 1 > c->pose_ref_end) c->pose_ref_end = entry + 1;
  if (deferred) {
    c->map_timestamp += 1;
    return SB_OK;
  }
  uint32_t cnt[4];
  if ((r = fetch_counts(c, cnt, 4))) return r;
  c->n_host = cnt[0];
  c->n_holes = 0;  // (dense)
  c->n_upper = cnt[0];
  c->n_updated = cnt[2];
  c->n_new = cnt[3];
  if ((r = update_active_submaps(c, pose))) return r;  // :547
  c->map_timestamp += 1;
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// SurfelMapping
// ---------------------------------------------------------------------------------------------------------
float conf_threshold(const sb_ctx* c) {  // SurfelMapping.cpp:333-340, time_init = 10
  float ct = c->confidence_threshold;
  if (c->timestamp < 10) {
    float alpha = (float)c->timestamp / 10.0f;
    ct = (float)((1.0 - (double)alpha) * (double)c->log_unstable_slam + (double)(alpha * c->confidence_threshold));
  }
  return ct;
}

// staging buffers for host-pointer scans grow with the largest scan seen (the projection itself only needs W*H pixels)
int grow_point_buffers(sb_ctx* c, size_t n) {
  if (n <= c->pts_cap) return SB_OK;
  size_t cap = n + n / 4 + 1024;
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (c->copy_stream) SB_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  DevPtr<float4> np;
  DevPtr<float> nl, nq;
  if (dev_alloc(np, cap * 16) != cudaSuccess || dev_alloc(nl, cap * 4) != cudaSuccess ||
      dev_alloc(nq, cap * 4) != cudaSuccess) {
    cudaGetLastError();
    return fail(c, SB_ERR_CAPACITY, "out of device memory for the scan staging buffers");
  }
  c->d_pts = std::move(np); c->d_labels = std::move(nl); c->d_probs = std::move(nq);
  for (auto& sl : c->prefetch) {  // prefetch slots are re-allocated lazily at the new capacity
    sl.pts.reset(); sl.labels.reset(); sl.probs.reset();
    sl.valid = false; sl.in_use = false; sl.has_released = false;
  }
  c->pts_cap = cap;
  return SB_OK;
}

int upload_scan(sb_ctx* c, const float* pts4, const float* labels, const float* probs, uint32_t n, int on_device,
                const float4** d_pts, const float** d_labels, const float** d_probs) {
  if (on_device) {
    *d_pts = reinterpret_cast<const float4*>(pts4);
    *d_labels = labels;
    *d_probs = probs;
    return SB_OK;
  }
  int rg = grow_point_buffers(c, n);  // GlBuffer::assign resizes (SurfelMapping.cpp:327-330): no cap on the scan size
  if (rg) return rg;
  if (c->copy_stream) {  // was this scan prefetched (same host buffer, same size, same optional arrays)?
    for (auto& sl : c->prefetch)
      if (sl.in_use) {  // the work that read this slot is already in the compute stream: mark the point after it
        SB_CUDA(c, cudaEventRecord(sl.released, c->stream));
        sl.has_released = true;
        sl.in_use = false;
      }
    for (auto& sl : c->prefetch) {
      if (!sl.valid || sl.host_pts != pts4 || sl.n != n || sl.has_labels != (labels != nullptr) ||
          sl.has_probs != (probs != nullptr))
        continue;
      SB_CUDA(c, cudaStreamWaitEvent(c->stream, sl.done, 0));
      sl.valid = false;
      sl.in_use = true;
      *d_pts = sl.pts;
      *d_labels = labels ? sl.labels.get() : nullptr;
      *d_probs = probs ? sl.probs.get() : nullptr;
      return SB_OK;
    }
  }
  if (n) SB_CUDA(c, cudaMemcpyAsync(c->d_pts, pts4, (size_t)n * 16, cudaMemcpyHostToDevice, c->stream));
  if (labels && n) SB_CUDA(c, cudaMemcpyAsync(c->d_labels, labels, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
  if (probs && n) SB_CUDA(c, cudaMemcpyAsync(c->d_probs, probs, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
  *d_pts = c->d_pts;
  *d_labels = labels ? c->d_labels.get() : nullptr;
  *d_probs = probs ? c->d_probs.get() : nullptr;
  return SB_OK;
}

// SurfelMap::render_composed, SurfelMap.cpp:1116-1165
int render_composed_internal(sb_ctx* c, const float* pose_old, const float* pose_new, float conf_thr) {
  frame_written(c, c->f_comp);
  const KParams& kp = c->kp;
  Launch L = L_(c);
  size_t Pm = (size_t)kp.Wm * kp.Hm;
  float inv_old[16], inv_new[16];
  sbg::rigid_inverse_f(pose_old, inv_old);
  sbg::rigid_inverse_f(pose_new, inv_new);
  uint32_t np = pose_table_count(c);
  launch_pose_products(L, mat4_from(inv_old), nullptr, c->poses, c->Mtab_old, np);
  launch_pose_products(L, mat4_from(inv_new), nullptr, c->poses, c->Mtab_new, np);
  RenderTargets t{nullptr, nullptr, c->key_comp};
  int thr = t_threshold(c);
  // GL_LEQUAL (SurfelMap.cpp:1126), old then new without clearing (:1146-1152); COLOR2 not attached (Q4)
  launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_old, conf_thr, thr, 1, 0, 1, t);
  launch_render_scatter(L, kp, c->A, c->res->counts, c->live, n_grid(c), c->Mtab_new, conf_thr, thr, 0, 1, 1, t);
  launch_render_resolve(L, kp, c->A, c->Mtab_old, c->Mtab_new, t, null_frame(), null_frame(), c->f_comp->d, null_frame(),
                        null_frame(), 1, 1);
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}

// SurfelMapping::updatePose, SurfelMapping.cpp:372-476 -- enqueue only. The increment, the track-loss decision, the
// recovery minimisation and the pose chaining stay on the device: two cooperative launches (GN_MAIN, GN_POST) around the
// rendering of the active map at the new pose. Returns with *tables_ready = true when GN_POST has also written the pose
// table entry of this scan and the table inv(P_cur) * poses[t] (Mtab_old) for the map update / model rendering.
// With a host all-reduce callback (sb_comm_set_callback) the minimisations are driven from the host instead.
// *index_fused = true: the render at the new pose has also written the map update's index keys (IndexFuse).
int update_pose_enqueue(sb_ctx* c, bool* tables_ready, bool* index_fused) {
  const sb_params& p = c->p;
  const bool sem = c->cur_has_semantics;
  *tables_ready = false;
  *index_fused = false;
  int r;
  Launch L = L_(c);
  const uint32_t np = pose_table_count(c);
  int max_iter = p.max_iterations;
  if (max_iter <= 0 || max_iter > kMaxGnIter) max_iter = kMaxGnIter;
  const int r0 = c->comm_on ? c->row_begin : 0, r1 = c->comm_on ? c->row_end : c->kp.H;
  if (!c->comm_cb) {
    // ---- device-resident path ----
    GnJob job;
    memset(&job, 0, sizeof(job));
    job.mode = GN_MAIN;  // objective_->setData(currentFrame_, map_->newMapFrame()); gn_->minimize(*objective_, T0)   :384-389
    job.a = icp_args(c, c->cur, c->f_new, p.icp_max_distance, p.icp_max_angle, r0, r1, sem);
    job.st = c->gn;
    job.pd = &c->res->pose;
    job.Mtab = c->Mtab_old;
    job.poses = c->poses;
    job.n_poses = np;
    job.initialize_identity = p.initialize_identity;
    job.fallback_mode = p.fallback_mode;
    job.timestamp = c->timestamp;
    job.max_iter = max_iter;
    job.eps = p.stopping_threshold;
    job.delta = p.delta;
    job.epoch_base = next_epoch_base(c, max_iter);
    if (launch_gn_persistent(L, c->kp, job, c->acc_slots, c->ticket, c->gn_pub, c->comm_on ? &c->comm : nullptr,
                             c->icp_coop_blocks) != 0) {
      cudaGetLastError();
      return fail(c, SB_ERR_CUDA, "cooperative launch of the Gauss-Newton kernel failed");
    }
    // :405-413: render_active at the new pose (its product table is ready), copied into lastModelFrame_.
    // It also writes the index keys of the map update (K6a) when that pass would see what it sees: without track-loss
    // recovery P_cur is bit for bit P_active (the same fp64 product, rounded once), GN_POST's table inv(P_cur) * poses[t]
    // equals this one except at entry t_map, which it sets to P_cur and no surfel refers to while pose_ref_end <=
    // t_map, and nothing writes the map before the update unless the loop-closure step runs in between.
    const bool fuse = !c->close_loops && c->pose_ref_end <= c->map_timestamp;
    // (fov_up, fov, min_depth, max_depth of the data image, then the same four of the model image: bitwise equal?)
    const int same_projection = memcmp(&c->kp.fov_up, &c->kp.m_fov_up, 4 * sizeof(float)) == 0 ? 1 : 0;
    const IndexFuse ix{c->key_index, &c->res->pose.fallback, same_projection};
    if ((r = render_single(c, nullptr, conf_threshold(c), 1, &c->res->pose.invP_active, true, c->last_model,
                           fuse ? &ix : nullptr)))
      return r;
    *index_fused = fuse;
    // :414-449: statistics pass at identity, track-loss recovery, pose chaining, pose-table entry, table for the update
    GnJob post;
    memset(&post, 0, sizeof(post));
    post.mode = GN_POST;
    post.a = icp_args(c, c->cur, c->f_new, p.icp_max_distance, p.icp_max_angle, 0, c->kp.H, sem);
    post.fb = icp_args(c, c->cur, c->last, p.fallback_max_distance, p.fallback_max_angle, r0, r1,
                       sem && c->last_has_semantics);
    post.st = c->gn2;
    post.pd = &c->res->pose;
    post.stats32 = c->res->sums;
    post.poses = c->poses;
    post.poses_inv = c->poses_inv;
    post.t_map = c->map_timestamp;
    post.Mtab = c->Mtab_old;
    post.n_poses = np;
    post.fallback_mode = p.fallback_mode;
    post.timestamp = c->timestamp;
    post.max_iter = max_iter;
    post.eps = p.stopping_threshold;
    post.delta = p.delta;
    post.epoch_base = next_epoch_base(c, max_iter);
    if (launch_gn_persistent(L, c->kp, post, c->acc_slots, c->ticket, c->gn_pub, c->comm_on ? &c->comm : nullptr,
                             c->icp_coop_blocks) != 0) {
      cudaGetLastError();
      return fail(c, SB_ERR_CUDA, "cooperative launch of the Gauss-Newton kernel failed");
    }
    *tables_ready = true;
    return SB_OK;
  }
  // ---- host-driven path (all-reduce callback): one Jacobian launch and one callback per iteration ----
  double T0[16];
  if (!p.initialize_identity) memcpy(T0, c->lastIncrement, sizeof(T0)); else ident_d(T0);
  if ((r = icp_minimize_enqueue(c, c->cur, c->f_new, T0, p.max_iterations, p.stopping_threshold, p.delta,
                                p.icp_max_distance, p.icp_max_angle, sem)))
    return r;
  Mat4d T0v;
  memcpy(T0v.m, T0, sizeof(T0v.m));
  launch_pose_after_icp(L, c->gn, &c->res->pose, T0v, c->timestamp, p.fallback_mode);
  if ((r = render_single(c, nullptr, conf_threshold(c), 1, &c->res->pose.invP_active, false, c->last_model))) return r;
  {
    IcpArgs a = icp_args(c, c->cur, c->f_new, p.icp_max_distance, p.icp_max_angle, 0, c->kp.H, sem);
    Mat4 I;
    for (int i = 0; i < 16; ++i) I.m[i] = (i % 5 == 0) ? 1.0f : 0.0f;
    launch_icp_jacobian(L, c->kp, a, I, 0, c->res->sums, c->acc_slots, c->ticket + 16, c->icp_blocks);
  }
  if (p.fallback_mode) {  // read the track-loss flag and run the recovery minimisation only when it is set
    int& fb = c->host->result.pose.fallback;
    SB_CUDA(c, cudaMemcpyAsync(&fb, &c->res->pose.fallback, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(c, cudaStreamSynchronize(c->stream));
    if (fb) {
      if ((r = icp_minimize_callback(c, c->gn2, c->cur, c->last, T0, max_iter, p.stopping_threshold, p.delta,
                                     p.fallback_max_distance, p.fallback_max_angle, sem && c->last_has_semantics)))
        return r;
    }
  }
  launch_pose_finalize(L, c->gn2, &c->res->pose, 1, c->poses, c->poses_inv, c->map_timestamp);
  return SB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// loop closure: SurfelMapping::checkLoopClosure (SurfelMapping.cpp:527-795) over the CUDA operators; the control flow is
// include/suma_b200_loop.hpp (shared with the oracle twin)
// ---------------------------------------------------------------------------------------------------------
struct CudaLoopBackend {
  sb_ctx* c;
  int err = 0;
  float confidence_threshold() { return conf_threshold(c); }
  void render_inactive(const float* pose, float ct) {
    if (!err) err = render_single(c, pose, ct, 0);
  }
  void render_composed(const float* pose_old, const float* pose_new, float ct) {
    if (!err) err = render_composed_internal(c, pose_old, pose_new, ct);
  }
  int minimize_old(const double* T0, double* pose_out, double* out48) {  // objective_->setData(currentFrame_, oldMapFrame())
    int iters = 0;
    if (!err)
      err = icp_minimize_enqueue(c, c->cur, c->f_old, T0, c->p.max_iterations, c->p.stopping_threshold, c->p.delta,
                                 c->p.icp_max_distance, c->p.icp_max_angle, c->cur_has_semantics);
    if (!err) err = icp_minimize_fetch(c, pose_out, out48, &iters, nullptr, nullptr);
    return iters;
  }
  void evaluate(int model, const double* pose, int iteration, double* out48) {
    long long raw[32];
    memset(raw, 0, sizeof(raw));
    if (!err)
      err = icp_jacobian_raw(c, c->cur, model == 0 ? c->f_old : c->f_comp, pose, iteration, c->p.icp_max_distance,
                             c->p.icp_max_angle, 0, c->kp.H, c->cur_has_semantics, raw);
    sbg::unpack48(raw, out48);
  }
};

// host copy of the device-resident pose block after updatePose (shared by the end of every scan and the loop-closure step)
void absorb_pose_block(sb_ctx* c, const ResultBlock& rb, bool had_icp) {
  const PoseDev& pdh = rb.pose;
  memcpy(c->lastPose, pdh.lastPose, sizeof(c->lastPose));
  memcpy(c->currentPose, pdh.currentPose, sizeof(c->currentPose));
  memcpy(c->lastPose_old, c->currentPose_old, sizeof(c->lastPose_old));  // lastPose_old_ = currentPose_old_   :454
  memcpy(c->currentPose_old, pdh.currentPose, sizeof(c->currentPose));
  memcpy(c->currentPose_new, pdh.currentPose, sizeof(c->currentPose));
  memcpy(c->lastIncrement, pdh.lastIncrement, sizeof(c->lastIncrement));
  c->trackLoss = (uint32_t)pdh.trackLoss;
  if (had_icp) {
    double r48[48];
    sbg::unpack48(rb.sums, r48);
    c->stats[0] = pdh.icp_iterations;
    c->stats[1] = r48[43];
    c->stats[3] = r48[44];
    c->stats[2] = (double)((uint32_t)r48[42] - (uint32_t)r48[44]);  // Frame2Model.cpp:222-226
    c->stats[4] = r48[46];
    c->stats[5] = (float)r48[45];
    // result_new_, SurfelMapping.cpp:417-423
    suma_b200::loop::OptResult& rn = c->loop.result_new;
    rn.error = r48[43];
    rn.outlier = (uint32_t)(float)r48[44];
    rn.valid = (uint32_t)r48[42];
    rn.inlier = rn.valid - rn.outlier;
    rn.invalid = (uint32_t)(float)r48[46];
    rn.residual = rn.error / (rn.inlier + rn.outlier);
    rn.inlier_residual = (float)r48[45] / rn.inlier;
  }
  c->stats[6] = c->trackLoss;
}

// between updatePose() and updateMap() (SurfelMapping.cpp:196-200): needs the scan's poses on the host
int loop_closure_step(sb_ctx* c) {
  namespace lp = suma_b200::loop;
  if (c->comm_on || c->comm_cb) return fail(c, SB_ERR_STATE, "loop closure is not available in row-striped multi-GPU mode");
  const ResultBlock& rb = c->host->result;
  SB_CUDA(c, cudaMemcpyAsync(&c->host->result, c->res, sizeof(ResultBlock), cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (rb.pose.gn_error) return gn_fail(c);
  absorb_pose_block(c, rb, true);
  lp::Poses P;
  memcpy(P.current.m, c->currentPose, 128);
  memcpy(P.current_old.m, c->currentPose_old, 128);
  memcpy(P.current_new.m, c->currentPose_new, 128);
  memcpy(P.last_old.m, c->lastPose_old, 128);
  memcpy(P.last_increment.m, c->lastIncrement, 128);
  lp::M4 inc;
  memcpy(inc.m, rb.pose.increment, 128);
  c->loop.after_update_pose(c->timestamp, inc, P.current);
  CudaLoopBackend be{c};
  lp::check_loop_closure(c->loop, be, c->timestamp, P);
  if (be.err) return be.err;
  memcpy(c->currentPose_old, P.current_old.m, 128);
  return SB_OK;
}

}  // namespace

// =========================================================================================================
// C ABI
// =========================================================================================================
extern "C" {

int sb_default_params(sb_params* p) {
  if (!p) return SB_ERR_INVALID;
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
  return SB_OK;
}

int sb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

// Head-room of the exact ICP sums. The largest per-pixel term is |v_d x n_m|^2 <= |v_d|^2 (unit normals), or r^2 for F,
// with the residual r at most about the longer range of a data / model pair on one beam. |v_d| is the data range plus
// the translation of the pose the data is moved by: kIcpPoseMargin metres of it are allowed for. At 75 m, 128x4096
// (5.6e18 of 9.2e18) is accepted; the largest image accepted at 75 m has 858 993 pixels.
constexpr double kIcpPoseMargin = 25.0;

// Parameters the library cannot run with exactly: nullptr when fine, otherwise the reason.
static const char* check_params(const sb_params* p) {
  if (!p) return "no parameters";
  if (p->data_width <= 0 || p->data_height <= 0 || p->model_width <= 0 || p->model_height <= 0) return "image size <= 0";
  if ((size_t)p->data_width * p->data_height > (1u << 24)) return "more than 2^24 data pixels";
  // the stencils of preprocessing reach 2 columns around the azimuth seam; one column cannot wrap onto itself twice
  if (p->data_width < 2) return "data width < 2";
  // k_render_scatter packs a small quad's pixel box origin as i0 | j0 << 16 (QuadStore::box)
  if (p->model_width > 65536 || p->model_height > 65536)
    return "model image side > 65536 (the render pass packs pixel boxes in 16 bits)";
  if (!(p->max_depth > p->min_depth) || !(p->model_max_depth > p->model_min_depth)) return "max depth <= min depth";
  // Q33.30 head-room of the exact ICP sums: no int64 sum may wrap (DESIGN.md section 2)
  const double range = (p->max_depth > p->model_max_depth ? p->max_depth : p->model_max_depth) + kIcpPoseMargin;
  if ((double)p->data_width * p->data_height * range * range * 1073741824.0 > 9223372036854775807.0)
    return "data pixels x (max depth + 25 m)^2 x 2^30 exceeds the int64 range of the exact ICP sums";
  return nullptr;
}

int sb_create(const sb_params* p, int device, sb_ctx** out) {
  if (!out) return SB_ERR_INVALID;
  if (const char* why = check_params(p)) {
    fprintf(stderr, "sb_create: %s\n", why);
    return SB_ERR_INVALID;
  }
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return SB_ERR_NOGPU;  // no CPU fallback
  if (device < 0 || device >= n) return SB_ERR_INVALID;
  sb_ctx* c = new sb_ctx();
  c->device = device;
  c->p = *p;
  if (cudaSetDevice(device) != cudaSuccess) {
    delete c;
    return SB_ERR_CUDA;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
  c->icp_blocks = icp_grid_blocks(c->sm_count);
  {
    // the Gauss-Newton loop is one cooperative launch (the host all-reduce callback aside): no device without it
    int coop = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device);
    int maxb = coop ? gn_persistent_max_blocks(c->sm_count) : 0;
    if (maxb <= 0) {
      fprintf(stderr, "sb_create: device %d cannot run the cooperative Gauss-Newton kernel\n", device);
      delete c;
      return SB_ERR_CUDA;
    }
    c->icp_coop_blocks = icp_balanced_blocks(p->data_width * p->data_height, maxb < c->icp_blocks ? maxb : c->icp_blocks);
    c->icp_blocks = icp_balanced_blocks(p->data_width * p->data_height, c->icp_blocks);
  }
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete c;
    return SB_ERR_CUDA;
  }
  derive(c);
  int r = alloc_buffers(c);
  if (r != SB_OK) {
    fprintf(stderr, "sb_create: %s\n", c->err.c_str());
    cudaStreamDestroy(c->stream);
    delete c;
    return r;
  }
  *out = c;
  return SB_OK;
}

int sb_destroy(sb_ctx* c) {
  if (!c) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  sb_comm_shutdown(c);
  for (auto& sl : c->prefetch) {
    if (sl.done) cudaEventDestroy(sl.done);
    if (sl.released) cudaEventDestroy(sl.released);
  }
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  for (cudaEvent_t e : c->state_ev)
    if (e) cudaEventDestroy(e);
  for (auto& r : c->prof.recs) {  // events of the per-kernel profiler (sb_profile_*)
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  for (cudaEvent_t e : c->prof.pool) cudaEventDestroy(e);
  cudaStreamDestroy(c->stream);
  delete c;  // frees the context's device and pinned memory
  return SB_OK;
}

int sb_reset(sb_ctx* c) {
  if (!c) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  return reset_state(c);
}

int sb_set_params(sb_ctx* c, const sb_params* p) {
  if (!c) return SB_ERR_INVALID;
  if (const char* why = check_params(p)) return fail(c, SB_ERR_INVALID, std::string("set_params: ") + why);
  if (p->data_width != c->p.data_width || p->data_height != c->p.data_height || p->model_width != c->p.model_width ||
      p->model_height != c->p.model_height)
    return fail(c, SB_ERR_STATE, "set_params: image sizes are fixed at sb_create (as in SurfelMapping's constructor)");
  c->p = *p;
  derive(c);
  c->memo.clear();
  return SB_OK;
}

int sb_get_params(const sb_ctx* c, sb_params* p) {
  if (!c || !p) return SB_ERR_INVALID;
  *p = c->p;
  return SB_OK;
}

const char* sb_last_error(const sb_ctx* c) { return c ? c->err.c_str() : "null context"; }

int sb_synchronize(sb_ctx* c) {
  if (!c) return SB_ERR_INVALID;
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}

void* sb_stream(sb_ctx* c) { return c ? (void*)c->stream : nullptr; }
uint64_t sb_launch_count(const sb_ctx* c) { return c ? c->launches : 0; }

int sb_frame_create(sb_ctx* c, int w, int h, sb_frame** out) {
  if (!c || !out) return fail(c, SB_ERR_INVALID, "frame_create: bad arguments");
  cudaSetDevice(c->device);
  FramePtr f;
  int r = frame_create(c, w, h, f);
  if (r) return r;
  *out = f.release();
  return SB_OK;
}
int sb_frame_destroy(sb_frame* f) {
  if (!f) return SB_ERR_INVALID;
  cudaStreamSynchronize(f->ctx->stream);
  frame_written(f->ctx, f);
  delete f;
  return SB_OK;
}
int sb_frame_copy(sb_frame* dst, const sb_frame* src) {
  if (!dst || !src || dst->d.W != src->d.W || dst->d.H != src->d.H) return SB_ERR_INVALID;
  sb_ctx* c = dst->ctx;
  frame_written(c, dst);
  SB_CUDA(c, cudaMemcpyAsync(dst->base, src->base, (size_t)src->d.W * src->d.H * 48, cudaMemcpyDeviceToDevice, c->stream));
  return SB_OK;
}
static float4* frame_plane(const sb_frame* f, int which) {
  return which == SB_MAP_VERTEX ? f->d.vertex : (which == SB_MAP_NORMAL ? f->d.normal : f->d.semantic);
}
int sb_frame_download(const sb_frame* f, int which, float* dst) {
  if (!f || !dst || which < 0 || which > 2) return SB_ERR_INVALID;
  sb_ctx* c = f->ctx;
  SB_CUDA(c, cudaMemcpyAsync(dst, frame_plane(f, which), (size_t)f->d.W * f->d.H * 16, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}
int sb_frame_upload(sb_frame* f, int which, const float* src) {
  if (!f || !src || which < 0 || which > 2) return SB_ERR_INVALID;
  sb_ctx* c = f->ctx;
  frame_written(c, f);
  SB_CUDA(c, cudaMemcpyAsync(frame_plane(f, which), src, (size_t)f->d.W * f->d.H * 16, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}
int sb_frame_size(const sb_frame* f, int* w, int* h) {
  if (!f) return SB_ERR_INVALID;
  if (w) *w = f->d.W;
  if (h) *h = f->d.H;
  return SB_OK;
}

int sb_preprocess(sb_ctx* c, const float* pts4, const float* labels, const float* probs, uint32_t n, uint32_t timestamp,
                  int on_device, sb_frame* out) {
  if (!c || !out || (!pts4 && n)) return fail(c, SB_ERR_INVALID, "preprocess: null argument");
  if (out->d.W != c->kp.W || out->d.H != c->kp.H) return fail(c, SB_ERR_INVALID, "preprocess: frame size mismatch");
  cudaSetDevice(c->device);
  const float4* dp; const float* dl; const float* dq;
  int r = upload_scan(c, pts4, labels, probs, n, on_device, &dp, &dl, &dq);
  if (r) return r;
  frame_written(c, out);
  launch_preprocess(L_(c), c->kp, dp, dl, dq, n, timestamp, c->prep, out->d, nullptr, nullptr, nullptr, nullptr);
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}

int sb_map_render(sb_ctx* c, const float pose_old[16], const float pose_new[16], float conf_thr, sb_frame* out) {
  if (!c || !pose_old || !pose_new || !out) return fail(c, SB_ERR_INVALID, "map_render: null argument");
  if (out->d.W != c->kp.Wm || out->d.H != c->kp.Hm) return fail(c, SB_ERR_INVALID, "map_render: frame size mismatch");
  cudaSetDevice(c->device);
  int r = render_full(c, pose_old, pose_new, conf_thr, out);
  if (r) return r;
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}
int sb_map_render_active(sb_ctx* c, const float pose[16], float conf_thr) {
  if (!c || !pose) return fail(c, SB_ERR_INVALID, "map_render_active: null argument");
  cudaSetDevice(c->device);
  int r = render_single(c, pose, conf_thr, 1);
  if (r) return r;
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}
int sb_map_render_inactive(sb_ctx* c, const float pose[16], float conf_thr) {
  if (!c || !pose) return fail(c, SB_ERR_INVALID, "map_render_inactive: null argument");
  cudaSetDevice(c->device);
  int r = render_single(c, pose, conf_thr, 0);
  if (r) return r;
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}
int sb_map_render_composed(sb_ctx* c, const float pose_old[16], const float pose_new[16], float conf_thr) {
  if (!c || !pose_old || !pose_new) return fail(c, SB_ERR_INVALID, "map_render_composed: null argument");
  cudaSetDevice(c->device);
  return render_composed_internal(c, pose_old, pose_new, conf_thr);
}
int sb_map_frame(sb_ctx* c, int which, sb_frame** out) {
  if (!c || !out || which < 0 || which > 2) return SB_ERR_INVALID;
  *out = which == SB_FRAME_OLD ? c->f_old : (which == SB_FRAME_NEW ? c->f_new : c->f_comp);
  return SB_OK;
}

void sb_icp_unpack(const int64_t raw32[32], double out48[48]) { sbg::unpack48((const long long*)raw32, out48); }

int sb_icp_jacobian(sb_ctx* c, const sb_frame* data, const sb_frame* model, const double pose[16], int iteration,
                    float max_distance, float max_angle_deg, int row_begin, int row_end, double out48[48],
                    int64_t raw32[32]) {
  int r = icp_check(c, data, model);
  if (r) return r;
  if (!pose || row_begin < 0 || row_end > c->kp.H || row_begin > row_end)
    return fail(c, SB_ERR_INVALID, "icp_jacobian: bad pose / row range");
  cudaSetDevice(c->device);
  long long raw[32];
  if ((r = icp_jacobian_raw(c, data, model, pose, iteration, max_distance, max_angle_deg, row_begin, row_end, true, raw)))
    return r;
  if (raw32) memcpy(raw32, raw, sizeof(raw));
  if (out48) sbg::unpack48(raw, out48);
  return SB_OK;
}

int sb_icp_minimize(sb_ctx* c, const sb_frame* data, const sb_frame* model, const double T0[16], int max_iter, double eps,
                    double delta, float max_distance, float max_angle_deg, double pose_out[16], double out48[48],
                    int* iters, double* history, int* history_len) {
  int r = icp_check(c, data, model);
  if (r) return r;
  if (!T0) return fail(c, SB_ERR_INVALID, "icp_minimize: null T0");
  // max_iter <= 0 is the reference's "no limit" (LieGaussNewton.cpp:24); the device loop stops after kMaxGnIter = 256
  // iterations at the latest. A caller-sized history buffer ((max_iter+1)*16 doubles) is only safe for 1..256.
  if (history && (max_iter <= 0 || max_iter > kMaxGnIter))
    return fail(c, SB_ERR_INVALID, "icp_minimize: with a history buffer max_iter must be in [1, 256]");
  cudaSetDevice(c->device);
  if ((r = icp_minimize_enqueue(c, data, model, T0, max_iter, eps, delta, max_distance, max_angle_deg, true))) return r;
  if ((r = icp_minimize_fetch(c, pose_out, out48, iters, history, history_len))) return r;
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}

void sb_se3_exp(const double x[6], double T[16]) { sbg::se3_exp(x, T); }

void sb_se3_log(const double M[16], double x[6]) {  // lie_algebra.cpp:36-71 (not on the hot path; libm fp64)
  for (int i = 0; i < 6; ++i) x[i] = 0.0;
  double d = 0.5 * (((M[0] + M[5]) + M[10]) - 1.0);
  double K[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (d < 1 - 1e-10) {
    double theta = acos(d);
    double f = theta / (2 * sin(theta));
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc) K[r * 3 + cc] = f * (M[cc * 4 + r] - M[r * 4 + cc]);
    x[3] = K[2 * 3 + 1]; x[4] = K[0 * 3 + 2]; x[5] = K[1 * 3 + 0];
  }
  double theta = sqrt((x[3] * x[3] + x[4] * x[4]) + x[5] * x[5]);
  x[0] = M[12]; x[1] = M[13]; x[2] = M[14];
  if (fabs(theta) > 1e-10) {
    double half = 0.5 * theta;
    double beta = 1 / (theta * theta) * (1 - theta * cos(half) / (2 * sin(half)));
    double t[3] = {M[12], M[13], M[14]};
    for (int r = 0; r < 3; ++r) {
      double acc = 0;
      for (int cc = 0; cc < 3; ++cc) {
        double k2 = (K[r * 3 + 0] * K[0 * 3 + cc] + K[r * 3 + 1] * K[1 * 3 + cc]) + K[r * 3 + 2] * K[2 * 3 + cc];
        double Vi = ((r == cc ? 1.0 : 0.0) + (-0.5) * K[r * 3 + cc]) + beta * k2;
        acc += Vi * t[cc];
      }
      x[r] = acc;
    }
  }
}

int sb_ldlt_solve6(const double A[36], const double b[6], double x[6]) {
  sbg::ldlt_solve6(A, b, x);
  return SB_OK;
}
int sb_gn_step(const double out48[48], double last_error, double eps, double delta, double pose[16], double dx[6]) {
  return sbg::gn_step(out48, last_error, eps, delta, pose, dx);
}

int sb_map_update(sb_ctx* c, const float pose[16], const sb_frame* frame) {
  if (!c || !pose || !frame) return fail(c, SB_ERR_INVALID, "map_update: null argument");
  if (frame->d.W != c->kp.W || frame->d.H != c->kp.H) return fail(c, SB_ERR_INVALID, "map_update: frame size mismatch");
  cudaSetDevice(c->device);
  int r = map_update(c, pose, frame);
  if (r) return r;
  SB_CUDA(c, cudaGetLastError());
  return SB_OK;
}

int sb_map_update_poses(sb_ctx* c, const float* poses16, uint32_t count) {
  if (!c || (!poses16 && count)) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  for (uint32_t t = 0; t < count && t < kMaxPoses; ++t) {
    int r = set_pose_entry(c, t, poses16 + 16 * (size_t)t);
    if (r) return r;
  }
  return SB_OK;
}
int sb_map_set_pose(sb_ctx* c, uint32_t t, const float pose[16]) {
  if (!c || !pose) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  return set_pose_entry(c, t, pose);
}
int sb_map_size(sb_ctx* c, uint32_t* n) {
  if (!c || !n) return SB_ERR_INVALID;
  *n = n_live(c);  // (no compaction: dead slots cost the readers nothing but a byte)
  return SB_OK;
}
int sb_map_timestamp(sb_ctx* c, uint32_t* t) {
  if (!c || !t) return SB_ERR_INVALID;
  *t = c->map_timestamp;
  return SB_OK;
}
int sb_map_download(sb_ctx* c, sb_surfel* dst, uint32_t cap, uint32_t* n) {
  if (!c || (!dst && cap)) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  int r = compact_map(c);
  if (r) return r;
  uint32_t k = c->n_host < cap ? c->n_host : cap;
  if (n) *n = k;
  if (k == 0) return SB_OK;
  // transpose the SoA lanes into 64-byte records inside the (idle) T lanes, then one D2H copy
  launch_soa_to_aos(L_(c), c->A, reinterpret_cast<sb_surfel*>(c->T.p0), k);
  SB_CUDA(c, cudaMemcpyAsync(dst, c->T.p0, (size_t)k * 64, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}
int sb_map_upload(sb_ctx* c, const sb_surfel* src, uint32_t n, uint32_t timestamp) {
  if (!c || (!src && n)) return SB_ERR_INVALID;
  if (n > kMaxSurfels) return fail(c, SB_ERR_CAPACITY, "map_upload: more than 4194304 surfels");
  cudaSetDevice(c->device);
  if (n) {
    SB_CUDA(c, cudaMemcpyAsync(c->T.p0, src, (size_t)n * 64, cudaMemcpyHostToDevice, c->stream));
    launch_aos_to_soa(L_(c), reinterpret_cast<const sb_surfel*>(c->T.p0), c->A, 0, n);
    SB_CUDA(c, cudaMemsetAsync(c->live, 1, n, c->stream));
  }
  for (uint32_t i = 0; i < n; ++i) {  // the pose-table entry of each surfel, as pose_index() reads it from the count field
    const float t = src[i].count;
    const uint32_t e = !(t >= 1.0f) ? 0u : t >= (float)(kMaxPoses - 1) ? kMaxPoses - 1 : (uint32_t)t;
    if (e + 1 > c->pose_ref_end) c->pose_ref_end = e + 1;
  }
  c->n_host = n;
  c->n_holes = 0;  // (overwritten: nothing to compact)
  c->n_upper = n;
  c->map_timestamp = timestamp;
  c->map_version += 1;
  SB_CUDA(c, cudaMemcpyAsync(c->res->counts, &c->n_host, 4, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  return SB_OK;
}
int sb_map_update_debug(sb_ctx* c, uint32_t* index_map, float* radius_map4, uint8_t* integrated, uint32_t* n_updated,
                        uint32_t* n_new) {
  if (!c) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  size_t Pd = (size_t)c->kp.W * c->kp.H;
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (index_map) {
    std::vector<unsigned long long> keys(Pd);
    SB_CUDA(c, cudaMemcpy(keys.data(), c->key_index, Pd * 8, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < Pd; ++i) index_map[i] = keys[i] == ~0ull ? 0u : (uint32_t)(keys[i] & 0xffffffffull) + 1u;
  }
  if (radius_map4) SB_CUDA(c, cudaMemcpy(radius_map4, c->radius_map, Pd * 16, cudaMemcpyDeviceToHost));
  if (integrated) SB_CUDA(c, cudaMemcpy(integrated, c->integrated, Pd, cudaMemcpyDeviceToHost));
  if (n_updated) *n_updated = c->n_updated;
  if (n_new) *n_new = c->n_new;
  return SB_OK;
}
int sb_map_submap_origin(sb_ctx* c, int32_t* i, int32_t* j, uint32_t* pending) {
  if (!c) return SB_ERR_INVALID;
  if (i) *i = c->origin_i;
  if (j) *j = c->origin_j;
  if (pending) *pending = (uint32_t)c->extraction.size();
  return SB_OK;
}

int sb_process_scan(sb_ctx* c, const float* pts4, const float* labels, const float* probs, uint32_t n, int on_device) {
  if (!c || (!pts4 && n)) return fail(c, SB_ERR_INVALID, "process_scan: null argument");
  cudaSetDevice(c->device);
  const sb_params& p = c->p;
  Launch L = L_(c);
  double t_all = now_s();
  // the upload can fail (out of memory for a larger scan): do it before any state of the context changes
  const float4* dp; const float* dl; const float* dq;
  int r = upload_scan(c, pts4, labels, probs, n, on_device, &dp, &dl, &dq);
  if (r) return r;
  // initialize(), SurfelMapping.cpp:323-331
  std::swap(c->cur, c->last);
  std::swap(c->cur_model, c->last_model);
  c->last_has_semantics = c->cur_has_semantics;
  c->cur_has_semantics = labels != nullptr;
  // ---- everything below is enqueued on the stream without a host round trip; ONE synchronisation at the end ----
  // preprocess(), :342-358
  frame_written(c, c->cur);
  launch_preprocess(L, c->kp, dp, dl, dq, n, c->timestamp, c->prep, c->cur->d, c->radius_map, c->key_index, c->integrated,
                    c->group_counts);
  c->prepped_for_update = true;
  float ct = conf_threshold(c);
  float Pold[16], Pnew[16];
  cast_f(c->currentPose_old, Pold);
  cast_f(c->currentPose_new, Pnew);
  if ((r = render_full(c, Pold, Pnew, ct, c->last_model))) return r;
  const bool had_icp = c->timestamp > 0;
  bool tables_ready = false, index_fused = false;
  bool loop_ran = false;
  if (had_icp) {
    if ((r = update_pose_enqueue(c, &tables_ready, &index_fused))) return r;
    if (c->close_loops) {  // checkLoopClosure(), :196-200; its renders overwrite the product table of the map update
      if ((r = loop_closure_step(c))) return r;
      tables_ready = false;
      loop_ran = true;
    }
  } else {
    launch_pose_finalize(L, c->gn2, &c->res->pose, 0, c->poses, c->poses_inv, c->map_timestamp);
  }
  // updateMap(), :797-804
  const uint32_t t_map = c->map_timestamp;
  if ((r = map_update(c, nullptr, c->cur, &c->res->pose.P_cur, &c->res->pose.invP_cur, tables_ready, index_fused)))
    return r;
  float ct2 = conf_threshold(c);
  if (p.render_after_update) {
    if ((r = render_full(c, nullptr, nullptr, ct2, c->cur_model, &c->res->pose.invP_cur, true))) return r;
  }
  // ---- the scan's results: pose block, statistics sums, surfel counts ----
  const ResultBlock& rb = c->host->result;
  SB_CUDA(c, cudaMemcpyAsync(&c->host->result, c->res, sizeof(ResultBlock), cudaMemcpyDeviceToHost, c->stream));
  const double t_enqueued = now_s();
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  const double t_synced = now_s();
  SB_CUDA(c, cudaGetLastError());
  // the map update has run on the device even when the scan fails below: the host's counts follow it, so that a later
  // compaction (download) covers the map as it is
  c->n_host = rb.counts[0];
  c->n_holes = c->lazy_update ? rb.counts[5] : 0;
  c->n_upper = rb.counts[0];
  c->n_updated = rb.counts[2];
  c->n_new = rb.counts[3];
  if (rb.pose.gn_error) return gn_fail(c);
  if (!loop_ran) absorb_pose_block(c, rb, had_icp);  // (the loop-closure step has already done it, and chose currentPose_old_)
  const Mat4 P_cur = rb.pose.P_cur;
  if (t_map < kMaxPoses) {  // host mirror of the pose table entry written by k_pose_finalize
    memcpy(&c->h_poses[16 * (size_t)t_map], P_cur.m, 64);
    sbg::rigid_inverse_f(P_cur.m, &c->h_poses_inv[16 * (size_t)t_map]);
  }
  if (p.render_after_update)  // the render's memo entry, now that the pose bits are known on the host
    c->memo.store(memo_key(c, P_cur.m, P_cur.m, ct2, c->cur_model));
  // submap paging (SurfelMap.cpp:547, 744-824) with the pose now known on the host. Re-inserting cached tiles changes
  // the map after the model was rendered: render again in that (rare) case, as the reference renders after paging.
  {
    const uint32_t n0 = c->n_host;
    if ((r = update_active_submaps(c, P_cur.m))) return r;
    if (c->n_host != n0 && p.render_after_update && (r = render_full(c, P_cur.m, P_cur.m, ct2, c->cur_model))) return r;
  }
  c->stats[7] = n_live(c);
  // The reference's three stage timers (preprocessing / icp / mapping) have no meaning here -- the stages overlap on
  // the stream; the slots carry the host-side split of the call instead: enqueue, wait for the device, bookkeeping.
  const double t_end = now_s();
  c->stats[8] = t_enqueued - t_all;
  c->stats[9] = t_synced - t_enqueued;
  c->stats[10] = t_end - t_synced;
  c->stats[11] = t_end - t_all;
  c->timestamp += 1;
  return SB_OK;
}

// Optional: start copying the NEXT scan's host buffers to the device on a separate copy stream while the current scan
// is being processed. A later sb_process_scan(..., on_device = 0) with the same host pointers and count uses the staged
// copy instead of copying again. (The reference uploads inside processScan, SurfelMapping.cpp:325-331; this is the usual
// double buffering of a sensor driver.) Buffers must stay unchanged until that sb_process_scan; pinned memory overlaps.
int sb_prefetch_scan(sb_ctx* c, const float* pts4, const float* labels, const float* probs, uint32_t n) {
  if (!c || (!pts4 && n)) return fail(c, SB_ERR_INVALID, "prefetch_scan: null argument");
  cudaSetDevice(c->device);
  int rg = grow_point_buffers(c, n);
  if (rg) return rg;
  if (!c->copy_stream) {
    SB_CUDA(c, cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (auto& sl : c->prefetch) {
      SB_CUDA(c, cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
      SB_CUDA(c, cudaEventCreateWithFlags(&sl.released, cudaEventDisableTiming));
    }
  }
  for (auto& sl : c->prefetch)
    if (!sl.pts) {  // first use, or the staging capacity grew
      SB_CUDA(c, dev_alloc(sl.pts, c->pts_cap * 16));
      SB_CUDA(c, dev_alloc(sl.labels, c->pts_cap * 4));
      SB_CUDA(c, dev_alloc(sl.probs, c->pts_cap * 4));
    }
  sb_ctx::PrefetchSlot* slot = nullptr;
  for (auto& sl : c->prefetch)  // a slot that neither holds an unconsumed scan nor feeds the scan in flight
    if (!sl.valid && !sl.in_use) {
      slot = &sl;
      break;
    }
  if (!slot) return fail(c, SB_ERR_STATE, "prefetch_scan: two scans are already staged");
  if (slot->has_released) SB_CUDA(c, cudaStreamWaitEvent(c->copy_stream, slot->released, 0));  // readers are done first
  if (n) SB_CUDA(c, cudaMemcpyAsync(slot->pts, pts4, (size_t)n * 16, cudaMemcpyHostToDevice, c->copy_stream));
  if (labels && n) SB_CUDA(c, cudaMemcpyAsync(slot->labels, labels, (size_t)n * 4, cudaMemcpyHostToDevice, c->copy_stream));
  if (probs && n) SB_CUDA(c, cudaMemcpyAsync(slot->probs, probs, (size_t)n * 4, cudaMemcpyHostToDevice, c->copy_stream));
  SB_CUDA(c, cudaEventRecord(slot->done, c->copy_stream));
  slot->host_pts = pts4;
  slot->n = n;
  slot->has_labels = labels != nullptr;
  slot->has_probs = probs != nullptr;
  slot->valid = true;
  return SB_OK;
}

void sb_default_loop_params(sb_loop_params* p) {  // SurfelMapping.h:223-235 overridden by config/default.xml:70-76
  if (!p) return;
  p->search_distance = 50.0f;
  p->min_trajectory_distance = 200.0f;
  p->min_verifications = 5;
  p->residual_threshold = 1.15f;
  p->outlier_threshold = 1.1f;
  p->valid_threshold = 0.95f;
}

int sb_set_loop_closure(sb_ctx* c, int enabled, const sb_loop_params* p) {
  if (!c) return SB_ERR_INVALID;
  sb_loop_params d;
  sb_default_loop_params(&d);
  if (p) d = *p;
  c->loop.p.search_distance = d.search_distance;
  c->loop.p.min_trajectory_distance = d.min_trajectory_distance;
  c->loop.p.min_verifications = d.min_verifications;
  c->loop.p.residual_threshold = d.residual_threshold;
  c->loop.p.outlier_threshold = d.outlier_threshold;
  c->loop.p.valid_threshold = d.valid_threshold;
  if (enabled && !c->close_loops) c->loop.reset();
  c->close_loops = enabled != 0;
  return SB_OK;
}

int sb_get_loop_info(sb_ctx* c, sb_loop_info* o) {
  if (!c || !o) return SB_ERR_INVALID;
  const suma_b200::loop::State& L = c->loop;
  memset(o, 0, sizeof(*o));
  o->enabled = c->close_loops ? 1u : 0u;
  o->loop_count = L.loop_count;
  o->time_without_loop_closure = L.time_without_loop_closure;
  o->candidates_tested = L.candidates_tested;
  o->loop_edges_added = L.loop_edges_added;
  o->unverified = (uint32_t)L.unverified.size();
  o->already_verified = L.already_verified ? 1u : 0u;
  o->found_candidate = L.found_candidate ? 1u : 0u;
  o->use_candidate = L.use_candidate ? 1u : 0u;
  o->optimisation_requested = L.optimisation_requested ? 1u : 0u;
  o->last_added_candidate = L.last_added_candidate;
  o->n_edges = (uint32_t)L.graph.edges.size();
  o->n_poses = (uint32_t)L.graph.poses.size();
  o->valid_ratio = L.stat_valid_ratio;
  o->outlier_ratio = L.stat_outlier_ratio;
  o->rel_error = L.stat_rel_error;
  o->residual_old = L.result_old.residual;
  o->residual_new = L.result_new.residual;
  memcpy(o->current_pose_old, c->currentPose_old, sizeof(o->current_pose_old));
  return SB_OK;
}

int sb_get_loop_edges(sb_ctx* c, sb_loop_edge* dst, uint32_t cap, uint32_t* n) {
  if (!c || (!dst && cap)) return SB_ERR_INVALID;
  const auto& E = c->loop.graph.edges;
  uint32_t k = (uint32_t)E.size() < cap ? (uint32_t)E.size() : cap;
  for (uint32_t i = 0; i < k; ++i) {
    dst[i].from = E[i].from;
    dst[i].to = E[i].to;
    memcpy(dst[i].rel_pose, E[i].rel.m, 128);
  }
  if (n) *n = (uint32_t)E.size();
  return SB_OK;
}

// SurfelMapping::integrateLoopClosures (SurfelMapping.cpp:212-258): the host application optimised the pose graph the
// library recorded (sb_get_loop_edges / sb_get_optimisation_request) and hands the poses of scans 0 .. n-1 back. The
// bookkeeping is State::integrate of include/suma_b200_loop.hpp (shared with the oracle twin and checked there against the
// reference's own code); here only its consequences reach the device: SurfelMap::updatePoses and the current pose.
int sb_integrate_loop_closures(sb_ctx* c, const double* poses16, uint32_t n, uint32_t* integrated) {
  namespace lp = suma_b200::loop;
  if (integrated) *integrated = 0;
  if (!c) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  lp::State& S = c->loop;
  if (!c->close_loops || !S.optimisation_requested) return SB_OK;  // nothing pending (the reference: !currentlyOptimizing_)
  std::vector<lp::M4> opt;
  if (poses16) {
    if (n <= (uint32_t)S.before_id) return fail(c, SB_ERR_INVALID, "integrate_loop_closures: fewer poses than the graph held at the request");
    opt.resize(n);
    for (uint32_t i = 0; i < n; ++i) memcpy(opt[i].m, poses16 + 16 * (size_t)i, 128);
  } else {  // identity "optimiser": the poses the graph held when the optimisation was requested
    opt.assign(S.graph.poses.begin(), S.graph.poses.begin() + (long)S.requested_size);
  }
  lp::M4 cur, cold, cnew;
  memcpy(cur.m, c->currentPose, 128);
  memcpy(cold.m, c->currentPose_old, 128);
  memcpy(cnew.m, c->currentPose_new, 128);
  std::vector<lp::M4> all = S.integrate(opt, cur, cold, cnew);
  if (all.empty()) return fail(c, SB_ERR_STATE, "integrate_loop_closures: no optimisation request pending");
  std::vector<float> pf(all.size() * 16);
  for (size_t t = 0; t < all.size(); ++t) lp::to_float(all[t], &pf[16 * t]);
  int r = sb_map_update_poses(c, pf.data(), (uint32_t)all.size());  // map_->updatePoses(casted_poses)   :232
  if (r) return r;
  memcpy(c->currentPose_old, cold.m, 128);  // currentPose_new_ = currentPose_old_ = currentPose_   :240
  memcpy(c->currentPose_new, cnew.m, 128);
  if ((r = sb_set_current_pose(c, cur.m))) return r;  // currentPose_ = difference * currentPose_   :236 (host + device copy)
  if (integrated) *integrated = (uint32_t)all.size();
  return SB_OK;
}

int sb_set_current_pose(sb_ctx* c, const double pose[16]) {  // SurfelMapping::setCurrentPose, SurfelMapping.cpp:880-882
  if (!c || !pose) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  memcpy(c->currentPose, pose, sizeof(c->currentPose));
  // the pose also lives on the device (PoseDev::currentPose): the next scan chains its increment onto it
  SB_CUDA(c, cudaMemcpyAsync(c->res->pose.currentPose, c->currentPose, sizeof(c->currentPose), cudaMemcpyHostToDevice,
                             c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  c->memo.clear();
  return SB_OK;
}

int sb_get_pose(sb_ctx* c, double pose[16]) {
  if (!c || !pose) return SB_ERR_INVALID;
  memcpy(pose, c->currentPose, sizeof(c->currentPose));
  return SB_OK;
}
int sb_get_last_pose(sb_ctx* c, double pose[16]) {
  if (!c || !pose) return SB_ERR_INVALID;
  memcpy(pose, c->lastPose, sizeof(c->lastPose));
  return SB_OK;
}
int sb_timestamp(sb_ctx* c, uint32_t* t) {
  if (!c || !t) return SB_ERR_INVALID;
  *t = c->timestamp;
  return SB_OK;
}
int sb_slam_frame(sb_ctx* c, int which, sb_frame** out) {
  if (!c || !out || which < 0 || which > 3) return SB_ERR_INVALID;
  sb_frame* f[4] = {c->cur, c->last, c->cur_model, c->last_model};
  *out = f[which];
  return SB_OK;
}
int sb_get_statistics(sb_ctx* c, double stats[16]) {
  if (!c || !stats) return SB_ERR_INVALID;
  memcpy(stats, c->stats, sizeof(c->stats));
  return SB_OK;
}


// ---- profiling ------------------------------------------------------------------------------------------------
int sb_profile_enable(sb_ctx* c, int on) {
  if (!c) return SB_ERR_INVALID;
  c->prof.on = on != 0;
  return SB_OK;
}
int sb_profile_kernels(void) { return K_COUNT; }
const char* sb_profile_name(int id) { return kernel_name(id); }
int sb_profile_collect(sb_ctx* c, double* total_ms, uint64_t* count, int cap) {
  if (!c || !total_ms || !count || cap < K_COUNT) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < K_COUNT; ++i) {
    total_ms[i] = 0.0;
    count[i] = 0;
  }
  for (auto& r : c->prof.recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
      total_ms[r.id] += ms;
      count[r.id] += 1;
    }
    c->prof.pool.push_back(r.e0);
    c->prof.pool.push_back(r.e1);
  }
  c->prof.recs.clear();
  return SB_OK;
}

// ---- multi-GPU ------------------------------------------------------------------------------------------------
int sb_comm_export(sb_ctx* c, uint8_t handle[64]) {
  if (!c || !handle) return SB_ERR_INVALID;
  cudaSetDevice(c->device);
  if (!c->mailbox) {
    // A CUDA IPC handle names the whole underlying allocation and cudaIpcOpenMemHandle returns ITS base: small
    // cudaMalloc requests are carved out of shared 2 MiB blocks, so an 8 KiB mailbox would be opened at the wrong
    // address on the peer. A 2 MiB allocation owns its block: exported pointer == base.
    SB_CUDA(c, dev_alloc(c->mailbox, 2u << 20));
  }
  // Every export starts a fresh session: stamps of an earlier session must not match the epochs of the next one (both
  // restart at 1). Peers cannot write yet -- they only learn this mailbox's address from the handle returned here.
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  SB_CUDA(c, cudaMemset(c->mailbox, 0, 2u << 20));
  cudaIpcMemHandle_t h;
  SB_CUDA(c, cudaIpcGetMemHandle(&h, c->mailbox));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle, &h, 64);
  return SB_OK;
}

int sb_comm_init(sb_ctx* c, int rank, int nranks, const uint8_t* handles, int row_begin, int row_end) {
  if (!c || !handles || nranks < 1 || nranks > 8 || rank < 0 || rank >= nranks)
    return fail(c, SB_ERR_INVALID, "comm_init: bad rank / nranks (max 8)");
  if (row_begin < 0 || row_end > c->kp.H || row_begin > row_end) return fail(c, SB_ERR_INVALID, "comm_init: bad rows");
  if (!c->mailbox) return fail(c, SB_ERR_STATE, "comm_init: call sb_comm_export first");
  cudaSetDevice(c->device);
  memset(&c->comm, 0, sizeof(c->comm));
  c->comm.rank = rank;
  c->comm.nranks = nranks;
  c->comm.epoch = c->comm_epoch;
  c->peer_ptrs.clear();
  for (int r = 0; r < nranks; ++r) {
    if (r == rank) {
      c->comm.mailbox[r] = c->mailbox;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + 64 * (size_t)r, 64);
    void* ptr = nullptr;
    SB_CUDA(c, cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    c->comm.mailbox[r] = (long long*)ptr;
    c->peer_ptrs.push_back(ptr);
  }
  SB_CUDA(c, cudaMemset(c->comm_epoch, 0, 64));
  c->row_begin = row_begin;
  c->row_end = row_end;
  c->comm_on = true;  // with nranks == 1 the exchange loops back to the own mailbox
  return SB_OK;
}

int sb_comm_set_callback(sb_ctx* c, sb_allreduce_fn fn, void* user, int row_begin, int row_end) {
  if (!c) return SB_ERR_INVALID;
  if (fn && (row_begin < 0 || row_end > c->kp.H || row_begin > row_end)) return fail(c, SB_ERR_INVALID, "comm: bad rows");
  if (fn && c->comm_on) return fail(c, SB_ERR_STATE, "comm: the fused peer-memory mode is already active");
  c->comm_cb = fn;
  c->comm_cb_user = user;
  if (fn) {
    c->row_begin = row_begin;
    c->row_end = row_end;
  }
  return SB_OK;
}

int sb_comm_shutdown(sb_ctx* c) {
  if (!c) return SB_ERR_INVALID;
  c->comm_cb = nullptr;
  for (void* p : c->peer_ptrs) cudaIpcCloseMemHandle(p);
  c->peer_ptrs.clear();
  c->comm_on = false;
  return SB_OK;
}

}  // extern "C"

// =========================================================================================================
// Checkpoints: sb_state_size / sb_state_save / sb_state_load (no counterpart in the reference, whose Posegraph::save/load
// are empty stubs). DESIGN.md section 9 lists which member of sb_ctx is saved, derived or context-local, and the format.
// =========================================================================================================
namespace {

static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "checkpoints are written little-endian");
const char kStateMagic[8] = {'S', 'B', 'S', 'T', 'A', 'T', 'E', '\0'};
constexpr uint32_t kStateFormat = 1;
constexpr size_t kStageBytes = 16u << 20;  // one half of the pinned double buffer
enum StateSection : uint32_t { S_HOST = 1, S_LOOP, S_POSES, S_RESULT, S_TILES, S_SURFELS, S_POOL, S_FRAMES };

#define SB_PARAM_FIELDS(X)                                                                                              \
  X(data_width) X(data_height) X(data_fov_up) X(data_fov_down) X(min_depth) X(max_depth) X(model_width)                 \
  X(model_height) X(model_fov_up) X(model_fov_down) X(model_min_depth) X(model_max_depth) X(max_iterations)            \
  X(stopping_threshold) X(delta) X(icp_max_distance) X(icp_max_angle) X(weighting) X(factor) X(initialize_identity)     \
  X(bilinear_sampling) X(fallback_mode) X(fallback_max_distance) X(fallback_max_angle) X(compose_rendering)             \
  X(max_loop_closure_distance) X(min_radius) X(max_radius) X(max_angle) X(map_max_distance) X(map_max_angle)            \
  X(unstable_age) X(confidence_mode) X(confidence_threshold) X(p_stable) X(p_prior) X(sigma_angle) X(sigma_distance)    \
  X(use_stability) X(active_timestamps) X(max_weight) X(weighting_scheme) X(averaging_scheme) X(update_always)          \
  X(submap_dimension) X(submap_extent) X(partial_extraction) X(label_offset_quirk) X(render_after_update)
#define SB_LOOP_PARAM_FIELDS(X)                                                                                         \
  X(search_distance) X(min_trajectory_distance) X(min_verifications) X(residual_threshold) X(outlier_threshold)         \
  X(valid_threshold) X(delta_timestamp)

// Field-by-field little-endian writer / reader: no padding byte of a C++ struct ever reaches a checkpoint, so that
// saving a loaded checkpoint reproduces it byte for byte.
struct Writer {
  std::vector<uint8_t> b;
  template <class T>
  void put(const T& v) {
    const uint8_t* p = reinterpret_cast<const uint8_t*>(&v);
    b.insert(b.end(), p, p + sizeof(T));
  }
  void bytes(const void* p, size_t n) {
    const uint8_t* q = static_cast<const uint8_t*>(p);
    b.insert(b.end(), q, q + n);
  }
  void align8() { b.resize((b.size() + 7) & ~size_t(7), 0); }
  size_t open(uint32_t id) {  // section header: id, 0, payload length (patched by close)
    put(id); put(uint32_t(0)); put(uint64_t(0));
    return b.size();
  }
  void close(size_t start) {
    align8();
    const uint64_t len = b.size() - start;
    memcpy(&b[start - 8], &len, 8);
  }
};
struct Reader {
  const uint8_t* p;
  size_t n, off = 0;
  bool ok = true;
  template <class T>
  T get() {
    T v{};
    if (!ok || n - off < sizeof(T)) { ok = false; return v; }
    memcpy(&v, p + off, sizeof(T));
    off += sizeof(T);
    return v;
  }
  void bytes(void* dst, size_t k) {
    if (!ok || n - off < k) { ok = false; return; }
    memcpy(dst, p + off, k);
    off += k;
  }
  uint32_t count(size_t elem) {  // a length prefix that cannot claim more elements than bytes remain
    uint32_t k = get<uint32_t>();
    if (ok && (uint64_t)k * elem > n - off) ok = false;
    return ok ? k : 0;
  }
  void align8() {
    size_t a = (off + 7) & ~size_t(7);
    if (a > n) ok = false; else off = a;
  }
};

namespace lp = suma_b200::loop;

// Everything a checkpoint holds except the three device-resident bulk sections (surfels, tile pool, frames).
struct StateImage {
  sb_params p;
  uint32_t timestamp = 0, trackLoss = 0;
  double currentPose[16], lastPose[16], currentPose_old[16], currentPose_new[16], lastIncrement[16], lastPose_old[16];
  float confidence_threshold = 0.f, log_unstable_slam = 0.f;
  double stats[16];
  uint32_t cur_has_semantics = 0, last_has_semantics = 0, close_loops = 0;
  uint32_t n_live = 0, map_timestamp = 0, pose_ref_end = 0, n_updated = 0, n_new = 0;
  int32_t origin_i = 0, origin_j = 0;
  std::vector<std::pair<int32_t, int32_t>> extraction;
  std::vector<std::pair<std::pair<int32_t, int32_t>, DevTile>> tiles;
  uint32_t n_slots = 0, tiles_pending = 0, pool_end = 0;
  std::vector<float> poses, poses_inv;  // the used entries of the device pose tables
  ResultBlock result;
  std::vector<uint2> tile_rec;
  lp::State loop;
};

void put_m4(Writer& w, const lp::M4& m) { w.bytes(m.m, sizeof(m.m)); }
lp::M4 get_m4(Reader& r) {
  lp::M4 m;
  r.bytes(m.m, sizeof(m.m));
  return m;
}
void put_edges(Writer& w, const std::vector<lp::Edge>& E) {
  w.put((uint32_t)E.size());
  for (const lp::Edge& e : E) { w.put(e.from); w.put(e.to); put_m4(w, e.rel); }
}
std::vector<lp::Edge> get_edges(Reader& r) {
  std::vector<lp::Edge> E(r.count(136));
  for (lp::Edge& e : E) { e.from = r.get<int32_t>(); e.to = r.get<int32_t>(); e.rel = get_m4(r); }
  return E;
}
void put_result(Writer& w, const lp::OptResult& o) {
  w.put(o.error); w.put(o.residual); w.put(o.inlier_residual);
  w.put(o.inlier); w.put(o.outlier); w.put(o.valid); w.put(o.invalid); w.put(o.outlier_ratio);
  put_m4(w, o.pose);
}
lp::OptResult get_result(Reader& r) {
  lp::OptResult o;
  o.error = r.get<double>(); o.residual = r.get<double>(); o.inlier_residual = r.get<double>();
  o.inlier = r.get<uint32_t>(); o.outlier = r.get<uint32_t>(); o.valid = r.get<uint32_t>(); o.invalid = r.get<uint32_t>();
  o.outlier_ratio = r.get<float>();
  o.pose = get_m4(r);
  return o;
}

void write_header(Writer& w, const StateImage& s, uint64_t total) {
  w.bytes(kStateMagic, 8);
  w.put(kStateFormat); w.put((uint32_t)SB_VERSION); w.put((uint32_t)sizeof(sb_surfel)); w.put(kMaxPoses);
  w.put(s.p.data_width); w.put(s.p.data_height); w.put(s.p.model_width); w.put(s.p.model_height);
  w.put(total);
#define X(f) w.put(s.p.f);
  SB_PARAM_FIELDS(X)
#undef X
#define X(f) w.put(s.loop.p.f);
  SB_LOOP_PARAM_FIELDS(X)
#undef X
  w.align8();
}

void write_host_sections(Writer& w, const StateImage& s) {
  size_t o = w.open(S_HOST);
  w.put(s.timestamp);
  for (const double* m : {s.currentPose, s.lastPose, s.currentPose_old, s.currentPose_new, s.lastIncrement, s.lastPose_old})
    w.bytes(m, 128);
  w.put(s.confidence_threshold); w.put(s.log_unstable_slam);
  w.bytes(s.stats, sizeof(s.stats));
  w.put(s.trackLoss); w.put(s.cur_has_semantics); w.put(s.last_has_semantics); w.put(s.close_loops);
  w.put(s.n_live); w.put(s.map_timestamp); w.put(s.pose_ref_end); w.put(s.n_updated); w.put(s.n_new);
  w.put(s.origin_i); w.put(s.origin_j);
  w.put((uint32_t)s.extraction.size());
  for (const auto& e : s.extraction) { w.put(e.first); w.put(e.second); }
  w.put((uint32_t)s.tiles.size());
  for (const auto& t : s.tiles) {
    w.put(t.first.first); w.put(t.first.second);
    w.put(t.second.slot); w.put((uint32_t)t.second.known); w.put(t.second.base); w.put(t.second.count);
  }
  w.put(s.n_slots); w.put(s.tiles_pending); w.put(s.pool_end);
  w.close(o);

  o = w.open(S_LOOP);
  const lp::State& L = s.loop;
  w.put((uint32_t)L.graph.poses.size());
  for (const lp::M4& m : L.graph.poses) put_m4(w, m);
  put_edges(w, L.graph.edges);
  w.put((uint32_t)L.trajectory_distances.size());
  w.bytes(L.trajectory_distances.data(), L.trajectory_distances.size() * sizeof(float));
  put_result(w, L.result_new);
  put_result(w, L.result_old);
  put_edges(w, L.unverified);
  put_edges(w, L.verified);
  w.put((uint32_t)L.already_verified); w.put(L.time_without_loop_closure); w.put(L.loop_count);
  w.put((uint32_t)L.found_candidate); w.put((uint32_t)L.use_candidate); w.put((uint32_t)L.optimisation_requested);
  w.put(L.last_added_candidate); w.put(L.candidates_tested); w.put(L.loop_edges_added);
  w.put(L.stat_valid_ratio); w.put(L.stat_outlier_ratio); w.put(L.stat_rel_error);
  w.put(L.before_id); w.put(L.before_loop_count); put_m4(w, L.before_pose); w.put((uint64_t)L.requested_size);
  w.close(o);

  o = w.open(S_POSES);
  w.put((uint32_t)(s.poses.size() / 16));
  w.bytes(s.poses.data(), s.poses.size() * 4);
  w.bytes(s.poses_inv.data(), s.poses_inv.size() * 4);
  w.close(o);

  o = w.open(S_RESULT);
  w.bytes(&s.result, sizeof(ResultBlock));
  w.close(o);

  o = w.open(S_TILES);
  w.put((uint32_t)s.tile_rec.size());
  for (const uint2& r : s.tile_rec) { w.put(r.x); w.put(r.y); }
  w.close(o);
}

// Opens section `id` and returns its payload length (0 and r.ok = false when the next section is another one).
uint64_t read_open(Reader& r, uint32_t id) {
  const uint32_t got = r.get<uint32_t>();
  r.get<uint32_t>();
  const uint64_t len = r.get<uint64_t>();
  if (!r.ok || got != id || len > r.n - r.off || (len & 7)) r.ok = false;
  return r.ok ? len : 0;
}
bool read_close(Reader& r, size_t start, uint64_t len) {
  r.align8();
  return r.ok && r.off - start == len;
}

// Parses the header and the host sections; nullptr when they are well formed, otherwise the reason.
const char* read_host(Reader& r, const sb_ctx* c, StateImage& s) {
  char magic[8];
  r.bytes(magic, 8);
  if (!r.ok || memcmp(magic, kStateMagic, 8) != 0) return "not a checkpoint (bad magic)";
  const uint32_t fmt = r.get<uint32_t>(), ver = r.get<uint32_t>(), ssz = r.get<uint32_t>(), mp = r.get<uint32_t>();
  if (!r.ok) return "truncated header";
  if (fmt != kStateFormat) return "unsupported checkpoint format version";
  if (ver != SB_VERSION) return "checkpoint written by another library version (SB_VERSION)";
  if (ssz != sizeof(sb_surfel) || mp != kMaxPoses) return "checkpoint written with another surfel size / pose capacity";
  int32_t dims[4];
  for (int32_t& d : dims) d = r.get<int32_t>();
  const uint64_t total = r.get<uint64_t>();
  if (!r.ok) return "truncated header";
  if (dims[0] != c->p.data_width || dims[1] != c->p.data_height || dims[2] != c->p.model_width ||
      dims[3] != c->p.model_height)
    return "checkpoint image geometry differs from the context's";
  if (total != r.n) return total > r.n ? "truncated checkpoint" : "checkpoint size does not match its header";
  memset(&s.p, 0, sizeof(s.p));
#define X(f) s.p.f = r.get<decltype(s.p.f)>();
  SB_PARAM_FIELDS(X)
#undef X
#define X(f) s.loop.p.f = r.get<decltype(s.loop.p.f)>();
  SB_LOOP_PARAM_FIELDS(X)
#undef X
  r.align8();
  if (!r.ok) return "truncated header";
  if (check_params(&s.p)) return "checkpoint parameters are not valid";
  if (s.p.data_width != dims[0] || s.p.data_height != dims[1] || s.p.model_width != dims[2] || s.p.model_height != dims[3])
    return "checkpoint parameters disagree with its image geometry";

  uint64_t len = read_open(r, S_HOST);
  size_t start = r.off;
  s.timestamp = r.get<uint32_t>();
  for (double* m : {s.currentPose, s.lastPose, s.currentPose_old, s.currentPose_new, s.lastIncrement, s.lastPose_old})
    r.bytes(m, 128);
  s.confidence_threshold = r.get<float>(); s.log_unstable_slam = r.get<float>();
  r.bytes(s.stats, sizeof(s.stats));
  s.trackLoss = r.get<uint32_t>(); s.cur_has_semantics = r.get<uint32_t>(); s.last_has_semantics = r.get<uint32_t>();
  s.close_loops = r.get<uint32_t>();
  s.n_live = r.get<uint32_t>(); s.map_timestamp = r.get<uint32_t>(); s.pose_ref_end = r.get<uint32_t>();
  s.n_updated = r.get<uint32_t>(); s.n_new = r.get<uint32_t>();
  s.origin_i = r.get<int32_t>(); s.origin_j = r.get<int32_t>();
  s.extraction.resize(r.count(8));
  for (auto& e : s.extraction) { e.first = r.get<int32_t>(); e.second = r.get<int32_t>(); }
  s.tiles.resize(r.count(24));
  for (auto& t : s.tiles) {
    t.first.first = r.get<int32_t>(); t.first.second = r.get<int32_t>();
    t.second.slot = r.get<uint32_t>(); t.second.known = r.get<uint32_t>() != 0;
    t.second.base = r.get<uint32_t>(); t.second.count = r.get<uint32_t>();
  }
  s.n_slots = r.get<uint32_t>(); s.tiles_pending = r.get<uint32_t>(); s.pool_end = r.get<uint32_t>();
  if (!read_close(r, start, len)) return "malformed state section";
  // A digest is no signature: every field that later sizes a copy or indexes device memory is range-checked here.
  if (s.n_live > kMaxSurfels || s.n_slots > kMaxTileSlots || s.pool_end > kTilePoolCap ||
      s.extraction.size() > kMaxTileSlots || s.tiles.size() > kMaxTileSlots)
    return "checkpoint exceeds the map / tile-pool capacity";
  if (s.pose_ref_end > kMaxPoses) return "malformed map state (pose-table reference beyond the table)";
  for (const auto& t : s.tiles)
    if (t.second.slot >= s.n_slots) return "malformed tile table";

  len = read_open(r, S_LOOP);
  start = r.off;
  lp::State& L = s.loop;
  L.graph.poses.resize(r.count(128));
  for (lp::M4& m : L.graph.poses) m = get_m4(r);
  L.graph.edges = get_edges(r);
  L.trajectory_distances.resize(r.count(4));
  r.bytes(L.trajectory_distances.data(), L.trajectory_distances.size() * 4);
  L.result_new = get_result(r);
  L.result_old = get_result(r);
  L.unverified = get_edges(r);
  L.verified = get_edges(r);
  L.already_verified = r.get<uint32_t>() != 0;
  L.time_without_loop_closure = r.get<uint32_t>(); L.loop_count = r.get<uint32_t>();
  L.found_candidate = r.get<uint32_t>() != 0; L.use_candidate = r.get<uint32_t>() != 0;
  L.optimisation_requested = r.get<uint32_t>() != 0;
  L.last_added_candidate = r.get<int32_t>(); L.candidates_tested = r.get<uint32_t>(); L.loop_edges_added = r.get<uint32_t>();
  L.stat_valid_ratio = r.get<float>(); L.stat_outlier_ratio = r.get<float>(); L.stat_rel_error = r.get<float>();
  L.before_id = r.get<int32_t>(); L.before_loop_count = r.get<uint32_t>(); L.before_pose = get_m4(r);
  L.requested_size = (size_t)r.get<uint64_t>();
  if (!read_close(r, start, len)) return "malformed loop-closure section";
  if (L.graph.poses.empty() || L.trajectory_distances.empty() || L.requested_size > L.graph.poses.size() ||
      (L.optimisation_requested && (L.before_id < 0 || (size_t)L.before_id >= L.graph.poses.size())))
    return "malformed loop-closure section";
  // the next scan's check reads graph pose and travelled distance timestamp - 1 (SurfelMapping.cpp:460-469)
  if (s.close_loops && s.timestamp > 0 &&
      (L.graph.poses.size() < s.timestamp || L.trajectory_distances.size() < s.timestamp))
    return "malformed loop-closure section (graph shorter than the sequence)";
  for (const std::vector<lp::Edge>* E : {&L.graph.edges, &L.unverified, &L.verified})
    for (const lp::Edge& e : *E)
      if (e.from < 0 || e.to < 0 || (size_t)e.from >= L.graph.poses.size() || (size_t)e.to >= L.graph.poses.size())
        return "malformed loop-closure section (edge outside the graph)";

  len = read_open(r, S_POSES);
  start = r.off;
  const uint32_t np = r.count(128);
  if (np > kMaxPoses) return "malformed pose tables";
  s.poses.resize((size_t)np * 16);
  s.poses_inv.resize((size_t)np * 16);
  r.bytes(s.poses.data(), s.poses.size() * 4);
  r.bytes(s.poses_inv.data(), s.poses_inv.size() * 4);
  if (!read_close(r, start, len)) return "malformed pose tables";

  len = read_open(r, S_RESULT);
  start = r.off;
  r.bytes(&s.result, sizeof(ResultBlock));
  if (!read_close(r, start, len)) return "malformed result block";
  if (s.result.counts[0] != s.n_live || s.result.counts[5] != 0) return "malformed result block (surfel counts)";

  len = read_open(r, S_TILES);
  start = r.off;
  s.tile_rec.resize(r.count(8));
  for (uint2& t : s.tile_rec) { t.x = r.get<uint32_t>(); t.y = r.get<uint32_t>(); }
  if (!read_close(r, start, len) || s.tile_rec.size() != s.n_slots) return "malformed tile records";
  if ((s.n_slots ? s.tile_rec[s.n_slots - 1].x : 0u) != s.pool_end) return "malformed tile records";
  // slot k holds [end of slot k - 1, rec[k].x), no more than the tile had surfels (or the extract cap allows)
  for (uint32_t k = 0; k < s.n_slots; ++k) {
    const uint32_t base = k ? s.tile_rec[k - 1].x : 0u;
    if (s.tile_rec[k].x < base || s.tile_rec[k].x - base > std::min(s.tile_rec[k].y, kExtractCap))
      return "malformed tile records";
  }
  for (const auto& t : s.tiles) {  // a tile already read back names exactly its slot's range
    const uint32_t base = t.second.slot ? s.tile_rec[t.second.slot - 1].x : 0u;
    if (t.second.known && (t.second.base != base || t.second.count != s.tile_rec[t.second.slot].x - base))
      return "malformed tile table";
  }
  return nullptr;
}

// The device-resident bulk of a checkpoint: (section id, device ranges in blob order)
struct DevRange {
  void* p;
  uint64_t bytes;
};
struct DevSection {
  uint32_t id;
  std::vector<DevRange> ranges;
  uint64_t bytes() const {
    uint64_t n = 0;
    for (const DevRange& r : ranges) n += r.bytes;
    return n;
  }
};
const sb_frame* const* frame_roles(const sb_ctx* c, const sb_frame* out[7]) {
  const sb_frame* f[7] = {c->cur, c->last, c->cur_model, c->last_model, c->f_old, c->f_new, c->f_comp};
  for (int i = 0; i < 7; ++i) out[i] = f[i];
  return out;
}
// surfels go through the (idle) scratch lanes T as one flat block; pool lanes and frames are copied where they are
std::vector<DevSection> dev_sections(sb_ctx* c, uint32_t n_live, uint32_t pool_end) {
  std::vector<DevSection> d(3);
  d[0].id = S_SURFELS;
  d[0].ranges.push_back(DevRange{c->T.p0, (uint64_t)n_live * 64});
  d[1].id = S_POOL;
  for (float4* lane : {c->pool.p0, c->pool.p1, c->pool.p2, c->pool.p3})
    d[1].ranges.push_back(DevRange{lane, (uint64_t)pool_end * 16});
  d[2].id = S_FRAMES;
  const sb_frame* f[7];
  frame_roles(c, f);
  for (const sb_frame* fr : f) d[2].ranges.push_back(DevRange{fr->base.get(), (uint64_t)fr->d.W * fr->d.H * 48});
  return d;
}

uint64_t host_digest(const uint8_t* b, uint64_t off, uint64_t len) {  // off, len: multiples of 8
  uint64_t h = 0;
  for (uint64_t i = 0; i < len; i += 8) {
    uint64_t w;
    memcpy(&w, b + off + i, 8);
    h += state_word_hash((off + i) / 8, w);
  }
  return h;
}

int state_staging(sb_ctx* c) {
  if (c->state_stage) return SB_OK;
  void* h = nullptr;
  SB_CUDA(c, cudaMallocHost(&h, 2 * kStageBytes));
  c->state_stage.reset(static_cast<uint8_t*>(h));
  for (cudaEvent_t& e : c->state_ev) SB_CUDA(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  SB_CUDA(c, dev_alloc(c->state_acc, sizeof(unsigned long long)));
  return SB_OK;
}

// Device ranges -> host bytes, in chunks through the pinned double buffer: the copy of chunk i from the pinned buffer
// to `dst` runs while chunk i + 1 crosses the bus.
int copy_out(sb_ctx* c, const std::vector<DevRange>& ranges, uint8_t* dst) {
  uint8_t* stage[2] = {c->state_stage.get(), c->state_stage.get() + kStageBytes};
  uint8_t* prev_dst = nullptr;
  size_t prev_n = 0;
  int buf = 0;
  for (const DevRange& r : ranges)
    for (uint64_t o = 0; o < r.bytes; o += kStageBytes) {
      const size_t n = (size_t)std::min<uint64_t>(kStageBytes, r.bytes - o);
      SB_CUDA(c, cudaMemcpyAsync(stage[buf], static_cast<uint8_t*>(r.p) + o, n, cudaMemcpyDeviceToHost, c->stream));
      SB_CUDA(c, cudaEventRecord(c->state_ev[buf], c->stream));
      if (prev_dst) {
        SB_CUDA(c, cudaEventSynchronize(c->state_ev[buf ^ 1]));
        memcpy(prev_dst, stage[buf ^ 1], prev_n);
      }
      prev_dst = dst;
      prev_n = n;
      dst += n;
      buf ^= 1;
    }
  if (prev_dst) {
    SB_CUDA(c, cudaEventSynchronize(c->state_ev[buf ^ 1]));
    memcpy(prev_dst, stage[buf ^ 1], prev_n);
  }
  return SB_OK;
}

// host bytes -> device ranges: the host fills one half while the other half crosses the bus
int copy_in(sb_ctx* c, const std::vector<DevRange>& ranges, const uint8_t* src) {
  uint8_t* stage[2] = {c->state_stage.get(), c->state_stage.get() + kStageBytes};
  bool used[2] = {false, false};
  int buf = 0;
  for (const DevRange& r : ranges)
    for (uint64_t o = 0; o < r.bytes; o += kStageBytes) {
      const size_t n = (size_t)std::min<uint64_t>(kStageBytes, r.bytes - o);
      if (used[buf]) SB_CUDA(c, cudaEventSynchronize(c->state_ev[buf]));
      memcpy(stage[buf], src, n);
      SB_CUDA(c, cudaMemcpyAsync(static_cast<uint8_t*>(r.p) + o, stage[buf], n, cudaMemcpyHostToDevice, c->stream));
      SB_CUDA(c, cudaEventRecord(c->state_ev[buf], c->stream));
      used[buf] = true;
      src += n;
      buf ^= 1;
    }
  // the next call starts filling the pinned halves again: both must have crossed the bus
  for (int b = 0; b < 2; ++b)
    if (used[b]) SB_CUDA(c, cudaEventSynchronize(c->state_ev[b]));
  return SB_OK;
}

// digest of the pool lanes and the frames (the surfels' is computed by the pack / unpack kernel), at their blob offsets
void digest_ranges(sb_ctx* c, const DevSection& s, uint64_t data_off) {
  for (const DevRange& r : s.ranges) {
    launch_state_digest(L_(c), r.p, r.bytes / 8, data_off / 8, c->state_acc);
    data_off += r.bytes;
  }
}

// Scans staged by sb_prefetch_scan are dropped: a checkpoint neither carries nor consumes them.
int discard_prefetch(sb_ctx* c) {
  if (!c->copy_stream) return SB_OK;
  SB_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  for (auto& sl : c->prefetch) sl.valid = sl.in_use = sl.has_released = false;
  return SB_OK;
}

// The state of a context between calls, as a checkpoint holds it (reads the small device blocks back).
int capture(sb_ctx* c, StateImage& s) {
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  s.p = c->p;
  s.timestamp = c->timestamp;
  s.trackLoss = c->trackLoss;
  memcpy(s.currentPose, c->currentPose, 128); memcpy(s.lastPose, c->lastPose, 128);
  memcpy(s.currentPose_old, c->currentPose_old, 128); memcpy(s.currentPose_new, c->currentPose_new, 128);
  memcpy(s.lastIncrement, c->lastIncrement, 128); memcpy(s.lastPose_old, c->lastPose_old, 128);
  s.confidence_threshold = c->confidence_threshold;
  s.log_unstable_slam = c->log_unstable_slam;
  memcpy(s.stats, c->stats, sizeof(s.stats));
  s.cur_has_semantics = c->cur_has_semantics; s.last_has_semantics = c->last_has_semantics;
  s.close_loops = c->close_loops;
  s.n_live = n_live(c);
  s.map_timestamp = c->map_timestamp; s.pose_ref_end = c->pose_ref_end;
  s.n_updated = c->n_updated; s.n_new = c->n_new;
  s.origin_i = c->origin_i; s.origin_j = c->origin_j;
  s.extraction = c->extraction;
  s.tiles.assign(c->tiles.begin(), c->tiles.end());
  s.n_slots = c->n_slots;
  s.tiles_pending = c->tiles_pending;
  s.tile_rec.resize(c->n_slots);
  if (c->n_slots)
    SB_CUDA(c, cudaMemcpy(s.tile_rec.data(), c->d_tile_rec, (size_t)c->n_slots * sizeof(uint2), cudaMemcpyDeviceToHost));
  s.pool_end = c->n_slots ? s.tile_rec[c->n_slots - 1].x : 0u;
  // the used entries of the pose tables: those the map can refer to, and any set beyond them through sb_map_set_pose
  uint32_t np = pose_table_count(c);
  for (uint32_t t = kMaxPoses; t > np; --t) {
    const float* e = &c->h_poses[16 * (size_t)(t - 1)];
    bool ident = true;
    for (int i = 0; i < 16; ++i) ident = ident && e[i] == ((i % 5 == 0) ? 1.0f : 0.0f);
    if (!ident) { np = t; break; }
  }
  s.poses.resize((size_t)np * 16);
  s.poses_inv.resize((size_t)np * 16);
  SB_CUDA(c, cudaMemcpy(s.poses.data(), c->poses, (size_t)np * 64, cudaMemcpyDeviceToHost));
  SB_CUDA(c, cudaMemcpy(s.poses_inv.data(), c->poses_inv, (size_t)np * 64, cudaMemcpyDeviceToHost));
  SB_CUDA(c, cudaMemcpy(&s.result, c->res, sizeof(ResultBlock), cudaMemcpyDeviceToHost));
  s.result.counts[0] = s.n_live;  // the map is restored dense: its physical end is the live count, no dead slots
  s.result.counts[5] = 0;
  s.loop = c->loop;
  return SB_OK;
}

// Commits a verified checkpoint (the bulk sections are already on the device).
int apply(sb_ctx* c, const StateImage& s) {
  c->p = s.p;
  derive(c);
  c->confidence_threshold = s.confidence_threshold;
  c->log_unstable_slam = s.log_unstable_slam;
  c->timestamp = s.timestamp;
  c->trackLoss = s.trackLoss;
  memcpy(c->currentPose, s.currentPose, 128); memcpy(c->lastPose, s.lastPose, 128);
  memcpy(c->currentPose_old, s.currentPose_old, 128); memcpy(c->currentPose_new, s.currentPose_new, 128);
  memcpy(c->lastIncrement, s.lastIncrement, 128); memcpy(c->lastPose_old, s.lastPose_old, 128);
  memcpy(c->stats, s.stats, sizeof(c->stats));
  c->cur_has_semantics = s.cur_has_semantics != 0; c->last_has_semantics = s.last_has_semantics != 0;
  c->close_loops = s.close_loops != 0;
  c->loop = s.loop;
  c->n_host = s.n_live; c->n_holes = 0; c->lazy_update = false; c->n_upper = s.n_live;
  c->prepped_for_update = false;
  c->map_timestamp = s.map_timestamp; c->pose_ref_end = s.pose_ref_end;
  c->n_updated = s.n_updated; c->n_new = s.n_new;
  c->origin_i = s.origin_i; c->origin_j = s.origin_j;
  c->extraction = s.extraction;
  c->tiles.clear();
  for (const auto& t : s.tiles) c->tiles[t.first] = t.second;
  c->n_slots = s.n_slots;
  c->tiles_pending = s.tiles_pending != 0;
  c->h_poses.assign((size_t)kMaxPoses * 16, 0.0f);
  for (uint32_t t = 0; t < kMaxPoses; ++t)
    for (int i = 0; i < 4; ++i) c->h_poses[16 * (size_t)t + 5 * i] = 1.0f;
  c->h_poses_inv = c->h_poses;
  memcpy(c->h_poses.data(), s.poses.data(), s.poses.size() * 4);
  memcpy(c->h_poses_inv.data(), s.poses_inv.data(), s.poses_inv.size() * 4);
  SB_CUDA(c, cudaMemcpyAsync(c->poses, c->h_poses.data(), (size_t)kMaxPoses * 64, cudaMemcpyHostToDevice, c->stream));
  SB_CUDA(c, cudaMemcpyAsync(c->poses_inv, c->h_poses_inv.data(), (size_t)kMaxPoses * 64, cudaMemcpyHostToDevice,
                             c->stream));
  c->host->result = s.result;
  SB_CUDA(c, cudaMemcpyAsync(c->res, &c->host->result, sizeof(ResultBlock), cudaMemcpyHostToDevice, c->stream));
  if (s.n_slots)
    SB_CUDA(c, cudaMemcpyAsync(c->d_tile_rec, s.tile_rec.data(), (size_t)s.n_slots * sizeof(uint2), cudaMemcpyHostToDevice,
                               c->stream));
  // scratch that a scan expects as the previous one left it: key images cleared by the pass that consumed them, group
  // totals zero (a context that stopped mid-scan may not hold these; a loaded one does)
  const size_t Pm = (size_t)c->kp.Wm * c->kp.Hm, Pk = preprocess_key_elems(c->kp.W, c->kp.H);
  SB_CUDA(c, cudaMemsetAsync(c->key_old, 0xff, Pm * 8 * 3, c->stream));
  for (int i = 0; i < 2; ++i) SB_CUDA(c, cudaMemsetAsync(c->prep.img[i], 0xff, Pk * 8, c->stream));
  SB_CUDA(c, cudaMemsetAsync(c->group_counts, 0, kGroupCounts * 4, c->stream));
  c->memo.clear();
  c->map_version += 1;
  SB_CUDA(c, cudaStreamSynchronize(c->stream));  // the copies read host vectors of `s` and members of the context
  return SB_OK;
}

// Serialises everything but the bulk data; returns the offsets of the three bulk payloads and the total size.
void layout(sb_ctx* c, const StateImage& s, Writer& head, std::vector<DevSection>& dev, uint64_t data_off[3],
            uint64_t* total) {
  Writer w;
  write_host_sections(w, s);
  dev = dev_sections(c, s.n_live, s.pool_end);
  Writer hdr;
  write_header(hdr, s, 0);
  uint64_t off = hdr.b.size() + w.b.size();
  for (int i = 0; i < 3; ++i) {
    data_off[i] = off + 16;
    off += 16 + dev[i].bytes();
  }
  *total = off + 8;
  head.b.clear();
  write_header(head, s, *total);
  head.bytes(w.b.data(), w.b.size());
}

int state_check(sb_ctx* c) {
  if (c->comm_on || c->comm_cb)
    return fail(c, SB_ERR_STATE, "checkpoints are not available while a multi-GPU exchange is set up");
  return SB_OK;
}

}  // namespace

extern "C" {

int sb_state_size(sb_ctx* c, uint64_t* bytes) {
  if (!c || !bytes) return fail(c, SB_ERR_INVALID, "state_size: null argument");
  int r;
  if ((r = state_check(c))) return r;
  cudaSetDevice(c->device);
  StateImage s;
  if ((r = capture(c, s))) return r;
  Writer head;
  std::vector<DevSection> dev;
  uint64_t off[3];
  layout(c, s, head, dev, off, bytes);
  return SB_OK;
}

int sb_state_save(sb_ctx* c, void* dst, uint64_t cap, uint64_t* written) {
  if (!c || !dst) return fail(c, SB_ERR_INVALID, "state_save: null argument");
  int r;
  if ((r = state_check(c))) return r;
  cudaSetDevice(c->device);
  StateImage s;
  if ((r = capture(c, s))) return r;
  Writer head;
  std::vector<DevSection> dev;
  uint64_t off[3], total = 0;
  layout(c, s, head, dev, off, &total);
  if (written) *written = total;
  if (cap < total) return fail(c, SB_ERR_INVALID, "state_save: buffer smaller than sb_state_size");
  if ((r = discard_prefetch(c))) return r;
  if ((r = state_staging(c))) return r;
  uint8_t* out = static_cast<uint8_t*>(dst);
  memcpy(out, head.b.data(), head.b.size());
  uint64_t digest = host_digest(out, 0, head.b.size());
  for (int i = 0; i < 3; ++i) {  // section headers of the bulk data
    const uint32_t id = dev[i].id, zero = 0;
    const uint64_t len = dev[i].bytes();
    memcpy(out + off[i] - 16, &id, 4); memcpy(out + off[i] - 12, &zero, 4); memcpy(out + off[i] - 8, &len, 8);
    digest += host_digest(out, off[i] - 16, 16);
  }
  SB_CUDA(c, cudaMemsetAsync(c->state_acc, 0, 8, c->stream));
  c->lb_gen = (c->lb_gen + 1) & 0x3fffffffu;
  if (c->lb_gen == 0) c->lb_gen = 1;
  launch_state_pack(L_(c), c->A, c->live, c->n_host, c->T.p0, s.n_live, c->lb_desc, c->lb_ticket, c->lb_gen, off[0] / 8,
                    c->state_acc);
  digest_ranges(c, dev[1], off[1]);
  digest_ranges(c, dev[2], off[2]);
  SB_CUDA(c, cudaGetLastError());
  for (int i = 0; i < 3; ++i)
    if ((r = copy_out(c, dev[i].ranges, out + off[i]))) return r;
  unsigned long long dd = 0;
  SB_CUDA(c, cudaMemcpyAsync(&c->host->sums[0], c->state_acc, 8, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  memcpy(&dd, &c->host->sums[0], 8);
  digest += dd;
  memcpy(out + total - 8, &digest, 8);
  return SB_OK;
}

int sb_state_load(sb_ctx* c, const void* src, uint64_t n) {
  if (!c || (!src && n)) return fail(c, SB_ERR_INVALID, "state_load: null argument");
  int r;
  if ((r = state_check(c))) return r;
  StateImage s;
  Reader rd{static_cast<const uint8_t*>(src), (size_t)n};
  if (const char* why = read_host(rd, c, s)) return fail(c, SB_ERR_INVALID, std::string("state_load: ") + why);
  cudaSetDevice(c->device);
  std::vector<DevSection> dev = dev_sections(c, s.n_live, s.pool_end);
  uint64_t off[3];
  for (int i = 0; i < 3; ++i) {
    const uint64_t len = read_open(rd, dev[i].id);
    off[i] = rd.off;
    if (!rd.ok || len != dev[i].bytes()) return fail(c, SB_ERR_INVALID, "state_load: malformed bulk section");
    rd.off += len;
  }
  if (rd.n - rd.off != 8) return fail(c, SB_ERR_INVALID, "state_load: checkpoint size does not match its sections");
  // ---- the header is sound: from here on the context changes ----
  if ((r = discard_prefetch(c))) return r;
  if ((r = state_staging(c))) return r;
  const uint8_t* in = static_cast<const uint8_t*>(src);
  uint64_t digest = host_digest(in, 0, off[0]);
  for (int i = 1; i < 3; ++i) digest += host_digest(in, off[i] - 16, 16);
  SB_CUDA(c, cudaMemsetAsync(c->state_acc, 0, 8, c->stream));
  for (int i = 0; i < 3; ++i)
    if ((r = copy_in(c, dev[i].ranges, in + off[i]))) return r;
  launch_state_unpack(L_(c), c->T.p0, s.n_live, c->A, c->live, off[0] / 8, c->state_acc);
  digest_ranges(c, dev[1], off[1]);
  digest_ranges(c, dev[2], off[2]);
  SB_CUDA(c, cudaGetLastError());
  SB_CUDA(c, cudaMemcpyAsync(&c->host->sums[0], c->state_acc, 8, cudaMemcpyDeviceToHost, c->stream));
  SB_CUDA(c, cudaStreamSynchronize(c->stream));
  unsigned long long dd = 0;
  memcpy(&dd, &c->host->sums[0], 8);
  digest += dd;
  uint64_t stored;
  memcpy(&stored, in + n - 8, 8);
  if (digest != stored) {
    // bulk sections are already overwritten: never leave a half-loaded context behind
    if ((r = reset_state(c))) return r;
    return fail(c, SB_ERR_INVALID, "state_load: checkpoint digest mismatch (corrupted data); the context was reset");
  }
  return apply(c, s);
}

}  // extern "C"
