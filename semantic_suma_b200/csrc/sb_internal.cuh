// sb_internal.cuh -- internal declarations shared by the kernels and the C-ABI layer of libsuma_b200.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cstddef>
#include <memory>
#include <vector>

#include "../../include/suma_b200.h"
#include "sb_math.cuh"

namespace sb {

constexpr uint32_t kMaxSurfels = 2048u * 2048u;  // SurfelMap.h:87
// The pose table starts at the reference's fixed size (SurfelMap.h:205) and doubles on demand up to 2^24 entries: a
// surfel keeps its entry in the float `count` field, which holds integers exactly only up to 2^24 (DESIGN.md section 12).
constexpr uint32_t kPoseCapInit = 10000u;
constexpr uint32_t kPoseCapMax = 1u << 24;
constexpr uint32_t kExtractCap = 500000u;        // SurfelMap.cpp:279
constexpr uint32_t kComposeAge = 100u;           // SurfelMap.h:144
constexpr int kMaxGnIter = 256;
constexpr uint32_t kTilePoolCap = 16u * 1024u * 1024u;  // surfels held by the HBM tile cache (1 GiB)
constexpr uint32_t kMaxTileSlots = 16384u;
constexpr int kGroupCounts = 256;  // group totals of a surfel-indexed compaction: kMaxSurfels / 256 threads / 64 blocks per group

// everything the kernels need from sb_params plus the derived constants the reference computes on the host
struct KParams {
  int W, H, Wm, Hm;
  float fov_up, fov, min_depth, max_depth;          // data image (abs values, Preprocessing.cpp:94-95)
  float m_fov_up, m_fov, m_min_depth, m_max_depth;  // model image (SurfelMap.cpp:440-443)
  int weighting, bilinear;
  float factor;
  int use_stability, unstable_age, confidence_mode, active_timestamps;
  int weighting_scheme, averaging_scheme, update_always;
  float confidence_threshold, p_stable, p_unstable, log_prior, log_unstable;
  float sigma_angle, sigma_distance, max_weight;
  float pixel_size, min_radius, max_radius, radconf_angle_thresh, update_angle_thresh, map_max_distance;
  float max_loop_closure_distance;
  int label_offset_quirk;
  uint32_t pose_cap;  // entries of the pose tables (pose_index() clamps to it: malformed input only)
};

// Frame.h:21-79: three RGBA32F images; one allocation, SoA of images
struct FrameDev {
  int W, H;
  float4* vertex;
  float4* normal;
  float4* semantic;
};

// Surfel store: structure of arrays of 16-byte lanes so that every pass streams exactly the lanes it needs with
// fully coalesced 128-bit accesses (the reference keeps 64-byte AoS records, Surfel.h:5-15):
//   p0 = (x, y, z, radius)   p1 = (nx, ny, nz, confidence)
//   p2 = (timestamp:u32, color, weight, count)   p3 = (r, g, b, w)  semantic label/255 x3 + probability
struct SurfelPlanes {
  float4* p0;
  float4* p1;
  float4* p2;
  float4* p3;
};

// ---- device state of one fused Gauss-Newton run (LieGaussNewton.cpp:13-79) ----
// GnHead is the part the host reads back after a run (and writes when it drives the loop itself)
struct GnHead {
  double pose[16];       // Tk_
  double last_error;     // last_error
  double out48[48];      // sums of the last evaluated iteration
  int k;                 // k_
  int done;              // loop left (converged or max iterations)
  int history_len;
  int error;             // a bounded spin of the persistent kernel timed out (missing block / peer GPU)
};
struct GnState : GnHead {
  double history[(kMaxGnIter + 1) * 16];
};

struct IcpArgs {
  const float4* data_v; const float4* data_n; const float4* data_s;
  const float4* model_v; const float4* model_n; const float4* model_s;
  float distance_thresh, angle_thresh;  // Frame2Model.cpp:66-67
  int row_begin, row_end;
  int Wm, Hm;    // size of the model images = textureSize(vertex_model) (Frame2Model_jacobians.geom:70): the rendered
                 // model frame, or the last data frame in the frame-to-frame fallback (SurfelMapping.cpp:442)
  // (this order leaves k_gn_persistent<2> with 24 bytes of spill loads; with has_semantics ahead of Wm it takes 68)
  int has_semantics;
};

// peer mailboxes for the multi-GPU one-shot all-reduce (fused into the Jacobian kernel's last block)
struct CommDev {
  int rank, nranks;
  long long* mailbox[8];  // mailbox[r]: rank r's mailbox (peer-mapped): [epoch parity 2][source rank 8][40] int64
  unsigned int* epoch;    // local all-reduce counter (identical on every rank by construction)
};

struct Mat4 {
  float m[16];
};
struct Mat4d {
  double m[16];
};

// Device-resident pose bookkeeping of SurfelMapping::updatePose (SurfelMapping.cpp:372-476): the per-scan pipeline is
// enqueued without a host round trip; the host reads this block back once, at the end of the scan.
struct PoseDev {
  double currentPose[16], lastPose[16], lastIncrement[16], increment[16], T0[16];
  Mat4 P_active, invP_active;  // currentPose_new * increment (render_active), and its inverse
  Mat4 P_cur, invP_cur;        // the scan's final pose (float) and inverse: map update + model rendering
  int fallback;                // track loss detected: the frame-to-frame minimisation runs
  int trackLoss;               // counter
  int icp_iterations;          // k_ of the frame-to-model minimisation
  int gn_error;                // the persistent Gauss-Newton kernel gave up (timeout): the scan's pose is invalid
  float t_err, r_err;
  int pad2[2];
};

// The per-scan results in one device block, so that the end of a scan is a single device-to-host copy into its pinned
// mirror. The offsets are those of the original hand-laid block; the copy moves all 8256 bytes.
struct ResultBlock {
  PoseDev pose;                       // device-resident pose bookkeeping of the pipeline
  char pad0[4096 - sizeof(PoseDev)];
  long long sums[64];                 // raw sums of a Jacobian pass (the first 32; the scan's statistics pass)
  char pad1[8192 - 4096 - 64 * sizeof(long long)];
  // [0] physical end of the surfel slots, [1] physical end after the update (base for new), [2] kept updated,
  // [3] kept new, [4] extracted, [5] dead slots below [1] after an in-place update, [6] / [7] end of the written range /
  // number kept of a compaction of the map (not read back), [8] smallest pose-table entry the extraction passes saw,
  // [9] / [10] surfels the update / the generation pass emit before the submap window (the reference's transform-feedback
  // counts, sb_map_update_debug)
  uint32_t counts[16];
};
static_assert(offsetof(ResultBlock, sums) == 4096, "result block layout");
static_assert(offsetof(ResultBlock, counts) == 8192, "result block layout");
static_assert(sizeof(ResultBlock) == 8256, "result block layout");

// Owning handle of one allocation. It converts to the plain pointer that launchers and sub-views take.
template <class T, class Free>
struct Owned : std::unique_ptr<T, Free> {
  using std::unique_ptr<T, Free>::unique_ptr;
  operator T*() const { return this->get(); }
};
struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <class T>
using DevPtr = Owned<T, CudaFree>;
template <class T>
using PinnedPtr = Owned<T, CudaFreeHost>;
template <class T>
cudaError_t dev_alloc(DevPtr<T>& p, size_t bytes) {
  void* raw = nullptr;
  cudaError_t e = cudaMalloc(&raw, bytes);
  p.reset(static_cast<T*>(raw));
  return e;
}

// ---------------- kernel ids (launch accounting + the optional CUDA-event profiler) ----------------
enum KernelId {
  K_FILL = 0, K_PROJECT_SCATTER, K_PREPROCESS_TILE, K_ICP_JACOBIAN, K_GN_INIT,
  K_ICP_FUSED, K_POSE_PRODUCTS, K_RENDER_SCATTER, K_RENDER_RESOLVE, K_INDEX_SCATTER, K_RADIUS, K_UPDATE_SURFELS,
  K_GEN_SURFELS, K_EXTRACT_FLAGS, K_COMPACT_SCATTER, K_AOS_TO_SOA, K_SOA_TO_AOS, K_ICP_POST, K_STATE_PACK,
  K_STATE_UNPACK, K_STATE_DIGEST, K_POOL_RECLAIM, K_POINT_LABELS, K_COUNT
};
const char* kernel_name(int id);

// per-kernel device time with CUDA events on the launching stream (off by default: zero overhead)
struct Profiler {
  bool on = false;
  struct Rec { int id; cudaEvent_t e0, e1; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  cudaEvent_t get() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }
};

// ---------------- launchers (implemented in the .cu files) ----------------
struct Launch {
  cudaStream_t stream;
  uint64_t* counter;  // number of kernels launched
  Profiler* prof;
};

struct ScopedKernel {
  const Launch& L;
  int slot = -1;
  ScopedKernel(const Launch& l, int id) : L(l) {
    ++*L.counter;
    if (L.prof && L.prof->on) {
      Profiler::Rec r{id, L.prof->get(), L.prof->get()};
      cudaEventRecord(r.e0, L.stream);
      L.prof->recs.push_back(r);
      slot = (int)L.prof->recs.size() - 1;
    }
  }
  ~ScopedKernel() {
    if (slot >= 0) cudaEventRecord(L.prof->recs[slot].e1, L.stream);
  }
};

// sb_preprocess.cu
// the two alternating z-buffer key images of the scan projection ([H][W+6] each, see sb_preprocess.cu) and their TMA maps
struct PrepKeys {
  DevPtr<unsigned long long> img[2];
  int cur = 0;
  bool tmap_ok[2] = {false, false};
  CUtensorMap tmap[2];
};
size_t preprocess_key_elems(int W, int H);
bool make_key_tensor_map(CUtensorMap* out, const unsigned long long* keys, int W, int H);
// per-point deskewing fused into K1a (DESIGN.md section 11): sweep-time source, s_ref, the sweep's motion as fp32
// axis-angle w and translation t, and where the moved points go (n float4, read by the tile pass instead of the input)
struct DeskewArgs {
  const float* times;  // mode 1: device pointer, one time per point
  int mode;            // 1 per-point times, 2 azimuth
  float ref_time, start_azimuth;
  int clockwise;
  float w[3], t[3];
  float4* out;
};
// K1-K3 (+ optionally K6b radius map and the re-arming of the index-map keys / integrated flags for the map update);
// deskew == nullptr: the points are projected as they are
void launch_preprocess(const Launch& L, const KParams& kp, const float4* pts, const float* labels, const float* probs,
                       uint32_t n, uint32_t timestamp, PrepKeys& keys, FrameDev out, float4* radius_map,
                       unsigned long long* index_keys, uint8_t* integrated, uint32_t* group_counts,
                       const DeskewArgs* deskew = nullptr);
// per-point labels of a scan (DESIGN.md section 13): the scan's own points, its key image (the one launch_preprocess
// read), its data frame and integrated flags, and the model frame (model.vertex == nullptr: none this scan)
struct PointLabelIO {
  const float4* pts;
  uint32_t n;
  const unsigned long long* keys;
  FrameDev frame;
  const uint8_t* integrated;
  FrameDev model;
  sb_point_label* out;
};
void launch_point_labels(const Launch& L, const KParams& kp, const PointLabelIO& io, const DeskewArgs* deskew);

// sb_icp.cu
void launch_icp_jacobian(const Launch& L, const KParams& kp, const IcpArgs& a, const Mat4& pose, int iteration,
                         long long* acc32, long long* slots, unsigned int* ticket, int blocks);
// ---- persistent Gauss-Newton kernel (sb_icp.cu) ----
enum GnMode { GN_PLAIN = 0, GN_MAIN = 1, GN_POST = 2 };
struct GnJob {
  int mode;
  IcpArgs a;    // GN_PLAIN / GN_MAIN: the objective; GN_POST: the statistics pass at identity (all rows)
  IcpArgs fb;   // GN_POST: the frame-to-frame recovery objective (row stripe in multi-GPU mode)
  GnState* st;  // state of the run (GN_PLAIN: prepared by k_gn_init)
  PoseDev* pd;  // GN_MAIN / GN_POST
  long long* stats32;                       // GN_POST: raw sums of the statistics pass, read by the host after the scan
  float* poses; float* poses_inv; uint32_t t_map, pose_cap;  // GN_POST: pose-table entry of this scan, table size
  // GN_MAIN / GN_POST: table inv(P) * poses[t] filled at the end over the window [pose_begin, pose_end) (or null)
  float* Mtab; uint32_t pose_begin, pose_end;
  int initialize_identity, fallback_mode;
  uint32_t timestamp;
  int max_iter;
  double eps, delta;
  unsigned int epoch_base;
};
void launch_gn_init(const Launch& L, GnState* st, const Mat4d& T0, long long* acc32);
int launch_gn_persistent(const Launch& L, const KParams& kp, const GnJob& job, long long* slots, unsigned int* ticket,
                         unsigned long long* pub, const CommDev* comm, int blocks);
int gn_persistent_max_blocks(int sm_count);
// one-thread bookkeeping kernels: first scan of a sequence and the host-callback exchange
void launch_pose_after_icp(const Launch& L, const GnState* gn, PoseDev* pd, const Mat4d& T0, uint32_t timestamp,
                           int fallback_mode);
void launch_pose_finalize(const Launch& L, const GnState* gn, PoseDev* pd, int had_icp, float* poses, float* poses_inv,
                          uint32_t t, uint32_t pose_cap);
int icp_grid_blocks(int sm_count);
int icp_balanced_blocks(int pixels, int max_blocks);

// sb_map.cu
struct RenderTargets {
  unsigned long long* key_old;   // may be null
  unsigned long long* key_new;   // may be null
  unsigned long long* key_comp;  // may be null
};
// The map update's index keys (K6a), written by the post-ICP render of the pipeline: that render and the index pass
// read the same map at the same pose with the same product table whenever the track-loss recovery does not run, so the
// render computes the keys from the transform, visibility test and centre projection it has already done.
struct IndexFuse {
  unsigned long long* keys;  // the index keys, armed this scan
  const int* fallback;       // PoseDev::fallback of the scan: set -> no keys here, the gated index pass writes them all
  int same_projection;       // model and data projection parameters are bitwise equal: the render's projection serves
};
// out[t] = A * poses[t] for t in [begin, end): the entries the live surfels of the map can refer to
void launch_pose_products(const Launch& L, const Mat4& A, const Mat4* A_dev, const float* poses, float* out,
                          uint32_t begin, uint32_t end);
// Surfel slots [0, counts[0]) of the map; a slot whose liveness byte is 0 holds a surfel removed by an in-place update.
// index != null: also write the index keys (IndexFuse).
void launch_render_scatter(const Launch& L, const KParams& kp, SurfelPlanes s, const uint32_t* n_dev, const uint8_t* live,
                           uint32_t n_upper, const float* M, float conf_thr, int t_thr, int emit_old, int emit_new,
                           int lequal, RenderTargets t, const IndexFuse* index = nullptr);
void launch_render_resolve(const Launch& L, const KParams& kp, SurfelPlanes s, const float* M_old, const float* M_new,
                           RenderTargets t, FrameDev f_old, FrameDev f_new, FrameDev f_comp, FrameDev f_out,
                           FrameDev f_copy, int keep_semantic, int lequal);
// gate != null: runs only if *gate is set (the repair of a fused scan on which the track-loss recovery ran)
void launch_index_scatter(const Launch& L, const KParams& kp, SurfelPlanes s, const uint32_t* n_dev, const uint8_t* live,
                          uint32_t n_upper, const float* M, unsigned long long* keys, const int* gate = nullptr);
void launch_radius(const Launch& L, const KParams& kp, FrameDev frame, float4* radius_map, unsigned long long* index_keys,
                   uint8_t* integrated, uint32_t* group_counts);
// ordered compaction of a surfel-indexed pass: items flagged in keep[0..n) of src go to dst[base..) in order, base =
// *base_dev (0 if null); out[0] = end of the written range, out[1] = number of items kept; dst_live (or null): liveness
// bytes of the destination, set for every slot written
void launch_compact(const Launch& L, SurfelPlanes src, const uint8_t* keep, const uint32_t* block_counts,
                    const uint32_t* group_counts, const uint32_t* n_dev, uint32_t n_upper, SurfelPlanes dst,
                    uint8_t* dst_live, const uint32_t* base_dev, uint32_t cap, uint32_t rel_cap, uint32_t* out);
// the live surfels of src, in order, to dst[0..); `live` is read for src and then set for dst. The group totals must be
// zero; out must not alias *n_dev.
void launch_compact_live(const Launch& L, SurfelPlanes src, const uint32_t* n_dev, uint32_t n_upper, uint8_t* live,
                         uint8_t* keep, uint32_t* block_counts, uint32_t* group_counts, SurfelPlanes dst, uint32_t* out);
// lazy = false: updated records into tmp + keep bytes for launch_compact; lazy = true: in place in src, removed surfels
// marked dead in `live`, counts[1] = physical end
void launch_update_surfels(const Launch& L, const KParams& kp, bool lazy, SurfelPlanes src, SurfelPlanes tmp,
                           uint32_t* counts, uint32_t n_upper, const Mat4& pose, const Mat4& inv_pose,
                           const Mat4* pose_dev, const Mat4* inv_pose_dev, const float* poses,
                           const float* poses_inv, const unsigned long long* index_keys, const float4* radius_map,
                           FrameDev frame, int timestamp, float2 submap_center, float submap_extent,
                           uint8_t* integrated, uint8_t* live, uint8_t* keep, uint32_t* block_counts,
                           uint32_t* group_counts);
// single-pass update / generate with in-place ordered compaction (decoupled look-back), appended behind counts[1];
// lazy_groups (the group totals of an in-place update, or null): counts[2] = their sum, counts[5] = counts[1] - sum
void launch_gen_compact(const Launch& L, const KParams& kp, FrameDev frame, const float4* radius_map,
                        const uint8_t* integrated, const float* poses, int timestamp, float2 submap_center,
                        float submap_extent, SurfelPlanes map, uint8_t* live, const uint32_t* lazy_groups,
                        unsigned long long* desc, uint32_t* ticket, uint32_t gen, uint32_t cap, uint32_t* counts);
// the live surfels of one submap tile, in order, into pool slot `slot`: rec[slot] = {end of the slot in the pool, surfels
// of the tile}; slot s starts at the end of slot s - 1. The group totals must be zero. *pose_min is lowered to the
// smallest pose-table entry of the live surfels of the map (those of the tile included).
void launch_extract_to_pool(const Launch& L, SurfelPlanes map, const uint32_t* n_dev, const uint8_t* live, uint32_t n_upper,
                            const float* poses, uint32_t pose_cap, uint32_t* pose_min, float2 center, float extent,
                            uint8_t* keep, uint32_t* block_counts,
                            uint32_t* group_counts, SurfelPlanes pool, uint32_t pool_cap, uint2* rec, uint32_t slot,
                            uint32_t tile_cap);
// Managed tile cache: dst[dst_base + d] = src[segs[i].x + d - segs[i].y] for d in [0, total), i the last segment with
// segs[i].y <= d (segs sorted by .y, segs[0].y == 0); nseg == 0: one segment that starts at src_base. src and dst must
// not overlap (the pool is compacted through the scratch set T).
void launch_pool_reclaim(const Launch& L, SurfelPlanes src, SurfelPlanes dst, const uint2* segs, uint32_t nseg,
                         uint32_t src_base, uint32_t dst_base, uint32_t total);
void launch_aos_to_soa(const Launch& L, const sb_surfel* aos, SurfelPlanes s, uint32_t offset, uint32_t n);
void launch_soa_to_aos(const Launch& L, SurfelPlanes s, sb_surfel* aos, uint32_t n);

// ---- checkpoint digest (sb_state_save / sb_state_load) ----
// The digest of a checkpoint is the sum mod 2^64 of state_word_hash(i, w) over its little-endian 64-bit words w at word
// offset i. Keyed by position, it changes when words move; being a sum, the blocks of a kernel and the host's part combine
// into the same value whatever order they are added in.
__host__ __device__ inline uint64_t state_mix64(uint64_t x) {  // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
__host__ __device__ inline uint64_t state_word_hash(uint64_t pos, uint64_t w) {
  return state_mix64(w ^ state_mix64(pos + 0x9e3779b97f4a7c15ull));
}
// The live surfels of map slots [0, n_phys), in order, into `flat` as four lanes of pitch n_live (p0[n_live], p1[...], ...),
// with their digest at blob word offset word_base added to *acc. Single pass: decoupled look-back (sb_map.cu).
void launch_state_pack(const Launch& L, SurfelPlanes map, const uint8_t* live, uint32_t n_phys, float4* flat,
                       uint32_t n_live, unsigned long long* desc, uint32_t* ticket, uint32_t gen, uint64_t word_base,
                       unsigned long long* acc);
// the reverse into a dense map: flat lanes of pitch n -> map slots [0, n), liveness set, digest added to *acc
void launch_state_unpack(const Launch& L, const float4* flat, uint32_t n, SurfelPlanes map, uint8_t* live,
                         uint64_t word_base, unsigned long long* acc);
// digest of n_words device words at blob word offset word_base, added to *acc
void launch_state_digest(const Launch& L, const void* words, uint64_t n_words, uint64_t word_base, unsigned long long* acc);

}  // namespace sb
