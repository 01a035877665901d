// sb_icp.cu -- K5: per-pixel projective association, point-to-plane residual, 6-DoF Jacobian and the reduction to
// J^T W J / J^T W r, plus the device-resident Gauss-Newton loop.
// Replaces Frame2Model::jacobianProducts (core/Frame2Model.cpp:136-261), its shader
// Frame2Model_jacobians.geom:67-247 and LieGaussNewton::minimize/step (core/LieGaussNewton.cpp:13-79).
//
// H100 mapping
//  * the reference sums 16 RGB texels through ROP float blending (order undefined) and reads 48 floats back with two
//    glFinish per iteration. Here every pixel's fp32 terms are converted to Q33.30 fixed point and summed as int64:
//    registers -> warp shuffles -> one 64-bit RED per value and block. Integer addition is associative, so the
//    result is bit-identical for any grid, any row striping and any number of GPUs.
//  * the Gauss-Newton step (6x6 LDL^T, SE3 exp, stop tests) runs in the last block to finish; iteration i+1 reads the
//    new pose from HBM. The whole minimisation is launched back-to-back with no host round trip.
//  * 6 range images of 2 MiB are L2-resident; the pass is latency/reduction bound, not HBM bound (DESIGN.md).
#include "sb_gn.cuh"
#include "sb_internal.cuh"

namespace sb {
using namespace sbm;

constexpr int kIcpThreads = 256;

int icp_grid_blocks(int sm_count) { return sm_count * 2; }

// number of blocks such that every thread gets the same number of pixels (the GN iteration time is the time of the
// slowest block): P/256 work units, u = ceil(units / max_blocks) units per block
int icp_balanced_blocks(int pixels, int max_blocks) {
  int units = (pixels + kIcpThreads - 1) / kIcpThreads;
  if (max_blocks < 1) max_blocks = 1;
  int u = (units + max_blocks - 1) / max_blocks;
  int blocks = (units + u - 1) / u;
  return blocks < 1 ? 1 : blocks;
}

__device__ __forceinline__ float4 tex_border(const float4* __restrict__ img, int W, int H, int x, int y) {
  if (x < 0 || x >= W || y < 0 || y >= H) return make_float4(0.f, 0.f, 0.f, 0.f);
  return __ldg(img + (size_t)y * W + x);
}

// texture(sampler2DRect, idx) with NEAREST or LINEAR filtering, CLAMP_TO_BORDER, border (0,0,0,0)
struct Bilin {
  int i0, j0;
  float w00, w10, w01, w11;
};
__device__ __forceinline__ Bilin bilin_setup(float u, float v) {
  Bilin b;
  float a = u - 0.5f, c = v - 0.5f;
  float fa = floorf(a), fc = floorf(c);
  b.i0 = (int)fa;
  b.j0 = (int)fc;
  float al = a - fa, be = c - fc;
  b.w00 = (1.0f - al) * (1.0f - be);
  b.w10 = al * (1.0f - be);
  b.w01 = (1.0f - al) * be;
  b.w11 = al * be;
  return b;
}
__device__ __forceinline__ float4 sample_bilin(const float4* __restrict__ img, int W, int H, const Bilin& b) {
  float4 t00 = tex_border(img, W, H, b.i0, b.j0);
  float4 t10 = tex_border(img, W, H, b.i0 + 1, b.j0);
  float4 t01 = tex_border(img, W, H, b.i0, b.j0 + 1);
  float4 t11 = tex_border(img, W, H, b.i0 + 1, b.j0 + 1);
  float4 r;
  r.x = ((b.w00 * t00.x + b.w10 * t10.x) + b.w01 * t01.x) + b.w11 * t11.x;
  r.y = ((b.w00 * t00.y + b.w10 * t10.y) + b.w01 * t01.y) + b.w11 * t11.y;
  r.z = ((b.w00 * t00.z + b.w10 * t10.z) + b.w01 * t01.z) + b.w11 * t11.z;
  r.w = ((b.w00 * t00.w + b.w10 * t10.w) + b.w01 * t01.w) + b.w11 * t11.w;
  return r;
}

// accumulators of one thread
struct Acc {
  long long s[29];  // 21 lower-triangle JtWJ | 6 JtWr | F | F_inlier
  int n_valid, n_outlier, n_invalid;
};

// Frame2Model_jacobians.geom:84-200 for one data pixel
__device__ __forceinline__ void icp_pixel_v(const KParams& kp, const IcpArgs& a, const float* M, int pix, float4 Vd, float4 Nd,
                                            int iteration, Acc& acc) {
  float e_d = Vd.w + Nd.w;
  if (!(e_d > 1.5f)) {
    acc.n_invalid += 1;
    return;
  }
  V3 v_d = xform_point(M, mk3(Vd.x, Vd.y, Vd.z));
  V3 n_d = xform_dir(M, mk3(Nd.x, Nd.y, Nd.z));
  // project2model, .geom:53-65
  float depth = len3(v_d);
  float yaw = atan2f_(v_d.y, v_d.x);
  float pitch = -asinf_(v_d.z / depth);
  float px = 0.5f * ((-yaw * kInvPi) + 1.0f);
  float py = 1.0f - (kRad2Deg * pitch + kp.fov_up) / kp.fov;
  float ix = px * (float)a.Wm, iy = py * (float)a.Hm;
  if (!(ix >= 0.0f && ix < (float)a.Wm && iy >= 0.0f && iy < (float)a.Hm)) {
    acc.n_invalid += 1;
    return;
  }
  float4 Vm, Nm;
  Bilin b;
  int tx = 0, ty = 0;
  if (kp.bilinear) {
    b = bilin_setup(ix, iy);
    Vm = sample_bilin(a.model_v, a.Wm, a.Hm, b);
    Nm = sample_bilin(a.model_n, a.Wm, a.Hm, b);
  } else {
    tx = (int)floorf(ix);
    ty = (int)floorf(iy);
    Vm = tex_border(a.model_v, a.Wm, a.Hm, tx, ty);
    Nm = tex_border(a.model_n, a.Wm, a.Hm, tx, ty);
  }
  float e_m = Vm.w + Nm.w;
  if (!(e_m > 1.5f)) {
    acc.n_invalid += 1;
    return;
  }
  V3 v_m = mk3(Vm.x, Vm.y, Vm.z), n_m = mk3(Nm.x, Nm.y, Nm.z);
  bool inlier = true;
  if (len3(sub3(v_m, v_d)) > a.distance_thresh) inlier = false;
  if (dot3(n_m, n_d) < a.angle_thresh) inlier = false;
  float residual = dot3(n_m, sub3(v_d, v_m));
  V3 cp = cross3(v_d, n_m);
  float weight = 1.0f;
  if (kp.weighting == 4 || kp.weighting == 1) {
    if (fabsf(residual) > kp.factor) weight = kp.factor / fabsf(residual);
  } else if (kp.weighting == 2 && iteration > 0) {
    if (fabsf(residual) > kp.factor) {
      weight = 0.0f;
    } else {
      float alpha = residual / kp.factor;
      weight = 1.0f - alpha * alpha;
      weight = weight * weight;
    }
  }
  if (a.has_semantics) {  // .geom:144-158
    float4 Sm = kp.bilinear ? sample_bilin(a.model_s, a.Wm, a.Hm, b) : tex_border(a.model_s, a.Wm, a.Hm, tx, ty);
    float4 Sd = __ldg(a.data_s + pix);
    float data_label = Sd.x * 255.0f, data_prob = Sd.w, model_label = Sm.x * 255.0f;
    if (is_movable(model_label)) {
      if (roundf_(data_label) != roundf_(model_label))
        weight = weight * (1.0f - data_prob);
      else
        weight = weight * data_prob;
    }
  }
  acc.n_valid += 1;
  float wr = weight * residual;
  acc.s[27] += fix30(wr * residual);
  if (inlier) {
    const float J[6] = {n_m.x, n_m.y, n_m.z, cp.x, cp.y, cp.z};
    int k = 0;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      float wc = weight * J[c];
#pragma unroll
      for (int r = c; r < 6; ++r) acc.s[k++] += fix30(wc * J[r]);
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) acc.s[21 + r] += fix30(wr * J[r]);
    acc.s[28] += fix30(wr * residual);
  } else {
    acc.n_outlier += 1;
  }
}

__device__ __forceinline__ void icp_pixel(const KParams& kp, const IcpArgs& a, const float* M, int pix, int iteration,
                                          Acc& acc) {
  icp_pixel_v(kp, a, M, pix, __ldg(a.data_v + pix), __ldg(a.data_n + pix), iteration, acc);
}

// Warp-level reduction of 32 values x 32 lanes with a transposing butterfly: at every step each lane keeps half of its
// values and trades the other half with its partner, so the whole reduction costs 16+8+4+2+1 = 31 exchanges instead of
// 32 x 5. Afterwards lane l holds the warp total of value l. (int64, so the association order is irrelevant.)
template <int kHalf>
__device__ __forceinline__ void transpose_reduce_stage(long long (&v)[32], int lane) {
  const bool upper = (lane & kHalf) != 0;
#pragma unroll
  for (int i = 0; i < kHalf; ++i) {
    long long keep = upper ? v[i + kHalf] : v[i];
    long long send = upper ? v[i] : v[i + kHalf];
    long long recv = __shfl_xor_sync(0xffffffffu, send, kHalf);
    v[i] = keep + recv;
  }
}
// One template instance per stage: every index into v[] must be a compile-time constant, or v[] lives in local memory.
// nvcc does not fully unroll a loop over the stage width, and the local-memory version costs ~6 us per Gauss-Newton
// iteration at 64x2048 on an H100.
__device__ __forceinline__ long long warp_transpose_reduce(long long (&v)[32], int lane) {
  transpose_reduce_stage<16>(v, lane);
  transpose_reduce_stage<8>(v, lane);
  transpose_reduce_stage<4>(v, lane);
  transpose_reduce_stage<2>(v, lane);
  transpose_reduce_stage<1>(v, lane);
  return v[0];
}

constexpr int kAccReplicas = 8;  // blocks spread their REDs over 8 replicas of the 32 accumulators (less contention)

// block-level reduction: lane l of warp 0 ends up with the block total of value l and adds it to one replica
__device__ __forceinline__ void block_reduce_to_replica(Acc& acc, long long* __restrict__ replicas) {
  __shared__ long long sm[kIcpThreads / 32][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long v[32];
#pragma unroll
  for (int i = 0; i < 29; ++i) v[i] = acc.s[i];
  v[29] = acc.n_valid;
  v[30] = acc.n_outlier;
  v[31] = acc.n_invalid;
  sm[warp][lane] = warp_transpose_reduce(v, lane);
  __syncthreads();
  if (warp == 0) {
    long long t = 0;
#pragma unroll
    for (int w = 0; w < kIcpThreads / 32; ++w) t += sm[w][lane];
    if (t != 0)
      atomicAdd((unsigned long long*)(replicas + (size_t)(blockIdx.x % kAccReplicas) * 32 + lane), (unsigned long long)t);
  }
}

// executed by warp 0 of the last block: lane l returns the total of value l over the replicas
__device__ __forceinline__ long long sum_replicas(const long long* __restrict__ replicas, int lane) {
  long long r[kAccReplicas];
#pragma unroll
  for (int i = 0; i < kAccReplicas; ++i) r[i] = *(const volatile long long*)(replicas + (size_t)i * 32 + lane);
  long long tot = 0;
#pragma unroll
  for (int i = 0; i < kAccReplicas; ++i) tot += r[i];
  return tot;
}
__device__ __forceinline__ void clear_replicas(long long* __restrict__ replicas, int lane) {
#pragma unroll
  for (int i = 0; i < kAccReplicas; ++i) replicas[(size_t)i * 32 + lane] = 0;
}

__device__ __forceinline__ void icp_accumulate(const KParams& kp, const IcpArgs& a, const float* M, int iteration,
                                               Acc& acc) {
#pragma unroll
  for (int i = 0; i < 29; ++i) acc.s[i] = 0;
  acc.n_valid = acc.n_outlier = acc.n_invalid = 0;
  const int begin = a.row_begin * kp.W, end = a.row_end * kp.W;
  for (int pix = begin + blockIdx.x * blockDim.x + threadIdx.x; pix < end; pix += gridDim.x * blockDim.x)
    icp_pixel(kp, a, M, pix, iteration, acc);
}

// ---- plain evaluation: one K5 pass, result = 32 int64 sums written to g_acc by the last block ----
__global__ void __launch_bounds__(kIcpThreads) k_icp_jacobian(KParams kp, IcpArgs a, Mat4 pose, int iteration,
                                                              long long* __restrict__ g_acc,
                                                              long long* __restrict__ slots, unsigned int* ticket) {
  float M[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) M[i] = pose.m[i];
  Acc acc;
  icp_accumulate(kp, a, M, iteration, acc);
  block_reduce_to_replica(acc, slots);
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned int t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last || threadIdx.x >= 32) return;
  __threadfence();
  long long tot = sum_replicas(slots, threadIdx.x);
  clear_replicas(slots, threadIdx.x);
  g_acc[threadIdx.x] = tot;
  if (threadIdx.x == 0) *ticket = 0;
}

void launch_icp_jacobian(const Launch& L, const KParams& kp, const IcpArgs& a, const Mat4& pose, int iteration,
                         long long* acc32, long long* slots, unsigned int* ticket, int blocks) {
  {
    ScopedKernel sk(L, K_ICP_JACOBIAN);
    k_icp_jacobian<<<blocks, kIcpThreads, 0, L.stream>>>(kp, a, pose, iteration, acc32, slots, ticket);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Device-side pose bookkeeping of SurfelMapping::updatePose (SurfelMapping.cpp:389-473): fp64, one thread, the same
// functions (sbg::*) the host-side API uses, so host and device agree bit for bit. Used by the last block of the
// persistent kernel (pipeline) and by the one-thread kernels below (first scan, host-callback exchange).
// ------------------------------------------------------------------------------------------------------------
__device__ void pose_after_icp_body(const double* gn_pose, int gn_k, PoseDev* pd, const double* T0, uint32_t timestamp,
                                    int fallback_mode) {
  double inc[16], inv_last[16], delta[16], Pn[16];
  for (int i = 0; i < 16; ++i) pd->T0[i] = T0[i];
  for (int i = 0; i < 16; ++i) inc[i] = gn_pose[i];  // increment = gn_->pose()   :395
  for (int i = 0; i < 16; ++i) pd->increment[i] = inc[i];
  pd->icp_iterations = gn_k;
  sbg::rigid_inverse_d(pd->lastIncrement, inv_last);
  mat4_mul<double>(inv_last, inc, delta);           // delta = lastIncrement_.inverse() * increment   :397
  mat4_mul<double>(pd->currentPose, inc, Pn);       // currentPose_new_ * increment   :406
  for (int i = 0; i < 16; ++i) pd->P_active.m[i] = (float)Pn[i];
  sbg::rigid_inverse_f(pd->P_active.m, pd->invP_active.m);
  float t_err = (float)sqrt((delta[12] * delta[12] + delta[13] * delta[13]) + delta[14] * delta[14]);  // :433
  float angle = (float)(0.5 * (((delta[0] + delta[5]) + delta[10]) - 1.0));
  float ca = angle < 1.0f ? angle : 1.0f;
  ca = ca > -1.0f ? ca : -1.0f;
  float r_err = acosf_(ca);
  pd->t_err = t_err;
  pd->r_err = r_err;
  int fb = (timestamp > 1 && ((double)t_err > 0.4 || (double)r_err > 0.1) && fallback_mode) ? 1 : 0;  // :437
  pd->fallback = fb;
  if (fb) pd->trackLoss += 1;
}

// lastPose_ = currentPose_; currentPose_ = currentPose_ * increment; ... (SurfelMapping.cpp:451-473) and the pose-table
// entry of this scan (SurfelMap.cpp:494-495)
__device__ void pose_finalize_body(const double* recovery_pose, PoseDev* pd, int had_icp, float* poses, float* poses_inv,
                                   uint32_t t, uint32_t pose_cap) {
  if (had_icp) {
    double inc[16], np[16];
    if (pd->fallback)
      for (int i = 0; i < 16; ++i) inc[i] = recovery_pose[i];  // increment = gn_->pose() of the recovery run   :446
    else
      for (int i = 0; i < 16; ++i) inc[i] = pd->increment[i];
    for (int i = 0; i < 16; ++i) pd->lastPose[i] = pd->currentPose[i];
    mat4_mul<double>(pd->currentPose, inc, np);  // :452
    for (int i = 0; i < 16; ++i) {
      pd->currentPose[i] = np[i];
      pd->lastIncrement[i] = inc[i];  // :473
      pd->increment[i] = inc[i];
    }
  }
  for (int i = 0; i < 16; ++i) pd->P_cur.m[i] = (float)pd->currentPose[i];
  sbg::rigid_inverse_f(pd->P_cur.m, pd->invP_cur.m);
  if (t < pose_cap) {  // (the host grows the table before it enqueues the scan)
    float inv[16];
    sbg::rigid_inverse_f(pd->P_cur.m, inv);
    for (int i = 0; i < 16; ++i) {
      poses[16 * (size_t)t + i] = pd->P_cur.m[i];
      poses_inv[16 * (size_t)t + i] = inv[i];
    }
  }
}

__global__ void k_gn_init(GnState* st, Mat4d T0, long long* acc32) {
  int i = threadIdx.x;
  if (i < 16) st->pose[i] = T0.m[i];
  if (i < 32) acc32[i] = 0;
  if (i < 48) st->out48[i] = 0.0;
  if (i == 0) {
    st->last_error = (double)3.402823466e+38f;  // numeric_limits<float>::max(), LieGaussNewton.cpp:48
    st->k = 0;
    st->done = 0;
    st->history_len = 0;
    st->error = 0;
  }
}

void launch_gn_init(const Launch& L, GnState* st, const Mat4d& T0, long long* acc32) {
  {
    ScopedKernel sk(L, K_GN_INIT);
    k_gn_init<<<1, 64, 0, L.stream>>>(st, T0, acc32);
  }
}

__global__ void k_pose_after_icp(const GnState* __restrict__ gn, PoseDev* __restrict__ pd, Mat4d T0, uint32_t timestamp,
                                 int fallback_mode) {
  if (threadIdx.x != 0) return;
  pose_after_icp_body(gn->pose, gn->k, pd, T0.m, timestamp, fallback_mode);
}
void launch_pose_after_icp(const Launch& L, const GnState* gn, PoseDev* pd, const Mat4d& T0, uint32_t timestamp,
                           int fallback_mode) {
  {
    ScopedKernel sk(L, K_GN_INIT);
    k_pose_after_icp<<<1, 32, 0, L.stream>>>(gn, pd, T0, timestamp, fallback_mode);
  }
}

__global__ void k_pose_finalize(const GnState* __restrict__ gn, PoseDev* __restrict__ pd, int had_icp,
                                float* __restrict__ poses, float* __restrict__ poses_inv, uint32_t t, uint32_t pose_cap) {
  if (threadIdx.x != 0) return;
  pose_finalize_body(gn->pose, pd, had_icp, poses, poses_inv, t, pose_cap);
}
void launch_pose_finalize(const Launch& L, const GnState* gn, PoseDev* pd, int had_icp, float* poses, float* poses_inv,
                          uint32_t t, uint32_t pose_cap) {
  {
    ScopedKernel sk(L, K_GN_INIT);
    k_pose_finalize<<<1, 32, 0, L.stream>>>(gn, pd, had_icp, poses, poses_inv, t, pose_cap);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Persistent Gauss-Newton kernel: ONE cooperative launch runs every iteration of a minimisation AND the bookkeeping
// around it. All blocks are co-resident; after the reduction the last block to arrive performs the GN step
// (warp-parallel 6x6 LDL^T, SE3 exp, pose update) and releases the other blocks through an epoch word in HBM. No kernel
// boundary and no host round trip per iteration (the reference does a 48-float read-back and two glFinish per
// iteration, Frame2Model.cpp:205-258).
//
// Three jobs (GnJob::mode):
//  GN_PLAIN  LieGaussNewton::minimize on a pre-initialised state (sb_icp_minimize).
//  GN_MAIN   updatePose, first half (SurfelMapping.cpp:372-406): T0 from the device-resident pose block, the
//            frame-to-model minimisation, then -- by the block that did the last step -- the increment, the pose of the
//            post-ICP rendering and the track-loss test; finally ALL blocks fill the table inv(P_active) * poses[t] that
//            render_active needs. (Round 1: four launches.)
//  GN_POST   updatePose, second half (:415-473): pass 0 is the statistics evaluation at identity against the freshly
//            rendered active model (result_new_); if the track was lost the same loop then runs the frame-to-frame
//            recovery minimisation; the finishing block chains the poses and writes the pose-table entry; finally all
//            blocks fill inv(P_cur) * poses[t] for the map update and the model rendering. (Round 1: five launches.)
//
// Epoch words never need a reset: launch j waits for base_j + iteration + 1 with base_{j+1} > every value launch j can
// publish (the host advances the base by max_iter + 8 per launch). The arrival ticket is returned to 0 by each step.
// Every spin is bounded (%globaltimer): a peer or a block that never shows up ends the launch with GnState::error set
// instead of hanging the stream.
// ------------------------------------------------------------------------------------------------------------
struct GnShared {
  double A[36];
  double O[48];
  double P[16];
  double E[16];
  double dx[6];
  int perm[6];
  int result;
};

__device__ __forceinline__ void tri_cr(int k, int& c, int& r) {  // k-th entry of the column-wise lower triangle
  const int start[6] = {0, 6, 11, 15, 18, 20};
  c = 0;
#pragma unroll
  for (int i = 1; i < 6; ++i)
    if (k >= start[i]) c = i;
  r = c + (k - start[c]);
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
constexpr unsigned long long kSpinTimeoutNs = 10ull * 1000ull * 1000ull * 1000ull;  // 10 s

// same arithmetic as sbg::ldlt_solve6 / sbg::gn_step, spread over the 32 lanes of one warp (per-element operation
// order unchanged, so the result is bit-identical to the sequential code)
__device__ void gn_step_warp(GnShared& sh, long long raw, int lane, double last_error, double eps, double delta_thr) {
  const double s = 1.0 / 1073741824.0;
  // unpack (Frame2Model.cpp:214-227)
  if (lane < 21) {
    int c, r;
    tri_cr(lane, c, r);
    double v = (double)raw * s;
    sh.O[c * 6 + r] = v;
    sh.O[r * 6 + c] = v;
  } else if (lane < 27) {
    sh.O[36 + (lane - 21)] = (double)raw * s;
  } else if (lane == 27) {
    sh.O[43] = (double)raw * s;
  } else if (lane == 28) {
    sh.O[45] = (double)raw * s;
  } else if (lane == 29) {
    sh.O[42] = (double)raw;
  } else if (lane == 30) {
    sh.O[44] = (double)raw;
  } else {
    sh.O[46] = (double)raw;
    sh.O[47] = 0.0;
  }
  __syncwarp();
  double* A = sh.A;
  for (int i = lane; i < 36; i += 32) A[i] = sh.O[i];  // already symmetric
  if (lane < 6) sh.perm[lane] = lane;
  __syncwarp();
#pragma unroll 1
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double best = fabs(A[k * 6 + k]);
    for (int i = k + 1; i < 6; ++i) {
      double v = fabs(A[i * 6 + i]);
      if (v > best) {
        best = v;
        piv = i;
      }
    }
    __syncwarp();  // every lane has read the diagonal before lanes k / piv swap it below (without it: correct in lockstep only)
    if (piv != k) {  // warp-uniform
      if (lane < 6) {
        double t = A[k * 6 + lane];
        A[k * 6 + lane] = A[piv * 6 + lane];
        A[piv * 6 + lane] = t;
      }
      __syncwarp();
      if (lane < 6) {
        double t = A[lane * 6 + k];
        A[lane * 6 + k] = A[lane * 6 + piv];
        A[lane * 6 + piv] = t;
      }
      if (lane == 0) {
        int t = sh.perm[k];
        sh.perm[k] = sh.perm[piv];
        sh.perm[piv] = t;
      }
      __syncwarp();
    }
    double dk = A[k * 6 + k];
    if (dk == 0.0) continue;
    if (lane > k && lane < 6) A[k * 6 + lane] = A[k * 6 + lane] / dk;
    __syncwarp();
    if (lane < 21) {
      int c, r;
      tri_cr(lane, c, r);
      if (c > k) {
        double v = A[c * 6 + r] - (A[k * 6 + r] * dk) * A[k * 6 + c];
        A[c * 6 + r] = v;
        A[r * 6 + c] = v;
      }
    }
    __syncwarp();
  }
  if (lane == 0) {
    double y[6], dx[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] = -sh.O[36 + sh.perm[i]];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int k = 0; k < i; ++k) y[i] = y[i] - A[k * 6 + i] * y[k];
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] = (A[i * 6 + i] == 0.0) ? 0.0 : y[i] / A[i * 6 + i];
#pragma unroll
    for (int i = 5; i >= 0; --i)
#pragma unroll
      for (int k = i + 1; k < 6; ++k) y[i] = y[i] - A[i * 6 + k] * y[k];
#pragma unroll
    for (int i = 0; i < 6; ++i) sh.dx[sh.perm[i]] = y[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) dx[i] = sh.dx[i];
    int result = 1;
    double current_error = sh.O[43];
    double linf = 0.0, maxc = sh.O[36];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      if (fabs(dx[i]) > linf) linf = fabs(dx[i]);
      if (sh.O[36 + i] > maxc) maxc = sh.O[36 + i];
    }
    if (linf < delta_thr) result = 0;
    if (fabs(maxc) < eps) result = 0;
    if (current_error < last_error && fabs(current_error - last_error) < eps) result = 0;
    sh.result = result;
    double E[16];
    sbg::se3_exp(dx, E);
#pragma unroll
    for (int i = 0; i < 16; ++i) sh.E[i] = E[i];
  }
  __syncwarp();
  double pn = 0.0;
  if (lane < 16) {
    int c = lane >> 2, r = lane & 3;
    const double* Ea = sh.E;
    const double* B = sh.P;
    pn = ((Ea[0 * 4 + r] * B[c * 4 + 0] + Ea[1 * 4 + r] * B[c * 4 + 1]) + Ea[2 * 4 + r] * B[c * 4 + 2]) +
         Ea[3 * 4 + r] * B[c * 4 + 3];
  }
  __syncwarp();
  if (lane < 16) sh.P[lane] = pn;
  __syncwarp();
}

// lane-parallel one-shot all-reduce of the 32 sums over the ranks' peer-mapped mailboxes (warp 0 of the last block).
// Every rank stores its sums into slot [epoch&1][rank] of EVERY rank's mailbox as 64 self-validating 8-byte words
// (32-bit half of a sum | epoch stamp << 32; an aligned 8-byte store arrives whole over NVLink), so no fence separates
// payload and flag and the cost is ONE one-way store latency: each lane then spins on its own two words per source rank
// in its local mailbox. Two slots: a rank can only be one exchange ahead of the slowest reader. False on timeout.
__device__ bool comm_allreduce32_warp(const CommDev& cd, long long& raw, int lane) {
  unsigned int epoch = 0;
  if (lane == 0) {
    epoch = *cd.epoch + 1u;  // stamps start at 1: a zeroed mailbox never matches
    *cd.epoch = epoch;
  }
  epoch = __shfl_sync(0xffffffffu, epoch, 0);
  const int slot = (int)(epoch & 1u);
  const unsigned long long tag = (unsigned long long)epoch << 32;
  const unsigned long long w_lo = tag | (unsigned long long)(unsigned int)((unsigned long long)raw & 0xffffffffull);
  const unsigned long long w_hi = tag | (unsigned long long)(unsigned int)((unsigned long long)raw >> 32);
  for (int r = 0; r < cd.nranks; ++r) {
    volatile unsigned long long* dst =
        reinterpret_cast<volatile unsigned long long*>(cd.mailbox[r]) + ((size_t)(slot * 8 + cd.rank)) * 64;
    dst[lane] = w_lo;
    dst[32 + lane] = w_hi;
  }
  volatile unsigned long long* mine = reinterpret_cast<volatile unsigned long long*>(cd.mailbox[cd.rank]);
  const unsigned long long t0 = globaltimer_ns();
  unsigned long long tot = 0;
  int ok = 1;
  for (int r = 0; r < cd.nranks && ok; ++r) {
    volatile unsigned long long* src = mine + ((size_t)(slot * 8 + r)) * 64;
    unsigned long long lo = src[lane], hi = src[32 + lane];
    unsigned int spins = 0;
    while ((unsigned int)(lo >> 32) != epoch || (unsigned int)(hi >> 32) != epoch) {
      if ((++spins & 1023u) == 0u && globaltimer_ns() - t0 > kSpinTimeoutNs) {
        ok = 0;
        break;
      }
      lo = src[lane];
      hi = src[32 + lane];
    }
    tot += (lo & 0xffffffffull) | (hi << 32);
  }
  ok = __all_sync(0xffffffffu, ok);
  raw = (long long)tot;
  return ok != 0;
}

__device__ __forceinline__ void load_mat_cg(const float* table, int idx, float* M) {  // coherent (L2) read of a pose
  const float4* t = reinterpret_cast<const float4*>(table + 16 * (size_t)idx);
  float4 a = __ldcg(t), b = __ldcg(t + 1), c = __ldcg(t + 2), d = __ldcg(t + 3);
  M[0] = a.x; M[1] = a.y; M[2] = a.z; M[3] = a.w;
  M[4] = b.x; M[5] = b.y; M[6] = b.z; M[7] = b.w;
  M[8] = c.x; M[9] = c.y; M[10] = c.z; M[11] = c.w;
  M[12] = d.x; M[13] = d.y; M[14] = d.z; M[15] = d.w;
}

// kGnCachePix = data pixels per thread kept in shared memory across the iterations of one launch: 2 covers 64x2048 on
// one GPU (1.7 pixels per thread); 4 is the instantiation a row stripe of a larger image takes (128x4096 over >= 2 GPUs
// -- the aggregate shared memory of the GPUs holds what one GPU's does not). Measured: the 4-deep unrolled body costs the
// 64x2048 launch 3.5 us, hence two instantiations instead of one.
template <int kGnCachePix>
__global__ void __launch_bounds__(kIcpThreads, 2) k_gn_persistent(KParams kp, GnJob job, long long* __restrict__ slots,
                                                               unsigned int* ticket, unsigned long long* pub,
                                                               CommDev cd) {
  __shared__ GnShared sh;
  __shared__ double s_pose[16];
  __shared__ double s_last_error;  // travels with the pose: the block that performs the next step is not the same one
  __shared__ int s_done, s_error;
  __shared__ float4 s_dv[kGnCachePix][kIcpThreads], s_dn[kGnCachePix][kIcpThreads];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  GnState* st = job.st;
  PoseDev* pd = job.pd;
  if (threadIdx.x == 0) s_error = 0;
  // The data frame does not change during a minimisation and a thread visits the same pixels in every iteration: keep
  // their vertex / normal texels in shared memory (thread-private slots), which takes one dependent L2 round trip out of
  // every iteration. Only when the whole stripe fits (<= kGnCachePix pixels per thread) and the objective is fixed.
  const int px_begin = job.a.row_begin * kp.W, px_end = job.a.row_end * kp.W;
  const int px_stride = gridDim.x * blockDim.x, px_first = px_begin + blockIdx.x * blockDim.x + threadIdx.x;
  const bool cached = job.mode != GN_POST && (px_end - px_begin) <= kGnCachePix * px_stride;
  if (cached) {
#pragma unroll
    for (int j = 0; j < kGnCachePix; ++j) {
      const int pix = px_first + j * px_stride;
      if (pix < px_end) {
        s_dv[j][threadIdx.x] = __ldg(job.a.data_v + pix);
        s_dn[j][threadIdx.x] = __ldg(job.a.data_n + pix);
      }
    }
  }
  for (unsigned int it = 0;; ++it) {
    // Warp 0 waits for the previous iteration's step (epoch word), then fetches the state written by that step with ONE
    // round of coherent loads spread over its lanes and broadcasts it through shared memory (every thread reading the
    // pose from L2 would hammer a single L2 sector with ~40k requests per iteration).
    if (warp == 0) {
      if (it == 0) {
        if (job.mode == GN_PLAIN) {  // state prepared by k_gn_init earlier on the stream
          if (lane < 16) s_pose[lane] = st->pose[lane];
          if (lane == 17) s_done = st->done;
        } else {
          // GN_MAIN: T0 = lastIncrement_ or identity (SurfelMapping.cpp:373-376); GN_POST: the statistics pass runs at
          // identity (objective_->initialize(Identity), :414)
          if (lane < 16) {
            double v = (lane % 5 == 0) ? 1.0 : 0.0;
            if (job.mode == GN_MAIN && !job.initialize_identity) v = pd->lastIncrement[lane];
            s_pose[lane] = v;
          }
          if (lane == 17) s_done = 0;
        }
      } else {
        // The step publishes the new pose as 32 self-validating 8-byte words (half a double + the epoch tag, bit 31 of the
        // tag = done): lane l polls word l, so pose AND release arrive in ONE L2 round trip (a flag followed by a fetch
        // of the pose costs two) and no fence is needed on either side of the hand-over.
        const unsigned int want = (job.epoch_base + it) & 0x7fffffffu;
        const unsigned long long t0 = globaltimer_ns();
        unsigned int spins = 0;
        unsigned long long w = *(volatile unsigned long long*)&pub[lane];
        unsigned long long w2 = lane < 2 ? *(volatile unsigned long long*)&pub[32 + lane] : 0ull;  // last_error halves
        bool timed_out = false;
        while ((((unsigned int)(w >> 32)) & 0x7fffffffu) != want ||
               (lane < 2 && (((unsigned int)(w2 >> 32)) & 0x7fffffffu) != want)) {
          if ((++spins & 4095u) == 0u && globaltimer_ns() - t0 > kSpinTimeoutNs) {
            timed_out = true;
            break;
          }
          w = *(volatile unsigned long long*)&pub[lane];
          if (lane < 2) w2 = *(volatile unsigned long long*)&pub[32 + lane];
        }
        if (__any_sync(0xffffffffu, timed_out)) {
          if (lane == 0) s_error = 1;
        }
        const unsigned int lo = __shfl_sync(0xffffffffu, (unsigned int)w, 2 * (lane & 15));
        const unsigned int hi = __shfl_sync(0xffffffffu, (unsigned int)w, 2 * (lane & 15) + 1);
        if (lane < 16) s_pose[lane] = __hiloint2double((int)hi, (int)lo);
        if (lane == 17) s_done = (int)((w >> 63) & 1ull);
        const unsigned int e_lo = __shfl_sync(0xffffffffu, (unsigned int)w2, 0);
        const unsigned int e_hi = __shfl_sync(0xffffffffu, (unsigned int)w2, 1);
        if (lane == 18) s_last_error = __hiloint2double((int)e_hi, (int)e_lo);
      }
    }
    __syncthreads();
    if (s_error) {  // a block (or a peer GPU) never arrived: give up instead of hanging the stream
      if (threadIdx.x == 0) {
        *(volatile int*)&st->error = 1;
        if (pd) *(volatile int*)&pd->gn_error = 1;
      }
      return;
    }
    if (s_done) {
      __threadfence();  // the finishing step fenced its pose-block writes before the done tag; acquire them
      break;
    }
    // Two sets of accumulator replicas, alternating per pass: the set of pass p is cleared by the block that consumed it
    // AFTER it has released pass p + 1 (nobody adds to it before pass p + 2, and that block's own arrival fence of pass
    // p + 1 orders the clearing stores before the release of p + 2). The arrival ticket counts on across the passes of a
    // launch for the same reason: no reset, hence no fence, between the step and the release.
    long long* const my_slots = slots + (size_t)(it & 1u) * kAccReplicas * 32;
    const bool stats_pass = job.mode == GN_POST && it == 0;
    const bool recovery = job.mode == GN_POST && it > 0;
    const int k = job.mode == GN_POST ? (int)it - 1 : (int)it;  // k_ of LieGaussNewton: one increment per completed step
    float M[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) M[i] = (float)s_pose[i];  // pose_.cast<float>(), Frame2Model.cpp:194
    Acc acc;
    if (cached) {
#pragma unroll
      for (int i = 0; i < 29; ++i) acc.s[i] = 0;
      acc.n_valid = acc.n_outlier = acc.n_invalid = 0;
#pragma unroll
      for (int j = 0; j < kGnCachePix; ++j) {
        const int pix = px_first + j * px_stride;
        if (pix < px_end) icp_pixel_v(kp, job.a, M, pix, s_dv[j][threadIdx.x], s_dn[j][threadIdx.x], k, acc);
      }
    } else {
      icp_accumulate(kp, recovery ? job.fb : job.a, M, stats_pass ? 0 : k, acc);
    }
    block_reduce_to_replica(acc, my_slots);
    // Warp 0 issued the block's slot adds, so warp 0 alone fences them and takes the arrival ticket; the other warps go
    // straight to the loop-top barrier and wait there for the next pose (in the stepping block as in every other).
    if (warp != 0) continue;
    __threadfence();  // every lane: its slot add before the ticket
    __syncwarp();
    unsigned int ticket_no = 0;
    if (lane == 0) ticket_no = atomicAdd(ticket, 1u);
    ticket_no = __shfl_sync(0xffffffffu, ticket_no, 0);
    if (ticket_no == (it + 1u) * gridDim.x - 1u) {
      __threadfence();
      long long raw = sum_replicas(my_slots, lane);
      int done = 0, error = 0;
      double pv = 0.0;  // lanes 0..15: the pose of the next pass
      if (stats_pass) {
        // result_new_ (SurfelMapping.cpp:415-423): the host unpacks these 32 sums after the scan
        job.stats32[lane] = raw;
        const int fb = job.fallback_mode ? *(volatile int*)&pd->fallback : 0;
        if (fb) {  // recovery_->setData(currentFrame_, lastFrame_); gn_->minimize(*recovery_, T0)   :442-444
          if (lane < 16) {
            pv = pd->T0[lane];
            st->pose[lane] = pv;
          }
          if (lane == 0) {
            st->last_error = (double)3.402823466e+38f;
            st->k = 0;
            st->history_len = 0;
          }
        } else {
          done = 1;
        }
      } else {
        double last_error = (double)3.402823466e+38f;  // LieGaussNewton.cpp:48
        if (k > 0) last_error = s_last_error;          // published with the pose by the previous step
        if (cd.epoch) error = comm_allreduce32_warp(cd, raw, lane) ? 0 : 1;
        if (lane < 16) sh.P[lane] = s_pose[lane];
        int hl = k;  // one pose has been pushed per completed iteration
        if (lane < 16) st->history[hl * 16 + lane] = s_pose[lane];  // history_.push_back(Tk_)
        ++hl;
        __syncwarp();
        gn_step_warp(sh, raw, lane, last_error, job.eps, job.delta);
        if (lane < 16) {
          pv = sh.P[lane];
          st->pose[lane] = pv;
        }
        for (int i = lane; i < 48; i += 32) st->out48[i] = sh.O[i];
        int kk = k;
        if (sh.result == 0) {
          done = 1;
        } else {
          ++kk;
          if (kk >= job.max_iter) {  // the loop pushes the pose once more and leaves (LieGaussNewton.cpp:24-27)
            if (lane < 16) st->history[hl * 16 + lane] = sh.P[lane];
            ++hl;
            done = 1;
          }
        }
        if (error) done = 1;
        if (lane == 0) {
          st->last_error = sh.O[43];
          st->k = kk;
          st->history_len = hl;
        }
        __syncwarp();
      }
      if (done && lane == 0 && !error) {
        if (job.mode == GN_MAIN) {
          double T0[16];
          for (int i = 0; i < 16; ++i) T0[i] = job.initialize_identity ? ((i % 5 == 0) ? 1.0 : 0.0) : pd->lastIncrement[i];
          pose_after_icp_body(sh.P, st->k, pd, T0, job.timestamp, job.fallback_mode);
        } else if (job.mode == GN_POST) {
          pose_finalize_body(st->pose, pd, 1, job.poses, job.poses_inv, job.t_map, job.pose_cap);
        }
      }
      if (lane == 0) {
        if (error) {
          st->error = 1;
          if (pd) pd->gn_error = 1;
        }
        st->done = done;
        if (done) *ticket = 0;  // the next launch counts from 0 again
      }
      if (done) {  // the finishing step: every write of this launch is visible before the done tag
        clear_replicas(my_slots, lane);
        __threadfence();
      }
      __syncwarp();
      // release: the pose straight from the registers of this warp (the state stores above drain in the background)
      {
        const double src = __shfl_sync(0xffffffffu, pv, lane >> 1);
        const unsigned int half = (lane & 1) ? (unsigned int)__double2hiint(src) : (unsigned int)__double2loint(src);
        const unsigned int tag = ((job.epoch_base + it + 1u) & 0x7fffffffu) | (done ? 0x80000000u : 0u);
        *(volatile unsigned long long*)&pub[lane] = ((unsigned long long)tag << 32) | (unsigned long long)half;
        if (lane < 2) {
          const double le = stats_pass ? 0.0 : sh.O[43];  // this step's error = last_error of the next one
          const unsigned int eh = lane ? (unsigned int)__double2hiint(le) : (unsigned int)__double2loint(le);
          *(volatile unsigned long long*)&pub[32 + lane] = ((unsigned long long)tag << 32) | (unsigned long long)eh;
        }
      }
      if (!done) clear_replicas(my_slots, lane);  // behind the release, see above
    }
  }
  // ---- all blocks: the table inv(P) * poses[t] of the rendering / map update that follows (render_surfels.vert:46), over
  // the entries the live surfels can refer to ----
  if (job.Mtab) {
    if (*(volatile int*)&pd->gn_error) return;
    const float* A = job.mode == GN_MAIN ? pd->invP_active.m : pd->invP_cur.m;
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = *(volatile const float*)&A[i];
    const uint32_t t0 = job.pose_begin, nt = job.pose_end - job.pose_begin;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nt; i += gridDim.x * blockDim.x) {
      const uint32_t t = t0 + i;
      float b[16], c[16];
      load_mat_cg(job.poses, (int)t, b);
      mat4_mul<float>(a, b, c);
      float4* o = reinterpret_cast<float4*>(job.Mtab + 16 * (size_t)t);
      o[0] = make_float4(c[0], c[1], c[2], c[3]);
      o[1] = make_float4(c[4], c[5], c[6], c[7]);
      o[2] = make_float4(c[8], c[9], c[10], c[11]);
      o[3] = make_float4(c[12], c[13], c[14], c[15]);
    }
  }
}

int gn_persistent_max_blocks(int sm_count) {
  int per_sm = 0;
  int per_sm4 = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gn_persistent<2>, kIcpThreads, 0) != cudaSuccess) return 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm4, k_gn_persistent<4>, kIcpThreads, 0) != cudaSuccess) return 0;
  return (per_sm < per_sm4 ? per_sm : per_sm4) * sm_count;
}

int launch_gn_persistent(const Launch& L, const KParams& kp, const GnJob& job, long long* slots, unsigned int* ticket,
                         unsigned long long* pub, const CommDev* comm, int blocks) {
  CommDev cd;
  if (comm) {
    cd = *comm;
  } else {
    memset(&cd, 0, sizeof(cd));
    cd.nranks = 1;
  }
  KParams kpv = kp;
  GnJob jv = job;
  void* args[] = {&kpv, &jv, &slots, &ticket, &pub, &cd};
  cudaError_t e;
  {
    ScopedKernel sk(L, job.mode == GN_POST ? K_ICP_POST : K_ICP_FUSED);
    // the deeper cache only where the shallow one does not hold the stripe but the deep one does
    const long long px = (long long)(job.a.row_end - job.a.row_begin) * kp.W, per_pass = (long long)blocks * kIcpThreads;
    const bool deep = job.mode != GN_POST && px > 2 * per_pass && px <= 4 * per_pass;
    e = cudaLaunchCooperativeKernel(deep ? (void*)k_gn_persistent<4> : (void*)k_gn_persistent<2>, dim3(blocks),
                                    dim3(kIcpThreads), args, 0, L.stream);
  }
  return e == cudaSuccess ? 0 : -1;
}

}  // namespace sb
