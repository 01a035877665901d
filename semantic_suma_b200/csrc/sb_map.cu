// sb_map.cu -- K4 (model rendering) and K6 (surfel update / initialise / merge) of the surfel map.
// Replaces SurfelMap::render* (core/SurfelMap.cpp:847-1165; render_surfels.{vert,geom,frag}, render_compose.frag)
// and SurfelMap::update (core/SurfelMap.cpp:492-698; gen_indexmap, init_radiusConf, update_surfels, gen_surfels,
// copy_surfels, extract_surfels).
//
// H100 mapping
//  * GL triangle rasterisation + 24-bit z-buffer  ->  one thread per surfel walks the quad's pixel bounding box
//    with exact integer edge functions and resolves visibility with a 64-bit atomicMin on
//    (depth24 << 40 | pass << 32 | surfel index): "earliest primitive wins" falls out of the key order.
//    One pass over the surfel lanes feeds the old / new / composed views at once (the reference draws the whole
//    buffer four times per render()).
//  * transform feedback (ordered stream compaction)  ->  surfel order (and therefore every surfel index) is identical to
//    the reference's. The surfel-indexed passes (update, tile extraction) publish per-block counts and 64-block group
//    totals from their predicate kernel, and k_compact finds each block's offset from those; the pixel-indexed generation
//    pass compacts in one kernel with a decoupled look-back.
//  * surfels live as four float4 lanes (SoA), every pass streams only the lanes it needs with 128-bit accesses.
#include "sb_gn.cuh"
#include "sb_internal.cuh"

namespace sb {
using namespace sbm;

constexpr int kThreads = 256;

const char* kernel_name(int id) {
  static const char* names[K_COUNT] = {"fill_u64", "project_scatter", "preprocess_tile",
                                       "icp_jacobian", "gn_init", "icp_fused", "pose_products", "render_scatter",
                                       "render_resolve", "index_scatter", "radius", "update_surfels", "gen_surfels",
                                       "extract_flags", "compact_scatter", "aos_to_soa", "soa_to_aos", "icp_post",
                                       "state_pack", "state_unpack", "state_digest"};
  return (id >= 0 && id < K_COUNT) ? names[id] : "?";
}

__device__ __forceinline__ int pose_index(float count) {
  int c = (int)count;
  c = c < 0 ? 0 : c;
  c = c >= (int)kMaxPoses ? (int)kMaxPoses - 1 : c;
  return c;
}

__device__ __forceinline__ void load_mat(const float* __restrict__ table, int idx, float* M) {
  const float4* t = reinterpret_cast<const float4*>(table + 16 * (size_t)idx);
  float4 a = __ldg(t), b = __ldg(t + 1), c = __ldg(t + 2), d = __ldg(t + 3);
  M[0] = a.x; M[1] = a.y; M[2] = a.z; M[3] = a.w;
  M[4] = b.x; M[5] = b.y; M[6] = b.z; M[7] = b.w;
  M[8] = c.x; M[9] = c.y; M[10] = c.z; M[11] = c.w;
  M[12] = d.x; M[13] = d.y; M[14] = d.z; M[15] = d.w;
}

// out[t] = A * poses[t]  (render_surfels.vert:46 evaluates (inv_pose * surfelPose) * v; the product is shared by all
// surfels created at time t)
__global__ void k_pose_products(Mat4 A, const Mat4* __restrict__ A_dev, const float* __restrict__ poses,
                                float* __restrict__ out, uint32_t count) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  float a[16], b[16], c[16];
  for (int i = 0; i < 16; ++i) a[i] = A_dev ? A_dev->m[i] : A.m[i];
  load_mat(poses, (int)t, b);
  mat4_mul<float>(a, b, c);
  for (int i = 0; i < 16; ++i) out[16 * (size_t)t + i] = c[i];
}

void launch_pose_products(const Launch& L, const Mat4& A, const Mat4* A_dev, const float* poses, float* out,
                          uint32_t count) {
  if (count == 0) return;
  {
    ScopedKernel sk(L, K_POSE_PRODUCTS);
    k_pose_products<<<(count + 127) / 128, 128, 0, L.stream>>>(A, A_dev, poses, out, count);
  }
}

// ------------------------------------------------------------------------------------------------------------
// K4 rasteriser
// ------------------------------------------------------------------------------------------------------------
struct RVert {  // the texture coordinates of quad corner i are (i & 1 ? 1 : -1, i & 2 ? 1 : -1), see corner_tx()
  long long X, Y;
  float z;
};

__device__ __forceinline__ long long floor_div256(long long a) { return a >> 8; }  // arithmetic shift = floor
__device__ __forceinline__ long long ceil_div256(long long a) { return -((-a) >> 8); }
__device__ __forceinline__ long long edge_fn(const RVert& P, const RVert& Q, long long X, long long Y) {
  return (Q.X - P.X) * (Y - P.Y) - (Q.Y - P.Y) * (X - P.X);
}

__device__ __forceinline__ bool edge_tie(const RVert& P, const RVert& Q) {  // rule for pixels exactly on an edge
  long long dx = Q.X - P.X, dy = Q.Y - P.Y;
  return dy > 0 || (dy == 0 && dx > 0);
}

// Triangle prepared for pixel-centre coverage tests with exact integer edge functions. The edge values at the first
// pixel centre of the bounding box and their per-pixel steps are int64 (no rounding anywhere):
// E(P + (256,0)) = E(P) - 256*dy, E(P + (0,256)) = E(P) + 256*dx.
struct TriSetup {
  long long eA, eB, eC;     // edge(B,C), edge(C,A), edge(A,B) at the first pixel centre
  long long sxA, sxB, sxC;  // step per pixel in x
  long long syA, syB, syC;  // step per pixel in y
  float farea;
  float zA, zB, zC;
  int i0, j0, ni, nj;       // bounding box origin and extent (inclusive), clamped to the image
  uint32_t ties;            // bit0..2: pixels exactly on edge A/B/C count as inside, bit3: B and C were swapped
  uint32_t valid;
};

__device__ __forceinline__ void tri_prepare(RVert A, RVert B, RVert C, int W, int H, TriSetup& t) {
  t.valid = 0;
  long long area = (B.X - A.X) * (C.Y - A.Y) - (B.Y - A.Y) * (C.X - A.X);
  if (area == 0) return;
  const bool swapped = area < 0;
  if (swapped) {
    RVert x = B;
    B = C;
    C = x;
    area = -area;
  }
  long long minX = min(A.X, min(B.X, C.X)), maxX = max(A.X, max(B.X, C.X));
  long long minY = min(A.Y, min(B.Y, C.Y)), maxY = max(A.Y, max(B.Y, C.Y));
  long long i0 = ceil_div256(minX - 128), i1 = floor_div256(maxX - 128);
  long long j0 = ceil_div256(minY - 128), j1 = floor_div256(maxY - 128);
  if (i0 < 0) i0 = 0;
  if (j0 < 0) j0 = 0;
  if (i1 > W - 1) i1 = W - 1;
  if (j1 > H - 1) j1 = H - 1;
  if (i0 > i1 || j0 > j1) return;
  t.farea = (float)area;
  const long long X0 = i0 * 256 + 128, Y0 = j0 * 256 + 128;
  t.eA = edge_fn(B, C, X0, Y0);
  t.eB = edge_fn(C, A, X0, Y0);
  t.eC = edge_fn(A, B, X0, Y0);
  t.sxA = -256 * (C.Y - B.Y); t.sxB = -256 * (A.Y - C.Y); t.sxC = -256 * (B.Y - A.Y);
  t.syA = 256 * (C.X - B.X); t.syB = 256 * (A.X - C.X); t.syC = 256 * (B.X - A.X);
  t.ties = (edge_tie(B, C) ? 1u : 0u) | (edge_tie(C, A) ? 2u : 0u) | (edge_tie(A, B) ? 4u : 0u) | (swapped ? 8u : 0u);
  t.zA = A.z; t.zB = B.z; t.zC = C.z;
  t.i0 = (int)i0; t.j0 = (int)j0; t.ni = (int)(i1 - i0); t.nj = (int)(j1 - j0);
  t.valid = 1;
}

constexpr int kRenderThreads = 256;
// A quad whose pixel bounding box is at most 12 x 5 is rasterised by its own lane (azimuth pixels are 2.5 x finer than
// elevation pixels at 64 x 2048, so the typical disc is ~6 x 2.5 pixels) ...
constexpr int kSmallW = 12, kSmallH = 5;
constexpr int kRoundItems = 4;   // box pixels a lane tests per round
constexpr int kFragBatch = 4;    // fragments a lane evaluates per batch (their depth keys are fetched together)
constexpr int kFragQueue = 32 * kRoundItems * 2;  // worst case: every tested pixel covered by both triangles
constexpr int kSmallSpan = 1 << 14;  // ... if its vertices lie within 64 pixels of the box origin: int32 edge functions are exact

// a surfel that passed every test of the vertex / geometry stage (render_surfels.geom:84-92)
struct Cand {
  float px, py, pz, nx, ny, nz, r, cx;
  uint32_t k, flags;  // flags: bit0 old-class surfel, bit1 new-class surfel, bit2 GL_LEQUAL composed mode
};

// render_surfels.geom:80-82: the quad's half axes r*u and r*v
__device__ __forceinline__ void quad_axes(const Cand& c, V3& ru, V3& rv) {
  const V3 nn = mk3(c.nx, c.ny, c.nz);
  V3 u = normalize3(mk3(nn.y - nn.z, -nn.x, nn.x));
  V3 v = normalize3(cross3(nn, u));
  ru = scale3(c.r, u);
  rv = scale3(c.r, v);
}

// render_surfels.geom:100-118: quad corner i = (pp -/+ ru) -/+ rv in window coordinates (1/256 pixel)
__device__ __forceinline__ RVert quad_corner(const KParams& kp, const Cand& c, V3 ru, V3 rv, int i) {
  const V3 pp = mk3(c.px, c.py, c.pz);
  const V3 h = (i & 1) ? add3(pp, ru) : sub3(pp, ru);
  const V3 corner = (i & 2) ? add3(h, rv) : sub3(h, rv);
  float x, y, z;
  project01(corner, kp.m_fov_up, kp.m_fov, kp.m_min_depth, kp.m_max_depth, x, y, z);
  if (c.cx - x > 0.5f) x += 1.0f;  // .geom:68
  if (x - c.cx > 0.5f) x -= 1.0f;  // .geom:69
  float xw = (0.5f * (2.0f * x - 1.0f) + 0.5f) * (float)kp.Wm;
  float yw = (0.5f * (2.0f * y - 1.0f) + 0.5f) * (float)kp.Hm;
  RVert q;
  q.z = 0.5f * (2.0f * z - 1.0f) + 0.5f;
  q.X = __float2ll_rn(xw * 256.0f);
  q.Y = __float2ll_rn(yw * 256.0f);
  return q;
}

// texture coordinates of quad corner i (render_surfels.geom:100-118)
__device__ __forceinline__ float corner_tx(int i) { return (i & 1) ? 1.0f : -1.0f; }
__device__ __forceinline__ float corner_ty(int i) { return (i & 2) ? 1.0f : -1.0f; }

// fragment stage (render_surfels.frag:19-33) + depth test + key update, shared by both rasterisers
__device__ __forceinline__ void emit_fragment(float tx, float ty, float z, size_t pix, uint32_t k, uint32_t flags,
                                              const RenderTargets& rt) {
  if (tx * tx + ty * ty > 1.0f) return;   // outside the disc
  if (!(z >= 0.0f && z <= 1.0f)) return;  // near / far clip
  unsigned long long d = (unsigned long long)depth24(z);
  const bool lequal = (flags & 4u) != 0;
  if (!lequal && d >= kDepthClear) return;  // GL_LESS against the cleared depth
  unsigned long long hi = d << 40;
  // keys only ever decrease: a (possibly stale) read that is already smaller proves the atomic cannot win, so most hidden
  // fragments never reach the L2 atomic unit
  if (flags & 1u) {  // old-class surfel
    if (rt.key_old) {
      unsigned long long key = hi | k;
      if (key < rt.key_old[pix]) atomicMin(rt.key_old + pix, key);
    }
    if (rt.key_comp) {  // old pass is drawn first: it wins depth ties under GL_LESS, loses them under GL_LEQUAL
      unsigned long long key = lequal ? (hi | (1ull << 32) | (unsigned long long)(0xffffffffu - k)) : (hi | k);
      if (key < rt.key_comp[pix]) atomicMin(rt.key_comp + pix, key);
    }
  }
  if (flags & 2u) {  // new-class surfel
    if (rt.key_new) {
      unsigned long long key = hi | k;
      if (key < rt.key_new[pix]) atomicMin(rt.key_new + pix, key);
    }
    if (rt.key_comp) {
      unsigned long long key = lequal ? (hi | (unsigned long long)(0xffffffffu - k)) : (hi | (1ull << 32) | k);
      if (key < rt.key_comp[pix]) atomicMin(rt.key_comp + pix, key);
    }
  }
}

// one triangle of a large quad, rasterised by a whole warp: the lanes stride over its bounding-box pixels (int64 edges)
// (corners tri, tri + 1, tri + 2 of the quad, B and C exchanged if the orientation fix swapped them)
__device__ __forceinline__ void raster_big_tri(const KParams& kp, const TriSetup& t, int tri, uint32_t k, uint32_t flags,
                                               const RenderTargets& rt, int lane) {
  if (!t.valid) return;
  const int wd = t.ni + 1, total = wd * (t.nj + 1);
  const bool tieA = t.ties & 1u, tieB = t.ties & 2u, tieC = t.ties & 4u;
  const int cA = tri, cB = (t.ties & 8u) ? tri + 2 : tri + 1, cC = (t.ties & 8u) ? tri + 1 : tri + 2;
  const float txA = corner_tx(cA), txB = corner_tx(cB), txC = corner_tx(cC);
  const float tyA = corner_ty(cA), tyB = corner_ty(cB), tyC = corner_ty(cC);
  for (int item = lane; item < total; item += 32) {
    const int dj = item / wd, di = item - dj * wd;
    const long long wA = t.eA + (long long)di * t.sxA + (long long)dj * t.syA;
    const long long wB = t.eB + (long long)di * t.sxB + (long long)dj * t.syB;
    const long long wC = t.eC + (long long)di * t.sxC + (long long)dj * t.syC;
    const bool in = (wA > 0 || (wA == 0 && tieA)) && (wB > 0 || (wB == 0 && tieB)) && (wC > 0 || (wC == 0 && tieC));
    if (!in) continue;
    float fB = (float)wB / t.farea, fC = (float)wC / t.farea;
    float fA = (1.0f - fB) - fC;
    float tx = (fA * txA + fB * txB) + fC * txC;
    float ty = (fA * tyA + fB * tyB) + fC * tyC;
    float z = (fA * t.zA + fB * t.zB) + fC * t.zC;
    emit_fragment(tx, ty, z, (size_t)(t.j0 + dj) * kp.Wm + (size_t)(t.i0 + di), k, flags, rt);
  }
}

// corner i of the quad, held by lanes i, i + 4, ... of the warp
__device__ __forceinline__ RVert shfl_corner(const RVert& mine, int i) {
  RVert q;
  q.X = __shfl_sync(0xffffffffu, mine.X, i);
  q.Y = __shfl_sync(0xffffffffu, mine.Y, i);
  q.z = __shfl_sync(0xffffffffu, mine.z, i);
  return q;
}

// a large quad (warp-uniform): every lane projects one corner, and each triangle collects its three corners by shuffles,
// so that no corner array stays live next to a triangle's set-up. The set-up itself goes to `st`, the warp's slot in
// shared memory, and the pixel loop reads it from there: held in registers next to the fragment evaluation it needed
// ~76 registers and spilled at the 64 that 4 blocks per SM allow.
__device__ __forceinline__ void raster_big(const KParams& kp, const Cand& c, const RenderTargets& rt, int lane,
                                           TriSetup& st) {
  V3 ru, rv;
  quad_axes(c, ru, rv);
  const RVert mine = quad_corner(kp, c, ru, rv, lane & 3);
#pragma unroll 1
  for (int tri = 0; tri < 2; ++tri) {
    const RVert A = shfl_corner(mine, tri), B = shfl_corner(mine, tri + 1), C = shfl_corner(mine, tri + 2);
    __syncwarp();  // every lane is done with the previous set-up
    if (lane == 0) tri_prepare(A, B, C, kp.Wm, kp.Hm, st);
    __syncwarp();
    raster_big_tri(kp, st, tri, c.k, c.flags, rt, lane);
  }
}

// ---- the quad records of a block, structure-of-arrays in shared memory (lanes read different quads) ----
struct QuadStore {
  int e[2][3][kRenderThreads];   // per triangle: edge functions at the first pixel centre of the quad's box
  int sx[2][3][kRenderThreads];  // per-pixel steps in x
  int sy[2][3][kRenderThreads];  // per-pixel steps in y
  float farea[2][kRenderThreads];
  float z[4][kRenderThreads];    // window depth of the four corners
  uint32_t box[kRenderThreads];   // i0 | j0 << 16
  uint32_t meta[kRenderThreads];  // ni | nj << 8 | per triangle (ties 3 bits, swapped 1 bit, valid 1 bit) << 16 / << 21 | flags << 26
  uint32_t k[kRenderThreads];
  int prefix[kRenderThreads + 1];  // exclusive prefix of the box pixel counts (0 for large / empty quads)
};

__device__ __forceinline__ int edge32(int Px, int Py, int Qx, int Qy) {  // edge_fn(P, Q, X0, Y0), P and Q relative to (X0, Y0)
  return (Qx - Px) * (0 - Py) - (Qy - Py) * (0 - Px);
}
__device__ __forceinline__ bool tie32(int Px, int Py, int Qx, int Qy) {
  int dx = Qx - Px, dy = Qy - Py;
  return dy > 0 || (dy == 0 && dx > 0);
}
// One triangle (corners A, B, C) of a small quad, everything relative to the quad's first pixel centre (X0, Y0): all
// magnitudes stay below 2^14 + 2^10, so the int32 edge functions, their steps and the area equal the int64 ones of
// tri_prepare() bit for bit. The set-up goes straight to slot `slot` of Q (so that only one triangle's is ever live);
// returns the triangle's meta bits, ties (3) | swapped (1) | valid (1), and 0 for a degenerate triangle, which stores
// nothing. Phase 2 takes the corner depths and texture coordinates from the swapped bit.
__device__ __forceinline__ uint32_t tri_small_store(QuadStore& Q, int slot, int tri, int Ax, int Ay, int Bx, int By,
                                                    int Cx, int Cy) {
  int area = (Bx - Ax) * (Cy - Ay) - (By - Ay) * (Cx - Ax);
  if (area == 0) return 0u;
  uint32_t swapped = 0u;
  if (area < 0) {  // same orientation fix as tri_prepare(): swap B and C
    int ti = Bx; Bx = Cx; Cx = ti;
    ti = By; By = Cy; Cy = ti;
    area = -area;
    swapped = 8u;
  }
  Q.farea[tri][slot] = (float)area;
  Q.e[tri][0][slot] = edge32(Bx, By, Cx, Cy);
  Q.e[tri][1][slot] = edge32(Cx, Cy, Ax, Ay);
  Q.e[tri][2][slot] = edge32(Ax, Ay, Bx, By);
  Q.sx[tri][0][slot] = -256 * (Cy - By); Q.sx[tri][1][slot] = -256 * (Ay - Cy); Q.sx[tri][2][slot] = -256 * (By - Ay);
  Q.sy[tri][0][slot] = 256 * (Cx - Bx); Q.sy[tri][1][slot] = 256 * (Ax - Cx); Q.sy[tri][2][slot] = 256 * (Bx - Ax);
  return (tie32(Bx, By, Cx, Cy) ? 1u : 0u) | (tie32(Cx, Cy, Ax, Ay) ? 2u : 0u) | (tie32(Ax, Ay, Bx, By) ? 4u : 0u) |
         swapped | 16u;
}

// K6a, gen_indexmap.vert:62-81 for one visible surfel k whose centre projects to (x, y, z) under the data image's
// parameters: its depth key and data pixel, false if it lands on none (k_index_scatter, and k_render_scatter<., true>
// for the pipeline; both then keep the smaller key with a stale pre-read and atomicMin, as emit_fragment does)
__device__ __forceinline__ bool index_key(const KParams& kp, float x, float y, float z, uint32_t k,
                                          unsigned long long& key, size_t& pix) {
  float fx = floorf(x * (float)kp.W), fy = floorf(y * (float)kp.H);
  if (!(fx >= 0.0f && fx < (float)kp.W && fy >= 0.0f && fy < (float)kp.H)) return false;
  float zn = 2.0f * z - 1.0f;
  if (!(zn >= -1.0f && zn <= 1.0f)) return false;
  uint32_t d24 = depth24(0.5f * zn + 0.5f);
  if (d24 >= kDepthClear) return false;
  pix = (size_t)(int)fy * kp.W + (size_t)(int)fx;
  key = ((unsigned long long)d24 << 32) | (unsigned long long)k;
  return true;
}

// render_surfels.vert:42-54 + .geom:76-122 + rasterisation + depth test for every surfel of the map.
//  stage A/B (one thread per surfel): confidence / age-class tests on two lanes, then transform, visibility and the
//    projection of the centre -- about half of the map drops out here;
//  compaction: the survivors are packed densely through shared memory, so that
//  stage C (corner projections + triangle set-up) runs on full warps and leaves one lean record per quad in shared memory;
//  rasterisation: the box pixels of ALL quads of the block form one flattened list that the 256 threads share evenly
//    (contiguous chunks: one binary search per thread, then a walk) -- quads differ by an order of magnitude in size
//    (a disc is ~6 x 2.5 pixels at 64 x 2048 but dozens of pixels wide from close by), and per-fragment work is a chain
//    of dependent L2 round trips, so every lane of every warp has to stay busy. Edge functions are int32, exact because a
//    "small" quad (box <= 12 x 5 pixels, vertices within 64 pixels) keeps every product below 2^31; the rare larger
//    quads are rasterised by whole warps with int64 edge functions.
//  (Round 1 stored int64 set-ups of every triangle per warp and ran stage C on half-empty warps: 15 of 32 lanes active.)
// kIndex: the render also writes the map update's index keys (K6a, index_key()) for every live surfel, see IndexFuse.
template <int kMinBlocks, bool kIndex>
__global__ void __launch_bounds__(kRenderThreads, kMinBlocks) k_render_scatter(KParams kp, SurfelPlanes s, const uint32_t* __restrict__ n_dev,
                                                                               const uint8_t* __restrict__ live,
                                                                               const float* __restrict__ Mtab, float conf_thr, int t_thr,
                                                                               int emit_old, int emit_new, int lequal, RenderTargets rt,
                                                                               IndexFuse ix) {
  __shared__ QuadStore Q;
  __shared__ float c_f[8][kRenderThreads];
  __shared__ uint32_t c_flags[kRenderThreads];
  __shared__ int s_warp_cnt[kRenderThreads / 32];
  __shared__ int s_nbig;
  __shared__ uint16_t s_big[kRenderThreads];
  // per warp: the fragment queue of the small quads, then the triangle set-up of its large quads (raster_big)
  __shared__ __align__(8) uint32_t s_fq[kRenderThreads / 32][kFragQueue];
  static_assert(sizeof(TriSetup) <= sizeof(s_fq[0]) && sizeof(s_fq[0]) % 8 == 0, "a warp's queue holds a TriSetup");
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_nbig = 0;
  const uint32_t k = blockIdx.x * blockDim.x + tid;
  bool alive = k < *n_dev;
  float4 p0, p1, p2;
  bool is_old = false, is_new = false, indexed = false;
  if (alive) {
    // the liveness byte is loaded together with the first two lanes: gating the lanes on it costs an L2 round trip
    const bool lv = live[k] != 0;
    p2 = __ldg(s.p2 + k);
    p1 = __ldg(s.p1 + k);
    if (kIndex) {  // the index map needs every live surfel: p0 joins the first loads instead of waiting for the tests
      p0 = __ldg(s.p0 + k);
      indexed = lv && *ix.fallback == 0;
    }
    alive = lv && (!kp.use_stability || p1.w > conf_thr);  // .geom:87 (cheap test first)
  }
  if (alive) {
    int creation = (int)p2.w, ts = (int)__float_as_uint(p2.x);
    is_old = emit_old && (creation < t_thr);                  // .geom:90
    is_new = emit_new && (creation >= t_thr || ts >= t_thr);  // .geom:91
    alive = is_old || is_new;
  }
  Cand c;
  if (alive || indexed) {
    if (!kIndex) p0 = __ldg(s.p0 + k);
    float M[16];
    load_mat(Mtab, pose_index(p2.w), M);
    V3 pp = xform_point(M, mk3(p0.x, p0.y, p0.z));
    V3 nn = xform_dir(M, mk3(p1.x, p1.y, p1.z));
    bool visible = dot3(nn, divs3(neg3(pp), len3(pp))) > 0.01f;  // .geom:84, the same test as gen_indexmap.vert
    float cx, cy, cz;
    project01(pp, kp.m_fov_up, kp.m_fov, kp.m_min_depth, kp.m_max_depth, cx, cy, cz);
    if (kIndex && indexed && visible) {
      float x = cx, y = cy, z = cz;
      if (!ix.same_projection) project01(pp, kp.fov_up, kp.fov, kp.min_depth, kp.max_depth, x, y, z);
      unsigned long long key;
      size_t pix;
      if (index_key(kp, x, y, z, k, key, pix) && key < ix.keys[pix]) atomicMin(ix.keys + pix, key);
    }
    alive = alive && visible && cx >= 0.0f && cy >= 0.0f && cz >= 0.0f && cx < 1.0f && cy < 1.0f && cz < 1.0f;
    c.px = pp.x; c.py = pp.y; c.pz = pp.z; c.nx = nn.x; c.ny = nn.y; c.nz = nn.z; c.r = p0.w; c.cx = cx;
  }
  // ---- dense packing of the survivors (their order inside the block is irrelevant: visibility is decided by the keys) ----
  const unsigned ballot = __ballot_sync(0xffffffffu, alive);
  if (lane == 0) s_warp_cnt[warp] = __popc(ballot);
  __syncthreads();
  int base = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kRenderThreads / 32; ++w) {
    const int cnt = s_warp_cnt[w];
    if (w < warp) base += cnt;
    total += cnt;
  }
  if (total == 0) return;
  if (alive) {
    const int slot = base + __popc(ballot & ((1u << lane) - 1u));
    c_f[0][slot] = c.px; c_f[1][slot] = c.py; c_f[2][slot] = c.pz; c_f[3][slot] = c.nx;
    c_f[4][slot] = c.ny; c_f[5][slot] = c.nz; c_f[6][slot] = c.r; c_f[7][slot] = c.cx;
    Q.k[slot] = k;
    c_flags[slot] = (is_old ? 1u : 0u) | (is_new ? 2u : 0u) | (lequal ? 4u : 0u);
  }
  __syncthreads();
  // ---- stage C on dense lanes: one quad record per survivor ----
  int npix = 0;
  if (tid < total) {
    c.px = c_f[0][tid]; c.py = c_f[1][tid]; c.pz = c_f[2][tid]; c.nx = c_f[3][tid];
    c.ny = c_f[4][tid]; c.nz = c_f[5][tid]; c.r = c_f[6][tid]; c.cx = c_f[7][tid];
    V3 ru, rv;
    quad_axes(c, ru, rv);
    RVert q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = quad_corner(kp, c, ru, rv, i);
    // pixel bounding box of the quad (union of the boxes of its two triangles), clamped to the image
    long long minX = min(min(q[0].X, q[1].X), min(q[2].X, q[3].X)), maxX = max(max(q[0].X, q[1].X), max(q[2].X, q[3].X));
    long long minY = min(min(q[0].Y, q[1].Y), min(q[2].Y, q[3].Y)), maxY = max(max(q[0].Y, q[1].Y), max(q[2].Y, q[3].Y));
    long long i0 = ceil_div256(minX - 128), i1 = floor_div256(maxX - 128);
    long long j0 = ceil_div256(minY - 128), j1 = floor_div256(maxY - 128);
    if (i0 < 0) i0 = 0;
    if (j0 < 0) j0 = 0;
    if (i1 > kp.Wm - 1) i1 = kp.Wm - 1;
    if (j1 > kp.Hm - 1) j1 = kp.Hm - 1;
    if (i0 <= i1 && j0 <= j1) {  // otherwise the quad covers no pixel centre
      const long long X0 = i0 * 256 + 128, Y0 = j0 * 256 + 128;
      const int ni = (int)(i1 - i0), nj = (int)(j1 - j0);
      bool small = ni < kSmallW && nj < kSmallH;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        long long dx = q[i].X - X0, dy = q[i].Y - Y0;
        small = small && dx > -kSmallSpan && dx < kSmallSpan && dy > -kSmallSpan && dy < kSmallSpan;
      }
      if (small) {
        int rx[4], ry[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          rx[i] = (int)(q[i].X - X0);
          ry[i] = (int)(q[i].Y - Y0);
        }
        const uint32_t m0 = tri_small_store(Q, tid, 0, rx[0], ry[0], rx[1], ry[1], rx[2], ry[2]);
        const uint32_t m1 = tri_small_store(Q, tid, 1, rx[1], ry[1], rx[2], ry[2], rx[3], ry[3]);
        if (m0 | m1) {
          Q.z[0][tid] = q[0].z; Q.z[1][tid] = q[1].z; Q.z[2][tid] = q[2].z; Q.z[3][tid] = q[3].z;
          Q.box[tid] = (uint32_t)i0 | ((uint32_t)j0 << 16);
          Q.meta[tid] = (uint32_t)ni | ((uint32_t)nj << 8) | (m0 << 16) | (m1 << 21) | (c_flags[tid] << 26);
          npix = (ni + 1) * (nj + 1);
        }
      } else {
        s_big[atomicAdd(&s_nbig, 1)] = (uint16_t)tid;
      }
    }
  }
  // ---- exclusive prefix of the pixel counts over the 256 slots ----
  int incl = npix;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  __syncthreads();  // everybody is done with s_warp_cnt (read above) before it is reused
  if (lane == 31) s_warp_cnt[warp] = incl;
  __syncthreads();
  int wbase = 0, T = 0;
#pragma unroll
  for (int w = 0; w < kRenderThreads / 32; ++w) {
    const int cnt = s_warp_cnt[w];
    if (w < warp) wbase += cnt;
    T += cnt;
  }
  Q.prefix[tid + 1] = wbase + incl;
  if (tid == 0) Q.prefix[0] = 0;
  __syncthreads();
  // ---- balanced rasterisation, two phases per round ----
  // Thread t owns the flattened box pixels [t*ch, (t+1)*ch). Coverage is ~50 % and a fragment costs ~5x a coverage test
  // plus a depth-key round trip to L2, so the phases are separated:
  //  phase 1: every lane runs the integer coverage tests of up to kRoundItems of its pixels and pushes the covered
  //           (quad, pixel, triangle) triples into the warp's queue in shared memory (ballot-ordered);
  //  phase 2: the lanes share the queue evenly -- all of them busy -- and evaluate fragments in batches: the depth keys of
  //           a batch are loaded first (independent loads in flight while the barycentric divides run), then compared.
  // (ncu on the one-phase version: 26 % of the stall samples on the key load, 12.6 of 32 lanes active.)
  if (T > 0) {
    uint32_t* fq = s_fq[warp];
    const int ch = (T + kRenderThreads - 1) / kRenderThreads;
    int item = tid * ch;
    const int end = min(item + ch, T);
    int slot = 0, wd = 1, cnt = 0, first = 0, di = 0, dj = 0;
    uint32_t meta = 0;
    bool have_owner = false;
    if (item < end) {
      int lo = 0, hi = kRenderThreads;  // largest slot with prefix[slot] <= item
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (Q.prefix[mid] <= item) lo = mid; else hi = mid;
      }
      slot = lo;
    }
    // plain targets: one key image per surfel class and no composed image -> the key can be fetched ahead of the fragment
    const bool plain = rt.key_comp == nullptr && !lequal;
    while (__any_sync(0xffffffffu, item < end)) {
      int qn = 0;  // queue length, warp-uniform
#pragma unroll 1
      for (int r = 0; r < kRoundItems; ++r) {
        const bool have = item < end;
        if (have && !have_owner) {  // enter the quad that owns `item`
          for (;;) {
            first = Q.prefix[slot];
            cnt = Q.prefix[slot + 1] - first;
            if (cnt != 0) break;
            ++slot;
          }
          meta = Q.meta[slot];
          wd = (int)(meta & 255u) + 1;
          const int local = item - first;
          dj = local / wd;
          di = local - dj * wd;
          have_owner = true;
        }
#pragma unroll
        for (int tri = 0; tri < 2; ++tri) {
          bool in = false;
          if (have) {
            const uint32_t m = (meta >> (16 + 5 * tri)) & 31u;  // ties (3) | swapped (1) | valid (1)
            if (m & 16u) {
              const int wA = Q.e[tri][0][slot] + di * Q.sx[tri][0][slot] + dj * Q.sy[tri][0][slot];
              const int wB = Q.e[tri][1][slot] + di * Q.sx[tri][1][slot] + dj * Q.sy[tri][1][slot];
              const int wC = Q.e[tri][2][slot] + di * Q.sx[tri][2][slot] + dj * Q.sy[tri][2][slot];
              in = (wA > 0 || (wA == 0 && (m & 1u))) && (wB > 0 || (wB == 0 && (m & 2u))) && (wC > 0 || (wC == 0 && (m & 4u)));
            }
          }
          const unsigned bm = __ballot_sync(0xffffffffu, in);
          if (in) fq[qn + __popc(bm & ((1u << lane) - 1u))] = (uint32_t)slot | ((uint32_t)di << 8) | ((uint32_t)dj << 12) | ((uint32_t)tri << 15);
          qn += __popc(bm);
        }
        if (have) {
          ++item;
          if (++di == wd) {
            di = 0;
            ++dj;
          }
          if (item - first == cnt) {  // leaving this quad
            have_owner = false;
            ++slot;
          }
        }
      }
      __syncwarp();
      // phase 2
      for (int i0q = 0; i0q < qn; i0q += 32 * kFragBatch) {
        // per fragment only the queue entry, the pixel and the fetched key stay live; the key image is chosen again from
        // the surfel class when it is used. The pixel index fits 32 bits: Q.box holds i0 and j0 in 16 bits each, and
        // sb_create refuses model images with a side over 65536 (check_params), so the index is at most 2^32 - 1.
        uint32_t ent[kFragBatch], pixs[kFragBatch];
        unsigned long long cur[kFragBatch];
#pragma unroll
        for (int b2 = 0; b2 < kFragBatch; ++b2) {
          const int i = i0q + 32 * b2 + lane;
          ent[b2] = i < qn ? fq[i] : 0xffffffffu;
          cur[b2] = 0ull;
          pixs[b2] = 0u;
          if (ent[b2] != 0xffffffffu) {
            const int sl = (int)(ent[b2] & 255u);
            const uint32_t box = Q.box[sl];
            pixs[b2] = ((box >> 16) + ((ent[b2] >> 12) & 7u)) * (uint32_t)kp.Wm + ((box & 0xffffu) + ((ent[b2] >> 8) & 15u));
            const uint32_t cls = (Q.meta[sl] >> 26) & 3u;  // 1 old, 2 new, 3 both (an old surfel re-observed recently)
            if (plain && cls != 3u) {
              const unsigned long long* img = (cls & 1u) ? rt.key_old : rt.key_new;
              if (img) cur[b2] = img[pixs[b2]];
            }
          }
        }
#pragma unroll
        for (int b2 = 0; b2 < kFragBatch; ++b2) {
          if (ent[b2] == 0xffffffffu) continue;
          const int sl = (int)(ent[b2] & 255u), fdi = (int)((ent[b2] >> 8) & 15u), fdj = (int)((ent[b2] >> 12) & 7u);
          const int tri = (int)((ent[b2] >> 15) & 1u);
          const uint32_t mt = Q.meta[sl];
          const uint32_t m = (mt >> (16 + 5 * tri)) & 31u;
          const int wB = Q.e[tri][1][sl] + fdi * Q.sx[tri][1][sl] + fdj * Q.sy[tri][1][sl];
          const int wC = Q.e[tri][2][sl] + fdi * Q.sx[tri][2][sl] + fdj * Q.sy[tri][2][sl];
          // corners of this triangle: (tri, tri+1, tri+2), B and C exchanged if the orientation fix swapped them
          const int cA = tri, cB = (m & 8u) ? tri + 2 : tri + 1, cC = (m & 8u) ? tri + 1 : tri + 2;
          const float farea = Q.farea[tri][sl];
          const float fB = (float)wB / farea, fC = (float)wC / farea;
          const float fA = (1.0f - fB) - fC;
          const float txA = corner_tx(cA), txB = corner_tx(cB), txC = corner_tx(cC);
          const float tyA = corner_ty(cA), tyB = corner_ty(cB), tyC = corner_ty(cC);
          const float tx = (fA * txA + fB * txB) + fC * txC;
          const float ty = (fA * tyA + fB * tyB) + fC * tyC;
          const float z = (fA * Q.z[cA][sl] + fB * Q.z[cB][sl]) + fC * Q.z[cC][sl];
          const uint32_t cls = (mt >> 26) & 3u;
          if (plain && cls != 3u) {
            unsigned long long* img = (cls & 1u) ? rt.key_old : rt.key_new;
            if (!img) continue;
            if (tx * tx + ty * ty > 1.0f) continue;   // outside the disc (render_surfels.frag:22-28)
            if (!(z >= 0.0f && z <= 1.0f)) continue;  // near / far clip
            const unsigned long long d = (unsigned long long)depth24(z);
            if (d >= kDepthClear) continue;           // GL_LESS against the cleared depth
            const unsigned long long key = (d << 40) | Q.k[sl];
            if (key < cur[b2]) atomicMin(img + pixs[b2], key);
          } else {
            emit_fragment(tx, ty, z, pixs[b2], Q.k[sl], mt >> 26, rt);
          }
        }
      }
      __syncwarp();
    }
  }
  // ---- large quads: one warp each ----
  const int nbig = s_nbig;
  for (int b = warp; b < nbig; b += kRenderThreads / 32) {
    const int slot = s_big[b];
    Cand cb;
    cb.px = c_f[0][slot]; cb.py = c_f[1][slot]; cb.pz = c_f[2][slot]; cb.nx = c_f[3][slot];
    cb.ny = c_f[4][slot]; cb.nz = c_f[5][slot]; cb.r = c_f[6][slot]; cb.cx = c_f[7][slot];
    cb.k = Q.k[slot]; cb.flags = c_flags[slot];
    raster_big(kp, cb, rt, lane, *reinterpret_cast<TriSetup*>(s_fq[warp]));
  }
}

void launch_render_scatter(const Launch& L, const KParams& kp, SurfelPlanes s, const uint32_t* n_dev, const uint8_t* live,
                           uint32_t n_upper, const float* M, float conf_thr, int t_thr, int emit_old, int emit_new,
                           int lequal, RenderTargets t, const IndexFuse* index) {
  if (n_upper == 0) return;
  {
    ScopedKernel sk(L, K_RENDER_SCATTER);
    const unsigned grid = (n_upper + kRenderThreads - 1) / kRenderThreads;
    // 4 resident blocks per SM (64 registers, no local memory, 46.6 KB shared memory): the kernel is bound by
    // instruction issue and dependent L2 round trips (renderbench.py times both instances)
    if (index)
      k_render_scatter<4, true><<<grid, kRenderThreads, 0, L.stream>>>(kp, s, n_dev, live, M, conf_thr, t_thr, emit_old,
                                                                       emit_new, lequal, t, *index);
    else
      k_render_scatter<4, false><<<grid, kRenderThreads, 0, L.stream>>>(kp, s, n_dev, live, M, conf_thr, t_thr, emit_old,
                                                                        emit_new, lequal, t, IndexFuse{});
  }
}

struct Px {
  float4 v, n, s;
};

__device__ __forceinline__ Px resolve_px(const SurfelPlanes& s, unsigned long long key, const float* __restrict__ M_old,
                                         const float* __restrict__ M_new, int fixed_pass, int lequal, bool need_semantic) {
  Px o;
  o.v = o.n = o.s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (key == ~0ull) return o;
  uint32_t low = (uint32_t)(key & 0xffffffffull);
  int pass = (int)((key >> 32) & 1ull);
  uint32_t k = low;
  if (lequal && fixed_pass < 0) {
    k = 0xffffffffu - low;
    pass = 1 - pass;
  }
  if (fixed_pass >= 0) pass = fixed_pass;
  float4 p0 = __ldg(s.p0 + k), p1 = __ldg(s.p1 + k), p2 = __ldg(s.p2 + k);
  float M[16];
  load_mat(pass ? M_new : M_old, pose_index(p2.w), M);
  V3 pp = xform_point(M, mk3(p0.x, p0.y, p0.z));
  V3 nn = xform_dir(M, mk3(p1.x, p1.y, p1.z));
  o.v = make_float4(pp.x, pp.y, pp.z, 1.0f);  // render_surfels.frag:30, .geom:95-97 (flat: surfel centre)
  o.n = make_float4(nn.x, nn.y, nn.z, 1.0f);
  if (need_semantic) o.s = __ldg(s.p3 + k);  // Q4: the single-view renderings keep the previous semantic image
  return o;
}

// resolve the key images into vertex / normal / semantic maps; optionally fuses render_compose.frag:26-48
__global__ void __launch_bounds__(kThreads) k_render_resolve(KParams kp, SurfelPlanes s, const float* __restrict__ M_old,
                                                            const float* __restrict__ M_new, RenderTargets t,
                                                            FrameDev f_old, FrameDev f_new, FrameDev f_comp,
                                                            FrameDev f_out, FrameDev f_copy, int keep_semantic, int lequal) {
  int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= kp.Wm * kp.Hm) return;
  // every key image that is read here is cleared again ("consume and clear"): no separate fill before the next view
  Px po, pn;
  unsigned long long ko_raw = ~0ull, kn_raw = ~0ull;
  if (t.key_old) {
    ko_raw = t.key_old[pix];
    t.key_old[pix] = ~0ull;
    po = resolve_px(s, ko_raw, M_old, M_new, 0, 0, !keep_semantic);
    f_old.vertex[pix] = po.v;
    f_old.normal[pix] = po.n;
    if (!keep_semantic) f_old.semantic[pix] = po.s;
  }
  if (t.key_new) {
    kn_raw = t.key_new[pix];
    t.key_new[pix] = ~0ull;
    pn = resolve_px(s, kn_raw, M_old, M_new, 1, 0, !keep_semantic);
    f_new.vertex[pix] = pn.v;
    f_new.normal[pix] = pn.n;
    if (!keep_semantic) f_new.semantic[pix] = pn.s;
    if (f_copy.vertex) {  // lastModelFrame_->copy(*map_->newMapFrame()), SurfelMapping.cpp:407, fused into this pass
      f_copy.vertex[pix] = pn.v;
      f_copy.normal[pix] = pn.n;
      f_copy.semantic[pix] = keep_semantic ? f_new.semantic[pix] : pn.s;
    }
  }
  if (f_comp.vertex && !t.key_comp && t.key_old && t.key_new) {
    // GL_LESS, old pass drawn before the new pass on an uncleared buffer (SurfelMap.cpp:893-906): the winner of the
    // union of both passes is the smaller of the two per-pass winners, depth first, then pass, then surfel index
    unsigned long long ko = ko_raw, kn = kn_raw;
    if (kn != ~0ull) kn |= (1ull << 32);
    Px pc = resolve_px(s, ko < kn ? ko : kn, M_old, M_new, -1, 0, !keep_semantic);
    f_comp.vertex[pix] = pc.v;
    f_comp.normal[pix] = pc.n;
    if (!keep_semantic) f_comp.semantic[pix] = pc.s;
  }
  if (t.key_comp) {
    unsigned long long kc = t.key_comp[pix];
    t.key_comp[pix] = ~0ull;
    Px pc = resolve_px(s, kc, M_old, M_new, -1, lequal, !keep_semantic);
    f_comp.vertex[pix] = pc.v;
    f_comp.normal[pix] = pc.n;
    if (!keep_semantic) f_comp.semantic[pix] = pc.s;
  }
  if (f_out.vertex && t.key_old && t.key_new) {  // render_compose.frag
    bool valid = po.v.w > 0.5f && po.n.w > 0.5f;
    bool new_valid = pn.v.w > 0.5f && pn.n.w > 0.5f;
    Px o = pn;
    if (!new_valid && valid &&
        (pn.v.w < 0.5f ||
         len3(sub3(mk3(pn.v.x, pn.v.y, pn.v.z), mk3(po.v.x, po.v.y, po.v.z))) < kp.max_loop_closure_distance))
      o = po;
    f_out.vertex[pix] = o.v;
    f_out.normal[pix] = o.n;
    f_out.semantic[pix] = o.s;
  }
}

void launch_render_resolve(const Launch& L, const KParams& kp, SurfelPlanes s, const float* M_old, const float* M_new,
                           RenderTargets t, FrameDev f_old, FrameDev f_new, FrameDev f_comp, FrameDev f_out,
                           FrameDev f_copy, int keep_semantic, int lequal) {
  int P = kp.Wm * kp.Hm;
  {
    ScopedKernel sk(L, K_RENDER_RESOLVE);
    k_render_resolve<<<(P + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(kp, s, M_old, M_new, t, f_old, f_new,
                                                                            f_comp, f_out, f_copy, keep_semantic, lequal);
  }
}

// ------------------------------------------------------------------------------------------------------------
// K6a: gen_indexmap.vert:62-81 -- nearest visible surfel per data pixel
// ------------------------------------------------------------------------------------------------------------
// gate != null: nothing to do unless *gate is set (the track-loss flag of a scan whose post-ICP render was to write the
// keys, see IndexFuse); the grid is then small and strides over the map.
constexpr uint32_t kIndexRepairBlocks = 512;
__global__ void __launch_bounds__(kThreads) k_index_scatter(KParams kp, SurfelPlanes s, const uint32_t* __restrict__ n_dev,
                                                           const uint8_t* __restrict__ live, const float* __restrict__ Mtab,
                                                           unsigned long long* __restrict__ keys, const int* __restrict__ gate) {
  if (gate && *gate == 0) return;
  const uint32_t n = *n_dev;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const bool lv = live[k] != 0;  // (loaded with the lanes, as in k_render_scatter)
    float4 p0 = __ldg(s.p0 + k), p1 = __ldg(s.p1 + k), p2 = __ldg(s.p2 + k);
    if (!lv) continue;
    float M[16];
    load_mat(Mtab, pose_index(p2.w), M);
    V3 v = xform_point(M, mk3(p0.x, p0.y, p0.z));
    V3 nrm = xform_dir(M, mk3(p1.x, p1.y, p1.z));
    if (!(dot3(nrm, divs3(neg3(v), len3(v))) > 0.01f)) continue;
    float x, y, z;
    project01(v, kp.fov_up, kp.fov, kp.min_depth, kp.max_depth, x, y, z);
    unsigned long long key;
    size_t pix;
    if (index_key(kp, x, y, z, k, key, pix) && key < keys[pix]) atomicMin(keys + pix, key);
  }
}

void launch_index_scatter(const Launch& L, const KParams& kp, SurfelPlanes s, const uint32_t* n_dev, const uint8_t* live,
                          uint32_t n_upper, const float* M, unsigned long long* keys, const int* gate) {
  if (n_upper == 0) return;
  {
    ScopedKernel sk(L, K_INDEX_SCATTER);
    // gated: a grid that costs next to nothing when the gate is clear and still covers the map when it is set
    const uint32_t blocks = (n_upper + kThreads - 1) / kThreads;
    const uint32_t grid = gate && blocks > kIndexRepairBlocks ? kIndexRepairBlocks : blocks;
    k_index_scatter<<<grid, kThreads, 0, L.stream>>>(kp, s, n_dev, live, M, keys, gate);
  }
}

// K6b: init_radiusConf.vert:41-68
// (+ re-arms the index-map key image and clears the "measurement integrated" flags of the pixel: the prologue of a
// stand-alone map update; in the per-scan pipeline the tiled preprocessing pass has already done all three)
__global__ void __launch_bounds__(kThreads) k_radius(KParams kp, FrameDev f, float4* __restrict__ radius_map,
                                                    unsigned long long* __restrict__ index_keys,
                                                    uint8_t* __restrict__ integrated, uint32_t* __restrict__ group_counts) {
  int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= kp.W * kp.H) return;
  index_keys[pix] = ~0ull;
  integrated[pix] = 0;
  // all kGroupCounts totals, also on an image of fewer pixels: the compaction reads every group the map spans
  for (int g = pix; g < kGroupCounts; g += kp.W * kp.H) group_counts[g] = 0;
  float4 V = __ldg(f.vertex + pix), N = __ldg(f.normal + pix);
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  V3 v = mk3(V.x, V.y, V.z), n = mk3(N.x, N.y, N.z);
  float d = len3(v);
  V3 view_dir = divs3(neg3(v), d);
  float angle = dot3(n, view_dir);
  if (V.w > 0.5f && N.w > 0.5f && angle > kp.radconf_angle_thresh) {
    float c = angle < 0.5f ? 0.5f : (angle > 1.0f ? 1.0f : angle);
    float radius = ((1.41f * d) * kp.pixel_size) / c;
    float lo = radius > kp.min_radius ? radius : kp.min_radius;
    radius = lo < kp.max_radius ? lo : kp.max_radius;
    o.x = radius;
    o.w = 1.0f;  // Q3: the confidence channel stays 0
  }
  radius_map[pix] = o;
}

void launch_radius(const Launch& L, const KParams& kp, FrameDev frame, float4* radius_map, unsigned long long* index_keys,
                   uint8_t* integrated, uint32_t* group_counts) {
  int P = kp.W * kp.H;
  {
    ScopedKernel sk(L, K_RADIUS);
    k_radius<<<(P + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(kp, frame, radius_map, index_keys, integrated,
                                                                       group_counts);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Single-pass ordered compaction (transform-feedback semantics) with decoupled look-back: every block publishes the
// number of items it keeps, obtains the number kept by all earlier blocks by walking back over the published
// descriptors, and writes its items to their final position -- one read and one write per surfel, no flag / count /
// scan passes. Blocks take their (virtual) index from a ticket so that earlier indices are always already running.
// Descriptor: [63:34] launch generation, [33:32] status (0 none, 1 block aggregate, 2 inclusive prefix), [31:0] value.
// ------------------------------------------------------------------------------------------------------------
struct Lookback {
  unsigned long long* desc;
  uint32_t* ticket;
  uint32_t gen;
};
__device__ __forceinline__ unsigned long long lb_pack(uint32_t gen, uint32_t status, uint32_t value) {
  return ((unsigned long long)gen << 34) | ((unsigned long long)status << 32) | (unsigned long long)value;
}

__device__ __forceinline__ uint32_t block_ticket(const Lookback& lb) {
  __shared__ uint32_t s_vb;
  if (threadIdx.x == 0) s_vb = atomicAdd(lb.ticket, 1u);
  __syncthreads();
  return s_vb;
}

// rank of this thread's item among the kept items of the block, and the block's count
template <int THREADS>
__device__ __forceinline__ uint32_t block_rank(bool kept, uint32_t& block_count) {
  __shared__ uint32_t s_warp[THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned m = __ballot_sync(0xffffffffu, kept);
  if (lane == 0) s_warp[warp] = __popc(m);
  __syncthreads();
  uint32_t before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) {
    uint32_t v = s_warp[w];
    if (w < warp) before += v;
    total += v;
  }
  block_count = total;
  return before + __popc(m & ((1u << lane) - 1u));
}

// Exclusive prefix of `count` over the blocks with a smaller virtual index. Every block publishes its own count FIRST and
// then sums the published counts of ALL its predecessors -- 256 descriptors per round with 8 loads in flight per lane.
// (Round 1 walked back 32 descriptors at a time and stopped at the first inclusive prefix: with all ~500 blocks of the
// generation pass resident and publishing at about the same moment that is a chain of ~16 dependent L2 round trips for
// the last blocks: 16 us for a pass that touches 11 MB.) No circular wait: a predecessor holds a smaller ticket, so it is
// running or finished, and it publishes before it waits for anything.
__device__ __forceinline__ uint32_t lookback_exclusive(const Lookback& lb, uint32_t vb, uint32_t count) {
  __shared__ uint32_t s_excl;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (lane == 0) atomicExch(lb.desc + vb, lb_pack(lb.gen, 1u, count));
    uint32_t sum = 0;
    for (uint32_t i0 = 0; i0 < vb; i0 += 256) {
      unsigned long long d[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t idx = i0 + 32 * j + lane;
        d[j] = idx < vb ? *(volatile unsigned long long*)(lb.desc + idx) : lb_pack(lb.gen, 1u, 0u);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t idx = i0 + 32 * j + lane;
        while (!((uint32_t)(d[j] >> 34) == lb.gen && ((d[j] >> 32) & 3ull) != 0ull))
          d[j] = *(volatile unsigned long long*)(lb.desc + idx);
        sum += (uint32_t)d[j];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) s_excl = sum;
  }
  __syncthreads();
  return s_excl;
}

// ------------------------------------------------------------------------------------------------------------
// K6c: update_surfels.vert:140-333, fused with the K6e predicate of copy_surfels.vert:38-56
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 data_tex(const float4* __restrict__ img, int W, int H, float fx, float fy) {
  if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) return make_float4(0.f, 0.f, 0.f, 0.f);
  return __ldg(img + (size_t)(int)fy * W + (size_t)(int)fx);
}

__device__ __forceinline__ V3 slerp(V3 v0, V3 v1, float weight) {  // update_surfels.vert:113-124
  float omega = acosf_(dot3(normalize3(v0), normalize3(v1)));
  float eta = 1.0f / sinf_(omega);
  float w0 = eta * sinf_(weight * omega);
  float w1 = eta * sinf_((1.0f - weight) * omega);
  return add3(scale3(w0, v0), scale3(w1, v1));
}

__device__ __forceinline__ bool submap_keep(const float* __restrict__ poses, float4 p0, float4 p2, float2 center,
                                            float extent) {
  float M[16];
  load_mat(poses, pose_index(p2.w), M);
  V3 w = xform_point(M, mk3(p0.x, p0.y, p0.z));
  if ((int)__float_as_uint(p2.x) < 0 || fabsf(w.x - center.x) > extent || fabsf(w.y - center.y) > extent) return false;
  return true;
}

// Epilogue of the predicate kernels of the surfel-indexed passes, called by every thread of the block: two-level counts, so
// that k_compact finds a block's output offset from <= 64 group totals + <= 63 block counts -- no scan pass. The
// kGroupCounts totals of 64 blocks each must be zero before the predicate kernel runs.
__device__ __forceinline__ void publish_block_count(bool kept, uint32_t* block_counts, uint32_t* group_counts) {
  const int cnt = __syncthreads_count(kept ? 1 : 0);
  if (threadIdx.x == 0) {
    block_counts[blockIdx.x] = (uint32_t)cnt;
    if (cnt) atomicAdd(group_counts + (blockIdx.x >> 6), (uint32_t)cnt);
  }
}

struct UpdateArgs {
  Mat4 pose;               // current sensor pose (by value: no upload on the critical path)
  Mat4 inv_pose;
  const Mat4* pose_dev;    // or resident on the device (pipeline mode)
  const Mat4* inv_pose_dev;
  const float* poses;      // pose table
  const float* poses_inv;  // inverse pose table
  const unsigned long long* index_keys;
  const float4* radius_map;
  int timestamp;
  float2 submap_center;
  float submap_extent;
};

__device__ __forceinline__ bool same_bits(float4 a, float4 b) {
  return __float_as_uint(a.x) == __float_as_uint(b.x) && __float_as_uint(a.y) == __float_as_uint(b.y) &&
         __float_as_uint(a.z) == __float_as_uint(b.z) && __float_as_uint(a.w) == __float_as_uint(b.w);
}

// kLazy = false (dense): the updated records go to tmp with a keep byte each, and k_compact moves the kept ones back.
// kLazy = true (in place): a lane is stored back into src only if its bits changed, a surfel that is not kept is marked
// dead in `live`, and nothing moves: counts[1] = the physical end (k_gen_compact appends behind it and sums the live
// count from the group totals). Dead slots are skipped in both modes, so a dense pass also compacts the map.
template <bool kLazy>
__global__ void __launch_bounds__(kThreads) k_update_surfels(KParams kp, SurfelPlanes src, SurfelPlanes tmp,
                                                            const uint32_t* n_dev, UpdateArgs ua,
                                                            FrameDev f, uint8_t* __restrict__ integrated,
                                                            uint8_t* __restrict__ live, uint8_t* __restrict__ keep,
                                                            uint32_t* __restrict__ block_counts,
                                                            uint32_t* __restrict__ group_counts, uint32_t* counts) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = *n_dev;
  if (kLazy && k == 0) counts[1] = n;
  bool kept = false;
  bool lv = false;
  // in place, the lanes are written by this kernel: plain loads, not the read-only path. The liveness byte is loaded
  // together with them (gating the lane loads on it would cost an L2 round trip per wave).
  float4 p0, p1, p2, p3 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (k < n) {
    lv = live[k] != 0;
    if (kLazy) {
      p0 = src.p0[k]; p1 = src.p1[k]; p2 = src.p2[k];
    } else {
      p0 = __ldg(src.p0 + k); p1 = __ldg(src.p1 + k); p2 = __ldg(src.p2 + k); p3 = __ldg(src.p3 + k);
    }
  }
  if (lv) {
    const int W = kp.W, H = kp.H;
    const int timestamp = ua.timestamp;
    int s_ts = (int)__float_as_uint(p2.x);
    int surfel_age = timestamp - s_ts;
    int creation = (int)p2.w;
    int ci = pose_index(p2.w);
    float SP[16];
    load_mat(ua.poses, ci, SP);
    const float* POSE = ua.pose_dev ? ua.pose_dev->m : ua.pose.m;
    const float* INV = ua.inv_pose_dev ? ua.inv_pose_dev->m : ua.inv_pose.m;
    V3 old_position = xform_point(SP, mk3(p0.x, p0.y, p0.z));
    V3 old_normal = xform_dir(SP, mk3(p1.x, p1.y, p1.z));
    float old_radius = p0.w, old_conf = p1.w, old_weight = p2.z;
    bool valid_out = true;
    if (old_conf < kp.confidence_threshold && kp.use_stability) valid_out = surfel_age < kp.unstable_age;
    float4 o0 = p0, o1 = p1, o2 = p2;
    bool avg_prob_set = false;  // o3 = p3 with w = avg_prob
    float avg_prob = 0.0f;
    o2.y = pack_rgb(0.3f, 0.3f, 0.3f);
    V3 vertex = xform_point(INV, old_position);
    V3 normal = normalize3(xform_dir(INV, old_normal));
    bool visible = dot3(normal, divs3(neg3(vertex), len3(vertex))) > 0.0f;
    float x, y, z;
    project01(vertex, kp.fov_up, kp.fov, kp.min_depth, kp.max_depth, x, y, z);
    float ix = floorf(x * (float)W) + 0.5f, iy = floorf(y * (float)H) + 0.5f;
    bool inside = (ix < (float)W && iy < (float)H && z < 1.0f) && !(ix < 0.0f && iy < 0.0f && z < 0.0f);
    // the measurement is only ever used under (valid && inside && visible): back-facing surfels skip the two gathers
    float4 Vt = make_float4(0.f, 0.f, 0.f, 0.f), Nt = Vt;
    if (visible && inside) {
      Vt = data_tex(f.vertex, W, H, ix, iy);
      Nt = data_tex(f.normal, W, H, ix, iy);
    }
    bool valid = (Vt.w > 0.5f) && (Nt.w > 0.5f);
    float penalty = 0.0f;
    float update_conf = kp.log_prior;
    size_t dpix = 0;
    bool mark_integrated = false;
    if (valid && inside && visible) {
      if (kLazy) p3 = src.p3[k];  // the only branch that reads or changes the semantic lane
      float4 St = data_tex(f.semantic, W, H, ix, iy);
      float4 Rt = data_tex(ua.radius_map, W, H, ix, iy);
      float data_label = St.x * 255.0f, data_prob = St.w;
      float model_label = p3.x * 255.0f, model_prob = p3.w;
      bool label_diff = roundf_(data_label) != roundf_(model_label);
      if (label_diff && is_movable(model_label)) penalty = 1.0f;
      V3 v = mk3(Vt.x, Vt.y, Vt.z), n = mk3(Nt.x, Nt.y, Nt.z);
      V3 v_global = xform_point(POSE, v);
      V3 n_global = normalize3(xform_dir(POSE, n));
      V3 view_dir = divs3(neg3(v), len3(v));
      float distance = fabsf(dot3(old_normal, sub3(v_global, old_position)));
      float angle = len3(cross3(n_global, old_normal));
      float new_radius = Rt.x, new_conf = Rt.y;
      dpix = (size_t)(int)iy * W + (size_t)(int)ix;
      if (distance < kp.map_max_distance && angle < kp.update_angle_thresh) {
        // the "measurement integrated" point is drawn only if the geometry stage emits this surfel, i.e. if it is
        // still valid at the end of the pass (update_surfels.geom:35-48): decided below
        float zn = 2.0f * z - 1.0f;
        mark_integrated = zn >= -1.0f && zn <= 1.0f && depth24(0.5f * zn + 0.5f) < kDepthClear;
        float confidence = old_conf + new_conf;
        o1.w = confidence;
        o2.x = __uint_as_float((uint32_t)timestamp);
        float avg_radius = new_radius < old_radius ? new_radius : old_radius;
        avg_radius = avg_radius > 0.0f ? avg_radius : 0.0f;  // update program's min_radius uniform is 0 (SurfelMap.cpp:422)
        o0.w = avg_radius;
        valid_out = true;
        o2.y = pack_rgb(0.0f, 0.7f, 0.0f);
        o2.w = (float)creation;
        float a = angle, d = distance;
        float pr = kp.p_stable;
        if (kp.confidence_mode == 1 || kp.confidence_mode == 3)
          pr = pr * expf_(((-a) * a) / (kp.sigma_angle * kp.sigma_angle));
        if (kp.confidence_mode == 2 || kp.confidence_mode == 3)
          pr = pr * expf_(((-d) * d) / (kp.sigma_distance * kp.sigma_distance));
        pr = pr > kp.p_unstable ? pr : kp.p_unstable;
        pr = pr < 1.0f ? pr : 1.0f;
        update_conf = logf_(pr / (1.0f - pr));
        if ((new_radius < old_radius && timestamp - creation < kp.active_timestamps) || kp.update_always) {
          float w1 = 0.9f, w2 = 0.1f;
          if (kp.weighting_scheme > 0) {
            w1 = old_weight;
            w2 = 1.0f;
            if (kp.weighting_scheme == 2) w2 = dot3(n, view_dir);
            float sw = w1 + w2;
            o2.z = kp.max_weight < sw ? kp.max_weight : sw;
            float sum = w1 + w2;
            w1 = w1 / sum;
            w2 = w2 / sum;
          }
          V3 avg_position = add3(scale3(w1, old_position), scale3(w2, v_global));
          V3 avg_normal = slerp(old_normal, n_global, w1);
          if (label_diff)
            avg_prob = w1 * model_prob + w2 * (1.0f - data_prob);
          else
            avg_prob = w1 * model_prob + w2 * data_prob;
          avg_prob_set = true;
          if (kp.averaging_scheme == 1) {
            avg_position = add3(old_position, scale3(w2 * distance, old_normal));
            avg_normal = slerp(old_normal, n_global, w1);
          }
          avg_normal = normalize3(avg_normal);
          float SPI[16];
          load_mat(ua.poses_inv, ci, SPI);
          avg_position = xform_point(SPI, avg_position);
          avg_normal = xform_dir(SPI, avg_normal);
          o0 = make_float4(avg_position.x, avg_position.y, avg_position.z, avg_radius);
          o1 = make_float4(avg_normal.x, avg_normal.y, avg_normal.z, confidence);
          o2.y = pack_rgb(1.0f, 0.0f, 1.0f);
        }
      } else {
        unsigned long long key = ua.index_keys[dpix];
        int idx = (key == ~0ull) ? -1 : (int)(uint32_t)(key & 0xffffffffull);
        if (idx == (int)k) {  // closest visible surfel of that pixel
          update_conf = logf_(kp.p_unstable / (1.0f - kp.p_unstable));
          o2.y = pack_rgb(0.0f, 1.0f, 1.0f);
        }
      }
    }
    update_conf = update_conf - penalty;
    if (kp.use_stability) {
      float c = (old_conf + update_conf) - kp.log_prior;
      o1.w = c < 20.0f ? c : 20.0f;
    } else {
      o1.w = old_conf;
    }
    if (o1.w < kp.log_unstable && kp.use_stability) valid_out = false;
    if (valid_out && mark_integrated) integrated[dpix] = 1;
    kept = valid_out && submap_keep(ua.poses, o0, o2, ua.submap_center, ua.submap_extent);
    const float4 o3 = avg_prob_set ? make_float4(p3.x, p3.y, p3.z, avg_prob) : p3;
    if (!kLazy) {
      tmp.p0[k] = o0;
      tmp.p1[k] = o1;
      tmp.p2[k] = o2;
      tmp.p3[k] = o3;
    } else if (!kept) {
      live[k] = 0;
    } else {  // bits, not values: -0.0, NaN payloads and confidences above 20 are stored exactly as the dense pass does
      if (!same_bits(o0, p0)) src.p0[k] = o0;
      if (!same_bits(o1, p1)) src.p1[k] = o1;
      if (!same_bits(o2, p2)) src.p2[k] = o2;
      if (avg_prob_set && __float_as_uint(avg_prob) != __float_as_uint(p3.w)) src.p3[k] = o3;
    }
  }
  if (!kLazy && k < n) keep[k] = kept ? 1 : 0;
  // (group totals are cleared by the per-pixel prologue of the map update)
  publish_block_count(kept, block_counts, group_counts);
}

// K6d + K6e in ONE pass: new surfels are appended in x-major pixel order behind the updated ones
__global__ void __launch_bounds__(kThreads) k_gen_compact(KParams kp, FrameDev f, const float4* __restrict__ radius_map,
                                                         const uint8_t* __restrict__ integrated,
                                                         const float* __restrict__ poses, int timestamp, float2 center,
                                                         float extent, SurfelPlanes dst, uint8_t* __restrict__ live,
                                                         const uint32_t* __restrict__ lazy_groups, Lookback lb,
                                                         uint32_t cap, uint32_t* __restrict__ counts) {
  const uint32_t vb = block_ticket(lb);
  int t = (int)(vb * blockDim.x + threadIdx.x);
  bool kept = false;
  float4 o0, o1, o2, o3;
  o0 = o1 = o2 = o3 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t < kp.W * kp.H) {
    int x = t / kp.H, y = t - x * kp.H;
    size_t pix = (size_t)y * kp.W + x;
    // the flag first: in the steady state most measurements were integrated into an existing surfel, and for those pixels
    // the three images below are never needed (1 byte instead of 49 per pixel)
    const bool integ = integrated[pix] != 0;
    float4 V = make_float4(0.f, 0.f, 0.f, 0.f), N = V, R = V;
    if (!integ) {
      V = __ldg(f.vertex + pix);
      N = __ldg(f.normal + pix);
      R = __ldg(radius_map + pix);
    }
    bool invalid = (V.w < 1.0f) || (N.w < 1.0f);
    invalid = invalid || (R.w < 0.5f);
    V3 v = mk3(V.x, V.y, V.z), n = mk3(N.x, N.y, N.z);
    V3 view_dir = divs3(neg3(v), len3(v));
    bool valid = !invalid && !integ && (dot3(n, view_dir) > 0.01f);
    if (valid) {
      V3 ng = normalize3(n);
      float4 S = __ldg(f.semantic + pix);
      float conf = is_movable(S.x * 255.0f) ? kp.log_prior - 0.5f : kp.log_prior;
      o0 = make_float4(v.x, v.y, v.z, R.x);
      o1 = make_float4(ng.x, ng.y, ng.z, conf);
      o2 = make_float4(__uint_as_float((uint32_t)timestamp), pack_rgb(0.0f, 0.0f, 1.0f), 1.0f, (float)timestamp);
      o3 = S;
      kept = submap_keep(poses, o0, o2, center, extent);
    }
  }
  uint32_t block_count;
  const uint32_t rank = block_rank<kThreads>(kept, block_count);
  const uint32_t excl = lookback_exclusive(lb, vb, block_count);
  const uint32_t base = counts[1];
  if (kept) {
    uint32_t d = base + excl + rank;
    if (d < cap) {
      dst.p0[d] = o0;
      dst.p1[d] = o1;
      dst.p2[d] = o2;
      dst.p3[d] = o3;
      live[d] = 1;
    }
  }
  if (vb == gridDim.x - 1 && lazy_groups && threadIdx.x < 32) {
    // after an in-place update (complete: stream order), which compacted nothing: the surfels it kept are the sum of the
    // group totals it published, and the rest of the slots below counts[1] are dead
    uint32_t v = 0;
    for (int g = threadIdx.x; g < kGroupCounts; g += 32) v += lazy_groups[g];
    v = __reduce_add_sync(0xffffffffu, v);
    if (threadIdx.x == 0) {
      counts[2] = v;
      counts[5] = base - v;
    }
  }
  if (vb == gridDim.x - 1 && threadIdx.x == 0) {
    uint32_t total = base + excl + block_count;
    counts[0] = total < cap ? total : cap;  // new physical end of the map
    counts[3] = excl + block_count;         // kept new surfels
    *lb.ticket = 0;
  }
}

// extract_surfels.vert:44-62: flags of the live surfels inside one submap tile; with poses == nullptr, of every live
// surfel (the compaction of a map with dead slots)
__global__ void __launch_bounds__(kThreads) k_extract_flags(SurfelPlanes s, const uint32_t* __restrict__ n_dev,
                                                           const uint8_t* __restrict__ live,
                                                           const float* __restrict__ poses, float2 center, float extent,
                                                           uint8_t* __restrict__ keep,
                                                           uint32_t* __restrict__ block_counts,
                                                           uint32_t* __restrict__ group_counts) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  bool kept = false;
  if (k < *n_dev) {
    if (live[k]) {
      kept = true;
      if (poses) {
        float4 p0 = __ldg(s.p0 + k), p2 = __ldg(s.p2 + k);
        float M[16];
        load_mat(poses, pose_index(p2.w), M);
        V3 w = xform_point(M, mk3(p0.x, p0.y, p0.z));
        kept = !(fabsf(w.x - center.x) > extent || fabsf(w.y - center.y) > extent);
      }
    }
    keep[k] = kept ? 1 : 0;
  }
  publish_block_count(kept, block_counts, group_counts);
}

// Ordered compaction (transform feedback semantics) of a surfel-indexed pass without a scan kernel: block b's offset =
// sum of the group totals before its group (<= 64 for 4M surfels) + the counts of the earlier blocks of its own group
// (<= 63), summed by one warp. The kept item of relative rank rel goes to dst[base + rel] iff rel < rel_cap and
// base + rel < cap (transform feedback drops what does not fit), with base = *base_dev (0 if null; base <= cap).
// The last block publishes out[0] = base + number written (the end of the written range), out[1] = number kept.
// dst_live (null for the tile pool): the liveness bytes of the destination slots, set for every slot written.
__global__ void __launch_bounds__(kThreads) k_compact(SurfelPlanes src, const uint8_t* __restrict__ keep,
                                                     const uint32_t* __restrict__ block_counts,
                                                     const uint32_t* __restrict__ group_counts,
                                                     const uint32_t* __restrict__ n_dev, SurfelPlanes dst,
                                                     uint8_t* __restrict__ dst_live,
                                                     const uint32_t* __restrict__ base_dev, uint32_t cap, uint32_t rel_cap,
                                                     uint32_t* __restrict__ out) {
  __shared__ uint32_t warp_cnt[kThreads / 32];
  __shared__ uint32_t s_offset;
  const uint32_t n = *n_dev;
  const uint32_t nblocks = (n + kThreads - 1) / kThreads;
  const uint32_t base = base_dev ? *base_dev : 0u;
  const uint32_t lim = min(rel_cap, cap - base);  // relative ranks below lim are written
  if (blockIdx.x >= nblocks) {
    if (nblocks == 0 && blockIdx.x == 0 && threadIdx.x == 0) {  // empty map
      out[0] = base;
      out[1] = 0;
    }
    return;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  const bool kept = (k < n) && keep[k];
  const unsigned m = __ballot_sync(0xffffffffu, kept);
  if (lane == 0) warp_cnt[warp] = __popc(m);
  if (warp == 0) {
    const uint32_t g = blockIdx.x >> 6, first = g << 6;
    uint32_t v = 0;
    for (uint32_t i = lane; i < g; i += 32) v += group_counts[i];
    for (uint32_t b = first + lane; b < blockIdx.x; b += 32) v += block_counts[b];
    v = __reduce_add_sync(0xffffffffu, v);
    if (lane == 0) s_offset = v;
  }
  __syncthreads();
  uint32_t before = 0;
  for (int w = 0; w < warp; ++w) before += warp_cnt[w];
  if (blockIdx.x == nblocks - 1 && threadIdx.x == 0) {
    const uint32_t total = s_offset + block_counts[blockIdx.x];
    out[0] = base + min(total, lim);
    out[1] = total;
  }
  if (!kept) return;
  const uint32_t rel = s_offset + before + __popc(m & ((1u << lane) - 1u));
  if (rel >= lim) return;
  const uint32_t d = base + rel;
  dst.p0[d] = src.p0[k];
  dst.p1[d] = src.p1[k];
  dst.p2[d] = src.p2[k];
  dst.p3[d] = src.p3[k];
  if (dst_live) dst_live[d] = 1;
}

void launch_compact(const Launch& L, SurfelPlanes src, const uint8_t* keep, const uint32_t* block_counts,
                    const uint32_t* group_counts, const uint32_t* n_dev, uint32_t n_upper, SurfelPlanes dst,
                    uint8_t* dst_live, const uint32_t* base_dev, uint32_t cap, uint32_t rel_cap, uint32_t* out) {
  uint32_t blocks = (n_upper + kThreads - 1) / kThreads;
  if (blocks == 0) blocks = 1;
  {
    ScopedKernel sk(L, K_COMPACT_SCATTER);
    k_compact<<<blocks, kThreads, 0, L.stream>>>(src, keep, block_counts, group_counts, n_dev, dst, dst_live, base_dev, cap,
                                                 rel_cap, out);
  }
}

void launch_compact_live(const Launch& L, SurfelPlanes src, const uint32_t* n_dev, uint32_t n_upper, uint8_t* live,
                         uint8_t* keep, uint32_t* block_counts, uint32_t* group_counts, SurfelPlanes dst, uint32_t* out) {
  if (n_upper > 0) {
    ScopedKernel sk(L, K_EXTRACT_FLAGS);
    k_extract_flags<<<(n_upper + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(src, n_dev, live, nullptr,
                                                                                 make_float2(0.f, 0.f), 0.f, keep,
                                                                                 block_counts, group_counts);
  }
  // (k_extract_flags has consumed the liveness bytes of the source slots before any is set for a destination slot)
  launch_compact(L, src, keep, block_counts, group_counts, n_dev, n_upper, dst, live, nullptr, kMaxSurfels, kMaxSurfels,
                 out);
}

// ---- submap tile cache in HBM: a leaving tile is compacted straight into a device-resident pool (the reference
// downloads it to host RAM, SurfelMap.cpp:708-742). Slot s of the pool starts where slot s - 1 ends (slot 0 at 0);
// rec[s] = {end of slot s in the pool, surfels of the tile}.
void launch_extract_to_pool(const Launch& L, SurfelPlanes map, const uint32_t* n_dev, const uint8_t* live, uint32_t n_upper,
                            const float* poses, float2 center, float extent, uint8_t* keep, uint32_t* block_counts,
                            uint32_t* group_counts, SurfelPlanes pool, uint32_t pool_cap, uint2* rec, uint32_t slot,
                            uint32_t tile_cap) {
  if (n_upper > 0) {
    ScopedKernel sk(L, K_EXTRACT_FLAGS);
    k_extract_flags<<<(n_upper + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(map, n_dev, live, poses, center, extent,
                                                                                 keep, block_counts, group_counts);
  }
  launch_compact(L, map, keep, block_counts, group_counts, n_dev, n_upper, pool, nullptr, slot ? &rec[slot - 1].x : nullptr,
                 pool_cap, tile_cap, &rec[slot].x);
}

void launch_update_surfels(const Launch& L, const KParams& kp, bool lazy, SurfelPlanes src, SurfelPlanes tmp,
                           uint32_t* counts, uint32_t n_upper, const Mat4& pose, const Mat4& inv_pose,
                           const Mat4* pose_dev, const Mat4* inv_pose_dev, const float* poses,
                           const float* poses_inv, const unsigned long long* index_keys, const float4* radius_map,
                           FrameDev frame, int timestamp, float2 submap_center, float submap_extent,
                           uint8_t* integrated, uint8_t* live, uint8_t* keep, uint32_t* block_counts,
                           uint32_t* group_counts) {
  if (n_upper == 0) return;
  UpdateArgs ua{pose, inv_pose, pose_dev, inv_pose_dev, poses, poses_inv, index_keys, radius_map, timestamp,
                submap_center, submap_extent};
  const unsigned grid = (n_upper + kThreads - 1) / kThreads;
  {
    ScopedKernel sk(L, K_UPDATE_SURFELS);
    if (lazy)
      k_update_surfels<true><<<grid, kThreads, 0, L.stream>>>(kp, src, tmp, counts, ua, frame, integrated, live, keep,
                                                             block_counts, group_counts, counts);
    else
      k_update_surfels<false><<<grid, kThreads, 0, L.stream>>>(kp, src, tmp, counts, ua, frame, integrated, live, keep,
                                                              block_counts, group_counts, counts);
  }
}

void launch_gen_compact(const Launch& L, const KParams& kp, FrameDev frame, const float4* radius_map,
                        const uint8_t* integrated, const float* poses, int timestamp, float2 submap_center,
                        float submap_extent, SurfelPlanes map, uint8_t* live, const uint32_t* lazy_groups,
                        unsigned long long* desc, uint32_t* ticket, uint32_t gen, uint32_t cap, uint32_t* counts) {
  int P = kp.W * kp.H;
  Lookback lb{desc, ticket, gen};
  {
    ScopedKernel sk(L, K_GEN_SURFELS);
    k_gen_compact<<<(P + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(kp, frame, radius_map, integrated, poses,
                                                                           timestamp, submap_center, submap_extent, map,
                                                                           live, lazy_groups, lb, cap, counts);
  }
}

// ---- 64-byte AoS records (Surfel.h) <-> SoA lanes, for upload / download at the ABI ----
__global__ void k_aos_to_soa(const float4* __restrict__ aos, SurfelPlanes s, uint32_t offset, uint32_t n) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  s.p0[offset + k] = aos[4 * (size_t)k + 0];
  s.p1[offset + k] = aos[4 * (size_t)k + 1];
  s.p2[offset + k] = aos[4 * (size_t)k + 2];
  s.p3[offset + k] = aos[4 * (size_t)k + 3];
}
__global__ void k_soa_to_aos(SurfelPlanes s, float4* __restrict__ aos, uint32_t n) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  aos[4 * (size_t)k + 0] = s.p0[k];
  aos[4 * (size_t)k + 1] = s.p1[k];
  aos[4 * (size_t)k + 2] = s.p2[k];
  aos[4 * (size_t)k + 3] = s.p3[k];
}
void launch_aos_to_soa(const Launch& L, const sb_surfel* aos, SurfelPlanes s, uint32_t offset, uint32_t n) {
  if (n == 0) return;
  {
    ScopedKernel sk(L, K_AOS_TO_SOA);
    k_aos_to_soa<<<(n + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(reinterpret_cast<const float4*>(aos), s, offset,
                                                                        n);
  }
}
void launch_soa_to_aos(const Launch& L, SurfelPlanes s, sb_surfel* aos, uint32_t n) {
  if (n == 0) return;
  {
    ScopedKernel sk(L, K_SOA_TO_AOS);
    k_soa_to_aos<<<(n + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(s, reinterpret_cast<float4*>(aos), n);
  }
}

// ---- checkpoints (sb_state_save / sb_state_load): ordered gather of the live map, scatter back, position-keyed digest ----
__device__ __forceinline__ uint64_t lane_digest(float4 v, uint64_t pos) {  // the two 64-bit words of one 16-byte lane
  const uint64_t w0 = ((uint64_t)__float_as_uint(v.y) << 32) | __float_as_uint(v.x);
  const uint64_t w1 = ((uint64_t)__float_as_uint(v.w) << 32) | __float_as_uint(v.z);
  return state_word_hash(pos, w0) + state_word_hash(pos + 1, w1);
}

// one atomic per block: the block's sum (exact mod 2^64, so the order of the blocks' additions does not matter)
__device__ __forceinline__ void block_digest_add(uint64_t h, unsigned long long* acc) {
  __shared__ uint64_t s_h[kThreads / 32];
  for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if ((threadIdx.x & 31) == 0) s_h[threadIdx.x >> 5] = h;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += s_h[w];
    atomicAdd(acc, (unsigned long long)t);
  }
}

__global__ void __launch_bounds__(kThreads) k_state_pack(SurfelPlanes s, const uint8_t* __restrict__ live, uint32_t n_phys,
                                                        float4* __restrict__ flat, uint32_t n_live, Lookback lb,
                                                        uint64_t word_base, unsigned long long* acc) {
  const uint32_t vb = block_ticket(lb);
  const uint32_t k = vb * blockDim.x + threadIdx.x;
  const bool kept = k < n_phys && live[k] != 0;
  float4 v0, v1, v2, v3;
  v0 = v1 = v2 = v3 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (kept) {
    v0 = s.p0[k]; v1 = s.p1[k]; v2 = s.p2[k]; v3 = s.p3[k];
  }
  uint32_t block_count;
  const uint32_t rank = block_rank<kThreads>(kept, block_count);
  const uint32_t excl = lookback_exclusive(lb, vb, block_count);
  uint64_t h = 0;
  if (kept) {
    const uint32_t d = excl + rank;  // < n_live: the host counted the live slots
    const float4 v[4] = {v0, v1, v2, v3};
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const size_t i = (size_t)l * n_live + d;
      flat[i] = v[l];
      h += lane_digest(v[l], word_base + 2 * i);
    }
  }
  block_digest_add(h, acc);
  if (vb == gridDim.x - 1 && threadIdx.x == 0) *lb.ticket = 0;
}

__global__ void __launch_bounds__(kThreads) k_state_unpack(const float4* __restrict__ flat, uint32_t n, SurfelPlanes s,
                                                          uint8_t* __restrict__ live, uint64_t word_base,
                                                          unsigned long long* acc) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t h = 0;
  if (k < n) {
    float4* dst[4] = {s.p0, s.p1, s.p2, s.p3};
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const size_t i = (size_t)l * n + k;
      const float4 v = flat[i];
      dst[l][k] = v;
      h += lane_digest(v, word_base + 2 * i);
    }
    live[k] = 1;
  }
  block_digest_add(h, acc);
}

__global__ void __launch_bounds__(kThreads) k_state_digest(const unsigned long long* __restrict__ w, uint64_t n,
                                                          uint64_t word_base, unsigned long long* acc) {
  uint64_t h = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    h += state_word_hash(word_base + i, w[i]);
  block_digest_add(h, acc);
}

void launch_state_pack(const Launch& L, SurfelPlanes map, const uint8_t* live, uint32_t n_phys, float4* flat,
                       uint32_t n_live, unsigned long long* desc, uint32_t* ticket, uint32_t gen, uint64_t word_base,
                       unsigned long long* acc) {
  if (n_phys == 0) return;
  Lookback lb{desc, ticket, gen};
  {
    ScopedKernel sk(L, K_STATE_PACK);
    k_state_pack<<<(n_phys + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(map, live, n_phys, flat, n_live, lb,
                                                                               word_base, acc);
  }
}

void launch_state_unpack(const Launch& L, const float4* flat, uint32_t n, SurfelPlanes map, uint8_t* live,
                         uint64_t word_base, unsigned long long* acc) {
  if (n == 0) return;
  {
    ScopedKernel sk(L, K_STATE_UNPACK);
    k_state_unpack<<<(n + kThreads - 1) / kThreads, kThreads, 0, L.stream>>>(flat, n, map, live, word_base, acc);
  }
}

void launch_state_digest(const Launch& L, const void* words, uint64_t n_words, uint64_t word_base, unsigned long long* acc) {
  if (n_words == 0) return;
  uint64_t blocks = (n_words + kThreads - 1) / kThreads;
  if (blocks > 1024) blocks = 1024;
  {
    ScopedKernel sk(L, K_STATE_DIGEST);
    k_state_digest<<<(unsigned)blocks, kThreads, 0, L.stream>>>(static_cast<const unsigned long long*>(words), n_words,
                                                                 word_base, acc);
  }
}

}  // namespace sb
