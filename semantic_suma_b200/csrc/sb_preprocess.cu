// sb_preprocess.cu -- K1-K3: spherical projection of a scan into vertex / normal / semantic range images.
// Replaces Preprocessing::process (core/Preprocessing.cpp:120-339) and its shaders gen_vertexmap.{vert,frag},
// gen_normalmap.frag, floodfill.frag.
//
// H100 mapping: the z-buffered point rasterisation (GL depth test GL_LESS, earliest primitive wins ties) becomes a
// 64-bit atomicMin on a packed (depth24 << 32 | point index) key image; the images (2 MiB each at 64x2048) stay
// L2-resident between the passes, so every pass is a plain coalesced float4 stream + a handful of L2 gathers.
#include <cuda.h>

#include "sb_internal.cuh"

namespace sb {
using namespace sbm;

// ---- K1a's per-point body, shared by the scatter and by the per-point labels (one source for the pixel arithmetic) ----
// The point i as the projection sees it. kDeskew: moved to the scan's reference time (DESIGN.md section 11).
template <bool kDeskew>
__device__ __forceinline__ float4 k1_point(const float4* __restrict__ pts, uint32_t i, const DeskewArgs& dk) {
  float4 p4 = __ldg(pts + i);
  if (kDeskew) {
    const float s = deskew_sweep_time(dk.mode, dk.mode == 1 ? __ldg(dk.times + i) : 0.0f,
                                      dk.mode == 2 ? atan2f_(p4.y, p4.x) : 0.0f, dk.ref_time, dk.start_azimuth,
                                      dk.clockwise);
    const V3 q = deskew_point(mk3(p4.x, p4.y, p4.z), s - dk.ref_time, mk3(dk.w[0], dk.w[1], dk.w[2]),
                              mk3(dk.t[0], dk.t[1], dk.t[2]));
    p4 = make_float4(q.x, q.y, q.z, p4.w);
  }
  return p4;
}

// gen_vertexmap.vert:83-89: the pixel (ix, iy) of pos at range d in a W x H image under (fov_up, fov); false: clipped
// (field of view, the seam at yaw -pi, NaN)
__device__ __forceinline__ bool k1_pixel(V3 pos, float d, int W, int H, float fov_up, float fov, int* ix, int* iy) {
  float yaw = atan2f_(pos.y, pos.x);
  float pitch = -asinf_(pos.z / d);
  float x = -yaw * kInvPi;
  float y = 1.0f - (2.0f * (kRad2Deg * pitch + fov_up)) / fov;
  float fx = floorf((0.5f * (x + 1.0f)) * (float)W);
  float fy = floorf((0.5f * (y + 1.0f)) * (float)H);
  if (!(fx >= 0.0f && fx < (float)W && fy >= 0.0f && fy < (float)H)) return false;
  *ix = (int)fx;
  *iy = (int)fy;
  return true;
}

// gen_vertexmap.vert:85-91: the data pixel and 24-bit depth of pos; false when the point scatters no key
__device__ __forceinline__ bool k1_project(const KParams& kp, V3 pos, int* ix, int* iy, uint32_t* d24) {
  const float d = len3(pos);
  if (!k1_pixel(pos, d, kp.W, kp.H, kp.fov_up, kp.fov, ix, iy)) return false;
  const float z = 2.0f * ((d - kp.min_depth) / (kp.max_depth - kp.min_depth)) - 1.0f;
  if (!(z >= -1.0f && z <= 1.0f)) return false;
  *d24 = depth24(0.5f * z + 0.5f);
  return *d24 < kDepthClear;  // GL_LESS against the cleared buffer
}

// K1a: gen_vertexmap.vert:73-91 -- one thread per point, scatter-min into the key image.
// kDeskew: the moved point is also written to dk.out, from where k_preprocess_tile reads the winners; the off instance
// does not touch dk.
template <bool kDeskew>
__global__ void __launch_bounds__(256) k_project_scatter(KParams kp, const float4* __restrict__ pts, uint32_t n,
                                                         unsigned long long* __restrict__ keys, DeskewArgs dk) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p4 = k1_point<kDeskew>(pts, i, dk);
  if (kDeskew) dk.out[i] = p4;
  int ix, iy;
  uint32_t d24;
  if (!k1_project(kp, mk3(p4.x, p4.y, p4.z), &ix, &iy, &d24)) return;
  // key image rows are [W + 6]: three mirror columns on both sides (see k_preprocess_tile)
  const int Wp = kp.W + 6;
  unsigned long long* row = keys + (size_t)iy * Wp;
  const unsigned long long key = ((unsigned long long)d24 << 32) | (unsigned long long)i;
  atomicMin(row + ix + 3, key);
  if (ix < 3) atomicMin(row + ix + 3 + kp.W, key);
  if (ix >= kp.W - 3) atomicMin(row + ix + 3 - kp.W, key);
}

// ------------------------------------------------------------------------------------------------------------
// K1b + K2 + K3 (+ K6b) in ONE shared-memory-tiled pass.
// gen_vertexmap.vert:92-102 / .frag:16-23 (resolve the depth-test winners), gen_normalmap.frag:41-99 (normals from the
// +x / +y neighbours, label erosion), floodfill.frag:34-84, init_radiusConf.vert:41-68.
//
// A block owns a kPrepTX x kPrepTY tile of the range image. It resolves the z-buffer keys of the tile plus a 3-pixel
// halo into shared memory (vertex + raw label; halo 3 = 1 for the erosion stencil + 2 for the flood-fill stencil),
// erodes the labels on the tile + 2, and finishes normals, flood fill and surfel radius for its own pixels from
// shared memory. One launch instead of four, every image written exactly once, the intermediate raw / eroded label
// images never reach HBM. The key tile itself is a dense 2-D box of the key image: with kTma it is staged by the TMA
// unit (cp.async.bulk.tensor.2d + mbarrier), otherwise by plain loads.
//
// Key image layout: [H][W + 6] -- three mirror columns on both sides of every row make the azimuth wrap-around of the
// stencils (gen_normalmap.frag wrap()) a plain box read; the scatter kernel writes seam pixels to both places.
// Two key images alternate between scans: this kernel reads image A and re-arms the own tile of image B (~0) for the
// next scan, so no fill pass exists and no block can clear a key a neighbour still has to read.
// ------------------------------------------------------------------------------------------------------------
constexpr int kPrepTX = 32, kPrepTY = 16, kPrepHalo = 3;
constexpr int kPrepSW = kPrepTX + 2 * kPrepHalo, kPrepSH = kPrepTY + 2 * kPrepHalo;  // 38 x 22
constexpr int kPrepThreads = 256;

struct PrepIO {
  const float4* pts;
  const float* labels;
  const float* probs;
  uint32_t n;
  int isfirst;
  const unsigned long long* keys;   // [H][W+6], read
  unsigned long long* keys_next;    // [H][W+6], re-armed for the next scan
  float4* vertex;
  float4* normal;
  float4* semantic;
  float4* radius_map;               // optional: init_radiusConf output of this frame (pipeline mode)
  unsigned long long* index_keys;   // optional: index-map key image to re-arm (pipeline mode)
  uint8_t* integrated;              // optional: "measurement integrated" flags to clear (pipeline mode)
  uint32_t* group_counts;           // optional: group totals of the update pass to clear (pipeline mode)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <bool kTma>
__global__ void __launch_bounds__(kPrepThreads) k_preprocess_tile(KParams kp, PrepIO io,
                                                                  const __grid_constant__ CUtensorMap tmap) {
  __shared__ __align__(128) unsigned long long s_key[kPrepSH][kPrepSW];
  __shared__ float4 s_v[kPrepSH][kPrepSW];
  __shared__ float2 s_sem[kPrepSH][kPrepSW];  // (label / 255, prob) of gen_vertexmap.frag's (l, l, l, prob)
  __shared__ float2 s_ero[kPrepSH][kPrepSW];  // (x, w) of the eroded label image: (l, l, l, prob) or (0, 0, 0, 1)
  __shared__ __align__(8) unsigned long long s_bar;
  const int W = kp.W, H = kp.H, Wp = W + 2 * kPrepHalo;
  const int x0 = blockIdx.x * kPrepTX, y0 = blockIdx.y * kPrepTY;
  const int tid = threadIdx.x;
  // ---- stage the key tile (padded column x0 .. x0+37 = image column x0-3 .. x0+34, rows y0-3 .. y0+18) ----
  if (kTma) {
    if (tid == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_bar)));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
      const uint32_t bytes = (uint32_t)sizeof(s_key);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&s_bar)), "r"(bytes) : "memory");
      asm volatile(
          "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
              smem_u32(&s_key[0][0])),
          "l"(reinterpret_cast<uint64_t>(&tmap)), "r"(smem_u32(&s_bar)), "r"(x0), "r"(y0 - kPrepHalo)
          : "memory");
    }
    // every thread waits for the bytes to land (phase 0)
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(&s_bar))
        : "memory");
  }
  // ---- phase 1: resolve the winners of tile + halo 3 ----
  for (int i = tid; i < kPrepSH * kPrepSW; i += kPrepThreads) {
    const int sy = i / kPrepSW, sx = i - sy * kPrepSW;
    const int gy = y0 + sy - kPrepHalo, px = x0 + sx;  // px: padded column
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    float2 sm = make_float2(0.f, 0.f);
    if (gy >= 0 && gy < H && px < Wp) {  // rows outside the image: CLAMP_TO_BORDER 0; columns: mirrored pads
      unsigned long long key = kTma ? s_key[sy][sx] : io.keys[(size_t)gy * Wp + px];
      if (key != ~0ull) {
        uint32_t k = (uint32_t)(key & 0xffffffffull);
        float4 p4 = __ldg(io.pts + k);
        float label = 0.0f, prob = 0.0f;
        if (io.labels) {  // Q1: attribute offsets 16 / 20 bytes on stride-4 buffers (Preprocessing.cpp:142-145)
          uint32_t li = kp.label_offset_quirk ? k + 4 : k;
          if (li < io.n) label = __ldg(io.labels + li);
        }
        if (io.probs) {
          uint32_t pi = kp.label_offset_quirk ? k + 5 : k;
          if (pi < io.n) prob = __ldg(io.probs + pi);
        }
        if (!(io.isfirst && is_movable(label))) v = make_float4(p4.x, p4.y, p4.z, 1.0f);  // .vert:95-102
        sm = make_float2(label / 255.0f, prob);                                            // .frag:20
      }
    }
    s_v[sy][sx] = v;
    s_sem[sy][sx] = sm;
  }
  __syncthreads();
  // ---- phase 2: label erosion (gen_normalmap.frag:69-85) on tile + halo 2 ----
  for (int i = tid; i < (kPrepSH - 2) * (kPrepSW - 2); i += kPrepThreads) {
    const int sy = 1 + i / (kPrepSW - 2), sx = 1 + (i - (sy - 1) * (kPrepSW - 2));
    const int gy = y0 + sy - kPrepHalo;
    float2 ero = make_float2(0.f, 0.f);  // rows outside the image sample as border colour 0
    if (gy >= 0 && gy < H) {
      ero = make_float2(0.f, 1.f);       // Q2: pixels without a vertex carry (0,0,0,1)
      if (s_v[sy][sx].w > 0.0f) {
        const float2 sp = s_sem[sy][sx];
        ero = sp;
        const float pl = sp.x;
        const float ul = s_sem[sy][sx + 1].x, vl = s_sem[sy + 1][sx].x, sl = s_sem[sy][sx - 1].x, tl = s_sem[sy - 1][sx].x;
        if ((pl != ul && ul != 0.0f) || (pl != vl && vl != 0.0f) || (pl != sl && sl != 0.0f) || (pl != tl && tl != 0.0f))
          ero = make_float2(0.f, 1.f);
      }
    }
    s_ero[sy][sx] = ero;
  }
  __syncthreads();
  // ---- phase 3: the block's own pixels: normal, flood fill, radius; every output written once ----
  for (int i = tid; i < kPrepTX * kPrepTY; i += kPrepThreads) {
    const int ty = i / kPrepTX, tx = i - ty * kPrepTX;
    const int gx = x0 + tx, gy = y0 + ty;
    if (gx >= W || gy >= H) continue;
    const int sx = tx + kPrepHalo, sy = ty + kPrepHalo;
    const size_t pix = (size_t)gy * W + gx;
    const float4 P = s_v[sy][sx];
    float4 nrm = make_float4(0.f, 0.f, 0.f, 1.f);  // Q2
    if (P.w > 0.0f) {                              // gen_normalmap.frag:47-66, 92-98
      float nw = 1.0f;
      const float4 U = s_v[sy][sx + 1], V = s_v[sy + 1][sx], S = s_v[sy][sx - 1], T = s_v[sy - 1][sx];
      if (U.w < 1.0f && V.w < 1.0f) nw = 0.0f;
      if (S.w < 1.0f && T.w < 1.0f) nw = 0.0f;
      if (!(U.w > 0.5f) || !(V.w > 0.5f)) nw = 0.0f;
      if (nw > 0.0f) {
        V3 pp = mk3(P.x, P.y, P.z);
        V3 u = normalize3(sub3(mk3(U.x, U.y, U.z), pp));
        V3 v = normalize3(sub3(mk3(V.x, V.y, V.z), pp));
        V3 w = cross3(u, v);
        float len = len3(w);
        nrm = make_float4(w.x / len, w.y / len, w.z / len, (len > 0.0000001f) ? 1.0f : 0.0f);
      } else {
        nrm = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    // floodfill.frag:34-84
    const float2 e0 = s_ero[sy][sx];
    float4 out = make_float4(e0.x, e0.x, e0.x, e0.y);
    if (e0.x == 0.0f) {
      const float lp = len3(mk3(P.x, P.y, P.z));
      bool done = false;
#pragma unroll
      for (int offset = 1; offset < 3; ++offset) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (done) continue;
          const int qx = sx + ((k == 0) ? offset : (k == 2 ? -offset : 0));
          const int qy = sy + ((k == 1) ? offset : (k == 3 ? -offset : 0));
          const float2 ql = s_ero[qy][qx];
          if (ql.x != 0.0f) {
            const float4 Q = s_v[qy][qx];
            const float lq = len3(mk3(Q.x, Q.y, Q.z));
            if (fabsf(lp - lq) < 0.007f * lp) {
              out = make_float4(ql.x, ql.x, ql.x, ql.y / (float)(offset + 1));
              done = true;
            }
          }
        }
      }
    }
    io.vertex[pix] = P;
    io.normal[pix] = nrm;
    io.semantic[pix] = out;
    if (io.radius_map) {  // init_radiusConf.vert:41-68
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      V3 v = mk3(P.x, P.y, P.z), n = mk3(nrm.x, nrm.y, nrm.z);
      float d = len3(v);
      V3 view_dir = divs3(neg3(v), d);
      float angle = dot3(n, view_dir);
      if (P.w > 0.5f && nrm.w > 0.5f && angle > kp.radconf_angle_thresh) {
        float c = angle < 0.5f ? 0.5f : (angle > 1.0f ? 1.0f : angle);
        float radius = ((1.41f * d) * kp.pixel_size) / c;
        float lo = radius > kp.min_radius ? radius : kp.min_radius;
        radius = lo < kp.max_radius ? lo : kp.max_radius;
        o.x = radius;
        o.w = 1.0f;  // Q3: the confidence channel stays 0
      }
      io.radius_map[pix] = o;
    }
    if (io.index_keys) io.index_keys[pix] = ~0ull;
    if (io.integrated) io.integrated[pix] = 0;
    if (io.group_counts)  // all of them, also on an image of fewer pixels (see k_radius)
      for (size_t g = pix; g < (size_t)kGroupCounts; g += (size_t)W * H) io.group_counts[g] = 0;
    // re-arm the other key image (own pixel and its mirror copies in the pads)
    unsigned long long* row = io.keys_next + (size_t)gy * Wp;
    row[gx + kPrepHalo] = ~0ull;
    if (gx < kPrepHalo) row[gx + kPrepHalo + W] = ~0ull;
    if (gx >= W - kPrepHalo) row[gx + kPrepHalo - W] = ~0ull;
  }
}

// ---- tensor map of the padded key image (driver entry point fetched through the runtime: no link against libcuda) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool make_key_tensor_map(CUtensorMap* out, const unsigned long long* keys, int W, int H) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p) {
      cudaGetLastError();
      return false;
    }
    fn = (EncodeTiledFn)p;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)(W + 2 * kPrepHalo), (cuuint64_t)H};
  const cuuint64_t strides[1] = {(cuuint64_t)(W + 2 * kPrepHalo) * 8};
  const cuuint32_t box[2] = {(cuuint32_t)kPrepSW, (cuuint32_t)kPrepSH};
  const cuuint32_t estr[2] = {1, 1};
  return fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, (void*)keys, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

size_t preprocess_key_elems(int W, int H) { return (size_t)(W + 2 * kPrepHalo) * H; }

void launch_preprocess(const Launch& L, const KParams& kp, const float4* pts, const float* labels, const float* probs,
                       uint32_t n, uint32_t timestamp, PrepKeys& keys, FrameDev out, float4* radius_map,
                       unsigned long long* index_keys, uint8_t* integrated, uint32_t* group_counts,
                       const DeskewArgs* deskew) {
  unsigned long long* cur = keys.img[keys.cur];
  unsigned long long* nxt = keys.img[keys.cur ^ 1];
  if (n > 0) {
    {
      ScopedKernel sk(L, K_PROJECT_SCATTER);
      if (deskew)
        k_project_scatter<true><<<(n + 255) / 256, 256, 0, L.stream>>>(kp, pts, n, cur, *deskew);
      else
        k_project_scatter<false><<<(n + 255) / 256, 256, 0, L.stream>>>(kp, pts, n, cur, DeskewArgs{});
    }
    if (deskew) pts = deskew->out;  // the tile pass resolves the winners from the deskewed points
  }
  PrepIO io{pts, labels, probs, n, timestamp < 10 ? 1 : 0, cur, nxt, out.vertex, out.normal, out.semantic, radius_map,
            index_keys, integrated, group_counts};
  dim3 grid((kp.W + kPrepTX - 1) / kPrepTX, (kp.H + kPrepTY - 1) / kPrepTY);
  {
    ScopedKernel sk(L, K_PREPROCESS_TILE);
    if (keys.tmap_ok[keys.cur])
      k_preprocess_tile<true><<<grid, kPrepThreads, 0, L.stream>>>(kp, io, keys.tmap[keys.cur]);
    else
      k_preprocess_tile<false><<<grid, kPrepThreads, 0, L.stream>>>(kp, io, keys.tmap[keys.cur]);
  }
  keys.cur ^= 1;
}

// ------------------------------------------------------------------------------------------------------------
// Per-point labels (DESIGN.md section 13): one thread per point, after the scan's last model render. The key image the
// scan's tile pass read stays untouched until the next scan's tile pass re-arms it (nothing else writes PrepKeys), so
// WON is the comparison of the point's own key with the pixel's.
// ------------------------------------------------------------------------------------------------------------
// rintf(255 x) as an unsigned id; NaN and negatives give 0, values past the range saturate (the oracle's rule)
__device__ __forceinline__ uint32_t label_id(float x) {
  const float f = rintf(x * 255.0f);
  return f > 0.0f ? (f < 4294967296.0f ? (uint32_t)f : 0xffffffffu) : 0u;
}

template <bool kDeskew>
__global__ void __launch_bounds__(256) k_point_labels(KParams kp, PointLabelIO io, DeskewArgs dk) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= io.n) return;
  const float4 p4 = k1_point<kDeskew>(io.pts, i, dk);
  const V3 pos = mk3(p4.x, p4.y, p4.z);
  int pixel = -1, map_pixel = -1;
  uint32_t flags = 0, frame_label = 0, map_label = 0;
  float frame_prob = 0.0f, map_prob = 0.0f, map_range = 0.0f;
  int ix, iy;
  uint32_t d24;
  if (k1_project(kp, pos, &ix, &iy, &d24)) {
    pixel = iy * kp.W + ix;
    const unsigned long long key = ((unsigned long long)d24 << 32) | (unsigned long long)i;
    if (io.keys[(size_t)iy * (kp.W + 6) + ix + 3] == key) flags |= SB_POINT_WON;
    if (io.frame.vertex[pixel].w > 0.0f) flags |= SB_POINT_VERTEX;
    if (io.integrated[pixel]) flags |= SB_POINT_INTEGRATED;
    const float4 s = io.frame.semantic[pixel];
    frame_label = label_id(s.x);
    frame_prob = s.w;
    int mx, my;
    if (k1_pixel(pos, len3(pos), kp.Wm, kp.Hm, kp.m_fov_up, kp.m_fov, &mx, &my)) {
      map_pixel = my * kp.Wm + mx;
      if (io.model.vertex) {
        const float4 mv = io.model.vertex[map_pixel];
        if (mv.w > 0.0f) {
          const float4 ms = io.model.semantic[map_pixel];
          flags |= SB_POINT_MAP;
          map_label = label_id(ms.x);
          map_prob = ms.w;
          map_range = len3(mk3(mv.x, mv.y, mv.z));
        }
      }
    }
  }
  uint4* out = reinterpret_cast<uint4*>(io.out + i);  // 32 bytes: two 16-byte stores
  out[0] = make_uint4((uint32_t)pixel, flags, frame_label, __float_as_uint(frame_prob));
  out[1] = make_uint4((uint32_t)map_pixel, map_label, __float_as_uint(map_prob), __float_as_uint(map_range));
}

void launch_point_labels(const Launch& L, const KParams& kp, const PointLabelIO& io, const DeskewArgs* deskew) {
  if (io.n == 0) return;
  ScopedKernel sk(L, K_POINT_LABELS);
  if (deskew)
    k_point_labels<true><<<(io.n + 255) / 256, 256, 0, L.stream>>>(kp, io, *deskew);
  else
    k_point_labels<false><<<(io.n + 255) / 256, 256, 0, L.stream>>>(kp, io, DeskewArgs{});
}

}  // namespace sb
