// sb_math.cuh -- scalar arithmetic of the hot path, shared by every kernel and by the host-side Gauss-Newton.
//
// Bit-reproducibility contract: the translation units that include this header are compiled with -fmad=false
// (device) and -ffp-contract=off (host), so every +,*,/,sqrt below is one correctly rounded IEEE-754 operation and
// a kernel gives the same bits on any launch shape. Transcendentals are fixed polynomial evaluations (Cephes-style
// single precision), because GLSL leaves atan/asin/acos/sin/exp/log precision implementation-defined
// (the reference calls them at gen_vertexmap.vert:80-81, Frame2Model_jacobians.geom:58-59,
// render_surfels.geom:49-50, update_surfels.vert:116-121,238-243).
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define SB_HD __host__ __device__ __forceinline__

namespace sbm {

constexpr float kPi = 3.14159265358979323846f;
constexpr float kInvPi = 0.31830988618379067154f;
constexpr float kPiO2 = 1.57079632679489661923f;
constexpr float kPiO4 = 0.78539816339744830962f;
constexpr float kRad2Deg = 57.29577951308232f;  // GLSL degrees()

SB_HD float bits2f(uint32_t u) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
SB_HD uint32_t f2bits(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}

SB_HD float atan_poly(float t) {  // |t| <= tan(pi/8)
  float z = t * t;
  float p = 8.05374449538e-2f;
  p = p * z - 1.38776856032e-1f;
  p = p * z + 1.99777106478e-1f;
  p = p * z - 3.33329491539e-1f;
  return (p * z) * t + t;
}

// GLSL atan(y, x); atan(0, 0) := 0
SB_HD float atan2f_(float y, float x) {
  float ax = fabsf(x), ay = fabsf(y);
  bool swap = ay > ax;
  float hi = swap ? ay : ax;
  float lo = swap ? ax : ay;
  if (hi == 0.0f) return 0.0f;
  float t = lo / hi;
  float r;
  if (t > 0.4142135623730950f)
    r = kPiO4 + atan_poly((t - 1.0f) / (t + 1.0f));
  else
    r = atan_poly(t);
  if (swap) r = kPiO2 - r;
  if (x < 0.0f) r = kPi - r;
  if (y < 0.0f) r = -r;
  return r;
}

SB_HD float asinf_(float x) {
  float a = fabsf(x);
  if (a < 1.0e-4f) return x;
  bool flag = a > 0.5f;
  float z, w;
  if (flag) {
    z = 0.5f * (1.0f - a);
    w = sqrtf(z);
  } else {
    w = a;
    z = w * w;
  }
  float p = 4.2163199048e-2f;
  p = p * z + 2.4181311049e-2f;
  p = p * z + 4.5470025998e-2f;
  p = p * z + 7.4953002686e-2f;
  p = p * z + 1.6666752422e-1f;
  float r = (p * z) * w + w;
  if (flag) {
    r = r + r;
    r = kPiO2 - r;
  }
  return x < 0.0f ? -r : r;
}

SB_HD float acosf_(float x) {
  if (x < -0.5f) return kPi - 2.0f * asinf_(sqrtf(0.5f * (1.0f + x)));
  if (x > 0.5f) return 2.0f * asinf_(sqrtf(0.5f * (1.0f - x)));
  return kPiO2 - asinf_(x);
}

SB_HD float sinf_(float xx) {
  if (xx != xx) return xx;
  float x = fabsf(xx);
  bool neg = xx < 0.0f;
  if (x > 8192.0f) return 0.0f;
  int j = (int)(1.27323954473516f * x);
  float y = (float)j;
  if (j & 1) {
    j += 1;
    y += 1.0f;
  }
  j &= 7;
  if (j > 3) {
    neg = !neg;
    j -= 4;
  }
  x = ((x - y * 0.78515625f) - y * 2.4187564849853515625e-4f) - y * 3.77489497744594108e-8f;
  float z = x * x, r, p;
  if (j == 1 || j == 2) {
    p = 2.443315711809948e-5f;
    p = p * z - 1.388731625493765e-3f;
    p = p * z + 4.166664568298827e-2f;
    r = (p * z) * z;
    r = r - 0.5f * z;
    r = r + 1.0f;
  } else {
    p = -1.9515295891e-4f;
    p = p * z + 8.3321608736e-3f;
    p = p * z - 1.6666654611e-1f;
    r = (p * z) * x + x;
  }
  return neg ? -r : r;
}

SB_HD float pow2i(int n) { return bits2f((uint32_t)(n + 127) << 23); }

SB_HD float expf_(float x) {
  if (x != x) return x;
  if (x > 88.0f) return bits2f(0x7f800000u);
  if (x < -87.0f) return 0.0f;
  float fn = floorf(1.44269504088896341f * x + 0.5f);
  int n = (int)fn;
  x = x - fn * 0.693359375f;
  x = x - fn * (-2.12194440e-4f);
  float z = x * x;
  float p = 1.9875691500e-4f;
  p = p * x + 1.3981999507e-3f;
  p = p * x + 8.3334519073e-3f;
  p = p * x + 4.1665795894e-2f;
  p = p * x + 1.6666665459e-1f;
  p = p * x + 5.0000001201e-1f;
  float r = (p * z + x) + 1.0f;
  int n1 = n >> 1, n2 = n - n1;
  return (r * pow2i(n1)) * pow2i(n2);
}

SB_HD float logf_(float x) {
  if (x != x) return x;
  if (x < 0.0f) return bits2f(0x7fc00000u);
  if (x == 0.0f) return bits2f(0xff800000u);
  if (x == bits2f(0x7f800000u)) return x;
  int e = 0;
  uint32_t b = f2bits(x);
  if (((b >> 23) & 0xffu) == 0u) {
    x = x * 8388608.0f;
    b = f2bits(x);
    e = -23;
  }
  e += (int)((b >> 23) & 0xffu) - 126;
  float m = bits2f((b & 0x807fffffu) | 0x3f000000u);
  if (m < 0.707106781186547524f) {
    e -= 1;
    m = (m + m) - 1.0f;
  } else {
    m = m - 1.0f;
  }
  float z = m * m;
  float p = 7.0376836292e-2f;
  p = p * m - 1.1514610310e-1f;
  p = p * m + 1.1676998740e-1f;
  p = p * m - 1.2420140846e-1f;
  p = p * m + 1.4249322787e-1f;
  p = p * m - 1.6668057665e-1f;
  p = p * m + 2.0000714765e-1f;
  p = p * m - 2.4999993993e-1f;
  p = p * m + 3.3333331174e-1f;
  float y = (p * m) * z;
  float fe = (float)e;
  y = y + (-2.12194440e-4f) * fe;
  y = y + (-0.5f) * z;
  float r = m + y;
  r = r + 0.693359375f * fe;
  return r;
}

// GLSL round(): ties away from zero (labels are integers +- rounding noise, ties never occur on the path)
SB_HD float roundf_(float x) { return roundf(x); }

// ---- fp64 sin/cos for SE3::exp: one fixed polynomial so the host and the device Gauss-Newton loops agree bit-wise
SB_HD void sincos_(double xx, double* s, double* c) {
  const double S0 = 1.58962301576546568060E-10, S1 = -2.50507477628578072866E-8, S2 = 2.75573136213857245213E-6,
               S3 = -1.98412698295895385996E-4, S4 = 8.33333333332211858878E-3, S5 = -1.66666666666666307295E-1;
  const double C0 = -1.13585365213876817300E-11, C1 = 2.08757008419747316778E-9, C2 = -2.75573141792967388112E-7,
               C3 = 2.48015872888517045348E-5, C4 = -1.38888888888730564116E-3, C5 = 4.16666666666665929218E-2;
  double x = fabs(xx);
  if (!(x < 1.0e9)) {
    *s = xx - xx;
    *c = xx - xx;
    return;
  }
  long long j = (long long)(x * 1.27323954473516268615);
  double y = (double)j;
  if (j & 1) {
    j += 1;
    y += 1.0;
  }
  j &= 7;
  bool sneg = xx < 0.0, cneg = false;
  if (j > 3) {
    sneg = !sneg;
    cneg = !cneg;
    j -= 4;
  }
  if (j > 1) cneg = !cneg;
  double z = ((x - y * 7.85398125648498535156E-1) - y * 3.77489470793079817668E-8) - y * 2.69515142907905952645E-15;
  double zz = z * z;
  double ps = S0;
  ps = ps * zz + S1; ps = ps * zz + S2; ps = ps * zz + S3; ps = ps * zz + S4; ps = ps * zz + S5;
  double pc = C0;
  pc = pc * zz + C1; pc = pc * zz + C2; pc = pc * zz + C3; pc = pc * zz + C4; pc = pc * zz + C5;
  double vs = z + (z * zz) * ps;
  double vc = (1.0 - 0.5 * zz) + (zz * zz) * pc;
  double sv = (j == 1 || j == 2) ? vc : vs;
  double cv = (j == 1 || j == 2) ? vs : vc;
  *s = sneg ? -sv : sv;
  *c = cneg ? -cv : cv;
}

// ---- 3-vectors with a fixed evaluation order --------------------------------------------------------------
struct V3 {
  float x, y, z;
};
SB_HD V3 mk3(float x, float y, float z) { return V3{x, y, z}; }
SB_HD float dot3(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
SB_HD float len3(V3 a) { return sqrtf(dot3(a, a)); }
SB_HD V3 sub3(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
SB_HD V3 add3(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
SB_HD V3 scale3(float s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
SB_HD V3 divs3(V3 a, float s) { return V3{a.x / s, a.y / s, a.z / s}; }
SB_HD V3 neg3(V3 a) { return V3{-a.x, -a.y, -a.z}; }
SB_HD V3 cross3(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
SB_HD V3 normalize3(V3 a) { return divs3(a, len3(a)); }

// column-major 4x4: M[c*4+r]
SB_HD V3 xform_point(const float* M, V3 p) {
  V3 r;
  r.x = ((M[0] * p.x + M[4] * p.y) + M[8] * p.z) + M[12];
  r.y = ((M[1] * p.x + M[5] * p.y) + M[9] * p.z) + M[13];
  r.z = ((M[2] * p.x + M[6] * p.y) + M[10] * p.z) + M[14];
  return r;
}
SB_HD V3 xform_dir(const float* M, V3 p) {
  V3 r;
  r.x = (M[0] * p.x + M[4] * p.y) + M[8] * p.z;
  r.y = (M[1] * p.x + M[5] * p.y) + M[9] * p.z;
  r.z = (M[2] * p.x + M[6] * p.y) + M[10] * p.z;
  return r;
}
template <typename T>
SB_HD void mat4_mul(const T* A, const T* B, T* C) {
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r)
      C[c * 4 + r] = ((A[0 * 4 + r] * B[c * 4 + 0] + A[1 * 4 + r] * B[c * 4 + 1]) + A[2 * 4 + r] * B[c * 4 + 2]) +
                     A[3 * 4 + r] * B[c * 4 + 3];
}

// spherical projection shared by every pass: x, y in [0,1) image coordinates, z normalised depth
SB_HD void project01(V3 p, float fov_up, float fov, float min_depth, float max_depth, float& x, float& y, float& z) {
  float depth = len3(p);
  float yaw = atan2f_(p.y, p.x);
  float pitch = -asinf_(p.z / depth);
  x = 0.5f * ((-yaw * kInvPi) + 1.0f);
  y = 1.0f - (kRad2Deg * pitch + fov_up) / fov;
  z = (depth - min_depth) / (max_depth - min_depth);
}

// ---- per-point deskewing (DESIGN.md section 11; restated by the oracle in orc_deskew.c) ----
// Sweep time s in [0, 1] of a point. mode 1: the caller's time, clamped, a non-finite one counts as s_ref. mode 2: the
// azimuth fraction frac(dir (a0 - yaw) / 2pi) of the raw point's yaw, dir = +1 for a clockwise spin.
SB_HD float deskew_sweep_time(int mode, float t, float yaw, float ref, float a0, int clockwise) {
  if (mode == 1) {
    if (!(fabsf(t) <= 3.402823466e38f)) return ref;
    return t < 0.0f ? 0.0f : (t > 1.0f ? 1.0f : t);
  }
  const float u = clockwise ? a0 - yaw : yaw - a0;
  const float q = u / 6.28318530717958647692f;
  return q - floorf(q);
}
// p' = Exp(tau w) p + tau t, tau = s - s_ref: Rodrigues with a = sin(th) / th, b = (1 - cos(th)) / th^2 = 2 sin^2(th/2) / th^2
// (no cancellation at small angles). tau == 0: the point's bits pass through (a -0 stays -0).
SB_HD V3 deskew_point(V3 p, float tau, V3 w, V3 t) {
  if (tau == 0.0f) return p;
  const V3 wt = scale3(tau, w);
  const float th2 = dot3(wt, wt);
  float a = 1.0f, b = 0.5f;
  if (th2 > 1e-30f) {
    const float th = sqrtf(th2);
    const float h = sinf_(0.5f * th);
    a = sinf_(th) / th;
    b = (2.0f * (h * h)) / th2;
  }
  const V3 c1 = cross3(wt, p);
  const V3 c2 = cross3(wt, c1);
  return mk3(((p.x + a * c1.x) + b * c2.x) + tau * t.x, ((p.y + a * c1.y) + b * c2.y) + tau * t.y,
             ((p.z + a * c1.z) + b * c2.z) + tau * t.z);
}

// movable classes (color_map.glsl:8-17): car, bicycle, bus, motorcycle, truck, other-vehicle, person, bicyclist,
// motorcyclist
SB_HD bool is_movable(float l) {
  return l == 10.0f || l == 11.0f || l == 13.0f || l == 15.0f || l == 18.0f || l == 20.0f || l == 30.0f ||
         l == 31.0f || l == 32.0f;
}

constexpr uint32_t kDepthClear = 0xFFFFFFu;  // 24-bit depth buffer cleared to 1.0
SB_HD uint32_t depth24(float zw) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__double2ll_rn((double)zw * 16777215.0);
#else
  return (uint32_t)llrint((double)zw * 16777215.0);
#endif
}

// exact accumulation: fp32 term -> Q33.30 fixed point (round to nearest even), summed as int64
SB_HD long long fix30(float t) {
#ifdef __CUDA_ARCH__
  return __float2ll_rn(t * 1073741824.0f);
#else
  return (long long)llrintf(t * 1073741824.0f);
#endif
}

// pack(), color.glsl:32-38
SB_HD float pack_rgb(float r, float g, float b) {
  int rgb = (int)roundf(r * 255.0f);
  rgb = (rgb << 8) + (int)roundf(g * 255.0f);
  rgb = (rgb << 8) + (int)roundf(b * 255.0f);
  return (float)rgb;
}

}  // namespace sbm
