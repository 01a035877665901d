/* suma_b200_deskew.h -- the host side of per-point deskewing (DESIGN.md section 11), shared by libsuma_b200 and the CPU
 * oracle so that both hand the same fp32 motion to the per-point formula.
 *
 * The motion over one sweep is a rigid transform M (column-major doubles): the increment the next Gauss-Newton run starts
 * from. It is split into an axis-angle omega = log_SO3(R_M) and the translation t_M, evaluated once per scan in fp64 and
 * rounded once to fp32. The per-point formula itself (sweep time, Exp((s - s_ref) omega) p + (s - s_ref) t_M) is restated
 * in fp32 by the kernel (sb_math.cuh) and the oracle (orc_deskew.c).
 */
#ifndef SUMA_B200_DESKEW_H_
#define SUMA_B200_DESKEW_H_

#include <math.h>

/* omega[3], t[3] of M; returns 1 when both round to all zeros (the motion is the identity: points pass through). The
 * angle comes from atan2(|v| / 2, (trace - 1) / 2) with v the skew part of R, which stays accurate for small angles where
 * acos of the trace does not. */
static inline int sb_deskew_motion(const double M[16], float omega[3], float t[3]) {
  const double vx = M[6] - M[9], vy = M[8] - M[2], vz = M[1] - M[4]; /* R32 - R23, R13 - R31, R21 - R12 */
  const double sv = sqrt((vx * vx + vy * vy) + vz * vz);
  const double c = 0.5 * (((M[0] + M[5]) + M[10]) - 1.0);
  double f = 0.0;
  if (sv > 0.0) f = atan2(0.5 * sv, c) / sv;
  omega[0] = (float)(f * vx);
  omega[1] = (float)(f * vy);
  omega[2] = (float)(f * vz);
  t[0] = (float)M[12];
  t[1] = (float)M[13];
  t[2] = (float)M[14];
  for (int i = 0; i < 3; ++i)
    if (omega[i] != 0.0f || t[i] != 0.0f) return 0;
  return 1;
}

#endif /* SUMA_B200_DESKEW_H_ */
