/* orc_deskew.h -- TEST INFRASTRUCTURE (CPU oracle): per-point deskewing before K1 (no counterpart in the reference;
 * DESIGN.md section 11). Built into its own library against liborc.so by oracle/deskew.py. */
#ifndef ORC_DESKEW_H_
#define ORC_DESKEW_H_

#include "orc.h"

#ifdef __cplusplus
extern "C" {
#endif

/* mode 0 off, 1 per-point times (times[n]), 2 azimuth; motion: the sweep's motion M (column-major, NULL = identity).
 * out4 = the moved points (w carried through). Returns 0 when nothing moved (mode 0 or M rounds to the identity: out4 is a
 * copy of pts4), 1 otherwise. */
int orc_deskew_points(const float* pts4, const float* times, uint32_t n, int32_t mode, float ref_time,
                      float start_azimuth, int32_t clockwise, const double motion[16], float* out4);
/* orc_preprocess of the deskewed points */
void orc_preprocess_deskew(const orc_params* p, const float* pts4, const float* labels, const float* probs,
                           const float* times, uint32_t n, uint32_t timestamp, int32_t mode, float ref_time,
                           float start_azimuth, int32_t clockwise, const double motion[16], float* vertex_map,
                           float* normal_map, float* semantic_map);
/* orc_slam_process_scan of the points deskewed with the slam's own lastIncrement_ when the scan begins (the motion the
 * next Gauss-Newton run starts from); times: NULL unless mode is 1; mode 0: orc_slam_process_scan itself */
void orc_slam_process_scan_timed(orc_slam* s, const float* pts4, const float* labels, const float* probs,
                                 const float* times, uint32_t n, int32_t mode, float ref_time, float start_azimuth,
                                 int32_t clockwise);

#ifdef __cplusplus
}
#endif
#endif /* ORC_DESKEW_H_ */
