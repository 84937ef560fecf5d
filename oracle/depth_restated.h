/* TEST INFRASTRUCTURE ONLY -- restatement of Fiesta::DepthConversion (FIESTA include/Fiesta.h:319-382), shared by
 * both oracles (the header needs cv_bridge/OpenCV/PCL and cannot be compiled here).  Fills `cloud` (3 floats per point, pixel
 * order) from a uint16 millimetre depth image; returns the number of points.
 *   image_cnt : value of image_cnt_ AFTER the increment at :321 (1 for the first image)
 *   last      : previous image (ignored when use_filter == 0 or image_cnt == 1)
 *   m_rel     : last_transform_.inverse() * transform_ , row-major (the per-pixel product at :366 is constant over the image;
 *               the caller supplies it because Eigen's 4x4 inverse is not restated here) */
#ifndef FIESTA_ORACLE_DEPTH_RESTATED_H
#define FIESTA_ORACLE_DEPTH_RESTATED_H
#include <math.h>
#include <stdint.h>
typedef struct {
  double fx, fy, cx, cy;              /* focal_x_, focal_y_, center_x_, center_y_ */
  int use_filter, margin;             /* use_depth_filter_, depth_filter_margin_ */
  double max_dist, min_dist, tolerance;
} oracle_depth_params;
static long oracle_depth_conversion(const uint16_t *img, const uint16_t *last, int rows, int cols, unsigned image_cnt,
                                    const oracle_depth_params *p, const double *m_rel, float *cloud) {
  const double k_depth_scaling_factor = 1000.0;                                   /* :328 */
  long n = 0;
  if (!p->use_filter) {                                                           /* :340-351 */
    for (int v = 0; v < rows; v++)
      for (int u = 0; u < cols; u++) {
        const double depth = img[(long)v * cols + u] / k_depth_scaling_factor;
        cloud[3 * n] = (float)((u - p->cx) * depth / p->fx);
        cloud[3 * n + 1] = (float)((v - p->cy) * depth / p->fy);
        cloud[3 * n + 2] = (float)depth;
        n++;
      }
    return n;
  }
  if (image_cnt == 1) return 0;                                                   /* :353 */
  for (int v = p->margin; v < rows - p->margin; v++)                              /* :356-378 */
    for (int u = p->margin; u < cols - p->margin; u++) {
      const double depth = img[(long)v * cols + u] / k_depth_scaling_factor;
      const float px = (float)((u - p->cx) * depth / p->fx), py = (float)((v - p->cy) * depth / p->fy), pz = (float)depth;
      if (depth > p->max_dist || depth < p->min_dist) continue;
      double h[4];
      for (int r = 0; r < 4; ++r)
        h[r] = ((m_rel[4 * r] * (double)px + m_rel[4 * r + 1] * (double)py) + m_rel[4 * r + 2] * (double)pz) + m_rel[4 * r + 3] * 1.0;
      const double cx_ = h[0] / h[3], cy_ = h[1] / h[3], cz_ = h[2] / h[3];
      const double uu = cx_ * p->fx / cz_ + p->cx, vv = cy_ * p->fy / cz_ + p->cy;
      if (uu >= 0 && uu < cols && vv >= 0 && vv < rows) {
        if (fabs(last[(long)(int)vv * cols + (int)uu] / k_depth_scaling_factor - cz_) < p->tolerance) {
          cloud[3 * n] = px; cloud[3 * n + 1] = py; cloud[3 * n + 2] = pz;
          n++;
        }
      }
    }
  return n;
}
#endif
