// TEST SCAFFOLDING ONLY -- runs camera_ray() of neurad-studio_b200/csrc/camera_rays.h on the host, ray by ray, with the
// instance raygen_camera_kernel uses for the same descriptor.  Never linked into libb200nerf.so.
#include <cstdint>

#include "../../neurad-studio_b200/csrc/camera_rays.h"

using namespace nff;

// f = {c2w[12], fx, fy, cx, cy, k1..k4, p1, p2, time, vel[3], rs_time, ttc}; i = {height, width, row0, row_step, n_rows, col0,
// col_step, n_cols, has_vel, rs_dir, fisheye}
extern "C" int emul_raygen_camera(const float* f, const int* iv, float* origins, float* dirs, float* area, float* times) {
  CameraArgs a{};
  for (int k = 0; k < 12; ++k) a.c2w[k] = f[k];
  a.fx = f[12], a.fy = f[13], a.cx = f[14], a.cy = f[15];
  bool distorted = false;
  for (int k = 0; k < 6; ++k) distorted |= (a.dist[k] = f[16 + k]) != 0.0f;
  a.time = f[22];
  for (int k = 0; k < 3; ++k) a.vel[k] = f[23 + k];
  a.rs_time = f[26], a.ttc = f[27];
  a.height = iv[0], a.width = iv[1], a.row0 = iv[2], a.row_step = iv[3], a.n_rows = iv[4];
  a.col0 = iv[5], a.col_step = iv[6], a.n_cols = iv[7], a.has_vel = iv[8], a.rs_dir = iv[9];
  const bool fisheye = iv[10] != 0;
  const int64_t n = (int64_t)a.n_rows * a.n_cols;
  for (int64_t i = 0; i < n; ++i) {
    float o[3], d[3];
    if (fisheye && distorted) camera_ray<true, true>(a, i, o, d, &area[i], &times[i]);
    else if (fisheye) camera_ray<true, false>(a, i, o, d, &area[i], &times[i]);
    else if (distorted) camera_ray<false, true>(a, i, o, d, &area[i], &times[i]);
    else camera_ray<false, false>(a, i, o, d, &area[i], &times[i]);
    for (int k = 0; k < 3; ++k) origins[3 * i + k] = o[k], dirs[3 * i + k] = d[k];
  }
  return 0;
}
