// camera_rays.h -- per-ray camera math of Cameras._generate_rays_from_coords (cameras/cameras.py:633-667, 793-815,
// 898-969) for PERSPECTIVE and FISHEYE cameras with the radial / tangential distortion of camera_utils.py:655-758 and the
// AD datasets' rolling shutter (top-to-bottom, left-to-right, right-to-left).
//
// Every operation is a single IEEE rounding the compiler may not contract (simt.h), in the reference's operation order,
// so the perspective rays are the reference's bits.  The fisheye mapping adds sinf / cosf, which may differ from torch's in
// the last bit.  The functions compile as plain C++ as well (tests/host_emul/emul_camera.cpp).
//
// Reference behaviour kept as it is:
//   * undistortion runs on the normalised coordinates of the pixel and of its +x / +y offsets: exactly 10 Newton steps,
//     a step only where |denominator| > 1e-3 (else 0).  The reference skips it when every parameter is 0; with zero
//     parameters one step returns x unchanged bit for bit, so the host picks the undistorted instance per camera;
//   * ZOD's fisheye is the r^2 polynomial above followed by the equidistant mapping theta = clip(|(u, v)|, 0, pi),
//     direction (u sin(theta) / theta, v sin(theta) / theta, -cos(theta)) -- not OpenCV's fisheye model;
//   * a coordinate exactly on the principal point gives theta = 0 and a NaN direction (0 * 0 / 0), and so NaN pixel_area
//     there and at the left and upper neighbours whose offset coordinates land on it;
//   * "Horizontal_reversed" negates the whole time offset, time_to_center_pixel included.
#pragma once

#include "simt.h"

namespace nff {
using namespace simt;

// b200nerf_camera.rs_direction
enum ShutterDirection : int { kRsVertical = 0, kRsHorizontal = 1, kRsHorizontalReversed = 2 };

struct CameraArgs {
  float c2w[12];
  float fx, fy, cx, cy;
  float dist[6];  // k1, k2, k3, k4, p1, p2
  int height, width, row0, row_step, n_rows, col0, col_step, n_cols;
  float time, vel[3], rs_time, ttc;
  int has_vel, rs_dir;
};

// ((x - cx) / fx, (y - cy) / fy) of the pixel centre (x, y) and of its +x / +y offsets (cameras.py:633-635)
NFF_D void camera_coords(const CameraArgs& a, float x, float y, float c[3][2]) {
  const float u0 = fdiv(fsub(x, a.cx), a.fx), v0 = fdiv(fsub(y, a.cy), a.fy);
  const float u1 = fdiv(fadd(fsub(x, a.cx), 1.0f), a.fx), v1 = fdiv(fadd(fsub(y, a.cy), 1.0f), a.fy);
  c[0][0] = u0, c[0][1] = v0;
  c[1][0] = u1, c[1][1] = v0;
  c[2][0] = u0, c[2][1] = v1;
}

// camera_utils.radial_and_tangential_undistort (camera_utils.py:655-758): (x, y) <- the undistorted coordinates of the
// distorted (xd, yd), k = {k1, k2, k3, k4, p1, p2}
NFF_D void radial_tangential_undistort(const float k[6], float* px, float* py) {
  const float xd = *px, yd = *py;
  const float k1 = k[0], k2 = k[1], k3 = k[2], k4 = k[3], p1 = k[4], p2 = k[5];
  const float p1x2 = fmul(2.0f, p1), p2x2 = fmul(2.0f, p2), k2x2 = fmul(2.0f, k2), k3x3 = fmul(3.0f, k3);
  const float p1x6 = fmul(6.0f, p1), p2x6 = fmul(6.0f, p2);
  float x = xd, y = yd;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {
    const float r = fadd(fmul(x, x), fmul(y, y));
    const float d = fadd(1.0f, fmul(r, fadd(k1, fmul(r, fadd(k2, fmul(r, fadd(k3, fmul(r, k4))))))));
    const float fx = fsub(fadd(fadd(fmul(d, x), fmul(fmul(p1x2, x), y)), fmul(p2, fadd(r, fmul(fmul(2.0f, x), x)))), xd);
    const float fy = fsub(fadd(fadd(fmul(d, y), fmul(fmul(p2x2, x), y)), fmul(p1, fadd(r, fmul(fmul(2.0f, y), y)))), yd);
    const float d_r = fadd(k1, fmul(r, fadd(k2x2, fmul(r, fadd(k3x3, fmul(fmul(r, 4.0f), k4))))));
    const float d_x = fmul(fmul(2.0f, x), d_r), d_y = fmul(fmul(2.0f, y), d_r);
    const float fx_x = fadd(fadd(fadd(d, fmul(d_x, x)), fmul(p1x2, y)), fmul(p2x6, x));
    const float fx_y = fadd(fadd(fmul(d_y, x), fmul(p1x2, x)), fmul(p2x2, y));
    const float fy_x = fadd(fadd(fmul(d_x, y), fmul(p2x2, y)), fmul(p1x2, x));
    const float fy_y = fadd(fadd(fadd(d, fmul(d_y, y)), fmul(p2x2, x)), fmul(p1x6, y));
    const float den = fsub(fmul(fy_x, fx_y), fmul(fx_x, fy_y));
    const float xn = fsub(fmul(fx, fy_y), fmul(fy, fx_y));
    const float yn = fsub(fmul(fy, fx_x), fmul(fx, fy_x));
    const bool step = fabsf(den) > 1e-3f;
    x = fadd(x, step ? fdiv(xn, den) : 0.0f);
    y = fadd(y, step ? fdiv(yn, den) : 0.0f);
  }
  *px = x, *py = y;
}

// camera-frame direction of normalised coordinates (u, v) after the OpenGL flip v -> -v (cameras.py:667, 796-815)
template <bool kFisheye>
NFF_D void camera_local_dir(float u, float v, float out[3]) {
  v = -v;
  if (!kFisheye) {
    out[0] = u, out[1] = v, out[2] = -1.0f;
  } else {
    float theta = fsqrt(fadd(fmul(u, u), fmul(v, v)));
    if (theta > 3.14159265358979323846f) theta = 3.14159265358979323846f;  // torch.clip(theta, 0, pi): keeps NaN
    const float s = sinf(theta);
    out[0] = fdiv(fmul(u, s), theta);
    out[1] = fdiv(fmul(v, s), theta);
    out[2] = -cosf(theta);
  }
}

// rotate by c2w: sum over columns of dir_j * R[i][j] (cameras.py:903-905), then normalise (camera_utils.py:596-610)
NFF_D void camera_world_dir(const float c2w[12], const float l[3], float out[3]) {
  float r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r[i] = fadd(fadd(fmul(l[0], c2w[4 * i + 0]), fmul(l[1], c2w[4 * i + 1])), fmul(l[2], c2w[4 * i + 2]));
  float n = fsqrt(fadd(fadd(fmul(r[0], r[0]), fmul(r[1], r[1])), fmul(r[2], r[2])));
  n = fmaxf(n, 8.8817841970012523e-16f);  // camera_utils.py:30 (_EPS = 4 * float64 eps, cast to fp32)
  out[0] = fdiv(r[0], n), out[1] = fdiv(r[1], n), out[2] = fdiv(r[2], n);
}

// rolling-shutter time offset of the pixel centre (x, y) (cameras.py:941-952)
NFF_D float rolling_shutter_offset(const CameraArgs& a, float x, float y) {
  if (a.rs_dir == kRsVertical) return fadd(fmul(fsub(fdiv(y, (float)a.height), 0.5f), a.rs_time), a.ttc);
  const float t = fadd(fmul(fsub(fdiv(x, (float)a.width), 0.5f), a.rs_time), a.ttc);
  return a.rs_dir == kRsHorizontalReversed ? -t : t;
}

// ray i of the strided pixel grid row0 + r * row_step, col0 + c * col_step
template <bool kFisheye, bool kDistorted>
NFF_D void camera_ray(const CameraArgs& a, int64_t i, float o[3], float d0[3], float* area, float* t) {
  const int r = (int)(i / a.n_cols), c = (int)(i % a.n_cols);
  const float y = (float)(a.row0 + r * a.row_step) + 0.5f, x = (float)(a.col0 + c * a.col_step) + 0.5f;
  float uv[3][2];
  camera_coords(a, x, y, uv);
  float d[3][3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    if (kDistorted) radial_tangential_undistort(a.dist, &uv[j][0], &uv[j][1]);
    float l[3];
    camera_local_dir<kFisheye>(uv[j][0], uv[j][1], l);
    camera_world_dir(a.c2w, l, d[j]);
  }
  float ex[3], ey[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ex[k] = fsub(d[0][k], d[1][k]);
    ey[k] = fsub(d[0][k], d[2][k]);
    d0[k] = d[0][k];
  }
  const float dx = fsqrt(fadd(fadd(fmul(ex[0], ex[0]), fmul(ex[1], ex[1])), fmul(ex[2], ex[2])));
  const float dy = fsqrt(fadd(fadd(fmul(ey[0], ey[0]), fmul(ey[1], ey[1])), fmul(ey[2], ey[2])));
  *area = fmul(dx, dy);
  o[0] = a.c2w[3], o[1] = a.c2w[7], o[2] = a.c2w[11];
  *t = a.time;
  if (a.has_vel) {
    const float toff = rolling_shutter_offset(a, x, y);
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = fadd(o[k], fmul(a.vel[k], toff));
    *t = fadd(*t, toff);
  }
}

}  // namespace nff
