// TEST SCAFFOLDING ONLY -- runs the per-tile device function of neurad-studio_b200/csrc/lidar_eval.cuh on the host.
//
// Same register blocks, the same padded target tiles and the same per-pair arithmetic (explicit FMAs) as
// chamfer_min_kernel, so the minima are the kernel's bit for bit; the target split of the grid only changes which CTA
// finds a minimum, not its value.  Never linked into libb200nerf.so.
#include <cstdint>

#include "../../neurad-studio_b200/csrc/lidar_eval.cuh"

using namespace nff;

extern "C" int emul_chamfer_min(const float* src, int64_t n_src, int src_stride, const float* dst, int64_t n_dst,
                                int dst_stride, float* out) {
  if (n_src < 1 || n_dst < 1 || src_stride < 3 || dst_stride < 3) return -1;
  static thread_local float tile[kChamferTile * 4];
  const int64_t block = (int64_t)kChamferThreads * kChamferPts;
  for (int64_t b0 = 0; b0 < n_src; b0 += block) {
    for (int tid = 0; tid < kChamferThreads; ++tid) {
      float sx[kChamferPts], sy[kChamferPts], sz[kChamferPts], m[kChamferPts];
      for (int p = 0; p < kChamferPts; ++p) {
        const float* s = src + chamfer_row(b0 + tid + p * kChamferThreads, n_src) * src_stride;
        sx[p] = s[0];
        sy[p] = s[1];
        sz[p] = s[2];
        m[p] = INFINITY;
      }
      for (int64_t t0 = 0; t0 < n_dst; t0 += kChamferTile) {
        for (int k = 0; k < kChamferTile; ++k) {
          const float* d = dst + chamfer_row(t0 + k, n_dst) * dst_stride;
          tile[4 * k] = d[0];
          tile[4 * k + 1] = d[1];
          tile[4 * k + 2] = d[2];
          tile[4 * k + 3] = 0.f;
        }
        chamfer_tile(tile, sx, sy, sz, m);
      }
      for (int p = 0; p < kChamferPts; ++p) {
        const int64_t i = b0 + tid + p * kChamferThreads;
        // through the key of the kernel's atomicMin and back
        if (i < n_src) out[i] = chamfer_unkey(chamfer_key(m[p]));
      }
    }
  }
  return 0;
}
