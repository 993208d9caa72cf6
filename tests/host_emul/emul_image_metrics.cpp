// TEST SCAFFOLDING ONLY -- runs the device functions of neurad-studio_b200/csrc/image_metrics.cuh on the host.
//
// The statistics use the kernels' NaN-keeping min / max and image_range; the SSIM walks the kernel's tiles with the
// kernel's shift, row moments (ssim_row_moments), tap order of the vertical pass and ssim_window, so every window's fp32
// value is the device's.  The sums are fp64 in index order (the device's fixed tree is another fp64 order).  Never
// linked into libb200nerf.so.
#include <cstdint>
#include <vector>

#include "../../neurad-studio_b200/csrc/image_metrics.cuh"

using namespace nff;

// out = [(batch + 1)][4] = {mse, psnr, ssim, data_range} of the batch, then of each image; strides = {batch, row, column,
// channel} in elements
extern "C" int emul_image_metrics(const float* a, const float* b, int B, int H, int W, int C, const int64_t* sa,
                                  const int64_t* sb, float data_range, double* out) {
  if (B < 1 || B > kImMaxBlocks || H < kSsimWin || W < kSsimWin || C < 1) return -1;
  const ImageView va{a, sa[0], sa[1], sa[2], sa[3]}, vb{b, sb[0], sb[1], sb[2], sb[3]};
  const StatsWalk w = stats_walk(va, vb, H, W, C);
  float mm[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  std::vector<double> se(B, 0.0);
  for (int bi = 0; bi < B; ++bi)
    for (int r = 0; r < w.n_r1 * w.n_r2; ++r) {
      const int r1 = r / w.n_r2, r2 = r - r1 * w.n_r2;
      const float* ra = a + bi * va.sb + r1 * w.a_r1 + r2 * w.a_r2;
      const float* rb = b + bi * vb.sb + r1 * w.b_r1 + r2 * w.b_r2;
      for (int i = 0; i < w.n_in; ++i) {
        const float x = ra[i * w.a_in], y = rb[i * w.b_in];
        mm[0] = nan_min(mm[0], x);
        mm[1] = nan_max(mm[1], x);
        mm[2] = nan_min(mm[2], y);
        mm[3] = nan_max(mm[3], y);
        const double d = (double)x - (double)y;
        se[bi] += d * d;
      }
    }
  const ImageRange R = image_range(mm[0], mm[1], mm[2], mm[3], data_range);

  const int tiles_x = (W - (kSsimWin - 1) + kSsimTile - 1) / kSsimTile, tiles_y = (H - (kSsimWin - 1) + kSsimTile - 1) / kSsimTile;
  const double n = (double)H * W * C, n_win = (double)(H - (kSsimWin - 1)) * (W - (kSsimWin - 1)) * C;
  std::vector<float> ta(kSsimIn * kSsimIn), tb(kSsimIn * kSsimIn), h(5 * kSsimIn * kSsimTile);
  double se_all = 0.0, ssim_all = 0.0;
  for (int bi = 0; bi < B; ++bi) {
    double ssim_sum = 0.0;
    for (int ty = 0; ty < tiles_y; ++ty)
      for (int tx = 0; tx < tiles_x; ++tx)
        for (int c = 0; c < C; ++c) {
          const int y0 = ty * kSsimTile, x0 = tx * kSsimTile;
          const float* pa = a + bi * va.sb + c * va.sc;
          const float* pb = b + bi * vb.sb + c * vb.sc;
          const int cy = ssim_shift_coord(y0, H), cx = ssim_shift_coord(x0, W);
          const float shift_a = pa[cy * va.sy + cx * va.sx], shift_b = pb[cy * vb.sy + cx * vb.sx];
          for (int r = 0; r < kSsimIn; ++r)
            for (int q = 0; q < kSsimIn; ++q) {
              const int y = y0 + r, x = x0 + q;
              const bool in = y < H && x < W;
              ta[r * kSsimIn + q] = in ? im_sub(pa[y * va.sy + x * va.sx], shift_a) : 0.f;
              tb[r * kSsimIn + q] = in ? im_sub(pb[y * vb.sy + x * vb.sx], shift_b) : 0.f;
            }
          for (int r = 0; r < kSsimIn; ++r)
            for (int q = 0; q < kSsimTile; ++q) {
              float m[5];
              ssim_row_moments(&ta[r * kSsimIn + q], &tb[r * kSsimIn + q], m);
              for (int k = 0; k < 5; ++k) h[(k * kSsimIn + r) * kSsimTile + q] = m[k];
            }
          double tile = 0.0;
          for (int r = 0; r < kSsimTile && y0 + r < H - (kSsimWin - 1); ++r)
            for (int q = 0; q < kSsimTile && x0 + q < W - (kSsimWin - 1); ++q) {
              float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
              for (int i = 0; i < kSsimWin; ++i)
                for (int k = 0; k < 5; ++k) m[k] = fmaf(ssim_tap(i), h[(k * kSsimIn + r + i) * kSsimTile + q], m[k]);
              tile += (double)ssim_window(m, shift_a, shift_b, R.c1, R.c2);
            }
          ssim_sum += tile;
        }
    double* o = out + (bi + 1) * kImOutPerImage;
    o[0] = se[bi] / n;
    o[1] = image_psnr(se[bi] / n);
    o[2] = ssim_sum / n_win;
    o[3] = (double)R.data_range;
    se_all += se[bi];
    ssim_all += o[2];
  }
  out[0] = se_all / (n * B);
  out[1] = image_psnr(se_all / (n * B));
  out[2] = ssim_all / B;
  out[3] = (double)R.data_range;
  return 0;
}

extern "C" void emul_ssim_taps(float* out) {
  for (int i = 0; i < kSsimWin; ++i) out[i] = ssim_tap(i);
}
