// image_metrics.cuh -- PSNR and SSIM of the camera half of NeuRADModel.get_image_metrics_and_images (models/neurad.py:
// 265-266, 585-586) over two images a, b of B x H x W x C fp32 values, with no host synchronisation.
//
// Both images are addressed by explicit element strides (batch, row, column, channel), so channels-last [H, W, C]
// renders and the [1, C, H, W] moveaxis views the reference passes to its metrics are read in place.
//
// SSIM is torchmetrics' structural_similarity_index_measure(preds, target) with its defaults -- STATED FROM MEMORY,
// UNPINNED AGAINST TORCHMETRICS (the package is neither part of the reference tree nor a dependency of this library;
// tests/test_zz_image_metrics_gpu.py compares with it wherever it is installed):
//   window   g[i] = exp(-((i - 5) / 1.5)^2 / 2), i = 0..10, normalised to sum 1 in fp32; the 2-D window is g x g, applied
//            per channel to a, b, a a, b b and a b;
//   range    R = max(max a - min a, max b - min b) over the whole batch unless the caller gives one; c1 = (0.01 R)^2,
//            c2 = (0.03 R)^2;
//   value    var_a = max(E[a a] - mu_a^2, 0), var_b alike, cov = E[a b] - mu_a mu_b,
//            ssim = (2 mu_a mu_b + c1)(2 cov + c2) / ((mu_a^2 + mu_b^2 + c1)(var_a + var_b + c2));
//   mean     torchmetrics reflect-pads by 5, filters, and crops 5 pixels from every border before the mean: the outputs
//            that remain are exactly the (H - 10) x (W - 10) windows that lie inside the unpadded image, so no padding
//            is ever read here.  The value is the mean of those windows over all channels, then over the batch.
//
// Three launches:
//   image_stats_kernel             min / max of each image and the fp64 sum of (a - b)^2 per batch image, as block partials
//                                  on a grid of at most kImMaxBlocks CTAs that does not depend on the GPU;
//   ssim_tile_kernel               a CTA owns kSsimTile x kSsimTile windows of one channel: the kSsimIn x kSsimIn inputs of
//                                  both images go to shared memory, a horizontal pass leaves the five row-filtered moments
//                                  there, a vertical pass finishes them in registers, and a fixed tree leaves one fp64
//                                  partial per CTA.  The C channels of a tile are neighbouring CTAs, so the sectors of a
//                                  channels-last row that one of them fetches serve the others from L2.
//   image_metrics_finalize_kernel  one CTA: the partials in a fixed order -> mse, psnr, ssim, data_range per image and for
//                                  the batch.
// Every sum is taken in an order fixed by the shapes alone: two calls give the same bits.  A NaN anywhere gives NaN, as
// torch.max / torch.mean do.
//
// fp32 E[a a] - mu_a^2 cancels on flat regions (torchmetrics subtracts in fp32 as well, but the tests here compare with
// float64).  So each tile filters a - m_a and b - m_b, m the image's value at the tile's centre: variances and the
// covariance of a window whose weights sum to 1 do not change under a shift, and the shift goes back into the means.
// The fp32-normalised window sums to 1 - 1e-7, which against c2 = 9e-4 is not nothing: ssim_window adds that term back.
//
// The device functions above the kernels compile as plain C++ as well (tests/host_emul/emul_image_metrics.cpp).
#pragma once

#include "simt.h"

namespace nff {

constexpr int kImThreads = 256;
constexpr int kImMaxBlocks = 256;       // stats grid cap, and so the most images in one call
constexpr int kSsimWin = 11;            // window taps; sigma = 1.5
constexpr int kSsimTile = 32;           // windows per tile side
constexpr int kSsimIn = kSsimTile + kSsimWin - 1;  // 42 input pixels per tile side
constexpr int kSsimPitch = kSsimIn + 1;
constexpr int kSsimStrip = kSsimTile * kSsimTile / kImThreads;  // 4 windows of one column per thread
constexpr int kSsimMaxTiles = 1 << 18;  // tile partials the context holds: 2^28 windows x channels in one call
constexpr int kImOutPerImage = 4;       // mse, psnr, ssim, data_range

// torch.exp(-(arange(-5, 6) / 1.5) ** 2 / 2) / sum, in fp32 (tests/test_image_metrics_cpu.py recomputes them)
NFF_HD float ssim_tap(int i) {
  constexpr float g[kSsimWin] = {0x1.0d957p-10f, 0x1.f1fdf8p-8f, 0x1.26eb18p-5f, 0x1.bff0fcp-4f, 0x1.b43c3ep-3f, 0x1.10656p-2f,
                                 0x1.b43c3ep-3f, 0x1.bff0fcp-4f, 0x1.26eb18p-5f, 0x1.f1fdf8p-8f, 0x1.0d957p-10f};
  return g[i];
}

// single IEEE roundings the compiler may not contract, on the device and in the host emulation alike
NFF_HD float im_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
NFF_HD float im_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
NFF_HD float im_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
NFF_HD float im_div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// min / max that keep a NaN, as torch.min / torch.max do
NFF_HD float nan_min(float a, float b) { return (a != a || b != b) ? NAN : (b < a ? b : a); }
NFF_HD float nan_max(float a, float b) { return (a != a || b != b) ? NAN : (b > a ? b : a); }

struct ImageView {
  const float* p;
  int64_t sb, sy, sx, sc;  // element strides of batch, row, column, channel
};

// The walk of image_stats_kernel: n_r1 x n_r2 rows of n_in elements.  Pixels whose channels are evenly spaced in both
// images (sx == C sc: channels-last tensors and their moveaxis views) are walked as rows of W C elements, anything
// else as C x H rows of W elements.
struct StatsWalk {
  int n_in, n_r1, n_r2;
  int64_t a_in, a_r1, a_r2, b_in, b_r1, b_r2;
};
NFF_HD StatsWalk stats_walk(const ImageView& a, const ImageView& b, int H, int W, int C) {
  StatsWalk w;
  if (C == 1 || (a.sx == C * a.sc && b.sx == C * b.sc)) {
    w.n_in = W * C;
    w.n_r1 = 1;
    w.n_r2 = H;
    w.a_in = C == 1 ? a.sx : a.sc;
    w.b_in = C == 1 ? b.sx : b.sc;
    w.a_r1 = w.b_r1 = 0;
  } else {
    w.n_in = W;
    w.n_r1 = C;
    w.n_r2 = H;
    w.a_in = a.sx;
    w.b_in = b.sx;
    w.a_r1 = a.sc;
    w.b_r1 = b.sc;
  }
  w.a_r2 = a.sy;
  w.b_r2 = b.sy;
  return w;
}

struct ImageRange {
  float data_range, c1, c2;
};
// data_range <= 0: derive it from the extrema of the two images
NFF_HD ImageRange image_range(float a_min, float a_max, float b_min, float b_max, float data_range) {
  ImageRange r;
  r.data_range = data_range > 0.f ? data_range : nan_max(im_sub(a_max, a_min), im_sub(b_max, b_min));
  const float k1 = im_mul(0.01f, r.data_range), k2 = im_mul(0.03f, r.data_range);
  r.c1 = im_mul(k1, k1);
  r.c2 = im_mul(k2, k2);
  return r;
}

// The five moments a, b, a a, b b, a b of 11 neighbouring pixels of one row, filtered tap by tap in ascending order.
NFF_HD void ssim_row_moments(const float* a, const float* b, float m[5]) {
  m[0] = m[1] = m[2] = m[3] = m[4] = 0.f;
  for (int i = 0; i < kSsimWin; ++i) {
    const float g = ssim_tap(i), x = a[i], y = b[i];
    m[0] = fmaf(g, x, m[0]);
    m[1] = fmaf(g, y, m[1]);
    m[2] = fmaf(g, im_mul(x, x), m[2]);
    m[3] = fmaf(g, im_mul(y, y), m[3]);
    m[4] = fmaf(g, im_mul(x, y), m[4]);
  }
}

// 1 - (sum of the taps)^2: the fp32-normalised taps sum to 1 - 5.03e-8, so the 2-D window's weight is S = 1 - kSsimDefect
// and E[x x] - mu^2 is not quite invariant under a shift of x.
constexpr float kSsimDefect = 0x1.bp-24f;  // 1.00582836e-7 in fp32

// E[(x + m_x)(y + m_y)] - E[x + m_x] E[y + m_y] = (E[x y] - E[x] E[y]) + (1 - S)(m_x E[y] + m_y E[x] + S m_x m_y) for a
// window of weight S; this is the bracket (with S = 1 inside it: an error of kSsimDefect^2).
NFF_HD float ssim_shift_term(float m_x, float e_x, float m_y, float e_y) { return fmaf(m_x, e_y, fmaf(m_y, e_x, im_mul(m_x, m_y))); }

// SSIM of one window of a, b from the filtered moments m of the shifted images a - shift_a, b - shift_b.  The three
// second moments take one expression, so identical images give var_a = var_b = cov bit for bit and exactly 1.
NFF_HD float ssim_window(const float m[5], float shift_a, float shift_b, float c1, float c2) {
  const float var_a = fmaxf(fmaf(kSsimDefect, ssim_shift_term(shift_a, m[0], shift_a, m[0]), im_sub(m[2], im_mul(m[0], m[0]))), 0.f);
  const float var_b = fmaxf(fmaf(kSsimDefect, ssim_shift_term(shift_b, m[1], shift_b, m[1]), im_sub(m[3], im_mul(m[1], m[1]))), 0.f);
  const float cov = fmaf(kSsimDefect, ssim_shift_term(shift_a, m[0], shift_b, m[1]), im_sub(m[4], im_mul(m[0], m[1])));
  const float mu_a = fmaf(-kSsimDefect, shift_a, im_add(m[0], shift_a)), mu_b = fmaf(-kSsimDefect, shift_b, im_add(m[1], shift_b));
  const float num = im_mul(im_add(im_mul(2.f, im_mul(mu_a, mu_b)), c1), im_add(im_mul(2.f, cov), c2));
  const float den = im_mul(im_add(im_add(im_mul(mu_a, mu_a), im_mul(mu_b, mu_b)), c1), im_add(im_add(var_a, var_b), c2));
  // a NaN moment must reach the mean: fmaxf alone would turn a NaN variance into 0
  return (m[2] != m[2] || m[3] != m[3]) ? NAN : im_div(num, den);
}

// Pixel of the tile whose value is the tile's shift: the centre of its input window, clamped into the image.
NFF_HD int ssim_shift_coord(int origin, int size) {
  const int c = origin + kSsimIn / 2;
  return c < size ? c : size - 1;
}

NFF_HD double image_psnr(double mse) { return 10.0 * log10(1.0 / mse); }

#if defined(__CUDACC__)
// ---- block helpers (kImThreads threads)
__device__ __forceinline__ double im_block_sum(double v, double* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();  // s_warp may still be read from an earlier call
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_warp[w];
  return t;  // valid on thread 0
}

// mm = [a_min, a_max, b_min, b_max]; the result is valid on every thread
__device__ __forceinline__ void im_block_minmax(float (&mm)[4], float (*s_mm)[4]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mm[0] = nan_min(mm[0], __shfl_xor_sync(0xffffffffu, mm[0], o));
    mm[1] = nan_max(mm[1], __shfl_xor_sync(0xffffffffu, mm[1], o));
    mm[2] = nan_min(mm[2], __shfl_xor_sync(0xffffffffu, mm[2], o));
    mm[3] = nan_max(mm[3], __shfl_xor_sync(0xffffffffu, mm[3], o));
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 4; ++k) s_mm[threadIdx.x >> 5][k] = mm[k];
  __syncthreads();
  for (int k = 0; k < 4; ++k) mm[k] = s_mm[0][k];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
    mm[0] = nan_min(mm[0], s_mm[w][0]);
    mm[1] = nan_max(mm[1], s_mm[w][1]);
    mm[2] = nan_min(mm[2], s_mm[w][2]);
    mm[3] = nan_max(mm[3], s_mm[w][3]);
  }
}

// The extrema of the whole batch from launch 1's block partials, on every thread.
__device__ __forceinline__ ImageRange im_range_from_partials(const float* __restrict__ mm_part, int n_part, float data_range,
                                                             float (*s_mm)[4]) {
  float mm[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < n_part; i += blockDim.x) {
    mm[0] = nan_min(mm[0], mm_part[4 * i + 0]);
    mm[1] = nan_max(mm[1], mm_part[4 * i + 1]);
    mm[2] = nan_min(mm[2], mm_part[4 * i + 2]);
    mm[3] = nan_max(mm[3], mm_part[4 * i + 3]);
  }
  im_block_minmax(mm, s_mm);
  return image_range(mm[0], mm[1], mm[2], mm[3], data_range);
}

// ---- launch 1: grid (blocks per image, B).  Block (k, bi) walks rows k, k + gridDim.x, .. of image bi and leaves
// mm_part[bi gridDim.x + k] = its extrema and se_part[..] = its fp64 sum of (a - b)^2.
__global__ void __launch_bounds__(kImThreads) image_stats_kernel(ImageView a, ImageView b, StatsWalk w,
                                                                float* __restrict__ mm_part, double* __restrict__ se_part) {
  __shared__ double s_warp[kImThreads / 32];
  __shared__ float s_mm[kImThreads / 32][4];
  const float* pa = a.p + (int64_t)blockIdx.y * a.sb;
  const float* pb = b.p + (int64_t)blockIdx.y * b.sb;
  float mm[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  double se = 0.0;
  const int n_rows = w.n_r1 * w.n_r2;
  for (int r = blockIdx.x; r < n_rows; r += gridDim.x) {
    const int r1 = r / w.n_r2, r2 = r - r1 * w.n_r2;
    const float* ra = pa + r1 * w.a_r1 + r2 * w.a_r2;
    const float* rb = pb + r1 * w.b_r1 + r2 * w.b_r2;
#pragma unroll 4
    for (int i = threadIdx.x; i < w.n_in; i += kImThreads) {
      const float x = ra[i * w.a_in], y = rb[i * w.b_in];
      mm[0] = nan_min(mm[0], x);
      mm[1] = nan_max(mm[1], x);
      mm[2] = nan_min(mm[2], y);
      mm[3] = nan_max(mm[3], y);
      const double d = (double)x - (double)y;
      se = fma(d, d, se);
    }
  }
  const int slot = blockIdx.y * gridDim.x + blockIdx.x;
  const double t = im_block_sum(se, s_warp);
  im_block_minmax(mm, s_mm);
  if (threadIdx.x == 0) {
    se_part[slot] = t;
    for (int k = 0; k < 4; ++k) mm_part[4 * slot + k] = mm[k];
  }
}

// ---- launch 2: block = ((bi tiles_y + ty) tiles_x + tx) C + c
struct SsimArgs {
  ImageView a, b;
  int H, W, C, tiles_x, tiles_y;
  int n_stats;       // block partials of launch 1
  float data_range;  // <= 0: derive
};

__global__ void __launch_bounds__(kImThreads) ssim_tile_kernel(SsimArgs g, const float* __restrict__ mm_part,
                                                              double* __restrict__ ssim_part) {
  __shared__ float s_a[kSsimIn][kSsimPitch], s_b[kSsimIn][kSsimPitch];
  __shared__ float s_h[5][kSsimIn][kSsimTile];
  __shared__ double s_warp[kImThreads / 32];
  __shared__ float s_mm[kImThreads / 32][4];
  const int t = threadIdx.x;
  int id = blockIdx.x;
  const int c = id % g.C;
  id /= g.C;
  const int x0 = (id % g.tiles_x) * kSsimTile;
  id /= g.tiles_x;
  const int y0 = (id % g.tiles_y) * kSsimTile;
  const int bi = id / g.tiles_y;
  const float* pa = g.a.p + bi * g.a.sb + c * g.a.sc;
  const float* pb = g.b.p + bi * g.b.sb + c * g.b.sc;

  const ImageRange R = im_range_from_partials(mm_part, g.n_stats, g.data_range, s_mm);
  const int cy = ssim_shift_coord(y0, g.H), cx = ssim_shift_coord(x0, g.W);
  const float shift_a = pa[cy * g.a.sy + cx * g.a.sx], shift_b = pb[cy * g.b.sy + cx * g.b.sx];

  // pixels past the image belong to no window of the image: zero
  for (int i = t; i < kSsimIn * kSsimIn; i += kImThreads) {
    const int r = i / kSsimIn, q = i - r * kSsimIn;
    const int y = y0 + r, x = x0 + q;
    const bool in = y < g.H && x < g.W;
    s_a[r][q] = in ? im_sub(pa[y * g.a.sy + x * g.a.sx], shift_a) : 0.f;
    s_b[r][q] = in ? im_sub(pb[y * g.b.sy + x * g.b.sx], shift_b) : 0.f;
  }
  __syncthreads();
  for (int i = t; i < kSsimIn * kSsimTile; i += kImThreads) {
    const int r = i / kSsimTile, q = i % kSsimTile;
    float m[5];
    ssim_row_moments(&s_a[r][q], &s_b[r][q], m);
#pragma unroll
    for (int k = 0; k < 5; ++k) s_h[k][r][q] = m[k];
  }
  __syncthreads();
  // thread (q, strip): windows (strip kSsimStrip + k, q), each the taps in ascending order over its 11 rows
  const int q = t % kSsimTile, r0 = (t / kSsimTile) * kSsimStrip;
  float acc[kSsimStrip][5];
#pragma unroll
  for (int k = 0; k < kSsimStrip; ++k)
#pragma unroll
    for (int m = 0; m < 5; ++m) acc[k][m] = 0.f;
#pragma unroll
  for (int j = 0; j < kSsimStrip + kSsimWin - 1; ++j) {
    float h[5];
#pragma unroll
    for (int m = 0; m < 5; ++m) h[m] = s_h[m][r0 + j][q];
#pragma unroll
    for (int k = 0; k < kSsimStrip; ++k) {
      if (j - k >= 0 && j - k < kSsimWin) {
#pragma unroll
        for (int m = 0; m < 5; ++m) acc[k][m] = fmaf(ssim_tap(j - k), h[m], acc[k][m]);
      }
    }
  }
  double sum = 0.0;
#pragma unroll
  for (int k = 0; k < kSsimStrip; ++k)
    if (y0 + r0 + k < g.H - (kSsimWin - 1) && x0 + q < g.W - (kSsimWin - 1))
      sum += (double)ssim_window(acc[k], shift_a, shift_b, R.c1, R.c2);
  const double total = im_block_sum(sum, s_warp);
  if (t == 0) ssim_part[blockIdx.x] = total;
}

// ---- launch 3: one CTA of kImThreads threads.  out = [batch | image 0 | image 1 ..] x [mse, psnr, ssim, data_range].
__global__ void __launch_bounds__(kImThreads) image_metrics_finalize_kernel(int B, int H, int W, int C, int stats_per_image,
                                                                           int tiles_per_image, float data_range,
                                                                           const float* __restrict__ mm_part,
                                                                           const double* __restrict__ se_part,
                                                                           const double* __restrict__ ssim_part,
                                                                           double* __restrict__ out) {
  __shared__ double s_warp[kImThreads / 32];
  __shared__ float s_mm[kImThreads / 32][4];
  const ImageRange R = im_range_from_partials(mm_part, B * stats_per_image, data_range, s_mm);
  const double n = (double)H * W * C, n_win = (double)(H - (kSsimWin - 1)) * (W - (kSsimWin - 1)) * C;
  double se_all = 0.0, ssim_all = 0.0;  // thread 0
  for (int bi = 0; bi < B; ++bi) {
    double v = 0.0;
    for (int i = threadIdx.x; i < tiles_per_image; i += kImThreads) v += ssim_part[(int64_t)bi * tiles_per_image + i];
    const double ssim = im_block_sum(v, s_warp) / n_win;
    if (threadIdx.x == 0) {
      double se = 0.0;
      for (int k = 0; k < stats_per_image; ++k) se += se_part[bi * stats_per_image + k];
      double* o = out + (bi + 1) * kImOutPerImage;
      o[0] = se / n;
      o[1] = image_psnr(se / n);
      o[2] = ssim;
      o[3] = (double)R.data_range;
      se_all += se;
      ssim_all += ssim;
    }
  }
  if (threadIdx.x == 0) {
    out[0] = se_all / (n * B);
    out[1] = image_psnr(se_all / (n * B));
    out[2] = ssim_all / B;
    out[3] = (double)R.data_range;
  }
}
#endif

}  // namespace nff
