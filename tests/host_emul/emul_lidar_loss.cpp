// TEST SCAFFOLDING ONLY -- runs the device functions of neurad-studio_b200/csrc/lidar_loss.cuh on the host.
//
// The selection makes the kernels' three radix passes with the same keys, digits, prefix test, ranks, ceil-statistic
// rule and lerp (the histograms are counted serially instead of with atomics, which changes no count).  The losses and
// gradients use the kernels' per-ray functions; the sums are fp64 in index order (the device's fixed tree is another
// fp64 order).  Never linked into libb200nerf.so.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../neurad-studio_b200/csrc/lidar_loss.cuh"

using namespace nff;

static float select_host(const float* x, int64_t n, float q, int lower_median) {
  SelectState s{};
  for (int64_t i = 0; i < n; ++i) s.nan_count += x[i] != x[i];
  const SelectRank r = select_rank((unsigned)n, q, lower_median != 0, s.nan_count);
  s.k_lo = r.k_lo;
  s.k_hi = r.k_hi;
  s.weight = r.weight;
  s.k = r.k_lo;
  s.lower_median = lower_median != 0;
  std::vector<unsigned> hist(kSelectBins);
  for (int pass = 0; pass < kSelectPasses; ++pass) {
    std::fill(hist.begin(), hist.end(), 0u);
    for (int64_t i = 0; i < n; ++i) {
      const unsigned key = select_key(x[i]);
      if (select_in_prefix(key, s.prefix, pass)) ++hist[select_digit(key, pass)];
    }
    unsigned before = 0;
    int bin = 0;
    while (before + hist[bin] <= s.k) before += hist[bin++];
    s.prefix |= (unsigned)bin << select_shift(pass);
    s.k -= before;
    if (pass == kSelectPasses - 1) {
      s.key_lo = s.prefix;
      int next = -1;
      for (int b = bin + 1; b < kSelectBins; ++b)
        if (hist[b]) {
          next = b;
          break;
        }
      select_second(s, s.k, hist[bin], next);
      if (s.need_above) {
        unsigned m = 0xffffffffu;
        for (int64_t i = 0; i < n; ++i) {
          const unsigned key = select_key(x[i]);
          if (key > s.key_lo && key < m) m = key;
        }
        s.key_hi = m;
      }
    }
  }
  return select_value(s);
}

extern "C" float emul_quantile(const float* x, int64_t n, float q, int lower_median) { return select_host(x, n, q, lower_median); }

// out = [depth_loss, intensity_loss, ray_drop_loss, quantile, depth_loss_0 ..]; prop [n_prop][n]
extern "C" int emul_lidar_losses(int64_t n, int n_prop, const float* pred, const float* prop, const float* distance,
                                 const uint8_t* did_return, const float* intensity, const float* gt, int64_t gt_stride,
                                 const float* logits, float nrd, float nrm, float q, float* out, uint8_t* mask, int* counts) {
  if (n < 1 || n > kLossMaxN || n_prop > kLossMaxProp) return -1;
  std::vector<float> loss(n);
  double prop_sum[kLossMaxProp] = {0, 0, 0, 0}, bce = 0;
  for (int64_t i = 0; i < n; ++i) {
    const bool ret = did_return[i] != 0;
    loss[i] = lidar_depth_loss(pred[i], distance[i], ret, nrd, nrm);
    for (int r = 0; r < n_prop; ++r) prop_sum[r] += (double)lidar_depth_loss(prop[r * n + i], distance[i], ret, nrd, nrm);
    bce += (double)bce_with_logits(logits[i], ret ? 0.f : 1.f);
  }
  const float qv = select_host(loss.data(), n, q, 0);
  double s0 = 0, c0 = 0, s1 = 0, c1 = 0;
  for (int64_t i = 0; i < n; ++i) {
    mask[i] = loss[i] < qv;
    if (!mask[i]) continue;
    s0 += loss[i];
    c0 += 1;
    if (did_return[i]) {
      const float d = gt[i * gt_stride] - intensity[i];
      s1 += (double)(d * d);
      c1 += 1;
    }
  }
  out[0] = (float)(s0 / c0);
  out[1] = (float)(s1 / c1);
  out[2] = (float)(bce / (double)n);
  out[3] = qv;
  for (int r = 0; r < n_prop; ++r) out[4 + r] = (float)(prop_sum[r] / (double)n);
  counts[0] = (int)c0;
  counts[1] = (int)c1;
  return 0;
}

// the per-ray body of lidar_loss_bwd_kernel
extern "C" int emul_lidar_losses_bwd(int64_t n, int n_prop, const float* pred, const float* prop, const float* distance,
                                     const uint8_t* did_return, const float* intensity, const float* gt, int64_t gt_stride,
                                     const float* logits, float nrd, float nrm, const uint8_t* mask, const int* counts,
                                     const float* grads, float* d_pred, float* d_prop, float* d_intensity, float* d_logits) {
  const float g_depth = counts[0] ? grads[0] / (float)counts[0] : 0.f;
  const float g_int = counts[1] ? grads[1] / (float)counts[1] : 0.f;
  const float g_drop = grads[2] / (float)n;
  for (int64_t i = 0; i < n; ++i) {
    const bool ret = did_return[i] != 0, m = mask[i] != 0;
    d_pred[i] = m ? lidar_depth_grad(pred[i], distance[i], ret, nrd, nrm, g_depth) : 0.f;
    for (int r = 0; r < n_prop; ++r)
      d_prop[r * n + i] = lidar_depth_grad(prop[r * n + i], distance[i], ret, nrd, nrm, grads[4 + r] / (float)n);
    float di = 0.f;
    if (m && ret) di = -((2.f * (gt[i * gt_stride] - intensity[i])) * g_int);
    d_intensity[i] = di;
    d_logits[i] = bce_with_logits_grad(logits[i], ret ? 0.f : 1.f, g_drop);
  }
  return 0;
}
