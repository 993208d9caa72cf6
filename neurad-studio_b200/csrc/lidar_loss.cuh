// lidar_loss.cuh -- the lidar terms of NeuRADModel.get_metrics_dict in training mode (models/neurad.py:486-520) as one
// forward and one backward operator over the n lidar rays of a batch, with no host synchronisation.
//
// Per ray (lidar_depth_loss): target = distance for returns, max(pred, non_return_lidar_distance) for non-returns, and
// the loss |target - pred|, times non_return_loss_mult for non-returns -- for the main depth and for every proposal
// depth.  The reference then takes torch.quantile(loss, q) and keeps the rays strictly below it.  Here that quantile is
// an exact radix select on order-preserving 32-bit keys (select_key): three histogram passes over 11 + 11 + 10 key bits
// find the floor order statistic v_k; the ceil one is v_k again when more than k + 1 keys are <= v_k, else the smallest
// key above it (the next non-empty bin of the last pass, or one atomicMin pass when that bin is the prefix's last).
// The rank and the interpolation are ATen's quantile_impl bit for bit: fp32 rank q * (n - 1), floor / ceil, and
// torch.lerp's two-branch formula with the FMAs the compiled torch kernels use; a NaN anywhere gives NaN.
//
// Reductions (depth_loss over the mask, intensity MSE over mask & did_return, BCE-with-logits over all rays, the plain
// per-round proposal means) are fp64 sums in a fixed order: a fixed grid, a fixed per-thread stride, a fixed tree per
// block and one CTA that adds the block partials in block order.  Two calls give the same bits.  An empty mask gives
// 0 / 0 = NaN, as torch.mean of an empty tensor does.
//
// The device functions above the kernels compile as plain C++ as well (tests/host_emul/emul_lidar_loss.cpp).
#pragma once

#include "simt.h"

namespace nff {

constexpr int kLossThreads = 256;
constexpr int kLossMaxBlocks = 256;  // fixed cap: the block partials, and so the sums' bits, do not depend on the GPU
constexpr int kLossMaxProp = 4;      // proposal rounds
constexpr int kSelectBins = 2048;    // 11-bit digits
constexpr int kSelectPasses = 3;     // key bits 31..21, 20..10, 9..0
constexpr int kRowSlots = kLossMaxProp + 1;  // per-round depth sums, BCE sum
constexpr int kMaskSlots = 4;                // masked depth sum and count, masked & returned intensity SE sum and count
constexpr int kLossMaxN = 1 << 24;           // torch.quantile's own limit

NFF_HD int select_shift(int pass) { return pass == 0 ? 21 : pass == 1 ? 10 : 0; }
NFF_HD int select_bins(int pass) { return pass == 2 ? 1024 : kSelectBins; }

// Order-preserving key: a < b as floats <=> key(a) < key(b).  -0 takes +0's key (torch's sort compares them equal), so a
// zero at the rank decodes as +0 where torch may return the -0 its sort left there; the depth losses are never -0.
// Every NaN takes the largest key, so NaNs sort last as in torch.sort.
NFF_HD unsigned select_key(float v) {
  if (v != v) return 0xffffffffu;
  unsigned u;
  memcpy(&u, &v, 4);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
NFF_HD float select_unkey(unsigned k) {
  if (k == 0xffffffffu) return NAN;
  const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  memcpy(&v, &u, 4);
  return v;
}
NFF_HD unsigned select_digit(unsigned key, int pass) { return (key >> select_shift(pass)) & (unsigned)(select_bins(pass) - 1); }
// key agrees with `prefix` on every bit above this pass's digit (the bits the earlier passes fixed)
NFF_HD bool select_in_prefix(unsigned key, unsigned prefix, int pass) {
  return pass == 0 || (key >> select_shift(pass - 1)) == (prefix >> select_shift(pass - 1));
}

// Ranks of ATen's quantile_impl (linear): rank = q * (n - 1) in fp32 (n - 1 when there is a NaN), k_lo = trunc(rank),
// k_hi = ceil(rank), weight = rank - k_lo.  lower_median: torch.median's (n - 1) / 2 (n - 1 with a NaN), no interpolation.
struct SelectRank {
  unsigned k_lo, k_hi;
  float weight;
};
NFF_HD SelectRank select_rank(unsigned n, float q, bool lower_median, unsigned nan_count) {
  SelectRank r;
  if (nan_count > 0) {
    r.k_lo = r.k_hi = n - 1;
    r.weight = 0.f;
  } else if (lower_median) {
    r.k_lo = r.k_hi = (n - 1) / 2;
    r.weight = 0.f;
  } else {
    const float rank = q * (float)(n - 1);
    r.k_lo = (unsigned)rank;
    r.k_hi = (unsigned)ceilf(rank);
    r.weight = rank - (float)r.k_lo;
  }
  return r;
}

// torch.lerp(lo, hi, w) (ATen's lerp: weight < 0.5 ? lo + w (hi - lo) : hi - (hi - lo)(1 - w)), with the single
// rounding of the FMA that the compiled CUDA and vectorised CPU kernels both use
NFF_HD float quantile_lerp(float lo, float hi, float w) {
  const float d = hi - lo;
  return fabsf(w) < 0.5f ? fmaf(w, d, lo) : fmaf(-d, 1.f - w, hi);
}

// State of one selection in device memory.  The host zeroes it (and the histogram) before the first pass.
struct SelectState {
  unsigned nan_count;  // pass 0 histogram kernel
  unsigned k;          // rank still to find inside the current prefix
  unsigned prefix;     // key bits fixed so far
  unsigned k_lo, k_hi;
  float weight;
  unsigned key_lo, key_hi;  // the two order statistics (key_hi valid once need_above == 0 or above_min is known)
  unsigned need_above;      // 1: key_hi = min key > key_lo, found by select_above_kernel
  unsigned above_min;       // atomicMin target, starts at 0xffffffff
  float value;              // the quantile
  unsigned lower_median;    // torch.median: v_k itself, no interpolation
  unsigned pad[4];
};

// After the last pass: the run of keys equal to key_lo holds `count` keys, and k_lo is the (k_in_run)-th of them.  The
// ceil statistic is key_lo when k_hi == k_lo or the run continues past k_lo; else the next non-empty bin above
// (`next_bin`, -1 if none in this prefix: then a pass over all keys finds the smallest key above key_lo).
NFF_HD void select_second(SelectState& s, unsigned k_in_run, unsigned count, int next_bin) {
  if (s.k_hi == s.k_lo || k_in_run + 1 < count) {
    s.key_hi = s.key_lo;
    s.need_above = 0;
  } else if (next_bin >= 0) {
    s.key_hi = (s.key_lo & ~1023u) | (unsigned)next_bin;
    s.need_above = 0;
  } else {
    s.need_above = 1;
  }
}
// torch.quantile interpolates even between equal ranks (lerp(-inf, -inf, 0) is NaN there too); torch.median does not
NFF_HD float select_value(const SelectState& s) {
  const float lo = select_unkey(s.key_lo), hi = select_unkey(s.key_hi);
  return s.lower_median ? lo : quantile_lerp(lo, hi, s.weight);
}

// ---- per ray
// a product the compiler may not fuse with the following subtraction (torch evaluates them as separate kernels)
NFF_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
// unreduced_depth_loss of one ray (neurad.py:491-494 / 516-519): torch.maximum propagates a NaN prediction
NFF_HD float lidar_target(float pred, float distance, bool did_return, float non_return_distance) {
  if (did_return) return distance;
  return (pred != pred || pred > non_return_distance) ? pred : non_return_distance;
}
NFF_HD float lidar_depth_loss(float pred, float distance, bool did_return, float non_return_distance, float non_return_mult) {
  const float l = fabsf(lidar_target(pred, distance, did_return, non_return_distance) - pred);
  return did_return ? l : l * non_return_mult;
}
// d loss / d pred for an upstream gradient g already divided by the mean's count: L1Loss's abs backward is g * sgn(x)
// with sgn(0) = sgn(NaN) = 0 (a non-return predicted at or beyond the non-return distance gets exactly 0); the target
// is detached
NFF_HD float lidar_depth_grad(float pred, float distance, bool did_return, float non_return_distance, float non_return_mult,
                              float g) {
  const float x = lidar_target(pred, distance, did_return, non_return_distance) - pred;
  const float a = did_return ? g : g * non_return_mult;
  const float sg = x > 0.f ? 1.f : x < 0.f ? -1.f : 0.f;
  return -(a * sg);
}
// BCEWithLogitsLoss (no weights) in ATen's stable form: (1 - y) x - log_sigmoid(x), log_sigmoid(x) = min(x, 0) -
// log1p(exp(-|x|))
NFF_HD float bce_with_logits(float x, float y) {
  const float log_sig = fminf(x, 0.f) - log1pf(expf(-fabsf(x)));
  return mul_rn(1.f - y, x) - log_sig;
}
NFF_HD float bce_with_logits_grad(float x, float y, float g) {
  return (1.f / (1.f + expf(-x)) - y) * g;
}

#if defined(__CUDACC__)
// ---- block helpers
template <int SLOTS>
__device__ __forceinline__ void block_sum_f64(double (&v)[SLOTS], double* out) {
  __shared__ double warp_sums[kLossThreads / 32][SLOTS];
#pragma unroll
  for (int s = 0; s < SLOTS; ++s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[s] += __shfl_down_sync(0xffffffffu, v[s], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) warp_sums[threadIdx.x >> 5][s] = v[s];
  }
  __syncthreads();
  if (threadIdx.x < SLOTS) {
    double t = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) t += warp_sums[w][threadIdx.x];
    out[threadIdx.x] = t;
  }
}

__device__ __forceinline__ void flush_hist(unsigned* s_hist, unsigned* hist) {
  __syncthreads();
  for (int b = threadIdx.x; b < kSelectBins; b += kLossThreads)
    if (s_hist[b]) atomicAdd(&hist[b], s_hist[b]);
}

// ---- selection kernels
// Histogram of pass `pass` over the keys that match the prefix; pass 0 also counts NaNs.
__global__ void __launch_bounds__(kLossThreads) select_hist_kernel(const float* __restrict__ vals, int n, int pass,
                                                                  SelectState* __restrict__ st, unsigned* __restrict__ hist) {
  __shared__ unsigned s_hist[kSelectBins];
  for (int b = threadIdx.x; b < kSelectBins; b += kLossThreads) s_hist[b] = 0u;
  __syncthreads();
  const unsigned prefix = pass == 0 ? 0u : st->prefix;
  unsigned nans = 0;
  for (int i = blockIdx.x * kLossThreads + threadIdx.x; i < n; i += gridDim.x * kLossThreads) {
    const float v = vals[i];
    const unsigned key = select_key(v);
    nans += v != v;
    if (select_in_prefix(key, prefix, pass)) atomicAdd(&s_hist[select_digit(key, pass)], 1u);
  }
  if (pass == 0 && nans) atomicAdd(&st->nan_count, nans);
  flush_hist(s_hist, hist);
}

// One CTA of 1024 threads, two bins each: find the bin that holds rank st->k, fix its digit, clear the histogram.
__global__ void __launch_bounds__(1024) select_scan_kernel(int n, float q, int lower_median, int pass, SelectState* __restrict__ st,
                                                           unsigned* __restrict__ hist) {
  __shared__ unsigned warp_tot[32];
  __shared__ int s_bin, s_next;
  __shared__ unsigned s_before, s_count;
  const int t = threadIdx.x;
  if (pass == 0 && t == 0) {
    const SelectRank r = select_rank((unsigned)n, q, lower_median != 0, st->nan_count);
    st->k_lo = r.k_lo;
    st->k_hi = r.k_hi;
    st->weight = r.weight;
    st->k = r.k_lo;
    st->prefix = 0u;
    st->lower_median = lower_median != 0;
  }
  if (t == 0) s_next = 0x7fffffff;
  __syncthreads();
  const unsigned k = st->k;
  const unsigned c0 = hist[2 * t], c1 = hist[2 * t + 1];
  unsigned incl = c0 + c1;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += y;
  }
  if ((t & 31) == 31) warp_tot[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    unsigned w = warp_tot[t];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, w, o);
      if (t >= o) w += y;
    }
    warp_tot[t] = w;  // inclusive over warps
  }
  __syncthreads();
  const unsigned excl = incl - (c0 + c1) + ((t >> 5) ? warp_tot[(t >> 5) - 1] : 0u);
  if (k >= excl && k < excl + c0) {
    s_bin = 2 * t;
    s_before = excl;
    s_count = c0;
  } else if (k >= excl + c0 && k < excl + c0 + c1) {
    s_bin = 2 * t + 1;
    s_before = excl + c0;
    s_count = c1;
  }
  __syncthreads();
  const int bin = s_bin;
  if (pass == kSelectPasses - 1) {
    if (2 * t > bin && c0) atomicMin(&s_next, 2 * t);
    if (2 * t + 1 > bin && c1) atomicMin(&s_next, 2 * t + 1);
  }
  hist[2 * t] = 0u;
  hist[2 * t + 1] = 0u;
  __syncthreads();
  if (t == 0) {
    st->prefix |= (unsigned)bin << select_shift(pass);
    st->k = k - s_before;
    if (pass == kSelectPasses - 1) {
      st->key_lo = st->prefix;
      st->above_min = 0xffffffffu;
      SelectState s = *st;
      select_second(s, k - s_before, s_count, s_next == 0x7fffffff ? -1 : s_next);
      st->key_hi = s.key_hi;
      st->need_above = s.need_above;
    }
  }
}

// The smallest key above key_lo, over all keys; a no-op unless the last scan asked for it.
__global__ void __launch_bounds__(kLossThreads) select_above_kernel(const float* __restrict__ vals, int n, SelectState* __restrict__ st) {
  if (!st->need_above) return;
  const unsigned lo = st->key_lo;
  unsigned m = 0xffffffffu;
  for (int i = blockIdx.x * kLossThreads + threadIdx.x; i < n; i += gridDim.x * kLossThreads) {
    const unsigned key = select_key(vals[i]);
    if (key > lo && key < m) m = key;
  }
  m = __reduce_min_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m != 0xffffffffu) atomicMin(&st->above_min, m);
}

__global__ void select_finish_kernel(SelectState* __restrict__ st, float* __restrict__ out) {
  SelectState s = *st;
  if (s.need_above) s.key_hi = s.above_min;
  const float v = select_value(s);
  st->key_hi = s.key_hi;
  st->value = v;
  if (out) *out = v;
}

// ---- loss kernels
struct LidarLossArgs {
  int n, n_prop, prop_stride, gt_intensity_stride;
  const float* pred;           // [n] main depth
  const float* prop;           // [n_prop][prop_stride] proposal depths
  const float* distance;       // [n]
  const uint8_t* did_return;   // [n]
  const float* intensity;      // [n] predicted
  const float* gt_intensity;   // [n] with stride gt_intensity_stride (column 3 of the lidar points)
  const float* logits;         // [n] ray-drop logits
  float non_return_distance, non_return_mult;
};

// Pass 0 of the selection fused with the per-ray losses: loss[i] (the main depth's unreduced loss), its key histogram,
// and the block partials of the proposal-depth and BCE sums.
__global__ void __launch_bounds__(kLossThreads) lidar_loss_rows_kernel(LidarLossArgs a, float* __restrict__ loss,
                                                                      SelectState* __restrict__ st, unsigned* __restrict__ hist,
                                                                      double* __restrict__ part) {
  __shared__ unsigned s_hist[kSelectBins];
  for (int b = threadIdx.x; b < kSelectBins; b += kLossThreads) s_hist[b] = 0u;
  __syncthreads();
  double acc[kRowSlots];
#pragma unroll
  for (int s = 0; s < kRowSlots; ++s) acc[s] = 0.0;
  unsigned nans = 0;
  for (int i = blockIdx.x * kLossThreads + threadIdx.x; i < a.n; i += gridDim.x * kLossThreads) {
    const bool ret = a.did_return[i] != 0;
    const float dist = a.distance[i];
    const float l = lidar_depth_loss(a.pred[i], dist, ret, a.non_return_distance, a.non_return_mult);
    loss[i] = l;
    nans += l != l;
    atomicAdd(&s_hist[select_digit(select_key(l), 0)], 1u);
#pragma unroll
    for (int r = 0; r < kLossMaxProp; ++r)
      if (r < a.n_prop)
        acc[r] += (double)lidar_depth_loss(a.prop[(int64_t)r * a.prop_stride + i], dist, ret, a.non_return_distance, a.non_return_mult);
    acc[kLossMaxProp] += (double)bce_with_logits(a.logits[i], ret ? 0.f : 1.f);
  }
  if (nans) atomicAdd(&st->nan_count, nans);
  flush_hist(s_hist, hist);
  block_sum_f64<kRowSlots>(acc, part + (int64_t)blockIdx.x * kRowSlots);
}

// mask = loss < quantile; block partials of the masked depth sum / count and the masked-and-returned intensity SE.
__global__ void __launch_bounds__(kLossThreads) lidar_loss_mask_kernel(LidarLossArgs a, const float* __restrict__ loss,
                                                                      const SelectState* __restrict__ st, uint8_t* __restrict__ mask,
                                                                      double* __restrict__ part) {
  const float qv = st->value;
  double acc[kMaskSlots] = {0.0, 0.0, 0.0, 0.0};
  for (int i = blockIdx.x * kLossThreads + threadIdx.x; i < a.n; i += gridDim.x * kLossThreads) {
    const float l = loss[i];
    const bool m = l < qv;
    mask[i] = m;
    if (m) {
      acc[0] += (double)l;
      acc[1] += 1.0;
      if (a.did_return[i]) {
        const float d = simt::fsub(a.gt_intensity[(int64_t)i * a.gt_intensity_stride], a.intensity[i]);
        acc[2] += (double)simt::fmul(d, d);
        acc[3] += 1.0;
      }
    }
  }
  block_sum_f64<kMaskSlots>(acc, part + (int64_t)blockIdx.x * kMaskSlots);
}

// One CTA: the block partials in block order.  out = [depth_loss, intensity_loss, ray_drop_loss, quantile,
// depth_loss_0 .. depth_loss_{n_prop-1}]; counts = [|mask|, |mask & did_return|].
__global__ void lidar_loss_final_kernel(int n, int n_prop, int blocks, const double* __restrict__ row_part,
                                        const double* __restrict__ mask_part, const SelectState* __restrict__ st,
                                        float* __restrict__ out, int* __restrict__ counts) {
  const int s = threadIdx.x;
  if (s < kRowSlots) {
    double t = 0.0;
    for (int b = 0; b < blocks; ++b) t += row_part[b * kRowSlots + s];
    if (s < n_prop) out[4 + s] = (float)(t / (double)n);
    if (s == kLossMaxProp) out[2] = (float)(t / (double)n);
  } else if (s < kRowSlots + 2) {
    const int j = (s - kRowSlots) * 2;  // 0: depth, 2: intensity
    double sum = 0.0, cnt = 0.0;
    for (int b = 0; b < blocks; ++b) {
      sum += mask_part[b * kMaskSlots + j];
      cnt += mask_part[b * kMaskSlots + j + 1];
    }
    out[j / 2] = (float)(sum / cnt);  // an empty mask: 0 / 0 = NaN, as torch.mean of an empty tensor
    counts[j / 2] = (int)cnt;
  } else if (s == kRowSlots + 2) {
    out[3] = st->value;
  }
}

// grads: the upstream gradients in the forward's `out` layout (the quantile's entry is not read); counts from the forward.
__global__ void __launch_bounds__(kLossThreads) lidar_loss_bwd_kernel(LidarLossArgs a, const uint8_t* __restrict__ mask,
                                                                     const int* __restrict__ counts, const float* __restrict__ grads,
                                                                     float* __restrict__ d_pred, float* __restrict__ d_prop,
                                                                     float* __restrict__ d_intensity, float* __restrict__ d_logits) {
  const int c_depth = counts[0], c_int = counts[1];
  // torch's mean backward: g / count in fp32 (only read when the count is > 0)
  const float g_depth = c_depth ? simt::fdiv(grads[0], (float)c_depth) : 0.f;
  const float g_int = c_int ? simt::fdiv(grads[1], (float)c_int) : 0.f;
  const float g_drop = simt::fdiv(grads[2], (float)a.n);
  float g_prop[kLossMaxProp];
#pragma unroll
  for (int r = 0; r < kLossMaxProp; ++r) g_prop[r] = r < a.n_prop ? simt::fdiv(grads[4 + r], (float)a.n) : 0.f;
  for (int i = blockIdx.x * kLossThreads + threadIdx.x; i < a.n; i += gridDim.x * kLossThreads) {
    const bool ret = a.did_return[i] != 0, m = mask[i] != 0;
    const float dist = a.distance[i];
    d_pred[i] = m ? lidar_depth_grad(a.pred[i], dist, ret, a.non_return_distance, a.non_return_mult, g_depth) : 0.f;
#pragma unroll
    for (int r = 0; r < kLossMaxProp; ++r)
      if (r < a.n_prop)
        d_prop[(int64_t)r * a.n + i] = lidar_depth_grad(a.prop[(int64_t)r * a.prop_stride + i], dist, ret, a.non_return_distance,
                                                        a.non_return_mult, g_prop[r]);
    float di = 0.f;
    if (m && ret) {  // MSELoss(gt, pred): d/d pred = -2 (gt - pred) g
      const float d = simt::fsub(a.gt_intensity[(int64_t)i * a.gt_intensity_stride], a.intensity[i]);
      di = -simt::fmul(simt::fmul(2.f, d), g_int);
    }
    d_intensity[i] = di;
    d_logits[i] = bce_with_logits_grad(a.logits[i], ret ? 0.f : 1.f, g_drop);
  }
}
#endif

}  // namespace nff
