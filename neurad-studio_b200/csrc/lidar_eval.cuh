// lidar_eval.cuh -- lidar evaluation: the exact chamfer distance of NeuRADModel.get_image_metrics_and_images
// (models/neurad.py:614-618, utils/math.py:745-798) as an all-pairs nearest-neighbour kernel.
//
// For every source point the kernel writes min_j |s_i - t_j|^2 over the target set.  The per-pair value is formed from
// direct differences in fp32 (dx = s - t, then dx*dx + dy*dy + dz*dz with two FMAs), never as |s|^2 + |t|^2 - 2 s.t:
// at 100 m ranges |p|^2 ~ 1e4, and that form cancels away the digits of the distance it is meant to measure.  No tensor
// cores are involved.
//
// Layout: a CTA holds CHAMFER_PTS source points per thread in registers and walks target tiles staged in shared memory
// (every thread reads the same target: broadcast LDS.128).  The grid's y dimension splits the target set so that a
// sweep fills every SM; the partial minima of the splits meet in an atomicMin on an order-preserving unsigned key.
// The min is a min over identical per-pair values, so neither the tile order nor the split changes a bit of it.
//
// NaN: a NaN coordinate gives NaN for its own point and for every point whose candidate set contains it, as torch.min
// does.  The per-pair min is PTX min.NaN.f32 (one FMNMX); plain fminf would drop the NaN.
//
// The device functions above the kernels compile as plain C++ as well (tests/host_emul/emul_chamfer.cpp), so the CPU
// tests run this exact per-pair arithmetic.
#pragma once

#include "simt.h"

namespace nff {

constexpr int kChamferThreads = 128;  // threads per CTA
constexpr int kChamferPts = 8;        // source points per thread (register block)
constexpr int kChamferTile = 512;     // target points per shared-memory tile (8 KB as float4)
constexpr int kChamferReduceThreads = 1024;

// |s - t|^2 from direct differences; explicit FMAs, so host and device round identically
NFF_HD float chamfer_sq(float sx, float sy, float sz, float tx, float ty, float tz) {
  const float dx = sx - tx, dy = sy - ty, dz = sz - tz;
  return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// min that propagates NaN (torch.min semantics)
NFF_HD float chamfer_min(float a, float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#else
  if (a != a || b != b) return NAN;
  return b < a ? b : a;
#endif
}

// order-preserving key of a squared distance (>= +0 or NaN) for an unsigned atomicMin: NaN -> 0 (wins every min),
// d -> bits(d) + 1 (bits(+inf) + 1 = 0x7f800001); 0xffffffff is the empty min
NFF_HD unsigned chamfer_key(float d) {
  if (d != d) return 0u;
  unsigned u;
  memcpy(&u, &d, 4);
  return u + 1u;
}
NFF_HD float chamfer_unkey(unsigned k) {
  if (k == 0u) return NAN;
  const unsigned u = k - 1u;
  float d;
  memcpy(&d, &u, 4);
  return d;
}

// One target tile against the thread's register block: m[p] = min(m[p], |s_p - t_k|^2) for k < kChamferTile.  Tiles are
// padded with copies of a real target point, so the loop has a fixed trip count.
NFF_HD void chamfer_tile(const float* tile /* [kChamferTile][4] */, const float (&sx)[kChamferPts], const float (&sy)[kChamferPts],
                         const float (&sz)[kChamferPts], float (&m)[kChamferPts]) {
#if defined(__CUDACC__)
#pragma unroll 4
#endif
  for (int k = 0; k < kChamferTile; ++k) {
    const float tx = tile[4 * k], ty = tile[4 * k + 1], tz = tile[4 * k + 2];
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int p = 0; p < kChamferPts; ++p) m[p] = chamfer_min(m[p], chamfer_sq(sx[p], sy[p], sz[p], tx, ty, tz));
  }
}

// Point (x, y, z) of row i (row stride `stride` floats) and the index clamp that pads tiles / register blocks
NFF_HD int64_t chamfer_row(int64_t i, int64_t n) { return i < n ? i : n - 1; }

#if defined(__CUDACC__)
// keys[i] = min(keys[i], key(min_{j in this CTA's target range} |src_i - dst_j|^2)); keys start at 0xffffffff
__global__ void __launch_bounds__(kChamferThreads) chamfer_min_kernel(const float* __restrict__ src, int n_src, int src_stride,
                                                                      const float* __restrict__ dst, int n_dst, int dst_stride,
                                                                      int tiles_per_split, unsigned* __restrict__ keys) {
  __shared__ __align__(16) float tile[kChamferTile * 4];
  const int n_tiles = (n_dst + kChamferTile - 1) / kChamferTile;
  const int tile0 = blockIdx.y * tiles_per_split;
  const int tile1 = min(tile0 + tiles_per_split, n_tiles);
  if (tile0 >= tile1) return;  // uniform per CTA
  const int64_t base = (int64_t)blockIdx.x * (kChamferThreads * kChamferPts) + threadIdx.x;
  float sx[kChamferPts], sy[kChamferPts], sz[kChamferPts], m[kChamferPts];
#pragma unroll
  for (int p = 0; p < kChamferPts; ++p) {
    const float* s = src + chamfer_row(base + p * kChamferThreads, n_src) * src_stride;
    sx[p] = __ldg(s);
    sy[p] = __ldg(s + 1);
    sz[p] = __ldg(s + 2);
    m[p] = __int_as_float(0x7f800000);
  }
  for (int t = tile0; t < tile1; ++t) {
    __syncthreads();
    for (int k = threadIdx.x; k < kChamferTile; k += kChamferThreads) {
      const float* d = dst + chamfer_row((int64_t)t * kChamferTile + k, n_dst) * dst_stride;
      *reinterpret_cast<float4*>(&tile[4 * k]) = make_float4(__ldg(d), __ldg(d + 1), __ldg(d + 2), 0.f);
    }
    __syncthreads();
    chamfer_tile(tile, sx, sy, sz, m);
  }
#pragma unroll
  for (int p = 0; p < kChamferPts; ++p) {
    const int64_t i = base + p * kChamferThreads;
    if (i < n_src) atomicMin(&keys[i], chamfer_key(m[p]));
  }
}

// One CTA: decode both key arrays in place into fp32 minima and sum each in fp64 in a fixed order (thread t takes
// i = t, t + 1024, ...; then a fixed shared-memory tree), so the scalar is bit-reproducible.
// out = (sum_src + sum_dst) * (normalize ? 1 / n_dst per term : 1), i.e. sum_src / M + sum_dst / M as utils/math.py:783-796.
__global__ void __launch_bounds__(kChamferReduceThreads) chamfer_reduce_kernel(unsigned* __restrict__ src_keys, int n_src,
                                                                               unsigned* __restrict__ dst_keys, int n_dst,
                                                                               int normalize_by_dst, double* __restrict__ out) {
  __shared__ double red[2][kChamferReduceThreads];
  double acc[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < n_src; i += kChamferReduceThreads) {
    const float d = chamfer_unkey(src_keys[i]);
    reinterpret_cast<float*>(src_keys)[i] = d;
    acc[0] += (double)d;
  }
  for (int i = threadIdx.x; i < n_dst; i += kChamferReduceThreads) {
    const float d = chamfer_unkey(dst_keys[i]);
    reinterpret_cast<float*>(dst_keys)[i] = d;
    acc[1] += (double)d;
  }
  red[0][threadIdx.x] = acc[0];
  red[1][threadIdx.x] = acc[1];
  __syncthreads();
  for (int w = kChamferReduceThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      red[0][threadIdx.x] += red[0][threadIdx.x + w];
      red[1][threadIdx.x] += red[1][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double a = red[0][0], b = red[1][0];
    *out = normalize_by_dst ? a / (double)n_dst + b / (double)n_dst : a + b;
  }
}
#endif

}  // namespace nff
