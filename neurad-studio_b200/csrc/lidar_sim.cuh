// lidar_sim.cuh -- the point clouds of simulated lidar sweeps: the return decision, points in world and sensor
// coordinates and an ordered compaction of the kept rays (viewer/render_state_machine.py:416-430,
// models/ad_model.py:107-113).
//
// Layout: a tile of kLsThreads x kLsPer consecutive rays of one sweep per CTA, each thread owning kLsPer consecutive
// rays, grid (tiles per sweep, sweeps).  Three launches:
//   1. lidar_sweep_count_kernel: keep flags, one count per tile;
//   2. lidar_sweep_scan_kernel (one CTA): exclusive scan of the tile counts in (sweep, tile) order, the per-sweep counts,
//      the total and each sweep's first row;
//   3. lidar_sweep_emit_kernel: the same flags again, a CTA scan of the thread counts, and the kept rays written at
//      their tile's offset plus their rank.
// Every row comes from a scan, never from an atomic, so the output is the order of a boolean index and the same bits on
// every run.  The kernels read the render's outputs once more instead of keeping a flag array: the flags cost less to
// recompute than to store and load.
#pragma once

#include "simt.h"

namespace nff {

constexpr int kLsThreads = 256;
constexpr int kLsPer = 4;
constexpr int kLsTile = kLsThreads * kLsPer;
constexpr int kLsScanThreads = 1024;

struct LidarSweepArgs {
  const b200nerf_lidar_sweep* sweeps;
  int64_t per;  // rays per sweep (beams * columns)
  int n_az, beams, tiles;  // columns, beams, tiles per sweep
  const float *origins, *dirs, *times, *depth, *intensity, *prob;
  int use_ray_drop;
  float threshold;
};

// the viewer's filter: ray_drop_prob < threshold with ray drop, depth < max distance without (NaN: not kept)
NFF_D bool lidar_keep(const LidarSweepArgs& a, int64_t i) {
  return a.use_ray_drop ? a.prob[i] < a.threshold : a.depth[i] < a.threshold;
}

// exclusive CTA scan of one int per thread; returns the CTA total
NFF_D int lidar_block_scan(int v, int* excl) {
  __shared__ int warp_sums[kLsThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kLsThreads / 32; ++w) {
    const int ws = warp_sums[w];
    before += w < warp ? ws : 0;
    total += ws;
  }
  *excl = before + x - v;
  return total;
}

__global__ void __launch_bounds__(kLsThreads) lidar_sweep_count_kernel(LidarSweepArgs a, int* __restrict__ tile_counts) {
  const int s = blockIdx.y;
  const int64_t j0 = (int64_t)blockIdx.x * kLsTile + (int64_t)threadIdx.x * kLsPer;
  int c = 0;
#pragma unroll
  for (int u = 0; u < kLsPer; ++u)
    if (j0 + u < a.per) c += lidar_keep(a, s * a.per + j0 + u);
  int excl;
  const int total = lidar_block_scan(c, &excl);
  if (threadIdx.x == 0) tile_counts[(int64_t)s * a.tiles + blockIdx.x] = total;
}

// one CTA: tile_offsets = exclusive scan of tile_counts; counts[s] = kept rays of sweep s, counts[n_sweeps] = total;
// offsets[s] = first row of sweep s
__global__ void __launch_bounds__(kLsScanThreads) lidar_sweep_scan_kernel(int n_sweeps, int tiles, const int* __restrict__ tile_counts,
                                                                          int* __restrict__ tile_offsets, int* __restrict__ counts,
                                                                          int* __restrict__ offsets) {
  __shared__ int warp_sums[kLsScanThreads / 32];
  __shared__ int carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int s = 0; s < n_sweeps; ++s) {
    const int start = carry;
    for (int t0 = 0; t0 < tiles; t0 += kLsScanThreads) {
      const int t = t0 + threadIdx.x;
      const int v = t < tiles ? tile_counts[(int64_t)s * tiles + t] : 0;
      int x = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
      }
      if (lane == 31) warp_sums[warp] = x;
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < kLsScanThreads / 32; ++w) {
        const int ws = warp_sums[w];
        before += w < warp ? ws : 0;
        total += ws;
      }
      const int base = carry;
      if (t < tiles) tile_offsets[(int64_t)s * tiles + t] = base + before + x - v;
      __syncthreads();  // every thread has read carry and warp_sums
      if (threadIdx.x == 0) carry = base + total;
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      offsets[s] = start;
      counts[s] = carry - start;
    }
  }
  if (threadIdx.x == 0) counts[n_sweeps] = carry;
}

__global__ void __launch_bounds__(kLsThreads) lidar_sweep_emit_kernel(LidarSweepArgs a, const int* __restrict__ tile_offsets,
                                                                      float* __restrict__ pts_sensor, float* __restrict__ pts_world,
                                                                      int* __restrict__ index) {
  const int s = blockIdx.y;
  const int64_t j0 = (int64_t)blockIdx.x * kLsTile + (int64_t)threadIdx.x * kLsPer;
  bool keep[kLsPer];
  int c = 0;
#pragma unroll
  for (int u = 0; u < kLsPer; ++u) {
    keep[u] = j0 + u < a.per && lidar_keep(a, s * a.per + j0 + u);
    c += keep[u];
  }
  int excl;
  lidar_block_scan(c, &excl);
  if (c == 0) return;
  int64_t row = (int64_t)tile_offsets[(int64_t)s * a.tiles + blockIdx.x] + excl;
  const b200nerf_lidar_sweep& w = a.sweeps[s];
  float m[12];
#pragma unroll
  for (int r = 0; r < 12; ++r) m[r] = w.l2w[r];
  // pose_inverse (utils/poses.py:42-55): [R^T | -R^T t]
  float tinv[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) tinv[r] = -fadd(fadd(fmul(m[r], m[3]), fmul(m[4 + r], m[7])), fmul(m[8 + r], m[11]));
#pragma unroll
  for (int u = 0; u < kLsPer; ++u) {
    if (!keep[u]) continue;
    const int64_t j = j0 + u, i = s * a.per + j;
    const float dep = a.depth[i];
    float p[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) p[r] = fadd(a.origins[3 * i + r], fmul(a.dirs[3 * i + r], dep));
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      pts_world[3 * row + r] = p[r];
      pts_sensor[5 * row + r] = fadd(fadd(fadd(fmul(m[r], p[0]), fmul(m[4 + r], p[1])), fmul(m[8 + r], p[2])), tinv[r]);
    }
    pts_sensor[5 * row + 3] = a.intensity[i];
    pts_sensor[5 * row + 4] = fsub(a.times[i], w.scan_time);
    index[3 * row] = s;
    index[3 * row + 1] = (int)(j / a.n_az);
    index[3 * row + 2] = (int)(j % a.n_az);
    ++row;
  }
}

}  // namespace nff
