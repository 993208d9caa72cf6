// b200nerf.cu -- kernels + C ABI of libb200nerf.so (sm_90a).  See include/b200nerf.h for the contract.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../include/b200nerf.h"
#include "nff_device.h"
#include "nff_lane.h"
#include "rgb_decoder.cuh"
#include "modules.cuh"

using namespace nff;

// ------------------------------------------------------------------------------------------- error plumbing
static thread_local std::string g_err;
static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                                   \
  do {                                                                                                   \
    cudaError_t e_ = (expr);                                                                             \
    if (e_ != cudaSuccess)                                                                               \
      return fail(B200NERF_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));                \
  } while (0)
#define REQUIRE(cond, msg) \
  do {                     \
    if (!(cond)) return fail(B200NERF_ERR_INVALID, std::string(msg)); \
  } while (0)

struct b200nerf_ctx {
  int device = 0;
  int sm_count = 0;
  FieldGrids fields[3]{};
  bool have_field[3] = {false, false, false};
  const float** d_actor_tables[3] = {nullptr, nullptr, nullptr};
  float* d_decoder[3] = {nullptr, nullptr, nullptr};
  float* d_main_mlp = nullptr;
  float* d_main_mlp_nn = nullptr;
  cudaStream_t param_stream = 0;  // stream of the set_* packing kernels / copies (b200nerf_set_param_stream)
  int act_alloc_actors = 0, act_alloc_times = 0;  // sizes the actor arrays are currently allocated for
  int layout = 0;    // 0: torch-mode grids (b200nerf_set_field_grids); 1: tiny-cuda-nn layout (b200nerf_set_field_grids_tcnn)
  int field_layout[3] = {0, 0, 0};
  int mlp_mode = 3;  // 3 = ray-per-lane in two kernels (sampling | shading + wgmma), 2 = the same as one fused kernel, 1 = warp-per-ray + wgmma (3xTF32), 0 = warp-per-ray + CUDA-core fp32 FFMA
  float* d_lane_scratch = nullptr;
  int lane_ctas = 0;
  unsigned* d_minmax = nullptr;      // [2] ordered-bit min / max of the depth steps (DepthRenderer "expected" clip)
  float* d_handoff = nullptr;        // [kS2+1][rays] spacing edges between the sampling and the shading kernel
  int64_t handoff_rays = 0;
  b200nerf_peer_outputs peers{};
  bool have_main_mlp = false;
  float beta = 0.f;
  float* d_lidar_mlp = nullptr;
  bool have_lidar = false;
  Appearance app{};
  bool have_app = false;
  Actors actors{};
  float *d_act_times = nullptr, *d_act_kf = nullptr, *d_act_bounds = nullptr, *d_act_radii = nullptr;
  uint8_t* d_act_present = nullptr;
  Sampling samp{};
  bool have_samp = false;
  float *d_u1 = nullptr, *d_u2 = nullptr;
  int* d_status = nullptr;
  int n_prop0 = 0, n_prop1 = 0, n_nerf = 0;
  // NeuRADModel.rgb_decoder (rgb_decoder.cuh): folded / re-laid-out parameters owned by the context
  bool have_rgb_decoder = false;
  int dec_in_dim = 0;
  unsigned char* d_dec_wimg[8] = {};  // [49][hi|lo] bf16 GMMA B tiles per 7x7 conv
  float* d_dec_wf32[8] = {};          // [49][ci][co] fp32 (CUDA-core reference kernel)
  float* d_dec_bias = nullptr;        // [8][32] folded conv + BN biases
  float* d_dec_small = nullptr;       // in conv w [32*in] b [32] | convT w [32*32*9] b [32] | out conv w [3*32] b [3]
  bool mlp_attr_set = false;            // mlp_tc_kernel's dynamic shared memory opt-in done on this device
  float** d_grad_actor_ptrs = nullptr;  // [kModMaxActors] per-actor gradient accumulators of the current encoding_bwd call
};

namespace {
struct DeviceGuard {
  int prev = 0;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() { cudaSetDevice(prev); }
};

int make_grid(const b200nerf_grid_desc* d, const float* table, Grid* g) {
  REQUIRE(d != nullptr, "grid descriptor is NULL");
  REQUIRE(d->num_levels >= 1 && d->num_levels <= kMaxLevels, "num_levels must be in [1,16]");
  REQUIRE(d->log2_hashmap_size >= 1 && d->log2_hashmap_size <= 30, "log2_hashmap_size out of range");
  g->table = table;
  g->T = 1u << d->log2_hashmap_size;
  g->mask = g->T - 1u;
  g->L = d->num_levels;
  g->F = d->features_per_level;
  for (int i = 0; i < kMaxLevels; ++i) g->res[i] = i < d->num_levels ? d->scalings[i] : 0.f;
  return 0;
}

// The fused kernels address a level's rows by 32-bit byte offsets pre-multiplied into the hash (grid_cell_b /
// cell_offsets_b: (h & mask) << log2(row bytes)), which is exact while log2 T + log2(4 F) <= 32.
bool fused_table_fits(int log2_hashmap_size, int F) {
  const int row_shift = F == 4 ? 4 : 2;
  return log2_hashmap_size + row_shift <= 32;
}

// The tiny-cuda-nn kernels hold entry indices (level offset + index in the level, a dense level's before its wrap: below
// twice its size) in 32 bits.
bool tcnn_entries_fit(const b200nerf_tcnn_grid_desc* d) {
  for (int l = 0; l < d->num_levels; ++l)
    if ((uint64_t)d->offset[l] + 2ull * d->size[l] > (1ull << 32)) return false;
  return true;
}
}  // namespace

// =================================================================================================== kernels
#ifndef NFF_WARPS
#define NFF_WARPS 8
#endif
constexpr int kSmemMaxOptIn = 227 * 1024;  // dynamic shared memory a CTA may opt in to on sm_90
constexpr int kRenderWarps = NFF_WARPS;  // warps (= rays in flight) per CTA; 16 warps/SM at <=128 registers

// CUDA-core MLP variant (exact fp32 FFMA): the reference/fallback numerics mode.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 16 / WARPS) nff_render_kernel(const __grid_constant__ RenderParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* mlp_s = reinterpret_cast<float*>(smem_raw);
  constexpr int kMlpBytes = (kMainMlpFloats * 4 + 15) / 16 * 16;
  WarpShared* ws = reinterpret_cast<WarpShared*>(smem_raw + kMlpBytes) + (threadIdx.x >> 5);
  for (int i = threadIdx.x; i < kMainMlpFloats; i += WARPS * 32) mlp_s[i] = P.main_mlp[i];
  __syncthreads();
  MlpFfma mlp{mlp_s};
  const int64_t stride = (int64_t)gridDim.x * WARPS;
  for (int64_t ray = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5); ray < P.n_rays; ray += stride)
    render_ray(P, *ws, mlp, ray, true);
}

// Tensor-core MLP variant (wgmma, 3xTF32): each group of 4 warps (a warp group) forms one 128-row tile.
using WarpSharedTc = WarpSharedT<kNff>;
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 16 / WARPS) nff_render_tc_kernel(const __grid_constant__ RenderParams P) {
  static_assert(WARPS % 4 == 0 && WARPS <= 16, "warp groups of 4");
  extern __shared__ __align__(128) unsigned char smem_tc[];
  TcShared* tcs = reinterpret_cast<TcShared*>(smem_tc);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), group = warp >> 2;
  WarpSharedTc* ws = reinterpret_cast<WarpSharedTc*>(smem_tc + tc_smem_bytes(WARPS * 32)) + warp;
  tc_stage_weights(*tcs, P.main_mlp_nn, threadIdx.x, WARPS * 32);
  tc::fence_async_smem();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
  __syncthreads();
  MlpTc mlp;
  mlp.t = tcs;
  mlp.stage = reinterpret_cast<float*>(smem_tc + kTcBytes) + group * kTcStageFloats;
  mlp.bar_id = 1 + group;
  const int64_t stride = (int64_t)gridDim.x * WARPS;
  for (int64_t base = (int64_t)blockIdx.x * WARPS; base < P.n_rays; base += stride) {
    const int64_t ray = base + warp;
    const bool active = ray < P.n_rays;
    render_ray(P, *ws, mlp, active ? ray : P.n_rays - 1, active);
  }
}



// Work units of the ray-per-lane kernels: with an image_width hint a CTA walks 32 x (threads/32)-pixel tiles and a warp
// renders an 8x4 patch (neighbours in both image directions); without it, kLaneThreads consecutive rays.  Inactive
// lanes (outside the image / beyond the last ray) get a valid fallback ray: they compute but never store.
__device__ __forceinline__ int64_t lane_units(const RenderParams& P) {
  const int W = P.rays.image_width;
  if (W <= 0) return (P.n_rays + kLaneThreads - 1) / kLaneThreads;
  constexpr int kTileH = kLaneThreads / 32;
  const int64_t H = (P.n_rays + W - 1) / W;
  return (int64_t)((W + 31) / 32) * ((H + kTileH - 1) / kTileH);
}
__device__ __forceinline__ bool lane_unit_ray(const RenderParams& P, int64_t unit, int tid, int64_t* ray_out) {
  const int W = P.rays.image_width;
  int64_t ray, fallback;
  bool active;
  if (W > 0) {
    constexpr int kTileH = kLaneThreads / 32;
    const int64_t H = (P.n_rays + W - 1) / W, tiles_x = (W + 31) / 32;
    const int warp = tid >> 5, lane_ = tid & 31;
    const int64_t px = (unit % tiles_x) * 32 + (warp & 3) * 8 + (lane_ & 7);
    const int64_t py = (unit / tiles_x) * kTileH + (warp >> 2) * 4 + (lane_ >> 3);
    ray = py * W + px;
    active = px < W && ray < P.n_rays;
    fallback = (py < H ? py : H - 1) * W + (px < W ? px : W - 1);
  } else {
    ray = unit * kLaneThreads + tid;
    active = ray < P.n_rays;
    fallback = P.n_rays - 1;
  }
  if (fallback >= P.n_rays) fallback = P.n_rays - 1;
  *ray_out = active ? ray : fallback;
  return active;
}

// Work distribution of the two-stage kernels.  The unit of work is a PATCH = the 32 rays of one warp (an 8x4 pixel patch of a
// 32x16 tile when the caller passes image_width, else 32 consecutive rays); patches are numbered tile by tile, so consecutive
// patches are spatial neighbours.  Whole tiles (16 patches = one per warp) are taken grid-stride, tile k * gridDim + blockIdx,
// for as many FULL rounds as there are -- all resident CTAs then work on adjacent tiles, which keeps their common working
// set of grid cells compact in L2 (giving every CTA one long contiguous range instead puts far-apart regions in flight, which
// thrashes L2).  The last, partial round is split evenly over ALL CTAs at patch granularity
// (sampling: round-robin over a CTA's warps, there is no CTA-level synchronisation at all; shading: over its 128-ray warp
// groups, one tensor-core tile = 4 consecutive patches).  With whole 512-ray CTA units a 230 400-ray image is 460 units, which
// no count of resident CTAs (132 SMs on an H100) divides evenly: the SMs with one unit more would set the launch time.
__device__ __forceinline__ int64_t lane_patches(const RenderParams& P) {
  return P.rays.image_width > 0 ? lane_units(P) * (kLaneThreads / 32) : (P.n_rays + 31) / 32;
}
__device__ __forceinline__ bool lane_patch_ray(const RenderParams& P, int64_t patch, int lane_, int64_t* ray_out) {
  constexpr int kPatchesPerUnit = kLaneThreads / 32;
  // same mapping as lane_unit_ray with (unit, warp) = (patch / 16, patch % 16)
  return lane_unit_ray(P, patch / kPatchesPerUnit, (int)(patch % kPatchesPerUnit) * 32 + lane_, ray_out);
}

// Two-stage variant of the ray-per-lane path.  Stage 1 (sampling: both proposal rounds) needs no shared memory beyond round
// 0's 516 B edge table and fits 64 registers, so it runs at 32 warps/SM with nearly the whole 256 KB L1/shared array as L1; stage 2 (main field + MLPs +
// compositing) is the tensor-core kernel at 16 warps/SM.  The hand-over is 33 spacing edges per ray ([edge][ray],
// 132 B/ray) -- still nothing per-sample in HBM.
#ifndef NFF_SAMPLE_CTAS
#define NFF_SAMPLE_CTAS 2
#endif
// LAYOUT 0: the reference's torch-mode grids; 1: tiny-cuda-nn layout (tcnn-trained checkpoints, SURVEY 8f f3).  ACTORS /
// TRACED = false leave the actor path / the trace stores out of the code: the untraced instances fit 64 registers without
// spilling (sample_lane_kernel picks the instance).
template <int LAYOUT, bool ACTORS, bool TRACED>
__global__ void __launch_bounds__(kLaneThreads, NFF_SAMPLE_CTAS) nff_sample_lane_kernel(const __grid_constant__ RenderParams P,
                                                                                        float* __restrict__ scratch,
                                                                                        float* __restrict__ handoff) {
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane_ = tid & 31;
  const LaneScratch sc = lane_scratch_of(scratch, blockIdx.x);
  // round 0's euclidean edges, when no ray has its own near / far
  __shared__ float e0_tab[kS0 + 1];
  const bool shared_edges = !P.rays.nears && !P.rays.fars;
  if (shared_edges) {
    if (tid <= kS0) e0_tab[tid] = lane_round0_edge(P.samp, tid);
    __syncthreads();
  }
  constexpr int kPPU = kLaneThreads / 32;  // patches per tile
  const int64_t n_patches = lane_patches(P);
  // full rounds: tile k * gridDim + blockIdx (the resident CTAs sweep over ADJACENT tiles together: their working set of
  // grid cells stays compact in L2); the last, partial round is dealt out patch by patch so that every SM ends together.
  // One loop (one copy of the body: the kernel has to stay inside the instruction cache).
  const int64_t full_rounds = n_patches / kPPU / gridDim.x;
  const int64_t r0 = full_rounds * gridDim.x * kPPU, rest = n_patches - r0;
  const int64_t p0 = r0 + rest * blockIdx.x / gridDim.x, p1 = r0 + rest * (blockIdx.x + 1) / gridDim.x;
  for (int64_t it = 0;; ++it) {
    int64_t patch;
    if (it < full_rounds) {
      patch = (it * gridDim.x + blockIdx.x) * kPPU + warp;
    } else {
      patch = p0 + warp + (it - full_rounds) * kPPU;
      if (patch >= p1) break;
    }
    int64_t ray;
    const bool active = lane_patch_ray(P, patch, lane_, &ray);
    const LaneRay R = lane_ray_setup<ACTORS>(P, sc, tid, ray);
    // inactive lanes write their (discarded) edges into the slab column instead of another ray's hand-over column
    float* col = active ? handoff + ray : sc.bins2 + tid;
    sample_ray_lane<LAYOUT, ACTORS, TRACED>(P, sc, R, tid, ray, active, col, active ? P.n_rays : (int64_t)kLaneThreads,
                                            shared_edges ? e0_tab : nullptr);
  }
}
// the instance of a launch: `actors` = the scene has actors, `traced` = a proposal-stage trace is recorded (traced renders
// take the instance with the actor path compiled in)
template <int LAYOUT>
static auto sample_lane_kernel(bool actors, bool traced) {
  return traced ? nff_sample_lane_kernel<LAYOUT, true, true>
         : actors ? nff_sample_lane_kernel<LAYOUT, true, false>
                  : nff_sample_lane_kernel<LAYOUT, false, false>;
}

template <int LAYOUT>
__global__ void __launch_bounds__(kLaneThreads, kLaneCtasPerSm) nff_shade_lane_kernel(const __grid_constant__ RenderParams P,
                                                                                      float* __restrict__ scratch,
                                                                                      const float* __restrict__ handoff) {
  extern __shared__ __align__(128) unsigned char smem_shade[];
  TcShared* tcs = reinterpret_cast<TcShared*>(smem_shade);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), group = warp >> 2;
  tc_stage_weights(*tcs, P.main_mlp_nn, tid, kLaneThreads, true);
  tc::fence_async_smem();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
  __syncthreads();
  MlpLaneTc mlp;
  mlp.t = tcs;
  mlp.panel_ = reinterpret_cast<float*>(smem_shade + kTcBytes);
  mlp.bar_id = 1 + group;
  const LaneScratch sc = lane_scratch_of(scratch, blockIdx.x);
  mlp.sh_tcnn = LAYOUT;
  // a warp group (one 128-row tensor-core tile) renders 4 consecutive patches; the groups of a CTA only meet at the two
  // block barrier before the loop, inside it they synchronise among their own 4 warps (named barriers).
  // Full rounds sweep adjacent tiles like the sampling kernel; the partial last round is dealt out group-unit by group-unit.
  constexpr int kPPU = kLaneThreads / 32;
  const int64_t n_patches = lane_patches(P);
  const int64_t full_rounds = n_patches / kPPU / gridDim.x;
  const int64_t r0 = full_rounds * gridDim.x * kPPU;
  const int64_t rest_groups = (n_patches - r0 + 3) / 4;
  const int64_t g0 = rest_groups * blockIdx.x / gridDim.x, g1 = rest_groups * (blockIdx.x + 1) / gridDim.x;
  for (int64_t it = 0;; ++it) {
    int64_t patch;
    if (it < full_rounds) {
      patch = (it * gridDim.x + blockIdx.x) * kPPU + warp;
    } else {
      const int64_t gu = g0 + group + (it - full_rounds) * (kLaneThreads / 128);
      if (gu >= g1) break;
      patch = r0 + gu * 4 + (warp & 3);
    }
    int64_t ray;
    const bool active = lane_patch_ray(P, patch, tid & 31, &ray);
    const LaneRay R = lane_ray_setup(P, sc, tid, ray);
    shade_ray_lane<MlpLaneTc, LAYOUT>(P, sc, R, mlp, tid, ray, active, handoff + ray, P.n_rays);
  }
}

// Ray-per-lane variant (nff_lane.h), single fused kernel: a warp = 32 adjacent rays at the same sample index.
__global__ void __launch_bounds__(kLaneThreads, kLaneCtasPerSm) nff_render_lane_kernel(const __grid_constant__ RenderParams P,
                                                                          float* __restrict__ scratch) {
  extern __shared__ __align__(128) unsigned char smem_lane[];
  TcShared* tcs = reinterpret_cast<TcShared*>(smem_lane);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), group = warp >> 2;
  tc_stage_weights(*tcs, P.main_mlp_nn, tid, kLaneThreads, true);
  tc::fence_async_smem();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
  __syncthreads();
  MlpLaneTc mlp;
  mlp.t = tcs;
  mlp.panel_ = reinterpret_cast<float*>(smem_lane + kTcBytes);
  mlp.bar_id = 1 + group;
  const LaneScratch sc = lane_scratch_of(scratch, blockIdx.x);
  for (int64_t unit = blockIdx.x; unit < lane_units(P); unit += gridDim.x) {
    int64_t ray;
    const bool active = lane_unit_ray(P, unit, tid, &ray);
    render_ray_lane(P, sc, mlp, tid, ray, active);
  }
}

// NeuRADModel.decode_features, lidar half (models/neurad.py:350-357): one thread per ray.
__global__ void lidar_decode_kernel(const float* __restrict__ mlp, const float* __restrict__ feats, int fdim,
                                    int64_t n, float* __restrict__ intensity, float* __restrict__ drop) {
  __shared__ __align__(16) float w[kLidarMlpFloats];
  for (int i = threadIdx.x; i < kLidarMlpFloats; i += blockDim.x) w[i] = mlp[i];
  __syncthreads();
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  float x[kNff + kApp];
#pragma unroll
  for (int i = 0; i < kNff + kApp; ++i) x[i] = i < fdim ? feats[r * fdim + i] : 0.f;
  float h[kHidden], h2[kHidden], o[2];
  dense<kNff + kApp, kHidden, kHidden, true>(w + kOffLidW0, w + kOffLidB0, x, h);
  dense<kHidden, kHidden, kHidden, true>(w + kOffLidW1, w + kOffLidB1, h, h2);
  dense<kHidden, 2, kLidOutP, false>(w + kOffLidW2, w + kOffLidB2, h2, o);
  if (intensity) intensity[r] = 1.0f / (1.0f + expf(-o[0]));
  if (drop) drop[r] = o[1];
}

// HashEncoding.forward (encodings.py:425-471), generic L / F: one thread per (point, level).
__global__ void hashgrid_fwd_kernel(Grid g, const float* __restrict__ x, float* __restrict__ out,
                                    int32_t* __restrict__ indices, int64_t n_points) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_points * g.L) return;
  int64_t p = i / g.L;
  int l = (int)(i % g.L);
  Cell c = grid_cell(x[3 * p], x[3 * p + 1], x[3 * p + 2], g.res[l]);
  uint32_t r[8];
  cell_rows(c, g.mask, r);
  if (indices) {
#pragma unroll
    for (int k = 0; k < 8; ++k) indices[(p * g.L + l) * 8 + k] = (int32_t)(r[k] + (uint32_t)l * g.T);
  }
  const float* base = g.table + (size_t)l * g.T * g.F;
  for (int f = 0; f < g.F; ++f) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __ldg(base + (size_t)r[k] * g.F + f);
    out[p * g.L * g.F + l * g.F + f] = trilerp(v, c);
  }
}

// tcnn.Encoding{HashGrid}.forward (stage operator of the tiny-cuda-nn layout): one thread per point.
template <int D>
__global__ void tcnn_hashgrid_fwd_kernel(Grid g, const float* __restrict__ x, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float p[D];
  for (int d = 0; d < D; ++d) p[d] = x[i * D + d];
  for (int l = 0; l < g.L; ++l) {
    uint32_t idx[1 << D];
    float frac[D];
    tcnn_corners<D>(g, l, p, idx, frac);
    for (int f = 0; f < g.F; ++f) {
      float v = 0.f;
      for (int c = 0; c < (1 << D); ++c) v = fmaf(tcnn_corner_weight<D>(c, frac), g.table[(size_t)idx[c] * g.F + f], v);
      out[i * (g.L * g.F) + l * g.F + f] = v;
    }
  }
}

__global__ void sh4_fwd_kernel(const float* __restrict__ dirs, float* __restrict__ out, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // SHEncoding receives get_normalized_directions(d) = (d+1)/2 from the field; as a stand-alone operator it is
  // the polynomial of utils/math.py:31-94 applied to its input as is.
  float x = dirs[3 * i], y = dirs[3 * i + 1], z = dirs[3 * i + 2];
  float c[16];
  sh4_poly(x, y, z, c);
#pragma unroll
  for (int k = 0; k < 16; ++k) out[16 * i + k] = c[k];
}

// PDFSampler (ray_samplers.py:309-361), generic S: one warp per ray, cdf in shared memory.
// Training mode (train_stratified, ray_samplers.py:321-329): u = linspace(0, 1 - 1/nb, nb) + rand / nb with `rand`
// [N, rand_cols] (rand_cols = 1: single_jitter, else nb); `u` then holds the linspace part.
__global__ void pdf_resample_kernel(const float* __restrict__ weights, const float* __restrict__ bins,
                                    const float* __restrict__ u, int n_rays, int S, int S_new, float hist_pad,
                                    float* __restrict__ new_bins, float* __restrict__ cdf_out,
                                    int32_t* __restrict__ inds, const float* __restrict__ rand = nullptr, int rand_cols = 0) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  float* cdf = sm + warp * (S + 1);
  int ray = blockIdx.x * (blockDim.x >> 5) + warp;
  if (ray >= n_rays) return;
  const float* w = weights + (size_t)ray * S;
  const float* b = bins + (size_t)ray * (S + 1);
  float part = 0.f;
  for (int s = ln; s < S; s += 32) part += __fadd_rn(w[s], hist_pad);
  float tot = warp_sum(part);
  float padding = fmaxf(__fsub_rn(1e-5f, tot), 0.f);
  float pad_each = __fdiv_rn(padding, (float)S);
  tot = __fadd_rn(tot, padding);
  float carry = 0.f;
  for (int s0 = 0; s0 < S; s0 += 32) {
    int s = s0 + ln;
    float pdf = s < S ? __fdiv_rn(__fadd_rn(__fadd_rn(w[s], hist_pad), pad_each), tot) : 0.f;
    float incl = warp_scan_add(pdf) + carry;
    carry = __shfl_sync(0xffffffffu, incl, 31);
    if (s < S) cdf[s + 1] = fminf(1.f, incl);
  }
  if (ln == 0) cdf[0] = 0.f;
  __syncwarp();
  if (cdf_out)
    for (int s = ln; s <= S; s += 32) cdf_out[(size_t)ray * (S + 1) + s] = cdf[s];
  for (int i = ln; i <= S_new; i += 32) {
    float uu = u[i];
    if (rand) uu = __fadd_rn(uu, __fdiv_rn(rand[(size_t)ray * rand_cols + (rand_cols == 1 ? 0 : i)], (float)(S_new + 1)));
    int lo = 0, hi = S + 1;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (cdf[mid] <= uu) lo = mid + 1; else hi = mid;
    }
    int below = min(max(lo - 1, 0), S), above = min(lo, S);
    float c0 = cdf[below], c1 = cdf[above];
    float t = nan_to_num(__fdiv_rn(__fsub_rn(uu, c0), __fsub_rn(c1, c0)));
    t = fminf(fmaxf(t, 0.f), 1.f);
    new_bins[(size_t)ray * (S_new + 1) + i] = __fadd_rn(b[below], __fmul_rn(t, __fsub_rn(b[above], b[below])));
    if (inds) inds[(size_t)ray * (S_new + 1) + i] = lo;
  }
}

// RaySamples.get_weights (rays.py:188-210) / nerfacc.render_weight_from_alpha: one warp per ray, generic S.
template <bool FROM_ALPHA>
__global__ void weights_kernel(const float* __restrict__ a, const float* __restrict__ b, int n_rays, int S,
                               float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  int ray = blockIdx.x * (blockDim.x >> 5) + warp;
  if (ray >= n_rays) return;
  float carry = FROM_ALPHA ? 1.f : 0.f;
  for (int s0 = 0; s0 < S; s0 += 32) {
    int s = s0 + ln;
    size_t idx = (size_t)ray * S + s;
    if (FROM_ALPHA) {
      float al = s < S ? a[idx] : 0.f;
      float incl = warp_scan_mul(1.f - al) * carry;
      float prev = __shfl_up_sync(0xffffffffu, incl, 1);
      float T = ln == 0 ? carry : prev;
      carry = __shfl_sync(0xffffffffu, incl, 31);
      if (s < S) out[idx] = al * T;
    } else {
      float dd = s < S ? __fmul_rn(a[idx], b[idx]) : 0.f;
      float incl = warp_scan_add(dd);
      float prev = __shfl_up_sync(0xffffffffu, incl, 1);
      float excl = carry + (ln == 0 ? 0.f : prev);
      carry += __shfl_sync(0xffffffffu, incl, 31);
      if (s < S) out[idx] = nan_to_num((1.f - expf(-dd)) * expf(-excl));
    }
  }
}

// ---------------------------------------------------------------------------------------- generic stage operators
// SpacedSampler.generate_ray_samples, eval mode (model_components/ray_samplers.py:80-132) for the reference's spacing
// functions: Uniform (:135-156), LinearDisparity (:159-180), Sqrt (:183-204), Log (:207-228), Power (:838-852).
struct SpacingArgs {
  int kind;
  Sampling power;  // kind == B200NERF_SPACING_POWER
};
__device__ __forceinline__ float spacing_apply(const SpacingArgs& a, float x) {
  switch (a.kind) {
    case 0: return x;
    case 1: return fdiv(1.0f, x);
    case 2: return spacing_fn(x, a.power);
    case 3: return fsqrt(x);
    default: return logf(x);
  }
}
__device__ __forceinline__ float spacing_invert(const SpacingArgs& a, float y) {
  switch (a.kind) {
    case 0: return y;
    case 1: return fdiv(1.0f, y);
    case 2: return spacing_fn_inv(y, a.power);
    case 3: return fmul(y, y);
    default: return expf(y);
  }
}
__global__ void spaced_sample_kernel(const SpacingArgs a, const float* __restrict__ nears, const float* __restrict__ fars,
                                     int64_t n_rays, int S, float* __restrict__ bins_s, float* __restrict__ bins_e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * (S + 1)) return;
  const int64_t ray = i / (S + 1);
  const int e = (int)(i % (S + 1));
  const float u = linspace01(e, S);
  if (bins_s && ray == 0) bins_s[e] = u;
  const float s_near = spacing_apply(a, nears ? nears[ray] : 0.0f), s_far = spacing_apply(a, fars[ray]);
  bins_e[i] = spacing_invert(a, fadd(fmul(u, s_far), fmul(fsub(1.0f, u), s_near)));
}
// Training mode of SpacedSampler.generate_ray_samples (train_stratified, ray_samplers.py:107-115): every edge moves
// inside [lower, upper] = the midpoints towards its neighbours, bins = lower + (upper - lower) * t_rand with t_rand
// [N, rand_cols] (rand_cols = 1: single_jitter, else S+1) drawn by the caller; per-ray spacing bins are an output.
__global__ void spaced_sample_jitter_kernel(const SpacingArgs a, const float* __restrict__ nears, const float* __restrict__ fars,
                                            const float* __restrict__ t_rand, int rand_cols, int64_t n_rays, int S,
                                            float* __restrict__ bins_s, float* __restrict__ bins_e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * (S + 1)) return;
  const int64_t ray = i / (S + 1);
  const int e = (int)(i % (S + 1));
  const float b = linspace01(e, S);
  const float lower = e == 0 ? b : fdiv(fadd(b, linspace01(e - 1, S)), 2.0f);
  const float upper = e == S ? b : fdiv(fadd(linspace01(e + 1, S), b), 2.0f);
  const float t = t_rand[ray * rand_cols + (rand_cols == 1 ? 0 : e)];
  const float u = fadd(lower, fmul(fsub(upper, lower), t));
  bins_s[i] = u;
  const float s_near = spacing_apply(a, nears ? nears[ray] : 0.0f), s_far = spacing_apply(a, fars[ray]);
  bins_e[i] = spacing_invert(a, fadd(fmul(u, s_far), fmul(fsub(1.0f, u), s_near)));
}
// spacing_to_euclidean_fn (ray_samplers.py:119-120) applied to per-ray spacing-domain edges, e.g. PDFSampler's output
// bins (ray_samplers.py:363-366): euclid = g^-1(x * g(far) + (1 - x) * g(near)).
__global__ void spacing_to_euclidean_kernel(const SpacingArgs a, const float* __restrict__ nears, const float* __restrict__ fars,
                                            const float* __restrict__ bins_s, int64_t n_rays, int S1, float* __restrict__ bins_e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S1) return;
  const int64_t ray = i / S1;
  const float u = bins_s[i];
  const float s_near = spacing_apply(a, nears ? nears[ray] : 0.0f), s_far = spacing_apply(a, fars[ray]);
  bins_e[i] = spacing_invert(a, fadd(fmul(u, s_far), fmul(fsub(1.0f, u), s_near)));
}
// Frustums.get_positions (cameras/rays.py:50-59) + SceneBox.get_normalized_positions (data/scene_box.py:63-79)
struct AabbArgs {
  int normalize;
  float lo[3], len[3];
};
__global__ void frustum_positions_kernel(const AabbArgs a, const float* __restrict__ origins, const float* __restrict__ dirs,
                                         const float* __restrict__ bins_e, int64_t n_rays, int S, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S) return;
  const int64_t ray = i / S;
  const int s = (int)(i % S);
  const float t = fadd(bins_e[ray * (S + 1) + s], bins_e[ray * (S + 1) + s + 1]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float p = fadd(origins[3 * ray + k], fdiv(fmul(dirs[3 * ray + k], t), 2.0f));
    if (a.normalize) p = fdiv(fsub(p, a.lo[k]), a.len[k]);
    out[3 * i + k] = p;
  }
}
// Field head activations of the reference's density + colour fields: density = trunc_exp(raw[...,0])
// (field_components/activations.py:28-35), rgb = Sigmoid(raw[...,1:1+C]).
__global__ void density_rgb_heads_kernel(const float* __restrict__ raw, int64_t n, int C, float* __restrict__ density,
                                         float* __restrict__ rgb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * (C + 1)) return;
  const int64_t p = i / (C + 1);
  const int k = (int)(i % (C + 1));
  const float v = raw[i];
  if (k == 0) density[p] = expf(v);
  else rgb[p * C + (k - 1)] = fdiv(1.0f, fadd(1.0f, expf(-v)));
}

// Renderers on dense [N,S] samples, one warp per ray (lane = sample):
//   values:        FeatureRenderer / RGBRenderer.combine_rgb (renderers.py:83-85, 103-148): sum_s w*v (+ bg*(1-acc))
//   accumulation:  AccumulationRenderer (renderers.py:322-350)
//   depth:         DepthRenderer "expected" (:396-416, the global clip is applied by depth_clip_kernel), "median"
//                  (:383-394), or NeuRAD's un-normalised render_depth_simple (models/neurad.py:727-734)
__device__ __forceinline__ unsigned order_bits(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unorder_bits(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
struct CompositeArgs {
  int C, value_nan_to_num, has_background, depth_method;
  float background[64];
};
__global__ void composite_kernel(const CompositeArgs a, const float* __restrict__ weights, const float* __restrict__ values,
                                 const float* __restrict__ starts, const float* __restrict__ ends, int64_t n_rays, int S,
                                 float* __restrict__ out_values, float* __restrict__ out_acc, float* __restrict__ out_depth,
                                 unsigned* __restrict__ minmax) {
  const int ln = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  float acc = 0.f, dsum = 0.f, smin = 3.4e38f, smax = -3.4e38f, median = 0.f;
  double carry = 0.0;
  int below = 0;
  const bool want_depth = a.depth_method != 0 && out_depth;
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + ln;
    const float w = s < S ? weights[ray * S + s] : 0.f;
    acc += w;
    if (want_depth) {
      const float mid = s < S ? fdiv(fadd(starts[ray * S + s], ends[ray * S + s]), 2.0f) : 0.f;
      dsum += fmul(w, mid);
      if (s < S) { smin = fminf(smin, mid); smax = fmaxf(smax, mid); }
      if (a.depth_method == 2) {  // torch.cumsum accumulates fp32 inputs in double on the CPU path; mirror that
        double c = (double)w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          double n = __shfl_up_sync(0xffffffffu, c, d);
          if (ln >= d) c += n;
        }
        c += carry;
        carry = __shfl_sync(0xffffffffu, c, 31);
        below += __popc(__ballot_sync(0xffffffffu, s < S && (float)c < 0.5f));
      }
    }
  }
  acc = warp_sum(acc);
  if (out_acc && ln == 0) out_acc[ray] = acc;
  if (want_depth) {
    dsum = warp_sum(dsum);
    if (a.depth_method == 2) {
      const int idx = below < S - 1 ? below : S - 1;
      median = fdiv(fadd(starts[ray * S + idx], ends[ray * S + idx]), 2.0f);
    }
    if (a.depth_method == 1) {
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        smin = fminf(smin, __shfl_xor_sync(0xffffffffu, smin, m));
        smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, m));
      }
      if (ln == 0) {
        atomicMin(&minmax[0], order_bits(smin));
        atomicMax(&minmax[1], order_bits(smax));
      }
    }
    if (ln == 0)
      out_depth[ray] = a.depth_method == 1 ? fdiv(dsum, fadd(acc, 1e-10f)) : a.depth_method == 2 ? median : dsum;
  }
  if (values && out_values) {
    const int C = a.C;
    for (int c0 = 0; c0 < C; c0 += 8) {  // 8 channels per pass keeps the per-lane partial sums in registers
      float part[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) part[k] = 0.f;
      for (int s = ln; s < S; s += 32) {
        const float w = weights[ray * S + s];
        const float* v = values + (ray * S + s) * C + c0;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (c0 + k < C) {
            float x = v[k];
            if (a.value_nan_to_num) x = nan_to_num(x);
            part[k] += fmul(w, x);
          }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float t = warp_sum(part[k]);
        if (ln == 0 && c0 + k < C) out_values[ray * C + c0 + k] = a.has_background ? fadd(t, fmul(a.background[c0 + k], fsub(1.0f, acc))) : t;
      }
    }
  }
}
__global__ void depth_clip_kernel(float* __restrict__ depth, int64_t n, const unsigned* __restrict__ minmax) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float lo = unorder_bits(minmax[0]), hi = unorder_bits(minmax[1]);
  depth[i] = fminf(fmaxf(depth[i], lo), hi);  // torch.clip
}

// Per-keyframe Gram-Schmidt of the 6-D rotations (utils/poses.py:107-114) + actor_bounds / radii
// (dynamic_actors.py:107-108, neurad_encoding.py:227).
__global__ void actors_prep_kernel(int n_times, int n_actors, const float* __restrict__ rot6, const float* __restrict__ pos,
                                   const float* __restrict__ sizes, float p0, float p1, float p2,
                                   float* __restrict__ kf, float* __restrict__ bounds, float* __restrict__ radii) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_times * n_actors) {
    float a1[3] = {rot6[6 * i], rot6[6 * i + 1], rot6[6 * i + 2]};
    float a2[3] = {rot6[6 * i + 3], rot6[6 * i + 4], rot6[6 * i + 5]};
    normalize3(a1);
    float dt = fadd(fadd(fmul(a1[0], a2[0]), fmul(a1[1], a2[1])), fmul(a1[2], a2[2]));
    a2[0] = fsub(a2[0], fmul(dt, a1[0]));
    a2[1] = fsub(a2[1], fmul(dt, a1[1]));
    a2[2] = fsub(a2[2], fmul(dt, a1[2]));
    normalize3(a2);
    float* o = kf + 9 * (size_t)i;
    o[0] = a1[0]; o[1] = a1[1]; o[2] = a1[2];
    o[3] = a2[0]; o[4] = a2[1]; o[5] = a2[2];
    o[6] = pos[3 * i]; o[7] = pos[3 * i + 1]; o[8] = pos[3 * i + 2];
  }
  if (i < n_actors) {
    float b0 = fadd(fmul(sizes[3 * i], 0.5f), p0), b1 = fadd(fmul(sizes[3 * i + 1], 0.5f), p1),
          b2 = fadd(fmul(sizes[3 * i + 2], 0.5f), p2);
    bounds[3 * i] = b0; bounds[3 * i + 1] = b1; bounds[3 * i + 2] = b2;
    radii[i] = fsqrt(fadd(fadd(fmul(b0, b0), fmul(b1, b1)), fmul(b2, b2)));
  }
}

// Repack nn.Linear [out,in] weights into the transposed, padded [in][outp] layout the kernels read.
__global__ void pack_linear_kernel(const float* __restrict__ w, const float* __restrict__ b, int out_f, int in_f,
                                   int outp, float* __restrict__ dst_w, float* __restrict__ dst_b) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < in_f * outp) {
    int k = i / outp, o = i % outp;
    dst_w[i] = o < out_f ? w[o * in_f + k] : 0.f;
  }
  if (i < outp) dst_b[i] = (i < out_f && b) ? b[i] : 0.f;
}


// MLP.forward (field_components/mlp.py:142-183) for NeuRAD's tiny MLPs on the tensor cores: up to 3 Linear layers,
// ReLU between them, in/out widths <= 64.  One CTA (one warp group) = one 128-row tile at a time (grid-stride), each
// layer a wgmma tile product through a shared-memory stage, weights in shared memory (see tc_mlp.cuh).
struct MlpArgs {
  const float* w[3];
  const float* b[3];
  int n_layers, in_dim;
  int k_real[3], n_real[3], k_pad[3], n_pad[3];
  int smem_off[3];  // float offsets of each layer's (hi) tile; lo follows at +n_pad*k_pad
  int bias_off;
  int mma_off;    // [128][tc::stage_pitch(kTcKMax)] stage of the tensor-core layers
  int stage_off;  // 2 x [128][max(kTcKMax, kTcNMax) + 1] row tiles (input rows in / output rows out, double buffered)
  float* hidden_pre[2];  // training: pre-activation rows [n_rows, n_real[l]] of hidden layer l, or NULL
  const float* relu_mask;  // backward: rows [n_rows, out_dim] of a pre-activation Z; the output is multiplied by (Z > 0), or NULL
};
template <int kTcKMax, int kTcNMax>
__global__ void __launch_bounds__(128) mlp_tc_kernel(const MlpArgs a, const float* __restrict__ x, float* __restrict__ y,
                                                     int64_t n_rows, int* __restrict__ status) {
  extern __shared__ __align__(128) float sm_mlp[];
  const int tid = threadIdx.x;
  for (int l = 0; l < a.n_layers; ++l) {
    float* hi = sm_mlp + a.smem_off[l];
    tc::stage_b_tile(hi, hi + a.n_pad[l] * a.k_pad[l], a.w[l], a.n_real[l], a.k_real[l], a.n_pad[l], a.k_pad[l], tid, 128);
    for (int i = tid; i < kTcNMax; i += 128) sm_mlp[a.bias_off + l * kTcNMax + i] = (i < a.n_real[l] && a.b[l]) ? a.b[l][i] : 0.f;
  }
  tc::fence_async_smem();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
  __syncthreads();
  float* mma_stage = sm_mlp + a.mma_off;
  constexpr int kMmaPitch = tc::stage_pitch(kTcKMax);
  const int out_dim = a.n_real[a.n_layers - 1];
  // Rows travel through shared-memory tiles with an odd pitch: the CTA's 128 rows are one contiguous block of global
  // memory, moved with coalesced accesses by all threads, while thread = row reads its own row from shared memory
  // without bank conflicts.  (Thread = row straight from global memory touches 32 different lines per load instruction:
  // 48 loads + 48 stores x 32 wavefronts made the LSU the limit.)  The NEXT tile's rows are fetched with cp.async into
  // the other buffer while this tile goes through the layers: with 8 warps per SM (two CTAs) nothing else
  // would hide the DRAM latency.
  constexpr int kPitch = (kTcKMax > kTcNMax ? kTcKMax : kTcNMax) + 1;
  float* stage0 = sm_mlp + a.stage_off;
  float* mask_tile = stage0 + 2 * 128 * kPitch;  // [128 * out_dim], present when a.relu_mask
  auto fetch_rows = [&](int64_t tile, float* buf) {  // asynchronous: 4-byte cp.async per element, no registers held
    const int rows_here = (int)(n_rows - tile * 128 < 128 ? n_rows - tile * 128 : 128);
    const float* src = x + tile * 128 * a.in_dim;
    const int n_el = rows_here * a.in_dim, qstep = 128 / a.in_dim, rstep = 128 - qstep * a.in_dim;
    int r = tid / a.in_dim, cidx = tid - r * a.in_dim;
    for (int e = tid; e < n_el; e += 128) {
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(buf + r * kPitch + cidx);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src + e) : "memory");
      r += qstep, cidx += rstep;
      if (cidx >= a.in_dim) cidx -= a.in_dim, ++r;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if ((int64_t)blockIdx.x * 128 < n_rows) fetch_rows(blockIdx.x, stage0);
  int it = 0;
  for (int64_t tile = blockIdx.x; tile * 128 < n_rows; tile += gridDim.x, ++it) {
    const int64_t row = tile * 128 + tid;
    const int rows_here = (int)(n_rows - tile * 128 < 128 ? n_rows - tile * 128 : 128);
    float* stage = stage0 + (it & 1) * (128 * kPitch);
    const int64_t next = tile + gridDim.x;
    // one cp.async group per iteration: the NEXT tile's input rows and (dgrad) THIS tile's mask rows, which are only needed
    // by the store loop at the end of the iteration
    const bool more = next * 128 < n_rows;
    if (a.relu_mask) {
      const float* src = a.relu_mask + tile * 128 * out_dim;
      const uint32_t dst0 = (uint32_t)__cvta_generic_to_shared(mask_tile);
      for (int e = tid; e < rows_here * out_dim; e += 128)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst0 + 4u * e), "l"(src + e) : "memory");
      if (!more) asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (more) fetch_rows(next, stage0 + ((it + 1) & 1) * (128 * kPitch));  // commits the group
    if (more || a.relu_mask)
      asm volatile("cp.async.wait_group 1;" ::: "memory");  // everything but this iteration's group: this tile's rows are in
    else
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    float v[kTcKMax];
#pragma unroll
    for (int k = 0; k < kTcKMax; ++k) v[k] = (row < n_rows && k < a.in_dim) ? stage[tid * kPitch + k] : 0.f;
    for (int l = 0; l < a.n_layers; ++l) {
      const float* hi = sm_mlp + a.smem_off[l];
      const float* lo = hi + a.n_pad[l] * a.k_pad[l];
      auto sync = [] { __syncthreads(); };
      float d[kTcNMax];
      switch (a.n_pad[l]) {  // the MMA's N is an immediate: one instantiation per padded width (host: multiple of 16)
        case 16: tc::tile_layer<kTcKMax, 16>(mma_stage, kMmaPitch, v, a.k_pad[l], hi, lo, d, sync); break;
        case 32: tc::tile_layer<kTcKMax, 32>(mma_stage, kMmaPitch, v, a.k_pad[l], hi, lo, d, sync); break;
        case 48: tc::tile_layer<kTcKMax, 48>(mma_stage, kMmaPitch, v, a.k_pad[l], hi, lo, d, sync); break;
        default:
          if constexpr (kTcNMax > 48) tc::tile_layer<kTcKMax, 64>(mma_stage, kMmaPitch, v, a.k_pad[l], hi, lo, d, sync);
          break;
      }
      const float* bias = sm_mlp + a.bias_off + l * kTcNMax;
      const bool last = l == a.n_layers - 1;
      float* hid = last ? nullptr : a.hidden_pre[l];  // warp-uniform
#pragma unroll
      for (int k = 0; k < kTcNMax; ++k) {
        float o = k < a.n_pad[l] ? d[k] + bias[k] : 0.f;
        if (hid && k < a.n_real[l]) stage[tid * kPitch + k] = o;  // (the input rows were consumed before this layer's barrier)
        v[k] = last ? o : fmaxf(o, 0.f);
      }
      if (hid) {  // the hidden pre-activation rows leave through the same tile, coalesced
        __syncthreads();
        const int W = a.n_real[l], n_el = rows_here * W, qstep = 128 / W, rstep = 128 - qstep * W;
        float* dst = hid + tile * 128 * W;
        int r = tid / W, cidx = tid - r * W;
        for (int e = tid; e < n_el; e += 128) {
          dst[e] = stage[r * kPitch + cidx];
          r += qstep, cidx += rstep;
          if (cidx >= W) cidx -= W, ++r;
        }
        __syncthreads();
      }
    }
    // every thread passed the layer loop's barriers after reading its input row: the tile can take the output rows
#pragma unroll
    for (int k = 0; k < kTcNMax; ++k)
      if (k < out_dim) stage[tid * kPitch + k] = v[k];
    if (a.relu_mask) asm volatile("cp.async.wait_group 0;" ::: "memory");  // this tile's mask rows (and the next tile's input)
    __syncthreads();
    {
      float* dst = y + tile * 128 * out_dim;
      const float* mask = a.relu_mask ? mask_tile : nullptr;
      const int n_el = rows_here * out_dim, qstep = 128 / out_dim, rstep = 128 - qstep * out_dim;
      int r = tid / out_dim, cidx = tid - r * out_dim;
      // 16 elements per thread at a time; the mask values (dgrad: the pre-activation rows, fetched into shared memory by
      // cp.async at the top of the iteration) are read as a batch before the stores that depend on them
      for (int e0 = tid; e0 < n_el; e0 += 128 * 16) {
        float mk[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) {
          const int e = e0 + 128 * u;
          mk[u] = (mask && e < n_el) ? mask[e] : 1.0f;
        }
#pragma unroll
        for (int u = 0; u < 16; ++u) {
          const int e = e0 + 128 * u;
          if (e < n_el) {
            dst[e] = mk[u] > 0.f ? stage[r * kPitch + cidx] : 0.f;
            r += qstep, cidx += rstep;
            if (cidx >= out_dim) cidx -= out_dim, ++r;
          }
        }
      }
    }
    __syncthreads();  // this buffer is the prefetch target of the next iteration
  }
}

// Cameras._generate_rays_from_coords, pinhole + rolling shutter (cameras/cameras.py:633-667,793-798,898-969)
struct PinholeArgs {
  float c2w[12];
  float fx, fy, cx, cy;
  int height, width, row0, row_step, n_rows, col0, col_step, n_cols;
  float time, vel[3], rs_time, ttc;
  int has_vel;
};
__device__ __forceinline__ void cam_dir(const PinholeArgs& a, float u, float v, float out[3], float* norm) {
  // direction (u, -v, -1) rotated by c2w: sum over columns of dir_j * R[i][j]  (cameras.py:902-904)
  float dx = u, dy = -v, dz = -1.0f;
  float r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r[i] = fadd(fadd(fmul(dx, a.c2w[4 * i + 0]), fmul(dy, a.c2w[4 * i + 1])), fmul(dz, a.c2w[4 * i + 2]));
  float n = fsqrt(fadd(fadd(fmul(r[0], r[0]), fmul(r[1], r[1])), fmul(r[2], r[2])));
  n = fmaxf(n, 8.8817841970012523e-16f);  // camera_utils.py:30 (_EPS = 4 * float64 eps, cast to fp32)
  out[0] = fdiv(r[0], n); out[1] = fdiv(r[1], n); out[2] = fdiv(r[2], n);
  *norm = n;
}
__global__ void raygen_pinhole_kernel(PinholeArgs a, float* __restrict__ origins, float* __restrict__ dirs,
                                      float* __restrict__ area, float* __restrict__ times) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)a.n_rows * a.n_cols) return;
  int r = (int)(i / a.n_cols), c = (int)(i % a.n_cols);
  float y = (float)(a.row0 + r * a.row_step) + 0.5f, x = (float)(a.col0 + c * a.col_step) + 0.5f;
  float u0 = fdiv(fsub(x, a.cx), a.fx), v0 = fdiv(fsub(y, a.cy), a.fy);
  float u1 = fdiv(fadd(fsub(x, a.cx), 1.0f), a.fx), v1 = fdiv(fadd(fsub(y, a.cy), 1.0f), a.fy);
  float d0[3], dxo[3], dyo[3], n0, n1;
  cam_dir(a, u0, v0, d0, &n0);
  cam_dir(a, u1, v0, dxo, &n1);
  cam_dir(a, u0, v1, dyo, &n1);
  float ex[3], ey[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ex[k] = fsub(d0[k], dxo[k]);
    ey[k] = fsub(d0[k], dyo[k]);
  }
  float dx = fsqrt(fadd(fadd(fmul(ex[0], ex[0]), fmul(ex[1], ex[1])), fmul(ex[2], ex[2])));
  float dy = fsqrt(fadd(fadd(fmul(ey[0], ey[0]), fmul(ey[1], ey[1])), fmul(ey[2], ey[2])));
  float o[3] = {a.c2w[3], a.c2w[7], a.c2w[11]};
  float t = a.time;
  if (a.has_vel) {
    float toff = fadd(fmul(fsub(fdiv(y, (float)a.height), 0.5f), a.rs_time), a.ttc);
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = fadd(o[k], fmul(a.vel[k], toff));
    t = fadd(t, toff);
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    origins[3 * i + k] = o[k];
    dirs[3 * i + k] = d0[k];
  }
  area[i] = fmul(dx, dy);
  times[i] = t;
}

// Lidars._generate_rays_from_points (cameras/lidars.py:399-460)
struct LidarArgs {
  float l2w[12];
  float scan_time, vel[3], h_div, v_div;
  int has_vel, stride;
};
__global__ void raygen_lidar_kernel(LidarArgs a, const float* __restrict__ pts, int64_t n, float* __restrict__ origins,
                                    float* __restrict__ dirs, float* __restrict__ area, float* __restrict__ times,
                                    float* __restrict__ distance) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = pts + i * a.stride;
  float px = p[0], py = p[1], pz = p[2], dt = a.stride >= 5 ? p[4] : 0.f;
  float pw[3], o[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    pw[k] = fadd(fadd(fadd(fmul(a.l2w[4 * k], px), fmul(a.l2w[4 * k + 1], py)), fmul(a.l2w[4 * k + 2], pz)), a.l2w[4 * k + 3]);
    o[k] = a.l2w[4 * k + 3];
    if (a.has_vel) o[k] = fadd(o[k], fmul(dt, a.vel[k]));
  }
  float d[3] = {fsub(pw[0], o[0]), fsub(pw[1], o[1]), fsub(pw[2], o[2])};
  float nrm = fsqrt(fadd(fadd(fmul(d[0], d[0]), fmul(d[1], d[1])), fmul(d[2], d[2])));
  nrm = fmaxf(nrm, 8.8817841970012523e-16f);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    origins[3 * i + k] = o[k];
    dirs[3 * i + k] = fdiv(d[k], nrm);
  }
  area[i] = fmul(a.h_div, a.v_div);
  times[i] = fadd(a.scan_time, dt);
  if (distance) distance[i] = nrm;
}


// Beam x azimuth lidar ray grid (viewer/render_state_machine.py:395-407: d = (cos v cos h, cos v sin h, sin v) over
// linspace elevations x arange azimuths) with a rolling-shutter sweep: per-ray time offset linear in azimuth over one
// revolution and origin shifted by velocity * dt (cameras/lidars.py:421-423, 625-639).  BASELINE config 4's input shape.
struct LidarGridArgs {
  float l2w[12];
  float elev0, elev1;   // radians
  double az_step;       // radians (torch.arange evaluates start + i*step in double, then casts)
  int beams, n_az;
  float scan_time, rev_time, vel[3], h_div, v_div;
  int has_vel;
};
__global__ void raygen_lidar_grid_kernel(LidarGridArgs a, float* __restrict__ origins, float* __restrict__ dirs,
                                         float* __restrict__ area, float* __restrict__ times) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)a.beams * a.n_az) return;
  const int b = (int)(i / a.n_az), k = (int)(i % a.n_az);
  // torch.linspace(e0, e1, beams): start + step*i for the first half, end - step*(n-1-i) for the second
  const float step = a.beams > 1 ? fdiv(fsub(a.elev1, a.elev0), (float)(a.beams - 1)) : 0.f;
  const float v = b < a.beams / 2 ? fadd(a.elev0, fmul(step, (float)b)) : fsub(a.elev1, fmul(step, (float)(a.beams - 1 - b)));
  const float h = (float)((double)k * a.az_step);
  const float cv = cosf(v), sv = sinf(v), ch = cosf(h), sh = sinf(h);
  const float dl[3] = {fmul(cv, ch), fmul(cv, sh), sv};
  float d[3], o[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    d[r] = fadd(fadd(fmul(a.l2w[4 * r], dl[0]), fmul(a.l2w[4 * r + 1], dl[1])), fmul(a.l2w[4 * r + 2], dl[2]));
    o[r] = a.l2w[4 * r + 3];
  }
  const float dt = fmul(fsub(fdiv(h, 6.283185307179586f), 0.5f), a.rev_time);
  if (a.has_vel) {
#pragma unroll
    for (int r = 0; r < 3; ++r) o[r] = fadd(o[r], fmul(dt, a.vel[r]));
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    origins[3 * i + r] = o[r];
    dirs[3 * i + r] = d[r];
  }
  area[i] = fmul(a.h_div, a.v_div);
  times[i] = fadd(a.scan_time, dt);
}

// ===================================================================================================== C ABI
// Rebase every per-ray pointer of a parameter block to ray `start` (slicing a bundle into several launches).
template <class T>
static inline void adv(T*& p, int64_t n) {
  if (p) p += n;
}
static void offset_rays(RenderParams& Q, int64_t start, int fdim) {
  if (start == 0) return;
  adv(Q.rays.origins, 3 * start); adv(Q.rays.directions, 3 * start); adv(Q.rays.pixel_area, start);
  adv(Q.rays.times, start); adv(Q.rays.nears, start); adv(Q.rays.fars, start);
  adv(Q.rays.sensor_idx, start); adv(Q.rays.is_lidar, start);
  adv(Q.out.features, (int64_t)fdim * start); adv(Q.out.depth, start); adv(Q.out.accumulation, start);
  adv(Q.out.prop_depth_0, start); adv(Q.out.prop_depth_1, start);
  b200nerf_trace& t = Q.trace;
  adv(t.prop_weights_0, kS0 * start); adv(t.prop_weights_1, kS1 * start);
  adv(t.bins_s_1, (kS1 + 1) * start); adv(t.bins_e_1, (kS1 + 1) * start);
  adv(t.bins_s_2, (kS2 + 1) * start); adv(t.bins_e_2, (kS2 + 1) * start);
  adv(t.inds_1, (kS1 + 1) * start); adv(t.inds_2, (kS2 + 1) * start);
  adv(t.sdf, kS2 * start); adv(t.alpha, kS2 * start); adv(t.field_feature, (int64_t)kS2 * kNff * start);
  adv(t.weights, kS2 * start);
  adv(t.actor_id_0, kS0 * start); adv(t.actor_id_1, kS1 * start); adv(t.actor_id_main, kS2 * start);
  Q.peers.row_offset += start;
}


extern "C" {

const char* b200nerf_last_error(void) { return g_err.c_str(); }
int b200nerf_version(void) { return B200NERF_VERSION; }

int b200nerf_create(int device_ordinal, b200nerf_ctx** out) {
  REQUIRE(out != nullptr, "out is NULL");
  int n = 0;
  CUDA_TRY(cudaGetDeviceCount(&n));
  REQUIRE(device_ordinal >= 0 && device_ordinal < n, "device ordinal out of range");
  DeviceGuard g(device_ordinal);
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device_ordinal));
  if (prop.major != 9 || prop.minor != 0)  // sm_90a code (wgmma, TMA) loads on compute capability 9.0 only
    return fail(B200NERF_ERR_UNSUPPORTED, "libb200nerf is built for sm_90a only (found sm_" +
                                              std::to_string(prop.major) + std::to_string(prop.minor) + ")");
  b200nerf_ctx* c = new (std::nothrow) b200nerf_ctx();
  REQUIRE(c != nullptr, "out of host memory");
  c->device = device_ordinal;
  c->sm_count = prop.multiProcessorCount;
  CUDA_TRY(cudaFuncSetAttribute(nff_render_kernel<kRenderWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)((kMainMlpFloats * 4 + 15) / 16 * 16 + kRenderWarps * sizeof(WarpShared))));
  CUDA_TRY(cudaFuncSetAttribute(nff_render_tc_kernel<kRenderWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)(tc_smem_bytes(kRenderWarps * 32) + kRenderWarps * sizeof(WarpSharedTc))));
  CUDA_TRY(cudaMalloc((void**)&c->d_status, sizeof(int)));
  CUDA_TRY(cudaMemset(c->d_status, 0, sizeof(int)));
  CUDA_TRY(cudaFuncSetAttribute(nff_render_lane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)lane_tc_smem_bytes()));
  c->lane_ctas = c->sm_count * (kLaneCtasPerSm > NFF_SAMPLE_CTAS ? kLaneCtasPerSm : NFF_SAMPLE_CTAS);
  CUDA_TRY(cudaMalloc((void**)&c->d_lane_scratch, sizeof(float) * lane_scratch_floats_per_cta() * c->lane_ctas));
  CUDA_TRY(cudaFuncSetAttribute(nff_shade_lane_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)lane_tc_smem_bytes()));
  CUDA_TRY(cudaFuncSetAttribute(nff_shade_lane_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)lane_tc_smem_bytes()));
  // (almost) all L1: the smallest carve-out that holds the 516 B edge table of each resident CTA
  for (int i = 0; i < 4; ++i) {
    CUDA_TRY(cudaFuncSetAttribute(sample_lane_kernel<0>(i & 1, i & 2), cudaFuncAttributePreferredSharedMemoryCarveout, 0));
    CUDA_TRY(cudaFuncSetAttribute(sample_lane_kernel<1>(i & 1, i & 2), cudaFuncAttributePreferredSharedMemoryCarveout, 0));
  }
  CUDA_TRY(cudaMalloc((void**)&c->d_minmax, 2 * sizeof(unsigned)));
  c->handoff_rays = (int64_t)1 << 21;
  CUDA_TRY(cudaMalloc((void**)&c->d_handoff, sizeof(float) * (kS2 + 1) * c->handoff_rays));
  CUDA_TRY(cudaMalloc((void**)&c->d_grad_actor_ptrs, sizeof(float*) * kModMaxActors));
  *out = c;
  return 0;
}

int b200nerf_destroy(b200nerf_ctx* c) {
  if (!c) return 0;
  DeviceGuard g(c->device);
  for (int i = 0; i < 3; ++i) {
    cudaFree((void*)c->d_actor_tables[i]);
    cudaFree(c->d_decoder[i]);
  }
  cudaFree(c->d_main_mlp);
  cudaFree(c->d_main_mlp_nn);
  cudaFree(c->d_lane_scratch);
  cudaFree(c->d_grad_actor_ptrs);
  cudaFree(c->d_handoff);
  cudaFree(c->d_minmax);
  cudaFree(c->d_lidar_mlp);
  cudaFree(c->d_act_times);
  cudaFree(c->d_act_kf);
  cudaFree(c->d_act_bounds);
  cudaFree(c->d_act_radii);
  cudaFree(c->d_act_present);
  cudaFree(c->d_u1);
  cudaFree(c->d_u2);
  cudaFree(c->d_status);
  for (int i = 0; i < 8; ++i) {
    cudaFree(c->d_dec_wimg[i]);
    cudaFree(c->d_dec_wf32[i]);
  }
  cudaFree(c->d_dec_bias);
  cudaFree(c->d_dec_small);
  delete c;
  return 0;
}

int b200nerf_set_field_grids(b200nerf_ctx* c, int field, const b200nerf_grid_desc* sd, const float* stable,
                             const b200nerf_grid_desc* ad, const float* const* atabs_host, int n_actors,
                             float static_scale, float actor_scale) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field selector out of range");
  REQUIRE(stable != nullptr, "static table is NULL");
  DeviceGuard g(c->device);
  FieldGrids fg{};
  if (int e = make_grid(sd, stable, &fg.stat)) return e;
  const int wantL = field == B200NERF_FIELD_MAIN ? 8 : 6, wantF = field == B200NERF_FIELD_MAIN ? 4 : 1;
  if (fg.stat.L != wantL || fg.stat.F != wantF)
    return fail(B200NERF_ERR_UNSUPPORTED,
                "fused kernel is specialised for NeuRAD's grid shapes (main: 8 levels x 4 features, proposal: 6 x 1)");
  if (!fused_table_fits(sd->log2_hashmap_size, wantF))
    return fail(B200NERF_ERR_UNSUPPORTED, "hash table too large for the fused kernels' 32-bit byte offsets");
  if (n_actors > 0) {
    REQUIRE(ad && atabs_host, "actor grid descriptor / tables missing");
    if (int e = make_grid(ad, nullptr, &fg.act)) return e;
    if (fg.act.L != 4 || fg.act.F != wantF)
      return fail(B200NERF_ERR_UNSUPPORTED, "actor grids must have 4 levels and the static grid's feature width");
    if (!fused_table_fits(ad->log2_hashmap_size, wantF))
      return fail(B200NERF_ERR_UNSUPPORTED, "actor hash table too large for the fused kernels' 32-bit byte offsets");
    cudaFree((void*)c->d_actor_tables[field]);
    c->d_actor_tables[field] = nullptr;
    CUDA_TRY(cudaMalloc((void**)&c->d_actor_tables[field], sizeof(float*) * n_actors));
    CUDA_TRY(cudaMemcpy((void*)c->d_actor_tables[field], atabs_host, sizeof(float*) * n_actors, cudaMemcpyHostToDevice));
    fg.actor_tables = c->d_actor_tables[field];
  }
  fg.static_scale = static_scale;
  fg.actor_scale = actor_scale;
  fg.decoder = c->d_decoder[field];
  c->fields[field] = fg;
  c->have_field[field] = true;
  c->field_layout[field] = 0;
  if (field == B200NERF_FIELD_MAIN) c->layout = 0;
  return 0;
}

namespace {
int make_tcnn_grid(const b200nerf_tcnn_grid_desc* d, const float* params, int want_dims, Grid* g) {
  REQUIRE(d != nullptr && params != nullptr, "tcnn grid descriptor / parameters are NULL");
  REQUIRE(d->num_levels >= 1 && d->num_levels <= kMaxLevels, "num_levels must be in [1,16]");
  REQUIRE(d->n_input_dims == want_dims, "tcnn grid has the wrong number of input dimensions (static: 3, actors: 4)");
  *g = Grid{};
  g->table = params;
  g->L = d->num_levels;
  g->F = d->features_per_level;
  g->n_dims = d->n_input_dims;
  for (int l = 0; l < d->num_levels; ++l) {
    g->res[l] = d->scalings[l];
    g->pos_scale[l] = d->scale[l];
    g->lvl_res[l] = d->resolution[l];
    g->lvl_off[l] = d->offset[l];
    REQUIRE(d->size[l] >= 1, "empty tcnn grid level");
    if (d->dense[l]) {
      g->dense_bits |= 1u << l;
      g->lvl_mask[l] = d->size[l];
    } else {
      REQUIRE((d->size[l] & (d->size[l] - 1)) == 0, "a hashed tcnn level must hold a power-of-two number of entries");
      g->lvl_mask[l] = d->size[l] - 1;
    }
  }
  return 0;
}
}  // namespace

int b200nerf_set_field_grids_tcnn(b200nerf_ctx* c, int field, const b200nerf_tcnn_grid_desc* sd, const float* sparams,
                                  const b200nerf_tcnn_grid_desc* ad, const float* aparams, int n_actors, float static_scale,
                                  float actor_scale) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field selector out of range");
  DeviceGuard g(c->device);
  FieldGrids fg{};
  if (int e = make_tcnn_grid(sd, sparams, 3, &fg.stat)) return e;
  const int wantL = field == B200NERF_FIELD_MAIN ? 8 : 6, wantF = field == B200NERF_FIELD_MAIN ? 4 : 1;
  if (fg.stat.L != wantL || fg.stat.F != wantF)
    return fail(B200NERF_ERR_UNSUPPORTED,
                "fused kernel is specialised for NeuRAD's grid shapes (main: 8 levels x 4 features, proposal: 6 x 1)");
  if (!tcnn_entries_fit(sd)) return fail(B200NERF_ERR_UNSUPPORTED, "tcnn grid has more entries than 32-bit indices address");
  if (n_actors > 0) {
    if (int e = make_tcnn_grid(ad, aparams, 4, &fg.act)) return e;
    if (fg.act.L != 4 || fg.act.F != wantF)
      return fail(B200NERF_ERR_UNSUPPORTED, "the 4-D actor grid must have 4 levels and the static grid's feature width");
    if (!tcnn_entries_fit(ad))
      return fail(B200NERF_ERR_UNSUPPORTED, "tcnn actor grid has more entries than 32-bit indices address");
  }
  fg.n_actors_f = (float)(n_actors > 0 ? n_actors : 1);
  fg.static_scale = static_scale;
  fg.actor_scale = actor_scale;
  fg.decoder = c->d_decoder[field];
  c->fields[field] = fg;
  c->have_field[field] = true;
  c->field_layout[field] = 1;
  if (field == B200NERF_FIELD_MAIN) c->layout = 1;
  return 0;
}

int b200nerf_set_proposal_decoder(b200nerf_ctx* c, int field, const float* weight, int in_dim) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field == B200NERF_FIELD_PROP0 || field == B200NERF_FIELD_PROP1, "decoder belongs to a proposal field");
  REQUIRE(weight && in_dim == 6, "density_decoder must be Linear(6, 1)");
  DeviceGuard g(c->device);
  if (!c->d_decoder[field]) CUDA_TRY(cudaMalloc((void**)&c->d_decoder[field], sizeof(float) * 8));
  CUDA_TRY(cudaMemcpyAsync(c->d_decoder[field], weight, sizeof(float) * in_dim, cudaMemcpyDeviceToDevice, c->param_stream));
  c->fields[field].decoder = c->d_decoder[field];
  return 0;
}

static int pack(cudaStream_t st, const float* w, const float* b, int out_f, int in_f, int outp, float* dw, float* db) {
  int n = in_f * outp > outp ? in_f * outp : outp;
  pack_linear_kernel<<<(n + 255) / 256, 256, 0, st>>>(w, b, out_f, in_f, outp, dw, db);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B200NERF_ERR_CUDA, std::string("pack_linear: ") + cudaGetErrorString(e));
  return 0;
}

int b200nerf_set_main_mlps(b200nerf_ctx* c, const float* gw0, const float* gb0, const float* gw1, const float* gb1,
                           const float* fw0, const float* fb0, const float* fw1, const float* fb1, const float* fw2,
                           const float* fb2, float beta) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(gw0 && gb0 && gw1 && gb1 && fw0 && fb0 && fw1 && fb1 && fw2 && fb2, "NULL MLP tensor");
  DeviceGuard g(c->device);
  if (!c->d_main_mlp) CUDA_TRY(cudaMalloc((void**)&c->d_main_mlp, sizeof(float) * kMainMlpFloats));
  float* m = c->d_main_mlp;
  if (int e = pack(c->param_stream, gw0, gb0, kHidden, kGeoIn, kHidden, m + kOffGeoW0, m + kOffGeoB0)) return e;
  if (int e = pack(c->param_stream, gw1, gb1, kNff + 1, kHidden, kGeoOutP, m + kOffGeoW1, m + kOffGeoB1)) return e;
  if (int e = pack(c->param_stream, fw0, fb0, kHidden, kNff + kSh, kHidden, m + kOffFeatW0, m + kOffFeatB0)) return e;
  if (int e = pack(c->param_stream, fw1, fb1, kHidden, kHidden, kHidden, m + kOffFeatW1, m + kOffFeatB1)) return e;
  if (int e = pack(c->param_stream, fw2, fb2, kNff, kHidden, kNff, m + kOffFeatW2, m + kOffFeatB2)) return e;
  if (!c->d_main_mlp_nn) CUDA_TRY(cudaMalloc((void**)&c->d_main_mlp_nn, sizeof(float) * kNnMlpFloats));
  {
    float* n = c->d_main_mlp_nn;
    const float* src[10] = {gw0, gb0, gw1, gb1, fw0, fb0, fw1, fb1, fw2, fb2};
    const int off[10] = {kNnGeoW0, kNnGeoB0, kNnGeoW1, kNnGeoB1, kNnFeatW0, kNnFeatB0, kNnFeatW1, kNnFeatB1, kNnFeatW2, kNnFeatB2};
    const int cnt[10] = {kHidden * kGeoIn, kHidden, (kNff + 1) * kHidden, kNff + 1, kHidden * (kNff + kSh), kHidden,
                         kHidden * kHidden, kHidden, kNff * kHidden, kNff};
    for (int i = 0; i < 10; ++i)
      CUDA_TRY(cudaMemcpyAsync(n + off[i], src[i], sizeof(float) * cnt[i], cudaMemcpyDeviceToDevice, c->param_stream));
  }
  // no synchronisation: the packing runs on the parameter stream (the caller's), render launches on it follow in order
  c->beta = beta;
  c->have_main_mlp = true;
  return 0;
}

int b200nerf_set_lidar_decoder(b200nerf_ctx* c, const float* w0, const float* b0, const float* w1, const float* b1,
                               const float* w2, const float* b2) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(w0 && b0 && w1 && b1 && w2 && b2, "NULL MLP tensor");
  DeviceGuard g(c->device);
  if (!c->d_lidar_mlp) CUDA_TRY(cudaMalloc((void**)&c->d_lidar_mlp, sizeof(float) * kLidarMlpFloats));
  float* m = c->d_lidar_mlp;
  if (int e = pack(c->param_stream, w0, b0, kHidden, kNff + kApp, kHidden, m + kOffLidW0, m + kOffLidB0)) return e;
  if (int e = pack(c->param_stream, w1, b1, kHidden, kHidden, kHidden, m + kOffLidW1, m + kOffLidB1)) return e;
  if (int e = pack(c->param_stream, w2, b2, 2, kHidden, kLidOutP, m + kOffLidW2, m + kOffLidB2)) return e;
  c->have_lidar = true;
  return 0;
}

int b200nerf_set_appearance(b200nerf_ctx* c, const float* emb, int num_embeds, int dim, int eps, float duration) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(dim >= 0 && dim <= kApp, "appearance_dim must be <= 16");
  REQUIRE(dim == 0 || (emb && num_embeds > 0 && eps > 0 && duration > 0.f), "bad appearance embedding");
  c->app.emb = emb;
  c->app.num_embeds = num_embeds;
  c->app.dim = dim;
  c->app.eps = eps;
  c->app.duration = duration;
  c->have_app = true;
  return 0;
}

int b200nerf_set_appearance_per_sensor(b200nerf_ctx* c, const float* emb, int num_embeds, int dim) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(dim >= 0 && dim <= kApp, "appearance_dim must be <= 16");
  REQUIRE(dim == 0 || (emb && num_embeds > 0), "bad appearance embedding");
  c->app.emb = emb;
  c->app.num_embeds = num_embeds;
  c->app.dim = dim;
  c->app.eps = 0;          // the kernels' per-sensor branch
  c->app.duration = 1.f;   // keeps the unused temporal index arithmetic finite
  c->have_app = true;
  return 0;
}

int b200nerf_set_actors(b200nerf_ctx* c, int n_actors, int n_times, const float* timestamps, const float* rot6,
                        const float* pos, const uint8_t* present, const float* sizes, const float* padding_host) {
  REQUIRE(c, "ctx is NULL");
  DeviceGuard g(c->device);
  if (n_actors <= 0 || n_actors != c->act_alloc_actors || n_times != c->act_alloc_times) {  // (re)allocate only on a shape change
    cudaFree(c->d_act_times); cudaFree(c->d_act_kf); cudaFree(c->d_act_bounds); cudaFree(c->d_act_radii);
    cudaFree(c->d_act_present);
    c->d_act_times = c->d_act_kf = c->d_act_bounds = c->d_act_radii = nullptr;
    c->d_act_present = nullptr;
    c->act_alloc_actors = c->act_alloc_times = 0;
  }
  c->actors = Actors{};
  if (n_actors <= 0) return 0;
  REQUIRE(n_times >= 1 && timestamps && rot6 && pos && present && sizes && padding_host, "NULL actor tensor");
  size_t ta = (size_t)n_times * n_actors;
  if (c->act_alloc_actors == 0) {
    CUDA_TRY(cudaMalloc((void**)&c->d_act_times, sizeof(float) * n_times));
    CUDA_TRY(cudaMalloc((void**)&c->d_act_kf, sizeof(float) * 9 * ta));
    CUDA_TRY(cudaMalloc((void**)&c->d_act_bounds, sizeof(float) * 3 * n_actors));
    CUDA_TRY(cudaMalloc((void**)&c->d_act_radii, sizeof(float) * n_actors));
    CUDA_TRY(cudaMalloc((void**)&c->d_act_present, ta));
    c->act_alloc_actors = n_actors;
    c->act_alloc_times = n_times;
  }
  CUDA_TRY(cudaMemcpyAsync(c->d_act_times, timestamps, sizeof(float) * n_times, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(c->d_act_present, present, ta, cudaMemcpyDeviceToDevice, c->param_stream));
  int n = (int)(ta > (size_t)n_actors ? ta : n_actors);
  actors_prep_kernel<<<(n + 127) / 128, 128, 0, c->param_stream>>>(n_times, n_actors, rot6, pos, sizes, padding_host[0], padding_host[1],
                                                                  padding_host[2], c->d_act_kf, c->d_act_bounds, c->d_act_radii);
  CUDA_TRY(cudaGetLastError());
  c->actors.n_actors = n_actors;
  c->actors.n_times = n_times;
  c->actors.times = c->d_act_times;
  c->actors.keyframes = c->d_act_kf;
  c->actors.present = c->d_act_present;
  c->actors.bounds = c->d_act_bounds;
  c->actors.radii = c->d_act_radii;
  return 0;
}

int b200nerf_set_sampling(b200nerf_ctx* c, int n_prop0, int n_prop1, int n_nerf, float lam, float scaling, float sky,
                          float hist_pad, const float* u1_host, const float* u2_host, const int* field_of_round,
                          float camera_area_scale) {
  REQUIRE(c, "ctx is NULL");
  if (n_prop0 != kS0 || n_prop1 != kS1 || n_nerf != kS2)
    return fail(B200NERF_ERR_UNSUPPORTED, "fused kernel is specialised for NeuRAD's 128/64/32 samples per ray");
  REQUIRE(u1_host && u2_host && field_of_round, "NULL sampling table");
  REQUIRE(lam != 0.f && lam != 1.f, "power_lambda 0 / 1 (log / identity spacing) is not supported");
  for (int i = 0; i < 2; ++i)
    REQUIRE(field_of_round[i] == B200NERF_FIELD_PROP0 || field_of_round[i] == B200NERF_FIELD_PROP1,
            "density_field_of_round entries must name a proposal field");
  DeviceGuard g(c->device);
  if (!c->d_u1) CUDA_TRY(cudaMalloc((void**)&c->d_u1, sizeof(float) * (kS1 + 1)));
  if (!c->d_u2) CUDA_TRY(cudaMalloc((void**)&c->d_u2, sizeof(float) * (kS2 + 1)));
  CUDA_TRY(cudaMemcpy(c->d_u1, u1_host, sizeof(float) * (kS1 + 1), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(c->d_u2, u2_host, sizeof(float) * (kS2 + 1), cudaMemcpyHostToDevice));
  Sampling s{};
  s.lam = lam;
  s.scaling = scaling;
  s.sky_distance = sky;
  s.hist_pad = hist_pad;
  s.cam_area_scale = camera_area_scale;
  double lam1 = lam - 1.0 < 0 ? -(lam - 1.0) : (lam - 1.0);
  s.lam_1 = (float)lam1;
  s.ratio = (float)(lam1 / (double)lam);
  s.u1 = c->d_u1;
  s.u2 = c->d_u2;
  s.field_of_round[0] = field_of_round[0];
  s.field_of_round[1] = field_of_round[1];
  c->samp = s;
  c->n_prop0 = n_prop0; c->n_prop1 = n_prop1; c->n_nerf = n_nerf;
  c->have_samp = true;
  return 0;
}

int b200nerf_nff_render_fwd(b200nerf_ctx* c, const b200nerf_rays* rays, int64_t n_rays, const b200nerf_outputs* out,
                            const b200nerf_trace* trace, void* stream) {
  REQUIRE(c && rays && out, "NULL argument");
  REQUIRE(n_rays >= 0, "negative ray count");
  REQUIRE(rays->image_width >= 0, "negative image_width");
  if (!(c->have_field[0] && c->have_main_mlp && c->have_samp && c->have_app))
    return fail(B200NERF_ERR_STATE, "set_field_grids(MAIN), set_main_mlps, set_sampling and set_appearance are required");
  for (int i = 0; i < 2; ++i) {
    int f = c->samp.field_of_round[i];
    if (!c->have_field[f] || !c->fields[f].decoder)
      return fail(B200NERF_ERR_STATE, "proposal field used by a sampling round has no grids / decoder set");
    if (c->actors.n_actors > 0 && !c->fields[f].actor_tables && !c->fields[f].act.table)
      return fail(B200NERF_ERR_STATE, "actors are set but a proposal field has no actor grids");
  }
  if (c->actors.n_actors > 0 && !c->fields[0].actor_tables && !c->fields[0].act.table)
    return fail(B200NERF_ERR_STATE, "actors are set but the main field has no actor grids");
  if (n_rays == 0) return 0;
  REQUIRE(rays->origins && rays->directions && rays->pixel_area && rays->times, "NULL ray tensor");
  REQUIRE(out->features && out->depth && out->accumulation && out->prop_depth_0 && out->prop_depth_1, "NULL output tensor");
  if ((out->intensity || out->ray_drop_logit) && !c->have_lidar)
    return fail(B200NERF_ERR_STATE, "intensity requested but set_lidar_decoder was not called");
  DeviceGuard g(c->device);
  RenderParams P{};
  for (int i = 0; i < 3; ++i) P.fields[i] = c->fields[i];
  P.main_mlp = c->d_main_mlp;
  P.main_mlp_nn = c->d_main_mlp_nn;
  P.status = c->d_status;
  P.lidar_mlp = c->d_lidar_mlp;
  P.beta = c->beta;
  P.nff_dim = kNff;
  P.actors = c->actors;
  P.samp = c->samp;
  P.app = c->app;
  P.rays = *rays;
  P.out = *out;
  if (trace) P.trace = *trace;
  P.peers = c->peers;
  if (c->peers.n_peers > 0 && c->mlp_mode < 2)
    return fail(B200NERF_ERR_UNSUPPORTED, "peer outputs are implemented by the ray-per-lane kernels (modes 2, 3) only");
  if (c->peers.n_peers > 0 && ((kNff + c->app.dim) & 3) != 0)
    return fail(B200NERF_ERR_UNSUPPORTED, "peer outputs need a feature width that is a multiple of 4");
  P.n_rays = n_rays;
  P.layout = c->layout;
  if (c->layout == 1) {
    if (c->mlp_mode != 3)
      return fail(B200NERF_ERR_UNSUPPORTED, "the tiny-cuda-nn layout is implemented by the two-stage renderer (mode 3) only");
    for (int i = 0; i < 2; ++i)
      if (c->field_layout[c->samp.field_of_round[i]] != 1)
        return fail(B200NERF_ERR_STATE, "main field has the tiny-cuda-nn layout but a proposal field used for sampling does not");
  } else {
    for (int i = 0; i < 2; ++i)
      if (c->field_layout[c->samp.field_of_round[i]] != 0)
        return fail(B200NERF_ERR_STATE, "a proposal field has the tiny-cuda-nn layout but the main field does not");
  }
  constexpr int WARPS = kRenderWarps;
  int64_t blocks_needed = (n_rays + WARPS - 1) / WARPS;
  int64_t max_blocks = (int64_t)c->sm_count * (16 / WARPS);  // persistent: resident CTAs only, grid-stride over rays
  int blocks = (int)(blocks_needed < max_blocks ? blocks_needed : max_blocks);
  cudaStream_t st = (cudaStream_t)stream;
  if (c->mlp_mode == 3) {
    // sampling kernel -> [33][rays] spacing edges -> shading kernel; bundles larger than the hand-over buffer are
    // rendered in slices (whole 16-row tile bands when an image_width hint is given)
    const size_t smem = lane_tc_smem_bytes();
    const b200nerf_trace& tr = P.trace;  // any proposal-stage trace pointer selects the traced sampling kernel
    const bool traced = tr.prop_weights_0 || tr.prop_weights_1 || tr.actor_id_0 || tr.actor_id_1 || tr.bins_s_1 ||
                        tr.bins_s_2 || tr.bins_e_1 || tr.bins_e_2 || tr.inds_1 || tr.inds_2;
    int64_t slice = c->handoff_rays;
    if (rays->image_width > 0) {
      const int64_t band = (int64_t)rays->image_width * (kLaneThreads / 32);
      REQUIRE(band <= slice, "image_width too large for the two-stage renderer");
      slice = slice / band * band;
    }
    const int fdim = kNff + c->app.dim;
    for (int64_t start = 0; start < n_rays; start += slice) {
      const int64_t cnt = n_rays - start < slice ? n_rays - start : slice;
      RenderParams Q = P;
      Q.n_rays = cnt;
      offset_rays(Q, start, fdim);
      int64_t need = (cnt + kLaneThreads - 1) / kLaneThreads;
      if (rays->image_width > 0) {
        const int64_t W = rays->image_width, H = (cnt + W - 1) / W;
        need = ((W + 31) / 32) * ((H + kLaneThreads / 32 - 1) / (kLaneThreads / 32));
      }
      // persistent grids: every resident CTA gets a balanced share of the patches (see lane_patches); bundles with fewer
      // patches than warps still spread over all SMs
      const int64_t max_a = (int64_t)c->sm_count * NFF_SAMPLE_CTAS, max_b = (int64_t)c->sm_count * kLaneCtasPerSm;
      const int64_t patches = rays->image_width > 0 ? need * (kLaneThreads / 32) : (cnt + 31) / 32, groups = (patches + 3) / 4;
      const int64_t grid_a = patches < max_a ? patches : max_a, grid_b = groups < max_b ? groups : max_b;
      const bool actors = c->actors.n_actors > 0;
      if (c->layout == 1) {
        sample_lane_kernel<1>(actors, traced)<<<(int)grid_a, kLaneThreads, 0, st>>>(Q, c->d_lane_scratch, c->d_handoff);
        nff_shade_lane_kernel<1><<<(int)grid_b, kLaneThreads, smem, st>>>(Q, c->d_lane_scratch, c->d_handoff);
      } else {
        sample_lane_kernel<0>(actors, traced)<<<(int)grid_a, kLaneThreads, 0, st>>>(Q, c->d_lane_scratch, c->d_handoff);
        nff_shade_lane_kernel<0><<<(int)grid_b, kLaneThreads, smem, st>>>(Q, c->d_lane_scratch, c->d_handoff);
      }
    }
  } else if (c->mlp_mode == 2) {
    const size_t smem = lane_tc_smem_bytes();
    int64_t need = (n_rays + kLaneThreads - 1) / kLaneThreads;
    if (rays->image_width > 0) {
      const int64_t W = rays->image_width, H = (n_rays + W - 1) / W;
      need = ((W + 31) / 32) * ((H + kLaneThreads / 32 - 1) / (kLaneThreads / 32));
    }
    int lane_blocks = (int)(need < c->lane_ctas ? need : c->lane_ctas);
    nff_render_lane_kernel<<<lane_blocks, kLaneThreads, smem, st>>>(P, c->d_lane_scratch);
  } else if (c->mlp_mode == 1) {
    const size_t smem = tc_smem_bytes(WARPS * 32) + WARPS * sizeof(WarpSharedTc);
    nff_render_tc_kernel<WARPS><<<blocks, WARPS * 32, smem, st>>>(P);
  } else {
    const size_t smem = (kMainMlpFloats * 4 + 15) / 16 * 16 + WARPS * sizeof(WarpShared);
    nff_render_kernel<WARPS><<<blocks, WARPS * 32, smem, st>>>(P);
  }
  CUDA_TRY(cudaGetLastError());
  if (out->intensity || out->ray_drop_logit) {
    int fdim = kNff + c->app.dim;
    lidar_decode_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, st>>>(c->d_lidar_mlp, out->features, fdim, n_rays,
                                                                          out->intensity, out->ray_drop_logit);
    CUDA_TRY(cudaGetLastError());
  }
  return 0;
}


static int mlp_fwd_impl(b200nerf_ctx* c, const float* x, int64_t n_rows, int in_dim, int n_layers,
                        const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                        float* y, float* const* hidden_pre_host, void* stream, const float* relu_mask = nullptr);
int b200nerf_mlp_fwd(b200nerf_ctx* c, const float* x, int64_t n_rows, int in_dim, int n_layers,
                     const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                     float* y, void* stream) {
  return mlp_fwd_impl(c, x, n_rows, in_dim, n_layers, weights_host, biases_host, out_dims_host, y, nullptr, stream);
}
int b200nerf_mlp_fwd_train(b200nerf_ctx* c, const float* x, int64_t n_rows, int in_dim, int n_layers,
                           const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                           float* y, float* const* hidden_pre_host, void* stream) {
  return mlp_fwd_impl(c, x, n_rows, in_dim, n_layers, weights_host, biases_host, out_dims_host, y, hidden_pre_host, stream);
}
int b200nerf_mlp_dgrad(b200nerf_ctx* c, const float* dy, int64_t n_rows, int dy_dim, const float* weight_t, int dx_dim,
                       const float* relu_z, float* dx, void* stream) {
  const float* w[1] = {weight_t};
  const int od[1] = {dx_dim};
  return mlp_fwd_impl(c, dy, n_rows, dy_dim, 1, w, nullptr, od, dx, nullptr, stream, relu_z);
}
static int mlp_fwd_impl(b200nerf_ctx* c, const float* x, int64_t n_rows, int in_dim, int n_layers,
                        const float* const* weights_host, const float* const* biases_host, const int* out_dims_host,
                        float* y, float* const* hidden_pre_host, void* stream, const float* relu_mask) {
  REQUIRE(c && weights_host && out_dims_host, "NULL argument");
  REQUIRE(n_layers >= 1 && n_layers <= 3, "MLP depth must be 1..3 Linear layers");
  constexpr int kWide = 64;
  REQUIRE(in_dim >= 1 && in_dim <= kWide, "in_dim must be <= 64");
  if (n_rows == 0) return 0;
  REQUIRE(x && y, "NULL argument");
  DeviceGuard g(c->device);
  MlpArgs a{};
  a.n_layers = n_layers;
  a.in_dim = in_dim;
  int k = in_dim, off = 0, wmax = in_dim;
  for (int l = 0; l < n_layers; ++l) {
    int n = out_dims_host[l];
    REQUIRE(n >= 1 && n <= kWide, "layer widths must be <= 64");
    wmax = n > wmax ? n : wmax;
    REQUIRE(weights_host[l] != nullptr, "NULL weight");
    a.w[l] = weights_host[l];
    a.b[l] = biases_host ? biases_host[l] : nullptr;
    a.k_real[l] = k;
    a.n_real[l] = n;
    a.k_pad[l] = (k + 7) / 8 * 8;
    a.n_pad[l] = (n + 15) / 16 * 16;
    a.smem_off[l] = off;
    off += 2 * a.n_pad[l] * a.k_pad[l];
    k = n;
  }
  a.bias_off = off;
  for (int l = 0; l + 1 < n_layers && l < 2; ++l) a.hidden_pre[l] = hidden_pre_host ? hidden_pre_host[l] : nullptr;
  a.relu_mask = relu_mask;
  // NeuRAD's own MLPs (<= 48 wide) use the 48-column tile; wider ones (config 1's 32 -> 64 -> 4) the 64-column tile
  const int tile_w = wmax <= 48 ? 48 : kWide;
  a.mma_off = off + 3 * tile_w;
  a.stage_off = a.mma_off + 128 * tc::stage_pitch(tile_w);
  size_t smem = sizeof(float) * (a.stage_off + 2 * 128 * (tile_w + 1) + (relu_mask ? 128 * out_dims_host[n_layers - 1] : 0));
  // function attributes are per device: one flag per context (several contexts, one per GPU, may share the process)
  REQUIRE(smem <= (size_t)kSmemMaxOptIn, "MLP too wide: its weights and row tiles exceed a CTA's shared memory");
  bool& attr_set = c->mlp_attr_set;
  if (!attr_set) {
    CUDA_TRY(cudaFuncSetAttribute(mlp_tc_kernel<48, 48>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMaxOptIn));
    CUDA_TRY(cudaFuncSetAttribute(mlp_tc_kernel<64, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMaxOptIn));
    attr_set = true;
  }
  int64_t tiles = (n_rows + 127) / 128;
  int grid = (int)(tiles < (int64_t)c->sm_count * 2 ? tiles : (int64_t)c->sm_count * 2);
  if (tile_w == 48)
    mlp_tc_kernel<48, 48><<<grid, 128, smem, (cudaStream_t)stream>>>(a, x, y, n_rows, c->d_status);
  else
    mlp_tc_kernel<64, 64><<<grid, 128, smem, (cudaStream_t)stream>>>(a, x, y, n_rows, c->d_status);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int make_spacing(int kind, float power_lambda, float power_scaling, SpacingArgs* a) {
  REQUIRE(kind >= B200NERF_SPACING_UNIFORM && kind <= B200NERF_SPACING_LOG, "unknown spacing kind");
  a->kind = kind;
  if (kind == B200NERF_SPACING_POWER) {
    REQUIRE(power_lambda != 0.f && power_lambda != 1.f, "power_lambda 0 / 1 (log / identity spacing) is not supported");
    REQUIRE(power_scaling > 0.f, "power_scaling must be positive");
    a->power.lam = power_lambda;
    a->power.scaling = power_scaling;
    double lam1 = power_lambda - 1.0 < 0 ? -(power_lambda - 1.0) : (power_lambda - 1.0);
    a->power.lam_1 = (float)lam1;
    a->power.ratio = (float)(lam1 / (double)power_lambda);
  }
  return 0;
}

int b200nerf_spaced_sample(b200nerf_ctx* c, int kind, float power_lambda, float power_scaling, const float* nears,
                           const float* fars, int64_t n_rays, int n_samples, float* bins_s, float* bins_e, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (n_rays == 0) return 0;
  REQUIRE(fars && bins_e, "NULL argument");
  SpacingArgs a{};
  if (int rc = make_spacing(kind, power_lambda, power_scaling, &a)) return rc;
  DeviceGuard g(c->device);
  const int64_t n = n_rays * (n_samples + 1);
  spaced_sample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, nears, fars, n_rays, n_samples, bins_s, bins_e);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------- module-level seams (SURVEY 8b)
int b200nerf_isotropic_gaussian_fwd(b200nerf_ctx* c, const float* origins, const float* directions,
                                    const float* pixel_area, const float* bins_e, int64_t n_rays, int n_samples,
                                    float* mean, float* std, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (n_rays == 0) return 0;
  REQUIRE(origins && directions && pixel_area && bins_e && mean && std, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t n = n_rays * n_samples;
  isotropic_gaussian_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(origins, directions, pixel_area, bins_e,
                                                                                           n_rays, n_samples, mean, std);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_neurad_encoding_fwd(b200nerf_ctx* c, int field, const float* mean, const float* std, const float* times,
                                 const float* flip, const float* directions, int directions_per_ray, int64_t n_rays, int n_samples,
                                 float* features, float* density, float* directions_out, int32_t* actor_id,
                                 void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field must be B200NERF_FIELD_MAIN / PROP0 / PROP1");
  if (!c->have_field[field]) return fail(B200NERF_ERR_STATE, "b200nerf_set_field_grids was not called for this field");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  const FieldGrids& fg = c->fields[field];
  REQUIRE(fg.stat.L * fg.stat.F <= kModMaxDim, "encoding rows wider than 64 features are not supported");
  REQUIRE(c->actors.n_actors == 0 || fg.act.L * fg.act.F <= fg.stat.L * fg.stat.F,
          "actor features must fit the static feature width (they are zero padded to it)");
  if (c->actors.n_actors > kModMaxActors) return fail(B200NERF_ERR_UNSUPPORTED, "more than 64 actors");
  if (density && !fg.decoder) return fail(B200NERF_ERR_STATE, "b200nerf_set_proposal_decoder was not called for this field");
  REQUIRE(!directions_out || directions, "directions_out needs directions");
  if (n_rays == 0) return 0;
  REQUIRE(mean && std, "NULL argument");
  REQUIRE(c->actors.n_actors == 0 || times, "times are required when the scene has actors");
  DeviceGuard g(c->device);
  EncodingArgs a{mean, std, times, directions, flip, features, density, directions_out, actor_id, n_rays, n_samples,
                 directions_per_ray ? 1 : 0};
  cudaError_t opt_in = cudaSuccess;
  if (!launch_neurad_encoding_fwd(fg, c->actors, a, (cudaStream_t)stream, opt_in))
    return fail(B200NERF_ERR_UNSUPPORTED, "encoding forward: 4 or 1 features per level, at most 8 levels");
  CUDA_TRY(opt_in);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_field_mid_fwd(b200nerf_ctx* c, const float* geo_out, const float* directions, int64_t n_points,
                           int geo_feat_dim, float* mlp_feature_in, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_points >= 0 && geo_feat_dim >= 1, "bad shape");
  if (n_points == 0) return 0;
  REQUIRE(geo_out && directions && mlp_feature_in, "NULL argument");
  DeviceGuard g(c->device);
  field_mid_kernel<<<(unsigned)((n_points + 127) / 128), 128, 0, (cudaStream_t)stream>>>(geo_out, directions, n_points, geo_feat_dim,
                                                                                          mlp_feature_in);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_field_tail_fwd(b200nerf_ctx* c, const float* geo_out, const float* mlp_feature_out, int64_t n_points,
                            int geo_feat_dim, float beta, float* feature, float* sdf, float* alpha, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_points >= 0 && geo_feat_dim >= 1, "bad shape");
  if (n_points == 0) return 0;
  REQUIRE(geo_out && mlp_feature_out && feature, "NULL argument");
  DeviceGuard g(c->device);
  field_tail_kernel<<<(unsigned)((n_points + 127) / 128), 128, 0, (cudaStream_t)stream>>>(geo_out, mlp_feature_out, n_points,
                                                                                           geo_feat_dim, beta, feature, sdf, alpha);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_spaced_sample_stratified(b200nerf_ctx* c, int kind, float power_lambda, float power_scaling, const float* nears,
                                      const float* fars, const float* t_rand, int rand_cols, int64_t n_rays, int n_samples,
                                      float* bins_s, float* bins_e, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  REQUIRE(rand_cols == 1 || rand_cols == n_samples + 1, "t_rand must be [N,1] (single_jitter) or [N,S+1]");
  SpacingArgs a{};
  if (int rc = make_spacing(kind, power_lambda, power_scaling, &a)) return rc;
  if (n_rays == 0) return 0;
  REQUIRE(fars && t_rand && bins_s && bins_e, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t n = n_rays * (n_samples + 1);
  spaced_sample_jitter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, nears, fars, t_rand, rand_cols, n_rays,
                                                                                             n_samples, bins_s, bins_e);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_spacing_to_euclidean(b200nerf_ctx* c, int kind, float power_lambda, float power_scaling, const float* nears,
                                  const float* fars, const float* bins_s, int64_t n_rays, int n_edges, float* bins_e,
                                  void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_edges >= 1, "bad bin grid");
  SpacingArgs a{};
  if (int rc = make_spacing(kind, power_lambda, power_scaling, &a)) return rc;
  if (n_rays == 0) return 0;
  REQUIRE(fars && bins_s && bins_e, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t n = n_rays * n_edges;
  spacing_to_euclidean_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, nears, fars, bins_s, n_rays, n_edges, bins_e);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// --------------------------------------------------------------------------- backward operators (SURVEY 8f, f2)
int b200nerf_neurad_encoding_bwd(b200nerf_ctx* c, int field, const float* mean, const float* std, const float* times,
                                 const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                 const float* density, const float* ddensity, float* grad_static_table,
                                 float* const* grad_actor_tables_host, float* grad_decoder, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field must be B200NERF_FIELD_MAIN / PROP0 / PROP1");
  if (!c->have_field[field]) return fail(B200NERF_ERR_STATE, "b200nerf_set_field_grids was not called for this field");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  // An empty batch's input tensors may have NULL data pointers, so a missing pointer only counts when there are rays;
  // every other check holds for empty batches too.
  const bool empty = n_rays == 0;
  REQUIRE(!(dfeatures && ddensity), "pass either dfeatures or (density, ddensity)");
  REQUIRE(empty || dfeatures || ddensity, "pass either dfeatures or (density, ddensity)");
  REQUIRE(empty || !ddensity || density, "density mode needs the forward density");
  const FieldGrids& fg = c->fields[field];
  if (ddensity && !fg.decoder) return fail(B200NERF_ERR_STATE, "b200nerf_set_proposal_decoder was not called for this field");
  REQUIRE(!grad_decoder || ddensity || empty, "grad_decoder belongs to the density mode");
  REQUIRE(!grad_decoder || !dfeatures, "grad_decoder belongs to the density mode");
  if (c->actors.n_actors > kModMaxActors) return fail(B200NERF_ERR_UNSUPPORTED, "more than 64 actors");
  if (empty) return 0;
  REQUIRE(mean && std, "NULL argument");
  REQUIRE(c->actors.n_actors == 0 || times, "times are required when the scene has actors");
  DeviceGuard g(c->device);
  float* const* d_ptrs = nullptr;
  if (grad_actor_tables_host && c->actors.n_actors > 0) {
    CUDA_TRY(cudaMemcpyAsync(c->d_grad_actor_ptrs, grad_actor_tables_host, sizeof(float*) * c->actors.n_actors,
                             cudaMemcpyHostToDevice, (cudaStream_t)stream));
    d_ptrs = c->d_grad_actor_ptrs;
  }
  EncodingBwdArgs a{mean, std, times, flip, dfeatures, density, ddensity, grad_static_table, d_ptrs, grad_decoder, n_rays,
                    n_samples};
  cudaError_t opt_in = cudaSuccess;
  if (!launch_neurad_encoding_bwd(fg, c->actors, a, (cudaStream_t)stream, opt_in))
    return fail(B200NERF_ERR_UNSUPPORTED, "encoding backward: features mode needs 4 features / level, density mode 1 (<= 8 levels)");
  CUDA_TRY(opt_in);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_neurad_encoding_pose_bwd(b200nerf_ctx* c, int field, const float* mean, const float* std, const float* times,
                                      const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                      const float* rotations_6d, const float* positions, float* grad_rotations_6d,
                                      float* grad_positions, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field must be B200NERF_FIELD_MAIN / PROP0 / PROP1");
  if (!c->have_field[field]) return fail(B200NERF_ERR_STATE, "b200nerf_set_field_grids was not called for this field");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (c->actors.n_actors > kModMaxActors) return fail(B200NERF_ERR_UNSUPPORTED, "more than 64 actors");
  if (n_rays == 0 || c->actors.n_actors == 0) return 0;
  REQUIRE(mean && std && times && dfeatures && rotations_6d && positions && grad_rotations_6d && grad_positions, "NULL argument");
  DeviceGuard g(c->device);
  PoseBwdArgs a{mean, std, times, flip, dfeatures, rotations_6d, positions, grad_rotations_6d, grad_positions, n_rays, n_samples};
  const unsigned grid = (unsigned)((n_rays + kModWarps - 1) / kModWarps);
  neurad_encoding_pose_bwd_kernel<<<grid, kModWarps * 32, 0, (cudaStream_t)stream>>>(c->fields[field], c->actors, a);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_neurad_encoding_mean_bwd(b200nerf_ctx* c, int field, const float* mean, const float* std, const float* times,
                                      const float* flip, int64_t n_rays, int n_samples, const float* dfeatures,
                                      const float* density, const float* ddensity, float* dmean, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(field >= 0 && field < 3, "field must be B200NERF_FIELD_MAIN / PROP0 / PROP1");
  if (!c->have_field[field]) return fail(B200NERF_ERR_STATE, "b200nerf_set_field_grids was not called for this field");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  // as in b200nerf_neurad_encoding_bwd: an empty batch's tensors may be NULL, every other check holds for it too
  const bool empty = n_rays == 0;
  REQUIRE(!(dfeatures && ddensity), "pass either dfeatures or (density, ddensity)");
  REQUIRE(empty || dfeatures || ddensity, "pass either dfeatures or (density, ddensity)");
  REQUIRE(empty || !ddensity || density, "density mode needs the forward density");
  const FieldGrids& fg = c->fields[field];
  if (ddensity && !fg.decoder) return fail(B200NERF_ERR_STATE, "b200nerf_set_proposal_decoder was not called for this field");
  if (c->actors.n_actors > kModMaxActors) return fail(B200NERF_ERR_UNSUPPORTED, "more than 64 actors");
  if (empty) return 0;
  REQUIRE(mean && std && dmean, "NULL argument");
  REQUIRE(c->actors.n_actors == 0 || times, "times are required when the scene has actors");
  DeviceGuard g(c->device);
  // require_actor_grad: the main field's grid only (fields/neurad_field.py:50,177)
  MeanBwdArgs a{mean, std, times, flip, dfeatures, density, ddensity, dmean, n_rays, n_samples, field == B200NERF_FIELD_MAIN ? 1 : 0};
  if (!launch_neurad_encoding_mean_bwd(fg, c->actors, a, (cudaStream_t)stream))
    return fail(B200NERF_ERR_UNSUPPORTED, "encoding mean backward: features mode needs 4 features / level, density mode 1 (<= 8 levels)");
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_isotropic_gaussian_bwd(b200nerf_ctx* c, const float* bins_e, int64_t n_rays, int n_samples, const float* dmean,
                                    float* dorigins, float* ddirections, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (n_rays == 0) return 0;
  REQUIRE(bins_e && dmean && dorigins && ddirections, "NULL argument");
  DeviceGuard g(c->device);
  const unsigned grid = (unsigned)((n_rays + kModWarps - 1) / kModWarps);
  isotropic_gaussian_bwd_kernel<<<grid, kModWarps * 32, 0, (cudaStream_t)stream>>>(bins_e, dmean, n_rays, n_samples, dorigins, ddirections);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_hashgrid_bwd(b200nerf_ctx* c, const b200nerf_grid_desc* desc, const float* x, const float* dout, int64_t n_points,
                          float* grad_table, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_points >= 0, "bad shape");
  Grid g{};
  if (int e = make_grid(desc, nullptr, &g)) return e;
  REQUIRE(g.L * g.F <= kModMaxDim, "encoding rows wider than 64 features are not supported");
  if (n_points == 0) return 0;
  REQUIRE(x && dout && grad_table, "NULL argument");
  DeviceGuard gd(c->device);
  hashgrid_bwd_kernel<<<(unsigned)((n_points + 127) / 128), 128, 0, (cudaStream_t)stream>>>(g, x, dout, n_points, grad_table);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_alpha_to_weights_bwd(b200nerf_ctx* c, const float* alphas, const float* dweights, int64_t n_rays, int s,
                                  float* dalphas, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && s >= 1, "bad shape");
  if (n_rays == 0) return 0;
  REQUIRE(alphas && dweights && dalphas, "NULL argument");
  DeviceGuard g(c->device);
  weights_bwd_kernel<true><<<(unsigned)((n_rays + 127) / 128), 128, 0, (cudaStream_t)stream>>>(alphas, nullptr, dweights, n_rays, s, dalphas);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_density_to_weights_bwd(b200nerf_ctx* c, const float* deltas, const float* densities, const float* dweights,
                                    int64_t n_rays, int s, float* ddensities, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && s >= 1, "bad shape");
  if (n_rays == 0) return 0;
  REQUIRE(deltas && densities && dweights && ddensities, "NULL argument");
  DeviceGuard g(c->device);
  weights_bwd_kernel<false><<<(unsigned)((n_rays + 127) / 128), 128, 0, (cudaStream_t)stream>>>(deltas, densities, dweights, n_rays, s,
                                                                                                 ddensities);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_composite_bwd(b200nerf_ctx* c, const float* weights, const float* values, int n_channels, const float* starts,
                           const float* ends, const float* dvalues_out, const float* daccumulation, const float* ddepth,
                           int64_t n_rays, int n_samples, float* dweights, float* dvalues, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1 && n_channels >= 0, "bad shape");
  if (n_rays == 0) return 0;
  REQUIRE(dweights || dvalues, "nothing to compute");
  REQUIRE(!dvalues_out || (weights && values && n_channels > 0), "dvalues_out needs weights and values");
  REQUIRE(!dvalues || dvalues_out, "dvalues needs dvalues_out");
  REQUIRE(!ddepth || (starts && ends), "ddepth needs starts and ends");
  DeviceGuard g(c->device);
  const int64_t n = n_rays * n_samples;
  composite_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(weights, values, n_channels, starts, ends, dvalues_out,
                                                                                      daccumulation, ddepth, n_rays, n_samples, dweights, dvalues);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_field_heads_bwd(b200nerf_ctx* c, const float* geo_out, const float* dfeature, const float* dsdf,
                             const float* dalpha, const float* dmlp_feature_in, int64_t n_points, int geo_feat_dim,
                             float beta, float* dgeo_out, float* dbeta, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_points >= 0 && geo_feat_dim >= 1, "bad shape");
  if (n_points == 0) return 0;
  REQUIRE(geo_out && dgeo_out, "NULL argument");
  DeviceGuard g(c->device);
  field_heads_bwd_kernel<<<(unsigned)((n_points + 127) / 128), 128, 0, (cudaStream_t)stream>>>(geo_out, dfeature, dsdf, dalpha, dmlp_feature_in,
                                                                                                n_points, geo_feat_dim, beta, dgeo_out, dbeta);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_relu_bwd(b200nerf_ctx* c, const float* z, float* dz, int64_t n, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n >= 0, "bad shape");
  if (n == 0) return 0;
  REQUIRE(z && dz, "NULL argument");
  DeviceGuard g(c->device);
  relu_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(z, dz, n);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_linear_wgrad(b200nerf_ctx* c, const float* x, const float* dy, int64_t n_rows, int in_dim, int out_dim,
                          int relu_x, float* dweight, float* dbias, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rows >= 0, "bad shape");
  REQUIRE(in_dim >= 1 && in_dim <= 64 && out_dim >= 1 && out_dim <= 64, "layer widths must be <= 64");
  if (n_rows == 0) return 0;
  REQUIRE(x && dy && dweight, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t tiles = (n_rows + kWgradRows - 1) / kWgradRows;
  const int grid = (int)(tiles < (int64_t)c->sm_count * 4 ? tiles : (int64_t)c->sm_count * 4);
  linear_wgrad_kernel<<<grid, kWgradThreads, 0, (cudaStream_t)stream>>>(x, dy, n_rows, in_dim, out_dim, relu_x, dweight, dbias);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_distortion_loss(b200nerf_ctx* c, const float* sdist, const float* weights, int64_t n_rays, int n_samples,
                             float* loss_per_ray, float* dweights, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0, "bad shape");
  REQUIRE(n_samples >= 1 && n_samples <= kLossMaxS, "the loss operators take at most 64 samples per ray");
  if (n_rays == 0) return 0;
  REQUIRE(sdist && weights && loss_per_ray, "NULL argument");
  DeviceGuard g(c->device);
  distortion_loss_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, (cudaStream_t)stream>>>(sdist, weights, n_rays, n_samples, loss_per_ray,
                                                                                             dweights);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_zipnerf_interlevel_loss(b200nerf_ctx* c, const float* sdist, const float* weights, int n_samples,
                                     const float* prop_sdist, const float* prop_weights, int n_prop_samples, float pulse_width,
                                     int64_t n_rays, float* loss_per_ray, float* dprop_weights, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_prop_samples >= 1, "bad shape");
  REQUIRE(n_samples >= 1 && n_samples <= kLossMaxS, "the loss operators take at most 64 samples of the final level per ray");
  REQUIRE(pulse_width > 0.f, "pulse_width must be positive");
  if (n_rays == 0) return 0;
  REQUIRE(sdist && weights && prop_sdist && prop_weights && loss_per_ray, "NULL argument");
  DeviceGuard g(c->device);
  zipnerf_interlevel_kernel<<<(unsigned)((n_rays + 63) / 64), 64, 0, (cudaStream_t)stream>>>(sdist, weights, n_samples, prop_sdist, prop_weights,
                                                                                             n_prop_samples, pulse_width, n_rays, loss_per_ray,
                                                                                             dprop_weights);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_linear_wgrad_tc(b200nerf_ctx* c, const float* x, const float* dy, int64_t n_rows, int in_dim, int out_dim,
                             int relu_x, float* dweight, float* dbias, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rows >= 0, "bad shape");
  REQUIRE(in_dim >= 1 && in_dim <= 64 && out_dim >= 1 && out_dim <= 64, "layer widths must be <= 64");
  if (n_rows == 0) return 0;
  REQUIRE(x && dy && dweight, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t chunks = (n_rows + kWgTcRows - 1) / kWgTcRows;
  const int grid = (int)(chunks < (int64_t)c->sm_count ? chunks : (int64_t)c->sm_count);
  CUDA_TRY(cudaFuncSetAttribute(linear_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgTcSmemBytes));
  linear_wgrad_tc_kernel<<<grid, 128, kWgTcSmemBytes, (cudaStream_t)stream>>>(x, dy, n_rows, in_dim, out_dim, relu_x, dweight, dbias);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_lidar_carving_mask(b200nerf_ctx* c, const float* bins_e, const uint8_t* is_lidar, const float* directions_norm,
                                const uint8_t* did_return, float carving_epsilon, float non_return_distance, int64_t n_rays,
                                int n_samples, uint8_t* mask, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (n_rays == 0) return 0;
  REQUIRE(bins_e && is_lidar && directions_norm && mask, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t n = n_rays * n_samples;
  lidar_carving_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(bins_e, is_lidar, directions_norm, did_return,
                                                                                           carving_epsilon, non_return_distance, n_rays, n_samples, mask);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_frustum_positions(b200nerf_ctx* c, const float* origins, const float* directions, const float* bins_e,
                               int64_t n_rays, int n_samples, const float* aabb_host, float* positions, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  if (n_rays == 0) return 0;
  REQUIRE(origins && directions && bins_e && positions, "NULL argument");
  AabbArgs a{};
  if (aabb_host) {
    a.normalize = 1;
    for (int k = 0; k < 3; ++k) {
      a.lo[k] = aabb_host[k];
      a.len[k] = aabb_host[3 + k] - aabb_host[k];  // fp32 subtraction, as aabb[1] - aabb[0] in the reference
      REQUIRE(a.len[k] > 0.f, "empty aabb");
    }
  }
  DeviceGuard g(c->device);
  const int64_t n = n_rays * n_samples;
  frustum_positions_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, origins, directions, bins_e, n_rays,
                                                                                          n_samples, positions);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_density_rgb_heads(b200nerf_ctx* c, const float* raw, int64_t n_points, int n_channels, float* density,
                               float* rgb, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_points >= 0 && n_channels >= 1, "bad shape");
  if (n_points == 0) return 0;
  REQUIRE(raw && density && rgb, "NULL argument");
  DeviceGuard g(c->device);
  const int64_t n = n_points * (n_channels + 1);
  density_rgb_heads_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(raw, n_points, n_channels, density, rgb);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_composite(b200nerf_ctx* c, const float* weights, const float* values, int n_channels, int value_nan_to_num,
                       const float* background_host, const float* starts, const float* ends, int depth_method,
                       int64_t n_rays, int n_samples, float* out_values, float* out_accumulation, float* out_depth,
                       void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sample grid");
  REQUIRE(depth_method >= B200NERF_DEPTH_NONE && depth_method <= B200NERF_DEPTH_SIMPLE, "unknown depth method");
  REQUIRE(n_channels >= 0 && n_channels <= 64, "at most 64 value channels");
  if (n_rays == 0) return 0;
  REQUIRE(weights, "NULL weights");
  REQUIRE(!(values || out_values) || (values && out_values && n_channels > 0), "values / out_values must come together");
  REQUIRE(depth_method == B200NERF_DEPTH_NONE || (starts && ends && out_depth), "depth needs starts, ends and out_depth");
  CompositeArgs a{};
  a.C = n_channels;
  a.value_nan_to_num = value_nan_to_num;
  a.has_background = background_host != nullptr;
  a.depth_method = depth_method;
  if (background_host) memcpy(a.background, background_host, sizeof(float) * n_channels);
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (depth_method == B200NERF_DEPTH_EXPECTED) {
    CUDA_TRY(cudaMemsetAsync(c->d_minmax, 0xff, sizeof(unsigned), st));
    CUDA_TRY(cudaMemsetAsync(c->d_minmax + 1, 0x00, sizeof(unsigned), st));
  }
  composite_kernel<<<(unsigned)((n_rays + 3) / 4), 128, 0, st>>>(a, weights, values, starts, ends, n_rays, n_samples, out_values,
                                                                 out_accumulation, out_depth, c->d_minmax);
  CUDA_TRY(cudaGetLastError());
  if (depth_method == B200NERF_DEPTH_EXPECTED) {
    depth_clip_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, st>>>(out_depth, n_rays, c->d_minmax);
    CUDA_TRY(cudaGetLastError());
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------- rgb decoder (f1)
namespace {
constexpr int kDecMaxIn = 64;
inline int64_t dec_small_floats() { return dec::kC * kDecMaxIn + dec::kC + dec::kC * dec::kC * 9 + dec::kC + 3 * dec::kC + 4; }
struct DecSmall {
  float *in_w, *in_b, *up_w, *up_b, *out_w, *out_b;
};
inline DecSmall dec_small(float* base) {
  DecSmall d;
  d.in_w = base;
  d.in_b = d.in_w + dec::kC * kDecMaxIn;
  d.up_w = d.in_b + dec::kC;
  d.up_b = d.up_w + dec::kC * dec::kC * 9;
  d.out_w = d.up_b + dec::kC;
  d.out_b = d.out_w + 3 * dec::kC;
  return d;
}
inline int64_t act_bytes(int64_t pixels) { return pixels * 128; }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// ACT buffer [batch][H][W][8 chunks][8 bf16] as a 5-D tensor; one copy = one chunk plane of a (kIR x kPW)-pixel window
inline bool act_window_map(CUtensorMap* map, const void* act, int batch, int H, int W) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return false;
  const cuuint64_t dims[5] = {8, 8, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)batch};
  const cuuint64_t strides[4] = {16, 128, (cuuint64_t)W * 128, (cuuint64_t)H * W * 128};
  const cuuint32_t box[5] = {8, 1, (cuuint32_t)dec::kPW, (cuuint32_t)dec::kIR, 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(act), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
}  // namespace

int b200nerf_set_rgb_decoder(b200nerf_ctx* c, const b200nerf_rgb_decoder_params* p) {
  REQUIRE(c && p, "NULL argument");
  REQUIRE(p->hidden_dim == dec::kC, "rgb_hidden_dim must be 32");
  REQUIRE(p->upsample == dec::kUp, "rgb_upsample_factor must be 3");
  REQUIRE(p->in_dim >= 1 && p->in_dim <= kDecMaxIn, "decoder in_dim must be in [1, 64]");
  REQUIRE(p->bn_eps > 0.f, "bn_eps must be positive");
  REQUIRE(p->in_conv.weight && p->in_conv.bias && p->up_conv.weight && p->up_conv.bias && p->out_conv.weight && p->out_conv.bias,
          "NULL decoder tensor");
  DeviceGuard g(c->device);
  if (!c->d_dec_bias) {
    for (int i = 0; i < 8; ++i) {
      CUDA_TRY(cudaMalloc((void**)&c->d_dec_wimg[i], (size_t)dec::kK7 * dec::kWRowBytes));
      CUDA_TRY(cudaMalloc((void**)&c->d_dec_wf32[i], sizeof(float) * dec::kTaps * dec::kC * dec::kC));
    }
    CUDA_TRY(cudaMalloc((void**)&c->d_dec_bias, sizeof(float) * 8 * dec::kC));
    CUDA_TRY(cudaMalloc((void**)&c->d_dec_small, sizeof(float) * dec_small_floats()));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tc_kernel<dec::EPI_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tc_kernel<dec::EPI_RES_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tc_kernel<dec::EPI_RES_RELU_RGB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tma_kernel<dec::EPI_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tma_kernel<dec::EPI_RES_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
    CUDA_TRY(cudaFuncSetAttribute(dec::dec_conv7_tma_kernel<dec::EPI_RES_RELU_RGB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(dec::ConvSmem)));
  }
  for (int b = 0; b < 4; ++b)
    for (int k = 0; k < 2; ++k) {
      const b200nerf_conv_bn_params& q = p->block[b][k];
      REQUIRE(q.conv_weight && q.conv_bias && q.bn_weight && q.bn_bias && q.bn_running_mean && q.bn_running_var, "NULL BasicBlock tensor");
      const int i = 2 * b + k, n = dec::kTaps * dec::kC * dec::kC;
      dec::dec_fold_conv_kernel<<<(n + 255) / 256, 256, 0, c->param_stream>>>(q.conv_weight, q.conv_bias, q.bn_weight, q.bn_bias, q.bn_running_mean,
                                                          q.bn_running_var, p->bn_eps, c->d_dec_wimg[i], c->d_dec_wf32[i],
                                                          c->d_dec_bias + i * dec::kC);
      CUDA_TRY(cudaGetLastError());
    }
  const DecSmall d = dec_small(c->d_dec_small);
  CUDA_TRY(cudaMemcpyAsync(d.in_w, p->in_conv.weight, sizeof(float) * dec::kC * p->in_dim, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(d.in_b, p->in_conv.bias, sizeof(float) * dec::kC, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(d.up_w, p->up_conv.weight, sizeof(float) * dec::kC * dec::kC * 9, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(d.up_b, p->up_conv.bias, sizeof(float) * dec::kC, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(d.out_w, p->out_conv.weight, sizeof(float) * 3 * dec::kC, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaMemcpyAsync(d.out_b, p->out_conv.bias, sizeof(float) * 3, cudaMemcpyDeviceToDevice, c->param_stream));
  CUDA_TRY(cudaStreamSynchronize(c->param_stream));  // the caller may release its parameter tensors when this returns
  c->dec_in_dim = p->in_dim;
  c->have_rgb_decoder = true;
  return 0;
}

int64_t b200nerf_rgb_decode_workspace_bytes(int batch, int height, int width) {
  if (batch <= 0 || height <= 0 || width <= 0) return 0;
  const int64_t lo = (int64_t)batch * height * width;
  return 3 * act_bytes(lo) + 3 * act_bytes(lo * dec::kUp * dec::kUp);
}

int b200nerf_rgb_decode_fwd(b200nerf_ctx* c, const float* features, int batch, int height, int width, float* rgb,
                            void* workspace, int64_t workspace_bytes, int impl, void* stream) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(batch >= 0 && height >= 0 && width >= 0, "negative image shape");
  REQUIRE(impl >= 0 && impl <= 2, "impl: 0 = wgmma + TMA loads, 1 = CUDA-core fp32 cross-check, 2 = wgmma + LDGSTS loads");
  if (!c->have_rgb_decoder) return fail(B200NERF_ERR_STATE, "set_rgb_decoder was not called");
  if (batch == 0 || height == 0 || width == 0) return 0;
  REQUIRE(features && rgb && workspace, "NULL argument");
  REQUIRE(workspace_bytes >= b200nerf_rgb_decode_workspace_bytes(batch, height, width), "workspace too small (see b200nerf_rgb_decode_workspace_bytes)");
  REQUIRE(((uintptr_t)workspace & 15) == 0, "workspace must be 16-byte aligned");
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t lo_px = (int64_t)batch * height * width, hi_px = lo_px * dec::kUp * dec::kUp;
  unsigned char* ws = (unsigned char*)workspace;
  uint4* lo[3];
  uint4* hi[3];
  for (int i = 0; i < 3; ++i) lo[i] = (uint4*)(ws + i * act_bytes(lo_px));
  for (int i = 0; i < 3; ++i) hi[i] = (uint4*)(ws + 3 * act_bytes(lo_px) + i * act_bytes(hi_px));
  const DecSmall d = dec_small(c->d_dec_small);
  dec::dec_input_kernel<<<(unsigned)((lo_px + 127) / 128), 128, sizeof(float) * (c->dec_in_dim * dec::kC + dec::kC), st>>>(
      features, lo_px, c->dec_in_dim, d.in_w, d.in_b, lo[0]);
  CUDA_TRY(cudaGetLastError());
  auto conv = [&](int layer, int epi, const uint4* in, const uint4* res, uint4* out, float* out_rgb, int H, int W) -> int {
    dec::ConvArgs a{};
    a.in = in; a.residual = res; a.out_act = out; a.out_rgb = out_rgb;
    a.w_img = c->d_dec_wimg[layer]; a.w_f32 = c->d_dec_wf32[layer]; a.bias = c->d_dec_bias + layer * dec::kC;
    a.out_w = d.out_w; a.out_b = d.out_b;
    a.batch = batch; a.H = H; a.W = W; a.status = c->d_status;
    if (impl == 0) {
      dec::ConvArgsTma t{};
      t.a = a;
      if (!act_window_map(&t.in_map, in, batch, H, W)) return fail(B200NERF_ERR_CUDA, "cuTensorMapEncodeTiled failed for the decoder's input window");
      const int64_t tiles = (int64_t)batch * ((H + dec::kTH - 1) / dec::kTH) * ((W + dec::kStrip - 1) / dec::kStrip);
      const int grid = (int)(tiles < c->sm_count ? tiles : c->sm_count);
      const size_t smem = sizeof(dec::ConvSmem);
      if (epi == dec::EPI_RELU) dec::dec_conv7_tma_kernel<dec::EPI_RELU><<<grid, dec::kConvThreads, smem, st>>>(t);
      else if (epi == dec::EPI_RES_RELU) dec::dec_conv7_tma_kernel<dec::EPI_RES_RELU><<<grid, dec::kConvThreads, smem, st>>>(t);
      else dec::dec_conv7_tma_kernel<dec::EPI_RES_RELU_RGB><<<grid, dec::kConvThreads, smem, st>>>(t);
    } else if (impl == 2) {
      const int64_t tiles = (int64_t)batch * ((H + dec::kTH - 1) / dec::kTH) * ((W + dec::kStrip - 1) / dec::kStrip);
      const int grid = (int)(tiles < c->sm_count ? tiles : c->sm_count);
      const size_t smem = sizeof(dec::ConvSmem);
      if (epi == dec::EPI_RELU) dec::dec_conv7_tc_kernel<dec::EPI_RELU><<<grid, dec::kConvThreads, smem, st>>>(a);
      else if (epi == dec::EPI_RES_RELU) dec::dec_conv7_tc_kernel<dec::EPI_RES_RELU><<<grid, dec::kConvThreads, smem, st>>>(a);
      else dec::dec_conv7_tc_kernel<dec::EPI_RES_RELU_RGB><<<grid, dec::kConvThreads, smem, st>>>(a);
    } else {
      const unsigned grid = (unsigned)((int64_t)batch * H * ((W + 127) / 128));
      if (epi == dec::EPI_RELU) dec::dec_conv7_ref_kernel<dec::EPI_RELU><<<grid, 128, 0, st>>>(a);
      else if (epi == dec::EPI_RES_RELU) dec::dec_conv7_ref_kernel<dec::EPI_RES_RELU><<<grid, 128, 0, st>>>(a);
      else dec::dec_conv7_ref_kernel<dec::EPI_RES_RELU_RGB><<<grid, 128, 0, st>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(B200NERF_ERR_CUDA, cudaGetErrorString(e));
    return 0;
  };
  const int H = height, W = width, HO = height * dec::kUp, WO = width * dec::kUp;
  // rgb_decoder.2, .3: BasicBlocks at feature resolution
  if (int e = conv(0, dec::EPI_RELU, lo[0], nullptr, lo[1], nullptr, H, W)) return e;
  if (int e = conv(1, dec::EPI_RES_RELU, lo[1], lo[0], lo[2], nullptr, H, W)) return e;
  if (int e = conv(2, dec::EPI_RELU, lo[2], nullptr, lo[1], nullptr, H, W)) return e;
  if (int e = conv(3, dec::EPI_RES_RELU, lo[1], lo[2], lo[0], nullptr, H, W)) return e;
  // rgb_decoder.4: 3x transposed conv
  dec::dec_upsample_kernel<<<(unsigned)((lo_px + 2 * dec::kUpThreads - 1) / (2 * dec::kUpThreads)), dec::kUpThreads,
                             sizeof(float) * (9 * dec::kC * dec::kC + dec::kC), st>>>(
      lo[0], batch, H, W, d.up_w, d.up_b, hi[0]);
  CUDA_TRY(cudaGetLastError());
  // rgb_decoder.5, .6 at image resolution; .7/.8 (1x1 conv + sigmoid) in the last epilogue
  if (int e = conv(4, dec::EPI_RELU, hi[0], nullptr, hi[1], nullptr, HO, WO)) return e;
  if (int e = conv(5, dec::EPI_RES_RELU, hi[1], hi[0], hi[2], nullptr, HO, WO)) return e;
  if (int e = conv(6, dec::EPI_RELU, hi[2], nullptr, hi[1], nullptr, HO, WO)) return e;
  if (int e = conv(7, dec::EPI_RES_RELU_RGB, hi[1], hi[2], nullptr, rgb, HO, WO)) return e;
  return 0;
}

int b200nerf_set_peer_outputs(b200nerf_ctx* c, const b200nerf_peer_outputs* peers) {
  REQUIRE(c, "ctx is NULL");
  if (!peers || peers->n_peers == 0) {
    c->peers = b200nerf_peer_outputs{};
    return 0;
  }
  REQUIRE(peers->n_peers > 0 && peers->n_peers <= B200NERF_MAX_PEERS, "n_peers must be in [1, 16]");
  REQUIRE(peers->self_rank >= -1 && peers->self_rank < peers->n_peers, "self_rank out of range");
  REQUIRE(peers->row_offset >= 0, "negative row_offset");
  for (int p = 0; p < peers->n_peers; ++p) {
    if (p == peers->self_rank) continue;
    REQUIRE(peers->features[p] && peers->depth[p] && peers->accumulation[p], "NULL peer buffer");
  }
  c->peers = *peers;
  return 0;
}

int b200nerf_set_param_stream(b200nerf_ctx* c, void* stream) {
  REQUIRE(c, "ctx is NULL");
  c->param_stream = (cudaStream_t)stream;
  return 0;
}

int b200nerf_set_mlp_mode(b200nerf_ctx* c, int mode) {
  REQUIRE(c, "ctx is NULL");
  REQUIRE(mode >= 0 && mode <= 3, "render mode: 0 = warp-per-ray + CUDA-core fp32, 1 = warp-per-ray + wgmma, 2 = ray-per-lane + wgmma, 3 = ray-per-lane in two kernels (sampling, shading)");
  c->mlp_mode = mode;
  return 0;
}

int b200nerf_check_status(b200nerf_ctx* c) {
  REQUIRE(c, "ctx is NULL");
  if (!c->d_status) return 0;
  DeviceGuard g(c->device);
  int st = 0;
  CUDA_TRY(cudaMemcpy(&st, c->d_status, sizeof(int), cudaMemcpyDeviceToHost));
  if (st != 0) {
    cudaMemset(c->d_status, 0, sizeof(int));
    return fail(B200NERF_ERR_CUDA, "device-side failure flag set (tensor-core pipeline timed out, code " + std::to_string(st) + ")");
  }
  return 0;
}

int b200nerf_hashgrid_fwd(b200nerf_ctx* c, const b200nerf_grid_desc* desc, const float* table, const float* x,
                          float* out, int32_t* indices, int64_t n_points, void* stream) {
  REQUIRE(c && desc, "NULL argument");
  REQUIRE(desc->features_per_level >= 1 && desc->features_per_level <= 8, "features_per_level must be in [1,8]");
  if (n_points == 0) return 0;
  REQUIRE(table && x && out, "NULL argument");
  DeviceGuard g(c->device);
  Grid gr{};
  if (int e = make_grid(desc, table, &gr)) return e;
  if (indices && (uint64_t)gr.L * gr.T > (1ull << 31))
    return fail(B200NERF_ERR_UNSUPPORTED, "row indices of more than 2^31 table rows do not fit int32");
  int64_t n = n_points * gr.L;
  hashgrid_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(gr, x, out, indices, n_points);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_tcnn_hashgrid_fwd(b200nerf_ctx* c, const b200nerf_tcnn_grid_desc* desc, const float* params, const float* x,
                               float* out, int64_t n_points, void* stream) {
  REQUIRE(c && desc, "NULL argument");
  REQUIRE(desc->features_per_level >= 1 && desc->features_per_level <= 8, "features_per_level must be in [1,8]");
  REQUIRE(desc->n_input_dims == 3 || desc->n_input_dims == 4, "n_input_dims must be 3 or 4");
  if (n_points == 0) return 0;
  REQUIRE(params && x && out, "NULL argument");
  DeviceGuard g(c->device);
  Grid gr{};
  if (int e = make_tcnn_grid(desc, params, desc->n_input_dims, &gr)) return e;
  const unsigned blocks = (unsigned)((n_points + 127) / 128);
  if (desc->n_input_dims == 3)
    tcnn_hashgrid_fwd_kernel<3><<<blocks, 128, 0, (cudaStream_t)stream>>>(gr, x, out, n_points);
  else
    tcnn_hashgrid_fwd_kernel<4><<<blocks, 128, 0, (cudaStream_t)stream>>>(gr, x, out, n_points);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_sh4_fwd(b200nerf_ctx* c, const float* dirs, float* out, int64_t n, void* stream) {
  REQUIRE(c, "NULL argument");
  if (n == 0) return 0;
  REQUIRE(dirs && out, "NULL argument");
  DeviceGuard g(c->device);
  sh4_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dirs, out, n);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_pdf_resample(b200nerf_ctx* c, const float* weights, const float* bins, const float* u, int n_rays,
                          int s_old, int s_new, float hist_pad, float* new_bins, float* cdf, int32_t* inds,
                          void* stream) {
  REQUIRE(c && weights && bins && u && new_bins, "NULL argument");
  REQUIRE(s_old >= 1 && s_old <= 2048 && s_new >= 1, "sample counts out of range");
  if (n_rays == 0) return 0;
  DeviceGuard g(c->device);
  const int warps = 4;
  size_t smem = sizeof(float) * warps * (s_old + 1);
  pdf_resample_kernel<<<(n_rays + warps - 1) / warps, warps * 32, smem, (cudaStream_t)stream>>>(
      weights, bins, u, n_rays, s_old, s_new, hist_pad, new_bins, cdf, inds);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_pdf_resample_stratified(b200nerf_ctx* c, const float* weights, const float* bins, const float* u_base,
                                     const float* rand, int rand_cols, int n_rays, int s_old, int s_new, float hist_pad,
                                     float* new_bins, float* cdf, int32_t* inds, void* stream) {
  REQUIRE(c && weights && bins && u_base && rand && new_bins, "NULL argument");
  REQUIRE(s_old >= 1 && s_old <= 2048 && s_new >= 1, "sample counts out of range");
  REQUIRE(rand_cols == 1 || rand_cols == s_new + 1, "rand must be [N,1] (single_jitter) or [N,S_new+1]");
  if (n_rays == 0) return 0;
  DeviceGuard g(c->device);
  const int warps = 4;
  size_t smem = sizeof(float) * warps * (s_old + 1);
  pdf_resample_kernel<<<(n_rays + warps - 1) / warps, warps * 32, smem, (cudaStream_t)stream>>>(
      weights, bins, u_base, n_rays, s_old, s_new, hist_pad, new_bins, cdf, inds, rand, rand_cols);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_density_to_weights(b200nerf_ctx* c, const float* deltas, const float* densities, int n_rays, int s,
                                float* weights, void* stream) {
  REQUIRE(c && deltas && densities && weights, "NULL argument");
  if (n_rays == 0) return 0;
  DeviceGuard g(c->device);
  weights_kernel<false><<<(n_rays + 3) / 4, 128, 0, (cudaStream_t)stream>>>(deltas, densities, n_rays, s, weights);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_alpha_to_weights(b200nerf_ctx* c, const float* alphas, int n_rays, int s, float* weights, void* stream) {
  REQUIRE(c && alphas && weights, "NULL argument");
  if (n_rays == 0) return 0;
  DeviceGuard g(c->device);
  weights_kernel<true><<<(n_rays + 3) / 4, 128, 0, (cudaStream_t)stream>>>(alphas, nullptr, n_rays, s, weights);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_raygen_pinhole(b200nerf_ctx* c, const float* c2w_host, float fx, float fy, float cx, float cy, int height,
                            int width, int row0, int row_step, int n_rows, int col0, int col_step, int n_cols,
                            float time, const float* velocity_host, float rs_time, float ttc, float* origins,
                            float* directions, float* pixel_area, float* times, void* stream) {
  REQUIRE(c && c2w_host && origins && directions && pixel_area && times, "NULL argument");
  REQUIRE(n_rows >= 0 && n_cols >= 0 && row_step >= 1 && col_step >= 1, "bad pixel grid");
  if (n_rows == 0 || n_cols == 0) return 0;
  DeviceGuard g(c->device);
  PinholeArgs a{};
  memcpy(a.c2w, c2w_host, sizeof(float) * 12);
  a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy;
  a.height = height; a.width = width;
  a.row0 = row0; a.row_step = row_step; a.n_rows = n_rows;
  a.col0 = col0; a.col_step = col_step; a.n_cols = n_cols;
  a.time = time; a.rs_time = rs_time; a.ttc = ttc;
  a.has_vel = velocity_host != nullptr;
  if (velocity_host) memcpy(a.vel, velocity_host, sizeof(float) * 3);
  int64_t n = (int64_t)n_rows * n_cols;
  raygen_pinhole_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, origins, directions,
                                                                                        pixel_area, times);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int b200nerf_raygen_lidar_points(b200nerf_ctx* c, const float* l2w_host, const float* points, int point_stride,
                                 int64_t n_points, float scan_time, const float* velocity_host, float h_div,
                                 float v_div, float* origins, float* directions, float* pixel_area, float* times,
                                 float* distance, void* stream) {
  REQUIRE(c && l2w_host && points && origins && directions && pixel_area && times, "NULL argument");
  REQUIRE(point_stride >= 3, "points need at least x,y,z");
  if (n_points == 0) return 0;
  DeviceGuard g(c->device);
  LidarArgs a{};
  memcpy(a.l2w, l2w_host, sizeof(float) * 12);
  a.scan_time = scan_time; a.h_div = h_div; a.v_div = v_div; a.stride = point_stride;
  a.has_vel = velocity_host != nullptr;
  if (velocity_host) memcpy(a.vel, velocity_host, sizeof(float) * 3);
  raygen_lidar_kernel<<<(unsigned)((n_points + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      a, points, n_points, origins, directions, pixel_area, times, distance);
  CUDA_TRY(cudaGetLastError());
  return 0;
}


int b200nerf_raygen_lidar_grid(b200nerf_ctx* c, const float* l2w_host, float elev_min_rad, float elev_max_rad, int beams,
                               int n_azimuth, double azimuth_step_rad, float scan_time, float revolution_time,
                               const float* velocity_host, float h_div, float v_div, float* origins, float* directions,
                               float* pixel_area, float* times, void* stream) {
  REQUIRE(c && l2w_host && origins && directions && pixel_area && times, "NULL argument");
  REQUIRE(beams >= 1 && n_azimuth >= 1, "bad lidar grid");
  DeviceGuard g(c->device);
  LidarGridArgs a{};
  memcpy(a.l2w, l2w_host, sizeof(float) * 12);
  a.elev0 = elev_min_rad; a.elev1 = elev_max_rad; a.az_step = azimuth_step_rad;
  a.beams = beams; a.n_az = n_azimuth;
  a.scan_time = scan_time; a.rev_time = revolution_time; a.h_div = h_div; a.v_div = v_div;
  a.has_vel = velocity_host != nullptr;
  if (velocity_host) memcpy(a.vel, velocity_host, sizeof(float) * 3);
  int64_t n = (int64_t)beams * n_azimuth;
  raygen_lidar_grid_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, origins, directions, pixel_area, times);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // extern "C"
