// modules.cuh -- kernels of the module-level operators (SURVEY.md 8b seams "Field", "Sampler", "Encoding op"): the
// reference's nn.Modules exchange [N,S,...] tensors, so these kernels read and write them (the fused renderer does not).
// Device logic lives in nff_modules.h (shared with the host emulation used by the CPU tests).
#pragma once

#include "nff_modules.h"

namespace nff {

constexpr int kModWarps = 8;
// dynamic shared memory above which a launch opts in (the 48 KB default limit also counts a kernel's static shared memory)
constexpr size_t kSmemOptIn = 47 * 1024;

// Frustums.get_fast_isotropic_gaussian(num_multisamples=1) (cameras/rays.py:109-124): one thread per sample.
__global__ void isotropic_gaussian_kernel(const float* __restrict__ origins, const float* __restrict__ dirs,
                                          const float* __restrict__ area, const float* __restrict__ bins_e,
                                          int64_t n_rays, int S, float* __restrict__ mean, float* __restrict__ std) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S) return;
  int64_t ray = i / S;
  int s = (int)(i % S);
  float o[3] = {origins[3 * ray], origins[3 * ray + 1], origins[3 * ray + 2]};
  float d[3] = {dirs[3 * ray], dirs[3 * ray + 1], dirs[3 * ray + 2]};
  Gauss g = sample_gaussian(o, d, area[ray], bins_e[ray * (S + 1) + s], bins_e[ray * (S + 1) + s + 1]);
  mean[3 * i] = g.x;
  mean[3 * i + 1] = g.y;
  mean[3 * i + 2] = g.z;
  std[i] = g.std;
}

struct EncodingArgs {
  const float* mean;    // [N,S,3]
  const float* std;     // [N,S]
  const float* times;   // [N] (the reference reads times[:, 0], neurad_encoding.py:194)
  const float* dirs;    // [N,3] (dirs_per_ray) or [N,S,3] or NULL
  const float* flip;    // [N] +1 / -1 or NULL: training-mode actor flip (neurad_encoding.py:212-219)
  float* features;      // [N*S, D] or NULL
  float* density;       // [N,S] or NULL: trunc_exp(Linear(D,1,bias=False)(features)) (neurad_field.py:208-213)
  float* dirs_out;      // [N,S,3] or NULL
  int32_t* actor_id;    // [N,S] or NULL
  int64_t n_rays;
  int32_t S, dirs_per_ray;
};

// NeuRADHashEncoding.forward (neurad_encoding.py:150-187), optionally followed by the proposal field's density head.
// One warp per ray: the lanes first build the ray's actor frames (lane = actor) in shared memory, then take 32 consecutive
// samples at a time.  F = 4 (main field) / F = 1 (proposal fields), at most 8 levels: a sample's feature row stays in
// registers (neurad_encode_point_t), and the warp's 32 rows -- one contiguous block of `features` -- go out through a
// shared-memory tile with an odd pitch so that the global stores are coalesced (lane = row wrote 32 different lines per
// store instruction).  EDIT: the frames carry the actor edit (only launched while one is active).
template <int F, bool EDIT>
__global__ void __launch_bounds__(kModWarps * 32) neurad_encoding_fwd_kernel(const FieldGrids fg, const Actors A,
                                                                              const EncodingArgs a) {
  constexpr int kRow = 8 * F, kPitch = kRow + 1;
  extern __shared__ __align__(16) unsigned char fwd_smem[];
  float* stage_all = reinterpret_cast<float*>(fwd_smem);  // [kModWarps][32][kPitch]
  ActorFrame* frames_all = reinterpret_cast<ActorFrame*>(stage_all + kModWarps * 32 * kPitch);  // [kModWarps][n_actors]
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kModWarps + warp;
  if (ray >= a.n_rays) return;
  float* stage = stage_all + warp * 32 * kPitch;
  ActorFrame* frames = frames_all + warp * A.n_actors;
  if (A.n_actors > 0) {
    int left, right;
    float frac;
    keyframe_bracket(A, a.times[ray], left, right, frac);
    for (int k = ln; k < A.n_actors; k += 32) actor_frame<EDIT>(A, k, left, right, frac, frames[k]);
  }
  __syncwarp();
  const int D = fg.stat.L * fg.stat.F;
  const float flip = a.flip ? a.flip[ray] : 1.0f;
  for (int s0 = 0; s0 < a.S; s0 += 32) {
    const int s = s0 + ln;
    if (s < a.S) {
      const int64_t i = ray * a.S + s;
      Gauss g = {a.mean[3 * i], a.mean[3 * i + 1], a.mean[3 * i + 2], a.std[i]};
      float dir[3] = {0.f, 0.f, 0.f};
      if (a.dirs) {
        const float* dp = a.dirs + 3 * (a.dirs_per_ray ? ray : i);
        dir[0] = dp[0]; dir[1] = dp[1]; dir[2] = dp[2];
      }
      float feat[kRow];
      const int aid = neurad_encode_point_t<8, F>(fg, frames, A.n_actors, g, feat, a.dirs ? dir : nullptr, flip);
      if (a.features) {
#pragma unroll
        for (int k = 0; k < kRow; ++k)
          if (k < D) stage[ln * kPitch + k] = feat[k];
      }
      if (a.density) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < kRow; ++k)
          if (k < D) acc = fmaf(feat[k], __ldg(fg.decoder + k), acc);
        a.density[i] = expf(acc);
      }
      if (a.dirs_out) {
        a.dirs_out[3 * i] = dir[0];
        a.dirs_out[3 * i + 1] = dir[1];
        a.dirs_out[3 * i + 2] = dir[2];
      }
      if (a.actor_id) a.actor_id[i] = aid;
    }
    if (a.features) {
      __syncwarp();
      const int rows = a.S - s0 < 32 ? a.S - s0 : 32, n_el = rows * D, qstep = 32 / D, rstep = 32 - qstep * D;
      float* dst = a.features + (ray * a.S + s0) * D;
      int r = ln / D, c = ln - r * D;
      for (int e = ln; e < n_el; e += 32) {
        dst[e] = stage[r * kPitch + c];
        r += qstep, c += rstep;
        if (c >= D) c -= D, ++r;
      }
      __syncwarp();
    }
  }
}
// Host dispatch (false: grid shapes b200nerf_set_field_grids does not admit).  `err`: the shared-memory opt-in's error,
// if it failed (the launch is then skipped).
inline bool launch_neurad_encoding_fwd(const FieldGrids& fg, const Actors& A, const EncodingArgs& a, cudaStream_t stream, cudaError_t& err) {
  err = cudaSuccess;
  const unsigned grid = (unsigned)((a.n_rays + kModWarps - 1) / kModWarps);
  if (grid == 0) return true;
  auto launch = [&](auto kernel, int F) {
    const size_t smem = sizeof(float) * kModWarps * 32 * (8 * F + 1) + sizeof(ActorFrame) * kModWarps * (size_t)A.n_actors;
    if (smem > kSmemOptIn) err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) kernel<<<grid, kModWarps * 32, smem, stream>>>(fg, A, a);
  };
  const bool edit = A.edit_last > A.edit_first;
  if (encode_bwd_fast_ok(fg, A.n_actors, 4))
    launch(edit ? neurad_encoding_fwd_kernel<4, true> : neurad_encoding_fwd_kernel<4, false>, 4);
  else if (encode_bwd_fast_ok(fg, A.n_actors, 1))
    launch(edit ? neurad_encoding_fwd_kernel<1, true> : neurad_encoding_fwd_kernel<1, false>, 1);
  else
    return false;
  return true;
}

// NeuRADField.forward between its two MLPs (fields/neurad_field.py:139-141): geo_out [P, G+1] (sdf | geo_embedding)
// and directions [P,3] -> the feature MLP's input [P, G+16] = [geo_embedding | SH4((d + 1) / 2)]
// (get_normalized_directions base_field.py:136-142, SHEncoding encodings.py:797-805).
// One CTA = 128 consecutive rows.  Per-row values (SH, sdf, alpha) are computed thread = row; the [rows, W] blocks are
// moved by all threads element-wise, so global accesses are coalesced (thread = row over a 47-float row touches 32
// different lines per instruction and made these copies LSU-bound).
__global__ void __launch_bounds__(128) field_mid_kernel(const float* __restrict__ geo_out, const float* __restrict__ dirs, int64_t n,
                                                        int G, float* __restrict__ x2) {
  __shared__ float sh[128 * 17];
  const int64_t r0 = (int64_t)blockIdx.x * 128, row = r0 + threadIdx.x;
  const int rows = (int)(n - r0 < 128 ? n - r0 : 128);
  if (row < n) {
    float c[16];
    sh4(dirs[3 * row], dirs[3 * row + 1], dirs[3 * row + 2], c);
#pragma unroll
    for (int k = 0; k < 16; ++k) sh[threadIdx.x * 17 + k] = c[k];
  }
  __syncthreads();
  const int W = G + kSh, n_el = rows * W, qstep = 128 / W, rstep = 128 - qstep * W;
  int i = threadIdx.x / W, k = threadIdx.x - i * W;
  for (int e = threadIdx.x; e < n_el; e += 128) {
    x2[r0 * W + e] = k < G ? geo_out[(r0 + i) * (G + 1) + 1 + k] : sh[i * 17 + k - G];
    i += qstep, k += rstep;
    if (k >= W) k -= W, ++i;
  }
}

// ... and after them (neurad_field.py:141-149): feature = geo_embedding + mlp_feature(...); sdf = geo_out[0];
// alpha = SigmoidDensity(sdf) = sigmoid(-sdf * (|beta| + 1e-4)) (model_components/utils.py:29-41; `beta` here is the
// already offset value the context holds).
__global__ void __launch_bounds__(128) field_tail_kernel(const float* __restrict__ geo_out, const float* __restrict__ mlp_out,
                                                         int64_t n, int G, float beta, float* __restrict__ feature,
                                                         float* __restrict__ sdf, float* __restrict__ alpha) {
  const int64_t r0 = (int64_t)blockIdx.x * 128, row = r0 + threadIdx.x;
  const int rows = (int)(n - r0 < 128 ? n - r0 : 128);
  const int n_el = rows * G, qstep = 128 / G, rstep = 128 - qstep * G;
  int i = threadIdx.x / G, k = threadIdx.x - i * G;
  for (int e = threadIdx.x; e < n_el; e += 128) {
    feature[r0 * G + e] = geo_out[(r0 + i) * (G + 1) + 1 + k] + mlp_out[r0 * G + e];
    i += qstep, k += rstep;
    if (k >= G) k -= G, ++i;
  }
  if (row < n) {
    const float sd = geo_out[row * (G + 1)];
    if (sdf) sdf[row] = sd;
    if (alpha) alpha[row] = frcp(fadd(1.0f, expf(fmul(sd, beta))));
  }
}

// =============================================================================================== backward operators
// SURVEY 8f row f2: the gradients of the module-level operators with respect to the trained parameters.

struct EncodingBwdArgs {
  const float* mean;       // [N,S,3]
  const float* std;        // [N,S]
  const float* times;      // [N]
  const float* flip;       // [N] or NULL
  const float* dfeatures;  // [N*S, D]            (features mode)
  const float* density;    // [N,S]  forward output (density mode: NeuRADProposalField.get_density)
  const float* ddensity;   // [N,S]  dL/d density  (density mode)
  float* grad_static;      // [L*T, F] accumulated (+=), or NULL
  float* const* grad_actor_tables;  // device array [n_actors] of [La*Ta, F] accumulators (entries may be NULL), or NULL
  float* grad_decoder;     // [D] accumulated, density mode, or NULL
  int64_t n_rays;
  int32_t S;
};

// Backward of neurad_encoding_fwd_kernel: scatter-add into the hash tables (RED.ADD.F32 / .v4).  Density mode folds the
// proposal head in: g = dL/d density * density (trunc_exp' = exp), dfeat_k = g * decoder_k, d decoder_k += g * feat_k.
// MODE 1: features (F = 4, L <= 8), MODE 2: density (F = 1, L <= 8) -- the shapes b200nerf_set_field_grids admits.
// A CTA of 128 threads owns 128 / kBwdSegments rays; a ray's samples are cut into kBwdSegments (4) contiguous segments, one
// per thread (adjacent lanes = the segments of one ray), so a thread sees CONSECUTIVE samples and can run-length aggregate
// the coarse levels' reductions in registers (nff_modules.h: encoding_bwd_segment has the why and the measurements).
constexpr int kBwdThreads = 128, kBwdRays = kBwdThreads / kBwdSegments;
#ifndef NFF_BWD_MINB_F4
#define NFF_BWD_MINB_F4 2  // resident CTAs the features-mode variant is compiled for (register budget of its 8 * 4 * K sums)
#endif
#ifndef NFF_BWD_WARP_MERGE
#define NFF_BWD_WARP_MERGE 3  // coarsest levels whose pending sums are merged across the warp before they are flushed
#endif
// What is still pending when a thread finishes its segment is, on the coarsest levels, the SAME cell for most lanes of a
// warp (every ray starts at the sensors; a level-0 cell is tens of metres wide): lanes holding the same (table, cell)
// add their 8 * F sums with shuffles and one of them issues the reductions.  At most kMergeRounds distinct cells are
// merged per level; lanes left over flush their own sums afterwards (agg_flush_all).  All 32 lanes must call this.
template <int K, int F>
__device__ __forceinline__ void warp_merge_pending(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables,
                                                   ScatterAgg<K, F>& ag) {
  constexpr int kMergeRounds = 4, KW = NFF_BWD_WARP_MERGE < K ? NFF_BWD_WARP_MERGE : K;
  const int lane = threadIdx.x & 31;
  float* gt = ag.tab == -2 ? nullptr : (ag.tab < 0 ? grad_static : (grad_actor_tables ? grad_actor_tables[ag.tab] : nullptr));
  const Grid& gr = ag.tab < 0 ? fg.stat : fg.act;
#pragma unroll
  for (int l = 0; l < KW; ++l) {
    const unsigned long long id = ((unsigned long long)(unsigned)ag.tab << 32) | ag.key[l];
    unsigned todo = __ballot_sync(0xffffffffu, gt != nullptr && ag.key[l] != kAggEmpty);
    for (int round = 0; round < kMergeRounds && todo; ++round) {
      const int src = __ffs(todo) - 1;
      const unsigned long long want = __shfl_sync(0xffffffffu, id, src);
      const bool mine = ((todo >> lane) & 1u) && id == want;
      const unsigned group = __ballot_sync(0xffffffffu, mine);
      if (group != (1u << src)) {  // somebody shares the leader's cell (warp-uniform branch)
#pragma unroll
        for (int j = 0; j < 8 * F; ++j) {
          const float t = warp_sum(mine ? ag.acc[l][j] : 0.0f);
          ag.acc[l][j] = lane == src ? t : (mine ? 0.0f : ag.acc[l][j]);
        }
        if (mine && lane != src) ag.key[l] = kAggEmpty;
      }
      if (lane == src) agg_flush_level<F>(gt + (size_t)l * gr.T * F, gr.mask, ag.key[l], ag.acc[l]);
      todo &= ~group;
    }
  }
}
template <int MODE>
__global__ void __launch_bounds__(kBwdThreads, MODE == 1 ? NFF_BWD_MINB_F4 : 4) neurad_encoding_bwd_kernel(const FieldGrids fg, const Actors A, const EncodingBwdArgs a) {
  static_assert(MODE == 1 || MODE == 2, "features or density mode");
  extern __shared__ __align__(16) unsigned char bwd_smem[];
  ActorFrame* frames = reinterpret_cast<ActorFrame*>(bwd_smem);  // [kBwdRays][n_actors]
  __shared__ float dec_part[kBwdThreads / 32][8];
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const int slot = threadIdx.x / kBwdSegments, seg = threadIdx.x % kBwdSegments;
  const int64_t ray = (int64_t)blockIdx.x * kBwdRays + slot;
  if (A.n_actors > 0) {  // the CTA's rays x actors frames, built cooperatively
    for (int i = threadIdx.x; i < kBwdRays * A.n_actors; i += kBwdThreads) {
      const int sl = i / A.n_actors, k = i - sl * A.n_actors;
      const int64_t r = (int64_t)blockIdx.x * kBwdRays + sl;
      if (r < a.n_rays) {
        int left, right;
        float frac;
        keyframe_bracket(A, a.times[r], left, right, frac);
        actor_frame(A, k, left, right, frac, frames[sl * A.n_actors + k]);
      }
    }
    __syncthreads();
  }
  float dec_acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) dec_acc[k] = 0.f;
  // (no early exit: the warp-wide merge below needs all 32 lanes)
  const bool live = ray < a.n_rays;
  const float flip = live && a.flip ? a.flip[ray] : 1.0f;
  const int seg_len = (a.S + kBwdSegments - 1) / kBwdSegments;
  const int s0 = seg * seg_len, n = live ? max(min(a.S, s0 + seg_len) - s0, 0) : 0;
  const ActorFrame* fr = frames + slot * A.n_actors;
  const int64_t i0 = live ? ray * a.S + s0 : 0;
  if (MODE == 1) {
    ScatterAgg<NFF_BWD_AGG_F4, 4> ag;
    encoding_bwd_segment_pending<4, false, NFF_BWD_AGG_F4>(fg, a.grad_static, a.grad_actor_tables, fr, A.n_actors, a.mean, a.std,
                                                           a.dfeatures, nullptr, nullptr, i0, n, flip, dec_acc, ag);
    warp_merge_pending(fg, a.grad_static, a.grad_actor_tables, ag);
    agg_flush_all(fg, a.grad_static, a.grad_actor_tables, ag);
  } else {
    ScatterAgg<NFF_BWD_AGG_F1, 1> ag;
    if (a.grad_decoder)
      encoding_bwd_segment_pending<1, true, NFF_BWD_AGG_F1>(fg, a.grad_static, a.grad_actor_tables, fr, A.n_actors, a.mean, a.std, nullptr,
                                                            a.density, a.ddensity, i0, n, flip, dec_acc, ag);
    else
      encoding_bwd_segment_pending<1, false, NFF_BWD_AGG_F1>(fg, a.grad_static, a.grad_actor_tables, fr, A.n_actors, a.mean, a.std, nullptr,
                                                             a.density, a.ddensity, i0, n, flip, dec_acc, ag);
    warp_merge_pending(fg, a.grad_static, a.grad_actor_tables, ag);
    agg_flush_all(fg, a.grad_static, a.grad_actor_tables, ag);
  }
  if (MODE == 2 && a.grad_decoder) {  // warp, then block reduction; one atomic per CTA and decoder weight
    const int D = fg.stat.L * fg.stat.F;
#pragma unroll
    for (int k = 0; k < 8; ++k) {  // static indices: dec_acc stays in registers
      const float t = warp_sum(dec_acc[k]);
      if (ln == 0) dec_part[warp][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < D) {
      float t = 0.f;
      for (int w = 0; w < kBwdThreads / 32; ++w) t += dec_part[w][threadIdx.x];
      atomicAdd(a.grad_decoder + threadIdx.x, t);
    }
  }
}
// Host dispatch; false when the bound grids do not have the shapes the variants are written for (cannot happen behind
// b200nerf_set_field_grids, which admits NeuRAD's shapes only -- the caller turns it into an error instead of guessing).
// `err`: the shared-memory opt-in's error, if it failed (the launch is then skipped).
inline bool launch_neurad_encoding_bwd(const FieldGrids& fg, const Actors& A, const EncodingBwdArgs& a, cudaStream_t stream,
                                       cudaError_t& err) {
  err = cudaSuccess;
  const unsigned grid = (unsigned)((a.n_rays + kBwdRays - 1) / kBwdRays);
  // 64 B per ray and actor: 2 KB per actor, above the 48 KB default from 24 actors on, 128 KB at kModMaxActors
  const size_t smem = sizeof(ActorFrame) * kBwdRays * (size_t)A.n_actors;
  if (grid == 0) return true;
  auto launch = [&](auto kernel) {
    if (smem > kSmemOptIn) err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) kernel<<<grid, kBwdThreads, smem, stream>>>(fg, A, a);
  };
  if (!a.ddensity && encode_bwd_fast_ok(fg, A.n_actors, 4))
    launch(neurad_encoding_bwd_kernel<1>);
  else if (a.ddensity && encode_bwd_fast_ok(fg, A.n_actors, 1))
    launch(neurad_encoding_bwd_kernel<2>);
  else
    return false;
  return true;
}

// nerfacc.render_weight_from_alpha / RaySamples.get_weights backward: one thread per ray, sequential scans (S is at
// most a few hundred; the [N,S] rows are read with a stride, so this is a latency-tolerant but simple first version).
template <bool FROM_ALPHA>
__global__ void weights_bwd_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ dw,
                                   int64_t n_rays, int S, float* __restrict__ out) {
  const int64_t ray = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  if (FROM_ALPHA)
    alpha_weights_bwd_ray(a + ray * S, dw + ray * S, S, out + ray * S);
  else
    density_weights_bwd_ray(a + ray * S, b + ray * S, dw + ray * S, S, out + ray * S);
}

// Renderers backward (FeatureRenderer / AccumulationRenderer / render_depth_simple): out_c = sum_s w_s v_sc,
// acc = sum_s w_s, depth = sum_s w_s (start_s + end_s)/2  =>  dv_sc = w_s dout_c;
// dw_s = sum_c dout_c v_sc + dacc + ddepth (start_s + end_s)/2.   One thread per (ray, sample).
__global__ void composite_bwd_kernel(const float* __restrict__ weights, const float* __restrict__ values, int C,
                                     const float* __restrict__ starts, const float* __restrict__ ends,
                                     const float* __restrict__ dvalues_out, const float* __restrict__ dacc,
                                     const float* __restrict__ ddepth, int64_t n_rays, int S, float* __restrict__ dweights,
                                     float* __restrict__ dvalues) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S) return;
  const int64_t ray = i / S;
  float dw = dacc ? dacc[ray] : 0.f;
  if (ddepth) dw = fmaf(ddepth[ray], (starts[i] + ends[i]) * 0.5f, dw);
  if (dvalues_out) {
    const float w = weights[i];
    for (int c = 0; c < C; ++c) {
      const float go = dvalues_out[ray * C + c];
      if (dweights) dw = fmaf(go, values[i * C + c], dw);
      if (dvalues) dvalues[i * C + c] = w * go;
    }
  }
  if (dweights) dweights[i] = dw;
}

// NeuRADField heads backward (neurad_field.py:139-149): given dL/dfeature [P,G], dL/dsdf [P] (or NULL), dL/dalpha [P]
// (or NULL) and dL/d(mlp_feature input) [P,G+16] (or NULL; its SH part has no trained parameter behind it):
//   d geo_out[:,0]  = dsdf + dalpha * (-beta * alpha * (1 - alpha))
//   d geo_out[:,1:] = dfeature + dx2[:, :G]              d mlp_feature_out = dfeature (the caller reuses the tensor)
//   d beta         += sum dalpha * (-sdf * alpha * (1 - alpha))
__global__ void __launch_bounds__(128) field_heads_bwd_kernel(const float* __restrict__ geo_out, const float* __restrict__ dfeature,
                                                              const float* __restrict__ dsdf, const float* __restrict__ dalpha,
                                                              const float* __restrict__ dx2, int64_t n, int G, float beta,
                                                              float* __restrict__ dgeo, float* __restrict__ dbeta) {
  __shared__ float g0s[128];
  const int64_t r0 = (int64_t)blockIdx.x * 128, row = r0 + threadIdx.x;
  const int rows = (int)(n - r0 < 128 ? n - r0 : 128);
  float db = 0.f;
  if (row < n) {  // thread = row: the sdf column
    const float sd = geo_out[row * (G + 1)];
    float g0 = dsdf ? dsdf[row] : 0.f;
    if (dalpha) {
      const float al = frcp(fadd(1.0f, expf(fmul(sd, beta))));
      const float t = dalpha[row] * al * (1.0f - al);
      g0 -= beta * t;
      db = -sd * t;
    }
    g0s[threadIdx.x] = g0;
  }
  __syncthreads();
  // all threads, element-wise over the CTA's [rows, G+1] block of dgeo (coalesced)
  const int W = G + 1, n_el = rows * W, qstep = 128 / W, rstep = 128 - qstep * W;
  int i = threadIdx.x / W, k = threadIdx.x - i * W;
  for (int e = threadIdx.x; e < n_el; e += 128) {
    float v;
    if (k == 0)
      v = g0s[i];
    else
      v = (dfeature ? dfeature[(r0 + i) * G + k - 1] : 0.f) + (dx2 ? dx2[(r0 + i) * (G + kSh) + k - 1] : 0.f);
    dgeo[r0 * W + e] = v;
    i += qstep, k += rstep;
    if (k >= W) k -= W, ++i;
  }
  if (dbeta) {
    db = warp_sum(db);
    if ((threadIdx.x & 31) == 0 && db != 0.f) atomicAdd(dbeta, db);
  }
}

// dZ *= (Z > 0): ReLU backward on a hidden pre-activation.
__global__ void relu_bwd_kernel(const float* __restrict__ z, float* __restrict__ dz, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(z[i] > 0.f)) dz[i] = 0.f;
}

// Weight / bias gradient of one Linear layer of the tiny MLPs: dW[o][i] += sum_p dY[p][o] * act(X[p][i]),
// db[o] += sum_p dY[p][o]; K, N <= 64.  A CTA walks row tiles of 32, stages X / dY in shared memory and keeps its
// share of the N*K outputs in registers (first version on the CUDA cores: K = rows is the long GEMM dimension here and
// the output is at most 64 x 64; a split-K wgmma version is the next step for this operator).
constexpr int kWgradThreads = 256, kWgradRows = 32;
// global -> shared copy of one [rows][W] row block into a tile of pitch ld (>= W, pad columns zero-filled), asynchronous
// (cp.async: no registers, completion through commit / wait groups).  16-byte copies when the rows are whole quads.
__device__ __forceinline__ void wgrad_fetch(const float* __restrict__ src, int rows, int W, int ld, float* tile, int tid) {
  const uint32_t dst0 = (uint32_t)__cvta_generic_to_shared(tile);
  if (ld == W && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    for (int e = tid; e < rows * (W >> 2); e += kWgradThreads)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst0 + 16u * e), "l"(src + 4 * e) : "memory");
  } else {
    for (int e = tid; e < rows * ld; e += kWgradThreads) {
      const int r = e / ld, c = e - r * ld;
      const int ok = c < W;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst0 + 4u * e), "l"(src + (int64_t)r * W + (ok ? c : 0)),
                   "r"(ok ? 4 : 0)
                   : "memory");
    }
  }
}
__global__ void __launch_bounds__(kWgradThreads) linear_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                     int64_t n_rows, int K, int N, int relu_x,
                                                                     float* __restrict__ dW, float* __restrict__ db) {
  // two stages: the next tile's rows are in flight while this one is multiplied (a CTA that waited for its own loads
  // would stall at the first shared-memory store after them)
  __shared__ __align__(16) float xs2[2][kWgradRows * 64];
  __shared__ __align__(16) float dys2[2][kWgradRows * 64];
  const int ldx = (K + 3) & ~3, ldy = (N + 3) & ~3;  // rows padded to whole quads (pad columns zero)
  const WgradMap m = wgrad_map(K, N, kWgradThreads);
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  float bacc = 0.f;  // thread o < N accumulates db[o]
  const int64_t n_tiles = (n_rows + kWgradRows - 1) / kWgradRows;
  auto fetch = [&](int64_t t, int buf) {
    const int64_t r0 = t * kWgradRows;
    const int rows = (int)(n_rows - r0 < kWgradRows ? n_rows - r0 : kWgradRows);
    wgrad_fetch(x + r0 * K, rows, K, ldx, xs2[buf], threadIdx.x);
    wgrad_fetch(dy + r0 * N, rows, N, ldy, dys2[buf], threadIdx.x);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if ((int64_t)blockIdx.x < n_tiles) fetch(blockIdx.x, 0);
  int it = 0;
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
    const int64_t r0 = t * kWgradRows;
    const int rows = (int)(n_rows - r0 < kWgradRows ? n_rows - r0 : kWgradRows);
    if (t + gridDim.x < n_tiles) {
      fetch(t + gridDim.x, (it + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float* xs = xs2[it & 1];
    const float* dys = dys2[it & 1];
    wgrad_tile(threadIdx.x, m, xs, dys, rows, ldx, ldy, relu_x != 0, acc);
    if (db && threadIdx.x < N)
      for (int r = 0; r < rows; ++r) bacc += dys[r * ldy + threadIdx.x];
    __syncthreads();  // this stage is the fetch target of the next iteration
  }
  // the row groups' partial blocks are summed through shared memory (both x stages are free now: 4096 floats), then one
  // atomic per output and CTA
  const int g = threadIdx.x / m.blocks, b = threadIdx.x - g * m.blocks;
  float* part = &xs2[0][0];  // [(G - 1) * blocks][16] <= 255 * 16 floats
  if (g > 0 && g < m.G) {
#pragma unroll
    for (int j = 0; j < 16; ++j) part[((g - 1) * m.blocks + b) * 16 + j] = acc[j];
  }
  __syncthreads();
  if (g == 0) {
    for (int gg = 1; gg < m.G; ++gg)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] += part[((gg - 1) * m.blocks + b) * 16 + j];
    wgrad_flush(b, m, K, N, acc, [&](int e, float v) { atomicAdd(dW + e, v); });
  }
  if (db && threadIdx.x < N) atomicAdd(db + threadIdx.x, bacc);
}

// Training regularisers of NeuRAD (models/neurad.py:524,541-545), one thread per ray; per-ray losses out (the caller
// takes the mean like losses.py:176,704) and, optionally, the gradient with respect to the weights that carry one.
__global__ void distortion_loss_kernel(const float* __restrict__ c, const float* __restrict__ w, int64_t n_rays, int S,
                                       float* __restrict__ loss, float* __restrict__ dw) {
  const int64_t ray = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  float cl[kLossMaxS + 1], wl[kLossMaxS], dl[kLossMaxS];
  for (int i = 0; i <= S; ++i) cl[i] = c[ray * (S + 1) + i];
  for (int i = 0; i < S; ++i) wl[i] = w[ray * S + i];
  loss[ray] = distortion_loss_ray(cl, wl, S, dw ? dl : nullptr);
  if (dw)
    for (int i = 0; i < S; ++i) dw[ray * S + i] = dl[i];
}

__global__ void zipnerf_interlevel_kernel(const float* __restrict__ c, const float* __restrict__ w, int S,
                                          const float* __restrict__ cp, const float* __restrict__ wp, int Sp, float pulse_width,
                                          int64_t n_rays, float* __restrict__ loss, float* __restrict__ dwp) {
  const int64_t ray = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  float cl[kLossMaxS + 1], wl[kLossMaxS];
  for (int i = 0; i <= S; ++i) cl[i] = c[ray * (S + 1) + i];
  for (int i = 0; i < S; ++i) wl[i] = w[ray * S + i];
  // the proposal level is read and its gradient written in place in global memory (row-strided, once each)
  loss[ray] = zipnerf_interlevel_ray(cl, wl, S, cp + ray * (Sp + 1), wp + ray * Sp, Sp, pulse_width, dwp ? dwp + ray * Sp : nullptr);
}

// NeuRADModel._compute_is_close_to_lidar (models/neurad.py:677-700), training mode: which samples of a LIDAR ray lie
// within carving_epsilon of the measured return (directions_norm = the measured distance), or, for rays without a return,
// closer than non_return_lidar_distance.  Camera rays get 0.  One thread per (ray, sample); bins_e [N,S+1].
__global__ void lidar_carving_mask_kernel(const float* __restrict__ bins_e, const uint8_t* __restrict__ is_lidar,
                                          const float* __restrict__ directions_norm, const uint8_t* __restrict__ did_return,
                                          float carving_epsilon, float non_return_distance, int64_t n_rays, int S,
                                          uint8_t* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S) return;
  const int64_t ray = i / S;
  const int s = (int)(i % S);
  uint8_t m = 0;
  if (is_lidar[ray]) {
    const float mid = fmul(fadd(bins_e[ray * (S + 1) + s], bins_e[ray * (S + 1) + s + 1]), 0.5f);
    const bool close_to_hit = fabsf(fsub(directions_norm[ray], mid)) < carving_epsilon;
    if (did_return)
      m = did_return[ray] ? close_to_hit : (mid < non_return_distance);
    else
      m = close_to_hit;
  }
  mask[i] = m;
}

// ---------------------------------------------------------------------------------- weight gradient on wgmma
// dW[o][i] += sum_r dY[r][o] * act(X[r][i]) as a split-K GEMM on the tensor cores, built from the pieces of
// mlp_tc_kernel (tc_mlp.cuh): the tile's 128 rows are the OUTPUT rows o, a chunk of 48 input rows r is K.  Per chunk
// thread o stages its column dY[r0..r0+48)[o] as A, the CTA stages X^T as the B tile (N padded to 64), and the
// accumulators stay in registers across the CTA's chunks; at the end one atomic per output and CTA adds them to dW.  EXPERIMENTAL: b200nerf_linear_wgrad (CUDA cores) stays the default until this variant has been timed.
constexpr int kWgTcRows = 48;  // rows per chunk = K of the chunk's MMAs
constexpr int kWgTcN = 64;     // MMA N: the layer's input width, padded
constexpr int kWgTcPitch = tc::stage_pitch(kWgTcN);
// [hi | lo] B tile (24 KB), then the A stage (26 KB); at the end the D rows (pitch kWgTcPitch) reuse the whole buffer
constexpr size_t kWgTcSmemBytes = sizeof(float) * (2 * kWgTcN * kWgTcRows + 128 * tc::stage_pitch(kWgTcRows));
static_assert(kWgTcSmemBytes >= 128 * kWgTcPitch * sizeof(float), "D rows do not fit");
__device__ __forceinline__ void wg_stage_xt(float* hi, float* lo, const float* __restrict__ x, int64_t r0, int64_t n_rows, int K, int n_pad,
                                            bool relu_x, int tid, int nthreads) {
  // B(n = i, k = r) = act(X[r0 + r][i]); i runs fastest so that the global reads are contiguous
  for (int e = tid; e < n_pad * kWgTcRows; e += nthreads) {
    const int r = e / n_pad, i = e - r * n_pad;
    float v = (i < K && r0 + r < n_rows) ? x[(r0 + r) * K + i] : 0.0f;
    if (relu_x) v = fmaxf(v, 0.0f);
    const float h = tc::tf32_hi(v);
    const uint32_t off = tc::b_elem_offset(i, r, kWgTcRows);
    hi[off] = h;
    lo[off] = v - h;
  }
}
__global__ void __launch_bounds__(128) linear_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t n_rows,
                                                              int K, int N, int relu_x, float* __restrict__ dW, float* __restrict__ db) {
  extern __shared__ __align__(128) float sm[];  // kWgTcSmemBytes
  const int tid = threadIdx.x;
  float* b_hi = sm;
  float* b_lo = sm + kWgTcN * kWgTcRows;
  float* a_stage = sm + 2 * kWgTcN * kWgTcRows;
  float acc[kWgTcN];
#pragma unroll
  for (int i = 0; i < kWgTcN; ++i) acc[i] = 0.f;
  float bacc = 0.f;
  bool any = false;
  const int64_t n_chunks = (n_rows + kWgTcRows - 1) / kWgTcRows;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const int64_t r0 = ch * kWgTcRows;
    float v[kWgTcRows];
#pragma unroll
    for (int r = 0; r < kWgTcRows; ++r) {
      v[r] = (tid < N && r0 + r < n_rows) ? dy[(r0 + r) * N + tid] : 0.f;
      bacc += v[r];
    }
    tc::store_row<kWgTcRows>(a_stage, tc::stage_pitch(kWgTcRows), v, kWgTcRows);
    wg_stage_xt(b_hi, b_lo, x, r0, n_rows, K, kWgTcN, relu_x != 0, tid, 128);
    tc::fence_async_smem();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
    __syncthreads();
    tc::tile_mma<kWgTcN>(a_stage, tc::stage_pitch(kWgTcRows), kWgTcRows, b_hi, b_lo, acc);
    __syncthreads();  // the A stage and the B tile may be overwritten after this
    any = true;
  }
  if (any) {  // this CTA contributed: drain its accumulator (uniform across the CTA)
    tc::tile_store_d<kWgTcN>(sm, kWgTcPitch, acc);
    __syncthreads();
    float d[kWgTcN];
    tc::load_row<kWgTcN>(sm, kWgTcPitch, d, kWgTcN);
    if (tid < N) {
#pragma unroll
      for (int i = 0; i < kWgTcN; ++i)
        if (i < K) atomicAdd(dW + tid * K + i, d[i]);
      if (db) atomicAdd(db + tid, bacc);
    }
  }
}

// Gradient of the main field's features with respect to the actor trajectories (DynamicActors.actor_positions /
// actor_rotations_6d; require_actor_grad, fields/neurad_field.py:50): a second walk over the samples that only does work
// for the (few) samples inside an actor box -- position gradient of the actor grid lookup, then the pose chain
// (nff_modules.h: neurad_encode_point_pose_bwd), accumulated with atomics into the two bracketing keyframes.
struct PoseBwdArgs {
  const float* mean;       // [N,S,3]
  const float* std;        // [N,S]
  const float* times;      // [N]
  const float* flip;       // [N] or NULL
  const float* dfeatures;  // [N*S, D]
  const float* rot6;       // [T,A,6] raw parameters
  const float* pos;        // [T,A,3]
  float* grad_rot6;        // [T,A,6] accumulated
  float* grad_pos;         // [T,A,3] accumulated
  int64_t n_rays;
  int32_t S;
};
__global__ void __launch_bounds__(kModWarps * 32) neurad_encoding_pose_bwd_kernel(const FieldGrids fg, const Actors A,
                                                                                   const PoseBwdArgs a) {
  __shared__ ActorFrame frames[kModWarps][kModMaxActors];
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kModWarps + warp;
  if (ray >= a.n_rays || A.n_actors == 0) return;
  int left, right;
  float frac;
  keyframe_bracket(A, a.times[ray], left, right, frac);
  for (int k = ln; k < A.n_actors; k += 32) actor_frame(A, k, left, right, frac, frames[warp][k]);
  __syncwarp();
  const int D = fg.stat.L * fg.stat.F;
  const float flip = a.flip ? a.flip[ray] : 1.0f;
  for (int s = ln; s < a.S; s += 32) {
    const int64_t i = ray * a.S + s;
    Gauss g = {a.mean[3 * i], a.mean[3 * i + 1], a.mean[3 * i + 2], a.std[i]};
    neurad_encode_point_pose_bwd(fg, A, frames[warp], a.rot6, a.pos, left, right, frac, g, flip, a.dfeatures + i * D, a.grad_rot6,
                                 a.grad_pos);
  }
}

// Gradient of NeuRADHashEncoding.forward (or NeuRADProposalField.get_density) with respect to the sample means, for
// camera pose optimisation: dmean [N,S,3], written with plain stores (each sample owns its row, no atomics).  The
// thread mapping is the forward's (neurad_encoding_fwd_kernel): one warp per ray builds the ray's actor frames in shared
// memory once, then lane = sample.  The scatter backward's segment-per-thread walk exists to run-length aggregate
// REDUCTIONS into shared table rows; here there is nothing to aggregate, and lane = sample makes the mean / std / dmean
// accesses of a warp contiguous.  MODE 1: features (F = 4), MODE 2: density (F = 1).
struct MeanBwdArgs {
  const float* mean;       // [N,S,3]
  const float* std;        // [N,S]
  const float* times;      // [N]
  const float* flip;       // [N] or NULL
  const float* dfeatures;  // [N*S, D]  (features mode)
  const float* density;    // [N,S]     (density mode: forward output)
  const float* ddensity;   // [N,S]     (density mode)
  float* dmean;            // [N,S,3]   written
  int64_t n_rays;
  int32_t S, actor_grad;
};
template <int MODE>
__global__ void __launch_bounds__(kModWarps * 32) neurad_encoding_mean_bwd_kernel(const FieldGrids fg, const Actors A, const MeanBwdArgs a) {
  static_assert(MODE == 1 || MODE == 2, "features or density mode");
  constexpr int F = MODE == 1 ? 4 : 1;
  extern __shared__ __align__(16) unsigned char mean_bwd_smem[];
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kModWarps + warp;
  if (ray >= a.n_rays) return;
  ActorFrame* frames = reinterpret_cast<ActorFrame*>(mean_bwd_smem) + warp * A.n_actors;
  if (A.n_actors > 0) {
    int left, right;
    float frac;
    keyframe_bracket(A, a.times[ray], left, right, frac);
    for (int k = ln; k < A.n_actors; k += 32) actor_frame(A, k, left, right, frac, frames[k]);
  }
  __syncwarp();
  const int D = fg.stat.L * fg.stat.F;
  const float flip = a.flip ? a.flip[ray] : 1.0f;
  for (int s = ln; s < a.S; s += 32) {
    const int64_t i = ray * a.S + s;
    const Gauss g = {a.mean[3 * i], a.mean[3 * i + 1], a.mean[3 * i + 2], a.std[i]};
    float gp[3];
    if (MODE == 1) {
      neurad_encode_point_mean_bwd_t<F>(fg, frames, A.n_actors, a.actor_grad != 0, g, flip, a.dfeatures + i * D, 1.0f, gp);
    } else {
      // trunc_exp backward (field_components/activations.py:38-41), as in encoding_bwd_segment_pending
      const float gd = a.ddensity[i] * fminf(fmaxf(a.density[i], 3.0590232e-07f), 3269017.372f);
      neurad_encode_point_mean_bwd_t<F>(fg, frames, A.n_actors, a.actor_grad != 0, g, flip, fg.decoder, gd, gp);
    }
    a.dmean[3 * i] = gp[0];
    a.dmean[3 * i + 1] = gp[1];
    a.dmean[3 * i + 2] = gp[2];
  }
}
inline bool launch_neurad_encoding_mean_bwd(const FieldGrids& fg, const Actors& A, const MeanBwdArgs& a, cudaStream_t stream) {
  const unsigned grid = (unsigned)((a.n_rays + kModWarps - 1) / kModWarps);
  if (grid == 0) return true;
  // 64 B per actor and warp: 32 KB at kModMaxActors, under the 48 KB default
  const size_t smem = sizeof(ActorFrame) * kModWarps * (size_t)A.n_actors;
  if (!a.ddensity && encode_bwd_fast_ok(fg, A.n_actors, 4))
    neurad_encoding_mean_bwd_kernel<1><<<grid, kModWarps * 32, smem, stream>>>(fg, A, a);
  else if (a.ddensity && encode_bwd_fast_ok(fg, A.n_actors, 1))
    neurad_encoding_mean_bwd_kernel<2><<<grid, kModWarps * 32, smem, stream>>>(fg, A, a);
  else
    return false;
  return true;
}

// Frustums.get_fast_isotropic_gaussian backward (cameras/rays.py:109-124): dmean [N,S,3] -> d origins [N,3],
// d directions [N,3] (written).  One warp per ray, lane = sample (coalesced dmean reads), then a warp sum.
__global__ void __launch_bounds__(kModWarps * 32) isotropic_gaussian_bwd_kernel(const float* __restrict__ bins_e, const float* __restrict__ dmean,
                                                                                int64_t n_rays, int S, float* __restrict__ dorigins,
                                                                                float* __restrict__ ddirs) {
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kModWarps + warp;
  if (ray >= n_rays) return;
  float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
  for (int s = ln; s < S; s += 32) {
    const int64_t i = ray * S + s;
    const float t = gaussian_t(bins_e[ray * (S + 1) + s], bins_e[ray * (S + 1) + s + 1]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float g = dmean[3 * i + k];
      go[k] += g;
      gd[k] = fmaf(t, g, gd[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    go[k] = warp_sum(go[k]);
    gd[k] = warp_sum(gd[k]);
  }
  if (ln == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      dorigins[3 * ray + k] = go[k];
      ddirs[3 * ray + k] = gd[k];
    }
  }
}

// HashEncoding.forward backward (the stand-alone grid of field_components/encodings.py:425-466, no anti-aliasing rescale):
// grad_table[row] += dout[p, l*F+f] * trilinear corner weight; one thread per point.
__global__ void hashgrid_bwd_kernel(Grid g, const float* __restrict__ x, const float* __restrict__ dout, int64_t n_points,
                                    float* __restrict__ grad_table) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_points) return;
  const Gauss q = {x[3 * p], x[3 * p + 1], x[3 * p + 2], 0.0f};  // std = 0: level_weight() == 1
  float d[kModMaxDim];
  const int D = g.L * g.F;
  for (int k = 0; k < D; ++k) d[k] = dout[p * D + k];
  encode_levels_bwd(grad_table, g, q, d);
}

}  // namespace nff
