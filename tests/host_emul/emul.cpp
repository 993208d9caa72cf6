// TEST SCAFFOLDING ONLY -- runs the device code of neurad-studio_b200/csrc/nff_device.h on the host.
//
// Each "warp" is 32 std::threads executing nff::render_ray in lock-step at warp collectives (see csrc/simt.h), so
// the exact kernel logic (scans, ballots, binary searches, actor culling, MLPs) can be checked against the oracle
// on a machine without a GPU.  Never linked into libb200nerf.so; the product has no CPU path.
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../neurad-studio_b200/csrc/nff_device.h"
#include "../../neurad-studio_b200/csrc/nff_lane.h"
#include "../../neurad-studio_b200/csrc/nff_modules.h"

using namespace nff;

static void pack_linear(const float* w, const float* b, int out_f, int in_f, int outp, float* dw, float* db) {
  for (int k = 0; k < in_f; ++k)
    for (int o = 0; o < outp; ++o) dw[k * outp + o] = o < out_f ? w[o * in_f + k] : 0.f;
  for (int o = 0; o < outp; ++o) db[o] = (o < out_f && b) ? b[o] : 0.f;
}

// ptrs / ints / floats layouts are documented in tests/host_emul/emul.py
// everything up to (not including) the rays: grids, MLPs, actors, sampling, appearance
struct Parsed {
  RenderParams P{};
  std::vector<float> kf, bounds, radii, mlp;
  int pi = 0, ii = 0, fi = 0;
};
static void parse_params(const void* const* ptrs, const int* ints, const float* floats, Parsed& Q) {
  RenderParams& P = Q.P;
  std::vector<float>&kf = Q.kf, &bounds = Q.bounds, &radii = Q.radii;
  int &pi = Q.pi, &ii = Q.ii, &fi = Q.fi;
  const int n_actors = ints[ii++];
  const int n_times = ints[ii++];
  for (int f = 0; f < 3; ++f) {
    FieldGrids& fg = P.fields[f];
    Grid* gs[2] = {&fg.stat, &fg.act};
    for (int k = 0; k < 2; ++k) {
      Grid& g = *gs[k];
      g.L = ints[ii++];
      g.F = ints[ii++];
      int log2T = ints[ii++];
      g.T = 1u << log2T;
      g.mask = g.T - 1u;
      for (int l = 0; l < kMaxLevels; ++l) g.res[l] = floats[fi++];
    }
    fg.stat.table = (const float*)ptrs[pi++];
    fg.actor_tables = (const float* const*)ptrs[pi++];
    fg.decoder = (const float*)ptrs[pi++];
    fg.static_scale = floats[fi++];
    fg.actor_scale = floats[fi++];
  }
  std::vector<float>& mlp = Q.mlp;
  mlp.resize(kMainMlpFloats);
  const float* t[10];
  for (int k = 0; k < 10; ++k) t[k] = (const float*)ptrs[pi++];
  pack_linear(t[0], t[1], kHidden, kGeoIn, kHidden, &mlp[kOffGeoW0], &mlp[kOffGeoB0]);
  pack_linear(t[2], t[3], kNff + 1, kHidden, kGeoOutP, &mlp[kOffGeoW1], &mlp[kOffGeoB1]);
  pack_linear(t[4], t[5], kHidden, kNff + kSh, kHidden, &mlp[kOffFeatW0], &mlp[kOffFeatB0]);
  pack_linear(t[6], t[7], kHidden, kHidden, kHidden, &mlp[kOffFeatW1], &mlp[kOffFeatB1]);
  pack_linear(t[8], t[9], kNff, kHidden, kNff, &mlp[kOffFeatW2], &mlp[kOffFeatB2]);
  P.beta = floats[fi++];
  P.nff_dim = kNff;
  // actors
  const float* a_times = (const float*)ptrs[pi++];
  const float* a_rot6 = (const float*)ptrs[pi++];
  const float* a_pos = (const float*)ptrs[pi++];
  const uint8_t* a_present = (const uint8_t*)ptrs[pi++];
  const float* a_sizes = (const float*)ptrs[pi++];
  float pad[3] = {floats[fi], floats[fi + 1], floats[fi + 2]};
  fi += 3;
  if (n_actors > 0) {
    kf.resize((size_t)9 * n_times * n_actors);
    bounds.resize(3 * n_actors);
    radii.resize(n_actors);
    for (int i = 0; i < n_times * n_actors; ++i) {
      float a1[3] = {a_rot6[6 * i], a_rot6[6 * i + 1], a_rot6[6 * i + 2]};
      float a2[3] = {a_rot6[6 * i + 3], a_rot6[6 * i + 4], a_rot6[6 * i + 5]};
      normalize3(a1);
      float dt = fadd(fadd(fmul(a1[0], a2[0]), fmul(a1[1], a2[1])), fmul(a1[2], a2[2]));
      for (int k = 0; k < 3; ++k) a2[k] = fsub(a2[k], fmul(dt, a1[k]));
      normalize3(a2);
      float* o = &kf[9 * (size_t)i];
      for (int k = 0; k < 3; ++k) { o[k] = a1[k]; o[3 + k] = a2[k]; o[6 + k] = a_pos[3 * i + k]; }
    }
    for (int i = 0; i < n_actors; ++i) {
      float b[3];
      for (int k = 0; k < 3; ++k) b[k] = bounds[3 * i + k] = fadd(fmul(a_sizes[3 * i + k], 0.5f), pad[k]);
      radii[i] = fsqrt(fadd(fadd(fmul(b[0], b[0]), fmul(b[1], b[1])), fmul(b[2], b[2])));
    }
    P.actors = Actors{n_actors, n_times, a_times, kf.data(), a_present, bounds.data(), radii.data()};
  }
  // sampling
  Sampling& s = P.samp;
  s.lam = floats[fi++]; s.scaling = floats[fi++]; s.sky_distance = floats[fi++]; s.hist_pad = floats[fi++];
  s.cam_area_scale = floats[fi++];
  double lam1 = std::fabs((double)s.lam - 1.0);
  s.lam_1 = (float)lam1;
  s.ratio = (float)(lam1 / (double)s.lam);
  s.u1 = (const float*)ptrs[pi++];
  s.u2 = (const float*)ptrs[pi++];
  s.field_of_round[0] = ints[ii++];
  s.field_of_round[1] = ints[ii++];
  // appearance
  P.app.emb = (const float*)ptrs[pi++];
  P.app.num_embeds = ints[ii++];
  P.app.dim = ints[ii++];
  P.app.eps = ints[ii++];
  P.app.duration = floats[fi++];
}

extern "C" {

// tiny-cuda-nn layout (SURVEY 8f row f3): after the ordinary parameter block the caller appends, per field and per grid
// (static 3-D, actor 4-D): tcnn_ints {n_dims, dense_bits, then per level res, off, mask} and tcnn_floats {per level scale};
// tcnn_ptrs {static params, actor params} per field.  lane_mode = 2 selects the LAYOUT = 1 instantiation.
static const void* const* g_tcnn_ptrs = nullptr;
static const int* g_tcnn_ints = nullptr;
static const float* g_tcnn_floats = nullptr;
static int g_bwd_generic = 0;  // 1: run the generic (MODE 0) scatter backward even where a fast path applies
// actor edit of the following lane-mode renders (b200nerf_set_actor_edit): lateral, longitudinal, height, rotation, index
static int g_edit_on = 0;
static double g_edit[5];
int emul_set_actor_edit(int on, const double* e) {
  g_edit_on = on;
  for (int i = 0; i < 5; ++i) g_edit[i] = on ? e[i] : 0.0;
  return 0;
}
int emul_set_bwd_generic(int on) { g_bwd_generic = on; return 0; }
int emul_set_tcnn(const void* const* ptrs, const int* ints, const float* floats) {
  g_tcnn_ptrs = ptrs; g_tcnn_ints = ints; g_tcnn_floats = floats;
  return 0;
}
static void apply_tcnn(RenderParams& P, int n_actors) {
  int pi = 0, ii = 0, fi = 0;
  for (int f = 0; f < 3; ++f) {
    FieldGrids& fg = P.fields[f];
    Grid* gs[2] = {&fg.stat, &fg.act};
    for (int k = 0; k < 2; ++k) {
      Grid& g = *gs[k];
      g.n_dims = g_tcnn_ints[ii++];
      g.dense_bits = (uint32_t)g_tcnn_ints[ii++];
      for (int l = 0; l < kMaxLevels; ++l) {
        g.lvl_res[l] = (uint32_t)g_tcnn_ints[ii++];
        g.lvl_off[l] = (uint32_t)g_tcnn_ints[ii++];
        g.lvl_mask[l] = (uint32_t)g_tcnn_ints[ii++];
        g.pos_scale[l] = g_tcnn_floats[fi++];
      }
      g.table = (const float*)g_tcnn_ptrs[pi++];
    }
    fg.n_actors_f = (float)(n_actors > 0 ? n_actors : 1);
  }
  P.layout = 1;
}

int emul_render(const void* const* ptrs, const int* ints, const float* floats, long long n_rays, int lane_mode) {
  Parsed Q;
  parse_params(ptrs, ints, floats, Q);
  RenderParams& P = Q.P;
  std::vector<float>& mlp = Q.mlp;
  int &pi = Q.pi;
  // rays
  P.rays.origins = (const float*)ptrs[pi++];
  P.rays.directions = (const float*)ptrs[pi++];
  P.rays.pixel_area = (const float*)ptrs[pi++];
  P.rays.times = (const float*)ptrs[pi++];
  P.rays.nears = (const float*)ptrs[pi++];
  P.rays.fars = (const float*)ptrs[pi++];
  P.rays.sensor_idx = (const int64_t*)ptrs[pi++];
  P.rays.is_lidar = (const uint8_t*)ptrs[pi++];
  // outputs
  P.out.features = (float*)ptrs[pi++];
  P.out.depth = (float*)ptrs[pi++];
  P.out.accumulation = (float*)ptrs[pi++];
  P.out.prop_depth_0 = (float*)ptrs[pi++];
  P.out.prop_depth_1 = (float*)ptrs[pi++];
  // trace
  P.trace.prop_weights_0 = (float*)ptrs[pi++];
  P.trace.prop_weights_1 = (float*)ptrs[pi++];
  P.trace.bins_s_1 = (float*)ptrs[pi++];
  P.trace.bins_e_1 = (float*)ptrs[pi++];
  P.trace.bins_s_2 = (float*)ptrs[pi++];
  P.trace.bins_e_2 = (float*)ptrs[pi++];
  P.trace.inds_1 = (int32_t*)ptrs[pi++];
  P.trace.inds_2 = (int32_t*)ptrs[pi++];
  P.trace.sdf = (float*)ptrs[pi++];
  P.trace.alpha = (float*)ptrs[pi++];
  P.trace.field_feature = (float*)ptrs[pi++];
  P.trace.weights = (float*)ptrs[pi++];
  P.trace.actor_id_0 = (int32_t*)ptrs[pi++];
  P.trace.actor_id_1 = (int32_t*)ptrs[pi++];
  P.trace.actor_id_main = (int32_t*)ptrs[pi++];
  P.n_rays = n_rays;

  if (lane_mode) {
    // ray-per-lane variant: no warp collectives, so plain sequential execution of every "thread" is exact
    std::vector<float> scratch(lane_scratch_floats_per_cta());
    LaneScratch sc = lane_scratch_of(scratch.data(), 0);
    std::vector<float> panel((size_t)kNff * kLaneThreads);
    MlpLaneFfma pol{mlp.data(), panel.data()};
    if (g_edit_on && !resolve_actor_edit(P.actors, g_edit[0], g_edit[1], g_edit[2], g_edit[3], g_edit[4])) return 2;
    if (lane_mode == 2) {
      apply_tcnn(P, P.actors.n_actors);
      pol.sh_tcnn = 1;
      if (P.actors.edit_last > P.actors.edit_first) {
        for (long long r = 0; r < n_rays; ++r) render_ray_lane<MlpLaneFfma, 1, true>(P, sc, pol, (int)(r % kLaneThreads), r, true);
        return 0;
      }
      for (long long r = 0; r < n_rays; ++r) render_ray_lane<MlpLaneFfma, 1>(P, sc, pol, (int)(r % kLaneThreads), r, true);
      return 0;
    }
    if (P.actors.edit_last > P.actors.edit_first) {
      for (long long r = 0; r < n_rays; ++r) render_ray_lane<MlpLaneFfma, 0, true>(P, sc, pol, (int)(r % kLaneThreads), r, true);
      return 0;
    }
    for (long long r = 0; r < n_rays; ++r) render_ray_lane(P, sc, pol, (int)(r % kLaneThreads), r, true);
    return 0;
  }
  // one emulated warp (32 threads) per hardware thread group; rays are distributed round-robin
  unsigned hw = std::thread::hardware_concurrency();
  int n_warps = hw >= 64 ? 2 : 1;
  if (n_warps > n_rays) n_warps = (int)n_rays;
  if (n_warps < 1) return 0;
  std::vector<simt::EmuWarp> warps(n_warps);
  std::vector<WarpShared> shared(n_warps);
  std::vector<std::thread> threads;
  for (int w = 0; w < n_warps; ++w)
    for (int l = 0; l < 32; ++l)
      threads.emplace_back([&, w, l]() {
        simt::t_lane = l;
        simt::t_warp = &warps[w];
        MlpFfma pol{mlp.data()};
        for (long long r = w; r < n_rays; r += n_warps) render_ray(P, shared[w], pol, r, true);
      });
  for (auto& th : threads) th.join();
  return 0;
}

// tcnn.Encoding{HashGrid}.forward through the device functions (tcnn_corners / tcnn_corner_weight), D = 3 or 4.
int emul_tcnn_hashgrid(const int* ints, const float* scales, const float* params, const float* x, long long n, float* out) {
  Grid g{};
  int ii = 0;
  g.n_dims = ints[ii++]; g.L = ints[ii++]; g.F = ints[ii++]; g.dense_bits = (uint32_t)ints[ii++];
  for (int l = 0; l < g.L; ++l) {
    g.lvl_res[l] = (uint32_t)ints[ii++]; g.lvl_off[l] = (uint32_t)ints[ii++]; g.lvl_mask[l] = (uint32_t)ints[ii++];
    g.pos_scale[l] = scales[l];
  }
  g.table = params;
  for (long long i = 0; i < n; ++i)
    for (int l = 0; l < g.L; ++l) {
      uint32_t idx[16];
      float frac[4];
      if (g.n_dims == 3) tcnn_corners<3>(g, l, x + 3 * i, idx, frac); else tcnn_corners<4>(g, l, x + 4 * i, idx, frac);
      for (int f = 0; f < g.F; ++f) {
        float v = 0.f;
        for (int c = 0; c < (1 << g.n_dims); ++c) {
          const float w = g.n_dims == 3 ? tcnn_corner_weight<3>(c, frac) : tcnn_corner_weight<4>(c, frac);
          v = std::fmaf(w, params[(size_t)idx[c] * g.F + f], v);
        }
        out[i * (g.L * g.F) + l * g.F + f] = v;
      }
    }
  return 0;
}

// Frustums.get_fast_isotropic_gaussian as the kernels compute it (nff_device.h: sample_gaussian).
int emul_gaussian(const float* origins, const float* dirs, const float* area, const float* bins_e, long long n_rays, int S,
                  float* mean, float* std) {
  for (long long r = 0; r < n_rays; ++r)
    for (int s = 0; s < S; ++s) {
      const long long i = r * S + s;
      Gauss g = sample_gaussian(origins + 3 * r, dirs + 3 * r, area[r], bins_e[r * (S + 1) + s], bins_e[r * (S + 1) + s + 1]);
      mean[3 * i] = g.x; mean[3 * i + 1] = g.y; mean[3 * i + 2] = g.z;
      std[i] = g.std;
    }
  return 0;
}

// NeuRADHashEncoding.forward as the module-level operator computes it (nff_modules.h: neurad_encode_point; same loop
// structure as neurad_encoding_fwd_kernel in modules.cuh).  extra = {mean [N,S,3], std [N,S], times [N] or NULL,
// dirs ([N,3] if dirs_per_ray else [N,S,3]) or NULL, features [N*S,D] or NULL, density [N,S] or NULL, dirs_out [N,S,3]
// or NULL, actor_id [N,S] (int32) or NULL, flip [N] or NULL}
int emul_encoding(const void* const* ptrs, const int* ints, const float* floats, const void* const* extra, long long n_rays,
                  int S, int field, int dirs_per_ray) {
  Parsed Q;
  parse_params(ptrs, ints, floats, Q);
  const FieldGrids& fg = Q.P.fields[field];
  const Actors& A = Q.P.actors;
  const float* mean = (const float*)extra[0];
  const float* std_ = (const float*)extra[1];
  const float* times = (const float*)extra[2];
  const float* dirs = (const float*)extra[3];
  float* features = (float*)extra[4];
  float* density = (float*)extra[5];
  float* dirs_out = (float*)extra[6];
  int32_t* actor_id = (int32_t*)extra[7];
  const float* flips = (const float*)extra[8];
  const int D = fg.stat.L * fg.stat.F;
  std::vector<ActorFrame> frames(A.n_actors > 0 ? A.n_actors : 1);
  for (long long r = 0; r < n_rays; ++r) {
    if (A.n_actors > 0) {
      int left, right;
      float frac;
      keyframe_bracket(A, times[r], left, right, frac);
      for (int a = 0; a < A.n_actors; ++a) actor_frame(A, a, left, right, frac, frames[a]);
    }
    const float flip = flips ? flips[r] : 1.0f;
    for (int s = 0; s < S; ++s) {
      const long long i = r * S + s;
      Gauss g = {mean[3 * i], mean[3 * i + 1], mean[3 * i + 2], std_[i]};
      float dir[3] = {0.f, 0.f, 0.f};
      if (dirs) {
        const float* dp = dirs + 3 * (dirs_per_ray ? r : i);
        dir[0] = dp[0]; dir[1] = dp[1]; dir[2] = dp[2];
      }
      float feat[kModMaxDim];
      int aid;  // same dispatch as launch_neurad_encoding_fwd (modules.cuh); g_bwd_generic also selects the generic forward
      if (!g_bwd_generic && encode_bwd_fast_ok(fg, A.n_actors, 4))
        aid = neurad_encode_point_t<8, 4>(fg, frames.data(), A.n_actors, g, feat, dirs ? dir : nullptr, flip);
      else if (!g_bwd_generic && encode_bwd_fast_ok(fg, A.n_actors, 1))
        aid = neurad_encode_point_t<8, 1>(fg, frames.data(), A.n_actors, g, feat, dirs ? dir : nullptr, flip);
      else
        aid = neurad_encode_point(fg, frames.data(), A.n_actors, g, feat, dirs ? dir : nullptr, flip);
      if (features)
        for (int k = 0; k < D; ++k) features[i * D + k] = feat[k];
      if (density) {
        float acc = 0.f;
        for (int k = 0; k < D; ++k) acc = std::fmaf(feat[k], fg.decoder[k], acc);
        density[i] = std::exp(acc);
      }
      if (dirs_out)
        for (int k = 0; k < 3; ++k) dirs_out[3 * i + k] = dir[k];
      if (actor_id) actor_id[i] = aid;
    }
  }
  return 0;
}

// Backward of the module-level encoding (nff_modules.h: neurad_encode_point_bwd; loop structure of
// neurad_encoding_bwd_kernel).  extra = {mean, std, times|NULL, flip|NULL, dfeatures|NULL, density|NULL, ddensity|NULL,
// grad_static|NULL, grad_actor_ptrs (array of n_actors float*)|NULL, grad_decoder|NULL}
int emul_encoding_bwd(const void* const* ptrs, const int* ints, const float* floats, const void* const* extra, long long n_rays,
                      int S, int field) {
  Parsed Q;
  parse_params(ptrs, ints, floats, Q);
  const FieldGrids& fg = Q.P.fields[field];
  const Actors& A = Q.P.actors;
  const float* mean = (const float*)extra[0];
  const float* std_ = (const float*)extra[1];
  const float* times = (const float*)extra[2];
  const float* flips = (const float*)extra[3];
  const float* dfeatures = (const float*)extra[4];
  const float* density = (const float*)extra[5];
  const float* ddensity = (const float*)extra[6];
  float* grad_static = (float*)extra[7];
  float* const* grad_actors = (float* const*)extra[8];
  float* grad_decoder = (float*)extra[9];
  const int D = fg.stat.L * fg.stat.F;
  std::vector<ActorFrame> frames(A.n_actors > 0 ? A.n_actors : 1);
  for (long long r = 0; r < n_rays; ++r) {
    if (A.n_actors > 0) {
      int left, right;
      float frac;
      keyframe_bracket(A, times[r], left, right, frac);
      for (int a = 0; a < A.n_actors; ++a) actor_frame(A, a, left, right, frac, frames[a]);
    }
    const float flip = flips ? flips[r] : 1.0f;
    // same dispatch and the same thread -> (ray, segment) cut as neurad_encoding_bwd_kernel (modules.cuh)
    const bool fast_feat = !g_bwd_generic && !ddensity && encode_bwd_fast_ok(fg, A.n_actors, 4);
    const bool fast_dens = !g_bwd_generic && ddensity && encode_bwd_fast_ok(fg, A.n_actors, 1);
    if (fast_feat || fast_dens) {
      const int seg_len = (S + kBwdSegments - 1) / kBwdSegments;
      for (int seg = 0; seg < kBwdSegments; ++seg) {
        const int s0 = seg * seg_len, n = std::min(S, s0 + seg_len) - s0;
        float dec8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (fast_feat)
          encoding_bwd_segment<4, false, NFF_BWD_AGG_F4>(fg, grad_static, grad_actors, frames.data(), A.n_actors, mean, std_, dfeatures, nullptr,
                                                         nullptr, r * S + s0, n, flip, dec8);
        else if (grad_decoder)
          encoding_bwd_segment<1, true, NFF_BWD_AGG_F1>(fg, grad_static, grad_actors, frames.data(), A.n_actors, mean, std_, nullptr, density,
                                                        ddensity, r * S + s0, n, flip, dec8);
        else
          encoding_bwd_segment<1, false, NFF_BWD_AGG_F1>(fg, grad_static, grad_actors, frames.data(), A.n_actors, mean, std_, nullptr, density,
                                                         ddensity, r * S + s0, n, flip, dec8);
        if (fast_dens && grad_decoder)
          for (int k = 0; k < D && k < 8; ++k) grad_decoder[k] += dec8[k];
      }
      continue;
    }
    for (int s = 0; s < S; ++s) {
      const long long i = r * S + s;
      Gauss g = {mean[3 * i], mean[3 * i + 1], mean[3 * i + 2], std_[i]};
      float dfeat[kModMaxDim];
      if (ddensity) {
        const float gd = ddensity[i] * std::fmin(std::fmax(density[i], 3.0590232e-07f), 3269017.372f);  // trunc_exp backward clamp
        if (grad_decoder) {
          float feat[kModMaxDim];
          neurad_encode_point(fg, frames.data(), A.n_actors, g, feat, nullptr, flip);
          for (int k = 0; k < D; ++k) grad_decoder[k] = std::fmaf(gd, feat[k], grad_decoder[k]);
        }
        for (int k = 0; k < D; ++k) dfeat[k] = gd * fg.decoder[k];
      } else {
        for (int k = 0; k < D; ++k) dfeat[k] = dfeatures[i * D + k];
      }
      neurad_encode_point_bwd(fg, grad_static, grad_actors, frames.data(), A.n_actors, g, flip, dfeat);
    }
  }
  return 0;
}

// weights backward rows (alpha_weights_bwd_ray / density_weights_bwd_ray)
int emul_weights_bwd(int from_alpha, const float* a, const float* b, const float* dw, long long n_rays, int S, float* out) {
  for (long long r = 0; r < n_rays; ++r) {
    if (from_alpha)
      alpha_weights_bwd_ray(a + r * S, dw + r * S, S, out + r * S);
    else
      density_weights_bwd_ray(a + r * S, b + r * S, dw + r * S, S, out + r * S);
  }
  return 0;
}

// linear_wgrad_kernel's tiling (modules.cuh) with `n_ctas` CTAs of 256 "threads" run one after the other.
int emul_linear_wgrad(const float* x, const float* dy, long long n_rows, int K, int N, int relu_x, int n_ctas, float* dW,
                      float* db) {
  constexpr int kThreads = 256, kRows = 32;
  const long long n_tiles = (n_rows + kRows - 1) / kRows;
  const int ldx = (K + 3) & ~3, ldy = (N + 3) & ~3;
  const WgradMap m = wgrad_map(K, N, kThreads);
  alignas(16) float xs[kRows * 64];   // the staged tiles: rows padded to whole quads, pad columns zero
  alignas(16) float dys[kRows * 64];
  for (int cta = 0; cta < n_ctas; ++cta)
    for (int tid = 0; tid < kThreads; ++tid) {
      float acc[16] = {};
      float bacc = 0.f;
      for (long long t = cta; t < n_tiles; t += n_ctas) {
        const long long r0 = t * kRows;
        const int rows = (int)(n_rows - r0 < kRows ? n_rows - r0 : kRows);
        for (int r = 0; r < rows; ++r) {
          for (int c = 0; c < ldx; ++c) xs[r * ldx + c] = c < K ? x[(r0 + r) * K + c] : 0.f;
          for (int c = 0; c < ldy; ++c) dys[r * ldy + c] = c < N ? dy[(r0 + r) * N + c] : 0.f;
        }
        wgrad_tile(tid, m, xs, dys, rows, ldx, ldy, relu_x != 0, acc);
        if (db && tid < N)
          for (int r = 0; r < rows; ++r) bacc += dys[r * ldy + tid];
      }
      const int g = tid / m.blocks, b = tid - g * m.blocks;
      if (g < m.G) wgrad_flush(b, m, K, N, acc, [&](int e, float v) { dW[e] += v; });  // (the kernel sums the row groups in shared memory first)
      if (db && tid < N) db[tid] += bacc;
    }
  return 0;
}

// training regularisers (nff_modules.h: distortion_loss_ray / zipnerf_interlevel_ray), one "thread" per ray
int emul_distortion_loss(const float* c, const float* w, long long n_rays, int S, float* loss, float* dw) {
  for (long long r = 0; r < n_rays; ++r) loss[r] = distortion_loss_ray(c + r * (S + 1), w + r * S, S, dw ? dw + r * S : nullptr);
  return 0;
}
int emul_zipnerf_interlevel(const float* c, const float* w, int S, const float* cp, const float* wp, int Sp, float pulse_width,
                            long long n_rays, float* loss, float* dwp) {
  for (long long r = 0; r < n_rays; ++r)
    loss[r] = zipnerf_interlevel_ray(c + r * (S + 1), w + r * S, S, cp + r * (Sp + 1), wp + r * Sp, Sp, pulse_width,
                                     dwp ? dwp + r * Sp : nullptr);
  return 0;
}

// Trajectory gradients of the main field's features (nff_modules.h: neurad_encode_point_pose_bwd; loop structure of
// neurad_encoding_pose_bwd_kernel).  extra = {mean, std, times, flip|NULL, dfeatures, rot6 [T,A,6], pos [T,A,3],
// grad_rot6, grad_pos}
int emul_encoding_pose_bwd(const void* const* ptrs, const int* ints, const float* floats, const void* const* extra, long long n_rays,
                           int S, int field) {
  Parsed Q;
  parse_params(ptrs, ints, floats, Q);
  const FieldGrids& fg = Q.P.fields[field];
  const Actors& A = Q.P.actors;
  if (A.n_actors == 0) return 0;
  const float* mean = (const float*)extra[0];
  const float* std_ = (const float*)extra[1];
  const float* times = (const float*)extra[2];
  const float* flips = (const float*)extra[3];
  const float* dfeatures = (const float*)extra[4];
  const float* rot6 = (const float*)extra[5];
  const float* pos = (const float*)extra[6];
  float* grad_rot6 = (float*)extra[7];
  float* grad_pos = (float*)extra[8];
  const int D = fg.stat.L * fg.stat.F;
  std::vector<ActorFrame> frames(A.n_actors);
  for (long long r = 0; r < n_rays; ++r) {
    int left, right;
    float frac;
    keyframe_bracket(A, times[r], left, right, frac);
    for (int a = 0; a < A.n_actors; ++a) actor_frame(A, a, left, right, frac, frames[a]);
    const float flip = flips ? flips[r] : 1.0f;
    for (int s = 0; s < S; ++s) {
      const long long i = r * S + s;
      Gauss g = {mean[3 * i], mean[3 * i + 1], mean[3 * i + 2], std_[i]};
      neurad_encode_point_pose_bwd(fg, A, frames.data(), rot6, pos, left, right, frac, g, flip, dfeatures + i * D, grad_rot6, grad_pos);
    }
  }
  return 0;
}

// stand-alone HashEncoding backward (modules.cuh: hashgrid_bwd_kernel = encode_levels_bwd with unit level weights)
int emul_hashgrid_bwd(int L, int F, int log2T, const float* res, const float* x, const float* dout, long long n_points, float* grad_table) {
  Grid g{};
  g.L = L; g.F = F; g.T = 1u << log2T; g.mask = g.T - 1u;
  for (int l = 0; l < L; ++l) g.res[l] = res[l];
  for (long long p = 0; p < n_points; ++p) {
    const Gauss q = {x[3 * p], x[3 * p + 1], x[3 * p + 2], 0.0f};
    encode_levels_bwd(grad_table, g, q, dout + p * L * F);
  }
  return 0;
}
}
