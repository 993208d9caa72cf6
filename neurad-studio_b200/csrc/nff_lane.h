// nff_lane.h -- "one ray per lane" variant of the fused NFF render.
//
// Why: profiling the warp-per-ray kernel showed it bound by the L1 tag stage: a
// gather instruction whose 32 lanes are 32 consecutive samples of ONE ray touches ~13 different 128-byte lines
// (17 sectors) per request, and neither more loads in flight nor more ILP moved the time.  Here the 32 lanes of a warp
// are 32 ADJACENT RAYS at the SAME sample index: their positions differ by a pixel footprint, so at the coarse and
// middle levels of the grids the lanes fall into the same few cells and one request touches a handful of lines.
//
// Consequences of the mapping:
//   * all per-ray sequences (transmittance, cdf) are plain sequential loops in one lane -- the same summation order as
//     torch.cumsum / torch.cumprod in the reference, no warp scans;
//   * searchsorted becomes a merge walk (the quantiles u are ascending, the cdf is non-decreasing);
//   * per-ray arrays (weights, resampled bin edges, actor candidates) live in a global scratch slab laid out
//     [index][thread] so that every access is one coalesced line per warp; the slab is small (0.5 MB per CTA) and stays
//     in L2;
//   * the main-field MLP tile is 128 rays x ONE sample; features are composited into 32 per-lane accumulators.
#pragma once
#include "nff_device.h"

namespace nff {

#ifndef NFF_LANE_THREADS
#define NFF_LANE_THREADS 512
#endif
#ifndef NFF_F4_WEIGHTS
#define NFF_F4_WEIGHTS 0  // main-grid interpolation as a weighted sum over the 8 corners (weights shared by the 4 features)
#endif
constexpr int kLaneThreads = NFF_LANE_THREADS;  // threads (= rays in flight) per CTA (256: 2 CTAs/SM, 512: 1 CTA/SM)
constexpr int kLaneCtasPerSm = 512 / kLaneThreads;
constexpr int kCandFloats = 16;    // per candidate: 12 (world->box 3x4) + 3 (bounds) + 1 (actor id bits)
constexpr int kLaneMaxCand = 32;   // actor candidates per ray (they live in the global scratch slab, so this is cheap)

// per-CTA slab of the global scratch, all arrays [index][kLaneThreads]
struct LaneScratch {
  float* w;      // [kS0]       padded proposal weights of the current round
  float* bins1;  // [kS1 + 1]   spacing edges after round 0
  float* bins2;  // [kS2 + 1]   spacing edges after round 1
  float* cand;   // [kLaneMaxCand * kCandFloats]
};
NFF_HD size_t lane_scratch_floats_per_cta() {
  return (size_t)kLaneThreads * (kS0 + (kS1 + 1) + (kS2 + 1) + kLaneMaxCand * kCandFloats);
}
NFF_D LaneScratch lane_scratch_of(float* base, int cta) {
  float* p = base + (size_t)cta * lane_scratch_floats_per_cta();
  LaneScratch s;
  s.w = p;
  s.bins1 = s.w + (size_t)kS0 * kLaneThreads;
  s.bins2 = s.bins1 + (size_t)(kS1 + 1) * kLaneThreads;
  s.cand = s.bins2 + (size_t)(kS2 + 1) * kLaneThreads;
  return s;
}

// --------------------------------------------------------------------------------------------- actors, per lane
// Same computation as actor_candidates() (nff_device.h) for ONE ray: loop over all actors, keep those whose bounding
// sphere the ray line passes (neurad_encoding.py:225-240), store [R^T | -R^T t], bounds and id in the scratch column.
// EDIT: an actor edit is active (Actors::edit_first/last).  The cull then needs the edited centre, so the rotation is
// built before it; without an edit the cheap centre test rejects first and the edit code is not compiled in.
template <bool EDIT = false>
NFF_D int lane_actor_candidates(const Actors& A, float time, const float o[3], const float d[3], const LaneScratch& sc,
                                int tid, int* overflow) {
  int n = 0;
  if (A.n_actors == 0) return 0;
  int lo = 0, hi = A.n_times;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (ldg(A.times + mid) < time) lo = mid + 1; else hi = mid;
  }
  int right = lo, left = right - 1 < 0 ? 0 : right - 1;
  if (right > A.n_times - 1) right = A.n_times - 1;
  float tl = ldg(A.times + left), tr = ldg(A.times + right);
  float frac = fdiv(fsub(time, tl), fadd(fsub(tr, tl), 1e-6f));
  frac = fminf(fmaxf(frac, 0.0f), 1.0f);
#pragma unroll 1
  for (int a = 0; a < A.n_actors; ++a) {
    const float* kl = A.keyframes + ((size_t)left * A.n_actors + a) * 9;
    const float* kr = A.keyframes + ((size_t)right * A.n_actors + a) * 9;
    float p[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      float l_ = ldg(kl + i), r_ = ldg(kr + i);
      p[i] = fadd(l_, fmul(fsub(r_, l_), frac));
    }
    bool valid = (A.present[(size_t)left * A.n_actors + a] | A.present[(size_t)right * A.n_actors + a]) != 0;
    // distance from the box centre to the ray line (independent of the rotation, so without an edit it rejects first)
    auto near_ray = [&]() {
      float v[3] = {fsub(p[6], o[0]), fsub(p[7], o[1]), fsub(p[8], o[2])};
      float cx = fsub(fmul(v[1], d[2]), fmul(v[2], d[1]));
      float cy = fsub(fmul(v[2], d[0]), fmul(v[0], d[2]));
      float cz = fsub(fmul(v[0], d[1]), fmul(v[1], d[0]));
      float dist = fsqrt(fadd(fadd(fmul(cx, cx), fmul(cy, cy)), fmul(cz, cz)));
      return valid && dist < ldg(A.radii + a) * 1.001f;
    };
    if (!EDIT) {
      if (!near_ray()) continue;
      if (n >= kLaneMaxCand) {
        *overflow = 1;
        continue;
      }
    }
    float b1[3] = {p[0], p[1], p[2]};
    normalize3(b1);
    float dt = fadd(fadd(fmul(b1[0], p[3]), fmul(b1[1], p[4])), fmul(b1[2], p[5]));
    float b2[3] = {fsub(p[3], fmul(dt, b1[0])), fsub(p[4], fmul(dt, b1[1])), fsub(p[5], fmul(dt, b1[2]))};
    normalize3(b2);
    float b3[3] = {fsub(fmul(b1[1], b2[2]), fmul(b1[2], b2[1])), fsub(fmul(b1[2], b2[0]), fmul(b1[0], b2[2])),
                   fsub(fmul(b1[0], b2[1]), fmul(b1[1], b2[0]))};
    if (EDIT) {
      edit_box_pose(A, a, b1, b2, b3, p + 6);
      if (!near_ray()) continue;
      if (n >= kLaneMaxCand) {
        *overflow = 1;
        continue;
      }
    }
    float R[9] = {b1[0], b2[0], b3[0], b1[1], b2[1], b3[1], b1[2], b2[2], b3[2]};
    float* c = sc.cand + (size_t)n * kCandFloats * kLaneThreads + tid;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      c[(4 * i + 0) * kLaneThreads] = R[3 * i + 0];
      c[(4 * i + 1) * kLaneThreads] = R[3 * i + 1];
      c[(4 * i + 2) * kLaneThreads] = R[3 * i + 2];
      c[(4 * i + 3) * kLaneThreads] = -fadd(fadd(fmul(R[3 * i], p[6]), fmul(R[3 * i + 1], p[7])), fmul(R[3 * i + 2], p[8]));
      c[(12 + i) * kLaneThreads] = ldg(A.bounds + 3 * a + i);
    }
    c[15 * kLaneThreads] = (float)a;  // actor ids are small integers: exact in fp32
    ++n;
  }
  return n;
}

// inside-box test against this ray's candidates; highest actor index wins (candidates are stored in increasing order)
NFF_D int lane_actor_of_sample(const LaneScratch& sc, int tid, int n_cand, const Gauss& g, float pb[3], float M_out[12]) {
  int hit = -1;
  for (int c = 0; c < n_cand; ++c) {
    const float* p = sc.cand + (size_t)c * kCandFloats * kLaneThreads + tid;
    float M[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) M[i] = p[i * kLaneThreads];
    float q0 = fadd(fadd(fadd(fmul(M[0], g.x), fmul(M[1], g.y)), fmul(M[2], g.z)), M[3]);
    float q1 = fadd(fadd(fadd(fmul(M[4], g.x), fmul(M[5], g.y)), fmul(M[6], g.z)), M[7]);
    float q2 = fadd(fadd(fadd(fmul(M[8], g.x), fmul(M[9], g.y)), fmul(M[10], g.z)), M[11]);
    if (fabsf(q0) < p[12 * kLaneThreads] && fabsf(q1) < p[13 * kLaneThreads] && fabsf(q2) < p[14 * kLaneThreads]) {
      hit = (int)p[15 * kLaneThreads];
      pb[0] = q0; pb[1] = q1; pb[2] = q2;
#pragma unroll
      for (int i = 0; i < 12; ++i) M_out[i] = M[i];
    }
  }
  return hit;
}

// LAYOUT 0: the reference's torch layout (hashed [L*T,F] tables, one 3-D grid per actor); 1: tiny-cuda-nn layout (nff_device.h)
// ACTORS = false: the scene has no actors (n_cand == 0), the actor path is not compiled in.
template <int LAYOUT = 0, bool ACTORS = true>
NFF_D float lane_proposal_density(const FieldGrids& fg, const LaneScratch& sc, int tid, int n_cand, const Gauss& g,
                                  int* actor_id) {
  float pb[3], M[12];
  int a = ACTORS && n_cand > 0 ? lane_actor_of_sample(sc, tid, n_cand, g, pb, M) : -1;
  float acc;
  if (a >= 0) {
    Gauss ga = {pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    if (LAYOUT == 1) {
      const float x4[4] = {ga.x, ga.y, ga.z, fdiv((float)a, fg.n_actors_f)};  // neurad_encoding.py:273-275
      acc = tcnn_encode_f1_dot<4>(fg.act, 4, x4, ga.std, fg.decoder);
    } else {
      acc = encode_f1_dot<4, NFF_G_ACT>(fg.actor_tables[a], fg.act, ga, fg.decoder);
    }
  } else {
    Gauss gs = contract(g, fg.static_scale);
    if (LAYOUT == 1) {
      const float x3[3] = {gs.x, gs.y, gs.z};
      acc = tcnn_encode_f1_dot<3>(fg.stat, 6, x3, gs.std, fg.decoder);
    } else {
      acc = encode_f1_dot<6, NFF_G_PROP>(fg.stat.table, fg.stat, gs, fg.decoder);
    }
  }
  *actor_id = a;
  return expf(acc);
}

// F = 4 grid into the CTA's shared panel column [4l+f][tid] (rolled level loop: small code); `pitch` = panel row pitch.
// The stored values are `scale` (a power of two, folded into the level weight) times the features, exactly.
NFF_D void encode_f4_col(const float* NFF_RESTRICT table, const Grid& gr, int L, Gauss g, float* x /* = panel + tid */, int pitch,
                         float scale) {
  const uint32_t maskb = gr.mask << 4;
#pragma unroll 2
  for (int l = 0; l < L; ++l) {
    const float res = gr.res[l];
    const CellB<4> c = grid_cell_b<4>(g.x, g.y, g.z, res);
    uint32_t r[8];
    cell_offsets_b<4>(c, maskb, r);
    const char* base = level_base(table, l, gr.T, 16);
    float4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = ldg_at<float4>(base, r[k]);
    const float w = fmul(level_weight(res, g.std), scale);
    const float ix = 1.0f - c.ox, iy = 1.0f - c.oy, iz = 1.0f - c.oz;
#if NFF_F4_WEIGHTS
    // the 8 corner weights are shared by the row's 4 features: 14 multiplies for the weights (level weight folded in) and
    // 8 multiply-adds per feature (46 instructions) instead of four blend trees and four scalings (60); same value up to
    // the rounding order (<= 1e-7 relative, like the FMA-folded blends)
    const float z1 = c.oz * w, z0 = iz * w;
    const float y1z1 = c.oy * z1, y0z1 = iy * z1, y1z0 = c.oy * z0, y0z0 = iy * z0;
    const float wk[8] = {c.ox * y1z1, c.ox * y0z1, ix * y0z1, ix * y1z1, c.ox * y1z0, c.ox * y0z0, ix * y0z0, ix * y1z0};
    float a0 = wk[0] * v[0].x, a1 = wk[0] * v[0].y, a2 = wk[0] * v[0].z, a3 = wk[0] * v[0].w;
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      a0 = fmaf(wk[k], v[k].x, a0);
      a1 = fmaf(wk[k], v[k].y, a1);
      a2 = fmaf(wk[k], v[k].z, a2);
      a3 = fmaf(wk[k], v[k].w, a3);
    }
    x[(4 * l + 0) * pitch] = a0;
    x[(4 * l + 1) * pitch] = a1;
    x[(4 * l + 2) * pitch] = a2;
    x[(4 * l + 3) * pitch] = a3;
#else
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].x;
    x[(4 * l + 0) * pitch] = fmul(trilerp_b<4>(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].y;
    x[(4 * l + 1) * pitch] = fmul(trilerp_b<4>(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].z;
    x[(4 * l + 2) * pitch] = fmul(trilerp_b<4>(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].w;
    x[(4 * l + 3) * pitch] = fmul(trilerp_b<4>(f, c, ix, iy, iz), w);
#endif
  }
}

// --------------------------------------------------------------------------------- one proposal round, per lane
// RaySamples.get_weights (cameras/rays.py:188-210) with the sequential cumsum of the reference, then PDFSampler
// (ray_samplers.py:309-361) as a merge walk over (cdf, u).  EdgeFn(i) = i-th spacing edge of the current level.
struct LaneRoundIO {
  int S, S_new;
  const float* u_tab;
  float* bins_out;  // this lane's column of the new edges: element i at bins_out[i * bins_stride]
  int64_t bins_stride;
  float* tr_w;
  int32_t* tr_aid;
  float* tr_bins_s;
  float* tr_bins_e;
  int32_t* tr_inds;
};
// `bins_in` == nullptr: level-0 edges torch.linspace(0, 1, S+1); else the scratch column written by the previous round.
// `e_tab`: the round's S+1 euclidean edges when they are the same for every ray (round 0 without per-ray nears / fars),
// else nullptr.  TRACED = false: no trace pointer is set (the io.tr_* tests are not compiled in).
template <int LAYOUT = 0, bool ACTORS = true, bool TRACED = true>
NFF_D float lane_proposal_round(const RenderParams& P, const FieldGrids& fg, const LaneScratch& sc, int tid, int n_cand,
                                const LaneRoundIO& io, const float* bins_in, const float* e_tab, const float o[3],
                                const float d[3], float area, float s_near, float s_far, int64_t ray) {
  const Sampling& sp = P.samp;
  const int S = io.S, S_new = io.S_new;
  auto edge = [bins_in, S](int i) { return bins_in ? bins_in[(size_t)i * kLaneThreads] : linspace01(i, S); };
  auto euclid = [&](int i) { return e_tab ? e_tab[i] : to_euclid(edge(i), s_near, s_far, sp); };
  // running sums are kept in double: torch's CPU cumsum/cumprod (the oracle) accumulate in double
  // (acc_type<float, false>) and round per element; a sequential fp32 sum of 128 terms would be ~20x noisier
  double excl = 0.0, tot_d = 0.0;
  float depth_acc = 0.0f;
  float e_prev = euclid(0);
#pragma unroll 1
  for (int s = 0; s < S; ++s) {
    const float T = expf(-(float)excl);
    // Exact early termination: once exp(-sum) has underflowed to 0 it stays 0 (the sum only grows), so every later
    // weight of this round is exactly 0 whatever the density is (nan_to_num(x * 0) == 0) -- the gathers are skipped
    // when that holds for all 32 rays of the warp.  Not taken when per-sample actor ids are being traced.
    float w = 0.0f;
    if (!(vote_all_converged(T == 0.0f) && (!TRACED || io.tr_aid == nullptr))) {
      const float e0 = e_prev;
      const float e1 = euclid(s + 1);
      e_prev = e1;
      Gauss g = sample_gaussian(o, d, area, e0, e1);
      int aid;
      float dens = lane_proposal_density<LAYOUT, ACTORS>(fg, sc, tid, n_cand, g, &aid);
      float dd = fmul(fsub(e1, e0), dens);
      float alpha = fsub(1.0f, expf(-dd));
      excl += (double)dd;  // torch.cumsum order
      w = nan_to_num(fmul(alpha, T));
      depth_acc = fadd(depth_acc, fmul(w, fmul(fadd(e0, e1), 0.5f)));
      if (TRACED && io.tr_aid) io.tr_aid[ray * S + s] = aid;
    }
    if (TRACED && io.tr_w) io.tr_w[ray * S + s] = w;
    w = fadd(w, sp.hist_pad);
    sc.w[(size_t)s * kLaneThreads + tid] = w;
    tot_d += (double)w;
  }
  float tot = (float)tot_d;
  const float padding = fmaxf(fsub(1e-5f, tot), 0.0f);
  const float pad_each = fdiv(padding, (float)S);
  tot = fadd(tot, padding);
  // merge walk: k = number of cdf entries (cdf[0] = 0, cdf[j] = min(1, sum_{m<j} pdf_m)) that are <= u
  int k = 1;
  double run = (double)fdiv(fadd(sc.w[tid], pad_each), tot);  // unclamped cumsum up to index k
  float c_km1 = 0.0f, c_k = fminf(1.0f, (float)run);
  float w_next = sc.w[(size_t)kLaneThreads + tid];  // weight k, loaded one step ahead of the dependent compare
#pragma unroll 1
  for (int i = 0; i <= S_new; ++i) {
    const float u = ldg(io.u_tab + i);
    while (k <= S && c_k <= u) {
      ++k;
      c_km1 = c_k;
      if (k <= S) {
        const float wk = w_next;
        w_next = sc.w[(size_t)(k < S ? k : S - 1) * kLaneThreads + tid];
        run += (double)fdiv(fadd(wk, pad_each), tot);
        c_k = fminf(1.0f, (float)run);
      }
    }
    const int above = k > S ? S : k;
    const float b0 = edge(k - 1), b1 = edge(above);
    float t = nan_to_num(fdiv(fsub(u, c_km1), fsub(k > S ? c_km1 : c_k, c_km1)));
    t = fminf(fmaxf(t, 0.0f), 1.0f);
    const float nb = fadd(b0, fmul(t, fsub(b1, b0)));
    io.bins_out[(size_t)i * io.bins_stride] = nb;
    if (TRACED && io.tr_inds) io.tr_inds[ray * (S_new + 1) + i] = k;
    if (TRACED && io.tr_bins_s) io.tr_bins_s[ray * (S_new + 1) + i] = nb;
    if (TRACED && io.tr_bins_e) io.tr_bins_e[ray * (S_new + 1) + i] = to_euclid(nb, s_near, s_far, sp);
  }
  return depth_acc;
}

// ------------------------------------------------------------------------------------------- MLP policies, per lane
// Input: the 32 grid features of this lane's sample in registers, kAScale times the features (the grid encoders write
// the panel at that scale); the direction's SH encoding from the last set_dir.  CUDA-core version (host emulation / fp32
// mode):
struct MlpLaneFfma {
  static constexpr int kPitch = kLaneThreads;  // panel row pitch (floats)
  static constexpr float kAScale = 1.0f;
  const float* w;  // packed transposed weights (nff_params.h)
  float* panel_;   // [kNff][kLaneThreads]
  int sh_tcnn = 0;  // 1: tiny-cuda-nn's SphericalHarmonics convention (nff_device.h: sh4_tcnn)
  float sh_[kSh] = {};
  NFF_D float* panel() const { return panel_; }
  NFF_D void set_dir(const float dir[3], int /*tid*/) {
    if (sh_tcnn) sh4_tcnn(dir[0], dir[1], dir[2], sh_); else sh4(dir[0], dir[1], dir[2], sh_);
  }
  NFF_D void run(const float* x, float& sdf, float* feat, int /*tid*/) const {
    float h[kHidden], go[kNff + 1], in2[kNff + kSh], h2[kHidden];
    dense<kGeoIn, kHidden, kHidden, true>(w + kOffGeoW0, w + kOffGeoB0, x, h);
    dense<kHidden, kNff + 1, kGeoOutP, false>(w + kOffGeoW1, w + kOffGeoB1, h, go);
    sdf = go[0];
#pragma unroll
    for (int i = 0; i < kNff; ++i) in2[i] = go[i + 1];
#pragma unroll
    for (int i = 0; i < kSh; ++i) in2[kNff + i] = sh_[i];
    dense<kNff + kSh, kHidden, kHidden, true>(w + kOffFeatW0, w + kOffFeatB0, in2, h);
    dense<kHidden, kHidden, kHidden, true>(w + kOffFeatW1, w + kOffFeatB1, h, h2);
    dense<kHidden, kNff, kNff, false>(w + kOffFeatW2, w + kOffFeatB2, h2, h);
#pragma unroll
    for (int i = 0; i < kNff; ++i) feat[i] = in2[i] + h[i];
  }
};

#if defined(__CUDACC__)
// Tensor-core version: the tile is the 128 rays of a warp group at this sample index, run as two independent m64 halves
// (tile rows 64h..64h+63) that each go through all five layers with every activation in wgmma fragment registers:
//   * every layer is m64n32k16 wgmma on fp16 operands with fp32 accumulators.  fp32 accuracy comes from the split
//         a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo        (hi = x rounded to fp16, lo = x - hi rounded to fp16)
//     three wgmma per k16 step (DESIGN section 4 bounds it);
//   * the operands are scaled by powers of two to sit inside fp16's range: A by 2^kLaneTcA, layer l's B by 2^e_l, chosen
//     from the layer's largest weight when the tiles are staged.  Each layer's first wgmma starts its accumulators at zero
//     (scale-d = 0); after the wait one FMA per accumulator scales the products back exactly (by 2^-e_l) and adds the bias
//     times 2^kLaneTcA, so the next layer's A is 2^kLaneTcA times the activation;
//   * layer 0 loads its A fragments straight from the grid-feature panel (rows 0..31; a row pitch of 4 mod 32 banks keeps
//     those loads free of bank conflicts).  Layer 2's K columns 32..47, the SH encoding of the direction, come from panel
//     rows 32..47, which the row owner writes (set_dir) before the group barrier.  The writers store both already times
//     2^kLaneTcA (kAScale), so the fragments are the A operands as loaded;
//   * layers 1-4 take the previous layer's accumulator registers as their A operand: the fp32 accumulator fragment of an
//     m64nN wgmma (rows g / g+8, columns 8j+2t, +1) is the register A fragment of an f16 k16 step, pair by pair;
//   * layer 4's products are scaled by 2^-(kLaneTcA + e_4) in the same FMA that adds bias + geo_embedding (the
//     residual).  geo_embedding waits in the panel at the thread's own fragment positions (rows 0..31, consumed by layer 0)
//     while layers 2-3 run;
//   * the sdf neuron is a dot product of layer 0's fragments: 8 terms per thread, then a reduction over the quad;
//   * one commit and one wait per layer and half: 10 waits per sample;
//   * an A operand at or beyond fp16's overflow threshold would turn into inf inside the product: each layer checks the
//     largest of its packed fp16 hi words and raises P.status (kLaneTcRangeStatus) instead.
// The outputs (feature c of tile row R at panel[c][R], sdf at panel[48][R]) reach the row owner behind the second and
// last group barrier of the sample.  Panel positions of a tile row are only ever read and written as fragments by the
// warp whose fragments hold that row, and by the row owner on the far side of a barrier.
constexpr int kLanePanelPitch = kLaneThreads + 4;
constexpr int kLanePanelRows = kGeoIn + kSh + 1;  // grid features | SH | sdf
constexpr int kLaneTcA = 6;                       // A operands are 2^6 times the activations: |x| < 1023.75 stays finite
constexpr float kLaneTcAScale = 64.0f, kLaneTcAUnscale = 1.0f / 64.0f;
constexpr float kLaneTcOverflow = 65520.0f;       // the smallest fp32 value that rounds to inf in fp16
constexpr int kLaneTcRangeStatus = 4;             // P.status code: an MLP activation beyond the fp16 operand range
struct LaneTcShared {
  __half b[2 * 32 * (32 + 32 + 48 + 32 + 32)];  // hi|lo fp16 B tiles of the 5 layers, layer l times 2^e_l (22 KiB)
  // bias and w_sdf are read as float2 fragments (8-byte aligned)
  alignas(8) float bias[kTcLayers][32];          // layers 0-3 times 2^kLaneTcA; layer 4 as it is (added to its output)
  float down[kTcLayers];                         // 2^-e_l
  alignas(8) float w_sdf[32];
  float b_sdf;
  unsigned wmax[kTcLayers];                      // staging: the bits of the largest |weight| of each layer
};
constexpr int kLaneTcBytes = (sizeof(LaneTcShared) + 127) / 128 * 128;
constexpr size_t lane_tc_smem_bytes() { return (size_t)kLaneTcBytes + sizeof(float) * kLanePanelRows * kLanePanelPitch; }

// cooperative (whole CTA, which it synchronises once): B tiles, scales and biases from the nn.Linear-layout weights.
// e_l = 15 - (exponent of the layer's largest |weight|, frexp convention): the scaled weights stay below 2^15.
NFF_D void lane_tc_stage_weights(LaneTcShared& t, const float* NFF_RESTRICT nn, int tid, int nthreads) {
  if (tid < kTcLayers) t.wmax[tid] = 0u;
  __syncthreads();
#pragma unroll
  for (int l = 0; l < kTcLayers; ++l) {
    unsigned m = 0u;
    for (int i = tid; i < 32 * tc_layer_k(l); i += nthreads) m = max(m, __float_as_uint(fabsf(nn[tc_layer_w(l) + i])));
    m = __reduce_max_sync(0xffffffffu, m);
    if ((tid & 31) == 0 && m) atomicMax(&t.wmax[l], m);
  }
  __syncthreads();
#pragma unroll
  for (int l = 0; l < kTcLayers; ++l) {
    int E;
    frexpf(__uint_as_float(t.wmax[l]), &E);
    const int e = min(max(15 - E, -60), 60);
    const float up = __int_as_float((127 + e) << 23), down = __int_as_float((127 - e) << 23);
    const int K = tc_layer_k(l);
    __half* hi = t.b + tc_layer_off(l);
    tc::stage_b_tile_f16(hi, hi + 32 * K, nn + tc_layer_w(l), K, up, tid, nthreads);
    for (int i = tid; i < 32; i += nthreads) t.bias[l][i] = nn[tc_layer_b(l) + i] * (l < kTcLayers - 1 ? kLaneTcAScale : 1.0f);
    if (tid == 0) t.down[l] = down;
  }
  for (int i = tid; i < 32; i += nthreads) t.w_sdf[i] = nn[kNnGeoW1 + i];
  if (tid == 0) t.b_sdf = nn[kNnGeoB1];
}

struct MlpLaneTc {
  static constexpr int kPitch = kLanePanelPitch;
  static constexpr float kAScale = kLaneTcAScale;  // the panel's grid features and SH are the scaled A operands
  const LaneTcShared* t;  // staged by lane_tc_stage_weights; at the start of dynamic shared memory
  float* panel_;          // [kLanePanelRows][kPitch] shared memory
  int* status;            // RenderParams::status
  int bar_id;             // this warp group's named barrier
  int sh_tcnn = 0;        // 1: tiny-cuda-nn's SphericalHarmonics convention
  NFF_D float* panel() const { return panel_; }
  NFF_D void group_sync() const { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); }

  // Low descriptor word (tc::smem_desc_lo, LBO 128 B) of t->b, taken from the dynamic shared memory symbol rather than
  // from `t`: ptxas then computes it, and every descriptor derived from it, on the uniform datapath.  From the generic
  // pointer it built every descriptor of a half in per-thread registers and moved each into a uniform register pair
  // (DESIGN section 4).
  NFF_D static uint32_t b_desc_lo() {
    extern __shared__ __align__(128) unsigned char nff_lane_smem[];  // = the kernel's dynamic shared memory
    return tc::smem_desc_lo(tc::smem_u32(nff_lane_smem + offsetof(LaneTcShared, b)), 128u);
  }

  // acc (this thread's 16 fragment registers of one m64n32 half) = A * W^T over the KS k16 steps of a layer with K inputs
  // (the first wgmma starts from zero); a = the scaled A operands, 8 per k-step in fragment order; OFF = the half offset in
  // t->b of the layer's hi B tile (lo follows it).  Every descriptor is b_desc_lo() plus a compile-time constant.
  template <int KS, int K, int OFF>
  NFF_D void half_mma(float* acc, const float* a) const {
    uint32_t ah[4 * KS], al[4 * KS];
    // Range check on the packed hi words: with round-to-nearest-even rn16(x) is inf exactly when |x| >= kLaneTcOverflow.
    // __hmax2 returns the other operand where one is NaN, so a NaN operand does not raise the status (as fmaxf did not).
    __half2 amax = __float2half2_rn(0.0f);
#pragma unroll
    for (int i = 0; i < 4 * KS; ++i) {
      tc::f16x2_split(a[2 * i], a[2 * i + 1], ah[i], al[i]);
      amax = __hmax2(amax, __habs2(*reinterpret_cast<const __half2*>(&ah[i])));
    }
    if (__hge2_mask(amax, __half2half2(__ushort_as_half((unsigned short)0x7c00u))) != 0u && status)  // either half is inf
      atomicExch(status, kLaneTcRangeStatus);
    constexpr uint32_t sbo = (uint32_t)(K / 8) * 128u;  // (K / 8) core matrices of 128 B per 8-row n block
    constexpr uint32_t hi_off = (uint32_t)OFF * 2u / 16u, lo_off = (uint32_t)(OFF + 32 * K) * 2u / 16u;
    const uint32_t b_desc = b_desc_lo();
    tc::wg_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint32_t adv = (uint32_t)(ks * 2 * 128) / 16u;  // two 16-byte K-chunks per k-step
      const uint64_t dh = tc::smem_desc_of(b_desc + hi_off + adv, sbo), dl = tc::smem_desc_of(b_desc + lo_off + adv, sbo);
      if (ks == 0) tc::wgmma_f16_m64n32_zero(acc, ah, dh);
      else tc::wgmma_f16_m64n32(acc, ah + 4 * ks, dh);
      tc::wgmma_f16_m64n32(acc, al + 4 * ks, dh);
      tc::wgmma_f16_m64n32(acc, ah + 4 * ks, dl);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    // the accumulators are read, and the operand registers may be reused, only after the wait
    tc::reg_fence(acc, 16);
#pragma unroll
    for (int i = 0; i < 4 * KS; ++i) asm volatile("" : "+r"(ah[i]), "+r"(al[i])::"memory");
  }
  // scaled A operands of k16 steps [ks0, ks0 + n) from panel rows 16 ks0 .. (p = the panel at this thread's fragment row g)
  NFF_D static void load_a(float* a, const float* p, int q, int ks0, int n) {
#pragma unroll
    for (int i = 0; i < n; ++i) {
      const float* r = p + (16 * (ks0 + i) + 2 * q) * kPitch;
      a[8 * i + 0] = r[0];
      a[8 * i + 1] = r[kPitch];
      a[8 * i + 2] = r[8];
      a[8 * i + 3] = r[kPitch + 8];
      a[8 * i + 4] = r[8 * kPitch];
      a[8 * i + 5] = r[9 * kPitch];
      a[8 * i + 6] = r[8 * kPitch + 8];
      a[8 * i + 7] = r[9 * kPitch + 8];
    }
  }
  // accumulators times 2^-e_l (exact) plus 2^kLaneTcA times the bias: 2^kLaneTcA times the layer's output
  NFF_D static void rescale_bias(float* acc, float down, const float* bias, int q) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 b = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q);
      acc[4 * j + 0] = fmaf(acc[4 * j + 0], down, b.x);
      acc[4 * j + 1] = fmaf(acc[4 * j + 1], down, b.y);
      acc[4 * j + 2] = fmaf(acc[4 * j + 2], down, b.x);
      acc[4 * j + 3] = fmaf(acc[4 * j + 3], down, b.y);
    }
  }
  NFF_D static void relu(float* acc) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fmaxf(acc[i], 0.0f);
  }

  // SH encoding of the shading direction, times 2^kLaneTcA, into panel rows 32..47 of this thread's column.  Only layer 2's
  // fragment loads read those rows, and nothing else writes them: the next run's first group barrier orders the writes.
  NFF_D void set_dir(const float dir[3], int tid) const {
    float shv[kSh];
    if (sh_tcnn) sh4_tcnn(dir[0], dir[1], dir[2], shv); else sh4(dir[0], dir[1], dir[2], shv);
    float* col = panel_ + tid;
#pragma unroll
    for (int i = 0; i < kSh; ++i) col[(kGeoIn + i) * kPitch] = shv[i] * kLaneTcAScale;
  }

  NFF_D void run(const float* /* x: read as fragments from the panel */, float& sdf, float* feat, int tid) {
    float* col = panel_ + tid;
    group_sync();  // all 128 panel columns of the group are in
    const int ln = tid & 31, q = ln & 3;
    // accumulator fragment (row g (+8), columns 8j + 2q (+1)) of tile row 64h + 16 warp + g: panel column fr + 64 h
    float* const fr = panel_ + (tid & ~127) + 16 * ((tid >> 5) & 3) + (ln >> 2);
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      float* const p = fr + 64 * h;
      float a[24], acc[16];
      // layer 0: grid features -> hidden, ReLU, sdf
      load_a(a, p, q, 0, 2);
      half_mma<2, 32, tc_layer_off(0)>(acc, a);
      rescale_bias(acc, t->down[0], t->bias[0], q);
      relu(acc);
      float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 w = *reinterpret_cast<const float2*>(t->w_sdf + 8 * j + 2 * q);
        s0 = fmaf(acc[4 * j + 0], w.x, fmaf(acc[4 * j + 1], w.y, s0));
        s1 = fmaf(acc[4 * j + 2], w.x, fmaf(acc[4 * j + 3], w.y, s1));
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      if (q == 0) {  // the sums of the scaled activations are exactly 2^kLaneTcA times those of the activations
        p[(kGeoIn + kSh) * kPitch] = s0 * kLaneTcAUnscale + t->b_sdf;
        p[(kGeoIn + kSh) * kPitch + 8] = s1 * kLaneTcAUnscale + t->b_sdf;
      }
      // layer 1: -> geo_embedding (scaled), parked at this thread's fragment positions of panel rows 0..31
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] = acc[i];
      half_mma<2, 32, tc_layer_off(1)>(acc, a);
      rescale_bias(acc, t->down[1], t->bias[1], q);
      __syncwarp();  // the warp's layer-0 fragment loads of these rows are done
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float* r = p + (8 * j + 2 * q) * kPitch;
        r[0] = acc[4 * j + 0], r[kPitch] = acc[4 * j + 1], r[8] = acc[4 * j + 2], r[kPitch + 8] = acc[4 * j + 3];
      }
      // layer 2: [geo_embedding | SH] -> hidden, ReLU
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] = acc[i];
      load_a(a + 16, p, q, 2, 1);
      half_mma<3, 48, tc_layer_off(2)>(acc, a);
      rescale_bias(acc, t->down[2], t->bias[2], q);
      relu(acc);
      // layer 3: hidden -> hidden, ReLU
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] = acc[i];
      half_mma<2, 32, tc_layer_off(3)>(acc, a);
      rescale_bias(acc, t->down[3], t->bias[3], q);
      relu(acc);
      // layer 4: hidden -> features, products times 2^-(kLaneTcA + e_4) plus bias + geo_embedding; out to the same positions
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] = acc[i];
      half_mma<2, 32, tc_layer_off(4)>(acc, a);
      const float out4 = t->down[4] * kLaneTcAUnscale;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float* r = p + (8 * j + 2 * q) * kPitch;
        const float2 b = *reinterpret_cast<const float2*>(t->bias[4] + 8 * j + 2 * q);
        r[0] = fmaf(acc[4 * j + 0], out4, fmaf(r[0], kLaneTcAUnscale, b.x));
        r[kPitch] = fmaf(acc[4 * j + 1], out4, fmaf(r[kPitch], kLaneTcAUnscale, b.y));
        r[8] = fmaf(acc[4 * j + 2], out4, fmaf(r[8], kLaneTcAUnscale, b.x));
        r[kPitch + 8] = fmaf(acc[4 * j + 3], out4, fmaf(r[kPitch + 8], kLaneTcAUnscale, b.y));
      }
    }
    group_sync();  // every tile row's outputs are in
#pragma unroll
    for (int i = 0; i < kNff; ++i) feat[i] = col[i * kPitch];
    sdf = col[(kGeoIn + kSh) * kPitch];
  }
};
#endif

// --------------------------------------------------------------------------------------------- the whole ray
// NeuRADModel.get_nff_outputs (models/neurad.py:368-421), eval mode, for the ray owned by this lane.
// Per-ray constants shared by the sampling and the shading stage.
struct LaneRay {
  float o[3], d[3];
  float area, time, s_near, s_far;
  int n_cand;
};
// spacing-domain near / far of a ray (_get_ray_samples, neurad.py:443-449); rays without nears / fars use the defaults
constexpr float kDefaultNear = 0.0f, kDefaultFar = 1.0e6f;
NFF_D void lane_spacing_bounds(const Sampling& sp, float near_, float far_, float* s_near, float* s_far) {
  *s_near = spacing_fn(near_, sp);
  *s_far = spacing_fn(fminf(far_, sp.sky_distance), sp);
}
// Round 0's euclidean edge i (0 <= i <= kS0) of a bundle without nears / fars: the same for every ray, so the sampling kernel
// computes the kS0+1 of them once per CTA instead of once per ray and sample.
NFF_D float lane_round0_edge(const Sampling& sp, int i) {
  float s_near, s_far;
  lane_spacing_bounds(sp, kDefaultNear, kDefaultFar, &s_near, &s_far);
  return to_euclid(linspace01(i, kS0), s_near, s_far, sp);
}
template <bool ACTORS = true, bool EDIT = false>
NFF_D LaneRay lane_ray_setup(const RenderParams& P, const LaneScratch& sc, int tid, int64_t ray) {
  const Sampling& sp = P.samp;
  LaneRay R;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    R.o[i] = ldg(P.rays.origins + 3 * ray + i);
    R.d[i] = ldg(P.rays.directions + 3 * ray + i);
  }
  const bool lidar = P.rays.is_lidar ? P.rays.is_lidar[ray] != 0 : false;
  R.area = fmul(ldg(P.rays.pixel_area + ray), lidar ? 1.0f : sp.cam_area_scale);  // _scale_pixel_area (neurad.py:702-709)
  R.time = ldg(P.rays.times + ray);
  const float far_ = P.rays.fars ? ldg(P.rays.fars + ray) : kDefaultFar;
  const float near_ = P.rays.nears ? ldg(P.rays.nears + ray) : kDefaultNear;
  lane_spacing_bounds(sp, near_, far_, &R.s_near, &R.s_far);
  int overflow = 0;
  R.n_cand = ACTORS ? lane_actor_candidates<EDIT>(P.actors, R.time, R.o, R.d, sc, tid, &overflow) : 0;
#if defined(__CUDACC__)
  if (overflow && P.status) atomicExch(P.status, 3);
#endif
  return R;
}

// Sampling stage: both proposal rounds (ProposalNetworkSampler.generate_ray_samples, ray_samplers.py:623-666).  The
// final spacing edges go to this lane's column `bins2` (element i at bins2[i * bins2_stride]); prop depths to P.out.
// `e0_tab`: round 0's kS0+1 euclidean edges (lane_round0_edge) when the bundle has no per-ray nears / fars, else nullptr.
template <int LAYOUT = 0, bool ACTORS = true, bool TRACED = true>
NFF_D void sample_ray_lane(const RenderParams& P, const LaneScratch& sc, const LaneRay& R, int tid, int64_t ray, bool active,
                           float* bins2, int64_t bins2_stride, const float* e0_tab = nullptr) {
  const Sampling& sp = P.samp;
#pragma unroll 1
  for (int rd = 0; rd < 2; ++rd) {  // one copy of the round's code for both rounds (instruction-cache footprint)
    LaneRoundIO io{};
    io.S = rd == 0 ? kS0 : kS1;
    io.S_new = rd == 0 ? kS1 : kS2;
    io.u_tab = rd == 0 ? sp.u1 : sp.u2;
    io.bins_out = rd == 0 ? sc.bins1 + tid : bins2;
    io.bins_stride = rd == 0 ? (int64_t)kLaneThreads : bins2_stride;
    if (TRACED) {
      io.tr_w = !active ? nullptr : rd == 0 ? P.trace.prop_weights_0 : P.trace.prop_weights_1;
      io.tr_aid = !active ? nullptr : rd == 0 ? P.trace.actor_id_0 : P.trace.actor_id_1;
      io.tr_bins_s = !active ? nullptr : rd == 0 ? P.trace.bins_s_1 : P.trace.bins_s_2;
      io.tr_bins_e = !active ? nullptr : rd == 0 ? P.trace.bins_e_1 : P.trace.bins_e_2;
      io.tr_inds = !active ? nullptr : rd == 0 ? P.trace.inds_1 : P.trace.inds_2;
    }
    const float prop_depth = lane_proposal_round<LAYOUT, ACTORS, TRACED>(
        P, P.fields[sp.field_of_round[rd]], sc, tid, R.n_cand, io, rd == 0 ? nullptr : sc.bins1 + tid,
        rd == 0 ? e0_tab : nullptr, R.o, R.d, R.area, R.s_near, R.s_far, ray);
    // stored per round: a [2] array indexed by the rolled round counter would live in local memory
    if (active) (rd == 0 ? P.out.prop_depth_0 : P.out.prop_depth_1)[ray] = prop_depth;
  }
}

// Shading stage: main field on the 32 resampled intervals + compositing + outputs (neurad.py:368-401).
// ACTORS = false: the scene has no actors (n_cand == 0).  The actor path is not compiled in, and the shading direction is
// the ray's own for every sample, so its SH encoding is set once per ray.
template <class Mlp, int LAYOUT = 0, bool ACTORS = true>
NFF_D void shade_ray_lane(const RenderParams& P, const LaneScratch& sc, const LaneRay& R, Mlp& mlp, int tid, int64_t ray,
                          bool active, const float* bins2, int64_t bins2_stride) {
  const Sampling& sp = P.samp;
  const float* o = R.o;
  const float* d = R.d;
  const float area = R.area, time = R.time, s_near = R.s_near, s_far = R.s_far;
  const int n_cand = R.n_cand;

  // ---- main field: loop over the 32 samples of this ray (fields/neurad_field.py:128-152 + compositing) ----
  const FieldGrids& fm = P.fields[B200NERF_FIELD_MAIN];
  float fsum[kNff];
#pragma unroll
  for (int i = 0; i < kNff; ++i) fsum[i] = 0.0f;
  double T_d = 1.0;
  float acc = 0.0f, depth = 0.0f;
  float e_prev = to_euclid(bins2[0], s_near, s_far, sp);
  if (!ACTORS) mlp.set_dir(d, tid);
#pragma unroll 1
  for (int s = 0; s < kS2; ++s) {
    const float e0 = e_prev;
    float e1 = to_euclid(bins2[(size_t)(s + 1) * bins2_stride], s_near, s_far, sp);
    e_prev = e1;
    if (s == kS2 - 1) e1 = fadd(e1, fsub(sp.sky_distance, e1));  // sky sample (neurad.py:451-455)
    Gauss g = sample_gaussian(o, d, area, e0, e1);
    float* col = mlp.panel() + tid;  // this thread's column of the [32][Mlp::kPitch] shared panel
    int aid = -1;
    {
      float dir[3] = {d[0], d[1], d[2]};
      float pb[3], M[12];
      if (ACTORS && n_cand > 0) aid = lane_actor_of_sample(sc, tid, n_cand, g, pb, M);
      if (aid >= 0) {
        Gauss ga = {pb[0], pb[1], pb[2], g.std};
        ga = contract(ga, fm.actor_scale);
#pragma unroll
        for (int i = 16; i < 32; ++i) col[i * Mlp::kPitch] = 0.0f;  // F.pad(actor_features, (0, 32-16))
        if (LAYOUT == 1) {
          const float x4[4] = {ga.x, ga.y, ga.z, fdiv((float)aid, fm.n_actors_f)};
          tcnn_encode_f4<4>(fm.act, 4, x4, ga.std, col, Mlp::kPitch, Mlp::kAScale);
        } else {
          encode_f4_col(fm.actor_tables[aid], fm.act, 4, ga, col, Mlp::kPitch, Mlp::kAScale);
        }
        float q0 = fadd(fadd(fmul(M[0], d[0]), fmul(M[1], d[1])), fmul(M[2], d[2]));
        float q1 = fadd(fadd(fmul(M[4], d[0]), fmul(M[5], d[1])), fmul(M[6], d[2]));
        float q2 = fadd(fadd(fmul(M[8], d[0]), fmul(M[9], d[1])), fmul(M[10], d[2]));
        float n = fadd(fsqrt(fadd(fadd(fmul(q0, q0), fmul(q1, q1)), fmul(q2, q2))), 1.0e-7f);
        dir[0] = fdiv(q0, n); dir[1] = fdiv(q1, n); dir[2] = fdiv(q2, n);
      } else {
        Gauss gs = contract(g, fm.static_scale);
        if (LAYOUT == 1) {
          const float x3[3] = {gs.x, gs.y, gs.z};
          tcnn_encode_f4<3>(fm.stat, 8, x3, gs.std, col, Mlp::kPitch, Mlp::kAScale);
        } else {
          encode_f4_col(fm.stat.table, fm.stat, 8, gs, col, Mlp::kPitch, Mlp::kAScale);
        }
      }
      if (ACTORS) mlp.set_dir(dir, tid);
    }
    float x[kGeoIn];
#pragma unroll
    for (int i = 0; i < kGeoIn; ++i) x[i] = col[i * Mlp::kPitch];
    float sdf, feat[kNff];
    mlp.run(x, sdf, feat, tid);
    const float alpha = frcp(fadd(1.0f, expf(fmul(sdf, P.beta))));
    float w = fmul(alpha, (float)T_d);  // nerfacc.render_weight_from_alpha, torch.cumprod order
    T_d *= (double)fsub(1.0f, alpha);
    acc = fadd(acc, w);
    if (s < kS2 - 1) depth = fadd(depth, fmul(w, fmul(fadd(e0, e1), 0.5f)));
    if (s == kS2 - 1) w = fadd(fadd(w, 1.0f), -acc);  // remaining accumulation onto the sky sample (neurad.py:381)
#pragma unroll
    for (int i = 0; i < kNff; ++i) fsum[i] = fmaf(feat[i], w, fsum[i]);
    if (active) {
      if (P.trace.sdf) P.trace.sdf[ray * kS2 + s] = sdf;
      if (P.trace.alpha) P.trace.alpha[ray * kS2 + s] = alpha;
      if (P.trace.weights) P.trace.weights[ray * kS2 + s] = w;
      if (P.trace.actor_id_main) P.trace.actor_id_main[ray * kS2 + s] = aid;
      if (P.trace.field_feature) {
#pragma unroll
        for (int i = 0; i < kNff; ++i) P.trace.field_feature[(ray * kS2 + s) * kNff + i] = feat[i];
      }
    }
  }
  // ---- outputs ----
  const int fdim = P.nff_dim + P.app.dim;
  float app[kApp];
#pragma unroll
  for (int i = 0; i < kApp; ++i) app[i] = 0.0f;
  if (P.app.dim > 0) {  // _get_appearance_embedding (neurad.py:423-441)
    // eps == 0: the per-sensor branch (:440), row `sensor_idx` copied; otherwise the temporal branch (:430-439)
    const bool per_sensor = P.app.eps == 0;
    float sens = P.rays.sensor_idx ? (float)P.rays.sensor_idx[ray] : 0.0f;
    float eps_ = (float)P.app.eps;
    float tidx = fmul(fdiv(time, P.app.duration), eps_);
    float before = fminf(fmaxf(floorf(tidx), 0.0f), eps_ - 1.0f);
    float after = fminf(fmaxf(fadd(before, 1.0f), 0.0f), eps_ - 1.0f);
    float ratio = fsub(tidx, before);
    int ib = (int)fadd(before, fmul(sens, eps_)), ia = (int)fadd(after, fmul(sens, eps_));
    if (per_sensor) ib = ia = (int)sens;
#pragma unroll
    for (int i = 0; i < kApp; ++i) {
      if (i < P.app.dim) {
        float eb = ldg(P.app.emb + (size_t)ib * P.app.dim + i), ea = ldg(P.app.emb + (size_t)ia * P.app.dim + i);
        app[i] = per_sensor ? eb : fadd(fmul(eb, fsub(1.0f, ratio)), fmul(ea, ratio));
      }
    }
  }
#if defined(__CUDACC__)
  if (fdim == kNff + kApp) {
    // Coalesced feature rows.  The 8 lanes 8g..8g+7 of a warp own 8 CONSECUTIVE rays (an image-row segment of the
    // 8x4 patch, or 8 flat neighbours), i.e. 8*48 floats = 1536 contiguous bytes of the output.  Each segment is
    // staged through the warp's slice of the shared panel and written with three fully coalesced 512-byte STG.128
    // instructions -- to the local buffer and, for the fused multi-GPU gather, to every peer's buffer over NVLink
    // (st.global on peer-mapped addresses; small scattered remote writes are what made the naive version slow).
    const int ln = tid & 31;
    float* slice = mlp.panel() + (tid & ~31);  // rows 0..11 (stride Mlp::kPitch) x 32 columns of this warp
    const unsigned act_mask = __ballot_sync(0xffffffffu, active);
#pragma unroll 1
    for (int g = 0; g < 4; ++g) {
      __syncwarp();
      if ((ln >> 3) == g) {
        const int r = ln & 7;
#pragma unroll
        for (int j = 0; j < kNff; ++j) {
          const int slot = r * (kNff + kApp) + j;
          slice[(slot >> 5) * Mlp::kPitch + (slot & 31)] = fsum[j];
        }
#pragma unroll
        for (int j = 0; j < kApp; ++j) {
          const int slot = r * (kNff + kApp) + kNff + j;
          slice[(slot >> 5) * Mlp::kPitch + (slot & 31)] = app[j];
        }
      }
      __syncwarp();
      const int k = __popc((act_mask >> (8 * g)) & 0xffu);  // active rays of the segment form a prefix
      const int64_t ray0 = __shfl_sync(0xffffffffu, ray, 8 * g);
      if (k == 0) continue;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int f = t * 32 + ln;  // float4 index inside the segment's 96 float4
        if (f / 12 < k) {
          const float4 v = *reinterpret_cast<const float4*>(&slice[(f >> 3) * Mlp::kPitch + ((f & 7) << 2)]);
          reinterpret_cast<float4*>(P.out.features + ray0 * fdim)[f] = v;
          for (int p = 0; p < P.peers.n_peers; ++p) {
            if (p == P.peers.self_rank) continue;
            reinterpret_cast<float4*>(P.peers.features[p] + (P.peers.row_offset + ray0) * fdim)[f] = v;
          }
        }
      }
    }
    __syncwarp();
  } else
#endif
  if (active) {
    float* fo = P.out.features + ray * fdim;
#pragma unroll
    for (int i = 0; i < kNff; ++i) fo[i] = fsum[i];
    for (int i = 0; i < P.app.dim; ++i) fo[P.nff_dim + i] = app[i];
  }
  if (!active) return;
  P.out.depth[ray] = depth;
  P.out.accumulation[ray] = acc;
#if defined(__CUDACC__)
  for (int p = 0; p < P.peers.n_peers; ++p) {
    if (p == P.peers.self_rank) continue;
    P.peers.depth[p][P.peers.row_offset + ray] = depth;
    P.peers.accumulation[p][P.peers.row_offset + ray] = acc;
  }
#endif
}

// NeuRADModel.get_nff_outputs (models/neurad.py:368-421), eval mode, for the ray owned by this lane: both stages back to
// back with the resampled edges handed over through the CTA's scratch slab.
template <class Mlp, int LAYOUT = 0, bool EDIT = false>
NFF_D void render_ray_lane(const RenderParams& P, const LaneScratch& sc, Mlp& mlp, int tid, int64_t ray, bool active) {
  const LaneRay R = lane_ray_setup<true, EDIT>(P, sc, tid, ray);
  sample_ray_lane<LAYOUT>(P, sc, R, tid, ray, active, sc.bins2 + tid, kLaneThreads);
  shade_ray_lane<Mlp, LAYOUT>(P, sc, R, mlp, tid, ray, active, sc.bins2 + tid, kLaneThreads);
}

}  // namespace nff
