// nff_modules.h -- device code of the MODULE-LEVEL seams of the reference API (SURVEY.md section 8b: Field, Sampler,
// NeuRADHashEncoding as stand-alone operators) and of their backward operators (SURVEY 8f, row f2).
//
// The fused renderer (nff_lane.h / nff_device.h) never materialises a per-sample tensor; these operators do, because
// the reference's per-module API hands [N,S,...] tensors from one nn.Module to the next.  Everything here is written
// per thread (no warp collectives), so the test-only host emulation (tests/host_emul) can run it as plain loops.
#pragma once

#include "nff_device.h"

namespace nff {

constexpr int kModMaxActors = 64;  // actors per scene the module-level operators accept (frames live in shared memory)
constexpr int kModMaxDim = 64;     // max L*F of a NeuRADHashEncoding output row

// world -> box frame of one actor at one ray's time: [R^T | -R^T t] row major 3x4, padded half extents, validity
struct ActorFrame {
  float w2b[12];
  float bnd[3];
  int32_t valid;
};

// torch.searchsorted(pose_times, t) (left) + the lerp fraction of interpolate_trajectories_6d (utils/poses.py:117-134)
NFF_D void keyframe_bracket(const Actors& A, float time, int& left, int& right, float& frac) {
  int lo = 0, hi = A.n_times;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (ldg(A.times + mid) < time) lo = mid + 1; else hi = mid;
  }
  right = lo;
  left = right - 1 < 0 ? 0 : right - 1;
  if (right > A.n_times - 1) right = A.n_times - 1;
  float tl = ldg(A.times + left), tr = ldg(A.times + right);
  frac = fdiv(fsub(time, tl), fadd(fsub(tr, tl), 1e-6f));
  frac = fminf(fmaxf(frac, 0.0f), 1.0f);
}

// DynamicActors.get_boxes2world (model_components/dynamic_actors.py:251-268) for ONE actor: keyframe lerp of the
// Gram-Schmidt'ed 6-D rotation + position (utils/poses.py:90-150), rotation_6d_to_matrix
// (cameras/camera_utils.py:422-443), pose inverse (utils/poses.py:42-55).  Same op sequence as actor_candidates()
// of the fused kernel, without the ray-line cull (a conservative optimisation there; the in-box test decides).
// EDIT: apply the actor edit (edit_box_pose).  The backward operators use EDIT = false: their gradients are those of
// the unedited poses, the only ones the reference trains.
template <bool EDIT = false>
NFF_D void actor_frame(const Actors& A, int a, int left, int right, float frac, ActorFrame& f) {
  const float* kl = A.keyframes + ((size_t)left * A.n_actors + a) * 9;
  const float* kr = A.keyframes + ((size_t)right * A.n_actors + a) * 9;
  float p[9];
  for (int i = 0; i < 9; ++i) {
    float l_ = ldg(kl + i), r_ = ldg(kr + i);
    p[i] = fadd(l_, fmul(fsub(r_, l_), frac));
  }
  f.valid = (A.present[(size_t)left * A.n_actors + a] | A.present[(size_t)right * A.n_actors + a]) != 0;
  float b1[3] = {p[0], p[1], p[2]};
  normalize3(b1);
  float dt = fadd(fadd(fmul(b1[0], p[3]), fmul(b1[1], p[4])), fmul(b1[2], p[5]));
  float b2[3] = {fsub(p[3], fmul(dt, b1[0])), fsub(p[4], fmul(dt, b1[1])), fsub(p[5], fmul(dt, b1[2]))};
  normalize3(b2);
  float b3[3] = {fsub(fmul(b1[1], b2[2]), fmul(b1[2], b2[1])), fsub(fmul(b1[2], b2[0]), fmul(b1[0], b2[2])),
                 fsub(fmul(b1[0], b2[1]), fmul(b1[1], b2[0]))};
  if (EDIT) edit_box_pose(A, a, b1, b2, b3, p + 6);
  float R[9] = {b1[0], b2[0], b3[0], b1[1], b2[1], b3[1], b1[2], b2[2], b3[2]};
  for (int i = 0; i < 3; ++i) {
    f.w2b[4 * i + 0] = R[3 * i + 0];
    f.w2b[4 * i + 1] = R[3 * i + 1];
    f.w2b[4 * i + 2] = R[3 * i + 2];
    f.w2b[4 * i + 3] = -fadd(fadd(fmul(R[3 * i + 0], p[6]), fmul(R[3 * i + 1], p[7])), fmul(R[3 * i + 2], p[8]));
    f.bnd[i] = ldg(A.bounds + 3 * a + i);
  }
}

// _get_actor_indices, per-sample part (field_components/neurad_encoding.py:241-254): the actor whose padded box
// contains the sample mean (highest index wins = the reference's sequential index_put on CPU), or -1.
NFF_D int actor_containing(const ActorFrame* frames, int n_actors, float x, float y, float z, float pb[3]) {
  int hit = -1;
  for (int a = 0; a < n_actors; ++a) {
    const ActorFrame& f = frames[a];
    if (!f.valid) continue;
    const float* M = f.w2b;
    float q0 = fadd(fadd(fadd(fmul(M[0], x), fmul(M[1], y)), fmul(M[2], z)), M[3]);
    float q1 = fadd(fadd(fadd(fmul(M[4], x), fmul(M[5], y)), fmul(M[6], z)), M[7]);
    float q2 = fadd(fadd(fadd(fmul(M[8], x), fmul(M[9], y)), fmul(M[10], z)), M[11]);
    if (fabsf(q0) < f.bnd[0] && fabsf(q1) < f.bnd[1] && fabsf(q2) < f.bnd[2]) {
      hit = a;
      pb[0] = q0; pb[1] = q1; pb[2] = q2;
    }
  }
  return hit;
}

// HashEncoding.pytorch_fwd + _rescale_grid_features for one contracted gaussian, generic L / F:
// out[l*F + f] = trilerp_l,f * 1/max(1, 2*res_l*std)   (encodings.py:425-466, neurad_encoding.py:297-304).
NFF_D void encode_levels(const float* NFF_RESTRICT table, const Grid& gr, const Gauss& g, float* out) {
  for (int l = 0; l < gr.L; ++l) {
    Cell c = grid_cell(g.x, g.y, g.z, gr.res[l]);
    uint32_t r[8];
    cell_rows(c, gr.mask, r);
    const float* base = table + (size_t)l * gr.T * gr.F;
    const float w = level_weight(gr.res[l], g.std);
    for (int f = 0; f < gr.F; ++f) {
      float v[8];
      for (int k = 0; k < 8; ++k) v[k] = ldg(base + (size_t)r[k] * gr.F + f);
      out[l * gr.F + f] = fmul(trilerp(v, c), w);
    }
  }
}

// NeuRADHashEncoding.forward for one sample (field_components/neurad_encoding.py:150-187): static features, or the
// containing actor's features zero-padded to the static width; the direction goes to the box frame, renormalised
// with +EPS (:203-209).  Returns the actor index or -1.  `feat` must hold fg.stat.L * fg.stat.F floats.  `flip` (+1 / -1 per
// ray) is the training-mode random actor flip, drawn by the caller.
NFF_D int neurad_encode_point(const FieldGrids& fg, const ActorFrame* frames, int n_actors, const Gauss& g,
                              float* feat, float dir[3], float flip = 1.0f) {
  float pb[3];
  const int a = n_actors > 0 ? actor_containing(frames, n_actors, g.x, g.y, g.z, pb) : -1;
  const int D = fg.stat.L * fg.stat.F;
  if (a >= 0) {
    // training-mode actor flip (neurad_encoding.py:212-219): x -> -x in the box frame for the whole ray
    Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    encode_levels(fg.actor_tables[a], fg.act, ga, feat);
    for (int i = fg.act.L * fg.act.F; i < D; ++i) feat[i] = 0.0f;  // F.pad(actor_features, (0, D - Da))
    if (dir) {
      const float* M = frames[a].w2b;
      float q0 = fadd(fadd(fmul(M[0], dir[0]), fmul(M[1], dir[1])), fmul(M[2], dir[2]));
      float q1 = fadd(fadd(fmul(M[4], dir[0]), fmul(M[5], dir[1])), fmul(M[6], dir[2]));
      float q2 = fadd(fadd(fmul(M[8], dir[0]), fmul(M[9], dir[1])), fmul(M[10], dir[2]));
      float n = fadd(fsqrt(fadd(fadd(fmul(q0, q0), fmul(q1, q1)), fmul(q2, q2))), 1.0e-7f);
      dir[0] = fdiv(q0, n); dir[1] = fdiv(q1, n); dir[2] = fdiv(q2, n);
      if (flip < 0.0f) dir[0] = -dir[0];
    }
  } else {
    Gauss gs = contract(g, fg.static_scale);
    encode_levels(fg.stat.table, fg.stat, gs, feat);
  }
  return a;
}

// The same two functions for NeuRAD's shapes (F = 4 or 1 features, at most LMAX levels) with the level loop unrolled, so
// the feature row lives in REGISTERS (the generic versions index a local-memory array) and an F = 4 row is one 16-byte
// load per corner.  Same operations in the same order: bit-identical to encode_levels / neurad_encode_point.  Levels past
// gr.L are written as zeros (the F.pad of an actor sample's row).
template <int LMAX, int F>
NFF_D void encode_levels_t(const float* NFF_RESTRICT table, const Grid& gr, const Gauss& g, float* out /* [LMAX*F] */) {
  static_assert(F == 1 || F == 4, "NeuRAD's feature widths");
#pragma unroll
  for (int l = 0; l < LMAX; ++l) {
    if (l < gr.L) {
      Cell c = grid_cell(g.x, g.y, g.z, gr.res[l]);
      uint32_t r[8];
      cell_rows(c, gr.mask, r);
      const float* base = table + (size_t)l * gr.T * F;
      const float w = level_weight(gr.res[l], g.std);
      if (F == 4) {
        float vx[8], vy[8], vz[8], vw[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 q = ldg(reinterpret_cast<const float4*>(base) + r[k]);
          vx[k] = q.x, vy[k] = q.y, vz[k] = q.z, vw[k] = q.w;
        }
        out[l * F] = fmul(trilerp(vx, c), w);
        out[l * F + (F > 1 ? 1 : 0)] = fmul(trilerp(vy, c), w);
        out[l * F + (F > 2 ? 2 : 0)] = fmul(trilerp(vz, c), w);
        out[l * F + (F > 3 ? 3 : 0)] = fmul(trilerp(vw, c), w);
      } else {
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = ldg(base + r[k]);
        out[l * F] = fmul(trilerp(v, c), w);
      }
    } else {
#pragma unroll
      for (int f = 0; f < F; ++f) out[l * F + f] = 0.0f;
    }
  }
}
template <int LMAX, int F>
NFF_D int neurad_encode_point_t(const FieldGrids& fg, const ActorFrame* frames, int n_actors, const Gauss& g, float* feat /* [LMAX*F] */,
                                float dir[3], float flip = 1.0f) {
  float pb[3];
  const int a = n_actors > 0 ? actor_containing(frames, n_actors, g.x, g.y, g.z, pb) : -1;
  if (a >= 0) {
    Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    encode_levels_t<LMAX, F>(fg.actor_tables[a], fg.act, ga, feat);
    if (dir) {
      const float* M = frames[a].w2b;
      float q0 = fadd(fadd(fmul(M[0], dir[0]), fmul(M[1], dir[1])), fmul(M[2], dir[2]));
      float q1 = fadd(fadd(fmul(M[4], dir[0]), fmul(M[5], dir[1])), fmul(M[6], dir[2]));
      float q2 = fadd(fadd(fmul(M[8], dir[0]), fmul(M[9], dir[1])), fmul(M[10], dir[2]));
      float n = fadd(fsqrt(fadd(fadd(fmul(q0, q0), fmul(q1, q1)), fmul(q2, q2))), 1.0e-7f);
      dir[0] = fdiv(q0, n); dir[1] = fdiv(q1, n); dir[2] = fdiv(q2, n);
      if (flip < 0.0f) dir[0] = -dir[0];
    }
  } else {
    Gauss gs = contract(g, fg.static_scale);
    encode_levels_t<LMAX, F>(fg.stat.table, fg.stat, gs, feat);
  }
  return a;
}

// --------------------------------------------------------------------------------------------- backward pieces
// SURVEY 8f row f2.  Gradients flow to the parameters the reference trains through this path (hash tables, proposal
// density decoders, MLPs, beta); sample positions carry no gradient (PDFSampler detaches its bins,
// ray_samplers.py:363-364; pose / camera optimisation is out of scope for this row).
//
// d(out[l*F+f]) / d(table rows): the trilinear corner weights of `trilerp` times the anti-aliasing weight.  Corner
// order as cell_rows(): ccc, cfc, ffc, fcc, ccf, cff, fff, fcf.
NFF_D void corner_weights(const Cell& c, float w[8]) {
  const float ox = c.ox, oy = c.oy, oz = c.oz, ix = 1.0f - c.ox, iy = 1.0f - c.oy, iz = 1.0f - c.oz;
  w[0] = ox * oy * oz;
  w[1] = ox * iy * oz;
  w[2] = ix * iy * oz;
  w[3] = ix * oy * oz;
  w[4] = ox * oy * iz;
  w[5] = ox * iy * iz;
  w[6] = ix * iy * iz;
  w[7] = ix * oy * iz;
}

// Backward of encode_levels(): grad_table[row*F + f] += dfeat[l*F + f] * level_weight_l * corner_weight_k.  When a
// coordinate is an exact integer ceil == floor and two corners name the same row; both contributions are added,
// like the forward reads the row twice (encodings.py:436-466).
NFF_D void encode_levels_bwd(float* grad_table, const Grid& gr, const Gauss& g, const float* dfeat) {
  for (int l = 0; l < gr.L; ++l) {
    Cell c = grid_cell(g.x, g.y, g.z, gr.res[l]);
    uint32_t r[8];
    cell_rows(c, gr.mask, r);
    float cw[8];
    corner_weights(c, cw);
    float* base = grad_table + (size_t)l * gr.T * gr.F;
    const float w = level_weight(gr.res[l], g.std);
    if (gr.F == 4) {  // NeuRAD's main grids: a row is 16 bytes -> one vector reduction per corner instead of four
      const float g0 = dfeat[4 * l] * w, g1 = dfeat[4 * l + 1] * w, g2 = dfeat[4 * l + 2] * w, g3 = dfeat[4 * l + 3] * w;
      if (g0 == 0.0f && g1 == 0.0f && g2 == 0.0f && g3 == 0.0f) continue;
      for (int k = 0; k < 8; ++k) atomic_add4(base + (size_t)r[k] * 4, g0 * cw[k], g1 * cw[k], g2 * cw[k], g3 * cw[k]);
      continue;
    }
    for (int f = 0; f < gr.F; ++f) {
      const float gs = dfeat[l * gr.F + f] * w;
      if (gs == 0.0f) continue;
      for (int k = 0; k < 8; ++k) atomic_add(base + (size_t)r[k] * gr.F + f, gs * cw[k]);
    }
  }
}

// ---- scatter backward, round 2: registers only + run-length aggregation of the coarse levels ---------------------------
// What bounds the scatter: not instructions and not DRAM but the L2 atomic units of a FEW slices (the busiest
// slice's tag requests run far above the average).  Every ray starts at the
// sensor, so the coarse levels' cells around the sensors receive a reduction from every near-range sample of every ray,
// and same-address reductions serialise in the slice that owns the row.  Consecutive samples of a ray share their coarse
// cells, so a thread that walks a CONTIGUOUS segment of one ray keeps the current cell's 8 corner sums of the first K
// levels in registers and issues the reductions only when the cell changes (flush): the hot rows see one reduction per
// cell crossing instead of one per sample.  Fine levels (and levels whose resolution does not fit the 10-bit cell key) go
// straight to RED.  The first version's other cost is gone as well: the level loop is unrolled over a compile-time bound
// and the upstream gradient is read from its source (the dL/dfeatures row, or decoder weight * g in density mode), so no
// per-sample row lives in local memory, and density mode computes the interpolated feature for the decoder gradient in
// the same pass.
//   grad_table[row] += scale * src[l*F + f] * level_weight_l * corner_weight_k
//   dec_acc[l]      += scale * feature_l                 (F == 1, density mode; feature_l = trilerp * level_weight)
#ifndef NFF_BWD_SEGMENTS
#define NFF_BWD_SEGMENTS 4
#endif
constexpr int kBwdSegments = NFF_BWD_SEGMENTS;  // threads per ray: each walks ceil(S / kBwdSegments) consecutive samples
constexpr uint32_t kAggEmpty = 0xffffffffu;
#ifndef NFF_BWD_PAIR_X
#define NFF_BWD_PAIR_X 1  // F = 1: x-adjacent corners that are adjacent rows share one 8-byte vector reduction
#endif
#ifndef NFF_BWD_PROBE_SKIP
#define NFF_BWD_PROBE_SKIP 0  // MEASUREMENT PROBE ONLY (wrong gradients): drop the scatter of the first n levels to see what they cost
#endif
template <int K, int F>
struct ScatterAgg {
  int tab;                                // table the pending sums belong to: -1 static, >= 0 actor, -2 none yet
  uint32_t key[K > 0 ? K : 1];            // ix | iy << 10 | iz << 20 of the pending cell, per aggregated level
  float acc[K > 0 ? K : 1][8 * F];
};
template <int K, int F>
NFF_D void agg_init(ScatterAgg<K, F>& ag) {
  ag.tab = -2;
#pragma unroll
  for (int l = 0; l < K; ++l) {
    ag.key[l] = kAggEmpty;
#pragma unroll
    for (int j = 0; j < 8 * F; ++j) ag.acc[l][j] = 0.0f;
  }
}
template <int F>
NFF_D void scatter_cell(float* base, const uint32_t r[8], const float* v /* [8*F] corner-major */) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (F == 4) {
      if (!(v[4 * k] == 0.0f && v[4 * k + 1] == 0.0f && v[4 * k + 2] == 0.0f && v[4 * k + 3] == 0.0f))
        atomic_add4(base + (size_t)r[k] * 4, v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    } else if (!NFF_BWD_PAIR_X) {
      if (v[k] != 0.0f) atomic_add(base + r[k], v[k]);
    }
  }
  if (F == 1 && NFF_BWD_PAIR_X) {
    // The x prime of the hash is 1, so the floor-x and ceil-x corners of an edge (same y, z) are rows h ^ ix and
    // h ^ (ix + 1): for even ix they differ in bit 0 only, i.e. they are the two halves of one aligned 8-byte pair and
    // take ONE vector reduction.  What limits this kernel is the number of L2 reduction requests (~85 G/s whether they
    // carry 4 or 16 bytes), and half of all edges qualify.  Corner order (cell_rows): floor-x / ceil-x pairs are
    // (2,1) (3,0) (6,5) (7,4).
    constexpr int kF[4] = {2, 3, 6, 7}, kC[4] = {1, 0, 5, 4};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const uint32_t rf = r[kF[e]], rc = r[kC[e]];
      const float vf = v[kF[e]], vc = v[kC[e]];
      if ((rf ^ rc) == 1u) {
        if (vf != 0.0f || vc != 0.0f) atomic_add2(base + (rf & ~1u), (rf & 1u) ? vc : vf, (rf & 1u) ? vf : vc);
      } else {
        if (vf != 0.0f) atomic_add(base + rf, vf);
        if (vc != 0.0f) atomic_add(base + rc, vc);
      }
    }
  }
}
template <int F>
NFF_D void agg_flush_level(float* base, uint32_t mask, uint32_t& key, float* acc) {
  if (key == kAggEmpty) return;
  const uint32_t ix = key & 1023u, iy = (key >> 10) & 1023u, iz = key >> 20;
  Cell c;  // rows of the cell's 8 vertices (a sample on an exact integer coordinate gave its "ceil" corners weight 0)
  c.hx[0] = ix, c.hx[1] = ix + 1u;
  c.hy[0] = iy * 2654435761u, c.hy[1] = (iy + 1u) * 2654435761u;
  c.hz[0] = iz * 805459861u, c.hz[1] = (iz + 1u) * 805459861u;
  c.ox = c.oy = c.oz = 0.0f;
  uint32_t r[8];
  cell_rows(c, mask, r);
  scatter_cell<F>(base, r, acc);
  key = kAggEmpty;
#pragma unroll
  for (int j = 0; j < 8 * F; ++j) acc[j] = 0.0f;
}
template <int K, int F>
NFF_D void agg_flush_all(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables, ScatterAgg<K, F>& ag) {
  if (K == 0 || ag.tab == -2) return;
  float* gt = ag.tab < 0 ? grad_static : grad_actor_tables[ag.tab];
  const Grid& gr = ag.tab < 0 ? fg.stat : fg.act;
#pragma unroll
  for (int l = 0; l < K; ++l)
    if (gt) agg_flush_level<F>(gt + (size_t)l * gr.T * F, gr.mask, ag.key[l], ag.acc[l]);
}
// one sample against one table (grad_table may be NULL: no table gradient wanted, the decoder gradient still is)
template <int LMAX, int F, bool WANT_DEC, int K>
NFF_D void encode_levels_bwd_t(float* grad_table, const float* NFF_RESTRICT table, const Grid& gr, const Gauss& g,
                               const float* NFF_RESTRICT src, float scale, float* dec_acc /* [LMAX] registers */,
                               ScatterAgg<K, F>& ag) {
  static_assert(F == 1 || F == 4, "NeuRAD's feature widths");
#pragma unroll
  for (int l = 0; l < LMAX; ++l) {
    if (l < gr.L) {
      const float res = gr.res[l];
      Cell c = grid_cell(g.x, g.y, g.z, res);
      uint32_t r[8];
      cell_rows(c, gr.mask, r);
      const float w = level_weight(res, g.std);
      if (WANT_DEC) {
        const float* tb = table + (size_t)l * gr.T;
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = ldg(tb + r[k]);
        dec_acc[l] = fmaf(scale, fmul(trilerp(v, c), w), dec_acc[l]);
      }
      if (grad_table && l >= NFF_BWD_PROBE_SKIP) {
        float gv[F];
        if (F == 4) {
          const float4 d4 = ldg(reinterpret_cast<const float4*>(src) + l);
          gv[0] = scale * d4.x * w, gv[1] = scale * d4.y * w, gv[2] = scale * d4.z * w, gv[3] = scale * d4.w * w;
        } else {
          gv[0] = scale * ldg(src + l) * w;
        }
        float cw[8];
        corner_weights(c, cw);
        float* base = grad_table + (size_t)l * gr.T * F;
        const int la = l < K ? l : 0;  // compile-time after unrolling
        const uint32_t ix = c.hx[0], iy = (uint32_t)(int32_t)floorf(fmul(g.y, res)), iz = (uint32_t)(int32_t)floorf(fmul(g.z, res));
        if (l < K && (ix | iy | iz) < 1023u) {  // the cell fits the key (always, for contracted coordinates on a coarse level)
          const uint32_t key = ix | (iy << 10) | (iz << 20);
          if (key != ag.key[la]) {
            agg_flush_level<F>(base, gr.mask, ag.key[la], ag.acc[la]);
            ag.key[la] = key;
          }
#pragma unroll
          for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int f = 0; f < F; ++f) ag.acc[la][k * F + f] = fmaf(gv[f], cw[k], ag.acc[la][k * F + f]);
        } else {
          float v[8 * F];
#pragma unroll
          for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int f = 0; f < F; ++f) v[k * F + f] = gv[f] * cw[k];
          scatter_cell<F>(base, r, v);
        }
      }
    }
  }
}
// one sample: static table or the containing actor's table (LMAX covers both grids)
template <int LMAX, int F, bool WANT_DEC, int K>
NFF_D int neurad_encode_point_bwd_t(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables,
                                    const ActorFrame* frames, int n_actors, const Gauss& g, float flip, const float* src,
                                    float scale, float* dec_acc, ScatterAgg<K, F>& ag) {
  float pb[3];
  const int a = n_actors > 0 ? actor_containing(frames, n_actors, g.x, g.y, g.z, pb) : -1;
  if (K > 0 && a != ag.tab) {  // pending sums belong to another table
    agg_flush_all(fg, grad_static, grad_actor_tables, ag);
    ag.tab = a;
  }
  if (a >= 0) {
    Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    encode_levels_bwd_t<LMAX, F, WANT_DEC, K>(grad_actor_tables ? grad_actor_tables[a] : nullptr, fg.actor_tables[a], fg.act, ga, src,
                                              scale, dec_acc, ag);
  } else {
    const Gauss gs = contract(g, fg.static_scale);
    encode_levels_bwd_t<LMAX, F, WANT_DEC, K>(grad_static, fg.stat.table, fg.stat, gs, src, scale, dec_acc, ag);
  }
  return a;
}
// `n` consecutive samples [i0, i0 + n) of one ray.  F == 4: features mode (src = the sample's dL/dfeatures row);
// F == 1: density mode, g = dL/d density * exp(clamp(x, -15, 15)) (trunc_exp backward, field_components/activations.py:38-41;
// density = exp(x) and exp is monotonic, so the clamp is applied to the stored density), src = the decoder weights.
#ifndef NFF_BWD_PREFETCH
#define NFF_BWD_PREFETCH 1
#endif
template <int F, bool WANT_DEC, int K>
NFF_D void encoding_bwd_segment_pending(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables,
                                        const ActorFrame* frames, int n_actors, const float* mean, const float* std_,
                                        const float* dfeatures, const float* density, const float* ddensity, int64_t i0, int n,
                                        float flip, float* dec_acc /* [8] */, ScatterAgg<K, F>& ag /* pending sums out */) {
  agg_init(ag);
  const int D = fg.stat.L * fg.stat.F;
  for (int t = 0; t < n; ++t) {
    const int64_t i = i0 + t;
    const Gauss g = {mean[3 * i], mean[3 * i + 1], mean[3 * i + 2], std_[i]};
    if (NFF_BWD_PREFETCH && t + 1 < n) {  // the walk is sequential and few warps are resident: fetch the next sample's inputs now
      if (F == 4) prefetch_l1(dfeatures + (i + 1) * D);
      prefetch_l1(mean + 3 * (i + 2)), prefetch_l1(std_ + i + 2);  // (a 128-byte line past the array's end is a dropped hint)
    }
    if (F == 4) {
      neurad_encode_point_bwd_t<8, F, false, K>(fg, grad_static, grad_actor_tables, frames, n_actors, g, flip, dfeatures + i * D, 1.0f,
                                                dec_acc, ag);
    } else {
      const float gd = ddensity[i] * fminf(fmaxf(density[i], 3.0590232e-07f), 3269017.372f);
      neurad_encode_point_bwd_t<8, F, WANT_DEC, K>(fg, grad_static, grad_actor_tables, frames, n_actors, g, flip, fg.decoder, gd, dec_acc,
                                                   ag);
    }
  }
}
// ... and with the pending sums flushed by the thread itself (the host emulation; the kernel merges the coarsest levels'
// pending sums across the warp first, modules.cuh: warp_merge_pending)
template <int F, bool WANT_DEC, int K>
NFF_D void encoding_bwd_segment(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables, const ActorFrame* frames,
                                int n_actors, const float* mean, const float* std_, const float* dfeatures, const float* density,
                                const float* ddensity, int64_t i0, int n, float flip, float* dec_acc /* [8] */) {
  ScatterAgg<K, F> ag;
  encoding_bwd_segment_pending<F, WANT_DEC, K>(fg, grad_static, grad_actor_tables, frames, n_actors, mean, std_, dfeatures, density,
                                               ddensity, i0, n, flip, dec_acc, ag);
  agg_flush_all(fg, grad_static, grad_actor_tables, ag);
}
// levels aggregated per feature width (registers: 8 * F sums + a key per level)
#ifndef NFF_BWD_AGG_F1
#define NFF_BWD_AGG_F1 6
#endif
#ifndef NFF_BWD_AGG_F4
#define NFF_BWD_AGG_F4 4
#endif
// the grids these variants cover: NeuRAD's shapes (and anything up to 8 levels of width 1 / 4)
NFF_HD bool encode_bwd_fast_ok(const FieldGrids& fg, int n_actors, int F) {
  return fg.stat.F == F && fg.stat.L <= 8 && (n_actors == 0 || (fg.act.F == F && fg.act.L <= 8));
}

// Backward of neurad_encode_point(): routes dfeat to the static table or to the containing actor's table (the zero
// padded tail of an actor sample's feature row has no parameter behind it).  `flip` is the per-ray actor flip of
// training mode (+1 / -1, neurad_encoding.py:212-219).
NFF_D int neurad_encode_point_bwd(const FieldGrids& fg, float* grad_static, float* const* grad_actor_tables,
                                  const ActorFrame* frames, int n_actors, const Gauss& g, float flip, const float* dfeat) {
  float pb[3];
  const int a = n_actors > 0 ? actor_containing(frames, n_actors, g.x, g.y, g.z, pb) : -1;
  if (a >= 0) {
    Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    if (grad_actor_tables && grad_actor_tables[a]) encode_levels_bwd(grad_actor_tables[a], fg.act, ga, dfeat);
  } else if (grad_static) {
    Gauss gs = contract(g, fg.static_scale);
    encode_levels_bwd(grad_static, fg.stat, gs, dfeat);
  }
  return a;
}

// nerfacc.render_weight_from_alpha backward for one ray (sequential; S <= a few hundred): w_i = a_i * T_i,
// T_i = prod_{j<i} (1 - a_j)  =>  dL/da_i = T_i * (dw_i - R_i),  R_i = sum_{k>i} dw_k a_k prod_{i<j<k} (1 - a_j),
// with the suffix recurrence R_{S-1} = 0, R_{i-1} = dw_i a_i + (1 - a_i) R_i.  No division: at a_i == 1 exactly the
// later samples' weights are 0 but R_i is not, and the result equals autograd of the cumprod (torch's cumprod backward
// is exact at a zero factor), where dividing sum_{k>i} dw_k w_k by 1 - a_i would lose the occlusion term.
NFF_D void alpha_weights_bwd_ray(const float* alpha, const float* dw, int S, float* dalpha) {
  float T = 1.0f;
  // forward pass for the transmittances, stored in dalpha[] temporarily
  for (int i = 0; i < S; ++i) {
    dalpha[i] = T;
    T *= 1.0f - alpha[i];
  }
  float R = 0.0f;
  for (int i = S - 1; i >= 0; --i) {
    const float a = alpha[i];
    dalpha[i] = dalpha[i] * (dw[i] - R);
    R = dw[i] * a + (1.0f - a) * R;
  }
}

// RaySamples.get_weights backward for one ray: w_i = (1 - e^{-a_i}) * e^{-A_i}, a = delta * density,
// A_i = sum_{j<i} a_j  =>  dL/da_i = dw_i * e^{-a_i} * e^{-A_i} - sum_{k>i} dw_k * w_k;  d density_i = delta_i * dL/da_i.
NFF_D void density_weights_bwd_ray(const float* delta, const float* density, const float* dw, int S, float* ddensity) {
  float A = 0.0f;
  for (int i = 0; i < S; ++i) {
    ddensity[i] = A;  // stash A_i
    A += delta[i] * density[i];
  }
  float suffix = 0.0f;
  for (int i = S - 1; i >= 0; --i) {
    const float a = delta[i] * density[i];
    const float eA = expf(-ddensity[i]), ea = expf(-a);
    const float w = (1.0f - ea) * eA;
    ddensity[i] = delta[i] * (dw[i] * ea * eA - suffix);
    suffix += dw[i] * w;
  }
}

// ------------------------------------------------------------------------------ gradients to the actor trajectories
// The main field's grid is built with require_actor_grad (fields/neurad_field.py:50), so in the reference the box-frame
// POSITIONS of actor samples carry a gradient back to DynamicActors.actor_positions / actor_rotations_6d
// (optimize_trajectories, model_components/dynamic_actors.py:37).  The box-frame DIRECTIONS do not: in torch mode the SH
// encoding runs under no_grad (field_components/encodings.py:797-800).
//
// d trilerp / d (ox, oy, oz) for one feature's 8 corner values (corner order of cell_rows()).
NFF_D void trilerp_grad(const float f[8], const Cell& c, float g[3]) {
  const float ox = c.ox, oy = c.oy, oz = c.oz, ix = 1.0f - ox, iy = 1.0f - oy, iz = 1.0f - oz;
  const float f03 = f[0] * ox + f[3] * ix, f12 = f[1] * ox + f[2] * ix;
  const float f56 = f[5] * ox + f[6] * ix, f47 = f[4] * ox + f[7] * ix;
  g[0] = ((f[0] - f[3]) * oy + (f[1] - f[2]) * iy) * oz + ((f[4] - f[7]) * oy + (f[5] - f[6]) * iy) * iz;
  g[1] = (f03 - f12) * oz + (f47 - f56) * iz;
  g[2] = (f03 * oy + f12 * iy) - (f47 * oy + f56 * iy);
}

// dL/d(grid coordinate in [0,1]^3) of one contracted gaussian: sum_l res_l * level_weight_l * sum_f dfeat[l,f] *
// d trilerp_f / d offset  (HashEncoding.pytorch_fwd: offset = x * res_l - floor(x * res_l), encodings.py:430-434).
NFF_D void encode_levels_pos_grad(const float* NFF_RESTRICT table, const Grid& gr, const Gauss& g, const float* dfeat, float gu[3]) {
  gu[0] = gu[1] = gu[2] = 0.0f;
  for (int l = 0; l < gr.L; ++l) {
    Cell c = grid_cell(g.x, g.y, g.z, gr.res[l]);
    uint32_t r[8];
    cell_rows(c, gr.mask, r);
    const float* base = table + (size_t)l * gr.T * gr.F;
    const float w = level_weight(gr.res[l], g.std) * gr.res[l];
    for (int f = 0; f < gr.F; ++f) {
      const float df = dfeat[l * gr.F + f];
      if (df == 0.0f) continue;
      float v[8], dt[3];
      for (int k = 0; k < 8; ++k) v[k] = ldg(base + (size_t)r[k] * gr.F + f);
      trilerp_grad(v, c, dt);
      gu[0] = fmaf(df * w, dt[0], gu[0]);
      gu[1] = fmaf(df * w, dt[1], gu[1]);
      gu[2] = fmaf(df * w, dt[2], gu[2]);
    }
  }
}

NFF_D float dot3(const float a[3], const float b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
// backward of y = x / max(|x|, 1e-12) (F.normalize): gx = (gy - y (y . gy)) / |x|
NFF_D void normalize_bwd(const float x[3], const float gy[3], float gx[3]) {
  const float n = fmaxf(sqrtf(dot3(x, x)), 1e-12f);
  const float y[3] = {x[0] / n, x[1] / n, x[2] / n};
  const float d = dot3(y, gy);
  for (int i = 0; i < 3; ++i) gx[i] = (gy[i] - y[i] * d) / n;
}
// backward of the Gram-Schmidt pair  u1 = normalize(r1), u2 = normalize(r2 - (u1 . r2) u1)  (rotation_6d_to_matrix
// cameras/camera_utils.py:438-441 and the per-keyframe orthogonalisation of interpolate_trajectories_6d, utils/poses.py:
// 117-120): given dL/du1, dL/du2 -> dL/dr1, dL/dr2.
NFF_D void gram_schmidt_bwd(const float r1[3], const float r2[3], const float gu1[3], const float gu2[3], float gr1[3], float gr2[3]) {
  const float n1 = fmaxf(sqrtf(dot3(r1, r1)), 1e-12f);
  const float u1[3] = {r1[0] / n1, r1[1] / n1, r1[2] / n1};
  const float s = dot3(u1, r2);
  const float c2[3] = {r2[0] - s * u1[0], r2[1] - s * u1[1], r2[2] - s * u1[2]};
  float gc2[3];
  normalize_bwd(c2, gu2, gc2);
  const float t = dot3(gc2, u1);
  float g1[3];
  for (int i = 0; i < 3; ++i) {
    gr2[i] = gc2[i] - t * u1[i];
    g1[i] = gu1[i] - t * r2[i] - s * gc2[i];
  }
  normalize_bwd(r1, g1, gr1);
}

// Chain from dL/d(box-frame position) of ONE actor sample to the trajectory parameters of its actor:
//   q = B^T (p - t),  B = rows (b1, b2, b3) = rotation_6d_to_matrix(lerp of the Gram-Schmidt'ed keyframes),  t = lerp of
//   the keyframe positions  (dynamic_actors.py:251-262, utils/poses.py:90-150, 42-55).
// rot6 / pos are the RAW parameters [T,A,6] / [T,A,3]; grad_rot6 / grad_pos are accumulated with atomics (two keyframes).
NFF_D void actor_pose_bwd(const float* NFF_RESTRICT rot6, const float* NFF_RESTRICT pos, int n_actors, int a, int left, int right,
                          float frac, const float p[3], const float gq[3], float* grad_rot6, float* grad_pos) {
  // forward recompute: keyframe Gram-Schmidt, lerp, rotation_6d_to_matrix
  float A1[2][3], A2[2][3], P[2][3];
  const int kf[2] = {left, right};
  for (int e = 0; e < 2; ++e) {
    const float* r = rot6 + ((size_t)kf[e] * n_actors + a) * 6;
    const float* t = pos + ((size_t)kf[e] * n_actors + a) * 3;
    float r1[3] = {ldg(r), ldg(r + 1), ldg(r + 2)}, r2[3] = {ldg(r + 3), ldg(r + 4), ldg(r + 5)};
    const float n1 = fmaxf(sqrtf(dot3(r1, r1)), 1e-12f);
    for (int i = 0; i < 3; ++i) A1[e][i] = r1[i] / n1;
    const float s = dot3(A1[e], r2);
    float c2[3] = {r2[0] - s * A1[e][0], r2[1] - s * A1[e][1], r2[2] - s * A1[e][2]};
    const float n2 = fmaxf(sqrtf(dot3(c2, c2)), 1e-12f);
    for (int i = 0; i < 3; ++i) {
      A2[e][i] = c2[i] / n2;
      P[e][i] = ldg(t + i);
    }
  }
  float a1[3], a2[3], tt[3];
  for (int i = 0; i < 3; ++i) {
    a1[i] = A1[0][i] + (A1[1][i] - A1[0][i]) * frac;
    a2[i] = A2[0][i] + (A2[1][i] - A2[0][i]) * frac;
    tt[i] = P[0][i] + (P[1][i] - P[0][i]) * frac;
  }
  const float m1 = fmaxf(sqrtf(dot3(a1, a1)), 1e-12f);
  const float b1[3] = {a1[0] / m1, a1[1] / m1, a1[2] / m1};
  const float s2 = dot3(b1, a2);
  const float c2[3] = {a2[0] - s2 * b1[0], a2[1] - s2 * b1[1], a2[2] - s2 * b1[2]};
  const float m2 = fmaxf(sqrtf(dot3(c2, c2)), 1e-12f);
  const float b2[3] = {c2[0] / m2, c2[1] / m2, c2[2] / m2};
  const float b3[3] = {b1[1] * b2[2] - b1[2] * b2[1], b1[2] * b2[0] - b1[0] * b2[2], b1[0] * b2[1] - b1[1] * b2[0]};
  // q_i = sum_j b_j[i] v_j, v = p - t
  const float v[3] = {p[0] - tt[0], p[1] - tt[1], p[2] - tt[2]};
  float gt[3] = {-dot3(b1, gq), -dot3(b2, gq), -dot3(b3, gq)};
  float gb1[3], gb2[3], gb3[3];
  for (int i = 0; i < 3; ++i) {
    gb1[i] = v[0] * gq[i];
    gb2[i] = v[1] * gq[i];
    gb3[i] = v[2] * gq[i];
  }
  // b3 = b1 x b2
  gb1[0] += b2[1] * gb3[2] - b2[2] * gb3[1];
  gb1[1] += b2[2] * gb3[0] - b2[0] * gb3[2];
  gb1[2] += b2[0] * gb3[1] - b2[1] * gb3[0];
  gb2[0] += gb3[1] * b1[2] - gb3[2] * b1[1];
  gb2[1] += gb3[2] * b1[0] - gb3[0] * b1[2];
  gb2[2] += gb3[0] * b1[1] - gb3[1] * b1[0];
  float ga1[3], ga2[3];
  gram_schmidt_bwd(a1, a2, gb1, gb2, ga1, ga2);
  // lerp: left gets (1 - frac), right gets frac; then the keyframes' own Gram-Schmidt back to the raw 6-D parameters
  for (int e = 0; e < 2; ++e) {
    const float w = e == 0 ? 1.0f - frac : frac;
    if (w == 0.0f) continue;
    const float* r = rot6 + ((size_t)kf[e] * n_actors + a) * 6;
    const float r1[3] = {ldg(r), ldg(r + 1), ldg(r + 2)}, r2[3] = {ldg(r + 3), ldg(r + 4), ldg(r + 5)};
    const float gA1[3] = {w * ga1[0], w * ga1[1], w * ga1[2]}, gA2[3] = {w * ga2[0], w * ga2[1], w * ga2[2]};
    float gr1[3], gr2[3];
    gram_schmidt_bwd(r1, r2, gA1, gA2, gr1, gr2);
    float* go = grad_rot6 + ((size_t)kf[e] * n_actors + a) * 6;
    float* gp = grad_pos + ((size_t)kf[e] * n_actors + a) * 3;
    for (int i = 0; i < 3; ++i) {
      atomic_add(go + i, gr1[i]);
      atomic_add(go + 3 + i, gr2[i]);
      atomic_add(gp + i, w * gt[i]);
    }
  }
}

// Trajectory gradient of one sample of the main field (if it lies inside an actor): position gradient of the actor grid
// lookup -> box frame (scene contraction is the identity inside the unit ball: |q| / actor_scale < 1 for every padded box)
// -> actor_pose_bwd.  Returns the actor index or -1.
NFF_D int neurad_encode_point_pose_bwd(const FieldGrids& fg, const Actors& A, const ActorFrame* frames, const float* rot6,
                                       const float* pos, int left, int right, float frac, const Gauss& g, float flip,
                                       const float* dfeat, float* grad_rot6, float* grad_pos) {
  float pb[3];
  const int a = A.n_actors > 0 ? actor_containing(frames, A.n_actors, g.x, g.y, g.z, pb) : -1;
  if (a < 0) return a;
  Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
  const float inv = frcp(fg.actor_scale);
  if (!(fmaxf(fmaxf(fabsf(ga.x), fabsf(ga.y)), fabsf(ga.z)) * inv < 1.0f)) return a;  // contracted region: never for a padded box
  ga = contract(ga, fg.actor_scale);
  float gu[3];
  encode_levels_pos_grad(fg.actor_tables[a], fg.act, ga, dfeat, gu);
  const float k = 0.25f * inv;  // u = (q / scale + 2) / 4
  float gq[3] = {gu[0] * k * (flip < 0.0f ? -1.0f : 1.0f), gu[1] * k, gu[2] * k};
  const float p[3] = {g.x, g.y, g.z};
  actor_pose_bwd(rot6, pos, A.n_actors, a, left, right, frac, p, gq, grad_rot6, grad_pos);
  return a;
}

// ------------------------------------------------------------------------------ gradients to the sample positions
// Camera pose optimisation (cameras/camera_optimizers.py:173-182) moves the ray origins and directions, so the sample
// means (cameras/rays.py:109-124) carry a gradient through the hash-grid lookups.  Per sample and lookup:
//   u = contract(p), features_lf = trilerp_lf(u * res_l) * w_l(std_u)   (encodings.py:425-466, neurad_encoding.py:297-304)
// The std depends on p only through the contraction's std scaling (spatial_distortions.py:132-136), which changes the
// level weights w_l = 1 / max(1, 2 res_l std_u) where 2 res_l std_u >= 1 (torch's clamp_min passes the gradient at the
// bound): d w_l / d std_u = -2 res_l w_l^2.
//
// One contracted lookup: g_u = dL/du (the position term of encode_levels_pos_grad, with 16-byte row loads for F = 4)
// and g_s = dL/d std_u.  src / scale as in encode_levels_bwd_t (features mode: the dfeatures row, scale 1; density mode:
// the decoder weights, scale = dL/d density * trunc_exp').  WANT_STD = false skips the level-weight term (the caller
// knows the std does not depend on p).
template <int LMAX, int F, bool WANT_STD>
NFF_D void encode_levels_mean_grad_t(const float* NFF_RESTRICT table, const Grid& gr, const Gauss& g, const float* NFF_RESTRICT src,
                                     float scale, float gu[3], float& gs) {
  static_assert(F == 1 || F == 4, "NeuRAD's feature widths");
  gu[0] = gu[1] = gu[2] = 0.0f;
  gs = 0.0f;
#pragma unroll
  for (int l = 0; l < LMAX; ++l) {
    if (l < gr.L) {
      const float res = gr.res[l];
      const Cell c = grid_cell(g.x, g.y, g.z, res);
      uint32_t r[8];
      cell_rows(c, gr.mask, r);
      const float w = level_weight(res, g.std);
      const float* base = table + (size_t)l * gr.T * F;
      float v[F][8], df[F];
      if (F == 4) {
        const float4 d4 = ldg(reinterpret_cast<const float4*>(src) + l);
        df[0] = scale * d4.x, df[F > 1 ? 1 : 0] = scale * d4.y, df[F > 2 ? 2 : 0] = scale * d4.z, df[F > 3 ? 3 : 0] = scale * d4.w;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 q = ldg(reinterpret_cast<const float4*>(base) + r[k]);
          v[0][k] = q.x, v[F > 1 ? 1 : 0][k] = q.y, v[F > 2 ? 2 : 0][k] = q.z, v[F > 3 ? 3 : 0][k] = q.w;
        }
      } else {
        df[0] = scale * ldg(src + l);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[0][k] = ldg(base + r[k]);
      }
      const float wr = w * res;
      const bool clamped = WANT_STD && fmul(fmul(res, 2.0f), g.std) >= 1.0f;
      float acc_v = 0.0f;
#pragma unroll
      for (int f = 0; f < F; ++f) {
        float dt[3];
        trilerp_grad(v[f], c, dt);
        const float s = df[f] * wr;
        gu[0] = fmaf(s, dt[0], gu[0]);
        gu[1] = fmaf(s, dt[1], gu[1]);
        gu[2] = fmaf(s, dt[2], gu[2]);
        if (clamped) acc_v = fmaf(df[f], trilerp(v[f], c), acc_v);
      }
      if (clamped) gs = fmaf(acc_v, -2.0f * res * w * w, gs);
    }
  }
}

// Backward of contract() (ScaledSceneContraction(order=inf), spatial_distortions.py:103-114,132-136) for one gaussian:
// dL/du (contracted position) and dL/d std_u -> dL/dp.  x = p / scale, m = |x|_inf; outside the unit cube
// y = (2 - 1/m) x / m and std_u = std / scale * ((2m - 1)^(1/3) / m)^2 / 4, both functions of m.  At a tie of |x_i|
// the gradient of m is split evenly between the tied coordinates, as torch's backward of the inf-norm does
// (linalg_vector_norm_backward: sign(x) * mask / mask.sum()).
NFF_D void contract_bwd(const Gauss& g, float scale, const float gu[3], float gs, float gp[3]) {
  const float inv = frcp(scale);
  const float x[3] = {fdiv(g.x, scale), fdiv(g.y, scale), fdiv(g.z, scale)};
  const float m = fmaxf(fmaxf(fabsf(x[0]), fabsf(x[1])), fabsf(x[2]));
  const float gy[3] = {0.25f * gu[0], 0.25f * gu[1], 0.25f * gu[2]};
  if (m < 1.0f) {
    for (int i = 0; i < 3; ++i) gp[i] = gy[i] * inv;
    return;
  }
  const float im = 1.0f / m, a = 2.0f - im;
  // d/dm [(2 - 1/m) / m] = 2 (1 - m) / m^3;  d/dm [(2m - 1)^(2/3) / m^2] = (4/3) (2m - 1)^(-1/3) / m^2 - 2 (2m - 1)^(2/3) / m^3
  const float da = 2.0f * (1.0f - m) * im * im * im;
  const float c = cbrtf(2.0f * m - 1.0f);
  const float dq2 = (4.0f / 3.0f) / c * im * im - 2.0f * c * c * im * im * im;
  float gm = da * (gy[0] * x[0] + gy[1] * x[1] + gy[2] * x[2]) + 0.25f * gs * g.std * inv * dq2;
  const int ties = (fabsf(x[0]) == m) + (fabsf(x[1]) == m) + (fabsf(x[2]) == m);
  gm /= (float)ties;
  for (int i = 0; i < 3; ++i) {
    float gx = gy[i] * a * im;
    if (fabsf(x[i]) == m) gx += x[i] < 0.0f ? -gm : gm;
    gp[i] = gx * inv;
  }
}

// dL/d mean of one sample of field `fg` (NeuRADHashEncoding.forward, neurad_encoding.py:150-187): the static lookup
// through the contraction, or -- for a sample inside an actor box -- the actor lookup through its contraction, the
// training-mode x flip and the world -> box transform q = B^T (p - t) (neurad_encoding.py:174-219).  `actor_grad`
// is the reference's require_actor_grad (fields/neurad_field.py:50,177): for the proposal fields the actor branch runs
// under no_grad and its rows overwrite the static features (index_put), so an actor sample's gradient is exactly 0.
template <int F>
NFF_D void neurad_encode_point_mean_bwd_t(const FieldGrids& fg, const ActorFrame* frames, int n_actors, bool actor_grad, const Gauss& g,
                                          float flip, const float* src, float scale, float gp[3]) {
  gp[0] = gp[1] = gp[2] = 0.0f;
  float pb[3];
  const int a = n_actors > 0 ? actor_containing(frames, n_actors, g.x, g.y, g.z, pb) : -1;
  float gu[3], gs;
  if (a >= 0) {
    if (!actor_grad) return;
    const Gauss ga = {flip < 0.0f ? -pb[0] : pb[0], pb[1], pb[2], g.std};
    encode_levels_mean_grad_t<8, F, true>(fg.actor_tables[a], fg.act, contract(ga, fg.actor_scale), src, scale, gu, gs);
    float gq[3];
    contract_bwd(ga, fg.actor_scale, gu, gs, gq);
    if (flip < 0.0f) gq[0] = -gq[0];
    const float* M = frames[a].w2b;  // q_i = sum_j M[4i + j] p_j + M[4i + 3]
    for (int j = 0; j < 3; ++j) gp[j] = M[j] * gq[0] + M[4 + j] * gq[1] + M[8 + j] * gq[2];
    return;
  }
  encode_levels_mean_grad_t<8, F, true>(fg.stat.table, fg.stat, contract(g, fg.static_scale), src, scale, gu, gs);
  contract_bwd(g, fg.static_scale, gu, gs, gp);
}

// Frustums.get_fast_isotropic_gaussian backward for one ray (cameras/rays.py:109-124): mean_s = o + d t_s with
// t_s = start_s + (end_s - start_s) / 2 of the detached bins (exactly sample_gaussian's t); std_s does not depend on
// o or d.  d o += dmean_s, d d += t_s dmean_s.
NFF_D float gaussian_t(float start, float end) { return fadd(start, fdiv(fsub(end, start), 2.0f)); }

// ------------------------------------------------------------------------------------------------ training losses
// The two per-ray regularisers NeuRAD trains with (models/neurad.py:262,524,541-545), one thread per ray; both are
// functions of the `weights_list` / `ray_samples_list` the module walk returns.
constexpr int kLossMaxS = 64;  // samples of the final level the loss kernels accept

// lossfun_distortion (model_components/losses.py:160-172) for one ray: c [S+1] spacing-domain edges, w [S]:
//   sum_i w_i sum_j w_j |u_i - u_j| + sum_i w_i^2 (c_{i+1} - c_i) / 3,  u = bin midpoints.
// dw (optional) receives d loss / d w_i = 2 sum_j w_j |u_i - u_j| + 2 w_i (c_{i+1} - c_i) / 3.
NFF_D float distortion_loss_ray(const float* c, const float* w, int S, float* dw) {
  float inter = 0.0f, intra = 0.0f;
  for (int i = 0; i < S; ++i) {
    const float ui = (c[i + 1] + c[i]) / 2.0f;
    float inner = 0.0f;
    for (int j = 0; j < S; ++j) inner += w[j] * fabsf(ui - (c[j + 1] + c[j]) / 2.0f);
    inter += w[i] * inner;
    const float d = c[i + 1] - c[i];
    intra += w[i] * w[i] * d;
    if (dw) dw[i] = 2.0f * inner + 2.0f * w[i] * d / 3.0f;
  }
  return inter + intra / 3.0f;
}

// zipnerf_interlevel_loss (losses.py:645-705) for one ray and one proposal level: the final level's histogram (c [S+1],
// w [S], both detached in the reference) is normalised, blurred with a box of half width r (_blur_stepfun), integrated
// to a piecewise-quadratic cdf and resampled at the proposal edges cp [Sp+1] (_sorted_interp_quad); the loss is
// sum_s relu(w_s - wp_s)^2 / (wp_s + 1e-5).  Only wp carries a gradient: dwp (optional) receives it.
NFF_D float zipnerf_interlevel_ray(const float* c, const float* w, int S, const float* cp, const float* wp, int Sp, float r,
                                   float* dwp) {
  constexpr int kM = 2 * (kLossMaxS + 1);  // blurred knots
  float xs[kM + 2], ys[kM + 2], cdf[kM + 2];  // padded by one knot at either end (losses.py:691-693)
  const int M = 2 * (S + 1);
  // w = cat(w[:-1], w[-1] + (1 - sum w)); w_norm = w / diff(c)
  float acc = 0.0f;
  for (int i = 0; i < S; ++i) acc += w[i];
  // y1_k = (y_k - y_{k-1}) / (2r) with y_{-1} = y_S = 0: the derivative of the box-blurred step function at c_k -/+ r
  // merge the two sorted knot sequences c_k - r (slope +y1_k) and c_k + r (slope -y1_k)
  int ia = 0, ib = 0;
  // cumulative sums in double, like torch.cumsum on the CPU (the oracle's accumulate type): in fp32 the blurred pdf
  // picks up ~1e-5 relative noise that the division by (wp + 1e-5) below amplifies to 1e-2 in the gradient
  double slope = 0.0, raw = 0.0;
  float xprev = 0.0f;
  float* x_ = xs + 1;
  float* y_ = ys + 1;
  auto wn = [&](int k) -> float {  // normalised weight of bin k (0 outside)
    if (k < 0 || k >= S) return 0.0f;
    const float wk = k == S - 1 ? w[k] + (1.0f - acc) : w[k];
    return wk / (c[k + 1] - c[k]);
  };
  for (int m = 0; m < M; ++m) {
    const bool take_a = ib >= S + 1 || (ia < S + 1 && c[ia] - r <= c[ib] + r);
    const int k = take_a ? ia : ib;
    const float x = take_a ? c[k] - r : c[k] + r;
    const float y1 = (wn(k) - wn(k - 1)) / (2.0f * r);
    // yr = cumsum(diff(xr) * cumsum(y2)).clamp_min(0), prefixed with 0: the clamp applies to the finished cumsum, it
    // does not feed back into it; each cumsum result is rounded to fp32 before it is used, as torch stores it
    if (m > 0) raw += (double)((x - xprev) * (float)slope);
    x_[m] = x;
    y_[m] = m == 0 ? 0.0f : fmaxf((float)raw, 0.0f);
    slope += (double)(take_a ? y1 : -y1);
    xprev = x;
    if (take_a) ++ia; else ++ib;
  }
  // piecewise linear pdf -> piecewise quadratic cdf; pad with (0, 0, 0) in front and (1, 0, 1) behind
  xs[0] = 0.0f; ys[0] = 0.0f; cdf[0] = 0.0f;
  double run = 0.0;
  cdf[1] = 0.0f;
  for (int m = 1; m < M; ++m) {
    run += (double)(0.5f * (y_[m] + y_[m - 1]) * (x_[m] - x_[m - 1]));
    cdf[1 + m] = (float)run;
  }
  xs[M + 1] = 1.0f; ys[M + 1] = 0.0f; cdf[M + 1] = 1.0f;
  const int L = M + 2;
  // _sorted_interp_quad at the proposal edges, then the difference of neighbours
  float prev = 0.0f, loss = 0.0f;
  for (int e = 0; e <= Sp; ++e) {
    const float x = cp[e];
    int lo = 0, hi = L;  // torch.searchsorted(xp, x) (left): first index with xp[idx] >= x
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (xs[mid] < x) lo = mid + 1; else hi = mid;
    }
    const int left = lo - 1 < 0 ? 0 : lo - 1;
    const int right = lo > L - 1 ? L - 1 : lo;
    const float xp0 = xs[left], xp1 = xs[right];
    float off = nan_to_num((x - xp0) / (xp1 - xp0));
    off = fminf(fmaxf(off, 0.0f), 1.0f);
    const float v = cdf[left] + (x - xp0) * (ys[left] + ys[right] * off + ys[left] * (1.0f - off)) * 0.5f;
    if (e > 0) {
      const float ws = v - prev;
      const float d = ws - wp[e - 1];
      const float den = wp[e - 1] + 1e-5f;
      if (d > 0.0f) {
        loss += d * d / den;
        if (dwp) dwp[e - 1] = -2.0f * d / den - d * d / (den * den);
      } else if (dwp) {
        dwp[e - 1] = 0.0f;
      }
    }
    prev = v;
  }
  return loss;
}

// One tile of the weight gradient of a Linear layer, dW[o][i] += sum_r dY[r][o] * act(X[r][i]) (act = ReLU when the
// layer's input is a hidden activation stored as its pre-activation).  The N x K outputs are cut into 4 x 4 blocks
// (NB = ceil(N/4) x KB = ceil(K/4) of them, at most 256); with fewer blocks than threads the tile's rows are split
// over G = nthreads / blocks row groups.  Thread tid = g * blocks + b owns block b = ob * KB + ib for the rows
// r = g, g + G, ...: one 16-byte read of act(X[r][4ib..4ib+3]) and one of dY[r][4ob..4ob+3] feed 16 FMAs (the first
// version read two words per FMA and was bound by shared-memory bandwidth; a 1 x 4 blocking still spent half its
// issue slots on loads).  xs [rows][ldx], dys [rows][ldy]: pitches = K / N rounded up to a multiple of 4, the pad
// columns zero, 16-byte aligned.  acc[4*c + d] belongs to dW[4*ob + c][4*ib + d].
struct WgradMap {
  int KB, blocks, G;  // blocks = NB * KB; G row groups
};
NFF_HD WgradMap wgrad_map(int K, int N, int nthreads) {
  WgradMap m;
  m.KB = (K + 3) >> 2;
  m.blocks = ((N + 3) >> 2) * m.KB;
  m.G = nthreads / m.blocks;
  if (m.G < 1) m.G = 1;
  return m;
}
NFF_D void wgrad_tile(int tid, const WgradMap& m, const float* xs, const float* dys, int rows, int ldx, int ldy, bool relu_x,
                      float (&acc)[16]) {
  const int g = tid / m.blocks, b = tid - g * m.blocks;
  if (g >= m.G) return;  // threads past G * blocks idle
  const int ob = b / m.KB, ib = b - ob * m.KB;
  for (int r = g; r < rows; r += m.G) {
    float4 x = *reinterpret_cast<const float4*>(xs + r * ldx + 4 * ib);
    if (relu_x) x.x = fmaxf(x.x, 0.0f), x.y = fmaxf(x.y, 0.0f), x.z = fmaxf(x.z, 0.0f), x.w = fmaxf(x.w, 0.0f);
    const float4 d = *reinterpret_cast<const float4*>(dys + r * ldy + 4 * ob);
    acc[0] = fmaf(d.x, x.x, acc[0]), acc[1] = fmaf(d.x, x.y, acc[1]), acc[2] = fmaf(d.x, x.z, acc[2]), acc[3] = fmaf(d.x, x.w, acc[3]);
    acc[4] = fmaf(d.y, x.x, acc[4]), acc[5] = fmaf(d.y, x.y, acc[5]), acc[6] = fmaf(d.y, x.z, acc[6]), acc[7] = fmaf(d.y, x.w, acc[7]);
    acc[8] = fmaf(d.z, x.x, acc[8]), acc[9] = fmaf(d.z, x.y, acc[9]), acc[10] = fmaf(d.z, x.z, acc[10]), acc[11] = fmaf(d.z, x.w, acc[11]);
    acc[12] = fmaf(d.w, x.x, acc[12]), acc[13] = fmaf(d.w, x.y, acc[13]), acc[14] = fmaf(d.w, x.z, acc[14]), acc[15] = fmaf(d.w, x.w, acc[15]);
  }
}
// where block b's accumulators go: add(o * K + i, acc[4*c + d]) for o = 4*ob + c < N, i = 4*ib + d < K
template <class Add>
NFF_D void wgrad_flush(int b, const WgradMap& m, int K, int N, const float (&acc)[16], Add add) {
  const int ob = b / m.KB, ib = b - ob * m.KB;
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int c = 0; c < 4; ++c)
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int d = 0; d < 4; ++d)
      if (4 * ob + c < N && 4 * ib + d < K) add((4 * ob + c) * K + 4 * ib + d, acc[4 * c + d]);
}

}  // namespace nff
