// nff_params.h -- plain-old-data parameter blocks handed to the kernels (by value, in the kernel parameter
// space) plus compile-time limits.  Shared between the CUDA build and the test-only host emulation.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/b200nerf.h"

namespace nff {

constexpr int kMaxLevels = 16;     // per grid (HashEncoding default is 16 levels)
constexpr int kMaxCand = 16;       // actor candidates per ray (ray line passes within the box's bounding sphere)
constexpr int kS0 = 128;           // proposal samples, round 0   (SamplingSettings.num_proposal_samples[0])
constexpr int kS1 = 64;            // proposal samples, round 1
constexpr int kS2 = 32;            // nerf samples == warp width: one sample per lane in the shading phase
constexpr int kGeoIn = 32;         // main grid: 8 levels x 4 features
constexpr int kHidden = 32;
constexpr int kNff = 32;           // nff_out_dim
constexpr int kSh = 16;            // SH degree-4 basis
constexpr int kApp = 16;           // appearance_dim (max supported)
constexpr int kFeatOut = 64;       // max nff_out_dim + appearance_dim

// packed, transposed ([in][out_padded]) MLP weights of the main field, in floats
constexpr int kGeoOutP = 36;  // 33 padded to a multiple of 4
constexpr int kOffGeoW0 = 0;                                  // [32][32]
constexpr int kOffGeoB0 = kOffGeoW0 + kGeoIn * kHidden;       // [32]
constexpr int kOffGeoW1 = kOffGeoB0 + kHidden;                // [32][36]
constexpr int kOffGeoB1 = kOffGeoW1 + kHidden * kGeoOutP;     // [36]
constexpr int kOffFeatW0 = kOffGeoB1 + kGeoOutP;              // [48][32]
constexpr int kOffFeatB0 = kOffFeatW0 + (kNff + kSh) * kHidden;
constexpr int kOffFeatW1 = kOffFeatB0 + kHidden;              // [32][32]
constexpr int kOffFeatB1 = kOffFeatW1 + kHidden * kHidden;
constexpr int kOffFeatW2 = kOffFeatB1 + kHidden;              // [32][32]
constexpr int kOffFeatB2 = kOffFeatW2 + kHidden * kNff;
constexpr int kMainMlpFloats = kOffFeatB2 + kNff;             // 5828 floats = 23.3 KB
// lidar decoder 48->32->32->2(4)
constexpr int kLidOutP = 4;
constexpr int kOffLidW0 = 0;                                   // [48][32]
constexpr int kOffLidB0 = kOffLidW0 + (kNff + kApp) * kHidden;
constexpr int kOffLidW1 = kOffLidB0 + kHidden;                 // [32][32]
constexpr int kOffLidB1 = kOffLidW1 + kHidden * kHidden;
constexpr int kOffLidW2 = kOffLidB1 + kHidden;                 // [32][4]
constexpr int kOffLidB2 = kOffLidW2 + kHidden * kLidOutP;
constexpr int kLidarMlpFloats = kOffLidB2 + kLidOutP;

// main-field MLP in nn.Linear ([out,in]) layout, the source for the tensor-core B tiles
constexpr int kNnGeoW0 = 0;
constexpr int kNnGeoB0 = kNnGeoW0 + kHidden * kGeoIn;
constexpr int kNnGeoW1 = kNnGeoB0 + kHidden;          // [33][32]: row 0 = sdf, rows 1..32 = geo_embedding
constexpr int kNnGeoB1 = kNnGeoW1 + (kNff + 1) * kHidden;
constexpr int kNnFeatW0 = kNnGeoB1 + (kNff + 1);      // [32][48]
constexpr int kNnFeatB0 = kNnFeatW0 + kHidden * (kNff + kSh);
constexpr int kNnFeatW1 = kNnFeatB0 + kHidden;
constexpr int kNnFeatB1 = kNnFeatW1 + kHidden * kHidden;
constexpr int kNnFeatW2 = kNnFeatB1 + kHidden;
constexpr int kNnFeatB2 = kNnFeatW2 + kNff * kHidden;
constexpr int kNnMlpFloats = kNnFeatB2 + kNff;

struct Grid {
  const float* table;  // torch layout: [L*T, F]; tcnn layout: the flat parameter vector (fp16-representable values)
  uint32_t mask;       // T-1
  uint32_t T;
  int32_t L, F;
  float res[kMaxLevels];  // HashEncoding.scalings: position scale of the torch layout AND the anti-aliasing weights of both
  // tiny-cuda-nn HashGrid layout (SURVEY 8f row f3; LAYOUT == 1 kernels only; zero otherwise)
  float pos_scale[kMaxLevels];    // grid_scale(level): pos = fma(x, pos_scale, 0.5)
  uint32_t lvl_res[kMaxLevels];   // vertices per axis
  uint32_t lvl_off[kMaxLevels];   // first entry of the level
  uint32_t lvl_mask[kMaxLevels];  // hashed levels: entries - 1 (entries is a power of two); dense levels: entries
  uint32_t dense_bits;            // bit l: level l indexes linearly (x + y*res + z*res^2 [+ w*res^3])
  int32_t n_dims;                 // 3, or 4 for the shared actor grid (4th coordinate = actor index / n_actors)
};

struct FieldGrids {
  Grid stat;
  Grid act;                          // torch layout: .table unused, per-actor tables below; tcnn layout: the one 4-D grid
  const float* const* actor_tables;  // device array [n_actors] (torch layout)
  float static_scale, actor_scale;
  float n_actors_f;                  // tcnn layout: the 4-D actor grid's 4th coordinate is actor_index / n_actors
  const float* decoder;              // proposal fields: density_decoder.weight [L*F]; main: nullptr
};

struct Actors {
  int32_t n_actors, n_times;
  const float* times;      // [T]
  const float* keyframes;  // [T,A,9]: per-keyframe Gram-Schmidt'ed (a1,a2) + position (poses.py:107-114)
  const uint8_t* present;  // [T,A]
  const float* bounds;     // [A,3] = size/2 + padding
  const float* radii;      // [A]   = |bounds|
  // DynamicActors.actor_editing (model_components/dynamic_actors.py:181-249), eval mode: actors [edit_first, edit_last)
  // render at the edited pose t' = R shift + t, R' = Rz(yaw) R (edit_box_pose, nff_device.h).  Empty range: no edit.
  int32_t edit_first, edit_last;
  float edit_shift[3];       // (lateral, longitudinal, height), box frame
  float edit_cos, edit_sin;  // cos / sin of the yaw, taken in double and rounded once
};

// The edit fields of `A` from the reference's actor_editing dict, resolved on the host (A.n_actors must be set).
// - longitudinal, lateral and rotation all 0: no edit, even with a height (the reference tests only those three);
// - index -1: every actor; otherwise actor min(index, n_actors - 1), truncated toward zero like
//   torch.tensor([...], dtype=torch.int), a negative value wrapping like torch indexing.
// Returns false, leaving A unedited, for an index that truncates below -n_actors (an IndexError in the reference).
// With no actors there is nothing to edit and any values are accepted.
inline bool resolve_actor_edit(Actors& A, double lateral, double longitudinal, double height, double rotation, double index) {
  A.edit_first = A.edit_last = 0;
  A.edit_shift[0] = A.edit_shift[1] = A.edit_shift[2] = 0.f;
  A.edit_cos = 1.f;
  A.edit_sin = 0.f;
  const int n = A.n_actors;
  if (n <= 0 || (longitudinal == 0.0 && lateral == 0.0 && rotation == 0.0)) return true;
  int first = 0, last = n;
  if (index != -1.0) {
    const double m = (double)(n - 1) < index ? (double)(n - 1) : index;  // Python's min(index, n - 1), NaN included
    const double k = trunc(m);
    if (!(k >= -(double)n)) return false;  // also rejects NaN
    first = (int)k < 0 ? (int)k + n : (int)k;
    last = first + 1;
  }
  A.edit_first = first;
  A.edit_last = last;
  A.edit_shift[0] = (float)lateral;
  A.edit_shift[1] = (float)longitudinal;
  A.edit_shift[2] = (float)height;
  A.edit_cos = (float)cos(rotation);
  A.edit_sin = (float)sin(rotation);
  return true;
}

struct Sampling {
  float lam, scaling, sky_distance, hist_pad, cam_area_scale;
  float lam_1, ratio;  // |lam-1|, lam_1/lam
  const float* u1;     // [kS1+1]
  const float* u2;     // [kS2+1]
  int32_t field_of_round[2];
};

struct Appearance {
  const float* emb;
  // eps: embeddings per sensor, interpolated in time; 0: one embedding per sensor, copied (use_temporal_appearance = False)
  int32_t num_embeds, dim, eps;
  float duration;
};

struct RenderParams {
  FieldGrids fields[3];
  const float* main_mlp;   // packed (kMainMlpFloats)
  const float* main_mlp_nn;  // nn.Linear layout (kNnMlpFloats), source of the tensor-core B tiles
  const float* lidar_mlp;  // packed (kLidarMlpFloats) or nullptr
  int* status;             // device-side failure flag (tensor-core barrier timeout)
  float beta;
  int32_t nff_dim;
  int32_t layout;          // 0: the reference's torch layout; 1: tiny-cuda-nn layout (grids, SH convention)
  Actors actors;
  Sampling samp;
  Appearance app;
  b200nerf_rays rays;
  b200nerf_outputs out;
  b200nerf_trace trace;
  b200nerf_peer_outputs peers;
  int64_t n_rays;
};

}  // namespace nff
