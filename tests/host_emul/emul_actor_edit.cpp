// TEST SCAFFOLDING ONLY -- the actor-edit device code (resolve_actor_edit, edit_box_pose through actor_frame<true> and
// lane_actor_candidates<true>) run on the host.  Never linked into libb200nerf.so.
#include <vector>

#include "../../neurad-studio_b200/csrc/nff_lane.h"
#include "../../neurad-studio_b200/csrc/nff_modules.h"

using namespace nff;

extern "C" {

// resolve_actor_edit: returns 1 and the edited range [first, last), or 0 for a rejected index
int emul_resolve_actor_edit(int n_actors, const double* edit, int* first, int* last) {
  Actors A{};
  A.n_actors = n_actors;
  const bool ok = resolve_actor_edit(A, edit[0], edit[1], edit[2], edit[3], edit[4]);
  *first = A.edit_first;
  *last = A.edit_last;
  return ok ? 1 : 0;
}

// Edited frames of every actor at every ray's time.  `edit` = (lateral, longitudinal, height, rotation, index).
// frames [N,A,12]: actor_frame<true>'s world->box [R^T | -R^T t]; valid [N,A].
// cand [N,A]: 1 where lane_actor_candidates<true> keeps the actor for the ray; cand_w2b [N,A,12] its stored world->box.
int emul_actor_edit_frames(int n_actors, int n_times, const float* times, const float* rot6, const float* pos,
                           const uint8_t* present, const float* sizes, const float* pad, const double* edit, int n_rays,
                           const float* ray_times, const float* origins, const float* dirs, float* frames, int* valid,
                           int* cand, float* cand_w2b) {
  std::vector<float> kf((size_t)9 * n_times * n_actors), bounds(3 * n_actors), radii(n_actors);
  for (int i = 0; i < n_times * n_actors; ++i) {  // actors_prep_kernel: per-keyframe Gram-Schmidt, then the position
    float a1[3] = {rot6[6 * i], rot6[6 * i + 1], rot6[6 * i + 2]};
    float a2[3] = {rot6[6 * i + 3], rot6[6 * i + 4], rot6[6 * i + 5]};
    normalize3(a1);
    float dt = fadd(fadd(fmul(a1[0], a2[0]), fmul(a1[1], a2[1])), fmul(a1[2], a2[2]));
    for (int k = 0; k < 3; ++k) a2[k] = fsub(a2[k], fmul(dt, a1[k]));
    normalize3(a2);
    for (int k = 0; k < 3; ++k) {
      kf[9 * (size_t)i + k] = a1[k];
      kf[9 * (size_t)i + 3 + k] = a2[k];
      kf[9 * (size_t)i + 6 + k] = pos[3 * i + k];
    }
  }
  for (int a = 0; a < n_actors; ++a) {
    float b[3];
    for (int k = 0; k < 3; ++k) b[k] = bounds[3 * a + k] = fadd(fmul(sizes[3 * a + k], 0.5f), pad[k]);
    radii[a] = fsqrt(fadd(fadd(fmul(b[0], b[0]), fmul(b[1], b[1])), fmul(b[2], b[2])));
  }
  Actors A{};
  A.n_actors = n_actors;
  A.n_times = n_times;
  A.times = times;
  A.keyframes = kf.data();
  A.present = present;
  A.bounds = bounds.data();
  A.radii = radii.data();
  if (!resolve_actor_edit(A, edit[0], edit[1], edit[2], edit[3], edit[4])) return -1;
  std::vector<float> scratch(lane_scratch_floats_per_cta());
  const LaneScratch sc = lane_scratch_of(scratch.data(), 0);
  for (int r = 0; r < n_rays; ++r) {
    int left, right;
    float frac;
    keyframe_bracket(A, ray_times[r], left, right, frac);
    for (int a = 0; a < n_actors; ++a) {
      ActorFrame f;
      actor_frame<true>(A, a, left, right, frac, f);
      for (int k = 0; k < 12; ++k) frames[((size_t)r * n_actors + a) * 12 + k] = f.w2b[k];
      valid[(size_t)r * n_actors + a] = f.valid;
      cand[(size_t)r * n_actors + a] = 0;
    }
    int overflow = 0;
    const int n = lane_actor_candidates<true>(A, ray_times[r], origins + 3 * r, dirs + 3 * r, sc, 0, &overflow);
    if (overflow) return -2;
    for (int c = 0; c < n; ++c) {
      const float* p = sc.cand + (size_t)c * kCandFloats * kLaneThreads;
      const int a = (int)p[15 * kLaneThreads];
      cand[(size_t)r * n_actors + a] = 1;
      for (int k = 0; k < 12; ++k) cand_w2b[((size_t)r * n_actors + a) * 12 + k] = p[k * kLaneThreads];
    }
  }
  return 0;
}
}
