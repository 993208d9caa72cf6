// TEST SCAFFOLDING ONLY -- the host emulation (emul.cpp) plus the camera-pose gradient device code: dL/d mean of the
// module-level encoding and the isotropic-gaussian backward (csrc/nff_modules.h).  Built into its own library by
// tests/camopt_emul.py; never linked into libb200nerf.so.
#include "emul.cpp"

extern "C" {
// Gradient with respect to the sample means (nff_modules.h: neurad_encode_point_mean_bwd_t; loop structure of
// neurad_encoding_mean_bwd_kernel).  extra = {mean, std, times|NULL, flip|NULL, dfeatures|NULL, density|NULL,
// ddensity|NULL, dmean [N,S,3] (written)}
int emul_encoding_mean_bwd(const void* const* ptrs, const int* ints, const float* floats, const void* const* extra, long long n_rays,
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
  float* dmean = (float*)extra[7];
  const int D = fg.stat.L * fg.stat.F;
  const bool features_mode = !ddensity;
  if (!encode_bwd_fast_ok(fg, A.n_actors, features_mode ? 4 : 1)) return 1;
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
      const Gauss g = {mean[3 * i], mean[3 * i + 1], mean[3 * i + 2], std_[i]};
      if (features_mode) {
        neurad_encode_point_mean_bwd_t<4>(fg, frames.data(), A.n_actors, field == 0, g, flip, dfeatures + i * D, 1.0f, dmean + 3 * i);
      } else {
        const float gd = ddensity[i] * std::fmin(std::fmax(density[i], 3.0590232e-07f), 3269017.372f);
        neurad_encode_point_mean_bwd_t<1>(fg, frames.data(), A.n_actors, field == 0, g, flip, fg.decoder, gd, dmean + 3 * i);
      }
    }
  }
  return 0;
}

// isotropic_gaussian_bwd_kernel (modules.cuh) per ray, sequential sums: d origins = sum dmean, d dirs = sum t dmean
int emul_gaussian_bwd(const float* bins_e, long long n_rays, int S, const float* dmean, float* dorigins, float* ddirs) {
  for (long long r = 0; r < n_rays; ++r) {
    float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
    for (int s = 0; s < S; ++s) {
      const float t = gaussian_t(bins_e[r * (S + 1) + s], bins_e[r * (S + 1) + s + 1]);
      for (int k = 0; k < 3; ++k) {
        go[k] += dmean[3 * (r * S + s) + k];
        gd[k] = std::fmaf(t, dmean[3 * (r * S + s) + k], gd[k]);
      }
    }
    for (int k = 0; k < 3; ++k) dorigins[3 * r + k] = go[k], ddirs[3 * r + k] = gd[k];
  }
  return 0;
}
}
