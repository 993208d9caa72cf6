// nff_device.h -- device-side implementation of NeuRAD's neural-feature-field forward path.
//
// One warp renders one ray end to end: power-spaced initial bins -> proposal round 0 (128 samples) -> PDF
// resample -> proposal round 1 (64) -> PDF resample -> main field (32 samples, one per lane: hash grid, geo MLP,
// SH, feature MLP, sigmoid-SDF alpha) -> transmittance scan -> composite.  Bins / cdf live in shared memory,
// everything else in registers; nothing but the per-ray outputs goes back to HBM.
//
// Each function names the reference code it reproduces (paths relative to nerfstudio/).  Where the reference
// evaluates separate elementwise torch kernels, the same single-rounding fp32 ops are used via simt::fmul/fadd/..
// (no FMA contraction), so grid cells, hash rows and bin edges agree with the reference bit for bit given
// identical inputs; only transcendental functions and dot-product orders differ (<= a few ulp).
#pragma once
#include "nff_params.h"
#include "simt.h"

#ifndef NFF_G_PROP
#define NFF_G_PROP 1  // proposal-grid levels gathered per batch (8 loads each); 1 measured best (r01 variants)
#endif
#ifndef NFF_G_ACT
#define NFF_G_ACT 2
#endif
#ifndef NFF_ILP
#define NFF_ILP 2  // independent samples per lane in the proposal rounds (64 % 32*NFF_ILP == 0)
#endif
#ifndef NFF_F4_UNROLL
#define NFF_F4_UNROLL 2
#endif
#ifndef NFF_FAST_RCP
#define NFF_FAST_RCP 1  // anti-aliasing weights via MUFU.RCP (smooth factor, <= 1 ulp)
#endif
#ifndef NFF_PARITY_STD
#define NFF_PARITY_STD 0  // gaussian std / contraction scaling / level weight with the reference's own op sequence (pow(x, 1/3) as
                          // powf(x, 0.33333334f), true divisions); 0: cbrtf + reciprocal multiplies (<= 3e-7 relative, faster)
#endif
#ifndef NFF_PARITY_LERP
#define NFF_PARITY_LERP 0  // trilinear blend with the reference's separate products (encodings.py:454-466); 0: one product per
                           // blend folded into an FMA
#endif
#define NFF_STR2(x) #x
#define NFF_STR(x) NFF_STR2(x)

namespace nff {
using namespace simt;
constexpr int kF4Unroll = NFF_F4_UNROLL;

// ------------------------------------------------------------------------------------------------ helpers
NFF_D float nan_to_num(float v) {  // torch.nan_to_num defaults: nan->0, +-inf -> +-FLT_MAX
  if (v != v) return 0.0f;
  if (v > 3.4028234663852886e38f) return 3.4028234663852886e38f;
  if (v < -3.4028234663852886e38f) return -3.4028234663852886e38f;
  return v;
}
NFF_D float warp_sum(float v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += shfl_xor(v, m);
  return v;
}
NFF_D float warp_scan_add(float v) {  // inclusive
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    float n = shfl_up(v, d);
    if (lane() >= d) v += n;
  }
  return v;
}
NFF_D float warp_scan_mul(float v) {  // inclusive
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    float n = shfl_up(v, d);
    if (lane() >= d) v *= n;
  }
  return v;
}

// ------------------------------------------------------------------------------ power-law sample spacing
// utils/math.py:541-579 (power_fn / inv_power_fn, general branch) as used by PowerSampler
// (model_components/ray_samplers.py:838-852).  x**lam with lam == -1 is torch's reciprocal fast path.
NFF_D float pow_lam(float t, float e) { return e == -1.0f ? frcp(t) : powf(t, e); }
NFF_D float spacing_fn(float x, const Sampling& s) {
  float t = fadd(fdiv(fmul(x, s.scaling), s.lam_1), 1.0f);
  return fmul(s.ratio, fsub(pow_lam(t, s.lam), 1.0f));
}
NFF_D float spacing_fn_inv(float y, const Sampling& s) {
  if (s.lam == -1.0f) {
    // NeuRAD's power_lambda, same values as the general path: lam_1 == 2, so (y * -1) / 2 is exactly y * -0.5 (one
    // rounding of the same real number), and t**-1 is the reciprocal; the division by `scaling` stays IEEE
    const float t = fmaxf(fadd(fmul(y, -0.5f), 1.0f), 1e-10f);
    return fdiv(fmul(fsub(frcp(t), 1.0f), s.lam_1), s.scaling);
  }
  float t = fadd(fdiv(fmul(y, s.lam), s.lam_1), 1.0f);
  t = fmaxf(t, 1e-10f);
  float r = fmul(fsub(pow_lam(t, s.lam == -1.0f ? -1.0f : 1.0f / s.lam), 1.0f), s.lam_1);
  return fdiv(r, s.scaling);
}
// spacing_to_euclidean_fn (ray_samplers.py:119-120)
NFF_D float to_euclid(float u, float s_near, float s_far, const Sampling& s) {
  return spacing_fn_inv(fadd(fmul(u, s_far), fmul(fsub(1.0f, u), s_near)), s);
}
// torch.linspace(0, 1, n+1)[i] (symmetric evaluation of aten's linspace kernel)
NFF_D float linspace01(int i, int n) {
  float step = fdiv(1.0f, (float)n);
  return i < (n + 1) / 2 ? fmul(step, (float)i) : fsub(1.0f, fmul(step, (float)(n - i)));
}

// ------------------------------------------------------------------------------------ gaussian + contraction
struct Gauss {
  float x, y, z, std;
};
// Frustums.get_fast_isotropic_gaussian, num_multisamples = 1 (cameras/rays.py:109-124)
NFF_D Gauss sample_gaussian(const float o[3], const float d[3], float area, float start, float end) {
  float md = fdiv(fsub(end, start), 2.0f);
  float t = fadd(start, md);
  Gauss g;
  g.x = fadd(o[0], fmul(d[0], t));
  g.y = fadd(o[1], fmul(d[1], t));
  g.z = fadd(o[2], fmul(d[2], t));
  float cs = fmul(area, fmul(t, t));
  // reference: pow(x, 1/3) with the fp32 exponent 0.33333334f; cbrtf differs from it by < 3e-7 relative
  // (|ln x| * 1e-8) and costs ~12 instead of ~75 instructions
#if NFF_PARITY_STD
  g.std = powf(fmul(cs, md), 0.33333334f);
#else
  g.std = cbrtf(fmul(cs, md));
#endif
  return g;
}
// ScaledSceneContraction(order=inf) on a GaussiansStd (field_components/spatial_distortions.py:103-114,132-136)
NFF_D Gauss contract(Gauss g, float scale) {
  // Positions keep the reference's exact op sequence (IEEE divisions): the finest grid level multiplies any rounding
  // difference in x by its resolution (4096 / 8191 cells), so one ulp here is ~1e-4 in a feature.  The std only
  // scales the smooth anti-aliasing weights, so it uses reciprocals and cbrt (<= 3e-7 relative).
  float x = fdiv(g.x, scale), y = fdiv(g.y, scale), z = fdiv(g.z, scale);
#if NFF_PARITY_STD
  float sd = fdiv(g.std, scale);
#else
  float sd = fmul(g.std, frcp(scale));
#endif
  float mag = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z));
  if (!(mag < 1.0f)) {
    const float a = fsub(2.0f, frcp(mag));
    x = fmul(a, fdiv(x, mag));
    y = fmul(a, fdiv(y, mag));
    z = fmul(a, fdiv(z, mag));
#if NFF_PARITY_STD
    float q = fdiv(powf(fsub(fmul(2.0f, mag), 1.0f), 0.33333334f), mag);
#else
    float q = fmul(cbrtf(fsub(fmul(2.0f, mag), 1.0f)), frcp(mag));
#endif
    sd = fmul(sd, fmul(q, q));
  }
  Gauss r;
  r.x = fmul(fadd(x, 2.0f), 0.25f);
  r.y = fmul(fadd(y, 2.0f), 0.25f);
  r.z = fmul(fadd(z, 2.0f), 0.25f);
  r.std = fmul(sd, 0.25f);
  return r;
}

// -------------------------------------------------------------------------------------------- hash grid
// HashEncoding.hash_fn + pytorch_fwd (field_components/encodings.py:406-466): per level p = x*res;
// c = ceil(p), f = floor(p); rows = ((i*1) ^ (j*2654435761) ^ (k*805459861)) mod T (+ level*T); trilinear blend
// with weight (p - f) on the ceil corner.  int64 products mod 2^k == uint32 wrap-around products mod 2^k.
struct Cell {
  uint32_t hx[2], hy[2], hz[2];  // [0] = floor, [1] = ceil, already multiplied by the primes
  float ox, oy, oz;
};
NFF_D Cell grid_cell(float x, float y, float z, float res) {
  float px = fmul(x, res), py = fmul(y, res), pz = fmul(z, res);
  float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  Cell c;
  // ceil(p) == floor(p) + (p != floor(p)) for finite p
  const uint32_t ix = (uint32_t)(int32_t)fx, iy = (uint32_t)(int32_t)fy, iz = (uint32_t)(int32_t)fz;
  c.hx[0] = ix;
  c.hx[1] = ix + (px != fx ? 1u : 0u);
  c.hy[0] = iy * 2654435761u;
  c.hy[1] = (iy + (py != fy ? 1u : 0u)) * 2654435761u;
  c.hz[0] = iz * 805459861u;
  c.hz[1] = (iz + (pz != fz ? 1u : 0u)) * 805459861u;
  c.ox = fsub(px, fx);
  c.oy = fsub(py, fy);
  c.oz = fsub(pz, fz);
  return c;
}
// corner order of the reference: hashed_0..7 = ccc, cfc, ffc, fcc, ccf, cff, fff, fcf  (x,y,z; c=ceil f=floor)
NFF_D void cell_rows(const Cell& c, uint32_t mask, uint32_t r[8]) {
  r[0] = (c.hx[1] ^ c.hy[1] ^ c.hz[1]) & mask;
  r[1] = (c.hx[1] ^ c.hy[0] ^ c.hz[1]) & mask;
  r[2] = (c.hx[0] ^ c.hy[0] ^ c.hz[1]) & mask;
  r[3] = (c.hx[0] ^ c.hy[1] ^ c.hz[1]) & mask;
  r[4] = (c.hx[1] ^ c.hy[1] ^ c.hz[0]) & mask;
  r[5] = (c.hx[1] ^ c.hy[0] ^ c.hz[0]) & mask;
  r[6] = (c.hx[0] ^ c.hy[0] ^ c.hz[0]) & mask;
  r[7] = (c.hx[0] ^ c.hy[1] ^ c.hz[0]) & mask;
}
NFF_D float blend(float a, float wa, float b, float wb) { return fadd(fmul(a, wa), fmul(b, wb)); }
NFF_D float trilerp(const float f[8], const Cell& c) {
  float ix = fsub(1.0f, c.ox), iy = fsub(1.0f, c.oy), iz = fsub(1.0f, c.oz);
  float f03 = blend(f[0], c.ox, f[3], ix);
  float f12 = blend(f[1], c.ox, f[2], ix);
  float f56 = blend(f[5], c.ox, f[6], ix);
  float f47 = blend(f[4], c.ox, f[7], ix);
  float f0312 = blend(f03, c.oy, f12, iy);
  float f4756 = blend(f47, c.oy, f56, iy);
  return blend(f0312, c.oz, f4756, iz);
}

// Fused-path variant: same blend tree with the second product folded into an FMA (one rounding fewer per blend,
// 14 instead of 24 instructions); the stage operator b200nerf_hashgrid_fwd keeps the bit-exact form above.
#if NFF_PARITY_LERP
NFF_D float blend_f(float a, float wa, float b, float wb) { return fadd(fmul(a, wa), fmul(b, wb)); }
#else
NFF_D float blend_f(float a, float wa, float b, float wb) { return fmaf(a, wa, b * wb); }
#endif
// anti-aliasing weight 1/max(1, 2*res*std) (neurad_encoding.py:302)
NFF_D float level_weight(float res, float std) {
  const float t = fmaxf(fmul(fmul(res, 2.0f), std), 1.0f);
#if NFF_FAST_RCP && !NFF_PARITY_STD && defined(__CUDACC__)
  float r;  // bare MUFU.RCP (<= 1 ulp; t >= 1, so neither the denormal guard of __fdividef nor a Newton step is needed;
            // the value is the one __fdividef(1.0f, t) returns for t in [1, 2^126))
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(t));
  return r;
#else
  return frcp(t);
#endif
}
NFF_D float trilerp_f(const float f[8], const Cell& c, float ix, float iy, float iz) {
  float f03 = blend_f(f[0], c.ox, f[3], ix);
  float f12 = blend_f(f[1], c.ox, f[2], ix);
  float f56 = blend_f(f[5], c.ox, f[6], ix);
  float f47 = blend_f(f[4], c.ox, f[7], ix);
  float f0312 = blend_f(f03, c.oy, f12, iy);
  float f4756 = blend_f(f47, c.oy, f56, iy);
  return blend_f(f0312, c.oz, f4756, iz);
}

// ---- fused-path addressing: byte offsets straight out of the hash --------------------------------------------------
// The stage operator above exposes the reference's row indices; the fused kernels only need the ADDRESSES, and the
// index arithmetic was a large share of their instructions (per corner xor3 + and + zero-extend +
// 64-bit scale-and-add).  Here every hash term is pre-multiplied by the row size (a shift distributes over
// xor, and (h & mask) << s == (h << s) & (mask << s) while log2(T) + s <= 32), so a corner costs one LOP3
// ((hx ^ a) & maskb) and one 64-bit add.  The "ceil" corner is always floor + 1: where the reference's ceil equals its
// floor (p integral) the interpolation offset is exactly 0, so the value read there is multiplied by 0 either way
// (finite tables) -- same result, three compare/select pairs fewer per level.
template <int SH>  // log2(bytes per table row): F = 1 -> 2, F = 4 -> 4
struct CellB {
  uint32_t hx, hy, hz;  // floor corner, pre-scaled
  float ox, oy, oz;
};
template <int SH>
NFF_D CellB<SH> grid_cell_b(float x, float y, float z, float res) {
  const float px = fmul(x, res), py = fmul(y, res), pz = fmul(z, res);
  const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  CellB<SH> c;
  c.hx = (uint32_t)(int32_t)fx << SH;
  c.hy = (uint32_t)(int32_t)fy * (2654435761u << SH);
  c.hz = (uint32_t)(int32_t)fz * (805459861u << SH);
  c.ox = fsub(px, fx);
  c.oy = fsub(py, fy);
  c.oz = fsub(pz, fz);
  return c;
}
// byte offsets of the 8 corners in the reference's order (ccc, cfc, ffc, fcc, ccf, cff, fff, fcf)
NFF_D uint32_t xor_and(uint32_t a, uint32_t b, uint32_t m) {  // (a ^ b) & m: one LOP3
#if defined(__CUDACC__)
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0x28;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
  return d;
#else
  return (a ^ b) & m;
#endif
}
template <int SH>
NFF_D void cell_offsets_b(const CellB<SH>& c, uint32_t maskb, uint32_t r[8]) {
  const uint32_t hx1 = c.hx + (1u << SH), hy1 = c.hy + (2654435761u << SH), hz1 = c.hz + (805459861u << SH);
  const uint32_t a11 = hy1 ^ hz1, a01 = c.hy ^ hz1, a10 = hy1 ^ c.hz, a00 = c.hy ^ c.hz;
  r[0] = xor_and(hx1, a11, maskb);
  r[1] = xor_and(hx1, a01, maskb);
  r[2] = xor_and(c.hx, a01, maskb);
  r[3] = xor_and(c.hx, a11, maskb);
  r[4] = xor_and(hx1, a10, maskb);
  r[5] = xor_and(hx1, a00, maskb);
  r[6] = xor_and(c.hx, a00, maskb);
  r[7] = xor_and(c.hx, a10, maskb);
}
// base + zero-extended 32-bit byte offset as ONE instruction (IMAD.WIDE.U32 off * 1 + base)
template <class T>
NFF_D T ldg_at(const char* base, uint32_t byte_off) {
#if defined(__CUDACC__)
  uint64_t addr;
  asm("mad.wide.u32 %0, %1, 1, %2;" : "=l"(addr) : "r"(byte_off), "l"((uint64_t)base));
  return ldg(reinterpret_cast<const T*>(addr));
#else
  return ldg(reinterpret_cast<const T*>(base + byte_off));
#endif
}
// byte address of level l's first row, opaque to the compiler so that it is formed once per level and not re-associated
// into every corner's offset
NFF_D const char* level_base(const void* table, uint32_t l, uint32_t T, int row_bytes) {
  const char* p = reinterpret_cast<const char*>(table) + (size_t)l * T * (size_t)row_bytes;
#if defined(__CUDACC__)
  asm("" : "+l"(p));
#endif
  return p;
}
template <int SH>
NFF_D float trilerp_b(const float f[8], const CellB<SH>& c, float ix, float iy, float iz) {
  float f03 = blend_f(f[0], c.ox, f[3], ix);
  float f12 = blend_f(f[1], c.ox, f[2], ix);
  float f56 = blend_f(f[5], c.ox, f[6], ix);
  float f47 = blend_f(f[4], c.ox, f[7], ix);
  float f0312 = blend_f(f03, c.oy, f12, iy);
  float f4756 = blend_f(f47, c.oy, f56, iy);
  return blend_f(f0312, c.oz, f4756, iz);
}

// One grid, all levels, F = 1, fused with the proposal field's Linear(L,1) decoder:
//   sum_l dec[l] * interp_l * 1/max(1, 2*res_l*std)      (neurad_encoding.py:297-304, neurad_field.py:201,211)
template <int L, int G>
NFF_D float encode_f1_dot(const float* NFF_RESTRICT table, const Grid& gr, Gauss g, const float* NFF_RESTRICT dec) {
  // levels in groups of G: the 8*G gathers of a group are issued back to back before the first is consumed
  static_assert(L % G == 0, "group size must divide the level count");
  float acc = 0.0f;
  const uint32_t maskb = gr.mask << 2;
#pragma unroll
  for (int l0 = 0; l0 < L; l0 += G) {
    CellB<2> c[G];
    float f[G][8];
#pragma unroll
    for (int j = 0; j < G; ++j) {
      c[j] = grid_cell_b<2>(g.x, g.y, g.z, gr.res[l0 + j]);
      uint32_t r[8];
      cell_offsets_b<2>(c[j], maskb, r);
      const char* base = level_base(table, l0 + j, gr.T, 4);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[j][k] = ldg_at<float>(base, r[k]);
    }
#pragma unroll
    for (int j = 0; j < G; ++j) {
      float w = level_weight(gr.res[l0 + j], g.std);
      float v = trilerp_b<2>(f[j], c[j], 1.0f - c[j].ox, 1.0f - c[j].oy, 1.0f - c[j].oz);
      acc = fmaf(fmul(v, w), ldg(dec + l0 + j), acc);
    }
  }
  return acc;
}
// ---- tiny-cuda-nn HashGrid layout (SURVEY 8f row f3: tcnn-trained checkpoints) ---------------------------------------
// tcnn::GridEncoding (encodings/grid.h; configuration built at field_components/encodings.py:386-401) differs from the
// torch twin in four ways: the position is pos = fma(x, grid_scale(l), 0.5) with grid_scale = base * growth^l - 1 (vertex-
// centred), levels whose res^n vertices fit their share of the table index LINEARLY (x + y*res + z*res^2, no hash), every
// level has its own entry offset / size, and the actors share ONE 4-D grid whose 4th coordinate is actor_index / n_actors
// (neurad_encoding.py:270-281; a 4th prime, 3674653429, joins the hash).  Parameters are the fp16-rounded values of the
// checkpoint held as floats, the arithmetic is fp32 (tiny-cuda-nn itself accumulates in half: parity unpinned, see
// oracle/tcnn_oracle.py).  The anti-aliasing weights still use HashEncoding.scalings (neurad_encoding.py:300-302).
//
// Entry indices of the 2^D corners of level l, in the order bit d of the corner number = "ceil" along dimension d, and the
// interpolation offsets.
template <int D>
NFF_D void tcnn_corners(const Grid& gr, int l, const float* x, uint32_t* idx /* [1 << D] */, float* frac /* [D] */) {
  uint32_t pg[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float p = fmaf(x[d], gr.pos_scale[l], 0.5f);
    const float f = floorf(p);
    pg[d] = (uint32_t)(int32_t)f;
    frac[d] = fsub(p, f);
  }
  const uint32_t res = gr.lvl_res[l];
  if ((gr.dense_bits >> l) & 1u) {
    uint32_t base = 0, stride = 1, st[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      st[d] = stride;
      base += pg[d] * stride;
      stride *= res;
    }
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) {
      uint32_t i = base;
#pragma unroll
      for (int d = 0; d < D; ++d)
        if (c & (1 << d)) i += st[d];
      // tiny-cuda-nn takes `index % entries` and never clamps: the "+1" vertex of the last cell (pos >= res - 1, i.e. x
      // within half a cell of 1) wraps into the next row / the start of the level.  i < 2 * entries always.
      if (i >= gr.lvl_mask[l]) i -= gr.lvl_mask[l];
      idx[c] = gr.lvl_off[l] + i;
    }
  } else {
    constexpr uint32_t kPrimes[4] = {1u, 2654435761u, 805459861u, 3674653429u};
    uint32_t h0[D], h1[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      h0[d] = pg[d] * kPrimes[d];
      h1[d] = h0[d] + kPrimes[d];
    }
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) {
      uint32_t h = 0;
#pragma unroll
      for (int d = 0; d < D; ++d) h ^= (c & (1 << d)) ? h1[d] : h0[d];
      idx[c] = gr.lvl_off[l] + (h & gr.lvl_mask[l]);
    }
  }
}
// N-linear interpolation weight of corner c
template <int D>
NFF_D float tcnn_corner_weight(int c, const float* frac) {
  float w = 1.0f;
#pragma unroll
  for (int d = 0; d < D; ++d) w = fmul(w, (c & (1 << d)) ? frac[d] : fsub(1.0f, frac[d]));
  return w;
}
// F = 1 grid fused with the proposal decoder (the tcnn twin of encode_f1_dot); `x` has D coordinates in [0,1]
template <int D>
NFF_D float tcnn_encode_f1_dot(const Grid& gr, int L, const float* x, float std, const float* NFF_RESTRICT dec) {
  float acc = 0.0f;
#pragma unroll 1
  for (int l = 0; l < L; ++l) {
    uint32_t idx[1 << D];
    float frac[D];
    tcnn_corners<D>(gr, l, x, idx, frac);
    float f[1 << D];
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) f[c] = ldg(gr.table + idx[c]);
    float v = 0.0f;
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) v = fmaf(tcnn_corner_weight<D>(c, frac), f[c], v);
    acc = fmaf(fmul(v, level_weight(gr.res[l], std)), ldg(dec + l), acc);
  }
  return acc;
}
// F = 4 grid into a strided column (the tcnn twin of encode_f4_col / encode_f4_panel): out[(4l+f) * stride]
template <int D>
NFF_D void tcnn_encode_f4(const Grid& gr, int L, const float* x, float std, float* out, int stride) {
#pragma unroll 1
  for (int l = 0; l < L; ++l) {
    uint32_t idx[1 << D];
    float frac[D];
    tcnn_corners<D>(gr, l, x, idx, frac);
    const float4* t4 = reinterpret_cast<const float4*>(gr.table);
    float4 v[1 << D];
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) v[c] = ldg(t4 + idx[c]);
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) {
      const float w = tcnn_corner_weight<D>(c, frac);
      a0 = fmaf(w, v[c].x, a0);
      a1 = fmaf(w, v[c].y, a1);
      a2 = fmaf(w, v[c].z, a2);
      a3 = fmaf(w, v[c].w, a3);
    }
    const float lw = level_weight(gr.res[l], std);
    out[(4 * l + 0) * stride] = fmul(a0, lw);
    out[(4 * l + 1) * stride] = fmul(a1, lw);
    out[(4 * l + 2) * stride] = fmul(a2, lw);
    out[(4 * l + 3) * stride] = fmul(a3, lw);
  }
}
// tcnn SphericalHarmonics, degree 4 (encodings/spherical_harmonics.h): the reference passes (d + 1) / 2
// (fields/base_field.py:136-142) and tiny-cuda-nn maps it back with x * 2 - 1, i.e. the basis is evaluated at the direction
// itself, with the Condon-Shortley signs the torch twin (utils/math.py:31-94) does not have.
NFF_D void sh4_tcnn(float dx, float dy, float dz, float* c) {
  const float x = fsub(fmul(fmul(fadd(dx, 1.0f), 0.5f), 2.0f), 1.0f), y = fsub(fmul(fmul(fadd(dy, 1.0f), 0.5f), 2.0f), 1.0f),
              z = fsub(fmul(fmul(fadd(dz, 1.0f), 0.5f), 2.0f), 1.0f);
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  c[0] = 0.28209479177387814f;
  c[1] = -0.48860251190291987f * y;
  c[2] = 0.48860251190291987f * z;
  c[3] = -0.48860251190291987f * x;
  c[4] = 1.0925484305920792f * xy;
  c[5] = -1.0925484305920792f * yz;
  c[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
  c[7] = -1.0925484305920792f * xz;
  c[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
  c[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
  c[10] = 2.8906114426405538f * xy * z;
  c[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
  c[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
  c[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
  c[14] = 1.4453057213202769f * z * (x2 - y2);
  c[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// F = 4 (16-byte rows, one LDG.128 per corner); writes feature 4l+f of this lane's sample to panel[4l+f][lane].
NFF_D void encode_f4_panel(const float* NFF_RESTRICT table, const Grid& gr, int L, Gauss g, float (*panel)[33]) {
  const int ln = lane();
#pragma unroll kF4Unroll
  for (int l = 0; l < L; ++l) {
    const float res = gr.res[l];
    Cell c = grid_cell(g.x, g.y, g.z, res);
    uint32_t r[8];
    cell_rows(c, gr.mask, r);
    const float4* base = reinterpret_cast<const float4*>(table) + (size_t)l * gr.T;
    float4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = ldg(base + r[k]);
    float w = level_weight(res, g.std);
    const float ix = 1.0f - c.ox, iy = 1.0f - c.oy, iz = 1.0f - c.oz;
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].x;
    panel[4 * l + 0][ln] = fmul(trilerp_f(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].y;
    panel[4 * l + 1][ln] = fmul(trilerp_f(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].z;
    panel[4 * l + 2][ln] = fmul(trilerp_f(f, c, ix, iy, iz), w);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = v[k].w;
    panel[4 * l + 3][ln] = fmul(trilerp_f(f, c, ix, iy, iz), w);
  }
}

// ------------------------------------------------------------------------------------------------ actors
// Per-warp shared state.  One warp == one ray.
template <int ACT_ROWS>
struct WarpSharedT {
  // The sampling scratch (cdf, resampled bins, euclidean edges) is dead once the main-field phase starts and the
  // activation panel is dead until then, so they share storage: every KB of shared memory given back is L1 cache
  // for the hash-grid gathers (unified 256 KB L1/shared per SM on sm_90).
  union {
    struct {
      float cdf[kS0 + 4];
      float bins_b[kS1 + 4];
      float bins_e[kS0 + 4];  // euclidean edges of the current level
    };
    float act[ACT_ROWS][33];  // per-lane (column) grid features / MLP activations; also the composite transpose
  };
  float bins_a[kS0 + 4];
  float w2b[kMaxCand][12];  // world->box [R^T | -R^T t], row major 3x4
  float bnd[kMaxCand][3];
  int32_t cand_id[kMaxCand];
  int32_t n_cand;
  int32_t overflow;
};
using WarpShared = WarpSharedT<kNff + kSh>;  // CUDA-core MLP path (and the host emulation)

NFF_D void normalize3(float v[3]) {  // F.normalize: v / max(|v|, 1e-12)
  float n = fsqrt(fadd(fadd(fmul(v[0], v[0]), fmul(v[1], v[1])), fmul(v[2], v[2])));
  n = fmaxf(n, 1e-12f);
  v[0] = fdiv(v[0], n);
  v[1] = fdiv(v[1], n);
  v[2] = fdiv(v[2], n);
}

// DynamicActors.get_boxes2world (model_components/dynamic_actors.py:251-268) = interpolate_trajectories_6d
// (utils/poses.py:90-150) + rotation_6d_to_matrix (cameras/camera_utils.py:422-443) + pose inverse
// (utils/poses.py:42-55), followed by the ray-line culling of NeuRADHashEncoding._get_actor_indices
// (field_components/neurad_encoding.py:225-240).  Lanes stride over actors; survivors are compacted, in
// increasing actor order, into the warp's candidate list.
template <class WS>
NFF_D void actor_candidates(const Actors& A, float time, const float o[3], const float d[3], WS& ws) {
  if (lane() == 0) {
    ws.n_cand = 0;
    ws.overflow = 0;
  }
  syncwarp();
  if (A.n_actors == 0) return;
  // torch.searchsorted(pose_times, t) (left): first index with times[idx] >= t
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
  for (int base = 0; base < A.n_actors; base += 32) {
    int a = base + lane();
    bool keep = false;
    float R[9], t[3];
    if (a < A.n_actors) {
      const float* kl = A.keyframes + ((size_t)left * A.n_actors + a) * 9;
      const float* kr = A.keyframes + ((size_t)right * A.n_actors + a) * 9;
      float p[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        float l_ = ldg(kl + i), r_ = ldg(kr + i);
        p[i] = fadd(l_, fmul(fsub(r_, l_), frac));
      }
      bool valid = (A.present[(size_t)left * A.n_actors + a] | A.present[(size_t)right * A.n_actors + a]) != 0;
      float b1[3] = {p[0], p[1], p[2]};
      normalize3(b1);
      float dt = fadd(fadd(fmul(b1[0], p[3]), fmul(b1[1], p[4])), fmul(b1[2], p[5]));
      float b2[3] = {fsub(p[3], fmul(dt, b1[0])), fsub(p[4], fmul(dt, b1[1])), fsub(p[5], fmul(dt, b1[2]))};
      normalize3(b2);
      float b3[3] = {fsub(fmul(b1[1], b2[2]), fmul(b1[2], b2[1])), fsub(fmul(b1[2], b2[0]), fmul(b1[0], b2[2])),
                     fsub(fmul(b1[0], b2[1]), fmul(b1[1], b2[0]))};
      // boxes2world rotation has rows b1,b2,b3; world2box rotation is its transpose
      R[0] = b1[0]; R[1] = b2[0]; R[2] = b3[0];
      R[3] = b1[1]; R[4] = b2[1]; R[5] = b3[1];
      R[6] = b1[2]; R[7] = b2[2]; R[8] = b3[2];
      t[0] = -fadd(fadd(fmul(R[0], p[6]), fmul(R[1], p[7])), fmul(R[2], p[8]));
      t[1] = -fadd(fadd(fmul(R[3], p[6]), fmul(R[4], p[7])), fmul(R[5], p[8]));
      t[2] = -fadd(fadd(fmul(R[6], p[6]), fmul(R[7], p[7])), fmul(R[8], p[8]));
      // distance from the box centre to the ray line (|d| == 1 up to rounding; the reference renormalises the
      // first->last sample chord, same direction)
      float v[3] = {fsub(p[6], o[0]), fsub(p[7], o[1]), fsub(p[8], o[2])};
      float cx = fsub(fmul(v[1], d[2]), fmul(v[2], d[1]));
      float cy = fsub(fmul(v[2], d[0]), fmul(v[0], d[2]));
      float cz = fsub(fmul(v[0], d[1]), fmul(v[1], d[0]));
      float dist = fsqrt(fadd(fadd(fmul(cx, cx), fmul(cy, cy)), fmul(cz, cz)));
      // the cull is conservative (a point inside the box is within |bounds| of the centre); 1e-3 relative slack
      // makes the chord-vs-direction rounding difference irrelevant
      keep = valid && dist < ldg(A.radii + a) * 1.001f;
    }
    unsigned m = vote_ballot(keep);
    int slot = ws.n_cand + popc(m & ((1u << lane()) - 1u));
    if (keep) {
      if (slot < kMaxCand) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          ws.w2b[slot][4 * i + 0] = R[3 * i + 0];
          ws.w2b[slot][4 * i + 1] = R[3 * i + 1];
          ws.w2b[slot][4 * i + 2] = R[3 * i + 2];
          ws.w2b[slot][4 * i + 3] = t[i];
          ws.bnd[slot][i] = ldg(A.bounds + 3 * a + i);
        }
        ws.cand_id[slot] = a;
      } else {
        ws.overflow = 1;
      }
    }
    syncwarp();
    if (lane() == 0) {
      int n = ws.n_cand + popc(m);
      ws.n_cand = n > kMaxCand ? kMaxCand : n;
    }
    syncwarp();
  }
}

// The per-sample part of _get_actor_indices (neurad_encoding.py:241-254): is the sample mean inside a padded
// box?  Returns the candidate slot (highest actor index wins, matching the reference's sequential index_put on
// CPU) or -1; `pb` receives the position in the box frame.
template <class WS>
NFF_D int actor_of_sample(const WS& ws, const Gauss& g, float pb[3]) {
  int hit = -1;
  int n = ws.n_cand;
  for (int c = 0; c < n; ++c) {
    const float* M = ws.w2b[c];
    float q0 = fadd(fadd(fadd(fmul(M[0], g.x), fmul(M[1], g.y)), fmul(M[2], g.z)), M[3]);
    float q1 = fadd(fadd(fadd(fmul(M[4], g.x), fmul(M[5], g.y)), fmul(M[6], g.z)), M[7]);
    float q2 = fadd(fadd(fadd(fmul(M[8], g.x), fmul(M[9], g.y)), fmul(M[10], g.z)), M[11]);
    if (fabsf(q0) < ws.bnd[c][0] && fabsf(q1) < ws.bnd[c][1] && fabsf(q2) < ws.bnd[c][2]) {
      hit = c;
      pb[0] = q0; pb[1] = q1; pb[2] = q2;
    }
  }
  return hit;
}

// ------------------------------------------------------------------------------------- proposal density
// NeuRADProposalField.get_density (fields/neurad_field.py:208-213) for one sample:
// NeuRADHashEncoding.forward (static grid, or the containing actor's grid zero-padded) -> Linear(6,1) -> exp.
template <class WS>
NFF_D float proposal_density(const FieldGrids& fg, const WS& ws, const Gauss& g, int* actor_id) {
  float pb[3];
  int c = actor_of_sample(ws, g, pb);
  float acc;
  if (c >= 0) {
    Gauss ga = {pb[0], pb[1], pb[2], g.std};
    ga = contract(ga, fg.actor_scale);
    // actor features occupy the first 4 of the 6 decoder inputs; the zero padding contributes nothing
    acc = encode_f1_dot<4, NFF_G_ACT>(fg.actor_tables[ws.cand_id[c]], fg.act, ga, fg.decoder);
    *actor_id = ws.cand_id[c];
  } else {
    Gauss gs = contract(g, fg.static_scale);
    acc = encode_f1_dot<6, NFF_G_PROP>(fg.stat.table, fg.stat, gs, fg.decoder);
    *actor_id = -1;
  }
  return expf(acc);
}

// ----------------------------------------------------------------------------------------------- MLPs
// y = W x + b with W stored transposed [IN][OUTP] in shared memory: every lane owns one sample (row); a weight
// quad is one broadcast LDS.128 feeding 4 FFMAs.
template <int IN, int OUT, int OUTP, bool RELU>
NFF_D void dense(const float* NFF_RESTRICT W, const float* NFF_RESTRICT B, const float* x, float* y) {
  float acc[OUTP];
#pragma unroll
  for (int o = 0; o < OUTP; ++o) acc[o] = o < OUT ? B[o] : 0.0f;
#pragma unroll
  for (int k = 0; k < IN; ++k) {
    const float xk = x[k];
#pragma unroll
    for (int o4 = 0; o4 < OUTP / 4; ++o4) {
      const float4 w = *reinterpret_cast<const float4*>(W + k * OUTP + 4 * o4);
      acc[4 * o4 + 0] = fmaf(xk, w.x, acc[4 * o4 + 0]);
      acc[4 * o4 + 1] = fmaf(xk, w.y, acc[4 * o4 + 1]);
      acc[4 * o4 + 2] = fmaf(xk, w.z, acc[4 * o4 + 2]);
      acc[4 * o4 + 3] = fmaf(xk, w.w, acc[4 * o4 + 3]);
    }
  }
#pragma unroll
  for (int o = 0; o < OUT; ++o) y[o] = RELU ? fmaxf(acc[o], 0.0f) : acc[o];
}

// Same product, but the input row lives in the warp's shared-memory panel act[k][lane] and the k-loop stays rolled:
// keeps the kernel small enough for the instruction cache (the fully unrolled form is ~27k SASS instructions and
// stalls on instruction fetch).
template <int IN, int OUT, int OUTP>
NFF_D void dense_panel(const float* NFF_RESTRICT W, const float* NFF_RESTRICT B, const float (*act)[33], float* acc) {
  const int ln = lane();
#pragma unroll
  for (int o = 0; o < OUTP; ++o) acc[o] = o < OUT ? B[o] : 0.0f;
#pragma unroll 2
  for (int k = 0; k < IN; ++k) {
    const float xk = act[k][ln];
#pragma unroll
    for (int o4 = 0; o4 < OUTP / 4; ++o4) {
      const float4 w = *reinterpret_cast<const float4*>(W + k * OUTP + 4 * o4);
      acc[4 * o4 + 0] = fmaf(xk, w.x, acc[4 * o4 + 0]);
      acc[4 * o4 + 1] = fmaf(xk, w.y, acc[4 * o4 + 1]);
      acc[4 * o4 + 2] = fmaf(xk, w.z, acc[4 * o4 + 2]);
      acc[4 * o4 + 3] = fmaf(xk, w.w, acc[4 * o4 + 3]);
    }
  }
}

// components_from_spherical_harmonics(levels=4) (utils/math.py:31-94) on (d+1)/2 (fields/base_field.py:136-142)
NFF_D void sh4_poly(float x, float y, float z, float* c) {
  float xx = x * x, yy = y * y, zz = z * z;
  c[0] = 0.28209479177387814f;
  c[1] = 0.4886025119029199f * y;
  c[2] = 0.4886025119029199f * z;
  c[3] = 0.4886025119029199f * x;
  c[4] = 1.0925484305920792f * x * y;
  c[5] = 1.0925484305920792f * y * z;
  c[6] = 0.9461746957575601f * zz - 0.31539156525251999f;
  c[7] = 1.0925484305920792f * x * z;
  c[8] = 0.5462742152960396f * (xx - yy);
  c[9] = 0.5900435899266435f * y * (3.0f * xx - yy);
  c[10] = 2.890611442640554f * x * y * z;
  c[11] = 0.4570457994644658f * y * (5.0f * zz - 1.0f);
  c[12] = 0.3731763325901154f * z * (5.0f * zz - 3.0f);
  c[13] = 0.4570457994644658f * x * (5.0f * zz - 1.0f);
  c[14] = 1.445305721320277f * z * (xx - yy);
  c[15] = 0.5900435899266435f * x * (xx - 3.0f * yy);
}
NFF_D void sh4(float dx, float dy, float dz, float* c) {
  sh4_poly(fmul(fadd(dx, 1.0f), 0.5f), fmul(fadd(dy, 1.0f), 0.5f), fmul(fadd(dz, 1.0f), 0.5f), c);
}

// --------------------------------------------------------------------------------- proposal round + resample
// One proposal round for the warp's ray: densities (NeuRADProposalField.get_density) -> RaySamples.get_weights
// (cameras/rays.py:188-210) -> prop depth (render_depth_simple, models/neurad.py:727-734) -> PDFSampler
// (ray_samplers.py:309-361) producing S_new+1 new spacing-domain edges.  `bins_in` holds the S+1 spacing edges of
// the current level, `bins_out` receives the new ones (both in shared memory).  Chunks of 32 samples are a rolled
// loop; per-sample weights are parked in ws.cdf[] between the two passes.
struct RoundIO {
  int S, S_new;
  const float* u_tab;
  const float* bins_in;
  float* bins_out;
  float* tr_w;
  int32_t* tr_aid;
  float* tr_bins_s;
  float* tr_bins_e;
  int32_t* tr_inds;
};
template <class WS>
NFF_D float proposal_round(const RenderParams& P, const FieldGrids& fg, WS& ws, const RoundIO& io,
                           const float o[3], const float d[3], float area, float s_near, float s_far, int64_t ray) {
  const Sampling& sp = P.samp;
  const int S = io.S, S_new = io.S_new, ln = lane();
  float carry = 0.0f, depth_acc = 0.0f, part = 0.0f;
  // spacing -> euclidean for the S+1 edges, once (each edge is shared by two samples)
#pragma unroll 1
  for (int i = ln; i <= S; i += 32) ws.bins_e[i] = to_euclid(io.bins_in[i], s_near, s_far, sp);
  syncwarp();
  // NFF_ILP chunks (of 32 samples) are processed together: each lane carries NFF_ILP independent samples through
  // gaussian -> contraction -> gathers -> interpolation, which is what fills the issue slots of a kernel that runs
  // at 4 warps per scheduler
  constexpr int U = NFF_ILP;
#pragma unroll 1
  for (int s0 = 0; s0 < S; s0 += 32 * U) {
    float e0[U], e1[U], dd[U];
    int aid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int s = s0 + 32 * u + ln;
      e0[u] = ws.bins_e[s];
      e1[u] = ws.bins_e[s + 1];
      Gauss g = sample_gaussian(o, d, area, e0[u], e1[u]);
      float dens = proposal_density(fg, ws, g, &aid[u]);
      dd[u] = fmul(fsub(e1[u], e0[u]), dens);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int s = s0 + 32 * u + ln;
      float incl = warp_scan_add(dd[u]);
      float prev = shfl_up(incl, 1);
      float excl = carry + (ln == 0 ? 0.0f : prev);
      carry += shfl(incl, 31);
      float alpha = fsub(1.0f, expf(-dd[u]));
      float T = expf(-excl);
      float wj = nan_to_num(fmul(alpha, T));
      depth_acc = fadd(depth_acc, fmul(wj, fmul(fadd(e0[u], e1[u]), 0.5f)));
      if (io.tr_w) io.tr_w[ray * S + s] = wj;
      if (io.tr_aid) io.tr_aid[ray * S + s] = aid[u];
      wj = fadd(wj, sp.hist_pad);  // PDFSampler: histogram padding
      ws.cdf[s + 1] = wj;
      part += wj;
    }
  }
  const float prop_depth = warp_sum(depth_acc);
  float tot = warp_sum(part);
  const float padding = fmaxf(fsub(1e-5f, tot), 0.0f);
  const float pad_each = fdiv(padding, (float)S);
  tot = fadd(tot, padding);
  carry = 0.0f;
#pragma unroll 1
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + ln;
    float pdf = fdiv(fadd(ws.cdf[s + 1], pad_each), tot);
    float incl = warp_scan_add(pdf) + carry;
    carry = shfl(incl, 31);
    ws.cdf[s + 1] = fminf(1.0f, incl);
  }
  if (ln == 0) ws.cdf[0] = 0.0f;
  syncwarp();
  // inverse-cdf sampling: inds = searchsorted(cdf, u, side="right")
#pragma unroll 1
  for (int i = ln; i <= S_new; i += 32) {
    float u = ldg(io.u_tab + i);
    int lo = 0, hi = S + 1;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (ws.cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    int below = lo - 1 < 0 ? 0 : (lo - 1 > S ? S : lo - 1);
    int above = lo > S ? S : lo;
    float c0 = ws.cdf[below], c1 = ws.cdf[above];
    float b0 = io.bins_in[below], b1 = io.bins_in[above];
    float t = nan_to_num(fdiv(fsub(u, c0), fsub(c1, c0)));
    t = fminf(fmaxf(t, 0.0f), 1.0f);
    float nb = fadd(b0, fmul(t, fsub(b1, b0)));
    io.bins_out[i] = nb;
    if (io.tr_inds) io.tr_inds[ray * (S_new + 1) + i] = lo;
    if (io.tr_bins_s) io.tr_bins_s[ray * (S_new + 1) + i] = nb;
    if (io.tr_bins_e) io.tr_bins_e[ray * (S_new + 1) + i] = to_euclid(nb, s_near, s_far, sp);
  }
  syncwarp();
  return prop_depth;
}

// ------------------------------------------------------------------------------------ main-field MLP policies
// NeuRADField.forward after the grid lookup (fields/neurad_field.py:138-142): mlp_geo -> (sdf | geo_embedding),
// SH(dir), feature = geo_embedding + mlp_feature([geo_embedding, sh]).  Input: this lane's 32 grid features in
// ws.act[0..31][lane].
//
// CUDA-core path: fp32 FFMA, weights transposed in shared memory (exact-fp32 reference mode; also what the host
// emulation runs).
struct MlpFfma {
  const float* w;  // packed (nff_params.h), in shared memory
  template <class WS>
  NFF_D void run(WS& ws, const float dir[3], float& sdf, float* feat) const {
    const int ln = lane();
    const float* mlp = w;
    float mac[kGeoOutP];
    dense_panel<kGeoIn, kHidden, kHidden>(mlp + kOffGeoW0, mlp + kOffGeoB0, ws.act, mac);
#pragma unroll
    for (int i = 0; i < kHidden; ++i) ws.act[i][ln] = fmaxf(mac[i], 0.0f);
    dense_panel<kHidden, kNff + 1, kGeoOutP>(mlp + kOffGeoW1, mlp + kOffGeoB1, ws.act, mac);
    sdf = mac[0];
    float geo[kNff];  // geo_embedding, kept for the residual
#pragma unroll
    for (int i = 0; i < kNff; ++i) {
      geo[i] = mac[i + 1];
      ws.act[i][ln] = geo[i];
    }
    {
      float shv[kSh];
      sh4(dir[0], dir[1], dir[2], shv);
#pragma unroll
      for (int i = 0; i < kSh; ++i) ws.act[kNff + i][ln] = shv[i];
    }
    dense_panel<kNff + kSh, kHidden, kHidden>(mlp + kOffFeatW0, mlp + kOffFeatB0, ws.act, mac);
#pragma unroll
    for (int i = 0; i < kHidden; ++i) ws.act[i][ln] = fmaxf(mac[i], 0.0f);
    dense_panel<kHidden, kHidden, kHidden>(mlp + kOffFeatW1, mlp + kOffFeatB1, ws.act, mac);
#pragma unroll
    for (int i = 0; i < kHidden; ++i) ws.act[i][ln] = fmaxf(mac[i], 0.0f);
    dense_panel<kHidden, kNff, kNff>(mlp + kOffFeatW2, mlp + kOffFeatB2, ws.act, mac);
#pragma unroll
    for (int i = 0; i < kNff; ++i) feat[i] = geo[i] + mac[i];  // residual (neurad_field.py:141)
  }
};

#if defined(__CUDACC__)
}  // namespace nff
#include "tc_mlp.cuh"
namespace nff {
// Tensor-core path: a tile = the 4 warps (4 rays x 32 samples = 128 rows) of one warp group; every layer is a wgmma
// tile product through the group's shared-memory stage (tc_mlp.cuh: 3xTF32 split, fp32-level accuracy), the weights are
// staged once per CTA in shared memory.  The sdf neuron (row 0 of mlp_geo's last layer) is one 32-term dot product on
// the CUDA cores so that all tensor-core layers have N = 32.
constexpr int kTcLayers = 5;
constexpr int kTcPitch = tc::stage_pitch(48);     // stage row pitch (floats) for K <= 48, N = 32
constexpr int kTcStageFloats = 128 * kTcPitch;    // one warp group's stage (26 KB)
struct TcShared {
  float b[2 * 32 * (32 + 32 + 48 + 32 + 32)];  // hi|lo B tiles of the 5 layers (45 KB)
  float bias[kTcLayers][32];
  float w_sdf[32];
  float b_sdf;
};
constexpr int kTcBytes = (sizeof(TcShared) + 127) / 128 * 128;
// dynamic shared memory of a tensor-core render kernel up to its own part: TcShared, then one stage per warp group
constexpr size_t tc_smem_bytes(int threads) { return (size_t)kTcBytes + (size_t)(threads / 128) * kTcStageFloats * sizeof(float); }
NFF_D constexpr int tc_layer_k(int l) { return l == 2 ? 48 : 32; }
NFF_D constexpr int tc_layer_off(int l) { return l == 0 ? 0 : l == 1 ? 2048 : l == 2 ? 4096 : l == 3 ? 7168 : 9216; }

// cooperative (whole CTA): build the B tiles from the nn.Linear-layout weights in global memory.  `chained`: layers 1-4
// take their first 32 inputs straight from the previous layer's accumulator fragments (MlpLaneTc, nff_lane.h), so those
// K rows are permuted (tc::chained_k).
NFF_D void tc_stage_weights(TcShared& t, const float* NFF_RESTRICT nn, int tid, int nthreads, bool chained = false) {
  const int w_off[kTcLayers] = {kNnGeoW0, kNnGeoW1 + kHidden /* rows 1..32 */, kNnFeatW0, kNnFeatW1, kNnFeatW2};
  const int b_off[kTcLayers] = {kNnGeoB0, kNnGeoB1 + 1, kNnFeatB0, kNnFeatB1, kNnFeatB2};
#pragma unroll
  for (int l = 0; l < kTcLayers; ++l) {
    const int K = tc_layer_k(l);
    float* hi = t.b + tc_layer_off(l);
    tc::stage_b_tile(hi, hi + 32 * K, nn + w_off[l], 32, K, 32, K, tid, nthreads, chained && l > 0 ? 32 : 0);
    for (int i = tid; i < 32; i += nthreads) t.bias[l][i] = nn[b_off[l] + i];
  }
  for (int i = tid; i < 32; i += nthreads) t.w_sdf[i] = nn[kNnGeoW1 + i];
  if (tid == 0) t.b_sdf = nn[kNnGeoB1];
}

struct MlpTc {
  const TcShared* t;
  float* stage;  // this warp group's [128][kTcPitch] stage
  int bar_id;    // this warp group's named barrier

  // run layer l for this thread's row (K activations) on the tensor cores: the 32 outputs + bias -> out
  template <int K>
  NFF_D void layer(int l, const float* x, float* out) {
    const float* hi = t->b + tc_layer_off(l);
    const int id = bar_id;
    tc::tile_layer<48, 32>(stage, kTcPitch, x, K, hi, hi + 32 * K, out, [id] { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); });
#pragma unroll
    for (int i = 0; i < 32; ++i) out[i] += t->bias[l][i];
  }

  template <class WS>
  NFF_D void run(WS& ws, const float dir[3], float& sdf, float* feat) {
    const int ln = lane();
    float x[kNff + kSh], h[kHidden];
#pragma unroll
    for (int i = 0; i < kGeoIn; ++i) x[i] = ws.act[i][ln];
    layer<32>(0, x, h);
    float s = t->b_sdf;
#pragma unroll
    for (int i = 0; i < kHidden; ++i) {
      h[i] = fmaxf(h[i], 0.0f);
      s = fmaf(h[i], t->w_sdf[i], s);
    }
    sdf = s;
    layer<32>(1, h, x);  // x[0..31] = geo_embedding (kept for the residual)
    sh4(dir[0], dir[1], dir[2], x + kNff);
    layer<48>(2, x, h);
#pragma unroll
    for (int i = 0; i < kHidden; ++i) h[i] = fmaxf(h[i], 0.0f);
    float h2[kHidden];
    layer<32>(3, h, h2);
#pragma unroll
    for (int i = 0; i < kHidden; ++i) h2[i] = fmaxf(h2[i], 0.0f);
    layer<32>(4, h2, h);
#pragma unroll
    for (int i = 0; i < kNff; ++i) feat[i] = x[i] + h[i];
  }
};
#endif  // __CUDACC__

// --------------------------------------------------------------------------------------- the whole ray
// NeuRADModel.get_nff_outputs (models/neurad.py:368-421), eval mode.  `active == false` renders a (clamped, valid)
// ray without storing anything: warps of a tensor-core tile must all take part in the tile's barriers.
template <class WS, class Mlp>
NFF_D void render_ray(const RenderParams& P, WS& ws, Mlp& mlp, int64_t ray, bool active) {
  const Sampling& sp = P.samp;
  const int ln = lane();
  float o[3], d[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    o[i] = ldg(P.rays.origins + 3 * ray + i);
    d[i] = ldg(P.rays.directions + 3 * ray + i);
  }
  const bool lidar = P.rays.is_lidar ? P.rays.is_lidar[ray] != 0 : false;
  // _scale_pixel_area (neurad.py:702-709)
  float area = fmul(ldg(P.rays.pixel_area + ray), lidar ? 1.0f : sp.cam_area_scale);
  const float time = ldg(P.rays.times + ray);
  // _get_ray_samples (neurad.py:443-449)
  float far_ = P.rays.fars ? ldg(P.rays.fars + ray) : 1.0e6f;
  far_ = fminf(far_, sp.sky_distance);
  float near_ = P.rays.nears ? ldg(P.rays.nears + ray) : 0.0f;
  const float s_near = spacing_fn(near_, sp), s_far = spacing_fn(far_, sp);

  actor_candidates(P.actors, time, o, d, ws);
#if defined(__CUDACC__)
  if (ws.overflow && P.status && ln == 0) atomicExch(P.status, 3);  // > kMaxCand actors along one ray: fail loudly
#endif

  // level-0 spacing bins: torch.linspace(0, 1, S0+1) (ray_samplers.py:102)
  for (int i = ln; i <= kS0; i += 32) ws.bins_a[i] = linspace01(i, kS0);
  syncwarp();
  float prop_depth[2];
#pragma unroll 1
  for (int rd = 0; rd < 2; ++rd) {
    RoundIO io;
    io.S = rd == 0 ? kS0 : kS1;
    io.S_new = rd == 0 ? kS1 : kS2;
    io.u_tab = rd == 0 ? sp.u1 : sp.u2;
    io.bins_in = rd == 0 ? ws.bins_a : ws.bins_b;
    io.bins_out = rd == 0 ? ws.bins_b : ws.bins_a;
    io.tr_w = !active ? nullptr : rd == 0 ? P.trace.prop_weights_0 : P.trace.prop_weights_1;
    io.tr_aid = !active ? nullptr : rd == 0 ? P.trace.actor_id_0 : P.trace.actor_id_1;
    io.tr_bins_s = !active ? nullptr : rd == 0 ? P.trace.bins_s_1 : P.trace.bins_s_2;
    io.tr_bins_e = !active ? nullptr : rd == 0 ? P.trace.bins_e_1 : P.trace.bins_e_2;
    io.tr_inds = !active ? nullptr : rd == 0 ? P.trace.inds_1 : P.trace.inds_2;
    prop_depth[rd] = proposal_round(P, P.fields[sp.field_of_round[rd]], ws, io, o, d, area, s_near, s_far, ray);
  }
  const float prop_depth_0 = prop_depth[0], prop_depth_1 = prop_depth[1];

  // ---- main field: one sample per lane (fields/neurad_field.py:128-152) ----
  float e0 = to_euclid(ws.bins_a[ln], s_near, s_far, sp);
  float e1 = to_euclid(ws.bins_a[ln + 1], s_near, s_far, sp);
  if (ln == kS2 - 1) e1 = fadd(e1, fsub(sp.sky_distance, e1));  // sky sample (neurad.py:451-455)
  Gauss g = sample_gaussian(o, d, area, e0, e1);
  const FieldGrids& fm = P.fields[B200NERF_FIELD_MAIN];
  float dir[3] = {d[0], d[1], d[2]};
  int aid = -1;
  {
    float pb[3];
    int c = actor_of_sample(ws, g, pb);
    if (c >= 0) {
      aid = ws.cand_id[c];
      Gauss ga = {pb[0], pb[1], pb[2], g.std};
      ga = contract(ga, fm.actor_scale);
#pragma unroll
      for (int i = 16; i < 32; ++i) ws.act[i][ln] = 0.0f;  // F.pad(actor_features, (0, 32-16))
      encode_f4_panel(fm.actor_tables[aid], fm.act, 4, ga, ws.act);
      // direction into the box frame, renormalised with +EPS (neurad_encoding.py:203-209)
      const float* M = ws.w2b[c];
      float q0 = fadd(fadd(fmul(M[0], d[0]), fmul(M[1], d[1])), fmul(M[2], d[2]));
      float q1 = fadd(fadd(fmul(M[4], d[0]), fmul(M[5], d[1])), fmul(M[6], d[2]));
      float q2 = fadd(fadd(fmul(M[8], d[0]), fmul(M[9], d[1])), fmul(M[10], d[2]));
      float n = fadd(fsqrt(fadd(fadd(fmul(q0, q0), fmul(q1, q1)), fmul(q2, q2))), 1.0e-7f);
      dir[0] = fdiv(q0, n); dir[1] = fdiv(q1, n); dir[2] = fdiv(q2, n);
    } else {
      Gauss gs = contract(g, fm.static_scale);
      encode_f4_panel(fm.stat.table, fm.stat, 8, gs, ws.act);
    }
  }
  syncwarp();
  float sdf, feat[kNff];
  mlp.run(ws, dir, sdf, feat);
  // SigmoidDensity (model_components/utils.py:29-41): alpha = sigmoid(-sdf * beta)
  const float alpha = frcp(fadd(1.0f, expf(fmul(sdf, P.beta))));

  // nerfacc.render_weight_from_alpha (neurad.py:717): w_i = alpha_i * prod_{j<i} (1 - alpha_j)
  float incl = warp_scan_mul(fsub(1.0f, alpha));
  float prevT = shfl_up(incl, 1);
  float T = ln == 0 ? 1.0f : prevT;
  float w = fmul(alpha, T);
  const float acc = warp_sum(w);  // AccumulationRenderer (renderers.py:349)
  // depth over the non-sky samples (neurad.py:388-389, 727-734)
  float dterm = ln < kS2 - 1 ? fmul(w, fmul(fadd(e0, e1), 0.5f)) : 0.0f;
  const float depth = warp_sum(dterm);
  if (ln == kS2 - 1) w = fadd(fadd(w, 1.0f), -acc);  // remaining accumulation onto the sky sample (neurad.py:381)

  if (active && P.trace.sdf) P.trace.sdf[ray * kS2 + ln] = sdf;
  if (active && P.trace.alpha) P.trace.alpha[ray * kS2 + ln] = alpha;
  if (active && P.trace.weights) P.trace.weights[ray * kS2 + ln] = w;
  if (active && P.trace.actor_id_main) P.trace.actor_id_main[ray * kS2 + ln] = aid;
  if (active && P.trace.field_feature) {
#pragma unroll
    for (int i = 0; i < kNff; ++i) P.trace.field_feature[(ray * kS2 + ln) * kNff + i] = feat[i];
  }

  // FeatureRenderer: sum_s w_s * feat_s (renderers.py:85) via a padded shared-memory transpose
#pragma unroll
  for (int i = 0; i < kNff; ++i) ws.act[i][ln] = fmul(feat[i], w);
  syncwarp();
  float fsum = 0.0f;
#pragma unroll 8
  for (int s = 0; s < kS2; ++s) fsum = fadd(fsum, ws.act[ln][s]);
  syncwarp();

  if (!active) return;
  const int fdim = P.nff_dim + P.app.dim;
  float* fo = P.out.features + ray * fdim;
  fo[ln] = fsum;
  // _get_appearance_embedding (neurad.py:423-441); eps == 0: the per-sensor branch (:440), row `sensor_idx` copied
  float app = 0.0f;
  if (ln < P.app.dim) {
    const bool per_sensor = P.app.eps == 0;
    float sens = P.rays.sensor_idx ? (float)P.rays.sensor_idx[ray] : 0.0f;
    float eps_ = (float)P.app.eps;
    float tidx = fmul(fdiv(time, P.app.duration), eps_);
    float before = fminf(fmaxf(floorf(tidx), 0.0f), eps_ - 1.0f);
    float after = fminf(fmaxf(fadd(before, 1.0f), 0.0f), eps_ - 1.0f);
    float ratio = fsub(tidx, before);
    int ib = (int)fadd(before, fmul(sens, eps_)), ia = (int)fadd(after, fmul(sens, eps_));
    if (per_sensor) ib = ia = (int)sens;
    float eb = ldg(P.app.emb + (size_t)ib * P.app.dim + ln), ea = ldg(P.app.emb + (size_t)ia * P.app.dim + ln);
    app = per_sensor ? eb : fadd(fmul(eb, fsub(1.0f, ratio)), fmul(ea, ratio));
    fo[P.nff_dim + ln] = app;
  }
  if (ln == 0) {
    P.out.depth[ray] = depth;
    P.out.accumulation[ray] = acc;
    P.out.prop_depth_0[ray] = prop_depth_0;
    P.out.prop_depth_1[ray] = prop_depth_1;
  }
}

}  // namespace nff
