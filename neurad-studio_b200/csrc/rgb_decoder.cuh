// rgb_decoder.cuh -- NeuRADModel.rgb_decoder (models/neurad.py:201-216, model_components/cnns.py:19-46) in eval mode:
//   Conv2d(in->32, 1x1) + ReLU -> 2 x BasicBlock(32, 7x7, BN) -> ConvTranspose2d(32->32, k = s = 3) -> 2 x BasicBlock
//   -> Conv2d(32->3, 1x1) -> Sigmoid,            feature image [B,H,W,in] (row-major rays) -> rgb [B,3H,3W,3].
//
// 97 % of the work is the eight 7x7 convolutions (50 176 MAC per pixel each).  They run as implicit GEMMs on the
// Hopper warp-group tensor cores (wgmma): M = 128 consecutive pixels of one image row (two m64 tiles, one per warp
// group), N = 32 output channels, K = 49 taps x 32 input channels, fp32 accumulators in registers.  BatchNorm is folded
// into the conv weights/bias when the parameters are set.
//
// fp32-level accuracy from bf16 tensor-core inputs: every activation and weight is split into two bf16 numbers
// (hi = bf16(v), lo = bf16(v - hi)) and each k-step issues three MMAs  a_hi*w_hi + a_lo*w_hi + a_hi*w_lo  into the
// same accumulator; the dropped a_lo*w_lo term is <= 2^-16 |a||w| (~2^-18 typical).  This costs 1.5x the tensor time of a single TF32
// pass (bf16 runs at twice the TF32 rate) and needs exactly the bytes of fp32 storage.
//
// Activations between layers therefore live in HBM already split ("ACT" layout): per pixel 128 B = 8 chunks of 8 bf16,
// chunk c < 4: hi of channels 8c..8c+7, chunk 4+c: lo.  A conv CTA copies a (4+6) x (128+6) pixel window of it into
// shared memory as 8 planes [chunk][row][pixel][16 B]; in that layout the A operand of tap (dy,dx) for output row r is
// the SAME planes read from a shifted start address ((r+dy)*PW + dx)*16 B -- the canonical K-major no-swizzle GMMA
// layout with SBO = 128 B (8-pixel groups are contiguous) and LBO = the plane stride -- so the im2col matrix is never
// materialised.  The folded weights of one tap COLUMN dx ({hi,lo} x 7 taps x 32x32 bf16 = 28 KB, pre-arranged in the
// GMMA B layout by dec_fold_conv_kernel) are double-buffered in shared memory and streamed from L2 while the tensor
// core works on the previous column.
//
// Each A block is read once for ALL the output rows it feeds: input row i at shift dx feeds output row r through tap
// dy = i - r.  With the four accumulators side by side ([D0|D1|D2|D3]) and the tap tiles in descending dy, that is ONE
// MMA with N = 32..128.  The accumulators start from the folded bias.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

#include "tc_mlp.cuh"

namespace dec {

constexpr int kC = 32;           // hidden channels (rgb_hidden_dim)
constexpr int kUp = 3;           // rgb_upsample_factor
constexpr int kK7 = 7, kPad = 3; // BasicBlock kernel_size / padding
constexpr int kTaps = kK7 * kK7;
constexpr int kStrip = 128;      // pixels per MMA (M)
constexpr int kPW = kStrip + 2 * kPad;
constexpr int kTH = 4;           // output rows per tile
constexpr int kIR = kTH + 2 * kPad;
constexpr int kPlaneBytes = (kIR * kPW * 16 + 127) / 128 * 128;  // TMA destinations are 128-byte aligned
constexpr int kActBytes = 8 * kPlaneBytes;
constexpr int kWTileBytes = kC * kC * 2;                 // one 32x32 bf16 B tile
constexpr int kWRowBytes = kK7 * 2 * kWTileBytes;        // one tap column: {hi, lo} x 7 taps (dy descending)
constexpr int kConvThreads = 256;                        // two warp groups, 64 pixels of the strip each

struct ConvSmem {
  alignas(128) unsigned char act[kActBytes];
  alignas(128) unsigned char w[2][kWRowBytes];
  float bias[kC];
  float out_w[3 * kC];
  float out_b[4];
  alignas(8) uint64_t bar_w[2];    // TMA kernel: weight column landed in w[b]
  alignas(8) uint64_t bar_win;     // TMA kernel: input window landed
  volatile int abort;  // a completion barrier timed out: every thread leaves after the tile's last block-wide sync
};

static_assert(sizeof(ConvSmem) <= 227 * 1024, "ConvSmem exceeds the 227 KB a CTA may opt in to");

// ------------------------------------------------------------------------------------------------ bf16 split
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// two fp32 -> packed bf16x2 hi word and lo word (element 0 in the low half = lower address)
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// 32 channels of one pixel -> ACT (8 x uint4), registers only
__device__ __forceinline__ void store_act(uint4* dst, const float* v) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint4 h, l;
    split_pack2(v[8 * c + 0], v[8 * c + 1], h.x, l.x);
    split_pack2(v[8 * c + 2], v[8 * c + 3], h.y, l.y);
    split_pack2(v[8 * c + 4], v[8 * c + 5], h.z, l.z);
    split_pack2(v[8 * c + 6], v[8 * c + 7], h.w, l.w);
    dst[c] = h;
    dst[4 + c] = l;
  }
}
__device__ __forceinline__ void unpack2(uint32_t h, uint32_t l, float& a, float& b) {
  a = __uint_as_float(h << 16) + __uint_as_float(l << 16);
  b = __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u);
}
__device__ __forceinline__ void load_act(const uint4* src, float* v) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const uint4 h = src[c], l = src[4 + c];
    unpack2(h.x, l.x, v[8 * c + 0], v[8 * c + 1]);
    unpack2(h.y, l.y, v[8 * c + 2], v[8 * c + 3]);
    unpack2(h.z, l.z, v[8 * c + 4], v[8 * c + 5]);
    unpack2(h.w, l.w, v[8 * c + 6], v[8 * c + 7]);
  }
}

// ---------------------------------------------------------------------------------------- parameter preparation
// Conv2d [co][ci][7][7] + BatchNorm2d (eval) -> folded  w' = w * s[co],  b' = (b - mean) * s + beta,  s = gamma /
// sqrt(var + eps)  (BasicBlock.main_branch, cnns.py:37-43), written as
//   w_img : [dx][hi|lo][6 - dy] 32x32 bf16 tiles in the GMMA K-major no-swizzle B layout (n = co, k = ci):
//           byte offset of (n,k) = (n/8)*512 + (k/8)*128 + (n%8)*16 + (k%8)*2.  Tiles of one tap COLUMN are contiguous
//           in DESCENDING dy, so that [W(dy), W(dy-1), W(dy-2)] is one N = 96 B operand (see issue_window_row)
//   w_f32 : [dy][dx][ci][co] fp32 (CUDA-core reference kernel)
//   bias  : [co]
__global__ void dec_fold_conv_kernel(const float* __restrict__ w, const float* __restrict__ b, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ var,
                                     float eps, unsigned char* __restrict__ w_img, float* __restrict__ w_f32, float* __restrict__ bias) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kC) {
    const float s = gamma[i] / sqrtf(var[i] + eps);
    bias[i] = (b[i] - mean[i]) * s + beta[i];
  }
  if (i >= kTaps * kC * kC) return;
  const int co = i / (kC * kTaps), ci = (i / kTaps) % kC, tap = i % kTaps;  // i = flat index of w[co][ci][dy][dx]
  const float s = gamma[co] / sqrtf(var[co] + eps);
  const float v = w[i] * s;
  w_f32[(tap * kC + ci) * kC + co] = v;
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  const int off = (co >> 3) * 512 + (ci >> 3) * 128 + (co & 7) * 16 + (ci & 7) * 2;
  const int dy = tap / kK7, dx = tap % kK7;
  unsigned char* tile = w_img + (size_t)dx * kWRowBytes + (size_t)(kK7 - 1 - dy) * kWTileBytes;
  *reinterpret_cast<__nv_bfloat16*>(tile + off) = hi;
  *reinterpret_cast<__nv_bfloat16*>(tile + kK7 * kWTileBytes + off) = lo;
}

// ------------------------------------------------------------------------------------- 1x1 input conv + ReLU
// rgb_decoder.0/.1: features fp32 [P, in_dim] -> ACT [P]; w [32][in_dim], b [32] (Conv2d 1x1 layout)
__global__ void dec_input_kernel(const float* __restrict__ x, int64_t n_pix, int in_dim, const float* __restrict__ w,
                                 const float* __restrict__ b, uint4* __restrict__ out) {
  extern __shared__ float sw[];  // [in_dim][32] transposed + bias
  for (int i = threadIdx.x; i < in_dim * kC; i += blockDim.x) sw[(i % in_dim) * kC + i / in_dim] = w[i];
  for (int i = threadIdx.x; i < kC; i += blockDim.x) sw[in_dim * kC + i] = b[i];
  __syncthreads();
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pix) return;
  float acc[kC];
#pragma unroll
  for (int k = 0; k < kC; ++k) acc[k] = sw[in_dim * kC + k];
  for (int c = 0; c < in_dim; ++c) {
    const float v = x[p * in_dim + c];
#pragma unroll
    for (int k = 0; k < kC; ++k) acc[k] = fmaf(v, sw[c * kC + k], acc[k]);
  }
#pragma unroll
  for (int k = 0; k < kC; ++k) acc[k] = fmaxf(acc[k], 0.f);
  store_act(out + p * 8, acc);
}

// --------------------------------------------------------------------------- ConvTranspose2d, kernel = stride = 3
// rgb_decoder.4: out[3y+i][3x+j][co] = b[co] + sum_ci in[y][x][ci] * w[ci][co][i][j].  One thread owns TWO input pixels
// and produces their 2 x 9 output pixels; the weights [ij][ci][co] sit in shared memory and every read is a warp-wide
// broadcast feeding 8 FMAs (2 pixels x 4 channels).
constexpr int kUpThreads = 128;
__global__ void __launch_bounds__(kUpThreads) dec_upsample_kernel(const uint4* __restrict__ in, int batch, int H, int W,
                                                                   const float* __restrict__ w, const float* __restrict__ b,
                                                                   uint4* __restrict__ out) {
  extern __shared__ __align__(16) float sw[];  // [i*3+j][ci][co] + bias
  for (int i = threadIdx.x; i < kC * kC * kUp * kUp; i += blockDim.x) {
    const int ci = i / (kC * 9), co = (i / 9) % kC, ij = i % 9;
    sw[(ij * kC + ci) * kC + co] = w[i];
  }
  for (int i = threadIdx.x; i < kC; i += blockDim.x) sw[9 * kC * kC + i] = b[i];
  __syncthreads();
  const int64_t n_in = (int64_t)batch * H * W;
  const int64_t p0 = ((int64_t)blockIdx.x * kUpThreads + threadIdx.x) * 2;
  if (p0 >= n_in) return;
  const bool two = p0 + 1 < n_in;
  float v0[kC], v1[kC];
  load_act(in + p0 * 8, v0);
  load_act(in + (two ? p0 + 1 : p0) * 8, v1);
  const int64_t WO = (int64_t)W * kUp;
  int64_t base[2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int64_t p = p0 + q, img = p / ((int64_t)H * W), y = (p / W) % H, x = p % W;
    base[q] = (img * H * kUp + y * kUp) * WO + x * kUp;
  }
#pragma unroll 1
  for (int ij = 0; ij < 9; ++ij) {
    float a0[kC], a1[kC];
#pragma unroll
    for (int k = 0; k < kC; ++k) a0[k] = a1[k] = sw[9 * kC * kC + k];
    const float4* wt = reinterpret_cast<const float4*>(sw + ij * kC * kC);
#pragma unroll
    for (int c = 0; c < kC; ++c) {
#pragma unroll
      for (int k4 = 0; k4 < kC / 4; ++k4) {
        const float4 ww = wt[c * (kC / 4) + k4];
        a0[4 * k4 + 0] = fmaf(v0[c], ww.x, a0[4 * k4 + 0]); a1[4 * k4 + 0] = fmaf(v1[c], ww.x, a1[4 * k4 + 0]);
        a0[4 * k4 + 1] = fmaf(v0[c], ww.y, a0[4 * k4 + 1]); a1[4 * k4 + 1] = fmaf(v1[c], ww.y, a1[4 * k4 + 1]);
        a0[4 * k4 + 2] = fmaf(v0[c], ww.z, a0[4 * k4 + 2]); a1[4 * k4 + 2] = fmaf(v1[c], ww.z, a1[4 * k4 + 2]);
        a0[4 * k4 + 3] = fmaf(v0[c], ww.w, a0[4 * k4 + 3]); a1[4 * k4 + 3] = fmaf(v1[c], ww.w, a1[4 * k4 + 3]);
      }
    }
    const int64_t off = (int64_t)(ij / 3) * WO + ij % 3;
    store_act(out + (base[0] + off) * 8, a0);
    if (two) store_act(out + (base[1] + off) * 8, a1);
  }
}

// ------------------------------------------------------------------------------------------------ epilogues
enum { EPI_RELU = 0, EPI_RES_RELU = 1, EPI_RES_RELU_RGB = 2 };
// acc = conv + folded bias for one pixel.  EPI_RELU: first conv of a BasicBlock.  EPI_RES_RELU: second conv:
// relu(x + main_branch(x)) (cnns.py:31-32).  EPI_RES_RELU_RGB: the last block, followed by rgb_decoder.7/.8
// (Conv2d 32->3 1x1 + Sigmoid) while the pixel is still in registers -> fp32 rgb.
template <int EPI>
__device__ __forceinline__ void conv_epilogue(float* acc, const uint4* __restrict__ residual, int64_t pix, uint4* __restrict__ out_act,
                                              float* __restrict__ out_rgb, const float* out_w, const float* out_b) {
  if (EPI != EPI_RELU) {
    float x[kC];
    load_act(residual + pix * 8, x);
#pragma unroll
    for (int k = 0; k < kC; ++k) acc[k] += x[k];
  }
#pragma unroll
  for (int k = 0; k < kC; ++k) acc[k] = fmaxf(acc[k], 0.f);
  if (EPI == EPI_RES_RELU_RGB) {
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      float s = out_b[o];
#pragma unroll
      for (int k = 0; k < kC; ++k) s = fmaf(acc[k], out_w[o * kC + k], s);
      out_rgb[pix * 3 + o] = 1.0f / (1.0f + expf(-s));
    }
  } else {
    store_act(out_act + pix * 8, acc);
  }
}

struct ConvArgs {
  const uint4* in;        // ACT [B][H][W]
  const uint4* residual;  // ACT (EPI_RES_*) or nullptr
  uint4* out_act;         // ACT or nullptr
  float* out_rgb;         // [B][H][W][3] (EPI_RES_RELU_RGB)
  const unsigned char* w_img;  // [7 dx][kWRowBytes]
  const float* w_f32;     // [49][ci][co]
  const float* bias;      // [32] folded
  const float* out_w;     // [3][32] (EPI_RES_RELU_RGB)
  const float* out_b;     // [3]
  int batch, H, W;
  int* status;
};

// ------------------------------------------------------------------------------- 7x7 conv on the tensor cores
// Both operands K-major, no swizzle.  A: LBO = plane stride, SBO = 128 B (8 pixels).  B: LBO = 128 B, SBO = 512 B.
constexpr uint32_t kDescSboA = 128u, kDescLboB = 128u, kDescSboB = 512u;

template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t a_desc, uint64_t b_desc) {
  static_assert(N == 32 || N == 64 || N == 96 || N == 128, "one to four 32-channel accumulators");
  if constexpr (N == 32) tc::wgmma_bf16_m64n32(d, a_desc, b_desc);
  else if constexpr (N == 64) tc::wgmma_bf16_m64n64(d, a_desc, b_desc);
  else if constexpr (N == 96) tc::wgmma_bf16_m64n96(d, a_desc, b_desc);
  else tc::wgmma_bf16_m64n128(d, a_desc, b_desc);
}

// Input row I of the window at tap column dx feeds output rows r_min..r_max through taps dy = I - r: one wgmma per
// operand pair with N = 32 * (rows fed), accumulating into those rows' registers (acc + 16 * r_min).
template <int I>
__device__ __forceinline__ void issue_window_row(float* acc, uint32_t a_row, uint32_t w_buf) {
  constexpr int kLast = kK7 - 1;
  constexpr int r_min = I > kLast ? I - kLast : 0, r_max = I < kTH - 1 ? I : kTH - 1, nr = r_max - r_min + 1;
  constexpr uint32_t slot = (uint32_t)(kLast - (I - r_min));  // first (largest-dy) tile of the N-concatenated B
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {  // 16 input channels (two 8-channel chunks) per MMA
    const uint32_t ah = a_row + (uint32_t)(I * kPW * 16 + 2 * ks * kPlaneBytes);
    const uint32_t al = ah + (uint32_t)(4 * kPlaneBytes);
    const uint32_t bh = w_buf + slot * kWTileBytes + (uint32_t)(ks * 256);
    const uint32_t bl = bh + (uint32_t)(kK7 * kWTileBytes);
    const uint64_t dah = tc::smem_desc(ah, kPlaneBytes, kDescSboA), dal = tc::smem_desc(al, kPlaneBytes, kDescSboA);
    const uint64_t dbh = tc::smem_desc(bh, kDescLboB, kDescSboB), dbl = tc::smem_desc(bl, kDescLboB, kDescSboB);
    wgmma_bf16<32 * nr>(acc + 16 * r_min, dah, dbh);
    wgmma_bf16<32 * nr>(acc + 16 * r_min, dal, dbh);
    wgmma_bf16<32 * nr>(acc + 16 * r_min, dah, dbl);
  }
}
template <int... I>
__device__ __forceinline__ void issue_window_rows(float* acc, uint32_t a_row, uint32_t w_buf, std::integer_sequence<int, I...>) {
  (issue_window_row<I>(acc, a_row, w_buf), ...);
}

// Epilogue on the fragments of one output row (pixels lane/4 and lane/4 + 8 of the warp's 16, channels 8j + 2*(lane%4)
// + {0,1}): 32-bit ACT words per thread; the rgb head reduces its dot products over the 4 lanes of a pixel.
template <int EPI>
__device__ __forceinline__ void conv_epilogue_frag(const float* d, const ConvArgs& a, int64_t pix0, bool ok0, int64_t pix1, bool ok1,
                                                   int t, const float* out_w, const float* out_b) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int64_t pix = q ? pix1 : pix0;
    const bool ok = q ? ok1 : ok0;
    float v[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[2 * j] = d[4 * j + 2 * q];
      v[2 * j + 1] = d[4 * j + 2 * q + 1];
    }
    if (EPI != EPI_RELU && ok) {
      const uint32_t* res = reinterpret_cast<const uint32_t*>(a.residual + pix * 8);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float x0, x1;
        unpack2(res[4 * j + t], res[4 * (4 + j) + t], x0, x1);
        v[2 * j] += x0;
        v[2 * j + 1] += x1;
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
    if (EPI == EPI_RES_RELU_RGB) {
      float s[3];
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        s[o] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[o] = fmaf(v[2 * j], out_w[o * kC + 8 * j + 2 * t], s[o]);
          s[o] = fmaf(v[2 * j + 1], out_w[o * kC + 8 * j + 2 * t + 1], s[o]);
        }
        s[o] += __shfl_xor_sync(0xffffffffu, s[o], 1);
        s[o] += __shfl_xor_sync(0xffffffffu, s[o], 2);
      }
      if (ok && t < 3) a.out_rgb[pix * 3 + t] = 1.0f / (1.0f + expf(-(out_b[t] + s[t])));
    } else if (ok) {
      uint32_t* dst = reinterpret_cast<uint32_t*>(a.out_act + pix * 8);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t h, l;
        split_pack2(v[2 * j], v[2 * j + 1], h, l);
        dst[4 * j + t] = h;
        dst[4 * (4 + j) + t] = l;
      }
    }
  }
}

// 16-byte asynchronous global -> shared copy (LDGSTS); src_bytes = 0 writes zeros (the conv's padding) without
// reading.  Many of these are in flight per thread, which is what hides the L2 latency of the window / weight loads.
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc::smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(dst), "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(tc::smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(tc::smem_u32(bar))
               : "memory");
}

struct ConvArgsTma {
  alignas(64) CUtensorMap in_map;  // ACT input as [B][H][W][8][8 x bf16], box (8,1,kPW,kIR,1)
  ConvArgs a;
};

// Two warp groups split the 128-pixel strip, each holding the accumulators of all 4 output rows of its 64 pixels.  TMA:
// the window is 8 tensor copies from a 5-D map over the ACT buffer (its zero fill IS the conv's padding), a weight column
// one 28 KB bulk copy, issued by thread 0 on transaction-count mbarriers.  Otherwise every thread issues 16-byte LDGSTS.
// Column dx + 2 is loaded into the buffer column dx has just finished with; the next tile's loads overlap the epilogue.
template <int EPI, bool TMA>
__device__ __forceinline__ void conv7_body(const ConvArgs& a, const CUtensorMap* in_map) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  ConvSmem& S = *reinterpret_cast<ConvSmem*>(smem_raw);
  const int tid = threadIdx.x, wgp = tid >> 7, wq = (tid >> 5) & 3, ln = tid & 31, g = ln >> 2, t = ln & 3;
  if (tid < kC) S.bias[tid] = a.bias[tid];
  if (EPI == EPI_RES_RELU_RGB) {
    if (tid < 3 * kC) S.out_w[tid] = a.out_w[tid];
    if (tid < 3) S.out_b[tid] = a.out_b[tid];
  }
  if (tid == 0) {
    tc::mbar_init(&S.bar_w[0], 1);
    tc::mbar_init(&S.bar_w[1], 1);
    tc::mbar_init(&S.bar_win, 1);
    S.abort = 0;
  }
  __syncthreads();
  const uint32_t act_u32 = tc::smem_u32(S.act);
  const uint32_t w_u32[2] = {tc::smem_u32(S.w[0]), tc::smem_u32(S.w[1])};
  const int tiles_x = (a.W + kStrip - 1) / kStrip, tiles_y = (a.H + kTH - 1) / kTH;
  const int64_t n_tiles = (int64_t)a.batch * tiles_y * tiles_x;
  uint32_t n_w[2] = {0u, 0u}, n_win = 0u;  // TMA: completions waited for so far (phase parity = count & 1)

  auto load_window = [&](int64_t tile) {  // TMA: thread 0 only; LDGSTS: every thread, no commit (joins column 0's group)
    const int tx = (int)(tile % tiles_x), ty = (int)((tile / tiles_x) % tiles_y);
    const int64_t img = tile / ((int64_t)tiles_x * tiles_y);
    if constexpr (TMA) {
      constexpr uint32_t kWinBytes = 8u * kIR * kPW * 16u;
      mbar_expect_tx(&S.bar_win, kWinBytes);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        tma_load_5d(act_u32 + (uint32_t)(c * kPlaneBytes), in_map, 0, c, tx * kStrip - kPad, ty * kTH - kPad, (int)img, &S.bar_win);
    } else {
      const int x0 = tx * kStrip, y0 = ty * kTH;
      const uint4* in_img = a.in + img * (int64_t)a.H * a.W * 8;
      for (int i = tid; i < kIR * kPW * 8; i += kConvThreads) {
        const int c = i & 7, ip = (i >> 3) % kPW, ir = (i >> 3) / kPW;
        const int y = y0 - kPad + ir, x = x0 - kPad + ip;
        const bool inside = y >= 0 && y < a.H && x >= 0 && x < a.W;
        const uint4* src = inside ? in_img + ((int64_t)y * a.W + x) * 8 + c : in_img;
        cp_async16(act_u32 + (uint32_t)(c * kPlaneBytes + (ir * kPW + ip) * 16), src, inside ? 16u : 0u);
      }
    }
  };
  auto load_column = [&](int dx, int buf) {
    if constexpr (TMA) {
      mbar_expect_tx(&S.bar_w[buf], kWRowBytes);
      bulk_load(w_u32[buf], a.w_img + (size_t)dx * kWRowBytes, kWRowBytes, &S.bar_w[buf]);
    } else {
      const uint4* src = reinterpret_cast<const uint4*>(a.w_img + (size_t)dx * kWRowBytes);
      for (int i = tid; i < kWRowBytes / 16; i += kConvThreads) cp_async16(w_u32[buf] + (uint32_t)(i * 16), src + i, 16u);
      cp_async_commit();
    }
  };
  auto load_tile_start = [&](int64_t tile) {
    if (!TMA || tid == 0) {
      load_window(tile);
      load_column(0, 0);
      load_column(1, 1);
    }
  };
  if ((int64_t)blockIdx.x < n_tiles) load_tile_start(blockIdx.x);

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int tx = (int)(tile % tiles_x), ty = (int)((tile / tiles_x) % tiles_y);
    const int64_t img = tile / ((int64_t)tiles_x * tiles_y);
    const int x0 = tx * kStrip, y0 = ty * kTH;
    // accumulators start from the folded bias: row r in acc[16r, 16r + 16), fragment layout of an m64n32 tile
    float acc[kTH * 16];
#pragma unroll
    for (int r = 0; r < kTH; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[16 * r + 4 * j + 0] = acc[16 * r + 4 * j + 2] = S.bias[8 * j + 2 * t];
        acc[16 * r + 4 * j + 1] = acc[16 * r + 4 * j + 3] = S.bias[8 * j + 2 * t + 1];
      }
    if constexpr (TMA) {
      if (!tc::mbar_wait(&S.bar_win, n_win & 1u)) S.abort = 1;
      ++n_win;
    }
    const uint32_t a_row = act_u32 + (uint32_t)(64 * wgp * 16);  // this warp group's first pixel in window row 0
#pragma unroll 1
    for (int dx = 0; dx < kK7; ++dx) {
      const int buf = dx & 1;
      if constexpr (TMA) {
        if (!tc::mbar_wait(&S.bar_w[buf], n_w[buf] & 1u)) S.abort = 1;
        ++n_w[buf];
      } else {
        if (dx + 1 < kK7) cp_async_wait<1>(); else cp_async_wait<0>();  // column dx (and the window) have landed
        tc::fence_async_smem();  // generic-proxy writes -> visible to the tensor cores (async proxy)
        __syncthreads();
      }
      const uint32_t a_dx = a_row + (uint32_t)(dx * 16);
      tc::wg_fence();
      issue_window_rows(acc, a_dx, w_u32[buf], std::make_integer_sequence<int, kIR>{});
      tc::wg_commit();
      tc::wg_wait<0>();
      __syncthreads();  // both warp groups are done with w[buf] (after column 6: with the window too)
      if (dx + 2 < kK7 && (!TMA || tid == 0)) load_column(dx + 2, buf);
    }
    tc::reg_fence(acc, kTH * 16);
    if (S.abort) break;
    if (tile + gridDim.x < n_tiles) load_tile_start(tile + gridDim.x);
    // ---- epilogue from the registers: this thread's pixels x0 + 64 * wgp + 16 * wq + {g, g + 8}
    const int xa = x0 + 64 * wgp + 16 * wq + g, xb = xa + 8;
#pragma unroll
    for (int r = 0; r < kTH; ++r) {
      const int y = y0 + r;
      const int64_t row = (img * a.H + y) * a.W;
      const bool yok = y < a.H;
      conv_epilogue_frag<EPI>(acc + 16 * r, a, row + xa, yok && xa < a.W, row + xb, yok && xb < a.W, t, S.out_w, S.out_b);
    }
  }
  if (!TMA) cp_async_wait<0>();
  if (S.abort && tid == 0 && a.status) atomicExch(a.status, 2);
}

template <int EPI>
__global__ void __launch_bounds__(kConvThreads, 1) dec_conv7_tma_kernel(const __grid_constant__ ConvArgsTma P) {
  conv7_body<EPI, true>(P.a, &P.in_map);
}
template <int EPI>
__global__ void __launch_bounds__(kConvThreads, 1) dec_conv7_tc_kernel(const ConvArgs a) {
  conv7_body<EPI, false>(a, nullptr);
}


// ------------------------------------------------------------------ 7x7 conv on the CUDA cores (fp32 reference)
// Same inputs, outputs and epilogues as dec_conv7_tc_kernel; one thread per output pixel, the weights of one tap row
// (7 x 32 x 32 fp32 = 28 KB) staged in shared memory.  ~20x slower; kept as the in-library cross-check of the
// tensor-core path (b200nerf_rgb_decode_fwd impl = 1) and for the numerics tests.
template <int EPI>
__global__ void __launch_bounds__(128) dec_conv7_ref_kernel(const ConvArgs a) {
  __shared__ float sw[kK7 * kC * kC];
  __shared__ float s_out[3 * kC + 4];
  const int tid = threadIdx.x;
  if (EPI == EPI_RES_RELU_RGB) {
    if (tid < 3 * kC) s_out[tid] = a.out_w[tid];
    if (tid < 3) s_out[3 * kC + tid] = a.out_b[tid];
  }
  const int tiles_x = (a.W + 127) / 128;
  const int64_t row_id = blockIdx.x / tiles_x;  // (img, y)
  const int x = (blockIdx.x % tiles_x) * 128 + tid;
  const int64_t img = row_id / a.H;
  const int y = (int)(row_id % a.H);
  float acc[kC];
#pragma unroll
  for (int k = 0; k < kC; ++k) acc[k] = a.bias[k];
  for (int dy = 0; dy < kK7; ++dy) {
    __syncthreads();
    for (int i = tid; i < kK7 * kC * kC; i += 128) sw[i] = a.w_f32[(size_t)dy * kK7 * kC * kC + i];
    __syncthreads();
    const int yy = y + dy - kPad;
    if (yy < 0 || yy >= a.H || x >= a.W) continue;
    for (int dx = 0; dx < kK7; ++dx) {
      const int xx = x + dx - kPad;
      if (xx < 0 || xx >= a.W) continue;
      float v[kC];
      load_act(a.in + ((img * a.H + yy) * (int64_t)a.W + xx) * 8, v);
      const float* wt = sw + dx * kC * kC;
#pragma unroll 4
      for (int c = 0; c < kC; ++c) {
#pragma unroll
        for (int k = 0; k < kC; ++k) acc[k] = fmaf(v[c], wt[c * kC + k], acc[k]);
      }
    }
  }
  if (x < a.W) conv_epilogue<EPI>(acc, a.residual, (img * a.H + y) * (int64_t)a.W + x, a.out_act, a.out_rgb, s_out, s_out + 3 * kC);
}

}  // namespace dec
