// tc_mlp.cuh -- tiny-MLP layers on Hopper's warp-group tensor cores (wgmma), sm_90a.
//
// A tile is 128 rows held one per thread by a warp group.  A layer D[128 x N] = A[128 x K] * W^T: every thread writes its
// row to the group's shared-memory stage, the group runs two m64nNk8 TF32 wgmma tiles with A fragments loaded from the
// stage into registers and B = the weights in shared memory (canonical K-major no-swizzle layout), the accumulators go
// back to the stage and every thread reads its own row of D.
// fp32 accuracy is recovered with the 3xTF32 split
//     x*w ~= x_hi*w_hi + x_lo*w_hi + x_hi*w_lo        (x_hi = x with the 13 low mantissa bits cleared)
// i.e. three wgmma per 8-wide k-step accumulating into the same registers; the dropped x_lo*w_lo term is ~2^-22 relative.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers stay untouched by other instructions while a wgmma that writes them is in flight
__device__ __forceinline__ void reg_fence(float* d, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Bounded wait: returns false instead of hanging the GPU if a copy never completes (a wrong tensor map must show up as a
// failed status, not as a wedged GPU).
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  for (int it = 0; it < (1 << 20); ++it) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    if (ok) return true;
  }
  return false;
}
__device__ __forceinline__ uint32_t elect_one() {  // one lane of the converged warp (the same one every time)
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred;
}

// wgmma with fp32 accumulators d (this thread's N/2 fragment registers of an m64 tile); scale-d = 1: D += A * B
// (accumulators are zeroed or preset by the caller).
// "+f" operands d[i .. i + 8)
#define TC_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define TC_D16(i) TC_D8(i), TC_D8(i + 8)
#define TC_D32(i) TC_D16(i), TC_D16(i + 16)
__device__ __forceinline__ void wgmma_tf32_m64n16(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\twgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
               : TC_D8(0)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_m64n32(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
               : TC_D16(0)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_m64n48(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\twgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1;\n\t}"
               : TC_D16(0), TC_D8(16)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_m64n64(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
               : TC_D32(0)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_bf16_m64n32(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
               : TC_D16(0)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_bf16_m64n64(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : TC_D32(0)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_bf16_m64n96(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\twgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
               : TC_D32(0), TC_D16(32)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_bf16_m64n128(float* d, uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : TC_D32(0), TC_D32(32)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
// m64n32k16 with fp16 operands and fp32 accumulators; A = this thread's 4 f16x2 fragment registers (row g / g+8,
// k 2t, 2t+1 / 2t+8, 2t+9; the lower k in the low half), B from a K-major descriptor.
__device__ __forceinline__ void wgmma_f16_m64n32(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
               : TC_D16(0)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
// the same with scale-d = 0: D = A * B, the accumulators' previous values are not read
__device__ __forceinline__ void wgmma_f16_m64n32_zero(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
               : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]),
                 "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(0));
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, const uint32_t* a, uint64_t b_desc) {
  static_assert(N == 16 || N == 32 || N == 48 || N == 64, "tf32 tile widths");
  if constexpr (N == 16) wgmma_tf32_m64n16(d, a, b_desc);
  else if constexpr (N == 32) wgmma_tf32_m64n32(d, a, b_desc);
  else if constexpr (N == 48) wgmma_tf32_m64n48(d, a, b_desc);
  else wgmma_tf32_m64n64(d, a, b_desc);
}

// ------------------------------------------------------------------------------------------- operand layouts
// B operand (weights, nn.Linear [N_real, K_real] row major in global memory) -> shared memory, canonical K-major
// no-swizzle layout (cute: ((8,n),2):((1,SBO),LBO) in 16-byte units): 8-row x 16-byte core matrices, core (nb, kc) at
// nb*SBO + kc*LBO with LBO = 128 B, SBO = (K_pad/4)*128 B; element (n,k) at  +(n%8)*16 + (k%4)*4.
__host__ __device__ constexpr uint32_t b_tile_floats(int n_pad, int k_pad) { return (uint32_t)(n_pad * k_pad); }
__device__ __forceinline__ uint32_t b_elem_offset(int n, int k, int k_pad) {
  return (uint32_t)((n >> 3) * (k_pad >> 2) * 32 + (k >> 2) * 32 + (n & 7) * 4 + (k & 3));  // in floats
}
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

// cooperative: all `nthreads` threads of the CTA
__device__ __forceinline__ void stage_b_tile(float* hi, float* lo, const float* __restrict__ w, int n_real, int k_real, int n_pad,
                                             int k_pad, int tid, int nthreads) {
  for (int i = tid; i < n_pad * k_pad; i += nthreads) {
    int n = i / k_pad, k = i % k_pad;
    float v = (n < n_real && k < k_real) ? w[n * k_real + k] : 0.0f;
    float h = tf32_hi(v);
    uint32_t off = b_elem_offset(n, k, k_pad);
    hi[off] = h;
    lo[off] = v - h;  // exact in fp32; the tensor core truncates it to TF32 (error ~2^-22 |v|)
  }
}

// fp16 hi/lo split of a pair: hi = (x0, x1) rounded to fp16, lo = the remainders x - hi (exact in fp32) rounded to fp16.
// x0 goes to the low half of each register.  FP16 has TF32's 11 significant bits, so hi + lo carries 22 of them.
__device__ __forceinline__ void f16x2_split(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// fp16 B tile, canonical K-major no-swizzle layout for k16 steps: 8-row x 16-byte core matrices (8 halves along K), core
// (nb, kc) at nb*SBO + kc*LBO with LBO = 128 B, SBO = (K_pad/8)*128 B; element (n,k) at +(n%8)*16 B + (k%8)*2 B.
__device__ __forceinline__ uint32_t b_elem_offset_f16(int n, int k, int k_pad) {
  return (uint32_t)((n >> 3) * (k_pad >> 3) * 64 + (k >> 3) * 64 + (n & 7) * 8 + (k & 7));  // in halves
}
// cooperative (all `nthreads` threads of the CTA): W[n_real x k_real] (row major, fp32) times `scale` (a power of two)
// -> fp16 hi / lo tiles [32 x k_real]
__device__ __forceinline__ void stage_b_tile_f16(__half* hi, __half* lo, const float* __restrict__ w, int k_real, float scale,
                                                 int tid, int nthreads) {
  for (int i = tid; i < 32 * k_real; i += nthreads) {
    const int n = i / k_real, k = i % k_real;
    const float v = w[i] * scale;
    const __half h = __float2half_rn(v);
    const uint32_t off = b_elem_offset_f16(n, k, k_real);
    hi[off] = h;
    lo[off] = __float2half_rn(v - __half2float(h));
  }
}
// 64-bit shared-memory matrix descriptor (sm_90 GMMA): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base offset 0, layout_type = no swizzle (0) [62,64)
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3ffffu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
// The same descriptor as two 32-bit words: lo = start and LBO fields, hi = SBO field.  A tile `off` bytes further on has
// lo + off / 16 (the start field cannot carry into the LBO field: shared memory ends below 2^18 bytes), so every
// descriptor of a CTA's resident B tiles is one lo word plus compile-time constants.  When that word comes from a shared
// memory symbol, ptxas forms the descriptors on the uniform datapath: no per-thread descriptor arithmetic and no R2UR
// move in front of each wgmma.
__device__ __forceinline__ uint32_t smem_desc_lo(uint32_t saddr, uint32_t lbo_bytes) {
  return ((saddr & 0x3ffffu) >> 4) | ((lbo_bytes >> 4) << 16);
}
__device__ __forceinline__ uint64_t smem_desc_of(uint32_t lo, uint32_t sbo_bytes) {
  return (uint64_t)lo | ((uint64_t)(sbo_bytes >> 4) << 32);
}

// ------------------------------------------------------------------------------------------------ tile ops
// Row pitch (floats) of a 128-row stage holding up to W columns.
__host__ __device__ constexpr int stage_pitch(int w) { return (w + 7) / 8 * 8 + 4; }

// This thread's `n` (multiple of 4) values -> its row of the stage.  row = thread index within the warp group.
template <int K_MAX>
__device__ __forceinline__ void store_row(float* stage, int pitch, const float* x, int n) {
  float4* dst = reinterpret_cast<float4*>(stage + (threadIdx.x & 127) * pitch);
#pragma unroll
  for (int c = 0; c < K_MAX; c += 4)
    if (c < n) dst[c / 4] = make_float4(x[c], x[c + 1], x[c + 2], x[c + 3]);
}
template <int N_MAX>
__device__ __forceinline__ void load_row(const float* stage, int pitch, float* y, int n) {
  const float4* src = reinterpret_cast<const float4*>(stage + (threadIdx.x & 127) * pitch);
#pragma unroll
  for (int c = 0; c < N_MAX; c += 4)
    if (c < n) {
      const float4 v = src[c / 4];
      y[c] = v.x, y[c + 1] = v.y, y[c + 2] = v.z, y[c + 3] = v.w;
    }
}

// acc[N] += stage[128 x k_pad] * W^T, 3xTF32, by a converged warp group once the stage is full.  acc: [half][N/2]
// fragments (rows 64*half + 16*warp + lane/4 (+8), columns 8j + 2*(lane%4) (+1)).
template <int N>
__device__ __forceinline__ void tile_mma(const float* stage, int pitch, int k_pad, const float* b_hi, const float* b_lo, float* acc) {
  const int wq = (threadIdx.x >> 5) & 3, ln = threadIdx.x & 31, g = ln >> 2, t = ln & 3;
  const uint32_t sbo = (uint32_t)(k_pad >> 2) * 128u;
  const uint64_t dh0 = smem_desc(smem_u32(b_hi), 128u, sbo), dl0 = smem_desc(smem_u32(b_lo), 128u, sbo);
  for (int ks = 0; ks < k_pad / 8; ++ks) {
    uint32_t ah[2][4], al[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float* r0 = stage + (64 * h + 16 * wq + g) * pitch + 8 * ks + t;
      const float* r1 = r0 + 8 * pitch;
      const float v[4] = {r0[0], r1[0], r0[4], r1[4]};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float vh = tf32_hi(v[i]);
        ah[h][i] = __float_as_uint(vh);
        al[h][i] = __float_as_uint(v[i] - vh);
      }
    }
    const uint64_t adv = (uint64_t)((ks * 2 * 128) >> 4);  // two 16-byte K-chunks (= 2 core matrices) per k-step
    wg_fence();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      wgmma_tf32<N>(acc + h * (N / 2), ah[h], dh0 + adv);
      wgmma_tf32<N>(acc + h * (N / 2), al[h], dh0 + adv);
      wgmma_tf32<N>(acc + h * (N / 2), ah[h], dl0 + adv);
    }
    wg_commit();
    wg_wait<0>();  // the fragment registers of this k-step are reused by the next
  }
  reg_fence(acc, N);
}
// accumulator fragments -> stage rows (each warp writes the rows of its own fragments; __syncwarp orders them after the
// warp's fragment reads of the same rows)
template <int N>
__device__ __forceinline__ void tile_store_d(float* stage, int pitch, const float* acc) {
  const int wq = (threadIdx.x >> 5) & 3, ln = threadIdx.x & 31, g = ln >> 2, t = ln & 3;
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* r0 = stage + (64 * h + 16 * wq + g) * pitch + 2 * t;
    float* r1 = r0 + 8 * pitch;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const float* d = acc + h * (N / 2) + 4 * j;
      *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[0], d[1]);
      *reinterpret_cast<float2*>(r1 + 8 * j) = make_float2(d[2], d[3]);
    }
  }
}

// One layer of the tile: x (this thread's k_pad inputs) -> out (its N outputs, no bias).  All 128 threads of the warp
// group; `sync` is the group's barrier.
template <int K_MAX, int N, class Sync>
__device__ __forceinline__ void tile_layer(float* stage, int pitch, const float* x, int k_pad, const float* b_hi, const float* b_lo,
                                           float* out, Sync&& sync) {
  store_row<K_MAX>(stage, pitch, x, k_pad);
  sync();  // every row is in; also: every thread has read its previous D row
  float acc[N];
#pragma unroll
  for (int i = 0; i < N; ++i) acc[i] = 0.0f;
  tile_mma<N>(stage, pitch, k_pad, b_hi, b_lo, acc);
  tile_store_d<N>(stage, pitch, acc);
  sync();
  load_row<N>(stage, pitch, out, N);
}

}  // namespace tc
