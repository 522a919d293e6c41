// unet_tc.cu -- wgmma / TMA / mbarrier implicit-GEMM 3x3 convolution for the U-Net backbone (sm_90a).
//
// Reference op: Keras Conv2D(3x3, padding='same', bias, ReLU) as composed by csbdeep's unet_block
// (stardist/models/model2d.py:310-349, SURVEY A.1).  Parity target for the float maps is 1e-5
// relative, i.e. fp32-faithful -- a single TF32/BF16 pass (10/8 mantissa bits) is not enough.
//
// Number format: every activation tensor lives in HBM as TWO fp16 planes (hi, lo) with
//   hi = fp16(v), lo = fp16(v - hi)      (22 significant bits, same 4 bytes/element as fp32)
// written by the producing kernel's epilogue, and weights are split the same way once per model.
// A convolution is then 3 fp16 tensor-core passes  hi*Whi + lo*Whi + hi*Wlo  accumulated in fp32
// registers (each fp16 x fp16 product is exact in fp32; the dropped lo*Wlo term is ~2^-22).
// Compared with 3xTF32 this doubles the MMA rate (fp16 wgmma) and needs no in-kernel split pass.
//
// One kernel, k_conv_wg<N, KC, FUSE>, does every tensor-core convolution of the network:
//   tile = 8 x 16 output pixels (M = 128) x N output channels, persistent CTAs sweeping the tiles;
//   K loop over (tap, KC-channel block): the A operand of a tap is one 4-D TMA box {KC channels, 16 x, 8 y, 1 image}
//   at tap-shifted coordinates (out-of-bounds elements are zero-filled by TMA == the 'same' zero padding), the B operand
//   = weights [tap][Cout][Cin] (K-major), 3-D TMA box {KC, N, 1}.  K-major SWIZZLE_128B (KC = 64) / SWIZZLE_64B (KC = 32).
//   Warp 8 = TMA producer (one lane), warpgroups 0 and 1 = MMA + epilogue for pixel rows [0,64) and [64,128) of the tile.
//   The producer runs ahead across tile boundaries through a ring of shared-memory stages, so the next tile's loads
//   overlap the epilogue of the current one.
//   3x3x3 (n_taps = 27): the tensor map's image axis is the z plane of ONE volume, tap dz reads plane z + dz - 1.
//   1x1 heads (n_taps = 1): channel 0 -> sigmoid -> prob, channels 1..R -> dist, fp32 outputs.
//   FUSE: the features convolution (Cout = 128) with the 1x1 heads computed on the fp32 accumulators in the epilogue.
//   The decoder's Concatenate([UpSampling(x), skip]) is two activation sources on the K axis; the up-sampled source is
//   materialised by its producer's epilogue (each pixel written 2x2, or 2x2x2 in 3-D).
// All mbarrier waits are bounded: on timeout an error flag is raised and the kernel drains.
#include <cuda.h>
#include <cuda_fp16.h>
#include <vector>
#include <algorithm>
#include <map>
#include <tuple>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

struct ConvParams {
  int H, W;              // output (== input) spatial size
  int c_src0;            // channels taken from source 0 (0 for a plain convolution)
  int c_total;           // Cin
  int c_out;             // output channels of the whole layer (row stride of the output planes; N per tile)
  int relu;
  int up2x;              // 1: write every output pixel to the 2x2 block of a (2H, 2W) tensor; 2: 2x2x2 block (3-D)
  float acc_scale;       // 2^-k: the weights were multiplied by 2^k before the hi/lo split (keeps w_lo out of the fp16 subnormals)
  const float* bias;
  __half* out_hi; __half* out_lo;
  unsigned int* error_flag;
  int n_taps;            // 9 (3x3), 27 (3x3x3) or 1 (1x1 heads)
  int heads_R;           // > 0: heads epilogue -> prob = sigmoid(ch 0), dist = ch 1..R, fp32 outputs
  float* prob; float* dist;
  // fused features -> heads (FUSE): fp32 head weights [128][36] (columns 0..R-1 = dist, 32 = prob, zero padded) and biases [36]
  const float* fuse_w; const float* fuse_b;
  int split_acc;         // 1: the two small products (lo*Whi, hi*Wlo) accumulate in their own registers, so the main
                         // accumulator takes one truncating add per k-step instead of three (DESIGN.md 5, network floats)
};

// ---------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: returns false after ~2 s without completion (a lost arrival then surfaces as an error, not a hang)
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return true;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    for (int it = 0; it < 256; ++it) { if (mbar_try_wait(bar, parity)) return true; }
    unsigned long long t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > 2000000000ull) return false;
  }
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}
__device__ __forceinline__ float lds32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
// K-major swizzled shared-memory matrix descriptor of wgmma: start addr>>4 [0,14), LBO>>4 [16,30) (unused for swizzled
// K-major), SBO>>4 [32,46) = stride of 8-row groups, swizzle mode [62,64) (1 = 128B, 2 = 64B).  Operand tiles start on
// 1024-byte boundaries, so the base-offset field stays 0; a k-step of 16 fp16 (32 B) inside the swizzled row is +2.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t sbo_bytes, uint32_t swizzle) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)swizzle << 62;
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int K> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(K) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R> __device__ __forceinline__ void wg_fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma.m64nNk16.f32.f16.f16, A and B from shared memory (K-major), D += A x B^T (acc = 0: D = A x B^T).
// Accumulator fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[j] holds row w*16 + l/4 + 8*((j/2)&1),
// column (j/4)*8 + (l%4)*2 + (j&1).
template <int N> struct Wg;
template <> struct Wg<32> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<48> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<64> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<80> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                 "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<112> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %58, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                 "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<128> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                 "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                 "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wg<144> {
  __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %74, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                 "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                 "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                 "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
               : "l"(a), "l"(b), "r"(acc));
  }
};

// ---------------------------------------------------------------------------------- the kernel
template <int N, int KC, bool FUSE>
struct WgCfg {
  static constexpr int ROWB = KC * 2;                       // bytes per operand row
  static constexpr int A_BYTES = 128 * ROWB;                // one A plane tile (a multiple of 1024)
  static constexpr int B_BYTES = N * ROWB;
  static constexpr int B_SLOT = (B_BYTES + 1023) / 1024 * 1024;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_SLOT;
  static constexpr int TX_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int FUSE_BYTES = FUSE ? (36 + N + N * 36) * 4 : 0;   // head biases, feature biases, head weights
  static constexpr int STAGES_RAW = (216 * 1024 - FUSE_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + FUSE_BYTES;
  static constexpr uint32_t SWZ = (ROWB == 128) ? 1u : 2u;
  static constexpr uint32_t SBO = 8 * ROWB;
  static constexpr int NREG = N / 2;                        // accumulator registers per thread (m64nN over 128 threads)
  static_assert(N % 16 == 0 && N <= 256, "wgmma N");
  static_assert(STAGES >= 2, "pipeline needs two stages");
  static_assert(SMEM <= 227 * 1024, "shared memory");
  static_assert(!FUSE || N == 128, "fused heads follow the 128-channel features convolution");
};

constexpr int kConsumerThreads = 256;                       // two warpgroups
constexpr int kThreads = kConsumerThreads + 128;            // + the producer warpgroup (one TMA lane)
// register split (setmaxnreg): the producer warpgroup needs few, the accumulators (2 x N/2 floats) need many;
// 128 * 40 + 256 * 232 <= 64K registers
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

template <int N, int KC, bool FUSE>
__global__ void __launch_bounds__(kThreads, 1)
k_conv_wg(const __grid_constant__ CUtensorMap tm_a0_hi, const __grid_constant__ CUtensorMap tm_a0_lo,
          const __grid_constant__ CUtensorMap tm_a1_hi, const __grid_constant__ CUtensorMap tm_a1_lo,
          const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, ConvParams P,
          int tiles_x, int tiles_y, int n_nb, int n_tiles) {
  using C = WgCfg<N, KC, FUSE>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;
  float* sHW = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES + 256);   // FUSE only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_cb = P.c_total / KC;
  const int n_kb = P.n_taps * n_cb;

  if (FUSE) {
    for (int e = threadIdx.x; e < 36; e += blockDim.x) sHW[e] = P.fuse_b[e];
    for (int e = threadIdx.x; e < N; e += blockDim.x) sHW[36 + e] = P.bias[e];
    for (int e = threadIdx.x; e < N * 36; e += blockDim.x) sHW[36 + N + e] = P.fuse_w[e];
  }
  if (threadIdx.x == 0) {
    // empty: one arrival per consumer warp once its MMAs on the stage have retired
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kConsumerThreads / 32 && lane == 0) {
      uint32_t it = 0;
      bool ok = true;
      for (int tile = blockIdx.x; tile < n_tiles && ok; tile += gridDim.x) {
        const int nb = tile % n_nb, r = tile / n_nb;
        const int bx = r % tiles_x, by = (r / tiles_x) % tiles_y, img = r / (tiles_x * tiles_y);
        const int x0 = bx * 16, y0 = by * 8;
        for (int kb = 0; kb < n_kb; ++kb, ++it) {
          const uint32_t s = it % C::STAGES;
          if (it >= (uint32_t)C::STAGES && !mbar_wait(&empty_bar[s], ((it / C::STAGES) - 1) & 1)) {
            atomicExch(P.error_flag, 1u); ok = false; break;
          }
          const int tap = kb / n_cb, cb = kb - tap * n_cb;
          const int t9 = tap % 9;
          const int dy = (P.n_taps == 1) ? 0 : t9 / 3 - 1, dx = (P.n_taps == 1) ? 0 : t9 % 3 - 1;
          const int plane = (P.n_taps == 27) ? img + tap / 9 - 1 : img;
          const int ch = cb * KC;
          unsigned char* st = smem + s * C::STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], C::TX_BYTES);
          if (ch < P.c_src0) {
            tma_load_4d(st, &tm_a0_hi, &full_bar[s], ch, x0 + dx, y0 + dy, plane);
            tma_load_4d(st + C::A_BYTES, &tm_a0_lo, &full_bar[s], ch, x0 + dx, y0 + dy, plane);
          } else {
            tma_load_4d(st, &tm_a1_hi, &full_bar[s], ch - P.c_src0, x0 + dx, y0 + dy, plane);
            tma_load_4d(st + C::A_BYTES, &tm_a1_lo, &full_bar[s], ch - P.c_src0, x0 + dx, y0 + dy, plane);
          }
          tma_load_3d(st + 2 * C::A_BYTES, &tm_w_hi, &full_bar[s], ch, nb * N, tap);
          tma_load_3d(st + 2 * C::A_BYTES + C::B_SLOT, &tm_w_lo, &full_bar[s], ch, nb * N, tap);
        }
      }
    }
    return;
  }

  // ===================== MMA + epilogue (warpgroup wg: pixel rows [64 wg, 64 wg + 64) of the tile) =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  const int wg = threadIdx.x >> 7, w = warp & 3;
  float acc[C::NREG], cor[C::NREG];
#pragma unroll
  for (int j = 0; j < C::NREG; ++j) cor[j] = 0.f;
  uint32_t it = 0;
  bool ok = true;
  for (int tile = blockIdx.x; tile < n_tiles && ok; tile += gridDim.x) {
    const int nb = tile % n_nb, r = tile / n_nb;
    const int bx = r % tiles_x, by = (r / tiles_x) % tiles_y, img = r / (tiles_x * tiles_y);
    wg_fence_regs<C::NREG>(acc); wg_fence_regs<C::NREG>(cor);
    for (int kb = 0; kb < n_kb; ++kb, ++it) {
      const uint32_t s = it % C::STAGES;
      ok = __all_sync(0xffffffffu, mbar_wait(&full_bar[s], (it / C::STAGES) & 1));
      if (!ok) { atomicExch(P.error_flag, 2u); break; }
      const uint32_t a_hi = smem_u32(smem + s * C::STAGE_BYTES) + (uint32_t)(wg * 64 * C::ROWB), a_lo = a_hi + C::A_BYTES;
      const uint32_t b_hi = smem_u32(smem + s * C::STAGE_BYTES) + 2 * C::A_BYTES, b_lo = b_hi + C::B_SLOT;
      const uint64_t dah = make_desc(a_hi, C::SBO, C::SWZ), dal = make_desc(a_lo, C::SBO, C::SWZ);
      const uint64_t dbh = make_desc(b_hi, C::SBO, C::SWZ), dbl = make_desc(b_lo, C::SBO, C::SWZ);
      wg_fence();
      if (P.split_acc) {
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks) {
          const uint32_t first = (kb | ks) ? 1u : 0u;
          Wg<N>::mma(acc, dah + 2u * ks, dbh + 2u * ks, first);
          Wg<N>::mma(cor, dal + 2u * ks, dbh + 2u * ks, first);
          Wg<N>::mma(cor, dah + 2u * ks, dbl + 2u * ks, 1u);
        }
      } else {
#pragma unroll
        for (int ks = 0; ks < KC / 16; ++ks) {
          Wg<N>::mma(acc, dah + 2u * ks, dbh + 2u * ks, (kb | ks) ? 1u : 0u);
          Wg<N>::mma(acc, dal + 2u * ks, dbh + 2u * ks, 1u);
          Wg<N>::mma(acc, dah + 2u * ks, dbl + 2u * ks, 1u);
        }
      }
      wg_commit();
      wg_wait<1>();                             // the previous stage's MMAs have retired: hand its slot back
      if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % C::STAGES]);
    }
    wg_wait<0>();
    wg_fence_regs<C::NREG>(acc); wg_fence_regs<C::NREG>(cor);
    if (!ok) break;
    if (n_kb > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % C::STAGES]);

    // ---- epilogue: this thread holds pixels (y, x0 + lane/4) and (y, x0 + lane/4 + 8), channels c8*8 + (lane%4)*2 + {0,1}
    const int y = by * 8 + wg * 4 + w;
    const int xa = bx * 16 + (lane >> 2);
    const int cq = (lane & 3) * 2;
    if (FUSE) {
      // features (bias + ReLU, fp32 straight from the accumulators) -> 1x1 heads on the CUDA cores -> prob / dist.
      // The 128-channel feature map never goes to HBM.  Each thread sums its 32 channels of both pixels into the head
      // outputs, the four threads of a quad (which together hold all 128 channels) reduce with shuffles.  Two passes
      // over the outputs (dist 0..15, then dist 16..31 + prob) bound the live registers.
      const uint32_t sFB_s = smem_u32(sHW + 36), sW_s = smem_u32(sHW + 36 + N);
      // one accumulator from here on (the correction registers hold the constant 0 until the next tile's first MMA
      // overwrites them), which keeps the head sums below the register budget
#pragma unroll
      for (int j = 0; j < C::NREG; ++j) { acc[j] += cor[j]; cor[j] = 0.f; }
#pragma unroll
      for (int grp = 0; grp < 2; ++grp) {
        float o0[17], o1[17];
#pragma unroll
        for (int o = 0; o < 17; ++o) { o0[o] = 0.f; o1[o] = 0.f; }
#pragma unroll
        for (int c8 = 0; c8 < N / 8; ++c8) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = c8 * 8 + cq + e;
            const float fb = lds32(sFB_s + 4u * (uint32_t)c);
            float f0 = acc[c8 * 4 + e] * P.acc_scale + fb;
            float f1 = acc[c8 * 4 + 2 + e] * P.acc_scale + fb;
            if (P.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
            const uint32_t wrow = sW_s + 4u * (uint32_t)(c * 36 + grp * 16);
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              const float4 wv = lds128(wrow + 16u * qq);
              o0[4 * qq] = fmaf(f0, wv.x, o0[4 * qq]); o0[4 * qq + 1] = fmaf(f0, wv.y, o0[4 * qq + 1]);
              o0[4 * qq + 2] = fmaf(f0, wv.z, o0[4 * qq + 2]); o0[4 * qq + 3] = fmaf(f0, wv.w, o0[4 * qq + 3]);
              o1[4 * qq] = fmaf(f1, wv.x, o1[4 * qq]); o1[4 * qq + 1] = fmaf(f1, wv.y, o1[4 * qq + 1]);
              o1[4 * qq + 2] = fmaf(f1, wv.z, o1[4 * qq + 2]); o1[4 * qq + 3] = fmaf(f1, wv.w, o1[4 * qq + 3]);
            }
            if (grp) { const float wv = lds32(sW_s + 4u * (uint32_t)(c * 36 + 32)); o0[16] = fmaf(f0, wv, o0[16]); o1[16] = fmaf(f1, wv, o1[16]); }
          }
        }
#pragma unroll
        for (int o = 0; o < 17; ++o) {
          o0[o] += __shfl_xor_sync(0xffffffffu, o0[o], 1); o0[o] += __shfl_xor_sync(0xffffffffu, o0[o], 2);
          o1[o] += __shfl_xor_sync(0xffffffffu, o1[o], 1); o1[o] += __shfl_xor_sync(0xffffffffu, o1[o], 2);
        }
        // quad thread q writes pixel q >> 1, outputs (q & 1) * 8 .. + 7 of this pass (and the prob)
        const int q = lane & 3;
        const int x = xa + ((q >> 1) ? 8 : 0);
        if (y < P.H && x < P.W) {
          const size_t pix = ((size_t)img * P.H + y) * P.W + x;
          const int ob = grp * 16 + (q & 1) * 8;
          float v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float a = (q & 1) ? o0[8 + k] : o0[k], b = (q & 1) ? o1[8 + k] : o1[k];
            v[k] = ((q >> 1) ? b : a) + sHW[ob + k];
          }
          if (P.heads_R == 32) {
            float4* d4 = reinterpret_cast<float4*>(P.dist + pix * 32 + ob);
            d4[0] = make_float4(v[0], v[1], v[2], v[3]); d4[1] = make_float4(v[4], v[5], v[6], v[7]);
          } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) if (ob + k < P.heads_R) P.dist[pix * P.heads_R + ob + k] = v[k];
          }
          if (grp && (q & 1) == 0) P.prob[pix] = 1.f / (1.f + expf(-(((q >> 1) ? o1[16] : o0[16]) + sHW[32])));
        }
      }
      continue;
    }
    const float* bias = P.bias + nb * N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int x = xa + 8 * h;
      if (y >= P.H || x >= P.W) continue;
      const size_t pix = ((size_t)img * P.H + y) * P.W + x;
      if (P.heads_R > 0) {
        // heads: channel 0 -> sigmoid -> prob, channels 1..R -> dist (fp32)
#pragma unroll
        for (int c8 = 0; c8 < N / 8; ++c8)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ch = c8 * 8 + cq + e, j = c8 * 4 + 2 * h + e;
            if (ch > P.heads_R) continue;
            const float v = (acc[j] + cor[j]) * P.acc_scale + __ldg(bias + ch);
            if (ch == 0) P.prob[pix] = 1.f / (1.f + expf(-v));
            else P.dist[pix * P.heads_R + (ch - 1)] = v;
          }
        continue;
      }
#pragma unroll
      for (int c8 = 0; c8 < N / 8; ++c8) {
        const int ch = c8 * 8 + cq, j = c8 * 4 + 2 * h;
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + ch));
        float v0 = (acc[j] + cor[j]) * P.acc_scale + bb.x, v1 = (acc[j + 1] + cor[j + 1]) * P.acc_scale + bb.y;
        if (P.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        if (!(fabsf(v0) <= 65504.f) || !(fabsf(v1) <= 65504.f)) atomicOr(P.error_flag, 0x80000000u);   // fp16 range of the hi plane exceeded (or NaN)
        const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
        const __half2 hi = __halves2half2(h0, h1);
        const __half2 lo = __halves2half2(__float2half_rn(v0 - __half2float(h0)), __float2half_rn(v1 - __half2float(h1)));
        const int oc = nb * N + ch;
        if (!P.up2x) {
          const size_t off = pix * P.c_out + oc;
          *reinterpret_cast<__half2*>(P.out_hi + off) = hi;
          *reinterpret_cast<__half2*>(P.out_lo + off) = lo;
        } else {
          // nearest up-sampling written by the producer: 2x2 pixels, and both planes 2z, 2z+1 for a volume (up2x == 2)
          const int H2 = 2 * P.H, W2 = 2 * P.W;
          const int nrep = (P.up2x == 2) ? 8 : 4;
          for (int rep = 0; rep < nrep; ++rep) {
            const size_t plane = (P.up2x == 2) ? (size_t)(2 * img + (rep >> 2)) : (size_t)img;
            const size_t off = ((plane * H2 + (2 * y + ((rep >> 1) & 1))) * W2 + (2 * x + (rep & 1))) * P.c_out + oc;
            *reinterpret_cast<__half2*>(P.out_hi + off) = hi;
            *reinterpret_cast<__half2*>(P.out_lo + off) = lo;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------- small SIMT companions
// stem: Cin (1..4) -> COUT, fp32 input, split fp16 output
template <int COUT>
__global__ void __launch_bounds__(128)
k_stem_split(const float* __restrict__ in, int N_, int H, int W, int Cin, const float* __restrict__ wgt,
             const float* __restrict__ bias, int relu, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
             unsigned int* __restrict__ err) {
  extern __shared__ float sw[];
  for (int e = threadIdx.x; e < 9 * Cin * COUT; e += blockDim.x) sw[e] = wgt[e];
  for (int e = threadIdx.x; e < COUT; e += blockDim.x) sw[9 * Cin * COUT + e] = bias[e];
  __syncthreads();
  const long long npix = (long long)N_ * H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int x = (int)(p % W), y = (int)((p / W) % H);
  const long long img = p / ((long long)W * H);
  float acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = sw[9 * Cin * COUT + o];
  for (int dy = 0; dy < 3; ++dy) {
    const int yy = y + dy - 1;
    if (yy < 0 || yy >= H) continue;
    for (int dx = 0; dx < 3; ++dx) {
      const int xx = x + dx - 1;
      if (xx < 0 || xx >= W) continue;
      const float* ip = in + ((img * H + yy) * W + xx) * Cin;
      for (int c = 0; c < Cin; ++c) {
        const float v = ip[c];
        const float* wr = sw + ((dy * 3 + dx) * Cin + c) * COUT;
#pragma unroll
        for (int o = 0; o < COUT; ++o) acc[o] = fmaf(v, wr[o], acc[o]);
      }
    }
  }
  __align__(16) __half hi[COUT];
  __align__(16) __half lo[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) {
    float v = acc[o];
    if (relu) v = fmaxf(v, 0.f);
    if (!(fabsf(v) <= 65504.f)) atomicOr(err, 0x80000000u);
    const __half h = __float2half_rn(v);
    hi[o] = h; lo[o] = __float2half_rn(v - __half2float(h));
  }
#pragma unroll
  for (int j = 0; j < COUT / 8; ++j) {
    reinterpret_cast<uint4*>(out_hi + p * COUT)[j] = reinterpret_cast<const uint4*>(hi)[j];
    reinterpret_cast<uint4*>(out_lo + p * COUT)[j] = reinterpret_cast<const uint4*>(lo)[j];
  }
}

__global__ void k_maxpool_split(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int N_, int H, int W, int C,
                                __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const int Ho = H / 2, Wo = W / 2, C2 = C / 2;
  const long long total = (long long)N_ * Ho * Wo * C2;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c2 = (int)(e % C2); long long r = e / C2;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); const long long img = r / Ho;
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t off = (((size_t)img * H + 2 * yo + (k >> 1)) * W + 2 * xo + (k & 1)) * C + 2 * c2;
      const float2 h = __half22float2(*reinterpret_cast<const __half2*>(in_hi + off));
      const float2 l = __half22float2(*reinterpret_cast<const __half2*>(in_lo + off));
      m0 = fmaxf(m0, h.x + l.x); m1 = fmaxf(m1, h.y + l.y);
    }
    const __half h0 = __float2half_rn(m0), h1 = __float2half_rn(m1);
    const size_t o = (size_t)e * 2;
    *reinterpret_cast<__half2*>(out_hi + o) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(out_lo + o) = __halves2half2(__float2half_rn(m0 - __half2float(h0)), __float2half_rn(m1 - __half2float(h1)));
  }
}

// heads on split features: prob = sigmoid(x.Wp+bp), dist = x.Wd+bd.
// One thread per pixel keeps 32 output accumulators in registers per pass (feature value read once from
// shared memory, weights as broadcast LDS.128), results staged through shared memory for coalesced stores.
template <int CF>
__global__ void __launch_bounds__(128)
k_heads_split(const __half* __restrict__ f_hi, const __half* __restrict__ f_lo, long long npix, const float* __restrict__ wp,
              const float* __restrict__ bp, const float* __restrict__ wd, const float* __restrict__ bd, int R,
              float* __restrict__ prob, float* __restrict__ dist) {
  extern __shared__ __align__(16) float sm[];
  const int NO = R + 1, NOP = (NO + 31) / 32 * 32;
  float* sW = sm;                        // [CF][NOP]  (o = 0 prob, 1.. dist, zero padded)
  float* sB = sW + CF * NOP;             // [NOP]
  float* sF = sB + NOP;                  // [128][CF+1]
  float* sO = sF + 128 * (CF + 1);       // [128][33]
  for (int e = threadIdx.x; e < CF * NOP; e += blockDim.x) {
    const int f = e / NOP, o = e % NOP;
    sW[e] = (o == 0) ? wp[f] : (o < NO ? wd[(size_t)f * R + (o - 1)] : 0.f);
  }
  for (int o = threadIdx.x; o < NOP; o += blockDim.x) sB[o] = (o == 0) ? bp[0] : (o < NO ? bd[o - 1] : 0.f);
  const long long p0 = (long long)blockIdx.x * 128;
  for (int e = threadIdx.x; e < 128 * (CF / 2); e += blockDim.x) {
    const int px = e / (CF / 2), f2 = e % (CF / 2);
    float2 v = make_float2(0.f, 0.f);
    if (p0 + px < npix) {
      const float2 h = __half22float2(*reinterpret_cast<const __half2*>(f_hi + (p0 + px) * CF + 2 * f2));
      const float2 l = __half22float2(*reinterpret_cast<const __half2*>(f_lo + (p0 + px) * CF + 2 * f2));
      v.x = h.x + l.x; v.y = h.y + l.y;
    }
    sF[px * (CF + 1) + 2 * f2] = v.x; sF[px * (CF + 1) + 2 * f2 + 1] = v.y;
  }
  __syncthreads();
  const int px = threadIdx.x;
  const float* fr = sF + px * (CF + 1);
  for (int ob = 0; ob < NOP; ob += 32) {
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = sB[ob + j];
#pragma unroll 4
    for (int f = 0; f < CF; ++f) {
      const float a = fr[f];
      const float4* w4 = reinterpret_cast<const float4*>(sW + f * NOP + ob);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 w = w4[j];
        acc[4 * j] = fmaf(a, w.x, acc[4 * j]); acc[4 * j + 1] = fmaf(a, w.y, acc[4 * j + 1]);
        acc[4 * j + 2] = fmaf(a, w.z, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(a, w.w, acc[4 * j + 3]);
      }
    }
    if (ob == 0) acc[0] = 1.f / (1.f + expf(-acc[0]));
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 32; ++j) sO[px * 33 + j] = acc[j];
    __syncthreads();
    // coalesced stores: outputs ob..ob+31 of 128 pixels
    for (int e = threadIdx.x; e < 128 * 32; e += blockDim.x) {
      const int q = e / 32, j = e % 32, o = ob + j;
      if (p0 + q >= npix || o >= NO) continue;
      const float v = sO[q * 33 + j];
      if (o == 0) prob[p0 + q] = v; else dist[(p0 + q) * R + (o - 1)] = v;
    }
  }
}

// (pz,py,px) max-pooling of one volume on split planes (3-D U-Net)
__global__ void k_maxpool3d_split(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int D, int H, int W, int C,
                                  int pz, int py, int px, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const int Do = D / pz, Ho = H / py, Wo = W / px, C2 = C / 2;
  const long long total = (long long)Do * Ho * Wo * C2;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c2 = (int)(e % C2); long long r = e / C2;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); const int zo = (int)(r / Ho);
    float m0 = -INFINITY, m1 = -INFINITY;
    for (int a = 0; a < pz; ++a)
      for (int b = 0; b < py; ++b)
        for (int c = 0; c < px; ++c) {
          const size_t off = ((((size_t)zo * pz + a) * H + (size_t)yo * py + b) * W + (size_t)xo * px + c) * C + 2 * c2;
          const float2 h = __half22float2(*reinterpret_cast<const __half2*>(in_hi + off));
          const float2 l = __half22float2(*reinterpret_cast<const __half2*>(in_lo + off));
          m0 = fmaxf(m0, h.x + l.x); m1 = fmaxf(m1, h.y + l.y);
        }
    const __half h0 = __float2half_rn(m0), h1 = __float2half_rn(m1);
    const size_t o = (size_t)e * 2;
    *reinterpret_cast<__half2*>(out_hi + o) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(out_lo + o) = __halves2half2(__float2half_rn(m0 - __half2float(h0)), __float2half_rn(m1 - __half2float(h1)));
  }
}
// fp32 -> split fp16 planes (output of the CUDA-core stem of the 3-D network)
__global__ void k_split_f32(const float* __restrict__ in, long long n, __half* __restrict__ hi, __half* __restrict__ lo, unsigned int* __restrict__ err) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float v = in[e];
    if (!(fabsf(v) <= 65504.f)) atomicOr(err, 0x80000000u);
    const __half h = __float2half_rn(v);
    hi[e] = h; lo[e] = __float2half_rn(v - __half2float(h));
  }
}

// weights (3,3,Cin,Cout) fp32 -> [tap][Cout][Cin] fp16 hi / lo
__global__ void k_split_weights(const float* __restrict__ w, int n_taps, int Cin, int Cout, float scale, __half* __restrict__ w_hi, __half* __restrict__ w_lo) {
  const long long total = (long long)n_taps * Cin * Cout;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(e % Cin); long long r = e / Cin;
    const int co = (int)(r % Cout); const int tap = (int)(r / Cout);
    const float v = w[((size_t)tap * Cin + ci) * Cout + co] * scale;
    const __half h = __float2half_rn(v);
    w_hi[e] = h; w_lo[e] = __float2half_rn(v - __half2float(h));
  }
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int make_act_map(CUtensorMap* m, const __half* base, int n, int h, int w, int c, int kc) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { sdb::set_error("cuTensorMapEncodeTiled entry point not available"); return 1; }
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)h * w * c * 2};
  cuuint32_t box[4] = {(cuuint32_t)kc, 16, 8, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  const CUtensorMapSwizzle sw = (kc * 2 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { sdb::set_error("cuTensorMapEncodeTiled(activation) failed: " + std::to_string((int)r)); return 1; }
  return 0;
}
// weights [n_taps][cout][cin]; box = {kc, nbox output channels, 1 tap}
static int make_w_map(CUtensorMap* m, const __half* base, int cin, int cout, int kc, int nbox, int n_taps) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { sdb::set_error("cuTensorMapEncodeTiled entry point not available"); return 1; }
  cuuint64_t dims[3] = {(cuuint64_t)cin, (cuuint64_t)cout, (cuuint64_t)n_taps};
  cuuint64_t strides[2] = {(cuuint64_t)cin * 2, (cuuint64_t)cin * cout * 2};
  cuuint32_t box[3] = {(cuuint32_t)kc, (cuuint32_t)nbox, 1};
  cuuint32_t es[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = (kc * 2 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { sdb::set_error("cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r)); return 1; }
  return 0;
}

static int g_tc_split_acc = 1;   // see ConvParams::split_acc / sdb_tc_set_split_acc
static int g_tc_variant = 0;     // 0 = auto (persistent, 64-channel K blocks where the channel counts allow), 1 / 3 / 4: see sdb_tc_set_variant
static int g_num_sms = 0;
static unsigned int* g_err_flag = nullptr;      // device flag shared by all launches

template <int N, int KC, bool FUSE = false>
static int launch_wg(const CUtensorMap& a0h, const CUtensorMap& a0l, const CUtensorMap& a1h, const CUtensorMap& a1l,
                     const CUtensorMap& wh, const CUtensorMap& wl, const ConvParams& P, int n_img, cudaStream_t st) {
  using C = WgCfg<N, KC, FUSE>;
  static bool attr = false;
  if (!attr) { SDB_CUDA(cudaFuncSetAttribute(k_conv_wg<N, KC, FUSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM)); attr = true; }
  if (!g_num_sms) { int dev = 0; SDB_CUDA(cudaGetDevice(&dev)); SDB_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev)); }
  const int tiles_x = cdiv(P.W, 16), tiles_y = cdiv(P.H, 8), n_nb = P.heads_R > 0 ? 1 : P.c_out / N;
  const int n_tiles = tiles_x * tiles_y * n_nb * n_img;
  const int grid = (g_tc_variant == 1) ? n_tiles : std::min(n_tiles, g_num_sms);
  const int n_out = (P.heads_R > 0 && !FUSE) ? P.heads_R + 1 : P.c_out;
  sdb::ProfSpan sp;
  sdb::profile_begin("conv_tc", st, &sp);
  k_conv_wg<N, KC, FUSE><<<grid, kThreads, C::SMEM, st>>>(a0h, a0l, a1h, a1l, wh, wl, P, tiles_x, tiles_y, n_nb, n_tiles);
  sdb::profile_end("conv_tc", st, &sp);
  sdb::profile_add_units("conv_tc", (2.0 * P.n_taps * P.c_total * n_out + (FUSE ? 2.0 * N * (P.heads_R + 1) : 0.0)) * (double)P.H * P.W * n_img);     // algorithmic FLOPs
  sdb::g_launch_count++;
  SDB_CUDA(cudaGetLastError());
  return 0;
}

// activation maps of both sources and the weight maps for KC-channel blocks and N-channel output tiles
static int make_conv_maps(CUtensorMap* a0h, CUtensorMap* a0l, CUtensorMap* a1h, CUtensorMap* a1l, CUtensorMap* wh, CUtensorMap* wl,
                          const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo, int c_src1,
                          int n, int h, int w, const void* w_hi, const void* w_lo, int cout, int kc, int nbox, int n_taps) {
  if (make_act_map(a1h, (const __half*)src1_hi, n, h, w, c_src1, kc) || make_act_map(a1l, (const __half*)src1_lo, n, h, w, c_src1, kc)) return 1;
  if (c_src0 > 0) {
    if (make_act_map(a0h, (const __half*)src0_hi, n, h, w, c_src0, kc) || make_act_map(a0l, (const __half*)src0_lo, n, h, w, c_src0, kc)) return 1;
  } else { *a0h = *a1h; *a0l = *a1l; }
  const int cin = c_src0 + c_src1;
  return make_w_map(wh, (const __half*)w_hi, cin, cout, kc, nbox, n_taps) || make_w_map(wl, (const __half*)w_lo, cin, cout, kc, nbox, n_taps);
}

// K block: 64 channels (128-byte swizzled rows) when both sources allow it, else 32; variant 4 forces 32, variant 3 forces 64 where possible
static int pick_kc(int c_src0, int c_src1) {
  const bool k64 = (c_src0 % 64 == 0) && (c_src1 % 64 == 0);
  return (g_tc_variant == 4 || !k64) ? 32 : 64;
}

// 3x3 (n_taps 9) or 3x3x3 (n_taps 27) convolution, Cout in {32, 64, 128, 256} (256 = two 128-channel output tiles)
static int conv_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo, int c_src1,
                   int n, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias, int cout, int relu,
                   int up2x, void* out_hi, void* out_lo, int n_taps, cudaStream_t st) {
  const int cin = c_src0 + c_src1;
  if (!g_err_flag) { SDB_CUDA(cudaMalloc(&g_err_flag, 4)); SDB_CUDA(cudaMemset(g_err_flag, 0, 4)); }
  const int kc = pick_kc(c_src0, c_src1);
  const int nt = std::min(cout, 128);
  CUtensorMap a0h, a0l, a1h, a1l, wh, wl;
  if (make_conv_maps(&a0h, &a0l, &a1h, &a1l, &wh, &wl, src0_hi, src0_lo, c_src0, src1_hi, src1_lo, c_src1, n, h, w, w_hi, w_lo, cout, kc, nt, n_taps))
    return 1;
  ConvParams P;
  P.H = h; P.W = w; P.c_src0 = c_src0; P.c_total = cin; P.c_out = cout; P.relu = relu; P.up2x = up2x; P.bias = d_bias; P.acc_scale = 1.0f / w_scale;
  P.out_hi = (__half*)out_hi; P.out_lo = (__half*)out_lo; P.error_flag = g_err_flag; P.n_taps = n_taps; P.heads_R = 0; P.prob = nullptr; P.dist = nullptr;
  P.fuse_w = nullptr; P.fuse_b = nullptr; P.split_acc = g_tc_split_acc;
#define SDB_WG(NN, KK) return launch_wg<NN, KK>(a0h, a0l, a1h, a1l, wh, wl, P, n, st)
  if (kc == 64) { if (nt == 32) SDB_WG(32, 64); if (nt == 64) SDB_WG(64, 64); SDB_WG(128, 64); }
  if (nt == 32) SDB_WG(32, 32); if (nt == 64) SDB_WG(64, 32); SDB_WG(128, 32);
#undef SDB_WG
}

}  // namespace

// conv3x3 on split-fp16 activations.  src0 (optional, c_src0 channels) and src1 (c_src1 channels) are
// [n,h,w,c] hi/lo planes; weights are the pre-split [9][cout][cin] planes; output hi/lo planes are
// [n,h,w,cout] or, with up2x, [n,2h,2w,cout] with every pixel replicated 2x2 (nearest up-sampling).
extern "C" int sdb_conv3x3_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                              int c_src1, int n, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias, int cout,
                              int relu, int up2x, void* out_hi, void* out_lo, sdb_stream_t stream) {
  if ((c_src0 + c_src1) % 32 || c_src0 % 32 || c_src1 % 32) { sdb::set_error("conv3x3_tc: channel counts must be multiples of 32"); return 1; }
  if (cout != 32 && cout != 64 && cout != 128 && cout != 256) { sdb::set_error("conv3x3_tc: cout must be 32/64/128/256"); return 1; }
  return conv_tc(src0_hi, src0_lo, c_src0, src1_hi, src1_lo, c_src1, n, h, w, w_hi, w_lo, w_scale, d_bias, cout, relu, up2x ? 1 : 0,
                 out_hi, out_lo, 9, (cudaStream_t)stream);
}

// 1x1 heads on the tensor cores: features [n,h,w,cfeat] (split fp16) x head weights [1][NP][cfeat] (split fp16,
// row 0 = prob, rows 1..R = dist, zero padded to NP in {48,80,112,144}) -> prob = sigmoid(.) [n,h,w], dist [n,h,w,R] fp32
extern "C" int sdb_heads_tc(const void* f_hi, const void* f_lo, int cfeat, int n, int h, int w, const void* w_hi, const void* w_lo,
                            float w_scale, const float* d_bias, int np, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cfeat % 64) { sdb::set_error("heads_tc: feature channels must be a multiple of 64"); return 1; }
  if (n_rays + 1 > np) { sdb::set_error("heads_tc: padded head count too small"); return 1; }
  if (np != 48 && np != 80 && np != 112 && np != 144) { sdb::set_error("heads_tc: np must be one of 48, 80, 112, 144"); return 1; }
  if (!g_err_flag) { SDB_CUDA(cudaMalloc(&g_err_flag, 4)); SDB_CUDA(cudaMemset(g_err_flag, 0, 4)); }
  CUtensorMap ah, al, wh, wl;
  if (make_conv_maps(&ah, &al, &ah, &al, &wh, &wl, nullptr, nullptr, 0, f_hi, f_lo, cfeat, n, h, w, w_hi, w_lo, np, 64, np, 1)) return 1;
  ConvParams P;
  P.H = h; P.W = w; P.c_src0 = 0; P.c_total = cfeat; P.c_out = np; P.relu = 0; P.up2x = 0; P.bias = d_bias; P.acc_scale = 1.0f / w_scale;
  P.out_hi = nullptr; P.out_lo = nullptr; P.error_flag = g_err_flag; P.n_taps = 1; P.heads_R = n_rays; P.prob = d_prob; P.dist = d_dist;
  P.fuse_w = nullptr; P.fuse_b = nullptr; P.split_acc = g_tc_split_acc;
  if (np == 48) return launch_wg<48, 64>(ah, al, ah, al, wh, wl, P, n, st);
  if (np == 80) return launch_wg<80, 64>(ah, al, ah, al, wh, wl, P, n, st);
  if (np == 112) return launch_wg<112, 64>(ah, al, ah, al, wh, wl, P, n, st);
  return launch_wg<144, 64>(ah, al, ah, al, wh, wl, P, n, st);
}

// features conv (3x3, Cin <= 64 -> 128, bias, ReLU) fused with the 1x1 heads: prob = sigmoid(f . w_p + b_p),
// dist_k = f . w_k + b_k computed on the fp32 accumulators in the epilogue; the feature map is never stored.
// heads_w: fp32 [128][36] (columns 0..R-1 dist, column 32 prob, rest zero), heads_b: fp32 [36]; n_rays <= 32.
extern "C" int sdb_conv3x3_heads_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                                    int c_src1, int n, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias,
                                    int relu, const float* d_heads_w, const float* d_heads_b, int n_rays, float* d_prob, float* d_dist,
                                    sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int cin = c_src0 + c_src1, cout = 128;
  if (cin % 32 || c_src0 % 32 || c_src1 % 32) { sdb::set_error("conv3x3_heads_tc: channel counts must be multiples of 32"); return 1; }
  if (n_rays < 1 || n_rays > 32) { sdb::set_error("conv3x3_heads_tc: n_rays must be in [1,32]"); return 1; }
  if (!g_err_flag) { SDB_CUDA(cudaMalloc(&g_err_flag, 4)); SDB_CUDA(cudaMemset(g_err_flag, 0, 4)); }
  CUtensorMap a0h, a0l, a1h, a1l, wh, wl;
  if (make_conv_maps(&a0h, &a0l, &a1h, &a1l, &wh, &wl, src0_hi, src0_lo, c_src0, src1_hi, src1_lo, c_src1, n, h, w, w_hi, w_lo, cout, 32, cout, 9))
    return 1;
  ConvParams P;
  P.H = h; P.W = w; P.c_src0 = c_src0; P.c_total = cin; P.c_out = cout; P.relu = relu; P.up2x = 0; P.bias = d_bias; P.acc_scale = 1.0f / w_scale;
  P.out_hi = nullptr; P.out_lo = nullptr; P.error_flag = g_err_flag; P.n_taps = 9; P.heads_R = n_rays; P.prob = d_prob; P.dist = d_dist;
  P.fuse_w = d_heads_w; P.fuse_b = d_heads_b; P.split_acc = g_tc_split_acc;
  return launch_wg<128, 32, true>(a0h, a0l, a1h, a1l, wh, wl, P, n, st);
}

// 3x3x3 convolution of ONE volume [d,h,w,c] (split fp16 planes) on the tensor cores: the z planes are the tensor map's
// image axis and the 27 weight taps [27][cout][cin] (tap = dz*9 + dy*3 + dx).  up2x: 0 none, 2 = nearest 2x2x2.
extern "C" int sdb_conv3x3x3_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                                int c_src1, int d, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias, int cout,
                                int relu, int up2x, void* out_hi, void* out_lo, sdb_stream_t stream) {
  const int cin = c_src0 + c_src1;
  if (cin % 32 || c_src0 % 32 || c_src1 % 32) { sdb::set_error("conv3x3x3_tc: channel counts must be multiples of 32"); return 1; }
  if (cout != 32 && cout != 64 && cout != 128) { sdb::set_error("conv3x3x3_tc: cout must be 32/64/128"); return 1; }
  if (up2x != 0 && up2x != 2) { sdb::set_error("conv3x3x3_tc: up2x must be 0 or 2"); return 1; }
  return conv_tc(src0_hi, src0_lo, c_src0, src1_hi, src1_lo, c_src1, d, h, w, w_hi, w_lo, w_scale, d_bias, cout, relu, up2x,
                 out_hi, out_lo, 27, (cudaStream_t)stream);
}

// A/B switch for tests and profiling: 0 = auto (default), 1 = one tile per CTA (non-persistent grid),
// 3 = persistent with 64-channel K blocks where the channel counts allow, 4 = persistent with 32-channel K blocks
extern "C" int sdb_tc_set_variant(int variant) {
  if (variant != 0 && variant != 1 && variant != 3 && variant != 4) { sdb::set_error("tc_set_variant: 0 (auto), 1, 3 or 4"); return 1; }
  g_tc_variant = variant;
  return 0;
}

extern "C" int sdb_tc_set_split_acc(int on) { g_tc_split_acc = on ? 1 : 0; return 0; }

// non-zero when any tensor-core conv launch since the last call hit a bounded-wait timeout (then results are invalid)
extern "C" int sdb_tc_error_check(sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (!g_err_flag) return 0;
  unsigned int v = 0;
  SDB_CUDA(cudaMemcpyAsync(&v, g_err_flag, 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (v) {
    SDB_CUDA(cudaMemsetAsync(g_err_flag, 0, 4, st));
    if (v & 0x7fffffffu) { sdb::set_error("tensor-core conv: pipeline wait timed out (code " + std::to_string(v & 0x7fffffffu) + ")"); return 1; }
    sdb::set_error("tensor-core conv: fp16 overflow -- an activation exceeded 65504 (or is NaN) in the split-fp16 representation; normalise the input or use the fp32 CUDA-core path");
    return 2;
  }
  return 0;
}

extern "C" int sdb_split_weights(const float* d_w, int cin, int cout, float w_scale, void* w_hi, void* w_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = 9LL * cin * cout;
  SDB_LAUNCH(k_split_weights, (int)std::min<long long>(cdiv(total, 256), 1024), 256, 0, st, d_w, 9, cin, cout, w_scale, (__half*)w_hi, (__half*)w_lo);
  return 0;
}
// (3,3,3,Cin,Cout) -> [27][Cout][Cin] split planes
extern "C" int sdb_split_weights_3d(const float* d_w, int cin, int cout, float w_scale, void* w_hi, void* w_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = 27LL * cin * cout;
  SDB_LAUNCH(k_split_weights, (int)std::min<long long>(cdiv(total, 256), 1024), 256, 0, st, d_w, 27, cin, cout, w_scale, (__half*)w_hi, (__half*)w_lo);
  return 0;
}

extern "C" int sdb_stem_split(const float* d_in, int n, int h, int w, int cin, const float* d_w, const float* d_b, int cout, int relu,
                              void* out_hi, void* out_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cin > 4 || (cout != 32 && cout != 64)) { sdb::set_error("stem_split: cin <= 4 and cout in {32,64}"); return 1; }
  if (!g_err_flag) { SDB_CUDA(cudaMalloc(&g_err_flag, 4)); SDB_CUDA(cudaMemset(g_err_flag, 0, 4)); }
  const size_t smem = (size_t)(9 * cin * cout + cout) * sizeof(float);
  const long long npix = (long long)n * h * w;
  if (cout == 32) SDB_LAUNCH((k_stem_split<32>), cdiv(npix, 128), 128, smem, st, d_in, n, h, w, cin, d_w, d_b, relu, (__half*)out_hi, (__half*)out_lo, g_err_flag);
  else SDB_LAUNCH((k_stem_split<64>), cdiv(npix, 128), 128, smem, st, d_in, n, h, w, cin, d_w, d_b, relu, (__half*)out_hi, (__half*)out_lo, g_err_flag);
  return 0;
}

extern "C" int sdb_maxpool_split(const void* in_hi, const void* in_lo, int n, int h, int w, int c, void* out_hi, void* out_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if ((h & 1) || (w & 1) || (c & 1)) { sdb::set_error("maxpool_split: needs even h, w, c"); return 1; }
  const long long total = (long long)n * (h / 2) * (w / 2) * (c / 2);
  SDB_LAUNCH(k_maxpool_split, (int)std::min<long long>(cdiv(total, 256), 132 * 16), 256, 0, st, (const __half*)in_hi, (const __half*)in_lo, n, h, w, c,
             (__half*)out_hi, (__half*)out_lo);
  return 0;
}

extern "C" int sdb_maxpool3d_split(const void* in_hi, const void* in_lo, int d, int h, int w, int c, int pz, int py, int px,
                                   void* out_hi, void* out_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (pz < 1 || py < 1 || px < 1 || d % pz || h % py || w % px || (c & 1)) { sdb::set_error("maxpool3d_split: sizes must be divisible by the pool, c even"); return 1; }
  const long long total = (long long)(d / pz) * (h / py) * (w / px) * (c / 2);
  SDB_LAUNCH(k_maxpool3d_split, (int)std::min<long long>(cdiv(total, 256), 132 * 16), 256, 0, st, (const __half*)in_hi, (const __half*)in_lo, d, h, w, c,
             pz, py, px, (__half*)out_hi, (__half*)out_lo);
  return 0;
}
extern "C" int sdb_split_f32(const float* d_in, long long n, void* out_hi, void* out_lo, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (!g_err_flag) { SDB_CUDA(cudaMalloc(&g_err_flag, 4)); SDB_CUDA(cudaMemset(g_err_flag, 0, 4)); }
  if (n <= 0) return 0;
  SDB_LAUNCH(k_split_f32, (int)std::min<long long>(cdiv(n, 256), 132 * 32), 256, 0, st, d_in, n, (__half*)out_hi, (__half*)out_lo, g_err_flag);
  return 0;
}

extern "C" int sdb_heads_split(const void* f_hi, const void* f_lo, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                               const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cfeat != 128) { sdb::set_error("heads_split: only 128 feature channels supported"); return 1; }
  const int NO = n_rays + 1, NOP = (NO + 31) / 32 * 32;
  const size_t smem = (size_t)(128 * NOP + NOP + 128 * 129 + 128 * 33) * sizeof(float);
  static bool attr = false;
  if (!attr) { SDB_CUDA(cudaFuncSetAttribute(k_heads_split<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  if (smem > 200 * 1024) { sdb::set_error("heads_split: n_rays too large"); return 1; }
  SDB_LAUNCH((k_heads_split<128>), cdiv(npix, 128), 128, smem, st, (const __half*)f_hi, (const __half*)f_lo, npix, d_wp, d_bp, d_wd, d_bd, n_rays, d_prob, d_dist);
  return 0;
}
