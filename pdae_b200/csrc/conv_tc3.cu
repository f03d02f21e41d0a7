// conv_tc3 -- 3x3 convolution with the GroupNorm-apply / AdaGN / SiLU prologue FUSED into the operand path (sm_90a).
//
// Reference op chain (model/module.py:278-297, 361-384):   h = conv3x3(SiLU(GN(x)))   and
// out = conv3x3(SiLU((1+zs)*(GN(h)*(1+s)+sh)+zsh)) [+ skip_1x1(x_raw)] + residual.  The GroupNorm / AdaGN / z-modulation
// algebra is folded by gn_coef_ch into per-(image, channel) coefficients (a, b); this kernel applies
// SiLU(a*x + b) while it builds the tensor-core A operand, so the activated tensor never exists in HBM.
//
//   warp 13     : TMA producer of the weight (B) tiles                       [tap][Cout][Cin] bf16, SWIZZLE_128B
//   warp 12     : TMA producer of the RAW (pre-normalisation) halo: per 64-channel k-block ONE 4-D box (64 ch x 10 x 18 px,
//                 out-of-image pixels zero-filled = the conv padding) lands, 128B-swizzled, directly in the operand stage.
//   warps 8-11  : TRANSFORM group: rewrites that stage IN PLACE, x -> SiLU(a*x+b) (shared memory -> shared memory, no
//                 global-load latency on its path, no extra buffer); padding pixels stay zero.
//   warps 0-7   : two consumer warpgroups (output rows 0-7 / 8-15 of the 16 x 8 tile): wgmma into fp32 registers, then the
//                 epilogue from the accumulator fragments: +bias (+residual) -> swizzled staging -> per-channel GroupNorm
//                 sums (for the NEXT GroupNorm) -> TMA store        (as conv_tc2)
// All nine taps of the k-block address that single tile: tap (dy, dx) is the wgmma descriptor started (dy*10 + dx) rows
// into it with a stride-byte-offset of 10 rows (1280 B) between its 8-pixel row groups -- the 128B swizzle is a function
// of the absolute shared-memory address, so a row-shifted window of a tile written with address-based swizzling is a valid
// K-major operand.  Shared-memory operand writes per k-block drop from 9 x 16 KB (one TMA box per tap, conv_tc2) to 23 KB,
// and the separate gn_apply pass over HBM disappears.
//
// X3 = split-operand mode (fp32-grade products): the source is fp32; the transform writes TWO halo tiles
// hi = bf16(v), lo = bf16(v - hi); weights come as one merged [W_hi | W_lo] tile; per tap the consumers accumulate
// a_hi*W_hi + a_hi*W_lo + a_lo*W_hi.
//
// The 1x1 skip convolution of a channel-changing ResBlock (model/module.py:268-276) rides along as extra k-blocks whose
// transform is the identity and whose single tap is the centre window.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pdae {

constexpr int T3_BK = 64;
constexpr int T3_TW = 8, T3_TH = 16;                  // output tile (pixels): 8 wide x 16 tall, one image
constexpr int T3_P = T3_TW + 2;                       // halo pitch (pixels per halo row)
constexpr int T3_HROWS = T3_TH + 2;
constexpr int T3_HALO = T3_P * T3_HROWS;              // 180 halo pixels = 180 shared-memory rows of 128 B
constexpr int T3_HALO_BYTES = 23 * 1024;              // 180 * 128 = 23040 B, padded to a 1024-B multiple (swizzle atom alignment)
constexpr int T3_STG_BYTES = 128 * 128;
constexpr int T3_MAX_SA = 4, T3_MAX_SB = 12;
constexpr int T3_XF_WARPS = 4;
// 448 threads = 14 warps: at most 4 warps per scheduler partition, so each thread may hold 128 registers (the consumers keep
// BN / 2 fp32 accumulators each).
constexpr int T3_THREADS = 256 + 32 * T3_XF_WARPS + 32 + 32;
constexpr int T3_W_RAWPROD = 8 + T3_XF_WARPS, T3_W_BPROD = 9 + T3_XF_WARPS;   // warps 0-7: consumers, 8-11: transform group
constexpr int T3_XF_SLOTS = 4 * T3_XF_WARPS;                                  // pixel slots per pass (8 threads x 16 B per pixel)
constexpr int T3_XF_PASSES = (T3_HALO + T3_XF_SLOTS - 1) / T3_XF_SLOTS;     // 12 passes of 16 pixel slots

struct ConvTc3Args {
  int C1, C2;                           // pre-activation conv input = virtual channel concat C1 | C2 (tensor maps tmS1 | tmS2)
  const float* ab;                      // [B][2][C1+C2]: a | b of SiLU(a*x+b)
  int S1, S2;                           // raw input of the fused 1x1 skip conv: S1 | S2 channels (tensor maps tmK1 | tmK2)
  const float* bias;
  const float* res_f32;                 // X3 only: fp32 NHWC residual read straight from global memory by the epilogue
  float* ch_stats;                      // [B][Cout][2] (sum, sum^2) accumulators of the OUTPUT or nullptr; DET: the slots
                                        // [B][tiles_x * tiles_y][Cout][2], one per (image, tile of the image), plain stores
  int B, H, W, Cout;
  int tiles_x, tiles_y, tiles_m, tiles_total;
  int kblocks, kblocks2;
  int sa, sb;                           // pipeline depths: halo stages / weight-tile stages
  int has_res, out_bf16, silu;
};

// ---- small PTX helpers (same protocol as conv_tc2.cu) -------------------------------------------------------------------
namespace t3 {
__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mb_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mb_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}
// Slow path of a wait: mbarrier.try_wait with a SUSPEND-TIME HINT, so a waiting warp sleeps in hardware (it is woken by the
// completing arrive) instead of re-issuing the poll: most of the CTA's warps are waiting at any time, and hot polling takes
// issue slots away from the warps that have work.
__device__ __forceinline__ uint32_t mb_try_sleep(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity), "r"(20000u)
      : "memory");
  return done;
}
__device__ __noinline__ void mb_wait_slow(uint32_t bar, uint32_t parity) {
  uint32_t n = 0;
  while (!mb_try_sleep(bar, parity))
    if (++n > 4000000u) __trap();  // a protocol bug must trap, never hang the GPU
}
__device__ __forceinline__ void mb_wait(uint32_t bar, uint32_t parity) {
  if (mb_try(bar, parity)) return;   // fast path: already complete
  mb_wait_slow(bar, parity);
}
__device__ __forceinline__ void tma_ld4(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_ld3(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_st4(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m), "r"(src),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// One elected lane of a fully converged warp.  The producer loops are executed by ALL 32 lanes (warp-uniform control flow and
// operands, which the compiler keeps in uniform registers); only the TMA instruction itself is predicated on the elected lane.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// barrier of the 256 consumer threads (the other warps never join it)
__device__ __forceinline__ void cons_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// byte offset of (row, 16-byte chunk) inside a SWIZZLE_128B tile whose base is 1024-B aligned
__device__ __forceinline__ uint32_t swz(int row, int chunk16) { return (uint32_t)(row * 128 + ((chunk16 ^ (row & 7)) << 4)); }

// SiLU of the fused prologue.  bf16 mode: one MUFU (tanh.approx), the result is rounded to bf16 anyway.  Split mode: ex2 + rcp
// approximations (rel. error ~1e-7), well inside the 2^-17 the hi/lo pair resolves.
template <bool X3>
__device__ __forceinline__ float act(float x, int silu) {
  if (!silu) return x;
  if (X3) return __fdividef(x, 1.0f + __expf(-x));
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
}  // namespace t3

// DET: deterministic statistics (pdae_conv_tc3_set_deterministic): no atomics; each tile's per-channel sums go to the tile's own
// slot, which depends on the tile alone (not on the CTA that ran it).
template <int BN, bool X3, bool OB, bool DET = false>
__global__ void __launch_bounds__(T3_THREADS, 1)
conv_tc3_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmB2,
                const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR,
                const __grid_constant__ CUtensorMap tmS1, const __grid_constant__ CUtensorMap tmS2,
                const __grid_constant__ CUtensorMap tmK1, const __grid_constant__ CUtensorMap tmK2, ConvTc3Args p) {
  using namespace t3;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_a_full[T3_MAX_SA], bar_a_empty[T3_MAX_SA], bar_raw[T3_MAX_SA];
  __shared__ __align__(8) uint64_t bar_b_full[T3_MAX_SB], bar_b_empty[T3_MAX_SB];
  __shared__ __align__(8) uint64_t bar_res;
  __shared__ float st_acc[2][BN];   // [sum | sum^2][channel] of the current (image, n-tile)
  __shared__ float st_part[2][256]; // per-chunk partial sums [sum | sum^2][row run * CW + column]

  // Split mode: W_hi and W_lo of a (tap, k-block) arrive as ONE 2*BN-row tile [W_hi | W_lo]; per k-step the consumers run
  // a_hi x W_hi, a_hi x W_lo and a_lo x W_hi into the same accumulators.
  constexpr int B_BYTES = (X3 ? 2 * BN : BN) * T3_BK * 2;
  constexpr int A_STAGE = (X3 ? 2 : 1) * T3_HALO_BYTES;
  constexpr int CW = OB ? 64 : 32;             // accumulator columns per staging tile (128-byte rows)
  constexpr int NCH = BN / CW;
  constexpr int RPT = CW / 2;                  // statistics: rows per thread (256 threads = CW columns x 128 / RPT row runs)
  const uint32_t smem0 = (s_u32(smem_raw) + 1023u) & ~1023u;
  const int SA = p.sa, SB = p.sb;
  const uint32_t a_base = smem0;
  const uint32_t b_base = a_base + (uint32_t)(SA * A_STAGE);
  const uint32_t stg_out = b_base + (uint32_t)(SB * B_BYTES);
  const uint32_t stg_res = stg_out + (uint32_t)T3_STG_BYTES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_it = p.kblocks + p.kblocks2;
  const int per_cta = (p.tiles_total + (int)gridDim.x - 1) / (int)gridDim.x;
  const int tile_begin = (int)blockIdx.x * per_cta;
  const int tile_end = min(p.tiles_total, tile_begin + per_cta);
  const int tiles_img = p.tiles_x * p.tiles_y;

  for (int j = threadIdx.x; j < BN; j += T3_THREADS) {
    st_acc[0][j] = 0.f;
    st_acc[1][j] = 0.f;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < SA; ++s) {
      mb_init(s_u32(&bar_a_full[s]), T3_XF_WARPS);   // one elected arrive per transform warp
      mb_init(s_u32(&bar_a_empty[s]), 8);            // one arrive per consumer warp
      mb_init(s_u32(&bar_raw[s]), 1);
    }
    for (int s = 0; s < SB; ++s) {
      mb_init(s_u32(&bar_b_full[s]), 1);
      mb_init(s_u32(&bar_b_empty[s]), 8);
    }
    mb_init(s_u32(&bar_res), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmS1) : "memory");
  }
  __syncthreads();

  if (warp == T3_W_BPROD) {
    // ================= weight-tile TMA producer (warp-uniform loop, elected lane issues) =================
    int s = 0;
    uint32_t ph = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      const int n0 = (tile / p.tiles_m) * BN;
      for (int it = 0; it < total_it; ++it) {
        const bool skipk = it >= p.kblocks;
        const int ntap = skipk ? 1 : 9;
        for (int tap = 0; tap < ntap; ++tap) {
          mb_wait(s_u32(&bar_b_empty[s]), ph ^ 1u);
          const uint32_t full = s_u32(&bar_b_full[s]);
          const uint32_t dst = b_base + (uint32_t)(s * B_BYTES);
          if (elect_one()) {
            mb_expect_tx(full, (uint32_t)B_BYTES);
            if (!skipk) tma_ld3(dst, &tmB, full, it * T3_BK, n0, tap * (X3 ? 2 : 1));
            else tma_ld3(dst, &tmB2, full, (it - p.kblocks) * T3_BK, n0, 0);
          }
          __syncwarp();
          if (++s == SB) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else if (warp == T3_W_RAWPROD) {
    // ================= raw-halo TMA producer (warp-uniform loop, elected lane issues) =================
    // item (tile, k-block) -> ONE box of the pre-activation tensor: 64 channels x 10 x 18 pixels starting one pixel up-left of
    // the output tile; out-of-image coordinates are zero-filled by the TMA unit.  Split mode: fp32 source, two 32-channel
    // boxes (128 B rows each) land in the stage's hi / lo regions and are split in place by the transform group.
    constexpr uint32_t RAW_TX = (uint32_t)(T3_HALO * 128 * (X3 ? 2 : 1));
    int s = 0;
    uint32_t ph = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      int mt = tile % p.tiles_m;
      const int tx = mt % p.tiles_x;
      mt /= p.tiles_x;
      const int ty = mt % p.tiles_y;
      const int b0 = mt / p.tiles_y;
      const int x0 = tx * T3_TW - 1, y0 = ty * T3_TH - 1;
      for (int it = 0; it < total_it; ++it) {
        const CUtensorMap* m;
        int c0;
        if (it < p.kblocks) {
          const int kc = it * T3_BK;
          if (kc < p.C1) { m = &tmS1; c0 = kc; } else { m = &tmS2; c0 = kc - p.C1; }
        } else {
          const int kc = (it - p.kblocks) * T3_BK;
          if (kc < p.S1) { m = &tmK1; c0 = kc; } else { m = &tmK2; c0 = kc - p.S1; }
        }
        mb_wait(s_u32(&bar_a_empty[s]), ph ^ 1u);
        const uint32_t full = s_u32(&bar_raw[s]);
        const uint32_t dst = a_base + (uint32_t)(s * A_STAGE);
        if (elect_one()) {
          mb_expect_tx(full, RAW_TX);
          tma_ld4(dst, m, full, c0, x0, y0, b0);
          if (X3) tma_ld4(dst + (uint32_t)T3_HALO_BYTES, m, full, c0 + 32, x0, y0, b0);
        }
        __syncwarp();
        if (++s == SA) { s = 0; ph ^= 1u; }
      }
    }
  } else if (warp >= 8 && warp < 8 + T3_XF_WARPS) {
    // ================= transform group: raw halo (in the operand stage) -> SiLU(a*x+b) [-> hi | lo], IN PLACE =================
    const int tt = (int)threadIdx.x - 256;   // 0..T3_XF_SLOTS*8-1
    const int slot = tt >> 3, ch8 = tt & 7;  // pixel slot (T3_XF_SLOTS per pass), 8-channel chunk (16 B of bf16 operand)
    const int C = p.C1 + p.C2;
    int s = 0;
    uint32_t ph = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      int mt = tile % p.tiles_m;
      const int tx = mt % p.tiles_x;
      mt /= p.tiles_x;
      const int ty = mt % p.tiles_y;
      const int b0 = mt / p.tiles_y;
      const int x0 = tx * T3_TW - 1, y0 = ty * T3_TH - 1;   // image coordinates of halo pixel (0, 0)
      // halo pixels of this thread that are real image pixels (the others are conv padding and stay zero)
      uint32_t inimg = 0, interior = 0;
#pragma unroll
      for (int j = 0; j < T3_XF_PASSES; ++j) {
        const int hp = j * T3_XF_SLOTS + slot;
        const int hy = hp / T3_P, hx = hp - hy * T3_P;
        const int gy = y0 + hy, gx = x0 + hx;
        if (hp < T3_HALO && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) {
          inimg |= 1u << j;
          if (hy >= 1 && hy <= T3_TH && hx >= 1 && hx <= T3_TW) interior |= 1u << j;
        }
      }
      for (int it = 0; it < total_it; ++it) {
        const bool skipk = it >= p.kblocks;
        float ca[8], cb[8];
        if (!skipk) {
          const float* ap = p.ab + ((long long)b0 * 2) * C + it * T3_BK + ch8 * 8;
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(ap)), a1 = __ldg(reinterpret_cast<const float4*>(ap + 4));
          const float4 q0 = __ldg(reinterpret_cast<const float4*>(ap + C)), q1 = __ldg(reinterpret_cast<const float4*>(ap + C + 4));
          ca[0] = a0.x; ca[1] = a0.y; ca[2] = a0.z; ca[3] = a0.w; ca[4] = a1.x; ca[5] = a1.y; ca[6] = a1.z; ca[7] = a1.w;
          cb[0] = q0.x; cb[1] = q0.y; cb[2] = q0.z; cb[3] = q0.w; cb[4] = q1.x; cb[5] = q1.y; cb[6] = q1.z; cb[7] = q1.w;
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) { ca[j] = 1.f; cb[j] = 0.f; }
        }
        const int silu = skipk ? 0 : p.silu;
        mb_wait(s_u32(&bar_raw[s]), ph);
        const uint32_t hi_base = a_base + (uint32_t)(s * A_STAGE);
        // bf16 mode: the raw input of the 1x1 skip conv IS the operand -- nothing to do.  Split mode: it still needs the hi/lo
        // split, but only where the centre tap reads it.
        const uint32_t todo = skipk ? (X3 ? interior : 0u) : inimg;
#pragma unroll
        for (int j = 0; j < T3_XF_PASSES; ++j) {
          if (todo & (1u << j)) {
            const int hp = j * T3_XF_SLOTS + slot;
            float v[8];
            if (X3) {
              // raw fp32: channels 0-31 of the k-block sit in the hi region, 32-63 in the lo region (128-B swizzled rows)
              const uint32_t rrow = hi_base + (ch8 < 4 ? 0u : (uint32_t)T3_HALO_BYTES) + (uint32_t)hp * 128u;
              const int q = (ch8 & 3) * 2;
              asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3])
                           : "r"(rrow + (uint32_t)((q ^ (hp & 7)) << 4)));
              asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7])
                           : "r"(rrow + (uint32_t)(((q + 1) ^ (hp & 7)) << 4)));
            } else {
              uint32_t w[4];
              asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                           : "r"(hi_base + swz(hp, ch8)));
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                v[2 * e] = __uint_as_float(w[e] << 16);
                v[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
              }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = act<X3>(fmaf(ca[e], v[e], cb[e]), silu);
            uint32_t h[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) h[e] = pack_bf16(v[2 * e], v[2 * e + 1]);
            uint32_t l[4];
            if (X3) {
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float r0 = v[2 * e] - __uint_as_float(h[e] << 16);
                const float r1 = v[2 * e + 1] - __uint_as_float(h[e] & 0xffff0000u);
                l[e] = pack_bf16(r0, r1);
              }
              // the 8 lanes that share this pixel row have read their raw chunks (above) before any of them overwrites the
              // row: same warp, same branch, program order; the 8-lane barrier makes it hold under independent scheduling
              __syncwarp(0xFFu << (lane & 24));
            }
            const uint32_t dst = hi_base + swz(hp, ch8);
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
            if (X3)
              asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dst + (uint32_t)T3_HALO_BYTES), "r"(l[0]), "r"(l[1]),
                           "r"(l[2]), "r"(l[3])
                           : "memory");
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mb_arrive(s_u32(&bar_a_full[s]));
        if (++s == SA) { s = 0; ph ^= 1u; }
      }
    }
  } else if (warp < 8) {
    // ================= consumers: warpgroup wg computes output rows [8 wg, 8 wg + 8) of the 16 x 8 tile, then both run the
    // epilogue straight from the accumulator fragments (as conv_tc2) =================
    constexpr uint32_t A_SBO = (uint32_t)T3_P * 128u;   // 8-pixel row groups of the halo are one halo row (10 px) apart
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int ct = threadIdx.x;                // 0..255
    const bool elected = ct == 0;
    int rc = 0;
    int sa = 0, sb = 0;
    uint32_t pha = 0, phb = 0;
    const uint32_t obuf = stg_out, rbuf = stg_res;
    const uint32_t rbar = s_u32(&bar_res);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      const int nt = tile / p.tiles_m;
      int mt = tile - nt * p.tiles_m;
      const int tx = mt % p.tiles_x;
      mt /= p.tiles_x;
      const int ty = mt % p.tiles_y;
      const int b0 = mt / p.tiles_y;
      const int x0 = tx * T3_TW, y0 = ty * T3_TH, n0 = nt * BN;
      if (!X3 && p.has_res && elected) {       // residual chunk 0 (lands while the main loop runs)
        mb_expect_tx(rbar, T3_STG_BYTES);
        tma_ld4(rbuf, &tmR, rbar, n0, x0, y0, b0);
      }
      // ---- main loop: per k-block one halo stage, per tap one weight stage; a weight stage is released once the MMAs
      // reading it have retired, the halo stage at the end of its k-block ----
      uint32_t started = 0;                    // 0 until the tile's first MMA (which overwrites)
      int pend_b = -1;
      for (int it = 0; it < total_it; ++it) {
        mb_wait(s_u32(&bar_a_full[sa]), pha);
        const bool skipk = it >= p.kblocks;
        const int ntap = skipk ? 1 : 9;
        const uint32_t a_hi = a_base + (uint32_t)(sa * A_STAGE) + (uint32_t)wg * (8u * A_SBO);
        int ty3 = skipk ? 1 : 0, tx3 = skipk ? 1 : 0;    // tap = (ty3, tx3); the 1x1 skip conv reads the centre tap
        for (int tp = 0; tp < ntap; ++tp) {
          const uint32_t off = (uint32_t)(ty3 * T3_P + tx3) * 128u;
          if (++tx3 == 3) { tx3 = 0; ++ty3; }
          const uint64_t ad_hi = wgmma::desc_sw128(a_hi + off, 16u, A_SBO);
          mb_wait(s_u32(&bar_b_full[sb]), phb);
          const uint64_t bd = wgmma::desc_sw128(b_base + (uint32_t)(sb * B_BYTES), 16u, 1024u);
          wgmma::fence();
#pragma unroll
          for (int k = 0; k < T3_BK / 16; ++k)
            wgmma::mma<BN, 0>(acc, ad_hi + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), started | (uint32_t)(k != 0));
          if (X3) {
            const uint64_t ad_lo = wgmma::desc_sw128(a_hi + (uint32_t)T3_HALO_BYTES + off, 16u, A_SBO);
            const uint64_t bd_lo = bd + (uint64_t)((BN * 128) >> 4);   // W_lo: the second BN rows of the merged tile
#pragma unroll
            for (int k = 0; k < T3_BK / 16; ++k) {
              wgmma::mma<BN, 0>(acc, ad_hi + (uint64_t)(2 * k), bd_lo + (uint64_t)(2 * k), 1u);   // a_hi x W_lo
              wgmma::mma<BN, 0>(acc, ad_lo + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), 1u);      // a_lo x W_hi
            }
          }
          wgmma::commit();
          started = 1u;
          wgmma::wait<1>();
          if (pend_b >= 0 && lane == 0) mb_arrive(s_u32(&bar_b_empty[pend_b]));
          pend_b = sb;
          if (++sb == SB) { sb = 0; phb ^= 1u; }
        }
        wgmma::wait<0>();
        if (lane == 0) {
          mb_arrive(s_u32(&bar_b_empty[pend_b]));
          mb_arrive(s_u32(&bar_a_empty[sa]));
        }
        pend_b = -1;
        if (++sa == SA) { sa = 0; pha ^= 1u; }
      }

#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        float v[CW / 2];
#pragma unroll
        for (int q = 0; q < CW / 2; ++q) v[q] = acc[c * (CW / 2) + q];
        if (p.bias) {
#pragma unroll
          for (int q = 0; q < CW / 2; q += 2) {
            const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c * CW + wgmma::frag_col(t, q)));
            v[q] += bv.x; v[q + 1] += bv.y;
          }
        }
        if (X3 && p.has_res) {
          // split mode: the fp32 residual comes straight from global memory -- no shared-memory staging, which leaves room
          // for a deeper weight pipeline
#pragma unroll
          for (int q = 0; q < CW / 2; q += 2) {
            const int r = 64 * wg + wgmma::frag_row(t, q);
            const float2 rv = __ldg(reinterpret_cast<const float2*>(
                p.res_f32 + (((long long)b0 * p.H + y0 + (r >> 3)) * p.W + x0 + (r & 7)) * p.Cout + n0 + c * CW + wgmma::frag_col(t, q)));
            v[q] += rv.x; v[q + 1] += rv.y;
          }
        }
        if (!X3 && p.has_res) {
          mb_wait(rbar, (uint32_t)(rc & 1));
#pragma unroll
          for (int q = 0; q < CW / 2; q += 2) {
            const int r = 64 * wg + wgmma::frag_row(t, q), cl = wgmma::frag_col(t, q);
            if (OB) {
              uint32_t w;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(rbuf + swz(r, cl >> 3) + (uint32_t)((cl & 7) * 2)));
              v[q] += __uint_as_float(w << 16);
              v[q + 1] += __uint_as_float(w & 0xffff0000u);
            } else {
              float2 rv;
              asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(rv.x), "=f"(rv.y)
                           : "r"(rbuf + swz(r, cl >> 2) + (uint32_t)((cl & 3) * 4)));
              v[q] += rv.x; v[q + 1] += rv.y;
            }
          }
          ++rc;
        }
        if (elected) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // previous TMA store has read the staging buffer
        cons_bar();
        if (!X3 && p.has_res && elected && c + 1 < NCH) {
          mb_expect_tx(rbar, T3_STG_BYTES);
          tma_ld4(rbuf, &tmR, rbar, n0 + (c + 1) * CW, x0, y0, b0);
        }
#pragma unroll
        for (int q = 0; q < CW / 2; q += 2) {
          const int r = 64 * wg + wgmma::frag_row(t, q), cl = wgmma::frag_col(t, q);
          if (OB) {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(obuf + swz(r, cl >> 3) + (uint32_t)((cl & 7) * 2)),
                         "r"(pack_bf16(v[q], v[q + 1]))
                         : "memory");
          } else {
            asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(obuf + swz(r, cl >> 2) + (uint32_t)((cl & 3) * 4)), "f"(v[q]),
                         "f"(v[q + 1])
                         : "memory");
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        cons_bar();
        if (elected) {
          tma_st4(&tmO, obuf, n0 + c * CW, x0, y0, b0);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (p.ch_stats) {
          // per-channel partial sums over this tile's rows, read back from the staged (rounded) values:
          // thread -> column (ct % CW), rows [(ct / CW) * RPT, +RPT); accumulated in shared memory across the CTA's tiles of an image
          const int col = ct % CW, r0 = (ct / CW) * RPT;
          const uint32_t cbyte = OB ? (uint32_t)((col & 7) * 2) : (uint32_t)((col & 3) * 4);
          const int cchunk = OB ? (col >> 3) : (col >> 2);
          float sacc = 0.f, qq = 0.f;
#pragma unroll 8
          for (int rr = r0; rr < r0 + RPT; ++rr) {
            float x;
            if (OB) {
              unsigned short h;
              asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(obuf + swz(rr, cchunk) + cbyte));
              x = __uint_as_float(((uint32_t)h) << 16);
            } else {
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(obuf + swz(rr, cchunk) + cbyte));
            }
            sacc += x;
            qq = fmaf(x, x, qq);
          }
          // the row runs of a column are added in a fixed order by one thread: repeated runs give identical statistics
          st_part[0][ct] = sacc;
          st_part[1][ct] = qq;
          cons_bar();
          if (ct < CW) {
            float s2 = 0.f, q2 = 0.f;
#pragma unroll
            for (int g = 0; g < 256 / CW; ++g) {
              s2 += st_part[0][g * CW + ct];
              q2 += st_part[1][g * CW + ct];
            }
            if constexpr (DET) {
              const int pimg = (tile - nt * p.tiles_m) % tiles_img;
              *reinterpret_cast<float2*>(p.ch_stats + (((long long)b0 * tiles_img + pimg) * p.Cout + n0 + c * CW + ct) * 2) =
                  make_float2(s2, q2);
            } else {
              st_acc[0][c * CW + ct] += s2;
              st_acc[1][c * CW + ct] += q2;
            }
          }
        }
      }
      if (!DET && p.ch_stats) {
        bool flush = tile + 1 >= tile_end;
        if (!flush) {
          const int nt2 = (tile + 1) / p.tiles_m;
          const int b2 = ((tile + 1) - nt2 * p.tiles_m) / tiles_img;
          flush = nt2 != nt || b2 != b0;
        }
        if (flush) {
          cons_bar();   // every thread's shared-memory atomics are done before these reads
          for (int j = ct; j < BN; j += 256) {
            float* dst = p.ch_stats + ((long long)b0 * p.Cout + n0 + j) * 2;
            atomicAdd(dst, st_acc[0][j]);
            atomicAdd(dst + 1, st_acc[1][j]);
            st_acc[0][j] = 0.f;
            st_acc[1][j] = 0.f;
          }
          cons_bar();
        }
      }
    }
    if (elected) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

typedef CUresult (*EncodeTiledFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn3 encode_fn3() {
  static EncodeTiledFn3 fn = nullptr;
  if (fn) return fn;
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  fn = (EncodeTiledFn3)sym;
  return fn;
}

template <int BN, bool X3, bool OB, bool DET = false>
static cudaError_t launch_tc3(const CUtensorMap& b, const CUtensorMap& b2, const CUtensorMap& o, const CUtensorMap& r,
                              const CUtensorMap* sk, const ConvTc3Args& args, int grid, size_t smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc3_kernel<BN, X3, OB, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, 221 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  conv_tc3_kernel<BN, X3, OB, DET><<<grid, T3_THREADS, smem, s>>>(b, b2, o, r, sk[0], sk[1], sk[2], sk[3], args);
  return cudaPeekAtLastError();
}

}  // namespace pdae

using namespace pdae;

struct pdae_conv_tc3_plan {
  CUtensorMap tmB, tmB2, tmO, tmR;
  CUtensorMap tmS[4];   // raw halo sources: conv input (C1 | C2), skip-conv input (S1 | S2)
  ConvTc3Args args;
  int BN, x3, grid;
  size_t smem;
  int det;              // pdae_conv_tc3_set_deterministic: the DET kernel
  float* det_stats;     // DET with several tiles per image: the [B][Cout][2] sums the slots are reduced into (else nullptr)
};

static int g_num_sms3 = 0;

extern "C" int pdae_conv_tc3_supported(int H, int W, int Cin, int Cout) {
  return (H % T3_TH == 0 && W % T3_TW == 0 && Cin % T3_BK == 0 && Cout % 64 == 0) ? 1 : 0;
}

extern "C" int pdae_conv_tc3_create(pdae_conv_tc3_plan** plan_out, const void* src1, int C1, const void* src2, int C2,
                                    int src_dtype, const float* ab, int silu, const void* w, const float* bias,
                                    const void* skp1, int S1, const void* skp2, int S2, const void* w_skip,
                                    const void* residual, void* out, int out_dtype, float* ch_stats, int B, int H, int W,
                                    int Cout, int bn_override) {
  PDAE_REQUIRE(plan_out && src1 && ab && w && out, "conv_tc3_create: null pointer");
  PDAE_REQUIRE(src_dtype == PDAE_BF16 || src_dtype == PDAE_F32, "conv_tc3_create: bad source dtype");
  PDAE_REQUIRE(out_dtype == PDAE_BF16 || out_dtype == PDAE_F32, "conv_tc3_create: bad out dtype");
  PDAE_REQUIRE(!(src_dtype == PDAE_F32 && residual && out_dtype != PDAE_F32),
               "conv_tc3_create: the split mode reads an fp32 residual (output must be fp32 too)");
  const bool x3 = src_dtype == PDAE_F32;
  const int Cin = C1 + C2, Cs = S1 + S2;
  PDAE_REQUIRE(C1 > 0 && C1 % T3_BK == 0 && C2 % T3_BK == 0 && (C2 == 0 || src2), "conv_tc3_create: bad C1=%d C2=%d", C1, C2);
  PDAE_REQUIRE(S1 % T3_BK == 0 && S2 % T3_BK == 0 && (Cs == 0 || (skp1 && w_skip && S1 > 0)) && (S2 == 0 || skp2),
               "conv_tc3_create: bad fused-skip operands S1=%d S2=%d", S1, S2);
  PDAE_REQUIRE(!(Cs > 0 && residual), "conv_tc3_create: a block has an identity residual OR a skip conv, not both");
  PDAE_REQUIRE(pdae_conv_tc3_supported(H, W, Cin, Cout), "conv_tc3_create: unsupported shape H=%d W=%d Cin=%d Cout=%d", H, W, Cin, Cout);
  PDAE_REQUIRE(!(((uintptr_t)src1 | (uintptr_t)src2 | (uintptr_t)skp1 | (uintptr_t)skp2 | (uintptr_t)w | (uintptr_t)w_skip |
                  (uintptr_t)out | (uintptr_t)residual | (uintptr_t)bias | (uintptr_t)ab) & 15),
               "conv_tc3_create: pointers must be 16-byte aligned");
  EncodeTiledFn3 enc = encode_fn3();
  PDAE_REQUIRE(enc != nullptr, "conv_tc3_create: cuTensorMapEncodeTiled unavailable (no driver)");
  if (g_num_sms3 == 0) {
    int dev = 0;
    PDAE_CUDA(cudaGetDevice(&dev));
    PDAE_CUDA(cudaDeviceGetAttribute(&g_num_sms3, cudaDevAttrMultiProcessorCount, dev));
  }
  pdae_conv_tc3_plan* pl = new pdae_conv_tc3_plan();
  ConvTc3Args& a = pl->args;
  a.C1 = C1; a.C2 = C2; a.ab = ab;
  a.S1 = S1; a.S2 = S2;
  a.bias = bias; a.ch_stats = ch_stats; a.res_f32 = x3 ? (const float*)residual : nullptr;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout;
  a.tiles_x = W / T3_TW; a.tiles_y = H / T3_TH; a.tiles_m = a.tiles_x * a.tiles_y * B;
  a.kblocks = Cin / T3_BK; a.kblocks2 = Cs / T3_BK;
  a.has_res = residual != nullptr; a.out_bf16 = out_dtype == PDAE_BF16; a.silu = silu;
  pl->x3 = x3 ? 1 : 0;
  int BN;
  // BN <= 128: each consumer thread holds BN / 2 fp32 accumulators within a 128-register budget
  if ((bn_override == 64 || bn_override == 128) && Cout % bn_override == 0) BN = bn_override;
  else BN = (Cout % 128 == 0) ? 128 : 64;
  pl->BN = BN;
  a.tiles_total = a.tiles_m * (Cout / BN);
  pl->grid = a.tiles_total < g_num_sms3 ? a.tiles_total : g_num_sms3;
  const int a_stage = (x3 ? 2 : 1) * T3_HALO_BYTES, b_bytes = (x3 ? 2 * BN : BN) * T3_BK * 2;
  const int staging = ((a.has_res && !x3) ? 2 : 1) * T3_STG_BYTES;   // split mode reads its residual from global memory
  const int budget = 220 * 1024 - 1024 - staging;
  // the transform is software-pipelined, so two halo stages suffice; the weight tiles need depth (bytes in flight from L2)
  int sa = 2;
  int sb = (budget - sa * a_stage) / b_bytes;
  if (sb > T3_MAX_SB) sb = T3_MAX_SB;
  if (budget - sa * a_stage - sb * b_bytes >= a_stage) sa = 3;
  if (!x3 && a.kblocks2 > 0) {
    // fused 1x1 skip conv in the fast mode: its k-blocks carry one tap per 23 KB raw box, so their cost is the TMA
    // latency / number of stages in flight -- trade weight-pipeline depth for a fourth halo stage
    int sbw = (budget - 4 * a_stage) / b_bytes;
    if (sbw > T3_MAX_SB) sbw = T3_MAX_SB;
    if (sbw >= 4) { sa = 4; sb = sbw; }
  }
  if (x3 && BN == 64) {
    // 64-wide split mode: a k-block is short on the tensor pipe against the round trip of its halo stage (raw TMA -> in-place
    // split -> MMAs -> release), so the stage count bounds the rate: prefer three halo stages
    int sbw = (budget - 3 * a_stage) / b_bytes;
    if (sbw > T3_MAX_SB) sbw = T3_MAX_SB;
    if (sbw >= 3) { sa = 3; sb = sbw; }
  }
  if (sb < 2) {
    delete pl;
    PDAE_REQUIRE(false, "conv_tc3_create: shared-memory budget too small (BN=%d x3=%d)", BN, (int)x3);
  }
  a.sa = sa; a.sb = sb;
  pl->smem = (size_t)sa * a_stage + (size_t)sb * b_bytes + staging + 1024;

  auto fail = [&](const char* what, int code) {
    delete pl;
    set_error("conv_tc3_create: cuTensorMapEncodeTiled(%s) failed with %d", what, code);
    return PDAE_EINVAL;
  };
  {   // raw halo boxes: 64 channels (bf16) / 32 channels (fp32: two boxes per k-block) x 10 x 18 pixels of one image
    const void* sp[4] = {src1, src2, skp1, skp2};
    const int sc[4] = {C1, C2, S1, S2};
    const int esz = x3 ? 4 : 2;
    for (int i = 0; i < 4; ++i) {
      if (!sp[i] || sc[i] <= 0) { pl->tmS[i] = CUtensorMap(); continue; }
      cuuint64_t dims[4] = {(cuuint64_t)sc[i], (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)sc[i] * esz, (cuuint64_t)W * sc[i] * esz, (cuuint64_t)H * W * sc[i] * esz};
      cuuint32_t box[4] = {(cuuint32_t)(x3 ? 32 : 64), (cuuint32_t)T3_P, (cuuint32_t)T3_HROWS, 1};
      cuuint32_t estr4[4] = {1, 1, 1, 1};
      CUresult r = enc(&pl->tmS[i], x3 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                       const_cast<void*>(sp[i]), dims, strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail("source", (int)r);
    }
    if (!src2 || C2 <= 0) pl->tmS[1] = pl->tmS[0];
    if (!skp1 || S1 <= 0) pl->tmS[2] = pl->tmS[0];
    if (!skp2 || S2 <= 0) pl->tmS[3] = pl->tmS[2];
  }
  const int nmat = x3 ? 2 : 1;
  {
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout, (cuuint64_t)(9 * nmat)};
    cuuint64_t strides[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cout * Cin * 2};
    cuuint32_t box[3] = {(cuuint32_t)T3_BK, (cuuint32_t)BN, (cuuint32_t)nmat};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("W", (int)r);
  }
  pl->tmB2 = pl->tmB;
  if (Cs > 0) {
    cuuint64_t dims[3] = {(cuuint64_t)Cs, (cuuint64_t)Cout, (cuuint64_t)nmat};
    cuuint64_t strides[2] = {(cuuint64_t)Cs * 2, (cuuint64_t)Cout * Cs * 2};
    cuuint32_t box[3] = {(cuuint32_t)T3_BK, (cuuint32_t)BN, (cuuint32_t)nmat};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmB2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w_skip), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("W_skip", (int)r);
  }
  {
    const int esz = a.out_bf16 ? 2 : 4;
    cuuint32_t estr4[4] = {1, 1, 1, 1};
    cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cout * esz, (cuuint64_t)W * Cout * esz, (cuuint64_t)H * W * Cout * esz};
    cuuint32_t box[4] = {(cuuint32_t)(a.out_bf16 ? 64 : 32), (cuuint32_t)T3_TW, (cuuint32_t)T3_TH, 1};
    const CUtensorMapDataType dt = a.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUresult r = enc(&pl->tmO, dt, 4, out, dims, strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("O", (int)r);
    pl->tmR = pl->tmO;
    if (a.has_res) {
      r = enc(&pl->tmR, dt, 4, const_cast<void*>(residual), dims, strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail("R", (int)r);
    }
  }
  *plan_out = pl;
  return PDAE_OK;
}

// Deterministic statistics: the tiles' per-channel sums go to fixed slots [B][P][Cout][2] (P = tiles per image) in `workspace`
// and are summed over P in order into the plan's ch_stats by the same run.  With one tile per image the slots ARE ch_stats and
// no workspace is needed.  Without statistics the DET kernel is the default one, and nothing changes.
static int tc3_tiles_img(const pdae_conv_tc3_plan* pl) { return pl->args.tiles_x * pl->args.tiles_y; }

extern "C" int64_t pdae_conv_tc3_det_workspace_bytes(const pdae_conv_tc3_plan* pl) {
  if (!pl) {
    set_error("conv_tc3_det_workspace_bytes: null plan");
    return PDAE_EINVAL;
  }
  const float* stats = pl->det ? pl->det_stats : pl->args.ch_stats;
  const int P = tc3_tiles_img(pl);
  if (!stats || P == 1) return 0;
  return (int64_t)pl->args.B * P * pl->args.Cout * 2 * (int64_t)sizeof(float);
}

extern "C" int pdae_conv_tc3_set_deterministic(pdae_conv_tc3_plan* pl, float* workspace, int64_t workspace_bytes) {
  PDAE_REQUIRE(pl, "conv_tc3_set_deterministic: null plan");
  PDAE_REQUIRE(!pl->det, "conv_tc3_set_deterministic: the plan is deterministic already");
  const int64_t need = pdae_conv_tc3_det_workspace_bytes(pl);
  PDAE_REQUIRE(workspace_bytes >= need && (need == 0 || workspace),
               "conv_tc3_set_deterministic: workspace of %lld bytes, %lld needed (pdae_conv_tc3_det_workspace_bytes)",
               (long long)workspace_bytes, (long long)need);
  PDAE_REQUIRE(!((uintptr_t)workspace & 7), "conv_tc3_set_deterministic: workspace must be 8-byte aligned");
  pl->det = 1;
  if (need > 0) {
    pl->det_stats = pl->args.ch_stats;
    pl->args.ch_stats = workspace;
  }
  return PDAE_OK;
}

extern "C" int pdae_conv_tc3_run(const pdae_conv_tc3_plan* pl, pdae_stream_t stream) {
  PDAE_REQUIRE(pl, "conv_tc3_run: null plan");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e;
#define T3_GO(BN, X3, D) (pl->args.out_bf16 ? launch_tc3<BN, X3, true, D>(pl->tmB, pl->tmB2, pl->tmO, pl->tmR, pl->tmS, pl->args, pl->grid, pl->smem, s) \
                                            : launch_tc3<BN, X3, false, D>(pl->tmB, pl->tmB2, pl->tmO, pl->tmR, pl->tmS, pl->args, pl->grid, pl->smem, s))
  if (pl->det) {
    if (pl->x3) e = pl->BN == 64 ? T3_GO(64, true, true) : T3_GO(128, true, true);
    else e = pl->BN == 64 ? T3_GO(64, false, true) : T3_GO(128, false, true);
    if (e == cudaSuccess && pl->det_stats)
      e = launch_stat_parts_reduce(pl->args.ch_stats, pl->args.B, tc3_tiles_img(pl), pl->args.Cout, pl->det_stats, s);
  } else if (pl->x3) e = pl->BN == 64 ? T3_GO(64, true, false) : T3_GO(128, true, false);
  else e = pl->BN == 64 ? T3_GO(64, false, false) : T3_GO(128, false, false);
#undef T3_GO
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("launch of conv_tc3_kernel<%d,%d> failed: %s", pl->BN, pl->x3, cudaGetErrorString(e));
    return PDAE_ECUDA;
  }
  return PDAE_OK;
}

extern "C" void pdae_conv_tc3_destroy(pdae_conv_tc3_plan* pl) { delete pl; }
