// wgrad_tc -- weight gradient of a stride-1 3x3 / 1x1 "same" convolution on the tensor cores (sm_90a): fp32-grade on split
// operands, or single-pass on plain bf16 operands (the bf16 autocast training step).
//
//   dW[tap][cin][cout] = sum over (b, y, x) of  act[b, y+dy, x+dx, cin] * dY[b, y, x, cout]        (autograd of F.conv2d,
//   model/module.py:241-243, 255-259 under trainer/train_representation_learning.py:112 loss.backward())
//
// As a GEMM the contraction runs over PIXELS while both operands are NHWC (channels contiguous): both are MN-major wgmma
// operands.  A TMA box [64 pixels][64 channels] with SWIZZLE_128B is exactly the canonical MN-major SW128 atom stack
// (8 pixel rows x 128 B per atom, stride-byte-offset 1024 B between 8-row groups); a second box one leading-byte-offset
// further supplies channels 64-127.  One k-step = 128 (M channels) x BN (N channels) x 16 pixels, as two m64 wgmmas (one per
// consumer warpgroup).
//
// SPLIT = true: operands arrive split, [hi | lo | hi] channel blocks (a = hi + lo, bf16 each): every product is
// a_hi*d_hi + a_lo*d_hi + a_hi*d_lo accumulated in fp32 registers -- the same fp32-grade scheme as the forward / dgrad convs.
// SPLIT = false: operands are plain bf16 tensors with C channels; a stage holds one block per operand and a k-step issues one
// wgmma per warpgroup (a third of the MMA work and of the operand bytes), still accumulated in fp32.
//
// Work item = (tap, M chunk of 128 channels, N chunk of BN channels, 64-pixel tile).  Items are dealt to the persistent CTAs
// in contiguous ranges (split-K over pixels); a CTA accumulates in registers while consecutive items belong to the same
// (tap, M chunk, N chunk) and then adds its partial sums to dW with fp32 reductions.
//   warp 8: TMA producer (warp-uniform loop, elect.sync), warps 0-7: two consumer warpgroups, warpgroup g owning accumulator
//   rows [64 g, 64 g + 64) (wgmma, then the reductions straight from the accumulator fragments).
// The tap shift is applied to whichever operand is the activation (4-D box at shifted coordinates, out-of-image = zero = padding).
// `a_is_act` selects which tensor sits on the M side: with dY there (M = cout), which is the preferred form whenever
// Cout % 128 == 0.  When neither channel count is a
// multiple of 128 (64 -> 64, 192 -> 64) the M side is the activation in 64-channel chunks and the two 64-row halves of the
// accumulator hold two different TAPS of it ("pair" mode; the odd ninth tap is paired with a discarded duplicate).
//
// S2 = true: a 3x3, stride-2, pad-1 conv on plain bf16 operands (the semantic encoder under autocast).  The pixel tiles cover
// the OUTPUT grid (dY is read there, unshifted); the activation is read through its parity view [B][H/2][2][W/2][2C]
// (conv_tc2.cu): tap (ky, kx) is the parity class (ky != 1, kx != 1) at the output tile shifted by -1 where the tap index is
// 0, the -1 coordinate being zero-filled by TMA (the padding).
//
// DET (pdae_wgrad_tc_set_deterministic): no float atomics.  Work unit = (group, pixel split), one per CTA: split s of a group
// covers k-tiles [s kpt, s kpt + kpt) and stores its partial tile with plain stores into slot s of a caller-owned workspace
// [splits][taps][Cin][Cout]; the run then adds the slots in split order into dW.  The split count follows the shape alone
// (the least estimated time of the units on a 132-SM H100 SXM, wg_det_splits), so the sums do not depend on the GPU; with one
// split a unit stores straight into dW.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pdae {

constexpr int WG_KT = 64;                 // pixels per k-tile (= rows of one TMA box)
constexpr int WG_BOX = wgmma::MN_BOX;     // bytes of one [64 px][64 ch] box (WG_KT rows of 128 B)
constexpr int WG_THREADS = 288;
constexpr int WG_MAX_ST = 4;              // stage ring depth cap of the split variant (its 48-64 KB stages fit 3-4)
constexpr int WG_MAX_ST_BF16 = 8;         // plain bf16 variant: 24-32 KB stages, up to 8 in the same shared-memory budget
constexpr int WG_SMEM_BUDGET = 220 * 1024;

struct WgradArgs {
  float* dw;
  long long sm, sn, stap;   // element strides of the (m, n, tap) indices inside dw
  int a_is_act;             // 1: M side = activation (shifted per tap), N side = dY; 0: M side = dY, N side = activation
  int Ma, Nb;               // real channel counts on the M / N side (split operands hold 3x: [hi | lo | hi])
  int mchunks, nchunks, taps, ksize;
  int pair;                 // 1: 64-channel M chunks, the 128 accumulator rows hold TWO taps (activation on the M side)
  int tw, th, tn, tiles_x, tiles_y, tiles_b, ktiles;
  int B, H, W;
  int stages;
  long long items;          // taps * mchunks * nchunks * ktiles
  int det_splits, det_kpt;  // DET: pixel splits per group and k-tiles per split
  long long det_slot;       // DET: elements of one slot (= of dW)
};

namespace wg {
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
__device__ __forceinline__ uint32_t mb_try(uint32_t bar, uint32_t parity, uint32_t hint) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity), "r"(hint)
      : "memory");
  return done;
}
__device__ __noinline__ void mb_wait(uint32_t bar, uint32_t parity) {
  uint32_t n = 0;
  while (!mb_try(bar, parity, 20000u))
    if (++n > 4000000u) __trap();  // a protocol bug must trap, never hang the GPU
}
__device__ __forceinline__ void tma_ld4(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_ld5(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// stride-2 activation box of tap `tap` (ky = tap / 3, kx = tap % 3) at channel c of a C-channel tensor, output tile (x0, y0, b0)
__device__ __forceinline__ void tma_ld_s2(uint32_t dst, const CUtensorMap* m, uint32_t bar, int C, int c, int tap, int x0, int y0,
                                          int b0) {
  const int ky = tap / 3, kx = tap - 3 * ky;
  tma_ld5(dst, m, bar, (kx != 1) * C + c, x0 - (kx == 0), ky != 1, y0 - (ky == 0), b0);
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
}  // namespace wg

template <int BN, bool SPLIT, bool S2 = false, bool DET = false>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, WgradArgs p) {
  using namespace wg;
  static_assert(!(SPLIT && S2), "stride-2 weight gradients take plain bf16 operands");
  extern __shared__ uint8_t smem_raw[];
  constexpr int MAX_ST = SPLIT ? WG_MAX_ST : WG_MAX_ST_BF16;
  __shared__ __align__(8) uint64_t bar_full[MAX_ST], bar_empty[MAX_ST];
  constexpr int NBOX_B = BN / 64;                       // 64-channel boxes of the N-side tile
  constexpr int A_BYTES = 2 * WG_BOX;                   // M = 128 channels = two boxes
  constexpr int B_BYTES = NBOX_B * WG_BOX;
  constexpr int NBLK = SPLIT ? 2 : 1;                   // channel blocks loaded per operand: (hi, lo) or the plain tensor
  constexpr int STAGE = NBLK * (A_BYTES + B_BYTES);
  const uint32_t smem0 = (s_u32(smem_raw) + 1023u) & ~1023u;
  const int S = p.stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long per_cta = (p.items + gridDim.x - 1) / gridDim.x;
  // DET: blockIdx.x = group * det_splits + split
  const long long det_g = DET ? blockIdx.x / p.det_splits : 0, det_s = DET ? blockIdx.x - det_g * p.det_splits : 0;
  const long long it_begin = DET ? det_g * p.ktiles + det_s * p.det_kpt : (long long)blockIdx.x * per_cta;
  const long long it_end = DET ? det_g * p.ktiles + min((long long)p.ktiles, (det_s + 1) * p.det_kpt)
                               : (it_begin + per_cta < p.items ? it_begin + per_cta : p.items);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mb_init(s_u32(&bar_full[s]), 1);
      mb_init(s_u32(&bar_empty[s]), 8);   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ================= TMA producer =================
    int s = 0;
    uint32_t ph = 0;
    for (long long it = it_begin; it < it_end; ++it) {
      const long long g = it / p.ktiles;
      int kt = (int)(it - g * p.ktiles);
      int gg = (int)g;
      const int nc = gg % p.nchunks; gg /= p.nchunks;
      const int mc = gg % p.mchunks;
      const int tap = gg / p.mchunks;
      const int tx = kt % p.tiles_x; kt /= p.tiles_x;
      const int ty = kt % p.tiles_y;
      const int bt = kt / p.tiles_y;
      const int x0 = tx * p.tw, y0 = ty * p.th, b0 = bt * p.tn;
      // the activation carries the tap shift; in pair mode the two M boxes are two taps of the same 64 channels
      int tj[2], ax[2], ay[2], am[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        tj[j] = p.pair ? min(2 * tap + j, p.taps - 1) : tap;
        const int dy = p.ksize == 3 ? tj[j] / 3 - 1 : 0, dx = p.ksize == 3 ? tj[j] % 3 - 1 : 0;
        ax[j] = p.a_is_act ? x0 + dx : x0;
        ay[j] = p.a_is_act ? y0 + dy : y0;
        am[j] = p.pair ? mc * 64 : mc * 128 + j * 64;
      }
      const int bdy = p.ksize == 3 ? tap / 3 - 1 : 0, bdx = p.ksize == 3 ? tap % 3 - 1 : 0;
      const int bx = p.a_is_act ? x0 : x0 + bdx, by = p.a_is_act ? y0 : y0 + bdy;
      const int n0 = nc * BN;
      mb_wait(s_u32(&bar_empty[s]), ph ^ 1u);
      const uint32_t full = s_u32(&bar_full[s]);
      const uint32_t base = smem0 + (uint32_t)(s * STAGE);
      if constexpr (S2) {
        if (elect_one()) {
          mb_expect_tx(full, (uint32_t)STAGE);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint32_t dst = base + (uint32_t)(j * WG_BOX);
            if (p.a_is_act) tma_ld_s2(dst, &tmA, full, p.Ma, am[j], tj[j], x0, y0, b0);
            else tma_ld4(dst, &tmA, full, am[j], x0, y0, b0);
          }
#pragma unroll
          for (int j = 0; j < NBOX_B; ++j) {
            const uint32_t dst = base + (uint32_t)(A_BYTES + j * WG_BOX);
            if (p.a_is_act) tma_ld4(dst, &tmB, full, n0 + j * 64, x0, y0, b0);
            else tma_ld_s2(dst, &tmB, full, p.Nb, n0 + j * 64, tap, x0, y0, b0);
          }
        }
      } else if (elect_one()) {
        mb_expect_tx(full, (uint32_t)STAGE);
#pragma unroll
        for (int h = 0; h < NBLK; ++h) {       // hi block (channel offset 0), lo block (channel offset Ma / Nb)
#pragma unroll
          for (int j = 0; j < 2; ++j)
            tma_ld4(base + (uint32_t)(h * A_BYTES + j * WG_BOX), &tmA, full, h * p.Ma + am[j], ax[j], ay[j], b0);
#pragma unroll
          for (int j = 0; j < NBOX_B; ++j)
            tma_ld4(base + (uint32_t)(NBLK * A_BYTES + h * B_BYTES + j * WG_BOX), &tmB, full, h * p.Nb + n0 + j * 64, bx, by, b0);
        }
      }
      __syncwarp();
      if (++s == S) { s = 0; ph ^= 1u; }
    }
  } else {
    // ================= consumers: warpgroup wg = M box wg (accumulator rows [64 wg, 64 wg + 64)) =================
    const int wgi = warp >> 2, t = threadIdx.x & 127;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // fp32 reductions of a finished (tap, M chunk, N chunk) group into dW, straight from the accumulator fragments
    auto flush = [&](long long gid) {
      int gg = (int)gid;
      const int nc = gg % p.nchunks; gg /= p.nchunks;
      const int mc = gg % p.mchunks;
      const int tap = gg / p.mchunks;
      const int tap_w = p.pair ? 2 * tap + wgi : tap;             // pair mode: rows 64-127 belong to the second tap
      if (tap_w >= p.taps) return;
      float* base = p.dw + det_s * p.det_slot + (long long)tap_w * p.stap + (long long)(nc * BN) * p.sn;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        const int m = wgmma::frag_row(t, i);
        const int ch_m = p.pair ? mc * 64 + m : mc * 128 + 64 * wgi + m;
        float* o = base + (long long)ch_m * p.sm + (long long)wgmma::frag_col(t, i) * p.sn;
        if constexpr (DET) *o = acc[i];
        else atomicAdd(o, acc[i]);
      }
    };
    int s = 0;
    uint32_t ph = 0;
    long long cur_g = -1;
    for (long long it = it_begin; it < it_end; ++it) {
      const long long g = it / p.ktiles;
      const bool first = g != cur_g;
      if (first) {
        if (cur_g >= 0) flush(cur_g);
        cur_g = g;
      }
      mb_wait(s_u32(&bar_full[s]), ph);
      const uint32_t base = smem0 + (uint32_t)(s * STAGE) + (uint32_t)(wgi * WG_BOX);
      if constexpr (SPLIT) {
        const uint64_t a_hi = wgmma::desc_mnmajor(base), a_lo = wgmma::desc_mnmajor(base + A_BYTES);
        const uint32_t bb = smem0 + (uint32_t)(s * STAGE) + 2u * A_BYTES;
        const uint64_t b_hi = wgmma::desc_mnmajor(bb), b_lo = wgmma::desc_mnmajor(bb + B_BYTES);
        wgmma::fence();
#pragma unroll
        for (int k = 0; k < WG_KT / 16; ++k) {         // 16 pixels per k-step
          const uint64_t o = (uint64_t)k * wgmma::K16_STEP_MNMAJOR;
          wgmma::mma<BN, 1>(acc, a_hi + o, b_hi + o, (uint32_t)(!(first && k == 0)));
          wgmma::mma<BN, 1>(acc, a_lo + o, b_hi + o, 1u);
          wgmma::mma<BN, 1>(acc, a_hi + o, b_lo + o, 1u);
        }
      } else {                                          // plain bf16: one wgmma per k-step
        const uint64_t a_d = wgmma::desc_mnmajor(base);
        const uint64_t b_d = wgmma::desc_mnmajor(smem0 + (uint32_t)(s * STAGE) + (uint32_t)A_BYTES);
        wgmma::fence();
#pragma unroll
        for (int k = 0; k < WG_KT / 16; ++k) {
          const uint64_t o = (uint64_t)k * wgmma::K16_STEP_MNMAJOR;
          wgmma::mma<BN, 1>(acc, a_d + o, b_d + o, (uint32_t)(!(first && k == 0)));
        }
      }
      wgmma::commit();
      wgmma::wait<0>();
      if (lane == 0) mb_arrive(s_u32(&bar_empty[s]));
      if (++s == S) { s = 0; ph ^= 1u; }
    }
    if (cur_g >= 0) flush(cur_g);
  }
}

typedef CUresult (*EncodeTiledFnW)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnW encode_fnw() {
  static EncodeTiledFnW fn = nullptr;
  if (fn) return fn;
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  fn = (EncodeTiledFnW)sym;
  return fn;
}

static int pow2_tile_w(int W, int cap) {
  int t = 1;
  while (t * 2 <= cap && W % (t * 2) == 0) t *= 2;
  return t;
}

template <int BN, bool SPLIT, bool S2 = false, bool DET = false>
static cudaError_t launch_wg(const CUtensorMap& a, const CUtensorMap& b, const WgradArgs& args, int grid, size_t smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<BN, SPLIT, S2, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, 221 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  wgrad_tc_kernel<BN, SPLIT, S2, DET><<<grid, WG_THREADS, smem, s>>>(a, b, args);
  return cudaPeekAtLastError();
}

}  // namespace pdae

using namespace pdae;

struct pdae_wgrad_tc_plan {
  CUtensorMap tmA, tmB;
  WgradArgs args;
  int BN, split, grid;
  int s2;           // stride-2 3x3 conv (wgrad_tc_kernel's S2)
  size_t smem;
  int det;          // pdae_wgrad_tc_set_deterministic: the DET kernel
  float* det_out;   // DET with several splits: dW, which the run sums the slots into (args.dw is then the workspace)
};

static int g_num_sms_w = 0;

extern "C" int pdae_wgrad_tc_supported(int H, int W, int Cin, int Cout, int ksize) {
  if (ksize != 1 && ksize != 3) return 0;
  if (Cin % 64 || Cout % 64) return 0;
  const int tw = pow2_tile_w(W, WG_KT), th = pow2_tile_w(H, WG_KT / tw);
  const int tn = WG_KT / (tw * th);
  return (W % tw == 0 && H % th == 0 && tw * th * tn == WG_KT && tn <= 64) ? 1 : 0;
}

// split: act / dy hold [hi | lo | hi] blocks of 3*C channels; otherwise plain bf16 with C channels.
// s2: 3x3 stride-2 pad-1 conv, H x W = the activation's size, dy on the H/2 x W/2 grid (plain bf16 only)
static int wgrad_create(pdae_wgrad_tc_plan** plan_out, const void* act, const void* dy, float* dw, int B, int H, int W, int Cin,
                        int Cout, int ksize, bool split, bool s2 = false) {
  PDAE_REQUIRE(plan_out && act && dy && dw, "wgrad_tc_create: null pointer");
  if (s2) {
    PDAE_REQUIRE(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                 "wgrad_tc_create_bf16_s2: B=%d H=%d W=%d: H and W must be even and positive", B, H, W);
    PDAE_REQUIRE(ksize == 3 && !split && pdae_conv_s2_tc_supported(H, W, Cin, Cout),
                 "wgrad_tc_create_bf16_s2: unsupported channels Cin=%d Cout=%d (multiples of 64)", Cin, Cout);
  } else {
    PDAE_REQUIRE(pdae_wgrad_tc_supported(H, W, Cin, Cout, ksize), "wgrad_tc_create: unsupported shape H=%d W=%d Cin=%d Cout=%d k=%d", H, W,
                 Cin, Cout, ksize);
  }
  PDAE_REQUIRE(!(((uintptr_t)act | (uintptr_t)dy) & 15) && !((uintptr_t)dw & 3),
               "wgrad_tc_create: act / dy must be 16-byte aligned (TMA), dw 4-byte aligned");
  const int Ha = H, Wa = W;          // activation size
  if (s2) { H /= 2; W /= 2; }        // from here on: the pixel grid the tiles cover (dY's)
  EncodeTiledFnW enc = encode_fnw();
  PDAE_REQUIRE(enc != nullptr, "wgrad_tc_create: cuTensorMapEncodeTiled unavailable (no driver)");
  if (g_num_sms_w == 0) {
    int dev = 0;
    PDAE_CUDA(cudaGetDevice(&dev));
    PDAE_CUDA(cudaDeviceGetAttribute(&g_num_sms_w, cudaDevAttrMultiProcessorCount, dev));
  }
  pdae_wgrad_tc_plan* pl = new pdae_wgrad_tc_plan();
  WgradArgs& a = pl->args;
  a.dw = dw;
  a.a_is_act = (Cout % 128 == 0) ? 0 : 1;        // prefer dY on the M side: coalesced reductions into dW[tap][cin][cout]
  a.pair = (a.a_is_act && Cin % 128) ? 1 : 0;    // neither side fills 128 accumulator rows: two taps of 64 channels do
  a.Ma = a.a_is_act ? Cin : Cout;
  a.Nb = a.a_is_act ? Cout : Cin;
  a.sm = a.a_is_act ? Cout : 1;
  a.sn = a.a_is_act ? 1 : Cout;
  a.stap = (long long)Cin * Cout;
  const int BN = (a.Nb % 128 == 0) ? 128 : 64;
  pl->BN = BN;
  pl->split = split ? 1 : 0;
  pl->s2 = s2 ? 1 : 0;
  a.mchunks = a.pair ? a.Ma / 64 : a.Ma / 128; a.nchunks = a.Nb / BN; a.taps = ksize * ksize; a.ksize = ksize;
  a.tw = pow2_tile_w(W, WG_KT); a.th = pow2_tile_w(H, WG_KT / a.tw); a.tn = WG_KT / (a.tw * a.th);
  a.tiles_x = W / a.tw; a.tiles_y = H / a.th; a.tiles_b = (B + a.tn - 1) / a.tn;
  a.ktiles = a.tiles_x * a.tiles_y * a.tiles_b;
  a.B = B; a.H = H; a.W = W;
  a.items = (long long)(a.pair ? (a.taps + 1) / 2 : a.taps) * a.mchunks * a.nchunks * a.ktiles;
  const int stage = (split ? 2 : 1) * (2 * WG_BOX + (BN / 64) * WG_BOX);
  const int max_st = split ? WG_MAX_ST : WG_MAX_ST_BF16;
  int stages = (WG_SMEM_BUDGET - 1024) / stage;
  if (stages > max_st) stages = max_st;
  a.stages = stages;
  pl->smem = (size_t)stages * stage + 1024;
  pl->grid = a.items < g_num_sms_w ? (int)a.items : g_num_sms_w;
  const void* At = a.a_is_act ? act : dy;
  const void* Bt = a.a_is_act ? dy : act;
  const int Ca = (split ? 3 : 1) * a.Ma, Cb = (split ? 3 : 1) * a.Nb;
  cuuint32_t estr4[4] = {1, 1, 1, 1};
  cuuint32_t box[4] = {64, (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
  cuuint32_t estr5[5] = {1, 1, 1, 1, 1};
  cuuint32_t box5[5] = {64, (cuuint32_t)a.tw, 1, (cuuint32_t)a.th, (cuuint32_t)a.tn};
  for (int i = 0; i < 2; ++i) {
    const int C = i ? Cb : Ca;
    CUresult r;
    if (s2 && (i == 0) == (a.a_is_act == 1)) {
      // the activation's parity view [B][Ha/2][2][Wa/2][2C] (conv_tc2.cu)
      const cuuint64_t c2 = 2ull * C;
      cuuint64_t dims[5] = {c2, (cuuint64_t)Wa / 2, 2, (cuuint64_t)Ha / 2, (cuuint64_t)B};
      cuuint64_t strides[4] = {c2 * 2, (cuuint64_t)Wa * C * 2, 2ull * Wa * C * 2, (cuuint64_t)Ha * Wa * C * 2};
      r = enc(i ? &pl->tmB : &pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(i ? Bt : At), dims, strides, box5, estr5,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
      r = enc(i ? &pl->tmB : &pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(i ? Bt : At), dims, strides, box,
              estr4, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) {
      delete pl;
      set_error("wgrad_tc_create: cuTensorMapEncodeTiled failed with %d", (int)r);
      return PDAE_EINVAL;
    }
  }
  *plan_out = pl;
  return PDAE_OK;
}

extern "C" int pdae_wgrad_tc_create(pdae_wgrad_tc_plan** plan_out, const void* act3_bf16, const void* dy3_bf16, float* dw, int B,
                                    int H, int W, int Cin, int Cout, int ksize) {
  return wgrad_create(plan_out, act3_bf16, dy3_bf16, dw, B, H, W, Cin, Cout, ksize, true);
}

extern "C" int pdae_wgrad_tc_create_bf16(pdae_wgrad_tc_plan** plan_out, const void* act_bf16, const void* dy_bf16, float* dw, int B,
                                         int H, int W, int Cin, int Cout, int ksize) {
  return wgrad_create(plan_out, act_bf16, dy_bf16, dw, B, H, W, Cin, Cout, ksize, false);
}

extern "C" int pdae_wgrad_tc_create_bf16_s2(pdae_wgrad_tc_plan** plan_out, const void* act_bf16, const void* dy_bf16, float* dw,
                                            int B, int H, int W, int Cin, int Cout) {
  return wgrad_create(plan_out, act_bf16, dy_bf16, dw, B, H, W, Cin, Cout, 3, false, true);
}

// ---- deterministic plans (kernel header, DET) ----------------------------------------------------------------------------
constexpr int WG_DET_SMS = 132;   // SMs of an H100 SXM: a constant, so that the split count follows the shape alone

// The split count with the least estimated time on WG_DET_SMS SMs running one unit each: waves x k-tiles per unit, plus the
// slot traffic (each split writes and the reduction reads one dW image: about n / 750000 k-tile times of a split-operand
// unit at HBM speed, three times that for the single-pass bf16 unit, whose k-tile is a third of the work).
static int wg_det_splits(const WgradArgs& a, int split, int* kpt) {
  const long long groups = a.items / a.ktiles, n = (long long)a.taps * a.stap;
  double best = 0.0;
  int bk = a.ktiles;
  for (int s = 1; s <= a.ktiles; ++s) {
    const int k = (a.ktiles + s - 1) / s;
    if (s > 1 && (a.ktiles + k - 1) / k != s) continue;                 // every split non-empty
    const double waves = (double)((groups * s + WG_DET_SMS - 1) / WG_DET_SMS);
    const double cost = waves * k + (s > 1 ? (double)s * n / 750000.0 * (split ? 1 : 3) : 0.0);
    if (s == 1 || cost < best) { best = cost; bk = k; }
  }
  if (kpt) *kpt = bk;
  return (a.ktiles + bk - 1) / bk;
}

extern "C" int64_t pdae_wgrad_tc_det_workspace_bytes(const pdae_wgrad_tc_plan* pl) {
  if (!pl) {
    set_error("wgrad_tc_det_workspace_bytes: null plan");
    return PDAE_EINVAL;
  }
  const int splits = wg_det_splits(pl->args, pl->split, nullptr);
  return splits > 1 ? (int64_t)splits * pl->args.taps * pl->args.stap * (int64_t)sizeof(float) : 0;
}

extern "C" int pdae_wgrad_tc_set_deterministic(pdae_wgrad_tc_plan* pl, float* workspace, int64_t workspace_bytes) {
  PDAE_REQUIRE(pl, "wgrad_tc_set_deterministic: null plan");
  PDAE_REQUIRE(!pl->det, "wgrad_tc_set_deterministic: the plan is deterministic already");
  const int64_t need = pdae_wgrad_tc_det_workspace_bytes(pl);
  PDAE_REQUIRE(workspace_bytes >= need && (need == 0 || workspace),
               "wgrad_tc_set_deterministic: workspace of %lld bytes, %lld needed (pdae_wgrad_tc_det_workspace_bytes)",
               (long long)workspace_bytes, (long long)need);
  PDAE_REQUIRE(!((uintptr_t)workspace & 3), "wgrad_tc_set_deterministic: workspace must be 4-byte aligned");
  WgradArgs& a = pl->args;
  a.det_splits = wg_det_splits(a, pl->split, &a.det_kpt);
  a.det_slot = (long long)a.taps * a.stap;
  pl->grid = (int)(a.items / a.ktiles) * a.det_splits;
  if (need > 0) {
    pl->det_out = a.dw;
    a.dw = workspace;
  }
  pl->det = 1;
  return PDAE_OK;
}

extern "C" int pdae_wgrad_tc_run(const pdae_wgrad_tc_plan* pl, pdae_stream_t stream) {
  PDAE_REQUIRE(pl, "wgrad_tc_run: null plan");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e;
  if (pl->det) {
#define WG_DET(BN, SPLIT, S2) launch_wg<BN, SPLIT, S2, true>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s)
    if (pl->s2) e = pl->BN == 128 ? WG_DET(128, false, true) : WG_DET(64, false, true);
    else if (pl->split) e = pl->BN == 128 ? WG_DET(128, true, false) : WG_DET(64, true, false);
    else e = pl->BN == 128 ? WG_DET(128, false, false) : WG_DET(64, false, false);
#undef WG_DET
    if (e == cudaSuccess && pl->det_out) e = launch_slot_sum(pl->args.dw, pl->args.det_splits, pl->args.det_slot, pl->det_out, s);
  } else if (pl->s2)
    e = pl->BN == 128 ? launch_wg<128, false, true>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s)
                      : launch_wg<64, false, true>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s);
  else if (pl->split)
    e = pl->BN == 128 ? launch_wg<128, true>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s)
                      : launch_wg<64, true>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s);
  else
    e = pl->BN == 128 ? launch_wg<128, false>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s)
                      : launch_wg<64, false>(pl->tmA, pl->tmB, pl->args, pl->grid, pl->smem, s);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("launch of wgrad_tc_kernel<%d, %s> failed: %s", pl->BN, pl->split ? "split" : "bf16", cudaGetErrorString(e));
    return PDAE_ECUDA;
  }
  return PDAE_OK;
}

extern "C" void pdae_wgrad_tc_destroy(pdae_wgrad_tc_plan* pl) { delete pl; }
