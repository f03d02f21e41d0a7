// Tensor-core implicit-GEMM convolution for sm_90a:  TMA (im2col-free, OOB zero fill = conv padding)
//   -> 128B-swizzled shared-memory stages -> wgmma (bf16 x bf16 -> fp32 accumulators in registers)
//   -> epilogue (+bias, +residual) -> fp32 NHWC.
//
// GEMM view per CTA: D[128 pixels][BN couts] = sum over (tap, 64-channel block) of
//     A_tap[128 pixels][64 ch] * W_tap[BN couts][64 ch]^T
// The 128-pixel M tile is a (tn images) x (th rows) x (tw cols) box of the NHWC activation, fetched by
// ONE 4-D TMA per (tap, channel block) at coordinates shifted by the tap offset; out-of-image
// coordinates are zero-filled by the TMA unit, which is exactly the conv's zero padding.  Both operands
// land K-major with the 128-byte swizzle, i.e. the canonical wgmma SW128 layout (8-row atoms of 1024 B).
//
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups (tile rows 0-63 / 64-127: wgmma + epilogue),
// warp 8 = TMA producer.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pdae {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;                         // bf16 elements = 128 bytes = one swizzle row
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;     // 16 KB
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_THREADS = 288;

struct ConvTcArgs {
  const float* bias;
  const float* residual;
  float* out;
  int B, H, W, Cout;
  int tw, th, tn;        // pixel box of one M tile (tw*th*tn == 128)
  int tiles_x, tiles_y;  // tiles per image row / column
  int taps, ksize, kblocks;  // kblocks = Cin/64
  int stages;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must surface as a trapped kernel (error code), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB, ConvTcArgs p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[TC_MAX_STAGES];
  __shared__ __align__(8) uint64_t bar_empty[TC_MAX_STAGES];

  constexpr int B_BYTES = BN * TC_BK * 2;
  constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SW128 atoms need 1024-B alignment
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.stages;

  // ---- tile coordinates ----
  int mt = blockIdx.x;
  const int tx = mt % p.tiles_x;
  mt /= p.tiles_x;
  const int ty = mt % p.tiles_y;
  const int bt = mt / p.tiles_y;
  const int x0 = tx * p.tw, y0 = ty * p.th, b0 = bt * p.tn;
  const int n0 = blockIdx.y * BN;
  const int total_k = p.taps * p.kblocks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ===== TMA producer =====
      for (int it = 0; it < total_k; ++it) {
        const int s = it % S;
        const uint32_t ph = (uint32_t)((it / S) & 1);
        mbar_wait(smem_u32(&bar_empty[s]), ph ^ 1u);
        const uint32_t full = smem_u32(&bar_full[s]);
        mbar_expect_tx(full, STAGE_BYTES);
        const int tap = it / p.kblocks, kb = it - tap * p.kblocks;
        const int dy = p.ksize == 3 ? tap / 3 - 1 : 0, dx = p.ksize == 3 ? tap % 3 - 1 : 0;
        const uint32_t sa = smem0 + (uint32_t)s * STAGE_BYTES;
        tma_load_4d(sa, &tmA, full, kb * TC_BK, x0 + dx, y0 + dy, b0);
        tma_load_3d(sa + TC_A_BYTES, &tmB, full, kb * TC_BK, n0, tap);
      }
    }
  } else {
    // ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2, t = threadIdx.x & 127;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int it = 0; it < total_k; ++it) {
      const int s = it % S;
      mbar_wait(smem_u32(&bar_full[s]), (uint32_t)((it / S) & 1));
      const uint32_t sa = smem0 + (uint32_t)s * STAGE_BYTES;
      const uint64_t adesc = wgmma::desc_sw128(sa + (uint32_t)wg * (64u * 128u), 16u, 1024u);
      const uint64_t bdesc = wgmma::desc_sw128(sa + TC_A_BYTES, 16u, 1024u);
      wgmma::fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k)  // 16 bf16 = 32 bytes along K inside the swizzle atom: +2 in the (addr>>4) field
        wgmma::mma<BN, 0>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((it | k) != 0));
      wgmma::commit();
      wgmma::wait<1>();  // the previous stage's MMAs have retired: release it
      if (prev >= 0 && lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&bar_empty[prev])) : "memory");
      prev = s;
    }
    wgmma::wait<0>();
    // ===== epilogue: registers -> (+bias, +residual) -> global fp32 NHWC =====
    const int ppi = p.th * p.tw;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int r = 64 * wg + wgmma::frag_row(t, i), col = n0 + wgmma::frag_col(t, i);
      const int ni = r / ppi, rem = r - ni * ppi;
      const int yy = rem / p.tw, xx = rem - yy * p.tw;
      const int b = b0 + ni;
      if (b >= p.B) continue;
      const long long pix = ((long long)b * p.H + (y0 + yy)) * p.W + (x0 + xx);
      float2 o = make_float2(acc[i], acc[i + 1]);
      if (p.bias) {
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        o.x += bv.x; o.y += bv.y;
      }
      if (p.residual) {
        const float2 rv = *reinterpret_cast<const float2*>(p.residual + pix * p.Cout + col);
        o.x += rv.x; o.y += rv.y;
      }
      *reinterpret_cast<float2*>(p.out + pix * p.Cout + col) = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  fn = (EncodeTiledFn)sym;
  return fn;
}

}  // namespace pdae

using namespace pdae;

struct pdae_conv_tc_plan {
  CUtensorMap tmA, tmB;
  ConvTcArgs args;
  int BN;
  dim3 grid;
  size_t smem;
};

static int pick_pow2_tile(int W, int cap) {
  int t = 1;
  while (t * 2 <= cap && W % (t * 2) == 0) t *= 2;
  return t;
}

extern "C" int pdae_conv_tc_create(pdae_conv_tc_plan** plan_out, const void* in_bf16, const void* w_bf16,
                                   const float* bias, const float* residual, float* out, int B, int H, int W, int Cin,
                                   int Cout, int ksize) {
  PDAE_REQUIRE(plan_out && in_bf16 && w_bf16 && out, "conv_tc_create: null pointer");
  PDAE_REQUIRE(ksize == 1 || ksize == 3, "conv_tc_create: ksize must be 1 or 3");
  PDAE_REQUIRE(Cin % TC_BK == 0 && Cout % 64 == 0, "conv_tc_create: Cin=%d Cout=%d not multiples of 64", Cin, Cout);
  PDAE_REQUIRE(((uintptr_t)in_bf16 & 15) == 0 && ((uintptr_t)w_bf16 & 15) == 0 && ((uintptr_t)out & 15) == 0,
               "conv_tc_create: pointers must be 16-byte aligned");
  EncodeTiledFn enc = get_encode_fn();
  PDAE_REQUIRE(enc != nullptr, "conv_tc_create: cuTensorMapEncodeTiled unavailable (no driver)");

  pdae_conv_tc_plan* pl = new pdae_conv_tc_plan();
  ConvTcArgs& a = pl->args;
  a.bias = bias; a.residual = residual; a.out = out;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout;
  a.tw = pick_pow2_tile(W, TC_BM);
  a.th = pick_pow2_tile(H, TC_BM / a.tw);
  a.tn = TC_BM / (a.tw * a.th);
  if (W % a.tw != 0 || H % a.th != 0 || a.tw * a.th * a.tn != TC_BM || a.tn > 256) {
    delete pl;
    PDAE_REQUIRE(false, "conv_tc_create: H=%d W=%d cannot be tiled into 128-pixel boxes", H, W);
  }
  a.tiles_x = W / a.tw; a.tiles_y = H / a.th;
  a.taps = ksize * ksize; a.ksize = ksize; a.kblocks = Cin / TC_BK;
  pl->BN = (Cout % 128 == 0) ? 128 : 64;
  const int stage_bytes = TC_A_BYTES + pl->BN * TC_BK * 2;
  a.stages = 3;
  if (a.taps * a.kblocks < a.stages) a.stages = a.taps * a.kblocks;
  pl->smem = (size_t)a.stages * stage_bytes + 1024;
  const int b_tiles = (B + a.tn - 1) / a.tn;
  pl->grid = dim3((unsigned)(a.tiles_x * a.tiles_y * b_tiles), (unsigned)(Cout / pl->BN), 1);

  {  // activations: [B][H][W][Cin] bf16, box (64 ch, tw, th, tn)
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
    cuuint32_t box[4] = {(cuuint32_t)TC_BK, (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(in_bf16), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      delete pl;
      PDAE_REQUIRE(false, "conv_tc_create: cuTensorMapEncodeTiled(A) failed with %d", (int)r);
    }
  }
  {  // weights: [taps][Cout][Cin] bf16, box (64 ch, BN couts, 1 tap)
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout, (cuuint64_t)a.taps};
    cuuint64_t strides[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cout * Cin * 2};
    cuuint32_t box[3] = {(cuuint32_t)TC_BK, (cuuint32_t)pl->BN, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w_bf16), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      delete pl;
      PDAE_REQUIRE(false, "conv_tc_create: cuTensorMapEncodeTiled(W) failed with %d", (int)r);
    }
  }
  // opt in to the largest dynamic shared-memory footprint any plan of this BN can ask for (3 stages)
  const int max_smem = 3 * stage_bytes + 1024;
  cudaError_t e = pl->BN == 128
                      ? cudaFuncSetAttribute(conv_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)
                      : cudaFuncSetAttribute(conv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
  if (e != cudaSuccess) {
    delete pl;
    set_error("conv_tc_create: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    return PDAE_ECUDA;
  }
  *plan_out = pl;
  return PDAE_OK;
}

extern "C" int pdae_conv_tc_run(const pdae_conv_tc_plan* pl, pdae_stream_t stream) {
  PDAE_REQUIRE(pl, "conv_tc_run: null plan");
  cudaStream_t s = (cudaStream_t)stream;
  if (pl->BN == 128)
    conv_tc_kernel<128><<<pl->grid, TC_THREADS, pl->smem, s>>>(pl->tmA, pl->tmB, pl->args);
  else
    conv_tc_kernel<64><<<pl->grid, TC_THREADS, pl->smem, s>>>(pl->tmA, pl->tmB, pl->args);
  PDAE_LAUNCH_CHECK("conv_tc_kernel");
  return PDAE_OK;
}

extern "C" void pdae_conv_tc_destroy(pdae_conv_tc_plan* pl) { delete pl; }
