// conv_tc v2 -- persistent, warp-specialised tensor-core implicit-GEMM convolution for sm_90a.
//
//   warp 8   : TMA producer  (4-D activation boxes with OOB zero fill = conv padding, 3-D weight boxes)
//   warps 0-7: two consumer warpgroups; warpgroup g owns rows [64 g, 64 g + 64) of every 128-pixel tile:
//              wgmma (bf16 x bf16 -> fp32 accumulators in registers) over the stage ring, then the epilogue straight
//              from the accumulator fragments: +bias (+residual fetched by TMA) -> 128B-swizzled staging tile in smem ->
//              per-channel GroupNorm partial sums (sum, sum^2) -> TMA store (fp32 or bf16 NHWC).
// One CTA per SM, contiguous tile range per CTA (consecutive tiles mostly share an image and the weight tile).  The producer
// runs ahead into the next tile while the consumers are in the epilogue.
//
// The BN=16 instantiation is the UNet image head (Cout=3 zero-padded to 16): it skips the TMA store and writes the
// first `cout_valid` columns as NCHW fp32 planes.
//
// S2 != 0: the three-by-three, stride-2, pad-1 convs of the semantic encoder (bf16 autocast training; the forward also in the
// "bf16" and "bf16x3" forward-only plans).  An NHWC tensor
// [B][H][W][C] is addressed through its PARITY VIEW, the same memory as [B][H/2][2][W/2][2C]: pixel (2 a + py, 2 b + px),
// channel c sits at the 5-D TMA coordinate (px C + c, b, py, a, image).  Each parity class is a dense stride-1 grid.
//   S2 = 1, forward: output row o reads input row 2 o + ky - 1 = parity (ky != 1) at row o - (ky == 0), so each tap is a box
//           of one parity class at the output tile shifted by -1 or 0; the only out-of-range coordinate is -1, whose TMA zero
//           fill is the padding.  The tiles cover the output grid like the tiles of a stride-1 conv over that grid, so the
//           epilogue is the ordinary one: bias, fp32 or bf16 store, optional per-channel statistics.
//   S2 = 2, data gradient as four sub-pixel phases: dX at parity (py, px) is a stride-1 correlation of dY with the taps
//           ky = 1 (py = 0) or ky = 0 at dY row + 1 and ky = 2 at dY row + 0 (py = 1), likewise kx: 1, 2, 2 or 4 taps, 9 over
//           the four phases (the forward's MMA count).  The phase is the fastest tile index, so every CTA's contiguous tile
//           range mixes the cheap and the expensive phases; each tile is stored through the parity view of dX.
//
// GM != 0: batched-GEMM modes of the attention backward (bf16 autocast training).  GM_A_MN / GM_B_MN: the A / B operand is
// MN-major, stored [K][M] / [K][N] with a row stride; each 64-wide MN block of a stage is one TMA box [64 k][64 mn] with
// SWIZZLE_128B (wgmma.cuh: the MN-major SW128 atom stack wgrad_tc also reads).  GM_SMGRAD: the softmax-gradient epilogue; the
// tile's accumulators hold dP = dO V^T for whole rows (N == BN), and the stored bf16 tile is
//   dS = alpha * P * (dP - rowsum(P * dP)),
// with P (bf16, the forward's probabilities) read for the same rows and columns, so dP never leaves the registers.  A 256-wide
// row does not fit one warpgroup's registers beside the epilogue: with GM_SPLITN the tile is 64 rows x 2 BN columns, both
// warpgroups reading the same A rows, warpgroup g computing columns [g BN, g BN + BN); the row sums meet in shared memory.
//
// GM_SPLITK: split-K for the Linear shape (H = W = 1, 1x1, M = batch), whose few output tiles would leave most SMs idle.  A
// work item is (tile, k range): item = tile * splitk + split covers k-blocks [split kchunk, split kchunk + kchunk).  Each
// item adds its partial tile into the zeroed fp32 output with red.global.add straight from the accumulator fragments
// (rows past the batch skipped), split 0 adding the bias as well.  fp32 output only: no residual, statistics or bf16 store.
//
// DET: the deterministic instantiations (pdae_conv_tc2_set_deterministic) use no float atomics.  Statistics: a tile stores
// each of its images' per-channel sums in the slot [B][tiles per image][Cout][2] of that (image, tile) (plain stores; the run
// then sums an image's slots in tile order); a tile holding several images sums each (image, column) with one thread, in row
// order.  With one tile per image the slots are [B][Cout][2] itself.  An image's sums therefore follow its own pixels only,
// never its batch or its place in a tile.  Split-K: item (tile, split) stores its partial tile in slot [split][B][Cout] and
// the run adds the splits in order, then the bias; the split count follows K and N alone.  The training GEMMs (GM_A_MN / GM_B_MN, the softmax-gradient
// epilogue) and the stride-2 data gradient record no statistics, yet their default instantiations still compile the atomic
// statistics flush; their DET instantiations are the same kernels with that code compiled out.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace pdae {

constexpr int T2_BM = 128;
constexpr int T2_BK = 64;
constexpr int T2_A_BYTES = T2_BM * T2_BK * 2;  // 16 KB
constexpr int T2_STG_BYTES = 128 * 128;        // staging tile: 128 rows x 128 B
constexpr int T2_MAX_STAGES = 8;
constexpr int T2_THREADS = 288;   // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int T2_CONSUMERS = 256;
constexpr int GM_A_MN = 1, GM_B_MN = 2, GM_SMGRAD = 4, GM_SPLITN = 8, GM_SPLITK = 16;   // conv_tc2_kernel's GM bits (kernel header)

struct ConvTc2Args {
  const float* bias;
  float* ch_stats;    // [B][Cout][2] fp32 partial (sum, sum^2) accumulators or nullptr
  float* out_nchw;    // BN==16 head: NCHW fp32 output; GM_SPLITK: the zeroed [B][Cout] fp32 output the partial tiles are added to
  const long long* fuse;  // BN==16 head: optional device-side descriptor of the fused DDIM update (see pdae_conv_tc2_set_head_fuse)
  int B, H, W, Cout;
  int tw, th, tn;
  int tiles_x, tiles_y, tiles_b, tiles_m, tiles_total;
  int taps, ksize, kblocks;
  int stages;
  int has_res, out_bf16, cout_valid;
  int w_batched;  // B operand is a per-image matrix (batched GEMM): 3rd TMA coordinate = image index
  int kblocks2;   // fused 1x1 skip conv: extra K blocks from a second (activation, weight) pair, accumulated into the same tile
  int kblocks2a;  // ... of which the first kblocks2a come from tmA2, the rest from tmA3 (virtual channel concat of two tensors)
  int w_stat;     // weights stationary: every B tile of the (single) n-tile is loaded ONCE per CTA into its own shared-memory
                  // region and reused by all of the CTA's tiles; pipeline stages then hold A tiles only
  float softmax_alpha;  // > 0: the epilogue stores softmax_row(alpha * acc) (bf16) instead of acc -- attention scores whose
                        // whole row lives in this tile's accumulators (N == BN); model/module.py:452-455,483-486
  int splitk, kchunk;   // GM_SPLITK: k ranges per tile, k-blocks per range
};
// GM_SMGRAD operands (a kernel parameter of its own: ConvTc2Args keeps its size, so the other modes compile as before)
struct SmGradArgs {
  const __nv_bfloat16* p;  // the probabilities P, indexed like the output: row stride ld, batch stride bs
  long long ld, bs;
  float alpha;             // the score scale folded into dS
};

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
__device__ __forceinline__ void tma_ld5(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_st5(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(m), "r"(src),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
// stride-2 data gradient: number of taps of sub-pixel phase (py, px) = ph (py = ph >> 1, px = ph & 1)
__device__ __forceinline__ int s2_phase_taps(int ph) { return (1 + (ph >> 1)) * (1 + (ph & 1)); }
// One elected lane of a fully converged warp: the producer / issuer loops run on all 32 lanes (warp-uniform operands stay in
// uniform registers); only the TMA instruction is predicated.  Under `if (lane == 0)` every descriptor was a
// per-lane value and each MMA paid an ELECT + 5 x R2UR.BROADCAST + branch waterfall.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// barrier of the 256 consumer threads (the producer warp never joins it)
__device__ __forceinline__ void cons_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// byte offset of (row, 16-byte chunk) inside a 128-row x 128-byte SWIZZLE_128B staging tile
__device__ __forceinline__ uint32_t swz(int row, int chunk16) { return (uint32_t)(row * 128 + ((chunk16 ^ (row & 7)) << 4)); }

template <int BN, bool OB, int S2 = 0, int GM = 0, bool DET = false>
__global__ void __launch_bounds__(T2_THREADS, 1)
conv_tc2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR,
                const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                const __grid_constant__ CUtensorMap tmA3, ConvTc2Args p, SmGradArgs sg) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[T2_MAX_STAGES], bar_empty[T2_MAX_STAGES];
  __shared__ __align__(8) uint64_t bar_res, bar_w;
  __shared__ float st_acc[2][BN < 32 ? 32 : BN];  // [sum | sum^2][channel] of the current (image, n-tile)
  __shared__ float st_part[2][8][32];              // per-chunk partial sums [sum | sum^2][row run][column] (CW * 8 runs / 32)

  constexpr bool SPN = (GM & GM_SPLITN) != 0;   // 64-row tiles, the B tile holds 2 BN rows (one BN-row half per warpgroup)
  constexpr bool SK = (GM & GM_SPLITK) != 0;    // work item = (tile, k range); partial tiles reduced into the output
  constexpr int B_BYTES = (SPN ? 2 : 1) * BN * T2_BK * 2;
  constexpr int STAGE_BYTES = T2_A_BYTES + ((B_BYTES + 1023) / 1024) * 1024;
  constexpr int CW = OB ? 64 : 32;             // accumulator columns per staging tile (128-byte rows)
  constexpr int NCH = BN < CW ? 1 : BN / CW;
  constexpr int RPT = CW / 2;                  // statistics: rows per thread (256 threads = CW columns x 128 / RPT row runs)
  const uint32_t smem0 = (s_u32(smem_raw) + 1023u) & ~1023u;
  const int S = p.stages;
  const uint32_t stage_stride = p.w_stat ? (uint32_t)T2_A_BYTES : (uint32_t)STAGE_BYTES;
  const uint32_t wbase = smem0 + (uint32_t)S * stage_stride;                       // stationary weights (w_stat only)
  const uint32_t stg_out = wbase + (p.w_stat ? (uint32_t)((p.taps * p.kblocks + p.kblocks2) * B_BYTES) : 0u);   // 16 KB output staging
  const uint32_t stg_res = stg_out + (uint32_t)T2_STG_BYTES;   // 16 KB residual staging (only if has_res)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_k = p.taps * p.kblocks;          // main conv
  const int total_all = total_k + p.kblocks2;      // + fused 1x1 skip conv
  // contiguous tile range per CTA: consecutive tiles of a CTA mostly belong to the same image, so the per-channel
  // GroupNorm partial sums can be accumulated in shared memory across tiles and flushed once per image
  const int per_cta = (p.tiles_total + (int)gridDim.x - 1) / (int)gridDim.x;
  const int tile_begin = (int)blockIdx.x * per_cta;
  const int tile_end = min(p.tiles_total, tile_begin + per_cta);

  for (int j = threadIdx.x; j < (BN < 32 ? 32 : BN); j += T2_THREADS) {
    st_acc[0][j] = 0.f;
    st_acc[1][j] = 0.f;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mb_init(s_u32(&bar_full[s]), 1);
      mb_init(s_u32(&bar_empty[s]), 8);   // one arrive per consumer warp
    }
    mb_init(s_u32(&bar_res), 1);
    mb_init(s_u32(&bar_w), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ================= TMA producer (warp-uniform loop, elected lane issues) =================
    int s = 0;
    uint32_t ph = 0;
    const bool ws = p.w_stat != 0;
    const uint32_t stage_tx = ws ? (uint32_t)T2_A_BYTES : (uint32_t)((SPN ? T2_A_BYTES / 2 : T2_A_BYTES) + B_BYTES);
    if (ws && tile_begin < tile_end) {   // all B tiles of the layer, once (single n-tile: n0 = 0)
      const uint32_t wb = s_u32(&bar_w);
      if (elect_one()) {
        mb_expect_tx(wb, (uint32_t)(total_all * B_BYTES));
        for (int it = 0; it < total_k; ++it)
          tma_ld3(wbase + (uint32_t)(it * B_BYTES), &tmB, wb, (it % p.kblocks) * T2_BK, 0, it / p.kblocks);
        for (int kb2 = 0; kb2 < p.kblocks2; ++kb2)
          tma_ld3(wbase + (uint32_t)((total_k + kb2) * B_BYTES), &tmB2, wb, kb2 * T2_BK, 0, 0);
      }
      __syncwarp();
    }
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      const int ph2 = S2 == 2 ? (tile & 3) : 0;      // stride-2 dgrad: sub-pixel phase of this tile
      const int tl = S2 == 2 ? (tile >> 2) : (SK ? tile / p.splitk : tile);
      const int kb0 = SK ? (tile - tl * p.splitk) * p.kchunk : 0;   // split-K: first k-block of this item
      const int nt = tl / p.tiles_m;
      int mt = tl - nt * p.tiles_m;
      const int tx = mt % p.tiles_x;
      mt /= p.tiles_x;
      const int ty = mt % p.tiles_y;
      const int bt = mt / p.tiles_y;
      const int x0 = tx * p.tw, y0 = ty * p.th, b0 = bt * p.tn, n0 = nt * BN;
      if constexpr (S2 != 0) {
        const int cin = p.kblocks * T2_BK;
        const int nx = 1 + (ph2 & 1);
        const int n_it = (S2 == 1 ? 9 : s2_phase_taps(ph2)) * p.kblocks;
        for (int it = 0; it < n_it; ++it) {
          const int j = it / p.kblocks, kb = it - j * p.kblocks;
          mb_wait(s_u32(&bar_empty[s]), ph ^ 1u);
          const uint32_t full = s_u32(&bar_full[s]);
          const uint32_t sa = smem0 + (uint32_t)s * stage_stride;
          if (elect_one()) {
            mb_expect_tx(full, stage_tx);
            int wtap;
            if (S2 == 1) {           // forward tap j = (ky, kx): parity (ky != 1, kx != 1) at the output tile - (k == 0)
              const int ky = j / 3, kx = j - 3 * ky;
              wtap = j;
              tma_ld5(sa, &tmA, full, (kx != 1) * cin + kb * T2_BK, x0 - (kx == 0), ky != 1, y0 - (ky == 0), b0);
            } else {                 // dgrad phase (py, px), tap j: ky = 1 (py = 0) or 0 / 2 at dY row + 1 / + 0 (py = 1)
              const int jy = j / nx, jx = j - jy * nx;
              const int ky = (ph2 >> 1) ? 2 * jy : 1, kx = (ph2 & 1) ? 2 * jx : 1;
              wtap = 3 * ky + kx;
              tma_ld4(sa, &tmA, full, kb * T2_BK, x0 + (kx == 0), y0 + (ky == 0), b0);
            }
            if (!ws) tma_ld3(sa + T2_A_BYTES, &tmB, full, kb * T2_BK, n0, wtap);
          }
          __syncwarp();
          if (++s == S) { s = 0; ph ^= 1u; }
        }
        continue;
      }
      int tap = 0, kb = kb0, dy = p.ksize == 3 ? -1 : 0, dx = dy;
      const int n_main = SK ? min(p.kchunk, p.kblocks - kb0) : total_k;
      for (int it = 0; it < n_main; ++it) {
        mb_wait(s_u32(&bar_empty[s]), ph ^ 1u);
        const uint32_t full = s_u32(&bar_full[s]);
        const uint32_t sa = smem0 + (uint32_t)s * stage_stride;
        if (elect_one()) {
          mb_expect_tx(full, stage_tx);
          if constexpr ((GM & GM_A_MN) != 0) {        // [K][M] operand: one [64 k][64 m] box per consumer warpgroup
            tma_ld3(sa, &tmA, full, x0, kb * T2_BK, b0);
            tma_ld3(sa + wgmma::MN_BOX, &tmA, full, x0 + 64, kb * T2_BK, b0);
          } else {
            tma_ld4(sa, &tmA, full, kb * T2_BK, x0 + dx, y0 + dy, b0);
          }
          if constexpr ((GM & GM_B_MN) != 0) {        // [K][N] operand: BN / 64 boxes [64 k][64 n]
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_ld3(sa + T2_A_BYTES + (uint32_t)j * wgmma::MN_BOX, &tmB, full, n0 + 64 * j, kb * T2_BK, b0);
          } else if constexpr (SPN) {                 // both BN-row halves of the 2 BN-wide tile
            tma_ld3(sa + T2_A_BYTES, &tmB, full, kb * T2_BK, n0, b0);
            tma_ld3(sa + T2_A_BYTES + BN * T2_BK * 2, &tmB, full, kb * T2_BK, n0 + BN, b0);
          } else {
            if (!ws) tma_ld3(sa + T2_A_BYTES, &tmB, full, kb * T2_BK, n0, p.w_batched ? b0 : tap);
          }
        }
        __syncwarp();
        if (++kb == p.kblocks) {
          kb = 0;
          ++tap;
          if (p.ksize == 3 && ++dx == 2) { dx = -1; ++dy; }
        }
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      for (int kb2 = 0; kb2 < p.kblocks2; ++kb2) {   // fused 1x1 skip conv: un-normalised input, centre tap
        mb_wait(s_u32(&bar_empty[s]), ph ^ 1u);
        const uint32_t full = s_u32(&bar_full[s]);
        const uint32_t sa = smem0 + (uint32_t)s * stage_stride;
        if (elect_one()) {
          mb_expect_tx(full, stage_tx);
          if (kb2 < p.kblocks2a) tma_ld4(sa, &tmA2, full, kb2 * T2_BK, x0, y0, b0);
          else tma_ld4(sa, &tmA3, full, (kb2 - p.kblocks2a) * T2_BK, x0, y0, b0);
          if (!ws) tma_ld3(sa + T2_A_BYTES, &tmB2, full, kb2 * T2_BK, n0, 0);
        }
        __syncwarp();
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    // ================= consumers: warpgroup wg computes rows [64 wg, 64 wg + 64) of each tile, then both run the epilogue ==========
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;           // thread inside the warpgroup (accumulator fragment owner)
    const int ct = threadIdx.x;                // 0..255 over both warpgroups
    const bool elected = ct == 0;
    const int ppi = p.th * p.tw;               // pixels per image inside a tile
    int rc = 0;                                // residual loads consumed (mbarrier phase)
    int s = 0;
    uint32_t ph = 0;
    const uint32_t obuf = stg_out, rbuf = stg_res;
    const uint32_t rbar = s_u32(&bar_res);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if (p.w_stat && tile_begin < tile_end) mb_wait(s_u32(&bar_w), 0u);   // stationary weights have landed
    for (int tile = tile_begin; tile < tile_end; ++tile) {
      const int ph2 = S2 == 2 ? (tile & 3) : 0;
      const int tl = S2 == 2 ? (tile >> 2) : (SK ? tile / p.splitk : tile);
      const int kb0 = SK ? (tile - tl * p.splitk) * p.kchunk : 0;
      const int nt = tl / p.tiles_m;
      int mt = tl - nt * p.tiles_m;
      const int tx = mt % p.tiles_x;
      mt /= p.tiles_x;
      const int ty = mt % p.tiles_y;
      const int bt = mt / p.tiles_y;
      const int x0 = tx * p.tw, y0 = ty * p.th, b0 = bt * p.tn, n0 = nt * BN;
      const int n_it = S2 == 2 ? s2_phase_taps(ph2) * p.kblocks : (SK ? min(p.kchunk, p.kblocks - kb0) : total_all);
      if constexpr (BN != 16) {
        if (p.has_res && elected) {            // residual chunk 0 of this tile (lands while the main loop runs)
          mb_expect_tx(rbar, T2_STG_BYTES);
          tma_ld4(rbuf, &tmR, rbar, n0, x0, y0, b0);
        }
      }
      // ---- main loop: wgmma over the stage ring; a stage is released once the MMAs reading it have retired ----
      int prev = -1;
      for (int it = 0; it < n_it; ++it) {
        mb_wait(s_u32(&bar_full[s]), ph);
        const uint32_t sa = smem0 + (uint32_t)s * stage_stride;
        if constexpr ((GM & ~GM_SPLITK) == 0) {
          const uint64_t ad = wgmma::desc_sw128(sa + (uint32_t)wg * (64u * 128u), 16u, 1024u);
          const uint64_t bd = wgmma::desc_sw128(p.w_stat ? wbase + (uint32_t)(it * B_BYTES) : sa + T2_A_BYTES, 16u, 1024u);
          wgmma::fence();
#pragma unroll
          for (int k = 0; k < T2_BK / 16; ++k)
            wgmma::mma<BN, 0>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (uint32_t)((it | k) != 0));
        } else {
          constexpr int TA = (GM & GM_A_MN) ? 1 : 0, TB = (GM & GM_B_MN) ? 1 : 0;
          constexpr uint64_t SA = TA ? wgmma::K16_STEP_MNMAJOR : wgmma::K16_STEP_KMAJOR;
          constexpr uint64_t SB = TB ? wgmma::K16_STEP_MNMAJOR : wgmma::K16_STEP_KMAJOR;
          const uint32_t a_s = SPN ? sa : sa + (uint32_t)wg * wgmma::MN_BOX;
          const uint32_t b_s = sa + T2_A_BYTES + (SPN ? (uint32_t)(wg * BN * T2_BK * 2) : 0u);
          const uint64_t ad = TA ? wgmma::desc_mnmajor(a_s) : wgmma::desc_kmajor(a_s);
          const uint64_t bd = TB ? wgmma::desc_mnmajor(b_s) : wgmma::desc_kmajor(b_s);
          wgmma::fence();
#pragma unroll
          for (int k = 0; k < T2_BK / 16; ++k)
            wgmma::mma<BN, TA, TB>(acc, ad + (uint64_t)k * SA, bd + (uint64_t)k * SB, (uint32_t)((it | k) != 0));
        }
        wgmma::commit();
        wgmma::wait<1>();
        if (prev >= 0 && lane == 0) mb_arrive(s_u32(&bar_empty[prev]));
        prev = s;
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      wgmma::wait<0>();
      if (prev >= 0 && lane == 0) mb_arrive(s_u32(&bar_empty[prev]));

      if constexpr (SK) {
        // split-K partial tile (H = W = 1: tile row r is batch row b0 + r): fp32 reductions into the zeroed output
        if constexpr (DET) {
          float* slot = p.out_nchw + (long long)(kb0 / p.kchunk) * p.B * p.Cout;
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2) {
            const int b = b0 + 64 * wg + wgmma::frag_row(t, i), col = n0 + wgmma::frag_col(t, i);
            if (b < p.B) *reinterpret_cast<float2*>(slot + (long long)b * p.Cout + col) = make_float2(acc[i], acc[i + 1]);
          }
          continue;
        }
        const bool add_bias = p.bias != nullptr && kb0 == 0;
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
          const int b = b0 + 64 * wg + wgmma::frag_row(t, i), col = n0 + wgmma::frag_col(t, i);
          float v0 = acc[i], v1 = acc[i + 1];
          if (add_bias) {
            const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
            v0 += bv.x; v1 += bv.y;
          }
          if (b < p.B)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p.out_nchw + (long long)b * p.Cout + col), "f"(v0), "f"(v1)
                         : "memory");
        }
        continue;
      }
      if constexpr (BN == 16) {
        // ---- image head: first cout_valid columns -> NCHW fp32 planes ----
        const long long hw = (long long)p.H * p.W;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) {
          const int r = 64 * wg + wgmma::frag_row(t, i), j = wgmma::frag_col(t, i);
          const int ni = r / ppi, rem = r - ni * ppi;
          const int yy = rem / p.tw, xx = rem - yy * p.tw;
          const int b = b0 + ni;
          if (b >= p.B) continue;
          const long long pix = (long long)(y0 + yy) * p.W + (x0 + xx);
          const float val = acc[i] + (p.bias ? __ldg(p.bias + j) : 0.f);
          if (j < p.cout_valid) p.out_nchw[((long long)b * p.cout_valid + j) * hw + pix] = val;
          // ---- fused DDIM update (diffusion/ddim.py:43-55, 66-79, 91-107, 123-138): this head's output is the last tensor the
          // step needs, so x_t -> x_{t-1} (or x_{t+1}) is finished here, in place, with the exact arithmetic of ddim_step_kernel.
          // The descriptor lives in device memory and is (re)written by the sampling loop; flags == 0 -> plain head conv.
          if (p.fuse) {
            const long long flags = __ldg(p.fuse);
            const int C = (int)((flags >> 8) & 0xff), Ce = (int)((flags >> 16) & 0xff);
            if ((flags & 1) && j < C) {
              const float* eps = reinterpret_cast<const float*>(__ldg(p.fuse + 1));
              float* xt = reinterpret_cast<float*>(__ldg(p.fuse + 2));
              const long long tb = reinterpret_cast<const long long*>(__ldg(p.fuse + 3))[b];
              const long long xi = ((long long)b * C + j) * hw + pix;
              if (flags & 8) {
                // DDPM ancestral step (gaussian_diffusion.py:112-126), the arithmetic of noise_p_sample_kernel; the grad head adds
                // the shift term first as the reference does (eps + shift_coef[t] * grad, one rounding each).
                const float* tab = reinterpret_cast<const float*>(__ldg(p.fuse + 4));
                float e = val;
                if (flags & 2) e = __fadd_rn(eps[((long long)b * Ce + j) * hw + pix],
                                             __fmul_rn(reinterpret_cast<const float*>(__ldg(p.fuse + 6))[tb], val));
                const float mean = __fsub_rn(__fmul_rn(tab[tb], xt[xi]),
                                             __fmul_rn(reinterpret_cast<const float*>(__ldg(p.fuse + 5))[tb], e));
                const float lv = reinterpret_cast<const float*>(__ldg(p.fuse + 7))[tb];
                const float mask = tb == 0 ? 0.0f : 1.0f;
                const float nz = reinterpret_cast<const float*>(__ldg(p.fuse + 8))[xi];
                xt[xi] = __fadd_rn(mean, __fmul_rn(__fmul_rn(mask, expf(__fmul_rn(0.5f, lv))), nz));
              } else {
                const float A = reinterpret_cast<const float*>(__ldg(p.fuse + 4))[tb];
                const float Bm = reinterpret_cast<const float*>(__ldg(p.fuse + 5))[tb];
                const float abar = reinterpret_cast<const float*>(__ldg(p.fuse + 7))[tb];
                const float s1m = (flags & 2) ? reinterpret_cast<const float*>(__ldg(p.fuse + 6))[tb] : 0.f;
                float g = val;
                if (flags & 16) {
                  // trajectory interpolation (ddim.py:149-174): this is the second shift head; the first one wrote g1.  The
                  // blend is (1 - alpha) * g1 + alpha * g2 as torch evaluates it in fp32: a1 = fp32(1 - alpha), a2 = fp32(alpha).
                  const unsigned long long ab = (unsigned long long)__ldg(p.fuse + 9);
                  const float a1 = __uint_as_float((unsigned)ab), a2 = __uint_as_float((unsigned)(ab >> 32));
                  g = __fadd_rn(__fmul_rn(a1, reinterpret_cast<const float*>(__ldg(p.fuse + 8))[xi]), __fmul_rn(a2, val));
                }
                float e = val;                                  // this head predicts epsilon itself
                if (flags & 2) e = __fsub_rn(eps[((long long)b * Ce + j) * hw + pix], __fmul_rn(s1m, g));   // own output = shift term
                else if (flags & 4) e = eps[((long long)b * Ce + j) * hw + pix];   // shift unused this step: epsilon from the other head
                const float ax = __fmul_rn(A, xt[xi]);
                float x0v = __fsub_rn(ax, __fmul_rn(Bm, e));
                x0v = fminf(fmaxf(x0v, -1.0f), 1.0f);
                const float e2 = __fdiv_rn(__fsub_rn(ax, x0v), Bm);
                xt[xi] = __fadd_rn(__fmul_rn(x0v, sqrtf(abar)), __fmul_rn(sqrtf(__fsub_rn(1.0f, abar)), e2));
              }
            }
          }
        }
      } else {
        // softmax-gradient epilogue (GM_SMGRAD): the thread's two rows (i / 2 % 2) are spread over the 4 lanes of a quad; P is
        // read for exactly the (row, column pair)s its fragments hold.  rowsum(P dP) first, then dS chunk by chunk below.
        constexpr bool SMG = (GM & GM_SMGRAD) != 0;
        const __nv_bfloat16* sg_row =
            SMG ? sg.p + (long long)b0 * sg.bs + (long long)(x0 + (SPN ? 0 : 64 * wg) + wgmma::frag_row(t, 0)) * sg.ld +
                      (SPN ? wg * BN : 0)
                : nullptr;
        auto ld_p = [&](int i) -> uint32_t {     // P at the columns of fragment registers i, i + 1
          return __ldg(reinterpret_cast<const unsigned int*>(sg_row + ((i >> 1) & 1) * 8 * sg.ld + wgmma::frag_col(t, i)));
        };
        float rs[2] = {0.f, 0.f};
        if constexpr (SMG) {
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            // (the empty asm keeps each chunk's loads behind the previous chunk's: the accumulators of a 256-wide row leave
            //  room for one chunk of P words, not for all of them)
            asm volatile("" ::: "memory");
#pragma unroll
            for (int i = c * (CW / 2); i < (c + 1) * (CW / 2); i += 2) {
              const uint32_t w = ld_p(i);
              rs[(i >> 1) & 1] = fmaf(__uint_as_float(w << 16), acc[i],
                                      fmaf(__uint_as_float(w & 0xffff0000u), acc[i + 1], rs[(i >> 1) & 1]));
            }
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 1);
            rs[h] += __shfl_xor_sync(0xffffffffu, rs[h], 2);
          }
          if constexpr (SPN) {
            // the other half of each row is in the other warpgroup: [warpgroup][row] partial sums, added in the same order by
            // both.  (The next tile writes them again only after the chunk loop's barriers, which follow these reads.)
            float* xs = &st_part[0][0][0];
            const int fr = wgmma::frag_row(t, 0);
            if ((t & 3) == 0) {
              xs[64 * wg + fr] = rs[0];
              xs[64 * wg + fr + 8] = rs[1];
            }
            cons_bar();
            rs[0] = xs[fr] + xs[64 + fr];
            rs[1] = xs[fr + 8] + xs[64 + fr + 8];
          }
        }
        if (GM == 0 && p.softmax_alpha > 0.f) {
          // softmax epilogue: the thread's two rows (i / 2 % 2) are spread over the 4 lanes of a quad
          const float sm_a = p.softmax_alpha * 1.4426950408889634f;
          float mx[2] = {-3.0e38f, -3.0e38f}, sum[2] = {0.f, 0.f};
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], acc[i]);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
          }
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) sum[(i >> 1) & 1] += exp2f((acc[i] - mx[(i >> 1) & 1]) * sm_a);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
            sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
            sum[h] = 1.0f / sum[h];
          }
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = exp2f((acc[i] - mx[(i >> 1) & 1]) * sm_a) * sum[(i >> 1) & 1];
        }
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          // this chunk's fragment registers: i in [c CW/2, (c+1) CW/2), column inside the chunk = frag_col - c CW
          float v[CW / 2];
#pragma unroll
          for (int q = 0; q < CW / 2; ++q) v[q] = acc[c * (CW / 2) + q];
          if constexpr (SMG) {                  // dS = alpha P (dP - rowsum(P dP))
#pragma unroll
            for (int q = 0; q < CW / 2; q += 2) {
              const uint32_t w = ld_p(c * (CW / 2) + q);
              const float r = rs[(q >> 1) & 1];
              v[q] = sg.alpha * __uint_as_float(w << 16) * (v[q] - r);
              v[q + 1] = sg.alpha * __uint_as_float(w & 0xffff0000u) * (v[q + 1] - r);
            }
          }
          if (p.bias) {
#pragma unroll
            for (int q = 0; q < CW / 2; q += 2) {
              const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + c * CW + wgmma::frag_col(t, q)));
              v[q] += bv.x; v[q + 1] += bv.y;
            }
          }
          if (p.has_res) {                      // the residual has the output's dtype: CW columns = one 128-byte row
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
          // the staging buffer must no longer be read by the previous TMA store
          if (elected) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          cons_bar();                           // (also: every thread has consumed the residual buffer)
          if (p.has_res && elected && c + 1 < NCH) {   // residual for the next chunk overlaps this chunk's store + statistics
            mb_expect_tx(rbar, T2_STG_BYTES);
            tma_ld4(rbuf, &tmR, rbar, n0 + (c + 1) * CW, x0, y0, b0);
          }
#pragma unroll
          for (int q = 0; q < CW / 2; q += 2) {
            const int r = 64 * wg + wgmma::frag_row(t, q), cl = wgmma::frag_col(t, q);
            if (OB) {
              __nv_bfloat162 b2 = __floats2bfloat162_rn(v[q], v[q + 1]);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(obuf + swz(r, cl >> 3) + (uint32_t)((cl & 7) * 2)),
                           "r"(*reinterpret_cast<uint32_t*>(&b2))
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
            if constexpr (S2 == 2) tma_st5(&tmO, obuf, (ph2 & 1) * p.Cout + n0 + c * CW, x0, ph2 >> 1, y0, b0);   // dX parity view
            else if constexpr (SPN) {       // staging rows [64 g, 64 g + 64) = warpgroup g's columns of the tile's 64 rows
              tma_st4(&tmO, obuf, n0 + c * CW, x0, y0, b0);
              tma_st4(&tmO, obuf + 64u * 128u, n0 + BN + c * CW, x0, y0, b0);
            } else tma_st4(&tmO, obuf, n0 + c * CW, x0, y0, b0);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          }
          if (p.ch_stats) {
            // per-channel partial sums over this tile's rows, read back from the staged (rounded) values:
            // thread -> column (ct % CW), rows [(ct / CW) * RPT, +RPT)
            const int col = ct % CW, r0 = (ct / CW) * RPT;
            const uint32_t cbyte = OB ? (uint32_t)((col & 7) * 2) : (uint32_t)((col & 3) * 4);
            const int cchunk = OB ? (col >> 3) : (col >> 2);
            auto ldv = [&](int rr) -> float {
              float x;
              if (OB) {
                unsigned short h;
                asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(obuf + swz(rr, cchunk) + cbyte));
                x = __uint_as_float(((uint32_t)h) << 16);
              } else {
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(obuf + swz(rr, cchunk) + cbyte));
              }
              return x;
            };
            if (DET && p.tn != 1) {
              // several images per tile: (image, column) pairs, each summed over the image's rows in order by one thread.  When
              // an image spans several tiles (a grid that is not a power of two, e.g. 6x6 in 2x2 boxes) each tile has its slot.
              const int tpi = p.tiles_x * p.tiles_y, pimg = ty * p.tiles_x + tx;
              for (int pr = ct; pr < p.tn * CW; pr += T2_CONSUMERS) {
                const int img = pr / CW, cc = pr - img * CW;
                if (b0 + img >= p.B) continue;
                const uint32_t cb = OB ? (uint32_t)((cc & 7) * 2) : (uint32_t)((cc & 3) * 4);
                const int ck = OB ? (cc >> 3) : (cc >> 2);
                float sacc = 0.f, qq = 0.f;
                for (int rr = img * ppi; rr < (img + 1) * ppi; ++rr) {
                  float x;
                  if (OB) {
                    unsigned short h;
                    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(obuf + swz(rr, ck) + cb));
                    x = __uint_as_float(((uint32_t)h) << 16);
                  } else {
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(obuf + swz(rr, ck) + cb));
                  }
                  sacc += x;
                  qq = fmaf(x, x, qq);
                }
                *reinterpret_cast<float2*>(p.ch_stats + (((long long)(b0 + img) * tpi + pimg) * p.Cout + n0 + c * CW + cc) * 2) =
                    make_float2(sacc, qq);
              }
            } else if (p.tn == 1) {
              // whole tile = one image: accumulate in shared memory across this CTA's consecutive tiles.  The row runs of a
              // column are added in a fixed order by one thread, so repeated runs give identical statistics.
              float sacc = 0.f, qq = 0.f;
#pragma unroll 8
              for (int rr = r0; rr < r0 + RPT; ++rr) {
                const float x = ldv(rr);
                sacc += x;
                qq = fmaf(x, x, qq);
              }
              float* part = &st_part[0][0][0];
              part[ct] = sacc;
              part[256 + ct] = qq;
              cons_bar();
              if (ct < CW) {
                float s2 = 0.f, q2 = 0.f;
#pragma unroll
                for (int g = 0; g < 256 / CW; ++g) {
                  s2 += part[g * CW + ct];
                  q2 += part[256 + g * CW + ct];
                }
                if constexpr (DET) {   // this tile's slot
                  const int pimg = (tl - nt * p.tiles_m) % (p.tiles_x * p.tiles_y);
                  *reinterpret_cast<float2*>(
                      p.ch_stats + (((long long)b0 * p.tiles_x * p.tiles_y + pimg) * p.Cout + n0 + c * CW + ct) * 2) =
                      make_float2(s2, q2);
                } else {
                  st_acc[0][c * CW + ct] += s2;
                  st_acc[1][c * CW + ct] += q2;
                }
              }
            } else if (ppi % RPT == 0) {
              // several whole images per tile and this thread's RPT rows lie inside ONE image
              float sacc = 0.f, qq = 0.f;
#pragma unroll 8
              for (int rr = r0; rr < r0 + RPT; ++rr) {
                const float x = ldv(rr);
                sacc += x;
                qq = fmaf(x, x, qq);
              }
              const int cur = r0 / ppi;
              if (b0 + cur < p.B) {
                float* dst = p.ch_stats + ((long long)(b0 + cur) * p.Cout + n0 + c * CW + col) * 2;
                if (ppi == RPT && p.tiles_x * p.tiles_y == 1) {  // whole image inside this tile and this thread covers all of
                                                                 // its rows: the only contributor -> plain store, no atomic
                  *reinterpret_cast<float2*>(dst) = make_float2(sacc, qq);
                } else {
                  atomicAdd(dst, sacc);
                  atomicAdd(dst + 1, qq);
                }
              }
            } else {
              float sacc = 0.f, qq = 0.f;
              int cur = r0 / ppi, nxt = (cur + 1) * ppi;  // `nxt` = first row of the next image
              float* dst0 = p.ch_stats + ((long long)b0 * p.Cout + n0 + c * CW + col) * 2;
              for (int rr = r0; rr < r0 + RPT; ++rr) {
                if (rr == nxt) {
                  if (b0 + cur < p.B) {
                    atomicAdd(dst0 + (long long)cur * p.Cout * 2, sacc);
                    atomicAdd(dst0 + (long long)cur * p.Cout * 2 + 1, qq);
                  }
                  sacc = qq = 0.f;
                  ++cur;
                  nxt += ppi;
                }
                const float x = ldv(rr);
                sacc += x;
                qq = fmaf(x, x, qq);
              }
              if (b0 + cur < p.B) {
                atomicAdd(dst0 + (long long)cur * p.Cout * 2, sacc);
                atomicAdd(dst0 + (long long)cur * p.Cout * 2 + 1, qq);
              }
            }
          }
        }
        if (!DET && p.ch_stats && p.tn == 1) {
          bool flush = tile + 1 >= tile_end;
          if (!flush) {
            const int nt2 = (tile + 1) / p.tiles_m;
            const int bt2 = ((tile + 1) - nt2 * p.tiles_m) / (p.tiles_x * p.tiles_y);
            flush = nt2 != nt || bt2 != bt;
          }
          if (flush) {
            cons_bar();   // every thread's shared-memory atomics are done before these reads
            for (int j = ct; j < BN; j += T2_CONSUMERS) {
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
    }
    if (elected) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

typedef CUresult (*EncodeTiledFn2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn2 encode_fn2() {
  static EncodeTiledFn2 fn = nullptr;
  if (fn) return fn;
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    return nullptr;
  }
  fn = (EncodeTiledFn2)sym;
  return fn;
}

static int pow2_tile(int W, int cap) {
  int t = 1;
  while (t * 2 <= cap && W % (t * 2) == 0) t *= 2;
  return t;
}

template <int BN, bool OB, int S2 = 0, int GM = 0, bool DET = false>
static cudaError_t launch_tc2(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& o, const CUtensorMap& r,
                              const CUtensorMap& a2, const CUtensorMap& b2, const CUtensorMap& a3, const ConvTc2Args& args,
                              const SmGradArgs& sg, int grid, size_t smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc2_kernel<BN, OB, S2, GM, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, 221 * 1024);  // + static (barriers, stats <= 2 KB) <= 227 KB
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  conv_tc2_kernel<BN, OB, S2, GM, DET><<<grid, T2_THREADS, smem, s>>>(a, b, o, r, a2, b2, a3, args, sg);
  return cudaPeekAtLastError();
}

// deterministic split-K: out[b][n] = (sum over the splits in order of part[split][b][n]) + bias[n]
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, int splitk, long long n, int Cout,
                                                            const float* __restrict__ bias, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = part[i];
  for (int k = 1; k < splitk; ++k) a += part[(long long)k * n + i];
  if (bias) a += bias[i % Cout];
  out[i] = a;
}

}  // namespace pdae

using namespace pdae;

struct pdae_conv_tc2_plan {
  CUtensorMap tmA, tmB, tmO, tmR, tmA2, tmB2, tmA3;
  ConvTc2Args args;
  SmGradArgs sg;
  int BN, grid;
  int s2;           // 0: stride-1 conv / GEMM; 1: stride-2 forward; 2: stride-2 data gradient (conv_tc2_kernel's S2)
  int gm;           // batched-GEMM operand / epilogue mode (conv_tc2_kernel's GM)
  size_t smem;
  int det;          // pdae_conv_tc2_set_deterministic: the DET kernel
  float* det_out;   // DET: where the run reduces the slots to (the [B][Cout][2] statistics or the split-K output), or nullptr
};

static int g_num_sms = 0;

struct Tc2Desc {
  const void* in; const void* w; const float* bias; const void* residual; void* out;
  int out_dtype; float* ch_stats;
  int B, H, W, Cin, Cout, ksize, cout_valid, bn_override;
  long long in_ld;            // elements between consecutive pixels of the A operand
  long long in_bs;            // elements between consecutive images of the A operand
  int w_batched;              // 0: weights [taps][Cout][Cin] ; 1: per-image matrix [B][Cout rows][Cin], strides below
  long long w_ld, w_bs;
  long long out_ld, out_bs;   // elements between consecutive pixels / images of the output
  const void* in2 = nullptr; const void* w2 = nullptr; int Cin2 = 0;   // fused 1x1 skip conv (bf16 NHWC input, [Cout][Cin2] weights)
  float softmax_alpha = 0.f;  // batched GEMM only: store softmax_row(alpha * out) as bf16 (needs N == BN)
  const void* in3 = nullptr; int Cin2a = 0;   // skip input = channel concat of in2 [..,Cin2a] and in3 [..,Cin2-Cin2a] (in3 == nullptr: in2 alone)
  int s2 = 0;   // stride-2 3x3 conv (kernel header): H, W are the OUTPUT / dY grid; 1: `in` is read through its parity view;
                // 2: data gradient, `out` (fp32 dX) is written through its parity view
  int gm = 0;   // batched GEMM only: GM_A_MN / GM_B_MN operands ([K][M] / [K][N], in_ld / w_ld between k rows), GM_SMGRAD epilogue
  const void* sg_p = nullptr; long long sg_ld = 0, sg_bs = 0; float sg_alpha = 0.f;   // GM_SMGRAD: P and alpha
};

static int tc2_create(pdae_conv_tc2_plan** plan_out, const Tc2Desc& d) {
  const int B = d.B, H = d.H, W = d.W, Cin = d.Cin, Cout = d.Cout, ksize = d.ksize, cout_valid = d.cout_valid;
  PDAE_REQUIRE(plan_out && d.in && d.w && d.out, "conv_tc2_create: null pointer");
  PDAE_REQUIRE(ksize == 1 || ksize == 3, "conv_tc2_create: ksize must be 1 or 3");
  PDAE_REQUIRE(Cin % T2_BK == 0, "conv_tc2_create: Cin=%d not a multiple of 64", Cin);
  const bool head = cout_valid > 0;
  PDAE_REQUIRE(head ? (Cout == 16 && cout_valid <= 16 && d.out_dtype == PDAE_F32 && !d.residual && !d.ch_stats) : (Cout % 64 == 0),
               "conv_tc2_create: unsupported Cout=%d (cout_valid=%d)", Cout, cout_valid);
  PDAE_REQUIRE(d.out_dtype == PDAE_F32 || d.out_dtype == PDAE_BF16, "conv_tc2_create: bad out dtype");
  PDAE_REQUIRE(!(d.gm & GM_SPLITK) || (H == 1 && W == 1 && ksize == 1 && !head && d.out_dtype == PDAE_F32 && !d.residual &&
                                       !d.ch_stats && !d.Cin2 && !d.w_batched && d.s2 == 0 && d.softmax_alpha == 0.f),
               "conv_tc2_create: split-K takes the Linear shape (H = W = 1, 1x1) with an fp32 output and no residual, "
               "statistics or fused skip");
  // (a residual is read in the output's dtype: fp32 with an fp32 output, bf16 with a bf16 output)
  PDAE_REQUIRE(((uintptr_t)d.in & 15) == 0 && ((uintptr_t)d.w & 15) == 0 && ((uintptr_t)d.out & 15) == 0 &&
                   ((uintptr_t)d.residual & 15) == 0 && ((uintptr_t)d.bias & 15) == 0,
               "conv_tc2_create: pointers must be 16-byte aligned");
  PDAE_REQUIRE(d.in_ld % 8 == 0 && d.in_bs % 8 == 0 && d.w_ld % 8 == 0 && d.w_bs % 8 == 0 && d.out_ld % 8 == 0 &&
                   d.out_bs % 8 == 0, "conv_tc2_create: strides must be multiples of 16 bytes");
  EncodeTiledFn2 enc = encode_fn2();
  PDAE_REQUIRE(enc != nullptr, "conv_tc2_create: cuTensorMapEncodeTiled unavailable (no driver)");
  if (g_num_sms == 0) {
    int dev = 0;
    PDAE_CUDA(cudaGetDevice(&dev));
    PDAE_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  pdae_conv_tc2_plan* pl = new pdae_conv_tc2_plan();
  ConvTc2Args& a = pl->args;
  a.bias = d.bias; a.ch_stats = d.ch_stats; a.out_nchw = head ? (float*)d.out : nullptr;
  a.fuse = nullptr;
  a.B = B; a.H = H; a.W = W; a.Cout = Cout;
  a.tw = pow2_tile(W, T2_BM);
  a.th = pow2_tile(H, T2_BM / a.tw);
  a.tn = T2_BM / (a.tw * a.th);
  const bool spn = (d.gm & GM_SPLITN) != 0;   // 64-row tiles (batched GEMM, H == 1)
  if (spn) a.tw = 64;
  if (W % a.tw != 0 || H % a.th != 0 || a.tw * a.th * a.tn != (spn ? 64 : T2_BM) || a.tn > 256 || (d.w_batched && a.tn != 1)) {
    delete pl;
    PDAE_REQUIRE(false, "conv_tc2_create: H=%d W=%d cannot be tiled into 128-pixel boxes%s", H, W,
                 d.w_batched ? " of a single image (batched GEMM)" : "");
  }
  a.tiles_x = W / a.tw; a.tiles_y = H / a.th; a.tiles_b = (B + a.tn - 1) / a.tn;
  a.tiles_m = a.tiles_x * a.tiles_y * a.tiles_b;
  a.taps = ksize * ksize; a.ksize = ksize; a.kblocks = Cin / T2_BK;
  a.has_res = d.residual != nullptr; a.out_bf16 = d.out_dtype == PDAE_BF16; a.cout_valid = cout_valid;
  a.w_batched = d.w_batched;
  a.kblocks2 = d.Cin2 / T2_BK;
  a.softmax_alpha = d.softmax_alpha;
  if (d.softmax_alpha > 0.f && !(d.w_batched && d.out_dtype == PDAE_BF16 && !d.residual && !d.bias && !d.ch_stats &&
                                 d.bn_override == Cout)) {
    delete pl;
    PDAE_REQUIRE(false, "conv_tc2_create: the softmax epilogue needs a bf16 batched GEMM whose row fits one tile (N=%d)", Cout);
  }
  int BN;
  if (head) BN = 16;
  else if (d.bn_override == 64 || d.bn_override == 128 || d.bn_override == 256) BN = d.bn_override;
  // (no automatic BN = 256: its 128 accumulator registers per consumer thread spill; only the softmax GEMM, whose row
  //  must fit one tile, asks for it)
  else BN = (Cout % 128 == 0) ? 128 : 64;
  if (!head && Cout % BN != 0) {
    delete pl;
    PDAE_REQUIRE(false, "conv_tc2_create: Cout=%d not a multiple of BN=%d", Cout, BN);
  }
  if (spn) BN /= 2;   // per warpgroup
  pl->BN = BN;
  pl->s2 = d.s2;
  pl->gm = d.gm;
  pl->sg.p = static_cast<const __nv_bfloat16*>(d.sg_p); pl->sg.ld = d.sg_ld; pl->sg.bs = d.sg_bs; pl->sg.alpha = d.sg_alpha;
  a.tiles_total = a.tiles_m * (head ? 1 : Cout / (spn ? 2 * BN : BN)) * (d.s2 == 2 ? 4 : 1);   // stride-2 dgrad: x 4 phases
  if (d.gm & GM_SPLITK) {
    // about one wave of (tile, k range) items; every range non-empty
    const int want = a.tiles_total >= g_num_sms ? 1 : g_num_sms / a.tiles_total;
    a.kchunk = (a.kblocks + want - 1) / want;
    a.splitk = (a.kblocks + a.kchunk - 1) / a.kchunk;
    a.tiles_total *= a.splitk;
    a.out_nchw = static_cast<float*>(d.out);
  }
  const int b_bytes = ((BN * T2_BK * 2 + 1023) / 1024) * 1024 * (spn ? 2 : 1);
  int stage_bytes = T2_A_BYTES + b_bytes;
  const int staging = head ? 0 : (a.has_res ? 2 : 1) * T2_STG_BYTES;
  const int total_all = a.taps * a.kblocks + a.kblocks2;
  pl->grid = a.tiles_total < g_num_sms ? a.tiles_total : g_num_sms;
  // Weights stationary in shared memory: when the whole layer's B operand fits beside >= 4 A-only stages and every CTA
  // runs several tiles of the single n-tile, the weights are fetched once per CTA instead of once per tile (the narrow
  // 64-channel layers are L2->SM bandwidth-bound: this removes a third of their bytes).
  int wbytes = 0;
  a.w_stat = 0;
  // (not for the stride-2 dgrad: its phases read different subsets of the taps)
  if (!head && !d.w_batched && d.s2 != 2 && !(d.gm & GM_SPLITK) && Cout == BN && b_bytes == BN * T2_BK * 2 &&
      a.tiles_total >= 2 * pl->grid) {
    const int wb = total_all * b_bytes;
    if ((220 * 1024 - 1024 - staging - wb) / T2_A_BYTES >= 4) {
      a.w_stat = 1;
      wbytes = wb;
      stage_bytes = T2_A_BYTES;
    }
  }
  int stages = (220 * 1024 - 1024 - staging - wbytes) / stage_bytes;
  if (stages > T2_MAX_STAGES) stages = T2_MAX_STAGES;
  if (stages > total_all) stages = total_all;
  if (stages < 2) stages = 2;
  a.stages = stages;
  pl->smem = (size_t)stages * stage_bytes + wbytes + staging + 1024;

  auto fail = [&](const char* what, int code) {
    delete pl;
    set_error("conv_tc2_create: cuTensorMapEncodeTiled(%s) failed with %d", what, code);
    return PDAE_EINVAL;
  };
  cuuint32_t estr4[4] = {1, 1, 1, 1};
  cuuint32_t estr5[5] = {1, 1, 1, 1, 1};
  if (d.s2 == 1) {
    // parity view of the [B][2H][2W][Cin] input: [B][H][2][W][2 Cin] (kernel header); box = one parity class of the tile
    const cuuint64_t c2 = 2ull * Cin;
    cuuint64_t dims[5] = {c2, (cuuint64_t)W, 2, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[4] = {c2 * 2, 2 * W * c2, 2 * W * c2 * 2, (cuuint64_t)H * 2 * W * c2 * 2};
    cuuint32_t box[5] = {(cuuint32_t)T2_BK, (cuuint32_t)a.tw, 1, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    CUresult r = enc(&pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(d.in), dims, strides, box, estr5,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("A (parity view)", (int)r);
  } else if (d.gm & GM_A_MN) {
    // [batch][K][M] with row stride in_ld: one [64 k][64 m] box per consumer warpgroup
    cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)Cin, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)d.in_ld * 2, (cuuint64_t)d.in_bs * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)T2_BK, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d.in), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("A (MN-major)", (int)r);
  } else {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)d.in_ld * 2, (cuuint64_t)W * d.in_ld * 2, (cuuint64_t)d.in_bs * 2};
    cuuint32_t box[4] = {(cuuint32_t)T2_BK, (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    CUresult r = enc(&pl->tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d.in), dims, strides, box, estr4,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("A", (int)r);
  }
  if (d.gm & GM_B_MN) {
    // [batch][K][N] with row stride w_ld: BN / 64 boxes [64 k][64 n] per stage
    cuuint64_t dims[3] = {(cuuint64_t)Cout, (cuuint64_t)Cin, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)d.w_ld * 2, (cuuint64_t)d.w_bs * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)T2_BK, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d.w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("W (MN-major)", (int)r);
  } else {
    cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)Cout, (cuuint64_t)(d.w_batched ? B : a.taps)};
    cuuint64_t strides[2] = {(cuuint64_t)d.w_ld * 2, (cuuint64_t)d.w_bs * 2};
    cuuint32_t box[3] = {(cuuint32_t)T2_BK, (cuuint32_t)BN, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d.w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("W", (int)r);
  }
  pl->tmO = pl->tmA;
  pl->tmR = pl->tmA;
  pl->tmA2 = pl->tmA;
  pl->tmB2 = pl->tmB;
  pl->tmA3 = pl->tmA;
  if (d.Cin2 > 0) {
    const int Ca = d.in3 ? d.Cin2a : d.Cin2, Cb = d.Cin2 - Ca;
    if (!d.in2 || !d.w2 || d.Cin2 % T2_BK != 0 || head || d.w_batched || ((uintptr_t)d.in2 & 15) || ((uintptr_t)d.w2 & 15) ||
        (d.in3 && (Ca <= 0 || Cb <= 0 || Ca % T2_BK != 0 || ((uintptr_t)d.in3 & 15)))) {
      delete pl;
      PDAE_REQUIRE(false, "conv_tc2_create: bad fused-skip operands (Cin2=%d, Cin2a=%d)", d.Cin2, d.Cin2a);
    }
    a.kblocks2a = Ca / T2_BK;
    cuuint32_t box[4] = {(cuuint32_t)T2_BK, (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    CUresult r = CUDA_SUCCESS;
    for (int part = 0; part < (d.in3 ? 2 : 1); ++part) {
      const int Cp = part ? Cb : Ca;
      cuuint64_t dims[4] = {(cuuint64_t)Cp, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
      cuuint64_t strides[3] = {(cuuint64_t)Cp * 2, (cuuint64_t)W * Cp * 2, (cuuint64_t)H * W * Cp * 2};
      r = enc(part ? &pl->tmA3 : &pl->tmA2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(part ? d.in3 : d.in2), dims,
              strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(part ? "A3" : "A2", (int)r);
    }
    cuuint64_t wd[3] = {(cuuint64_t)d.Cin2, (cuuint64_t)Cout, 1};
    cuuint64_t ws[2] = {(cuuint64_t)d.Cin2 * 2, (cuuint64_t)Cout * d.Cin2 * 2};
    cuuint32_t wb[3] = {(cuuint32_t)T2_BK, (cuuint32_t)BN, 1};
    cuuint32_t we[3] = {1, 1, 1};
    r = enc(&pl->tmB2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(d.w2), wd, ws, wb, we, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("W2", (int)r);
  }
  if (d.s2 == 2) {
    // parity view of the fp32 [B][2H][2W][Cout] data gradient: [B][H][2][W][2 Cout]; one phase per store box
    const cuuint64_t c2 = 2ull * Cout;
    cuuint64_t dims[5] = {c2, (cuuint64_t)W, 2, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[4] = {c2 * 4, 2 * W * c2 * 2, 2 * W * c2 * 4, (cuuint64_t)H * 2 * W * c2 * 4};
    cuuint32_t box[5] = {32, (cuuint32_t)a.tw, 1, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    CUresult r = enc(&pl->tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, d.out, dims, strides, box, estr5, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("O (parity view)", (int)r);
  } else if (!head) {
    const int esz = a.out_bf16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)d.out_ld * esz, (cuuint64_t)W * d.out_ld * esz, (cuuint64_t)d.out_bs * esz};
    cuuint32_t box[4] = {(cuuint32_t)(a.out_bf16 ? 64 : 32), (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
    CUresult r = enc(&pl->tmO, a.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.out, dims,
                     strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("O", (int)r);
    if (a.has_res) {
      cuuint64_t rstr[3] = {(cuuint64_t)Cout * esz, (cuuint64_t)W * Cout * esz, (cuuint64_t)H * W * Cout * esz};
      cuuint32_t rbox[4] = {(cuuint32_t)(a.out_bf16 ? 64 : 32), (cuuint32_t)a.tw, (cuuint32_t)a.th, (cuuint32_t)a.tn};
      r = enc(&pl->tmR, a.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
              const_cast<void*>((const void*)d.residual), dims, rstr, rbox, estr4,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail("R", (int)r);
    }
  }
  *plan_out = pl;
  return PDAE_OK;
}

extern "C" int pdae_conv_tc2_create(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16, const float* bias,
                                    const void* residual, void* out, int out_dtype, float* ch_stats, int B, int H, int W,
                                    int Cin, int Cout, int ksize, int cout_valid, int bn_override) {
  Tc2Desc d;
  d.in = in_bf16; d.w = w_bf16; d.bias = bias; d.residual = residual; d.out = out; d.out_dtype = out_dtype;
  d.ch_stats = ch_stats; d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.ksize = ksize; d.cout_valid = cout_valid;
  d.bn_override = bn_override;
  d.in_ld = Cin; d.in_bs = (long long)H * W * Cin;
  d.w_batched = 0; d.w_ld = Cin; d.w_bs = (long long)Cout * Cin;
  d.out_ld = Cout; d.out_bs = (long long)H * W * Cout;
  return tc2_create(plan_out, d);
}

// conv (ksize 1|3) + fused 1x1 skip conv:  out = conv(in, w) + in2 * w2^T + bias (+ residual); bias must already hold b + b_skip
extern "C" int pdae_conv_tc2_create_skip(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16, const float* bias,
                                         const void* in2_bf16, const void* w2_bf16, int Cin2, void* out, int out_dtype,
                                         float* ch_stats, int B, int H, int W, int Cin, int Cout, int ksize, int bn_override) {
  Tc2Desc d;
  d.in = in_bf16; d.w = w_bf16; d.bias = bias; d.residual = nullptr; d.out = out; d.out_dtype = out_dtype;
  d.ch_stats = ch_stats; d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.ksize = ksize; d.cout_valid = 0;
  d.bn_override = bn_override;
  d.in_ld = Cin; d.in_bs = (long long)H * W * Cin;
  d.w_batched = 0; d.w_ld = Cin; d.w_bs = (long long)Cout * Cin;
  d.out_ld = Cout; d.out_bs = (long long)H * W * Cout;
  d.in2 = in2_bf16; d.w2 = w2_bf16; d.Cin2 = Cin2;
  return tc2_create(plan_out, d);
}

// Same, the skip conv's input being the channel concat cat([in2a (Cin2a ch), in2b (Cin2b ch)]) of two NHWC bf16 tensors
// that is never materialised (unet.py:199 `torch.cat([h, hs.pop()], dim=1)` feeding module.py:297 skip_connection).
extern "C" int pdae_conv_tc2_create_skip2(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16,
                                          const float* bias, const void* in2a_bf16, int Cin2a, const void* in2b_bf16, int Cin2b,
                                          const void* w2_bf16, void* out, int out_dtype, float* ch_stats, int B, int H, int W,
                                          int Cin, int Cout, int ksize, int bn_override) {
  PDAE_REQUIRE(in2b_bf16 && Cin2b > 0, "conv_tc2_create_skip2: second skip source missing");
  Tc2Desc d;
  d.in = in_bf16; d.w = w_bf16; d.bias = bias; d.residual = nullptr; d.out = out; d.out_dtype = out_dtype;
  d.ch_stats = ch_stats; d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.ksize = ksize; d.cout_valid = 0;
  d.bn_override = bn_override;
  d.in_ld = Cin; d.in_bs = (long long)H * W * Cin;
  d.w_batched = 0; d.w_ld = Cin; d.w_bs = (long long)Cout * Cin;
  d.out_ld = Cout; d.out_bs = (long long)H * W * Cout;
  d.in2 = in2a_bf16; d.w2 = w2_bf16; d.Cin2 = Cin2a + Cin2b; d.in3 = in2b_bf16; d.Cin2a = Cin2a;
  return tc2_create(plan_out, d);
}

// Batched GEMM on the same kernel: for every batch item i,  out_i[M x N] = A_i[M x K] * Bm_i[N x K]^T  (both K-major bf16).
// a_ld / b_ld / out_ld: elements between consecutive rows; *_bs: elements between consecutive batch items.
extern "C" int pdae_gemm_tc2_create(pdae_conv_tc2_plan** plan_out, const void* a_bf16, long long a_ld, long long a_bs,
                                    const void* b_bf16, long long b_ld, long long b_bs, void* out, int out_dtype,
                                    long long out_ld, long long out_bs, int batch, int M, int N, int K) {
  Tc2Desc d;
  d.in = a_bf16; d.w = b_bf16; d.bias = nullptr; d.residual = nullptr; d.out = out; d.out_dtype = out_dtype;
  d.ch_stats = nullptr; d.B = batch; d.H = 1; d.W = M; d.Cin = K; d.Cout = N; d.ksize = 1; d.cout_valid = 0; d.bn_override = 0;
  d.in_ld = a_ld; d.in_bs = a_bs;
  d.w_batched = 1; d.w_ld = b_ld; d.w_bs = b_bs;
  d.out_ld = out_ld; d.out_bs = out_bs;
  return tc2_create(plan_out, d);
}

// P_i = softmax_rows(alpha * A_i * Bm_i^T) stored as bf16: the attention-probability GEMM with the softmax folded into the
// epilogue (the fp32 score matrix never leaves the registers).  N must be 64, 128 or 256 (one n-tile holds the whole row).
extern "C" int pdae_gemm_tc2_softmax_create(pdae_conv_tc2_plan** plan_out, const void* a_bf16, long long a_ld, long long a_bs,
                                            const void* b_bf16, long long b_ld, long long b_bs, void* out_bf16, long long out_ld,
                                            long long out_bs, int batch, int M, int N, int K, float alpha) {
  PDAE_REQUIRE(N == 64 || N == 128 || N == 256, "gemm_tc2_softmax_create: N=%d must be 64, 128 or 256", N);
  PDAE_REQUIRE(alpha > 0.f, "gemm_tc2_softmax_create: alpha must be positive");
  Tc2Desc d;
  d.in = a_bf16; d.w = b_bf16; d.bias = nullptr; d.residual = nullptr; d.out = out_bf16; d.out_dtype = PDAE_BF16;
  d.ch_stats = nullptr; d.B = batch; d.H = 1; d.W = M; d.Cin = K; d.Cout = N; d.ksize = 1; d.cout_valid = 0; d.bn_override = N;
  d.in_ld = a_ld; d.in_bs = a_bs;
  d.w_batched = 1; d.w_ld = b_ld; d.w_bs = b_bs;
  d.out_ld = out_ld; d.out_bs = out_bs;
  d.softmax_alpha = alpha;
  return tc2_create(plan_out, d);
}

// ---- batched GEMMs of the attention backward (bf16 autocast training) ---------------------------------------------------
// Every argument is checked before any CUDA call.
static int gemm_validate(const char* fn, const void* a, const void* b, const void* out, long long a_ld, long long a_bs,
                         long long b_ld, long long b_bs, long long out_ld, long long out_bs, int batch, int M, int N, int K) {
  PDAE_REQUIRE(a && b && out, "%s: null pointer", fn);
  PDAE_REQUIRE(!(((uintptr_t)a | (uintptr_t)b | (uintptr_t)out) & 15), "%s: pointers must be 16-byte aligned", fn);
  PDAE_REQUIRE(!((a_ld | a_bs | b_ld | b_bs | out_ld | out_bs) & 7) && a_ld > 0 && b_ld > 0 && out_ld > 0 && a_bs >= 0 &&
                   b_bs >= 0 && out_bs >= 0,
               "%s: strides must be positive multiples of 16 bytes", fn);
  PDAE_REQUIRE(batch > 0 && M > 0 && N > 0 && K > 0 && M % 128 == 0 && N % 64 == 0 && K % 64 == 0,
               "%s: batch=%d M=%d N=%d K=%d: need M %% 128 == 0, N %% 64 == 0, K %% 64 == 0", fn, batch, M, N, K);
  return PDAE_OK;
}

// out_i[M x N] (fp32) = A_i * B_i^T for every batch item i, each operand K-major (a_mn / b_mn = 0: A_i stored [M][K], B_i
// [N][K]) or MN-major (1: A_i stored [K][M], B_i [K][N]); *_ld = elements between consecutive stored rows, *_bs = between items.
extern "C" int pdae_gemm_tc2_create_major(pdae_conv_tc2_plan** plan_out, const void* a_bf16, int a_mn, long long a_ld,
                                          long long a_bs, const void* b_bf16, int b_mn, long long b_ld, long long b_bs, float* out,
                                          long long out_ld, long long out_bs, int batch, int M, int N, int K) {
  static const char* fn = "gemm_tc2_create_major";
  PDAE_REQUIRE(plan_out, "%s: null pointer", fn);
  PDAE_REQUIRE((a_mn == 0 || a_mn == 1) && (b_mn == 0 || b_mn == 1), "%s: major flags must be 0 (K-major) or 1 (MN-major)", fn);
  const int rc = gemm_validate(fn, a_bf16, b_bf16, out, a_ld, a_bs, b_ld, b_bs, out_ld, out_bs, batch, M, N, K);
  if (rc != PDAE_OK) return rc;
  Tc2Desc d;
  d.in = a_bf16; d.w = b_bf16; d.bias = nullptr; d.residual = nullptr; d.out = out; d.out_dtype = PDAE_F32;
  d.ch_stats = nullptr; d.B = batch; d.H = 1; d.W = M; d.Cin = K; d.Cout = N; d.ksize = 1; d.cout_valid = 0; d.bn_override = 0;
  d.in_ld = a_ld; d.in_bs = a_bs;
  d.w_batched = 1; d.w_ld = b_ld; d.w_bs = b_bs;
  d.out_ld = out_ld; d.out_bs = out_bs;
  d.gm = (a_mn ? GM_A_MN : 0) | (b_mn ? GM_B_MN : 0);
  return tc2_create(plan_out, d);
}

// dS_i = alpha * P_i * (dP_i - rowsum(P_i * dP_i)) stored as bf16, dP_i = dO_i * V_i^T (both K-major, strides as in
// pdae_gemm_tc2_create) computed in fp32 and consumed in the epilogue; P_i (bf16) has the output's shape, strides p_ld / p_bs.
// N in {64, 128, 256}: one n-tile holds a whole row.
extern "C" int pdae_gemm_tc2_softmax_grad_create(pdae_conv_tc2_plan** plan_out, const void* do_bf16, long long a_ld, long long a_bs,
                                                 const void* v_bf16, long long b_ld, long long b_bs, const void* p_bf16,
                                                 long long p_ld, long long p_bs, void* ds_bf16, long long out_ld, long long out_bs,
                                                 int batch, int M, int N, int K, float alpha) {
  static const char* fn = "gemm_tc2_softmax_grad_create";
  PDAE_REQUIRE(plan_out && p_bf16, "%s: null pointer", fn);
  PDAE_REQUIRE(!((uintptr_t)p_bf16 & 15), "%s: pointers must be 16-byte aligned", fn);
  const int rc = gemm_validate(fn, do_bf16, v_bf16, ds_bf16, a_ld, a_bs, b_ld, b_bs, out_ld, out_bs, batch, M, N, K);
  if (rc != PDAE_OK) return rc;
  PDAE_REQUIRE(!((p_ld | p_bs) & 7) && p_ld > 0 && p_bs >= 0, "%s: strides must be positive multiples of 16 bytes", fn);
  PDAE_REQUIRE(N == 64 || N == 128 || N == 256, "%s: N=%d must be 64, 128 or 256", fn, N);
  PDAE_REQUIRE(alpha > 0.f, "%s: alpha must be positive", fn);
  Tc2Desc d;
  d.in = do_bf16; d.w = v_bf16; d.bias = nullptr; d.residual = nullptr; d.out = ds_bf16; d.out_dtype = PDAE_BF16;
  d.ch_stats = nullptr; d.B = batch; d.H = 1; d.W = M; d.Cin = K; d.Cout = N; d.ksize = 1; d.cout_valid = 0; d.bn_override = N;
  d.in_ld = a_ld; d.in_bs = a_bs;
  d.w_batched = 1; d.w_ld = b_ld; d.w_bs = b_bs;
  d.out_ld = out_ld; d.out_bs = out_bs;
  d.gm = N == 256 ? GM_SMGRAD | GM_SPLITN : GM_SMGRAD;
  d.sg_p = p_bf16; d.sg_ld = p_ld; d.sg_bs = p_bs; d.sg_alpha = alpha;
  return tc2_create(plan_out, d);
}

// Split-K Linear: out[B][Cout] (fp32) += in[B][Cin] (bf16) * w[Cout][Cin]^T (bf16) (+ bias), the k ranges of each output tile
// spread over the SMs (kernel header).  `out` must be zeroed before every run.
extern "C" int pdae_conv_tc2_create_splitk(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16,
                                           const float* bias, float* out, int B, int Cin, int Cout) {
  PDAE_REQUIRE(B > 0 && Cin > 0 && Cout > 0 && Cout % 64 == 0, "conv_tc2_create_splitk: B=%d Cin=%d Cout=%d: need Cout %% 64 == 0",
               B, Cin, Cout);
  Tc2Desc d;
  d.in = in_bf16; d.w = w_bf16; d.bias = bias; d.residual = nullptr; d.out = out; d.out_dtype = PDAE_F32;
  d.ch_stats = nullptr; d.B = B; d.H = 1; d.W = 1; d.Cin = Cin; d.Cout = Cout; d.ksize = 1; d.cout_valid = 0; d.bn_override = 0;
  d.in_ld = Cin; d.in_bs = Cin;
  d.w_batched = 0; d.w_ld = Cin; d.w_bs = (long long)Cout * Cin;
  d.out_ld = Cout; d.out_bs = Cout;
  d.gm = GM_SPLITK;
  return tc2_create(plan_out, d);
}

// ---- 3x3, stride-2, pad-1 convs on plain bf16 operands (the semantic encoder's bf16 autocast training step) ----------------
// H, W: the conv's INPUT size (even); the output / dY grid is H/2 x W/2.  Every tile shape the 128- and 64-pixel boxes of
// conv_tc2 / wgrad_tc need exists for such a grid (power-of-two tiles, several images per box when the grid is small).
extern "C" int pdae_conv_s2_tc_supported(int H, int W, int Cin, int Cout) {
  return H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && Cin >= 64 && Cout >= 64 && Cin % 64 == 0 && Cout % 64 == 0;
}

static int s2_validate(const char* fn, const void* a, const void* b, const void* out, const float* bias, int B, int H, int W,
                       int Cin, int Cout) {
  PDAE_REQUIRE(a && b && out, "%s: null pointer", fn);
  PDAE_REQUIRE(!(((uintptr_t)a | (uintptr_t)b | (uintptr_t)out | (uintptr_t)bias) & 15), "%s: pointers must be 16-byte aligned", fn);
  PDAE_REQUIRE(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "%s: B=%d H=%d W=%d: H and W must be even and positive", fn, B,
               H, W);
  PDAE_REQUIRE(pdae_conv_s2_tc_supported(H, W, Cin, Cout), "%s: unsupported channels Cin=%d Cout=%d (multiples of 64)", fn, Cin,
               Cout);
  return PDAE_OK;
}

// out[B][H/2][W/2][Cout] (fp32) = conv3x3_stride2_pad1(in[B][H][W][Cin] (bf16), w[9][Cout][Cin] (bf16)) + bias
extern "C" int pdae_conv_tc2_create_s2(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16, const float* bias,
                                       float* out, int B, int H, int W, int Cin, int Cout) {
  PDAE_REQUIRE(plan_out, "conv_tc2_create_s2: null pointer");
  return pdae_conv_tc2_create_s2_ex(plan_out, in_bf16, w_bf16, bias, out, PDAE_F32, nullptr, B, H, W, Cin, Cout);
}

// The same forward with the stride-1 epilogue's options: out (fp32 or bf16 NHWC) and, optionally, the per-channel (sum, sum^2)
// of the stored values accumulated into ch_stats [B][Cout][2].  The output grid is tiled like a stride-1 grid of H/2 x W/2, so
// the epilogue (staging, statistics, TMA store) is the stride-1 one.  Cin is the operand's channel count: a split-operand copy
// [hi | lo | hi] passes 3 C with [W_hi | W_hi | W_lo] weights (the parity view does not care what the 64-channel blocks mean).
extern "C" int pdae_conv_tc2_create_s2_ex(pdae_conv_tc2_plan** plan_out, const void* in_bf16, const void* w_bf16, const float* bias,
                                          void* out, int out_dtype, float* ch_stats, int B, int H, int W, int Cin, int Cout) {
  PDAE_REQUIRE(plan_out, "conv_tc2_create_s2: null pointer");
  const int rc = s2_validate("conv_tc2_create_s2", in_bf16, w_bf16, out, bias, B, H, W, Cin, Cout);
  if (rc != PDAE_OK) return rc;
  PDAE_REQUIRE(out_dtype == PDAE_F32 || out_dtype == PDAE_BF16, "conv_tc2_create_s2: bad out_dtype %d (PDAE_F32 or PDAE_BF16)",
               out_dtype);
  PDAE_REQUIRE(!((uintptr_t)ch_stats & 7), "conv_tc2_create_s2: ch_stats must be 8-byte aligned");
  const int Ho = H / 2, Wo = W / 2;
  Tc2Desc d;
  d.in = in_bf16; d.w = w_bf16; d.bias = bias; d.residual = nullptr; d.out = out; d.out_dtype = out_dtype;
  d.ch_stats = ch_stats; d.B = B; d.H = Ho; d.W = Wo; d.Cin = Cin; d.Cout = Cout; d.ksize = 3; d.cout_valid = 0; d.bn_override = 0;
  d.in_ld = Cin; d.in_bs = (long long)H * W * Cin;
  d.w_batched = 0; d.w_ld = Cin; d.w_bs = (long long)Cout * Cin;
  d.out_ld = Cout; d.out_bs = (long long)Ho * Wo * Cout;
  d.s2 = 1;
  return tc2_create(plan_out, d);
}

// Data gradient of the same conv: dx[B][H][W][Cin] (fp32, every element written) from dy[B][H/2][W/2][Cout] (bf16) and the
// transposed weights wt[9][Cin][Cout] (bf16, wt[3 ky + kx][ci][co] = w[co][ci][ky][kx], NOT flipped: the phases pick the taps)
extern "C" int pdae_conv_tc2_create_s2_dgrad(pdae_conv_tc2_plan** plan_out, const void* dy_bf16, const void* wt_bf16, float* dx,
                                             int B, int H, int W, int Cin, int Cout) {
  PDAE_REQUIRE(plan_out, "conv_tc2_create_s2_dgrad: null pointer");
  const int rc = s2_validate("conv_tc2_create_s2_dgrad", dy_bf16, wt_bf16, dx, nullptr, B, H, W, Cin, Cout);
  if (rc != PDAE_OK) return rc;
  const int Ho = H / 2, Wo = W / 2;
  Tc2Desc d;   // a GEMM over the dY grid with K = Cout, N = Cin
  d.in = dy_bf16; d.w = wt_bf16; d.bias = nullptr; d.residual = nullptr; d.out = dx; d.out_dtype = PDAE_F32;
  d.ch_stats = nullptr; d.B = B; d.H = Ho; d.W = Wo; d.Cin = Cout; d.Cout = Cin; d.ksize = 3; d.cout_valid = 0; d.bn_override = 0;
  d.in_ld = Cout; d.in_bs = (long long)Ho * Wo * Cout;
  d.w_batched = 0; d.w_ld = Cout; d.w_bs = (long long)Cin * Cout;
  d.out_ld = Cin; d.out_bs = (long long)H * W * Cin;
  d.s2 = 2;
  return tc2_create(plan_out, d);
}

// ---- deterministic plans (kernel header, DET) ----------------------------------------------------------------------------
constexpr int T2_DET_SPLIT_ITEMS = 128;   // split-K: about this many (n-tile, split) items per row tile, whatever the batch or GPU

static int tc2_det_splitk(const pdae_conv_tc2_plan* pl, int* kchunk) {
  const int ntn = pl->args.Cout / pl->BN;
  const int want = ntn >= T2_DET_SPLIT_ITEMS ? 1 : T2_DET_SPLIT_ITEMS / ntn;
  const int kc = (pl->args.kblocks + want - 1) / want;
  if (kchunk) *kchunk = kc;
  return (pl->args.kblocks + kc - 1) / kc;
}

static bool tc2_det_mode_ok(const pdae_conv_tc2_plan* pl) {
  if (pl->gm == GM_SPLITK || (pl->gm == 0 && pl->s2 != 2)) return true;
  return pl->args.ch_stats == nullptr;   // training GEMMs and the stride-2 data gradient: no statistics, nothing to slot
}

extern "C" int64_t pdae_conv_tc2_det_workspace_bytes(const pdae_conv_tc2_plan* pl) {
  if (!pl) {
    set_error("conv_tc2_det_workspace_bytes: null plan");
    return PDAE_EINVAL;
  }
  const ConvTc2Args& a = pl->args;
  if (pl->gm == GM_SPLITK) return (int64_t)tc2_det_splitk(pl, nullptr) * a.B * a.Cout * (int64_t)sizeof(float);
  const float* stats = pl->det ? pl->det_out : a.ch_stats;
  if (!stats || a.tiles_x * a.tiles_y == 1) return 0;
  return (int64_t)a.B * a.tiles_x * a.tiles_y * a.Cout * 2 * (int64_t)sizeof(float);
}

// Switch a plan of a forward conv (stride 1 or 2), a batched GEMM without a special epilogue or a split-K Linear to the
// deterministic kernels.  `workspace` (pdae_conv_tc2_det_workspace_bytes, owned by the caller, no initialisation needed) holds
// the slots; the run reduces them.  A split-K plan's output no longer needs zeroing.
extern "C" int pdae_conv_tc2_set_deterministic(pdae_conv_tc2_plan* pl, float* workspace, int64_t workspace_bytes) {
  PDAE_REQUIRE(pl, "conv_tc2_set_deterministic: null plan");
  PDAE_REQUIRE(!pl->det, "conv_tc2_set_deterministic: the plan is deterministic already");
  PDAE_REQUIRE(tc2_det_mode_ok(pl), "conv_tc2_set_deterministic: mode %d (s2 %d) has no deterministic form", pl->gm, pl->s2);
  const int64_t need = pdae_conv_tc2_det_workspace_bytes(pl);
  PDAE_REQUIRE(workspace_bytes >= need && (need == 0 || workspace),
               "conv_tc2_set_deterministic: workspace of %lld bytes, %lld needed (pdae_conv_tc2_det_workspace_bytes)",
               (long long)workspace_bytes, (long long)need);
  PDAE_REQUIRE(!((uintptr_t)workspace & 7), "conv_tc2_set_deterministic: workspace must be 8-byte aligned");
  ConvTc2Args& a = pl->args;
  if (pl->gm == GM_SPLITK) {
    const int tiles = a.tiles_total / a.splitk;
    a.splitk = tc2_det_splitk(pl, &a.kchunk);
    a.tiles_total = tiles * a.splitk;
    pl->grid = a.tiles_total < g_num_sms ? a.tiles_total : g_num_sms;
    pl->det_out = a.out_nchw;
    a.out_nchw = workspace;
  } else if (need > 0) {
    pl->det_out = a.ch_stats;
    a.ch_stats = workspace;
  }
  pl->det = 1;
  return PDAE_OK;
}

extern "C" int pdae_conv_tc2_run(const pdae_conv_tc2_plan* pl, pdae_stream_t stream) {
  PDAE_REQUIRE(pl, "conv_tc2_run: null plan");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e;
#define T2_GO(BN, OB) launch_tc2<BN, OB>(pl->tmA, pl->tmB, pl->tmO, pl->tmR, pl->tmA2, pl->tmB2, pl->tmA3, pl->args, pl->sg, pl->grid, pl->smem, s)
#define T2_GO_S2(BN, OB, S2) \
  launch_tc2<BN, OB, S2>(pl->tmA, pl->tmB, pl->tmO, pl->tmR, pl->tmA2, pl->tmB2, pl->tmA3, pl->args, pl->sg, pl->grid, pl->smem, s)
#define T2_GO_GM(BN, OB, GM) \
  launch_tc2<BN, OB, 0, GM>(pl->tmA, pl->tmB, pl->tmO, pl->tmR, pl->tmA2, pl->tmB2, pl->tmA3, pl->args, pl->sg, pl->grid, pl->smem, s)
  const bool ob = pl->args.out_bf16 != 0;
  if (pl->det) {
#define T2_GO_DET(BN, OB, S2, GM) \
  launch_tc2<BN, OB, S2, GM, true>(pl->tmA, pl->tmB, pl->tmO, pl->tmR, pl->tmA2, pl->tmB2, pl->tmA3, pl->args, pl->sg, pl->grid, pl->smem, s)
    const ConvTc2Args& a = pl->args;
    if (pl->gm == GM_SPLITK) {
      e = pl->BN == 128 ? T2_GO_DET(128, false, 0, GM_SPLITK) : T2_GO_DET(64, false, 0, GM_SPLITK);
      if (e == cudaSuccess) {
        const long long n = (long long)a.B * a.Cout;
        splitk_reduce_kernel<<<cdiv(n, 256), 256, 0, s>>>(a.out_nchw, a.splitk, n, a.Cout, a.bias, pl->det_out);
        e = cudaPeekAtLastError();
      }
    } else if (pl->gm == (GM_SMGRAD | GM_SPLITN)) e = T2_GO_DET(128, true, 0, GM_SMGRAD | GM_SPLITN);
    else if (pl->gm == GM_SMGRAD) e = pl->BN == 128 ? T2_GO_DET(128, true, 0, GM_SMGRAD) : T2_GO_DET(64, true, 0, GM_SMGRAD);
    else if (pl->gm == GM_A_MN) e = pl->BN == 128 ? T2_GO_DET(128, false, 0, GM_A_MN) : T2_GO_DET(64, false, 0, GM_A_MN);
    else if (pl->gm == GM_B_MN) e = pl->BN == 128 ? T2_GO_DET(128, false, 0, GM_B_MN) : T2_GO_DET(64, false, 0, GM_B_MN);
    else if (pl->gm == (GM_A_MN | GM_B_MN))
      e = pl->BN == 128 ? T2_GO_DET(128, false, 0, GM_A_MN | GM_B_MN) : T2_GO_DET(64, false, 0, GM_A_MN | GM_B_MN);
    else if (pl->s2 == 2) e = pl->BN == 128 ? T2_GO_DET(128, false, 2, 0) : T2_GO_DET(64, false, 2, 0);
    else {
      if (pl->s2 == 1) e = pl->BN == 128 ? (ob ? T2_GO_DET(128, true, 1, 0) : T2_GO_DET(128, false, 1, 0))
                                         : (ob ? T2_GO_DET(64, true, 1, 0) : T2_GO_DET(64, false, 1, 0));
      else switch (pl->BN) {
        case 16: e = T2_GO(16, false); break;   // (the image head has no statistics)
        case 64: e = ob ? T2_GO_DET(64, true, 0, 0) : T2_GO_DET(64, false, 0, 0); break;
        case 128: e = ob ? T2_GO_DET(128, true, 0, 0) : T2_GO_DET(128, false, 0, 0); break;
        default: e = ob ? T2_GO_DET(256, true, 0, 0) : T2_GO_DET(256, false, 0, 0); break;
      }
      if (e == cudaSuccess && pl->det_out) e = launch_stat_parts_reduce(a.ch_stats, a.B, a.tiles_x * a.tiles_y, a.Cout, pl->det_out, s);
    }
#undef T2_GO_DET
  } else if (pl->gm == GM_SPLITK) e = pl->BN == 128 ? T2_GO_GM(128, false, GM_SPLITK) : T2_GO_GM(64, false, GM_SPLITK);
  else if (pl->gm == (GM_SMGRAD | GM_SPLITN)) e = T2_GO_GM(128, true, GM_SMGRAD | GM_SPLITN);
  else if (pl->gm == GM_SMGRAD) e = pl->BN == 128 ? T2_GO_GM(128, true, GM_SMGRAD) : T2_GO_GM(64, true, GM_SMGRAD);
  else if (pl->gm == GM_A_MN) e = pl->BN == 128 ? T2_GO_GM(128, false, GM_A_MN) : T2_GO_GM(64, false, GM_A_MN);
  else if (pl->gm == GM_B_MN) e = pl->BN == 128 ? T2_GO_GM(128, false, GM_B_MN) : T2_GO_GM(64, false, GM_B_MN);
  else if (pl->gm == (GM_A_MN | GM_B_MN))
    e = pl->BN == 128 ? T2_GO_GM(128, false, GM_A_MN | GM_B_MN) : T2_GO_GM(64, false, GM_A_MN | GM_B_MN);
  else if (pl->s2 == 1 && ob) e = pl->BN == 128 ? T2_GO_S2(128, true, 1) : T2_GO_S2(64, true, 1);
  else if (pl->s2 == 1) e = pl->BN == 128 ? T2_GO_S2(128, false, 1) : T2_GO_S2(64, false, 1);
  else if (pl->s2 == 2) e = pl->BN == 128 ? T2_GO_S2(128, false, 2) : T2_GO_S2(64, false, 2);
  else switch (pl->BN) {
    case 16: e = T2_GO(16, false); break;
    case 64: e = ob ? T2_GO(64, true) : T2_GO(64, false); break;
    case 128: e = ob ? T2_GO(128, true) : T2_GO(128, false); break;
    default: e = ob ? T2_GO(256, true) : T2_GO(256, false); break;
  }
#undef T2_GO
#undef T2_GO_S2
#undef T2_GO_GM
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("launch of conv_tc2_kernel<%d> (mode %d) failed: %s", pl->BN, pl->gm, cudaGetErrorString(e));
    return PDAE_ECUDA;
  }
  return PDAE_OK;
}

// Image-head plans only: attach the device-side descriptor of the fused sampling update, 10 x int64 =
// { flags, eps*, x_t*, t*, sqrt_recip_alphas_cumprod*, sqrt_recip_alphas_cumprod_m1*, sqrt_one_minus_alphas_cumprod*, alphas_cumprod_prev|next*,
//   g1*, fp32 bits of (1 - alpha) | fp32 bits of alpha << 32 }
// with flags = enabled | use_grad << 1 | eps_only << 2 | ddpm << 3 | interp << 4 | C << 8 | C_eps << 16.  The head keeps writing its own output;
// when enabled it also updates x_t in place (use_grad: this head produces the shift/gradient term and `eps` comes from the other head;
// interp: the gradient is the alpha-blend of g1 and this head's output).  ddpm: the DDPM ancestral step instead, with slots 4..8 =
// { noise_posterior_mean_x_t_coef*, noise_posterior_mean_noise_coef*, shift_coef*, posterior_log_variance_clipped*, noise* }.
extern "C" int pdae_conv_tc2_set_head_fuse(pdae_conv_tc2_plan* pl, const int64_t* fuse_desc_device) {
  PDAE_REQUIRE(pl && pl->BN == 16, "conv_tc2_set_head_fuse: not an image-head plan");
  pl->args.fuse = reinterpret_cast<const long long*>(fuse_desc_device);
  return PDAE_OK;
}

extern "C" void pdae_conv_tc2_destroy(pdae_conv_tc2_plan* pl) { delete pl; }
