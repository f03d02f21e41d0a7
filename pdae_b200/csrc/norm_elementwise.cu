// GroupNorm(32) stats / coefficients / apply (+SiLU, +AdaGN, +concat, +up/down resample), embeddings,
// per-step diffusion arithmetic and the latent-MLP row op.  All HBM-bound: vectorised, coalesced along
// the NHWC channel axis, one pass over the data each.
#include <stdarg.h>

#include "common.cuh"

namespace pdae {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---------------------------------------------------------------------------------------------
// stats: grid (pixel chunks, B). Thread = (channel quad, pixel row) ; per-channel partial sums in
// registers -> shared per-channel fp32 -> per-group fp64 atomics.
constexpr int STATS_PIX = 256;
// pixels per CTA of the statistics kernels: fewer for low-resolution layers so that >= ~4 CTAs per SM exist
static inline int stats_ppc(int B, int HW) {
  int ppc = STATS_PIX;
  while (ppc > 8 && (long long)B * ((HW + ppc - 1) / ppc) < 592) ppc >>= 1;
  return ppc;
}
// pixels per CTA of the deterministic statistics (ch_parts_kernel): from the image size alone, so an image's partial sums are
// grouped, and added, the same way in every batch.  Halved until one image spans >= 16 CTAs, which keeps a batch of one
// spread over several SMs at the low-resolution levels (8 pixels at least: 2 CTAs at 4x4, 8 at 8x8, 16 from 16x16 up).
static inline int stats_ppc_det(int HW) {
  int ppc = STATS_PIX;
  while (ppc > 8 && (HW + ppc - 1) / ppc < 16) ppc >>= 1;
  return ppc;
}

__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ s1, int C1,
                                                       const float* __restrict__ s2, int C2, int HW,
                                                       double* __restrict__ sums, int ppc) {
  extern __shared__ float sh[];  // [2][C]
  const int C = C1 + C2, L = C >> 2;
  const int Lb = L < 256 ? L : 256;
  const int R = 256 / Lb;
  const int tid = threadIdx.x;
  const int lane = tid % Lb, row = tid / Lb;
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * ppc;
  const int p1 = min(HW, p0 + ppc);
  for (int i = tid; i < 2 * C; i += 256) sh[i] = 0.f;
  __syncthreads();
  if (row < R) {
    for (int cq = lane; cq < L; cq += Lb) {
      const int c = cq * 4;
      const float* base;
      int cs, cc;
      if (c < C1) { base = s1; cs = C1; cc = c; } else { base = s2; cs = C2; cc = c - C1; }
      base += (long long)b * HW * cs + cc;
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
      for (int p = p0 + row; p < p1; p += R) {
        const float4 v = *reinterpret_cast<const float4*>(base + (long long)p * cs);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
      atomicAdd(&sh[c + 0], s.x); atomicAdd(&sh[c + 1], s.y); atomicAdd(&sh[c + 2], s.z); atomicAdd(&sh[c + 3], s.w);
      atomicAdd(&sh[C + c + 0], q.x); atomicAdd(&sh[C + c + 1], q.y); atomicAdd(&sh[C + c + 2], q.z); atomicAdd(&sh[C + c + 3], q.w);
    }
  }
  __syncthreads();
  if (tid < 64) {
    const int g = tid & 31, which = tid >> 5;
    const int cpg = C / 32;
    double a = 0.0;
    for (int j = 0; j < cpg; ++j) a += (double)sh[which * C + g * cpg + j];
    atomicAdd(&sums[((long long)b * 32 + g) * 2 + which], a);
  }
}

// per-channel (sum, sum^2) fp32 accumulators [B][C][2] -- the form the tensor-core conv epilogue produces
__global__ void __launch_bounds__(256) ch_stats_kernel(const float* __restrict__ src, int C, int HW, float* __restrict__ chs,
                                                       int ppc) {
  extern __shared__ float sh[];  // [2][C]
  const int L = C >> 2;
  const int Lb = L < 256 ? L : 256;
  const int R = 256 / Lb;
  const int tid = threadIdx.x;
  const int lane = tid % Lb, row = tid / Lb;
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * ppc;
  const int p1 = min(HW, p0 + ppc);
  for (int i = tid; i < 2 * C; i += 256) sh[i] = 0.f;
  __syncthreads();
  if (row < R) {
    for (int cq = lane; cq < L; cq += Lb) {
      const int c = cq * 4;
      const float* base = src + (long long)b * HW * C + c;
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
      for (int p = p0 + row; p < p1; p += R) {
        const float4 v = *reinterpret_cast<const float4*>(base + (long long)p * C);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
      atomicAdd(&sh[c + 0], s.x); atomicAdd(&sh[c + 1], s.y); atomicAdd(&sh[c + 2], s.z); atomicAdd(&sh[c + 3], s.w);
      atomicAdd(&sh[C + c + 0], q.x); atomicAdd(&sh[C + c + 1], q.y); atomicAdd(&sh[C + c + 2], q.z); atomicAdd(&sh[C + c + 3], q.w);
    }
  }
  __syncthreads();
  for (int c = tid; c < C; c += 256) {
    atomicAdd(&chs[((long long)b * C + c) * 2 + 0], sh[c]);
    atomicAdd(&chs[((long long)b * C + c) * 2 + 1], sh[C + c]);
  }
}

// ---- deterministic statistics: no float atomics; every partial has a fixed slot, and slots are summed in a fixed order ----
// Per-CTA per-channel (sum, sum^2) of a virtual concat [s1 (C1) | s2 (C2)] into part[b][blockIdx.x][C][2]: the thread partials
// of ch_stats_kernel, combined across the CTA's pixel rows in row order through shared memory.
__global__ void __launch_bounds__(256) ch_parts_kernel(const float* __restrict__ s1, int C1, const float* __restrict__ s2, int C2,
                                                       int HW, float* __restrict__ part, int ppc) {
  extern __shared__ float sh[];  // [R][2][C]
  const int C = C1 + C2, L = C >> 2;
  const int Lb = L < 256 ? L : 256;
  const int R = 256 / Lb;
  const int tid = threadIdx.x;
  const int lane = tid % Lb, row = tid / Lb;
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * ppc;
  const int p1 = min(HW, p0 + ppc);
  if (row < R) {
    for (int cq = lane; cq < L; cq += Lb) {
      const int c = cq * 4;
      const float* base;
      int cs, cc;
      if (c < C1) { base = s1; cs = C1; cc = c; } else { base = s2; cs = C2; cc = c - C1; }
      base += (long long)b * HW * cs + cc;
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
      for (int p = p0 + row; p < p1; p += R) {
        const float4 v = *reinterpret_cast<const float4*>(base + (long long)p * cs);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
      *reinterpret_cast<float4*>(sh + (size_t)row * 2 * C + c) = s;
      *reinterpret_cast<float4*>(sh + (size_t)row * 2 * C + C + c) = q;
    }
  }
  __syncthreads();
  for (int c = tid; c < C; c += 256) {
    float s = 0.f, q = 0.f;
    for (int r = 0; r < R; ++r) {
      s += sh[(size_t)r * 2 * C + c];
      q += sh[(size_t)r * 2 * C + C + c];
    }
    *reinterpret_cast<float2*>(part + (((long long)b * gridDim.x + blockIdx.x) * C + c) * 2) = make_float2(s, q);
  }
}

// part [B][P][C][2] -> chs [B][C][2].  Block = 32 channels x 8 partial lanes; lane r sums partials r, r + 8, ... in order, then
// lane 0 adds the 8 lane sums in order: the same sums for every grid and every run.
__global__ void __launch_bounds__(256) stat_parts_reduce_kernel(const float* __restrict__ part, int P, int C,
                                                                float* __restrict__ chs) {
  __shared__ float2 red[8][32];
  const int cl = threadIdx.x & 31, r = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl, b = blockIdx.y;
  float2 a = make_float2(0.f, 0.f);
  if (c < C) {
    for (int p = r; p < P; p += 8) {
      const float2 v = *reinterpret_cast<const float2*>(part + (((long long)b * P + p) * C + c) * 2);
      a.x += v.x; a.y += v.y;
    }
  }
  red[r][cl] = a;
  __syncthreads();
  if (r == 0 && c < C) {
    float2 t = red[0][cl];
    for (int k = 1; k < 8; ++k) { t.x += red[k][cl].x; t.y += red[k][cl].y; }
    *reinterpret_cast<float2*>(chs + ((long long)b * C + c) * 2) = t;
  }
}

cudaError_t launch_stat_parts_reduce(const float* part, int B, int P, int C, float* chs, cudaStream_t s) {
  stat_parts_reduce_kernel<<<dim3(cdiv(C, 32), B), 256, 0, s>>>(part, P, C, chs);
  return cudaPeekAtLastError();
}

// part [B][P][C][2] -> per-group fp64 sums [B][32][2] (gn_stats' form).  One block per image: thread (group, which, lane k)
// sums partials k, k + 4, ... over the group's channels in order, then four lane sums are added in order.
__global__ void __launch_bounds__(256) gn_group_reduce_kernel(const float* __restrict__ part, int P, int C,
                                                              double* __restrict__ sums) {
  __shared__ double red[4][64];
  const int gw = threadIdx.x & 63, k = threadIdx.x >> 6;
  const int g = gw & 31, which = gw >> 5, cpg = C / 32, b = blockIdx.x;
  double a = 0.0;
  for (int p = k; p < P; p += 4) {
    const float* row = part + (((long long)b * P + p) * C + g * cpg) * 2 + which;
    for (int j = 0; j < cpg; ++j) a += (double)row[2 * j];
  }
  red[k][gw] = a;
  __syncthreads();
  if (k == 0) sums[((long long)b * 32 + g) * 2 + which] = ((red[0][gw] + red[1][gw]) + red[2][gw]) + red[3][gw];
}

// GroupNorm coefficients from per-channel sums of a virtual concat [chs1 (C1) | chs2 (C2)]
__global__ void gn_coef_ch_kernel(const float* __restrict__ chs1, int C1, const float* __restrict__ chs2, int C2,
                                  const float* __restrict__ gamma, const float* __restrict__ beta, int HW, float eps,
                                  const float* __restrict__ emb, int emb_ld, const float* __restrict__ embz, int embz_ld,
                                  float* __restrict__ ab) {
  __shared__ double gs[32][2];
  const int b = blockIdx.x;
  const int C = C1 + C2, cpg = C / 32;
  if (threadIdx.x < 64) {
    const int g = threadIdx.x & 31, which = threadIdx.x >> 5;
    double a = 0.0;
    for (int j = 0; j < cpg; ++j) {
      const int c = g * cpg + j;
      a += (double)(c < C1 ? chs1[((long long)b * C1 + c) * 2 + which] : chs2[((long long)b * C2 + (c - C1)) * 2 + which]);
    }
    gs[g][which] = a;
  }
  __syncthreads();
  const double n = (double)HW * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mean = gs[g][0] / n;
    double var = gs[g][1] / n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    float a = gamma[c] * rstd;
    float bb = beta[c] - (float)mean * a;
    if (emb) {
      const float s = 1.0f + emb[(long long)b * emb_ld + c], shv = emb[(long long)b * emb_ld + C + c];
      a *= s;
      bb = bb * s + shv;
    }
    if (embz) {
      const float s = 1.0f + embz[(long long)b * embz_ld + c], shv = embz[(long long)b * embz_ld + C + c];
      a *= s;
      bb = bb * s + shv;
    }
    ab[((long long)b * 2 + 0) * C + c] = a;
    ab[((long long)b * 2 + 1) * C + c] = bb;
  }
}

__global__ void gn_coef_kernel(const double* __restrict__ sums, const float* __restrict__ gamma,
                               const float* __restrict__ beta, int C, int HW, float eps,
                               const float* __restrict__ emb, int emb_ld, const float* __restrict__ embz, int embz_ld,
                               float* __restrict__ ab) {
  const int b = blockIdx.x;
  const int cpg = C / 32;
  const double n = (double)HW * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mean = sums[((long long)b * 32 + g) * 2] / n;
    double var = sums[((long long)b * 32 + g) * 2 + 1] / n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    float a = gamma[c] * rstd;
    float bb = beta[c] - (float)mean * a;
    if (emb) {
      const float s = 1.0f + emb[(long long)b * emb_ld + c], shv = emb[(long long)b * emb_ld + C + c];
      a *= s;
      bb = bb * s + shv;
    }
    if (embz) {
      const float s = 1.0f + embz[(long long)b * embz_ld + c], shv = embz[(long long)b * embz_ld + C + c];
      a *= s;
      bb = bb * s + shv;
    }
    ab[((long long)b * 2 + 0) * C + c] = a;
    ab[((long long)b * 2 + 1) * C + c] = bb;
  }
}

// ---------------------------------------------------------------------------------------------
// apply: flat float4 work items over [pixels][C/4]; consecutive threads walk consecutive channel quads.
// FAST: approximate exp / division (MUFU) -- used when the result is rounded to bf16 anyway
template <bool FAST>
__device__ __forceinline__ float silu_t(float x) {
  if (FAST) {  // x*sigmoid(x) = h + h*tanh(h), h = x/2 : ONE MUFU op (tanh.approx) instead of ex2 + rcp
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
  }
  return silu_f(x);
}
template <bool FAST = false>
__device__ __forceinline__ float4 affine_act(float4 v, float4 a, float4 b, int silu) {
  float4 r;
  r.x = fmaf(a.x, v.x, b.x); r.y = fmaf(a.y, v.y, b.y); r.z = fmaf(a.z, v.z, b.z); r.w = fmaf(a.w, v.w, b.w);
  if (silu) { r.x = silu_t<FAST>(r.x); r.y = silu_t<FAST>(r.y); r.z = silu_t<FAST>(r.z); r.w = silu_t<FAST>(r.w); }
  return r;
}

// Non-resampling, bf16-activation fast path: 8 channels (16 B of bf16 output) per work item, fast SiLU.
template <typename T>
__device__ __forceinline__ void load8(const T* p, float4& v0, float4& v1) {
  if (sizeof(T) == 2) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    const float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]), f2 = __bfloat1622float2(h[2]),
                 f3 = __bfloat1622float2(h[3]);
    v0 = make_float4(f0.x, f0.y, f1.x, f1.y);
    v1 = make_float4(f2.x, f2.y, f3.x, f3.y);
  } else {
    v0 = *reinterpret_cast<const float4*>(p);
    v1 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + 4);
  }
}

// raw (unconverted) 8-channel load: 16 B for bf16, 32 B for fp32 -- kept raw so a batch of loads is cheap in registers
template <typename T> struct Raw8;
template <> struct Raw8<__nv_bfloat16> { uint4 u; };
template <> struct Raw8<float> { float4 a, b; };
__device__ __forceinline__ void ld_raw8(const __nv_bfloat16* p, Raw8<__nv_bfloat16>& r) { r.u = __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void ld_raw8(const float* p, Raw8<float>& r) {
  r.a = __ldg(reinterpret_cast<const float4*>(p));
  r.b = __ldg(reinterpret_cast<const float4*>(p) + 1);
}
__device__ __forceinline__ void cvt_raw8(const Raw8<__nv_bfloat16>& r, float4& v0, float4& v1) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&r.u);
  const float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]), f2 = __bfloat1622float2(h[2]),
               f3 = __bfloat1622float2(h[3]);
  v0 = make_float4(f0.x, f0.y, f1.x, f1.y);
  v1 = make_float4(f2.x, f2.y, f3.x, f3.y);
}
__device__ __forceinline__ void cvt_raw8(const Raw8<float>& r, float4& v0, float4& v1) { v0 = r.a; v1 = r.b; }

// One source, one channel octet per thread, pixels strided.  U loads are issued back to back before any dependent
// math / store (the compiler serialises them otherwise: one 16-B load in flight per thread caps the kernel at ~4 TB/s).
template <typename T, typename TRaw, int U>
__device__ __forceinline__ void apply8_loop(const T* __restrict__ p, int Cs, __nv_bfloat16* __restrict__ po,
                                            TRaw* __restrict__ pr, int C, int pix, int stride, int HW, float4 a0, float4 a1,
                                            float4 b0, float4 b1, int silu) {
  auto emit = [&](const Raw8<T>& r, int px) {
    float4 v0, v1;
    cvt_raw8(r, v0, v1);
    const float4 r0 = affine_act<true>(v0, a0, b0, silu), r1 = affine_act<true>(v1, a1, b1, silu);
    __nv_bfloat162 h[4] = {__floats2bfloat162_rn(r0.x, r0.y), __floats2bfloat162_rn(r0.z, r0.w),
                           __floats2bfloat162_rn(r1.x, r1.y), __floats2bfloat162_rn(r1.z, r1.w)};
    *reinterpret_cast<uint4*>(po + (long long)px * C) = *reinterpret_cast<uint4*>(h);
    if (pr) {
      if (sizeof(TRaw) == sizeof(T)) {  // same type: forward the raw bits
        *reinterpret_cast<Raw8<T>*>(pr + (long long)px * C) = r;
      } else {
        store4<TRaw>(pr + (long long)px * C, v0);
        store4<TRaw>(pr + (long long)px * C + 4, v1);
      }
    }
  };
  for (; pix + (U - 1) * stride < HW; pix += U * stride) {
    Raw8<T> r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) ld_raw8(p + (long long)(pix + u * stride) * Cs, r[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) emit(r[u], pix + u * stride);
  }
  for (; pix < HW; pix += stride) {
    Raw8<T> r;
    ld_raw8(p + (long long)pix * Cs, r);
    emit(r, pix);
  }
}

// Source selection for a virtual concat: with both sources of one type the (pointer, pitch) pair is SELECTED, so a warp
// whose lanes straddle the two sources runs the pixel loop once (a branch would run it twice with half the lanes idle).
template <typename TSrc, typename TSrc2, typename TRaw>
__device__ __forceinline__ void apply8_dispatch(const TSrc* __restrict__ s1, int C1, const TSrc2* __restrict__ s2, int C2, int b,
                                                int c, __nv_bfloat16* __restrict__ po, TRaw* __restrict__ pr, int C, int pix0,
                                                int stride, int HW, float4 a0, float4 a1, float4 b0, float4 b1, int silu) {
  if constexpr (sizeof(TSrc) == sizeof(TSrc2)) {
    const bool first = c < C1;
    const TSrc* p = first ? s1 + (long long)b * HW * C1 + c
                          : reinterpret_cast<const TSrc*>(s2) + (long long)b * HW * C2 + (c - C1);
    apply8_loop<TSrc, TRaw, 4>(p, first ? C1 : C2, po, pr, C, pix0, stride, HW, a0, a1, b0, b1, silu);
  } else {
    if (c < C1)
      apply8_loop<TSrc, TRaw, 4>(s1 + (long long)b * HW * C1 + c, C1, po, pr, C, pix0, stride, HW, a0, a1, b0, b1, silu);
    else
      apply8_loop<TSrc2, TRaw, 4>(s2 + (long long)b * HW * C2 + (c - C1), C2, po, pr, C, pix0, stride, HW, a0, a1, b0, b1, silu);
  }
}

template <typename TSrc, typename TSrc2, typename TRaw>
__global__ void __launch_bounds__(256) gn_apply8_kernel(const TSrc* __restrict__ s1, int C1, const TSrc2* __restrict__ s2,
                                                        int C2, const float* __restrict__ ab, int silu, int HW,
                                                        __nv_bfloat16* __restrict__ out_act, TRaw* __restrict__ out_raw) {
  // thread -> fixed channel octet (tid % L), pixels strided: no division and no coefficient reload inside the loop.
  // blockDim.x = L * floor(256 / L) with L = C/8 <= 256; the host falls back to the generic kernel otherwise.
  const int C = C1 + C2, L = C >> 3;
  const int b = blockIdx.y;
  const int cq = threadIdx.x % L, prow = threadIdx.x / L, ppc = blockDim.x / L;   // pixels per CTA pass (blockDim = L * ppc)
  const int c = cq * 8;
  float4 a0 = make_float4(1.f, 1.f, 1.f, 1.f), a1 = a0, b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
  if (ab) {
    const float* pa = ab + ((long long)b * 2 + 0) * C + c;
    const float* pb = ab + ((long long)b * 2 + 1) * C + c;
    a0 = *reinterpret_cast<const float4*>(pa); a1 = *reinterpret_cast<const float4*>(pa + 4);
    b0 = *reinterpret_cast<const float4*>(pb); b1 = *reinterpret_cast<const float4*>(pb + 4);
  }
  __nv_bfloat16* po = out_act + (long long)b * HW * C + c;
  TRaw* pr = out_raw ? out_raw + (long long)b * HW * C + c : nullptr;
  const int stride = gridDim.x * ppc, pix0 = blockIdx.x * ppc + prow;
  apply8_dispatch<TSrc, TSrc2, TRaw>(s1, C1, s2, C2, b, c, po, pr, C, pix0, stride, HW, a0, a1, b0, b1, silu);
}

template <typename TSrc, typename TSrc2, typename TAct, typename TRaw, int RS>
__global__ void __launch_bounds__(256) gn_apply_kernel(const TSrc* __restrict__ s1, int C1,
                                                       const TSrc2* __restrict__ s2, int C2,
                                                       const float* __restrict__ ab, int silu, int H, int W,
                                                       TAct* __restrict__ out_act, TRaw* __restrict__ out_raw) {
  const int C = C1 + C2, L = C >> 2;
  const int b = blockIdx.y;
  // iteration space: source pixels for NONE / UP2, output pixels for DOWN2
  const int Hi = RS == PDAE_RESAMPLE_DOWN2 ? H / 2 : H, Wi = RS == PDAE_RESAMPLE_DOWN2 ? W / 2 : W;
  const long long items = (long long)Hi * Wi * L;
  const int Ho = RS == PDAE_RESAMPLE_UP2 ? 2 * H : Hi, Wo = RS == PDAE_RESAMPLE_UP2 ? 2 * W : Wi;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items;
       it += (long long)gridDim.x * blockDim.x) {
    const int cq = (int)(it % L);
    const long long pix = it / L;
    const int x = (int)(pix % Wi), y = (int)(pix / Wi);
    const int c = cq * 4;
    // source 1 may be bf16 (a conv output kept in bf16); source 2 (a skip tensor) is always fp32
    const bool first = c < C1;
    const int cs = first ? C1 : C2, cc = first ? c : c - C1;
    const long long boff = (long long)b * H * W * cs + cc;
    auto ld = [&](long long pixoff) -> float4 {
      return first ? load4<TSrc>(s1 + boff + pixoff * cs) : load4<TSrc2>(s2 + boff + pixoff * cs);
    };
    float4 a = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ab) {
      a = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 0) * C + c);
      bb = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 1) * C + c);
    }
    if (RS == PDAE_RESAMPLE_DOWN2) {
      float4 accA = make_float4(0.f, 0.f, 0.f, 0.f), accR = accA;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const float4 v = ld((long long)(2 * y + dy) * W + 2 * x + dx);
          const float4 r = affine_act(v, a, bb, silu);
          accA.x += r.x; accA.y += r.y; accA.z += r.z; accA.w += r.w;
          accR.x += v.x; accR.y += v.y; accR.z += v.z; accR.w += v.w;
        }
      const long long o = (((long long)b * Ho + y) * Wo + x) * C + c;
      store4<TAct>(out_act + o, make_float4(accA.x * 0.25f, accA.y * 0.25f, accA.z * 0.25f, accA.w * 0.25f));
      if (out_raw) store4<TRaw>(out_raw + o, make_float4(accR.x * 0.25f, accR.y * 0.25f, accR.z * 0.25f, accR.w * 0.25f));
    } else {
      const float4 v = ld((long long)y * W + x);
      const float4 r = affine_act(v, a, bb, silu);
      if (RS == PDAE_RESAMPLE_UP2) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) {
            const long long o = (((long long)b * Ho + 2 * y + dy) * Wo + 2 * x + dx) * C + c;
            store4<TAct>(out_act + o, r);
            if (out_raw) store4<TRaw>(out_raw + o, v);
          }
      } else {
        const long long o = (((long long)b * Ho + y) * Wo + x) * C + c;
        store4<TAct>(out_act + o, r);
        if (out_raw) store4<TRaw>(out_raw + o, v);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// "bf16x3" precision: activations are written as THREE bf16 channel blocks [hi | lo | hi] (hi = bf16(a), lo = bf16(a - hi))
// so that a tensor-core conv whose weights are packed [W_hi | W_hi | W_lo] along Cin computes
// a_hi*W_hi + a_lo*W_hi + a_hi*W_lo = a*W to ~2^-16 relative -- fp32-grade results from bf16 MMAs (3x the MMA work).
// Sources fp32; raw output either fp32 (plain, C channels) or bf16 (split, 3C channels).
__device__ __forceinline__ void store_split3(__nv_bfloat16* pix_base, int C, int c, float4 r) {
  const __nv_bfloat162 h0 = __floats2bfloat162_rn(r.x, r.y), h1 = __floats2bfloat162_rn(r.z, r.w);
  const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
  const __nv_bfloat162 l0 = __floats2bfloat162_rn(r.x - f0.x, r.y - f0.y), l1 = __floats2bfloat162_rn(r.z - f1.x, r.w - f1.y);
  uint2 hi, lo;
  hi.x = *reinterpret_cast<const uint32_t*>(&h0); hi.y = *reinterpret_cast<const uint32_t*>(&h1);
  lo.x = *reinterpret_cast<const uint32_t*>(&l0); lo.y = *reinterpret_cast<const uint32_t*>(&l1);
  *reinterpret_cast<uint2*>(pix_base + c) = hi;
  *reinterpret_cast<uint2*>(pix_base + C + c) = lo;
  *reinterpret_cast<uint2*>(pix_base + 2 * C + c) = hi;
}

template <typename TRaw, int RS>
__global__ void __launch_bounds__(256) gn_apply_split3_kernel(const float* __restrict__ s1, int C1, const float* __restrict__ s2,
                                                              int C2, const float* __restrict__ ab, int silu, int H, int W,
                                                              __nv_bfloat16* __restrict__ out_act, TRaw* __restrict__ out_raw) {
  const int C = C1 + C2, L = C >> 2;
  const int b = blockIdx.y;
  const int Hi = RS == PDAE_RESAMPLE_DOWN2 ? H / 2 : H, Wi = RS == PDAE_RESAMPLE_DOWN2 ? W / 2 : W;
  const long long items = (long long)Hi * Wi * L;
  const int Ho = RS == PDAE_RESAMPLE_UP2 ? 2 * H : Hi, Wo = RS == PDAE_RESAMPLE_UP2 ? 2 * W : Wi;
  constexpr bool RAW_SPLIT = sizeof(TRaw) == 2;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (long long)gridDim.x * blockDim.x) {
    const int cq = (int)(it % L);
    const long long pix = it / L;
    const int x = (int)(pix % Wi), y = (int)(pix / Wi);
    const int c = cq * 4;
    const bool first = c < C1;
    const int cs = first ? C1 : C2, cc = first ? c : c - C1;
    const float* src = (first ? s1 : s2) + (long long)b * H * W * cs + cc;
    float4 a = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ab) {
      a = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 0) * C + c);
      bb = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 1) * C + c);
    }
    auto put = [&](int oy, int ox, float4 r, float4 v) {
      const long long o = ((long long)b * Ho + oy) * Wo + ox;
      store_split3(out_act + o * 3 * C, C, c, r);
      if (out_raw) {
        if (RAW_SPLIT) store_split3(reinterpret_cast<__nv_bfloat16*>(out_raw) + o * 3 * C, C, c, v);
        else store4<float>(reinterpret_cast<float*>(out_raw) + o * C + c, v);
      }
    };
    if (RS == PDAE_RESAMPLE_DOWN2) {
      float4 accA = make_float4(0.f, 0.f, 0.f, 0.f), accR = accA;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const float4 v = *reinterpret_cast<const float4*>(src + ((long long)(2 * y + dy) * W + 2 * x + dx) * cs);
          const float4 r = affine_act(v, a, bb, silu);
          accA.x += r.x; accA.y += r.y; accA.z += r.z; accA.w += r.w;
          accR.x += v.x; accR.y += v.y; accR.z += v.z; accR.w += v.w;
        }
      put(y, x, make_float4(accA.x * 0.25f, accA.y * 0.25f, accA.z * 0.25f, accA.w * 0.25f),
          make_float4(accR.x * 0.25f, accR.y * 0.25f, accR.z * 0.25f, accR.w * 0.25f));
    } else {
      const float4 v = *reinterpret_cast<const float4*>(src + ((long long)y * W + x) * cs);
      const float4 r = affine_act(v, a, bb, silu);
      if (RS == PDAE_RESAMPLE_UP2) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) put(2 * y + dy, 2 * x + dx, r, v);
      } else {
        put(y, x, r, v);
      }
    }
  }
}


// ---------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const int64_t* __restrict__ t, int B, int dim,
                                          const float* __restrict__ freqs, float* __restrict__ out) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * dim) return;
  const int b = idx / dim, j = idx % dim;
  float v = 0.f;
  if (j < 2 * half) {
    const int i = j < half ? j : j - half;
    // freqs[] is computed on the host with the reference's own fp32 op sequence (a 1-ulp difference in
    // exp() would be amplified ~1000x by t before the cos/sin).
    const float arg = __fmul_rn((float)t[b], freqs[i]);
    v = j < half ? cosf(arg) : sinf(arg);
  }
  out[idx] = v;
}

__global__ void embedding_add_kernel(float* __restrict__ emb, const float* __restrict__ table,
                                     const int64_t* __restrict__ idx, int B, int E) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * E) return;
  const int b = i / E, j = i % E;
  emb[i] += table[idx[b] * E + j];
}

__global__ void ddim_step_kernel(const float* __restrict__ x, const float* __restrict__ eps,
                                 const float* __restrict__ grad, const int64_t* __restrict__ t,
                                 const float* __restrict__ tA, const float* __restrict__ tB,
                                 const float* __restrict__ tS, const float* __restrict__ tab,
                                 float* __restrict__ out, long long per_sample, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_sample);
    const int64_t tb = t[b];
    const float A = tA[tb], Bm = tB[tb], abar = tab[tb];
    float e = eps[i];
    if (grad) e = __fsub_rn(e, __fmul_rn(tS[tb], grad[i]));
    const float ax = __fmul_rn(A, x[i]);
    float x0 = __fsub_rn(ax, __fmul_rn(Bm, e));
    x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
    const float e2 = __fdiv_rn(__fsub_rn(ax, x0), Bm);
    out[i] = __fadd_rn(__fmul_rn(x0, sqrtf(abar)), __fmul_rn(sqrtf(__fsub_rn(1.0f, abar)), e2));
  }
}

// One step of a sampling loop's bookkeeping, on the device so that the whole step is ONE CUDA-graph replay: read the loop
// index i from `counter`, broadcast it (t_loc, the index into the respaced DDIM tables) and the original-schedule timestep
// map[i] (t_net, the network's time input; ddim.py:39-41 t_transform), then advance the counter by `delta`.
__global__ void ddim_select_t_kernel(long long* __restrict__ counter, int delta, const int64_t* __restrict__ map, int map_len,
                                     int64_t* __restrict__ t_loc, int64_t* __restrict__ t_net, int B) {
  const long long i = *counter;
  const long long ic = i < 0 ? 0 : (i >= map_len ? map_len - 1 : i);
  const int64_t m = map[ic];
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    t_loc[b] = (int64_t)ic;
    t_net[b] = m;
  }
  __syncthreads();
  if (threadIdx.x == 0) *counter = i + delta;
}

__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                const int64_t* __restrict__ t, const float* __restrict__ c1,
                                const float* __restrict__ c2, float* __restrict__ out, long long per_sample,
                                long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int64_t tb = t[i / per_sample];
    out[i] = __fadd_rn(__fmul_rn(c1[tb], x0[i]), __fmul_rn(c2[tb], noise[i]));
  }
}

__global__ void noise_p_sample_kernel(const float* __restrict__ x, const float* __restrict__ eps,
                                      const float* __restrict__ noise, const float* __restrict__ lr,
                                      const int64_t* __restrict__ t, const float* __restrict__ cx,
                                      const float* __restrict__ ce, const float* __restrict__ logvar,
                                      const float* __restrict__ logbeta, float* __restrict__ out,
                                      long long per_sample, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int64_t tb = t[i / per_sample];
    const float mean = __fsub_rn(__fmul_rn(cx[tb], x[i]), __fmul_rn(ce[tb], eps[i]));
    float lv = logvar[tb];
    if (lr) {
      const float frac = __fmul_rn(__fadd_rn(lr[i], 1.0f), 0.5f);
      lv = __fadd_rn(lv, __fmul_rn(frac, __fsub_rn(logbeta[tb], lv)));
    }
    const float mask = tb == 0 ? 0.0f : 1.0f;
    out[i] = __fadd_rn(mean, __fmul_rn(__fmul_rn(mask, expf(__fmul_rn(0.5f, lv))), noise[i]));
  }
}

// noise_p_sample_kernel with eps (and lr) read at per-sample stride eps_ld (the two halves of a learned-sigma output) and an
// optional shift term added first: e = eps + shift[t] * grad, rounded after the product and after the sum like the reference.
__global__ void noise_p_sample_shift_kernel(const float* __restrict__ x, const float* __restrict__ eps,
                                            const float* __restrict__ grad, const float* __restrict__ tS,
                                            const float* __restrict__ noise, const float* __restrict__ lr, long long eps_ld,
                                            const int64_t* __restrict__ t, const float* __restrict__ cx,
                                            const float* __restrict__ ce, const float* __restrict__ logvar,
                                            const float* __restrict__ logbeta, float* __restrict__ out,
                                            long long per_sample, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / per_sample;
    const long long ei = b * eps_ld + (i - b * per_sample);
    const int64_t tb = t[b];
    float e = eps[ei];
    if (grad) e = __fadd_rn(e, __fmul_rn(tS[tb], grad[i]));
    const float mean = __fsub_rn(__fmul_rn(cx[tb], x[i]), __fmul_rn(ce[tb], e));
    float lv = logvar[tb];
    if (lr) {
      const float frac = __fmul_rn(__fadd_rn(lr[ei], 1.0f), 0.5f);
      lv = __fadd_rn(lv, __fmul_rn(frac, __fsub_rn(logbeta[tb], lv)));
    }
    const float mask = tb == 0 ? 0.0f : 1.0f;
    out[i] = __fadd_rn(mean, __fmul_rn(__fmul_rn(mask, expf(__fmul_rn(0.5f, lv))), noise[i]));
  }
}

// (1 - alpha) * g1 + alpha * g2 in fp32 as torch evaluates it: ab = { fp32(1 - alpha), fp32(alpha) } in device memory, so a
// captured step graph serves every alpha.
__global__ void grad_blend_kernel(const float* __restrict__ g1, const float* __restrict__ g2, const float* __restrict__ ab,
                                  float* __restrict__ out, long long n) {
  const float a1 = ab[0], a2 = ab[1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __fadd_rn(__fmul_rn(a1, g1[i]), __fmul_rn(a2, g2[i]));
}

// The gap measure's per-step terms (gaussian_diffusion.py:292-318) in fp32, in the reference's expression order (one rounding
// per product and per sum): true = c0 x0 + c1 xt; m1 = c0 (A xt - Bm eps) + c1 xt; m2 the same with eps + S grad; then
// (true - m1)^2 and (true - m2)^2.  Each block sums GAP_PER_BLOCK consecutive elements in fp64 in a fixed order and writes its
// two partials; the grid follows the element count only, so the partials -- and the final sum -- are the same on every run.
constexpr int GAP_THREADS = 256;
constexpr int GAP_ITEMS = 16;
constexpr long long GAP_PER_BLOCK = (long long)GAP_THREADS * GAP_ITEMS;

__device__ __forceinline__ void gap_block_sum(double& a, double& b, double (*red)[GAP_THREADS / 32]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0; b = 0.0;
    for (int w = 0; w < GAP_THREADS / 32; ++w) { a += red[0][w]; b += red[1][w]; }
  }
}

__global__ void __launch_bounds__(GAP_THREADS) gap_terms_partial_kernel(
    const float* __restrict__ x0, const float* __restrict__ xt, const float* __restrict__ eps, const float* __restrict__ grad,
    const int64_t* __restrict__ t, const float* __restrict__ c0, const float* __restrict__ c1, const float* __restrict__ tA,
    const float* __restrict__ tBm, const float* __restrict__ tS, double* __restrict__ partial, long long per_sample,
    long long total) {
  __shared__ double red[2][GAP_THREADS / 32];
  double s1 = 0.0, s2 = 0.0;
  const long long base = (long long)blockIdx.x * GAP_PER_BLOCK + threadIdx.x;
#pragma unroll 4
  for (int k = 0; k < GAP_ITEMS; ++k) {
    const long long i = base + (long long)k * GAP_THREADS;
    if (i < total) {
      const int64_t tb = t[i / per_sample];
      const float a0 = c0[tb], a1 = c1[tb], A = tA[tb], Bm = tBm[tb];
      const float x = xt[i], e = eps[i];
      const float cx = __fmul_rn(a1, x), ax = __fmul_rn(A, x);
      const float tru = __fadd_rn(__fmul_rn(a0, x0[i]), cx);
      const float m1 = __fadd_rn(__fmul_rn(a0, __fsub_rn(ax, __fmul_rn(Bm, e))), cx);
      const float eae = __fadd_rn(e, __fmul_rn(tS[tb], grad[i]));
      const float m2 = __fadd_rn(__fmul_rn(a0, __fsub_rn(ax, __fmul_rn(Bm, eae))), cx);
      const float d1 = __fsub_rn(tru, m1), d2 = __fsub_rn(tru, m2);
      s1 += (double)__fmul_rn(d1, d1);
      s2 += (double)__fmul_rn(d2, d2);
    }
  }
  gap_block_sum(s1, s2, red);
  if (threadIdx.x == 0) {
    partial[2 * blockIdx.x] = s1;
    partial[2 * blockIdx.x + 1] = s2;
  }
}

// One block: the partials in a fixed order, then the two means into row t[0] of out ([T][2]).
__global__ void __launch_bounds__(GAP_THREADS) gap_terms_final_kernel(const double* __restrict__ partial, int nblk,
                                                                      const int64_t* __restrict__ t, float* __restrict__ out,
                                                                      double total) {
  __shared__ double red[2][GAP_THREADS / 32];
  double s1 = 0.0, s2 = 0.0;
  for (int j = threadIdx.x; j < nblk; j += GAP_THREADS) {
    s1 += partial[2 * j];
    s2 += partial[2 * j + 1];
  }
  gap_block_sum(s1, s2, red);
  if (threadIdx.x == 0) {
    float* row = out + 2 * t[0];
    row[0] = (float)(s1 / total);
    row[1] = (float)(s2 / total);
  }
}

// OutT of the latent MLP's row kernels in the split-operand plan: a value v is stored as hi = bf16_rn(v) at p, lo =
// bf16_rn(v - hi) at p + blk and hi again at p + 2 blk -- the [hi | lo | hi] column blocks of a [B][3 blk] split operand,
// rounded as store_split3 rounds them.
struct Split3 {
  __nv_bfloat16 v;
};
template <typename OutT>
__device__ __forceinline__ void store_row(OutT* p, int, float v) { store1(p, v); }
__device__ __forceinline__ void store_row(Split3* p, int blk, float v) {
  __nv_bfloat16* q = reinterpret_cast<__nv_bfloat16*>(p);
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
  q[0] = hi;
  q[blk] = lo;
  q[2 * blk] = hi;
}

// one CTA per row: y = act(LN(h*(1+cond))) (* mask * scale, the inverted dropout of pdae_mul_mask_cols); cond row b at
// cond + b * cond_ld.  OutT = float: pdae_mlp_mod_ln_act.  OutT = bf16: the next Linear's tensor-core operand, bf16_rn of
// exactly the fp32 value (same reduction order, same expressions).  OutT = Split3: the split of that fp32 value (blk apart).
template <typename OutT>
__global__ void __launch_bounds__(256) mlp_mod_ln_act_kernel(const float* __restrict__ h, const float* __restrict__ cond,
                                                             int cond_ld, const float* __restrict__ lw,
                                                             const float* __restrict__ lb, float eps, int silu,
                                                             const float* __restrict__ mask, float scale,
                                                             OutT* __restrict__ out, int out_ld, int N, int blk) {
  __shared__ float red[2][8];
  const int b = blockIdx.x;
  const float* hr = h + (long long)b * N;
  const float* cr = cond ? cond + (long long)b * cond_ld : nullptr;
  float s = 0.f, q = 0.f;
  for (int j = threadIdx.x; j < N; j += 256) {
    float v = hr[j];
    if (cr) v = v * (1.0f + cr[j]);
    s += v;
    q = fmaf(v, v, q);
  }
  float mean = 0.f, rstd = 1.f;
  if (lw) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = q; }
    __syncthreads();
    double ds = 0.0, dq = 0.0;
    for (int w = 0; w < 8; ++w) { ds += red[0][w]; dq += red[1][w]; }
    const double m = ds / N;
    double var = dq / N - m * m;
    var = var < 0.0 ? 0.0 : var;
    mean = (float)m;
    rstd = (float)(1.0 / sqrt(var + (double)eps));
  }
  for (int j = threadIdx.x; j < N; j += 256) {
    float v = hr[j];
    if (cr) v = v * (1.0f + cr[j]);
    if (lw) v = (v - mean) * rstd * lw[j] + lb[j];
    if (silu) v = silu_f(v);
    if (mask) v *= mask[(long long)b * N + j] * scale;
    store_row(out + (long long)b * out_ld + j, blk, v);
  }
}

template <typename OutT>
__global__ void copy_cols_kernel(const float* __restrict__ src, OutT* __restrict__ dst, int dst_ld, int col0, int B,
                                 int N, int blk) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * N) return;
  const int b = (int)(i / N), j = (int)(i % N);
  store_row(dst + (long long)b * dst_ld + col0 + j, blk, src[i]);
}

}  // namespace pdae

using namespace pdae;

extern "C" const char* pdae_last_error(void) { return g_err; }
extern "C" int pdae_abi_version(void) { return 1; }
extern "C" int pdae_device_check(void) {
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("no CUDA device available");
    return PDAE_ENODEV;
  }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device is sm_%d%d; pdae_b200 is built for sm_90a only", prop.major, prop.minor);
    return PDAE_ENODEV;
  }
  return PDAE_OK;
}

extern "C" int pdae_gn_stats(const float* src1, int C1, const float* src2, int C2, int B, int HW, double* sums,
                             pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && sums, "gn_stats: null pointer");
  if (!src2) C2 = 0;
  const int C = C1 + C2;
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C % 32 == 0 && C > 0, "gn_stats: C1=%d C2=%d unsupported", C1, C2);
  PDAE_REQUIRE((size_t)2 * C * sizeof(float) <= 48 * 1024, "gn_stats: C too large");
  cudaStream_t s = (cudaStream_t)stream;
  PDAE_CUDA(cudaMemsetAsync(sums, 0, (size_t)B * 32 * 2 * sizeof(double), s));
  const int ppc = stats_ppc(B, HW);
  dim3 grid(cdiv(HW, ppc), B);
  gn_stats_kernel<<<grid, 256, 2 * C * sizeof(float), s>>>(src1, C1, src2, C2, HW, sums, ppc);
  PDAE_LAUNCH_CHECK("gn_stats_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_coef(const double* sums, const float* gamma, const float* beta, int B, int C, int HW, float eps,
                            const float* emb, int emb_ld, const float* embz, int embz_ld, float* ab,
                            pdae_stream_t stream) {
  PDAE_REQUIRE(sums && gamma && beta && ab, "gn_coef: null pointer");
  PDAE_REQUIRE(C % 32 == 0, "gn_coef: C %% 32 != 0");
  gn_coef_kernel<<<B, C < 1024 ? C : 1024, 0, (cudaStream_t)stream>>>(sums, gamma, beta, C, HW, eps, emb, emb_ld, embz,
                                                                      embz_ld, ab);
  PDAE_LAUNCH_CHECK("gn_coef_kernel");
  return PDAE_OK;
}

extern "C" int pdae_zero(void* ptr, int64_t bytes, pdae_stream_t stream) {
  PDAE_REQUIRE(ptr && bytes >= 0, "zero: bad args");
  PDAE_CUDA(cudaMemsetAsync(ptr, 0, (size_t)bytes, (cudaStream_t)stream));
  return PDAE_OK;
}

extern "C" int pdae_ch_stats(const float* src, int B, int HW, int C, float* chs, pdae_stream_t stream) {
  PDAE_REQUIRE(src && chs, "ch_stats: null pointer");
  PDAE_REQUIRE(C % 4 == 0 && C > 0 && (size_t)2 * C * sizeof(float) <= 48 * 1024, "ch_stats: C=%d unsupported", C);
  cudaStream_t s = (cudaStream_t)stream;
  PDAE_CUDA(cudaMemsetAsync(chs, 0, (size_t)B * C * 2 * sizeof(float), s));
  const int ppc = stats_ppc(B, HW);
  dim3 grid(cdiv(HW, ppc), B);
  ch_stats_kernel<<<grid, 256, 2 * C * sizeof(float), s>>>(src, C, HW, chs, ppc);
  PDAE_LAUNCH_CHECK("ch_stats_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_coef_ch(const float* chs1, int C1, const float* chs2, int C2, const float* gamma, const float* beta,
                               int B, int HW, float eps, const float* emb, int emb_ld, const float* embz, int embz_ld,
                               float* ab, pdae_stream_t stream) {
  PDAE_REQUIRE(chs1 && gamma && beta && ab, "gn_coef_ch: null pointer");
  if (!chs2) C2 = 0;
  const int C = C1 + C2;
  PDAE_REQUIRE(C % 32 == 0, "gn_coef_ch: C %% 32 != 0");
  gn_coef_ch_kernel<<<B, C < 1024 ? (C < 64 ? 64 : C) : 1024, 0, (cudaStream_t)stream>>>(chs1, C1, chs2, C2, gamma, beta, HW,
                                                                                          eps, emb, emb_ld, embz, embz_ld, ab);
  PDAE_LAUNCH_CHECK("gn_coef_ch_kernel");
  return PDAE_OK;
}

// Deterministic forms of pdae_ch_stats / pdae_gn_stats: per-CTA partials in the caller's workspace, summed in a fixed order.
// An image's CTAs follow HW only (stats_ppc_det), so the workspace is B times one image's slots.
extern "C" int64_t pdae_stats_det_workspace_bytes(int B, int HW, int C) {
  if (B <= 0 || HW <= 0 || C <= 0) {
    ::pdae::set_error("stats_det_workspace_bytes: B=%d HW=%d C=%d must be > 0", B, HW, C);
    return PDAE_EINVAL;
  }
  return (int64_t)B * cdiv(HW, stats_ppc_det(HW)) * C * 2 * (int64_t)sizeof(float);
}

static int launch_ch_parts(const char* fn, const float* src1, int C1, const float* src2, int C2, int B, int HW, float* ws,
                           int64_t ws_bytes, cudaStream_t s, int* P_out) {
  const int C = C1 + C2;
  PDAE_REQUIRE(B > 0 && HW > 0, "%s: B=%d HW=%d must be > 0", fn, B, HW);
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C > 0 && C <= 6144, "%s: C1=%d C2=%d unsupported", fn, C1, C2);
  const int ppc = stats_ppc_det(HW), P = cdiv(HW, ppc);
  const long long need = (long long)B * P * C * 2 * (long long)sizeof(float);
  PDAE_REQUIRE(ws_bytes >= need, "%s: workspace of %lld bytes, %lld needed (pdae_stats_det_workspace_bytes)", fn,
               (long long)ws_bytes, need);
  const int L = C / 4, Lb = L < 256 ? L : 256;
  const size_t smem = (size_t)(256 / Lb) * 2 * C * sizeof(float);
  ch_parts_kernel<<<dim3(P, B), 256, smem, s>>>(src1, C1, src2, C2, HW, ws, ppc);
  PDAE_LAUNCH_CHECK("ch_parts_kernel");
  *P_out = P;
  return PDAE_OK;
}

extern "C" int pdae_ch_stats_det(const float* src, int B, int HW, int C, float* chs, float* workspace, int64_t workspace_bytes,
                                 pdae_stream_t stream) {
  PDAE_REQUIRE(src && chs && workspace, "ch_stats_det: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  int P = 0;
  const int rc = launch_ch_parts("ch_stats_det", src, C, nullptr, 0, B, HW, workspace, workspace_bytes, s, &P);
  if (rc != PDAE_OK) return rc;
  PDAE_CUDA(launch_stat_parts_reduce(workspace, B, P, C, chs, s));
  return PDAE_OK;
}

extern "C" int pdae_gn_stats_det(const float* src1, int C1, const float* src2, int C2, int B, int HW, double* sums,
                                 float* workspace, int64_t workspace_bytes, pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && sums && workspace, "gn_stats_det: null pointer");
  if (!src2) C2 = 0;
  PDAE_REQUIRE((C1 + C2) % 32 == 0, "gn_stats_det: C1=%d C2=%d: C %% 32 != 0", C1, C2);
  cudaStream_t s = (cudaStream_t)stream;
  int P = 0;
  const int rc = launch_ch_parts("gn_stats_det", src1, C1, src2, C2, B, HW, workspace, workspace_bytes, s, &P);
  if (rc != PDAE_OK) return rc;
  gn_group_reduce_kernel<<<B, 256, 0, s>>>(workspace, P, C1 + C2, sums);
  PDAE_LAUNCH_CHECK("gn_group_reduce_kernel");
  return PDAE_OK;
}

template <typename TSrc, typename TSrc2, typename TAct, typename TRaw>
static int launch_apply(const void* s1v, int C1, const void* s2v, int C2, const float* ab, int silu, int resample, int B,
                        int H, int W, void* out_act, void* out_raw, cudaStream_t s) {
  const TSrc* s1 = (const TSrc*)s1v;
  const TSrc2* s2 = (const TSrc2*)s2v;
  const int L = (C1 + C2) / 4;
  const int Hi = resample == PDAE_RESAMPLE_DOWN2 ? H / 2 : H, Wi = resample == PDAE_RESAMPLE_DOWN2 ? W / 2 : W;
  const long long items = (long long)Hi * Wi * L;
  int gx = cdiv(items, 256);
  if (gx > 148 * 16) gx = 148 * 16;
  dim3 grid(gx, B);
  TAct* oa = (TAct*)out_act;
  TRaw* orw = (TRaw*)out_raw;
  if (resample == PDAE_RESAMPLE_NONE)
    gn_apply_kernel<TSrc, TSrc2, TAct, TRaw, PDAE_RESAMPLE_NONE><<<grid, 256, 0, s>>>(s1, C1, s2, C2, ab, silu, H, W, oa, orw);
  else if (resample == PDAE_RESAMPLE_UP2)
    gn_apply_kernel<TSrc, TSrc2, TAct, TRaw, PDAE_RESAMPLE_UP2><<<grid, 256, 0, s>>>(s1, C1, s2, C2, ab, silu, H, W, oa, orw);
  else
    gn_apply_kernel<TSrc, TSrc2, TAct, TRaw, PDAE_RESAMPLE_DOWN2><<<grid, 256, 0, s>>>(s1, C1, s2, C2, ab, silu, H, W, oa, orw);
  PDAE_LAUNCH_CHECK("gn_apply_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_apply(const void* src1, int src1_dtype, int C1, const void* src2, int src2_dtype, int C2,
                             const float* ab, int silu, int resample, int B, int H, int W, void* out_act, int act_dtype,
                             void* out_raw, int raw_dtype, pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && out_act, "gn_apply: null pointer");
  if (!src2) { C2 = 0; src2_dtype = PDAE_F32; }
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C1 + C2 > 0, "gn_apply: C1=%d C2=%d unsupported", C1, C2);
  PDAE_REQUIRE(resample >= 0 && resample <= 2, "gn_apply: bad resample mode");
  PDAE_REQUIRE(resample != PDAE_RESAMPLE_DOWN2 || (H % 2 == 0 && W % 2 == 0), "gn_apply: odd dims for DOWN2");
  if (!out_raw) raw_dtype = (act_dtype == PDAE_BF16 && src1_dtype == PDAE_BF16 && src2_dtype == PDAE_BF16) ? PDAE_BF16 : PDAE_F32;
  // each dtype is one bit of the dispatch key: any other value would alias a different combination
  PDAE_REQUIRE(((unsigned)src1_dtype | (unsigned)src2_dtype | (unsigned)act_dtype | (unsigned)raw_dtype) <= 1u,
               "gn_apply: unsupported dtype combination src1=%d src2=%d act=%d raw=%d", src1_dtype, src2_dtype, act_dtype, raw_dtype);
  cudaStream_t s = (cudaStream_t)stream;
  typedef __nv_bfloat16 bf;
  const int key = src1_dtype | (src2_dtype << 1) | (act_dtype << 2) | (raw_dtype << 3);
  if (resample == PDAE_RESAMPLE_NONE && act_dtype == PDAE_BF16 && C1 % 8 == 0 && C2 % 8 == 0 && (C1 + C2) / 8 <= 256) {
    const int HW = H * W;
    const int L8 = (C1 + C2) / 8;
    const int ppc = 256 / L8;
    const int nthr = L8 * ppc;
    int gx = cdiv(HW, ppc * 8);          // 8 pixels per thread (unrolled x4) keep loads in flight
    if (gx > 148 * 16) gx = 148 * 16;
    if (gx < 1) gx = 1;
    dim3 grid(gx, B);
    bool ok = true;
    switch (key) {
      case 0 | 0 | 4 | 8: gn_apply8_kernel<float, float, bf><<<grid, nthr, 0, s>>>((const float*)src1, C1, (const float*)src2, C2, ab, silu, HW, (bf*)out_act, (bf*)out_raw); break;
      case 0 | 0 | 4 | 0: gn_apply8_kernel<float, float, float><<<grid, nthr, 0, s>>>((const float*)src1, C1, (const float*)src2, C2, ab, silu, HW, (bf*)out_act, (float*)out_raw); break;
      case 1 | 0 | 4 | 0: gn_apply8_kernel<bf, float, float><<<grid, nthr, 0, s>>>((const bf*)src1, C1, (const float*)src2, C2, ab, silu, HW, (bf*)out_act, (float*)out_raw); break;
      case 1 | 2 | 4 | 8: gn_apply8_kernel<bf, bf, bf><<<grid, nthr, 0, s>>>((const bf*)src1, C1, (const bf*)src2, C2, ab, silu, HW, (bf*)out_act, (bf*)out_raw); break;
      case 1 | 0 | 4 | 8: gn_apply8_kernel<bf, float, bf><<<grid, nthr, 0, s>>>((const bf*)src1, C1, (const float*)src2, C2, ab, silu, HW, (bf*)out_act, (bf*)out_raw); break;
      case 0 | 2 | 4 | 0: gn_apply8_kernel<float, bf, float><<<grid, nthr, 0, s>>>((const float*)src1, C1, (const bf*)src2, C2, ab, silu, HW, (bf*)out_act, (float*)out_raw); break;
      case 0 | 2 | 4 | 8: gn_apply8_kernel<float, bf, bf><<<grid, nthr, 0, s>>>((const float*)src1, C1, (const bf*)src2, C2, ab, silu, HW, (bf*)out_act, (bf*)out_raw); break;
      case 1 | 2 | 4 | 0: gn_apply8_kernel<bf, bf, float><<<grid, nthr, 0, s>>>((const bf*)src1, C1, (const bf*)src2, C2, ab, silu, HW, (bf*)out_act, (float*)out_raw); break;
      default: ok = false;
    }
    if (ok) {
      PDAE_LAUNCH_CHECK("gn_apply8_kernel");
      return PDAE_OK;
    }
  }
  switch (key) {
    case 0 | 0 | 0 | 0: return launch_apply<float, float, float, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 0 | 0 | 4 | 0: return launch_apply<float, float, bf, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 0 | 0 | 4 | 8: return launch_apply<float, float, bf, bf>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 1 | 0 | 4 | 0: return launch_apply<bf, float, bf, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 1 | 2 | 4 | 8: return launch_apply<bf, bf, bf, bf>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 1 | 0 | 4 | 8: return launch_apply<bf, float, bf, bf>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 0 | 2 | 4 | 0: return launch_apply<float, bf, bf, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 0 | 2 | 4 | 8: return launch_apply<float, bf, bf, bf>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 1 | 2 | 4 | 0: return launch_apply<bf, bf, bf, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    // a bf16-stream tensor feeding a CUDA-core (fp32) conv
    case 1 | 0 | 0 | 0: return launch_apply<bf, float, float, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 1 | 2 | 0 | 0: return launch_apply<bf, bf, float, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    case 0 | 2 | 0 | 0: return launch_apply<float, bf, float, float>(src1, C1, src2, C2, ab, silu, resample, B, H, W, out_act, out_raw, s);
    default: break;
  }
  PDAE_REQUIRE(false, "gn_apply: unsupported dtype combination src1=%d src2=%d act=%d raw=%d", src1_dtype, src2_dtype, act_dtype,
               raw_dtype);
}

extern "C" int pdae_gn_apply_split3(const float* src1, int C1, const float* src2, int C2, const float* ab, int silu, int resample,
                                    int B, int H, int W, void* out_act3_bf16, void* out_raw, int raw_dtype,
                                    pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && out_act3_bf16, "gn_apply_split3: null pointer");
  if (!src2) C2 = 0;
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C1 + C2 > 0, "gn_apply_split3: C1=%d C2=%d unsupported", C1, C2);
  PDAE_REQUIRE(resample >= 0 && resample <= 2, "gn_apply_split3: bad resample mode");
  PDAE_REQUIRE(resample != PDAE_RESAMPLE_DOWN2 || (H % 2 == 0 && W % 2 == 0), "gn_apply_split3: odd dims for DOWN2");
  const int Hi = resample == PDAE_RESAMPLE_DOWN2 ? H / 2 : H, Wi = resample == PDAE_RESAMPLE_DOWN2 ? W / 2 : W;
  const long long items = (long long)Hi * Wi * ((C1 + C2) / 4);
  int gx = cdiv(items, 256);
  if (gx > 148 * 16) gx = 148 * 16;
  dim3 grid(gx, B);
  cudaStream_t s = (cudaStream_t)stream;
  typedef __nv_bfloat16 bf;
  bf* oa = (bf*)out_act3_bf16;
  const bool rs_bf = out_raw && raw_dtype == PDAE_BF16;
#define PDAE_SPLIT3(RS)                                                                                                   \
  do {                                                                                                                     \
    if (rs_bf) gn_apply_split3_kernel<bf, RS><<<grid, 256, 0, s>>>(src1, C1, src2, C2, ab, silu, H, W, oa, (bf*)out_raw);   \
    else gn_apply_split3_kernel<float, RS><<<grid, 256, 0, s>>>(src1, C1, src2, C2, ab, silu, H, W, oa, (float*)out_raw);   \
  } while (0)
  if (resample == PDAE_RESAMPLE_NONE) PDAE_SPLIT3(PDAE_RESAMPLE_NONE);
  else if (resample == PDAE_RESAMPLE_UP2) PDAE_SPLIT3(PDAE_RESAMPLE_UP2);
  else PDAE_SPLIT3(PDAE_RESAMPLE_DOWN2);
#undef PDAE_SPLIT3
  PDAE_LAUNCH_CHECK("gn_apply_split3_kernel");
  return PDAE_OK;
}

extern "C" int pdae_timestep_embedding(const int64_t* t, int B, int dim, const float* freqs, float* out,
                                       pdae_stream_t stream) {
  PDAE_REQUIRE(t && out && freqs && B > 0 && dim > 0, "timestep_embedding: bad args");
  timestep_embedding_kernel<<<cdiv((long long)B * dim, 256), 256, 0, (cudaStream_t)stream>>>(t, B, dim, freqs, out);
  PDAE_LAUNCH_CHECK("timestep_embedding_kernel");
  return PDAE_OK;
}

extern "C" int pdae_embedding_add(float* emb, const float* table, const int64_t* idx, int B, int E,
                                  pdae_stream_t stream) {
  PDAE_REQUIRE(emb && table && idx, "embedding_add: null pointer");
  embedding_add_kernel<<<cdiv((long long)B * E, 256), 256, 0, (cudaStream_t)stream>>>(emb, table, idx, B, E);
  PDAE_LAUNCH_CHECK("embedding_add_kernel");
  return PDAE_OK;
}

static inline int ew_grid(long long total) {
  int g = cdiv(total, 256);
  return g > 148 * 16 ? 148 * 16 : g;
}

extern "C" int pdae_ddim_step(const float* x, const float* eps, const float* grad, const int64_t* t, const float* tab_A,
                              const float* tab_Bm, const float* tab_s1m, const float* tab_ab, float* out, int B,
                              int64_t per_sample, pdae_stream_t stream) {
  PDAE_REQUIRE(x && eps && t && tab_A && tab_Bm && tab_ab && out, "ddim_step: null pointer");
  PDAE_REQUIRE(!grad || tab_s1m, "ddim_step: grad given without sqrt_one_minus_alphas_cumprod table");
  const long long total = (long long)B * per_sample;
  ddim_step_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(x, eps, grad, t, tab_A, tab_Bm, tab_s1m, tab_ab, out,
                                                                    per_sample, total);
  PDAE_LAUNCH_CHECK("ddim_step_kernel");
  return PDAE_OK;
}

extern "C" int pdae_ddim_select_t(int64_t* counter, int delta, const int64_t* timestep_map, int map_len, int64_t* t_loc,
                                  int64_t* t_net, int B, pdae_stream_t stream) {
  PDAE_REQUIRE(counter && timestep_map && t_loc && t_net && map_len > 0 && B > 0, "ddim_select_t: bad args");
  ddim_select_t_kernel<<<1, 256, 0, (cudaStream_t)stream>>>((long long*)counter, delta, timestep_map, map_len, t_loc, t_net, B);
  PDAE_LAUNCH_CHECK("ddim_select_t_kernel");
  return PDAE_OK;
}

extern "C" int pdae_q_sample(const float* x0, const float* noise, const int64_t* t, const float* tab_c1,
                             const float* tab_c2, float* out, int B, int64_t per_sample, pdae_stream_t stream) {
  PDAE_REQUIRE(x0 && noise && t && tab_c1 && tab_c2 && out, "q_sample: null pointer");
  const long long total = (long long)B * per_sample;
  q_sample_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(x0, noise, t, tab_c1, tab_c2, out, per_sample, total);
  PDAE_LAUNCH_CHECK("q_sample_kernel");
  return PDAE_OK;
}

extern "C" int pdae_noise_p_sample(const float* x, const float* eps, const float* noise, const float* learned_range,
                                   const int64_t* t, const float* tab_cx, const float* tab_ce, const float* tab_logvar,
                                   const float* tab_logbeta, float* out, int B, int64_t per_sample,
                                   pdae_stream_t stream) {
  PDAE_REQUIRE(x && eps && noise && t && tab_cx && tab_ce && tab_logvar && out, "noise_p_sample: null pointer");
  PDAE_REQUIRE(!learned_range || tab_logbeta, "noise_p_sample: learned_range needs log(betas)");
  const long long total = (long long)B * per_sample;
  noise_p_sample_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(x, eps, noise, learned_range, t, tab_cx, tab_ce,
                                                                         tab_logvar, tab_logbeta, out, per_sample, total);
  PDAE_LAUNCH_CHECK("noise_p_sample_kernel");
  return PDAE_OK;
}

extern "C" int pdae_noise_p_sample_shift(const float* x, const float* eps, const float* grad, const float* tab_shift,
                                         const float* noise, const float* learned_range, int64_t eps_ld, const int64_t* t,
                                         const float* tab_cx, const float* tab_ce, const float* tab_logvar,
                                         const float* tab_logbeta, float* out, int B, int64_t per_sample,
                                         pdae_stream_t stream) {
  PDAE_REQUIRE(x && eps && noise && t && tab_cx && tab_ce && tab_logvar && out, "noise_p_sample_shift: null pointer");
  PDAE_REQUIRE(!grad || tab_shift, "noise_p_sample_shift: grad given without shift_coef table");
  PDAE_REQUIRE(!learned_range || tab_logbeta, "noise_p_sample_shift: learned_range needs log(betas)");
  PDAE_REQUIRE(eps_ld >= per_sample, "noise_p_sample_shift: eps_ld < per_sample");
  const long long total = (long long)B * per_sample;
  noise_p_sample_shift_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(
      x, eps, grad, tab_shift, noise, learned_range, eps_ld, t, tab_cx, tab_ce, tab_logvar, tab_logbeta, out, per_sample, total);
  PDAE_LAUNCH_CHECK("noise_p_sample_shift_kernel");
  return PDAE_OK;
}

extern "C" int pdae_grad_blend(const float* g1, const float* g2, const float* ab, float* out, int64_t n, pdae_stream_t stream) {
  PDAE_REQUIRE(g1 && g2 && ab && out && n > 0, "grad_blend: bad args");
  grad_blend_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(g1, g2, ab, out, n);
  PDAE_LAUNCH_CHECK("grad_blend_kernel");
  return PDAE_OK;
}

static inline long long gap_blocks(long long total) { return (total + GAP_PER_BLOCK - 1) / GAP_PER_BLOCK; }

extern "C" int64_t pdae_gap_terms_workspace_bytes(int64_t total) {
  if (total <= 0) {
    ::pdae::set_error("gap_terms_workspace_bytes: total=%lld must be > 0", (long long)total);
    return PDAE_EINVAL;
  }
  return gap_blocks(total) * 2 * (int64_t)sizeof(double);
}

extern "C" int pdae_gap_terms(const float* x0, const float* x_t, const float* eps, const float* grad, const int64_t* t,
                              const float* tab_c0, const float* tab_c1, const float* tab_A, const float* tab_Bm,
                              const float* tab_shift, double* workspace, int64_t workspace_bytes, float* out, int B,
                              int64_t per_sample, pdae_stream_t stream) {
  PDAE_REQUIRE(x0 && x_t && eps && grad && t && tab_c0 && tab_c1 && tab_A && tab_Bm && tab_shift && workspace && out,
               "gap_terms: null pointer");
  PDAE_REQUIRE(B > 0 && per_sample > 0, "gap_terms: B=%d and per_sample=%lld must be > 0", B, (long long)per_sample);
  const long long total = (long long)B * per_sample;
  const long long nblk = gap_blocks(total);
  PDAE_REQUIRE(nblk <= 0x7fffffffLL, "gap_terms: %lld elements are too many", total);
  PDAE_REQUIRE(workspace_bytes >= nblk * 2 * (long long)sizeof(double),
               "gap_terms: workspace of %lld bytes, %lld needed (pdae_gap_terms_workspace_bytes)", (long long)workspace_bytes,
               nblk * 2 * (long long)sizeof(double));
  cudaStream_t s = (cudaStream_t)stream;
  gap_terms_partial_kernel<<<(unsigned)nblk, GAP_THREADS, 0, s>>>(x0, x_t, eps, grad, t, tab_c0, tab_c1, tab_A, tab_Bm,
                                                                  tab_shift, workspace, per_sample, total);
  PDAE_LAUNCH_CHECK("gap_terms_partial_kernel");
  gap_terms_final_kernel<<<1, GAP_THREADS, 0, s>>>(workspace, (int)nblk, t, out, (double)total);
  PDAE_LAUNCH_CHECK("gap_terms_final_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mlp_mod_ln_act(const float* h, const float* cond, const float* ln_w, const float* ln_b, float eps,
                                   int silu, float* out, int out_ld, int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(h && out && B > 0 && N > 0 && out_ld >= N, "mlp_mod_ln_act: bad args");
  PDAE_REQUIRE(!ln_w || ln_b, "mlp_mod_ln_act: LayerNorm weight without bias");
  mlp_mod_ln_act_kernel<float><<<B, 256, 0, (cudaStream_t)stream>>>(h, cond, N, ln_w, ln_b, eps, silu, nullptr, 1.0f, out,
                                                                    out_ld, N, 0);
  PDAE_LAUNCH_CHECK("mlp_mod_ln_act_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mlp_mod_ln_act_bf16(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b,
                                        float eps, int silu, const float* mask, float mask_scale, void* out_bf16, int out_ld,
                                        int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(h && out_bf16 && B > 0 && N > 0 && out_ld >= N && (!cond || cond_ld >= N), "mlp_mod_ln_act_bf16: bad args");
  PDAE_REQUIRE(!ln_w || ln_b, "mlp_mod_ln_act_bf16: LayerNorm weight without bias");
  mlp_mod_ln_act_kernel<__nv_bfloat16><<<B, 256, 0, (cudaStream_t)stream>>>(h, cond, cond_ld, ln_w, ln_b, eps, silu, mask,
                                                                            mask_scale, (__nv_bfloat16*)out_bf16, out_ld, N, 0);
  PDAE_LAUNCH_CHECK("mlp_mod_ln_act_kernel<bf16>");
  return PDAE_OK;
}

extern "C" int pdae_mlp_mod_ln_act_split3(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b,
                                          float eps, int silu, void* out_split3, int ld, int col0, int B, int N,
                                          pdae_stream_t stream) {
  PDAE_REQUIRE(h && out_split3 && B > 0 && N > 0 && col0 >= 0 && col0 + N <= ld && (!cond || cond_ld == 0 || cond_ld >= N),
               "mlp_mod_ln_act_split3: bad args (B=%d N=%d ld=%d col0=%d cond_ld=%d)", B, N, ld, col0, cond_ld);
  PDAE_REQUIRE(!ln_w || ln_b, "mlp_mod_ln_act_split3: LayerNorm weight without bias");
  mlp_mod_ln_act_kernel<Split3><<<B, 256, 0, (cudaStream_t)stream>>>(h, cond, cond_ld, ln_w, ln_b, eps, silu, nullptr, 1.0f,
                                                                     (Split3*)out_split3 + col0, 3 * ld, N, ld);
  PDAE_LAUNCH_CHECK("mlp_mod_ln_act_kernel<split3>");
  return PDAE_OK;
}

extern "C" int pdae_copy_cols(const float* src, float* dst, int dst_ld, int col0, int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(src && dst && col0 >= 0 && col0 + N <= dst_ld, "copy_cols: bad args");
  copy_cols_kernel<float><<<cdiv((long long)B * N, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, dst_ld, col0, B, N, 0);
  PDAE_LAUNCH_CHECK("copy_cols_kernel");
  return PDAE_OK;
}

extern "C" int pdae_copy_cols_bf16(const float* src, void* dst_bf16, int dst_ld, int col0, int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(src && dst_bf16 && B > 0 && N > 0 && col0 >= 0 && col0 + N <= dst_ld, "copy_cols_bf16: bad args");
  copy_cols_kernel<__nv_bfloat16><<<cdiv((long long)B * N, 256), 256, 0, (cudaStream_t)stream>>>(
      src, (__nv_bfloat16*)dst_bf16, dst_ld, col0, B, N, 0);
  PDAE_LAUNCH_CHECK("copy_cols_kernel<bf16>");
  return PDAE_OK;
}

extern "C" int pdae_copy_cols_split3(const float* src, void* dst_split3, int ld, int col0, int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(src && dst_split3 && B > 0 && N > 0 && col0 >= 0 && col0 + N <= ld,
               "copy_cols_split3: bad args (B=%d N=%d ld=%d col0=%d)", B, N, ld, col0);
  copy_cols_kernel<Split3><<<cdiv((long long)B * N, 256), 256, 0, (cudaStream_t)stream>>>(src, (Split3*)dst_split3, 3 * ld,
                                                                                         col0, B, N, ld);
  PDAE_LAUNCH_CHECK("copy_cols_kernel<split3>");
  return PDAE_OK;
}
