// Backward kernels (training config: shift half of the ShiftUNet + semantic encoder + plain UNet), fp32 CUDA-core math.
//   conv dgrad / wgrad (implicit GEMM, any k / stride / pad), column sums (bias grads),
//   GroupNorm(+AdaGN)+SiLU(+nearest-up / avg-pool) backward in three passes, softmax backward, SiLU' helpers.
// Reference: autograd through model/module.py:278-297,361-384,422-428 and the encoders.
#include "common.cuh"

namespace pdae {

constexpr int DBM = 64, DBN = 64, DBK = 16;

struct DgradArgs {
  const float* dy; const float* w; float* dx;
  int B, H, W, Cin, Cout, Ho, Wo, ksize, stride, pad, accumulate;
  long long M; int K;
};

// dx[b,y,x,ci] (+)= sum_{ky,kx,co} dy[b,(y+pad-ky)/s,(x+pad-kx)/s,co] * w[tap][co][ci]   (terms with non-integer / OOB coords vanish)
__global__ void __launch_bounds__(256) conv_dgrad_kernel(DgradArgs p) {
  __shared__ __align__(16) float As[DBK][DBM + 4];
  __shared__ __align__(16) float Bs[DBK][DBN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * DBM;
  const int n0 = blockIdx.y * DBN;
  const int a_row = tid & 63, a_k = tid >> 6;
  const long long am = m0 + a_row;
  const bool a_valid = am < p.M;
  int ab = 0, ay = 0, ax = 0;
  if (a_valid) {
    long long r = am;
    ax = (int)(r % p.W); r /= p.W;
    ay = (int)(r % p.H);
    ab = (int)(r / p.H);
  }
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += DBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int kl = a_k + 4 * i, kk = k0 + kl;
      float v = 0.f;
      if (a_valid && kk < p.K) {
        const int tap = kk / p.Cout, co = kk - tap * p.Cout;
        const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
        const int ty_ = ay + p.pad - ky, tx_ = ax + p.pad - kx;
        if (ty_ >= 0 && tx_ >= 0 && ty_ % p.stride == 0 && tx_ % p.stride == 0) {
          const int oy = ty_ / p.stride, ox = tx_ / p.stride;
          if (oy < p.Ho && ox < p.Wo) v = p.dy[(((long long)ab * p.Ho + oy) * p.Wo + ox) * p.Cout + co];
        }
      }
      As[kl][a_row] = v;
    }
    {
      const int kk = k0 + b_k;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kk < p.K) {
        const float* wp = p.w + (long long)kk * p.Cin + n0 + b_n;  // w[tap][co][ci], kk = tap*Cout + co
        if (n0 + b_n + 0 < p.Cin) v.x = wp[0];
        if (n0 + b_n + 1 < p.Cin) v.y = wp[1];
        if (n0 + b_n + 2 < p.Cin) v.z = wp[2];
        if (n0 + b_n + 3 < p.Cin) v.w = wp[3];
      }
      *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DBK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.Cin) continue;
      float* o = p.dx + m * p.Cin + n;
      *o = p.accumulate ? *o + acc[i][j] : acc[i][j];
    }
  }
}

struct WgradArgs {
  const float* x; const float* dy; float* dw;
  int B, H, W, Cin, Cout, Ho, Wo, ksize, stride, pad, in_nchw, a_silu;
  long long P;   // output pixels = reduction length
  int MK;        // taps*Cin rows of dw
  int chunk;     // pixels per split-K slice
};

// dw[tap*Cin+ci][co] += sum_{pixels} f(x[b, oy*s-p+ky, ox*s-p+kx, ci]) * dy[pixel][co]    (split over pixel chunks, atomics)
// DET: pixel chunk z stores its partial into slot z of p.dw ([chunks][MK][Cout]); the slots are summed in order afterwards
template <bool DET>
__global__ void __launch_bounds__(256) conv_wgrad_kernel(WgradArgs p) {
  __shared__ __align__(16) float As[DBK][DBM + 4];   // [pixel][row of dw]
  __shared__ __align__(16) float Bs[DBK][DBN];       // [pixel][co]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int r0 = blockIdx.x * DBM, n0 = blockIdx.y * DBN;
  const long long p0 = (long long)blockIdx.z * p.chunk;
  const long long p1 = min(p.P, p0 + p.chunk);
  // A-load role: thread -> row (tid % 64), pixel offsets (tid / 64) + 4*i
  const int a_r = tid & 63, a_p = tid >> 6;
  const int row = r0 + a_r;
  const bool row_ok = row < p.MK;
  int tap = 0, ci = 0, ky = 0, kx = 0;
  if (row_ok) { tap = row / p.Cin; ci = row - tap * p.Cin; ky = tap / p.ksize; kx = tap - ky * p.ksize; }
  const int b_p = tid >> 4, b_n = (tid & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long pk = p0; pk < p1; pk += DBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int pl = a_p + 4 * i;
      const long long pix = pk + pl;
      float v = 0.f;
      if (row_ok && pix < p1) {
        long long r = pix;
        const int ox = (int)(r % p.Wo); r /= p.Wo;
        const int oy = (int)(r % p.Ho);
        const int b = (int)(r / p.Ho);
        const int iy = oy * p.stride - p.pad + ky, ix = ox * p.stride - p.pad + kx;
        if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
          const long long off = p.in_nchw ? ((((long long)b * p.Cin + ci) * p.H + iy) * p.W + ix)
                                          : ((((long long)b * p.H + iy) * p.W + ix) * p.Cin + ci);
          v = p.x[off];
          if (p.a_silu) v = silu_f(v);
        }
      }
      As[pl][a_r] = v;
    }
    {
      const long long pix = pk + b_p;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (pix < p1) {
        const float* dp = p.dy + pix * p.Cout + n0 + b_n;
        if (n0 + b_n + 0 < p.Cout) v.x = dp[0];
        if (n0 + b_n + 1 < p.Cout) v.y = dp[1];
        if (n0 + b_n + 2 < p.Cout) v.z = dp[2];
        if (n0 + b_n + 3 < p.Cout) v.w = dp[3];
      }
      *reinterpret_cast<float4*>(&Bs[b_p][b_n]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DBK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty * 4 + i;
    if (r >= p.MK) continue;
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.Cout) continue;
      if constexpr (DET) p.dw[((long long)blockIdx.z * p.MK + r) * p.Cout + n] = acc[i][j];
      else atomicAdd(p.dw + (long long)r * p.Cout + n, acc[i][j]);
    }
  }
}

// out[n] += sum_m dy[m][n]   (DET: row chunk x stores its sums into slot x of out, [chunks][N])
template <bool DET>
__global__ void colsum_kernel(const float* __restrict__ dy, long long M, int N, float* __restrict__ out, int rows_per_cta) {
  const long long m0 = (long long)blockIdx.x * rows_per_cta, m1 = min(M, m0 + rows_per_cta);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float s = 0.f;
    for (long long m = m0; m < m1; ++m) s += dy[m * N + n];
    if constexpr (DET) out[(long long)blockIdx.x * N + n] = s;
    else atomicAdd(out + n, s);
  }
}

// N % 4 == 0: a warp reads 32 float4 columns (512 contiguous bytes) of one row, the 8 warps of a CTA take interleaved rows
// (four independent loads in flight per thread), partial sums meet in shared memory, one fp32 reduction per column and CTA
// (DET: one plain store per column into the CTA's slot of out, [chunks][N])
template <bool DET>
__global__ void __launch_bounds__(256) colsum_v4_kernel(const float* __restrict__ dy, long long M, int N, float* __restrict__ out,
                                                        int rows_per_cta) {
  __shared__ float4 part[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nv = N >> 2;
  const long long m0 = (long long)blockIdx.x * rows_per_cta, m1 = min(M, m0 + rows_per_cta);
  const float4* src = reinterpret_cast<const float4*>(dy);
  for (int cb = 0; cb < nv; cb += 32) {
    const int cv = cb + lane;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cv < nv) {
      long long m = m0 + w;
      for (; m + 24 < m1; m += 32) {
        const float4 a = src[m * nv + cv], b = src[(m + 8) * nv + cv], c = src[(m + 16) * nv + cv], d = src[(m + 24) * nv + cv];
        s.x += (a.x + b.x) + (c.x + d.x); s.y += (a.y + b.y) + (c.y + d.y);
        s.z += (a.z + b.z) + (c.z + d.z); s.w += (a.w + b.w) + (c.w + d.w);
      }
      for (; m < m1; m += 8) {
        const float4 a = src[m * nv + cv];
        s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
      }
    }
    part[w][lane] = s;
    __syncthreads();
    if (w == 0 && cv < nv) {
#pragma unroll
      for (int i = 1; i < 8; ++i) {
        const float4 t = part[i][lane];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      if constexpr (DET) {
        float* o = out + (long long)blockIdx.x * N + 4 * cv;
        o[0] = s.x; o[1] = s.y; o[2] = s.z; o[3] = s.w;
      } else {
        float* o = out + 4 * cv;
        atomicAdd(o, s.x); atomicAdd(o + 1, s.y); atomicAdd(o + 2, s.z); atomicAdd(o + 3, s.w);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm(+AdaGN)+SiLU(+resample) backward.  Forward: y = R( f(a*x + b) ), f = SiLU or id, R = none / nearest-up2 / avg-pool2.
// pass 1: per (b,c):  S1 = sum du,  S2 = sum du * x   with du = f'(u) * R^T(dy)
template <int RS>
__device__ __forceinline__ float4 gather_dy(const float* __restrict__ dy, int b, int y, int x, int H, int W, int C, int c) {
  if (RS == PDAE_RESAMPLE_NONE) {
    return *reinterpret_cast<const float4*>(dy + (((long long)b * H + y) * W + x) * C + c);
  } else if (RS == PDAE_RESAMPLE_UP2) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int dy_ = 0; dy_ < 2; ++dy_)
#pragma unroll
      for (int dx_ = 0; dx_ < 2; ++dx_) {
        const float4 v = *reinterpret_cast<const float4*>(dy + (((long long)b * 2 * H + 2 * y + dy_) * 2 * W + 2 * x + dx_) * C + c);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    return s;
  } else {
    const float4 v = *reinterpret_cast<const float4*>(dy + (((long long)b * (H / 2) + y / 2) * (W / 2) + x / 2) * C + c);
    return make_float4(0.25f * v.x, 0.25f * v.y, 0.25f * v.z, 0.25f * v.w);
  }
}
__device__ __forceinline__ float dsilu(float u) {
  const float s = 1.0f / (1.0f + expf(-u));
  return s * (1.0f + u * (1.0f - s));
}

// DET: the pixel rows of a CTA keep their own shared sums ([R][2][C], no shared atomics), added in row order; the CTA stores
// them into its slot S[b][blockIdx.x][C][2], and stat_parts_reduce sums the slots in order (the ch_parts_kernel pattern).
template <int RS, bool DET>
__global__ void __launch_bounds__(256) gn_bwd_sums_kernel(const float* __restrict__ s1, int C1, const float* __restrict__ s2,
                                                          int C2, const float* __restrict__ ab, const float* __restrict__ dy,
                                                          int silu, int H, int W, float* __restrict__ S, int ppc) {
  extern __shared__ float sh[];  // [2][C]; DET: [R][2][C]
  const int C = C1 + C2, L = C >> 2;
  const int Lb = L < 256 ? L : 256, R = 256 / Lb;
  const int tid = threadIdx.x, lane = tid % Lb, row = tid / Lb;
  const int b = blockIdx.y;
  const int HW = H * W;
  const int p0 = blockIdx.x * ppc, p1 = min(HW, p0 + ppc);     // ppc pixels per CTA (host: enough CTAs to fill the SMs)
  if (!DET) {
    for (int i = tid; i < 2 * C; i += 256) sh[i] = 0.f;
    __syncthreads();
  }
  if (row < R) {
    for (int cq = lane; cq < L; cq += Lb) {
      const int c = cq * 4;
      const float* base; int cs, cc;
      if (c < C1) { base = s1; cs = C1; cc = c; } else { base = s2; cs = C2; cc = c - C1; }
      base += (long long)b * HW * cs + cc;
      const float4 a = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 0) * C + c);
      const float4 bb = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 1) * C + c);
      float4 t1 = make_float4(0.f, 0.f, 0.f, 0.f), t2 = t1;
      for (int pix = p0 + row; pix < p1; pix += R) {
        const int y = pix / W, x = pix - y * W;
        const float4 xv = *reinterpret_cast<const float4*>(base + (long long)pix * cs);
        float4 g = gather_dy<RS>(dy, b, y, x, H, W, C, c);
        if (silu) {
          g.x *= dsilu(fmaf(a.x, xv.x, bb.x)); g.y *= dsilu(fmaf(a.y, xv.y, bb.y));
          g.z *= dsilu(fmaf(a.z, xv.z, bb.z)); g.w *= dsilu(fmaf(a.w, xv.w, bb.w));
        }
        t1.x += g.x; t1.y += g.y; t1.z += g.z; t1.w += g.w;
        t2.x = fmaf(g.x, xv.x, t2.x); t2.y = fmaf(g.y, xv.y, t2.y); t2.z = fmaf(g.z, xv.z, t2.z); t2.w = fmaf(g.w, xv.w, t2.w);
      }
      if constexpr (DET) {
        *reinterpret_cast<float4*>(sh + (size_t)row * 2 * C + c) = t1;
        *reinterpret_cast<float4*>(sh + (size_t)row * 2 * C + C + c) = t2;
      } else {
        atomicAdd(&sh[c + 0], t1.x); atomicAdd(&sh[c + 1], t1.y); atomicAdd(&sh[c + 2], t1.z); atomicAdd(&sh[c + 3], t1.w);
        atomicAdd(&sh[C + c + 0], t2.x); atomicAdd(&sh[C + c + 1], t2.y); atomicAdd(&sh[C + c + 2], t2.z); atomicAdd(&sh[C + c + 3], t2.w);
      }
    }
  }
  __syncthreads();
  if constexpr (DET) {
    for (int c = tid; c < C; c += 256) {
      float a = 0.f, q = 0.f;
      for (int r = 0; r < R; ++r) {
        a += sh[(size_t)r * 2 * C + c];
        q += sh[(size_t)r * 2 * C + C + c];
      }
      *reinterpret_cast<float2*>(S + (((long long)b * gridDim.x + blockIdx.x) * C + c) * 2) = make_float2(a, q);
    }
  } else {
    for (int c = tid; c < C; c += 256) {
      atomicAdd(&S[((long long)b * C + c) * 2 + 0], sh[c]);
      atomicAdd(&S[((long long)b * C + c) * 2 + 1], sh[C + c]);
    }
  }
}

// pass 2 (tiny): from S1,S2, the forward statistics and the modulation rows produce
//   k[b][0][c] = gt*rstd (dx = k*du - (cA + x*cB) ...), per-group cA, cB folded per channel into kk[b][1..2][c],
//   gradients of gamma/beta (atomics over b) and of the (scale|shift) rows of emb / embz.
// DET: the per-channel terms of the group sums sit in shared memory ([2][C] doubles) and one thread per group adds them in
// channel order; dgamma / dbeta point at per-image slots [B][C], which gn_param_reduce_kernel sums over b in order.
template <bool DET>
__global__ void gn_bwd_coef_kernel(const float* __restrict__ S, const double* __restrict__ sums, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, const float* __restrict__ emb, int emb_ld,
                                   const float* __restrict__ embz, int embz_ld, int C, int HW, float eps,
                                   float* __restrict__ kk, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                   float* __restrict__ demb, int demb_ld, float* __restrict__ dembz, int dembz_ld) {
  __shared__ double gA[32], gB[32];
  extern __shared__ double terms[];   // DET: [2][C]
  const int b = blockIdx.x;
  const int cpg = C / 32;
  const double n = (double)HW * cpg;
  if (!DET && threadIdx.x < 32) { gA[threadIdx.x] = 0.0; gB[threadIdx.x] = 0.0; }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mean = sums[((long long)b * 32 + g) * 2] / n;
    double var = sums[((long long)b * 32 + g) * 2 + 1] / n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const double rstd = 1.0 / sqrt(var + (double)eps);
    const float s = emb ? 1.0f + emb[(long long)b * emb_ld + c] : 1.0f;
    const float sh = emb ? emb[(long long)b * emb_ld + C + c] : 0.0f;
    const float zs = embz ? 1.0f + embz[(long long)b * embz_ld + c] : 1.0f;
    const float gt = gamma[c] * s * zs;                      // effective gain
    const double S1 = S[((long long)b * C + c) * 2], S2 = S[((long long)b * C + c) * 2 + 1];
    const double dbt = S1;                                   // d beta~  = sum du
    const double dgt = rstd * (S2 - mean * S1);              // d gamma~ = sum du * xhat
    // parameter / modulation gradients
    if constexpr (DET) {
      terms[c] = (double)gt * dbt;
      terms[C + c] = (double)gt * dgt;
      if (dgamma) dgamma[(long long)b * C + c] = (float)(dgt * s * zs);
      if (dbeta) dbeta[(long long)b * C + c] = (float)(dbt * s * zs);
    } else {
      atomicAdd(&gA[g], (double)gt * dbt);
      atomicAdd(&gB[g], (double)gt * dgt);
      if (dgamma) atomicAdd(dgamma + c, (float)(dgt * s * zs));
      if (dbeta) atomicAdd(dbeta + c, (float)(dbt * s * zs));
    }
    if (demb) {
      demb[(long long)b * demb_ld + c] = (float)((dgt * gamma[c] + dbt * beta[c]) * zs);
      demb[(long long)b * demb_ld + C + c] = (float)(dbt * zs);
    }
    if (dembz) {
      dembz[(long long)b * dembz_ld + c] = (float)(dgt * gamma[c] * s + dbt * (beta[c] * s + sh));
      dembz[(long long)b * dembz_ld + C + c] = (float)dbt;
    }
  }
  __syncthreads();
  if constexpr (DET) {
    if (threadIdx.x < 32) {
      double a = 0.0, q = 0.0;
      for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) { a += terms[c]; q += terms[C + c]; }
      gA[threadIdx.x] = a;
      gB[threadIdx.x] = q;
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mean = sums[((long long)b * 32 + g) * 2] / n;
    double var = sums[((long long)b * 32 + g) * 2 + 1] / n - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    const double rstd = 1.0 / sqrt(var + (double)eps);
    const float s = emb ? 1.0f + emb[(long long)b * emb_ld + c] : 1.0f;
    const float zs = embz ? 1.0f + embz[(long long)b * embz_ld + c] : 1.0f;
    const float gt = gamma[c] * s * zs;
    // dx = rstd*( gt*du - (1/n)*( gA + xhat*gB ) ),  xhat = (x-mean)*rstd   ==  k0*du + k1*x + k2
    const double k1 = -rstd * rstd * gB[g] / n;
    kk[((long long)b * 3 + 0) * C + c] = (float)(rstd * gt);
    kk[((long long)b * 3 + 1) * C + c] = (float)k1;
    kk[((long long)b * 3 + 2) * C + c] = (float)(-rstd * gA[g] / n - k1 * mean);
  }
}

// pass 3: dx = k0*du + k1*x + k2 (+ R^T(add)), du recomputed.  Channels c < C1 go to dx1 [B,H,W,C1]; channels of the second
// (skip) source go to dx2 [B,H,W,C2] when requested (full-UNet training needs the gradient of the skip tensors too).
template <int RS>
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const float* __restrict__ s1, int C1, const float* __restrict__ s2,
                                                           int C2, const float* __restrict__ ab, const float* __restrict__ kk,
                                                           const float* __restrict__ dy, int silu, int H, int W,
                                                           const float* __restrict__ add, int add_ld, float* __restrict__ dx1,
                                                           float* __restrict__ dx2) {
  const int C = C1 + C2;
  const int Cw = dx2 ? C : C1;     // channels to produce
  const int L = Cw >> 2;
  const int b = blockIdx.y;
  const long long items = (long long)H * W * L;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (long long)gridDim.x * blockDim.x) {
    const int cq = (int)(it % L);
    const long long pix = it / L;
    const int y = (int)(pix / W), x = (int)(pix - (long long)y * W);
    const int c = cq * 4;
    const bool first = c < C1;
    const float4 xv = first ? *reinterpret_cast<const float4*>(s1 + ((long long)b * H * W + pix) * C1 + c)
                            : *reinterpret_cast<const float4*>(s2 + ((long long)b * H * W + pix) * C2 + (c - C1));
    float4 g = gather_dy<RS>(dy, b, y, x, H, W, C, c);
    if (silu) {
      const float4 a = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 0) * C + c);
      const float4 bb = *reinterpret_cast<const float4*>(ab + ((long long)b * 2 + 1) * C + c);
      g.x *= dsilu(fmaf(a.x, xv.x, bb.x)); g.y *= dsilu(fmaf(a.y, xv.y, bb.y));
      g.z *= dsilu(fmaf(a.z, xv.z, bb.z)); g.w *= dsilu(fmaf(a.w, xv.w, bb.w));
    }
    const float4 k0 = *reinterpret_cast<const float4*>(kk + ((long long)b * 3 + 0) * C + c);
    const float4 k1 = *reinterpret_cast<const float4*>(kk + ((long long)b * 3 + 1) * C + c);
    const float4 k2 = *reinterpret_cast<const float4*>(kk + ((long long)b * 3 + 2) * C + c);
    float4 o;
    o.x = fmaf(k0.x, g.x, fmaf(k1.x, xv.x, k2.x)); o.y = fmaf(k0.y, g.y, fmaf(k1.y, xv.y, k2.y));
    o.z = fmaf(k0.z, g.z, fmaf(k1.z, xv.z, k2.z)); o.w = fmaf(k0.w, g.w, fmaf(k1.w, xv.w, k2.w));
    if (add) {  // skip-path gradient, gathered through the same resample^T (identity skip of an up/down block)
      const float4 av = gather_dy<RS>(add, b, y, x, H, W, add_ld, c);
      o.x += av.x; o.y += av.y; o.z += av.z; o.w += av.w;
    }
    if (first) *reinterpret_cast<float4*>(dx1 + ((long long)b * H * W + pix) * C1 + c) = o;
    else *reinterpret_cast<float4*>(dx2 + ((long long)b * H * W + pix) * C2 + (c - C1)) = o;
  }
}

// dgamma[c] = sum over b in order of part[b][c] (and dbeta from part + B*C): the deterministic gn_bwd_coef's second pass
__global__ void gn_param_reduce_kernel(const float* __restrict__ part, int B, int C, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (dgamma) {
    float a = 0.f;
    for (int b = 0; b < B; ++b) a += part[(long long)b * C + c];
    dgamma[c] = a;
  }
  if (dbeta) {
    float a = 0.f;
    for (int b = 0; b < B; ++b) a += part[((long long)B + b) * C + c];
    dbeta[c] = a;
  }
}

// out[i] = sum over s = 0, 1, ..., S-1 in order of part[s][i]: the ordered reduction of per-split slots
__global__ void __launch_bounds__(256) slot_sum_kernel(const float* __restrict__ part, int S, long long n, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = part[i];
  for (int k = 1; k < S; ++k) a += part[(long long)k * n + i];
  out[i] = a;
}

cudaError_t launch_slot_sum(const float* part, int S, long long n, float* out, cudaStream_t s) {
  slot_sum_kernel<<<cdiv(n, 256), 256, 0, s>>>(part, S, n, out);
  return cudaPeekAtLastError();
}

// dW[idx[b]][:] += d_emb[b][:]   (nn.Embedding backward, unet.py:190-192)
__global__ void embedding_bwd_kernel(const float* __restrict__ d_emb, const int64_t* __restrict__ idx, float* __restrict__ dw,
                                     int B, int E) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * E) return;
  const int b = i / E, j = i % E;
  atomicAdd(dw + idx[b] * E + j, d_emb[i]);
}

// deterministic form: dW[r][j] = sum over b in order of d_emb[b][j] where idx[b] == r, for every row r (rows without a label get 0)
__global__ void embedding_bwd_det_kernel(const float* __restrict__ d_emb, const int64_t* __restrict__ idx, float* __restrict__ dw,
                                         int B, int E, int rows) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * E) return;
  const int r = (int)(i / E), j = (int)(i % E);
  float a = 0.f;
  for (int b = 0; b < B; ++b)
    if (idx[b] == r) a += d_emb[(long long)b * E + j];
  dw[i] = a;
}

// dS = alpha * P * (dP - rowsum(dP * P)), in place on dP  (softmax backward with the ch^-1/2 scale folded in)
__global__ void softmax_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP, long long rows, int cols, float alpha) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* p = P + row * cols;
  float* d = dP + row * cols;
  float s = 0.f;
  for (int j = lane; j < cols; j += 32) s = fmaf(p[j], d[j], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  for (int j = lane; j < cols; j += 32) d[j] = alpha * p[j] * (d[j] - s);
}

// out = g * silu'(x)   (gradient through the SiLU in front of the emb Linears); out = a + b ; out = a * scalar
__global__ void dsilu_mul_kernel(const float* __restrict__ g, const float* __restrict__ x, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = g[i] * dsilu(x[i]);
}
// a[i] *= mask[i] * scale   (inverted dropout with a caller-drawn 0/1 mask; used in both directions)
__global__ void mul_mask_kernel(float* __restrict__ a, const float* __restrict__ mask, float scale, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] *= mask[i] * scale;
}
__global__ void add_inplace_kernel(float* __restrict__ a, const float* __restrict__ b, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] += b[i];
}
// dst[b][c] (ld dst_ld) = src NCHW plane transposed to NHWC or reverse (small tensors: image heads / inputs)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C * HW) return;
  const int p = (int)(i % HW);
  const int c = (int)((i / HW) % C);
  const int b = (int)(i / ((long long)HW * C));
  dst[((long long)b * HW + p) * C + c] = src[i];
}


// ---------------------------------------------------------------------------------------------------------------------
// MLPLNAct backward (model/mlp_skip_net.py:123-141):  v = h*(1+c);  u = (v-mean)*rstd;  y0 = u*lw+lb;  y = SiLU(y0)
// one CTA per row; mean / rstd recomputed like the forward kernel.  dy is read with leading dimension dy_ld (the
// gradient of the skip-concat buffer's left columns).  dlw / dlb accumulate over rows with atomics (zero them first).
// BF16 (the autocast training step): cond / dcond rows have leading dimension cond_ld (a column block of the layers' bank),
// dy is multiplied by mask * scale as it is read (what pdae_mul_mask_cols does in place), and dh / dcond are also stored as
// bf16 (the GEMM operands of the data and weight gradients) next to their fp32 values.
template <bool BF16>
__global__ void __launch_bounds__(256) mlp_mod_ln_act_bwd_kernel(const float* __restrict__ h, const float* __restrict__ cond,
                                                                 int cond_ld, const float* __restrict__ lw,
                                                                 const float* __restrict__ lb, float eps, int silu,
                                                                 const float* __restrict__ dy, int dy_ld,
                                                                 const float* __restrict__ mask, float scale,
                                                                 float* __restrict__ dh, __nv_bfloat16* __restrict__ dh_bf,
                                                                 float* __restrict__ dcond, __nv_bfloat16* __restrict__ dcond_bf,
                                                                 float* __restrict__ dlw, float* __restrict__ dlb, int N) {
  __shared__ float red[2][8];
  __shared__ float bc[2];
  const int b = blockIdx.x;
  const float* hr = h + (long long)b * N;
  const float* cr = cond ? cond + (long long)b * cond_ld : nullptr;
  const float* gr = dy + (long long)b * dy_ld;
  const float* mr = BF16 && mask ? mask + (long long)b * N : nullptr;
  auto block_sum2 = [&](float a, float c2, float& oa, float& oc) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      c2 += __shfl_xor_sync(0xffffffffu, c2, o);
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = c2; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double da = 0.0, dc = 0.0;
      for (int w = 0; w < 8; ++w) { da += red[0][w]; dc += red[1][w]; }
      bc[0] = (float)da; bc[1] = (float)dc;
    }
    __syncthreads();
    oa = bc[0]; oc = bc[1];
  };
  float mean = 0.f, rstd = 1.f;
  if (lw) {
    float s = 0.f, q = 0.f;
    for (int j = threadIdx.x; j < N; j += 256) {
      float v = hr[j];
      if (cr) v = v * (1.0f + cr[j]);
      s += v;
      q = fmaf(v, v, q);
    }
    __syncthreads();
    if (true) {
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
  }
  // pass 1: du = dy * dSiLU(y0) * lw ; sums of du and du*u
  float s1 = 0.f, s2 = 0.f;
  for (int j = threadIdx.x; j < N; j += 256) {
    float v = hr[j];
    if (cr) v = v * (1.0f + cr[j]);
    const float u = lw ? (v - mean) * rstd : v;
    const float y0 = lw ? u * lw[j] + lb[j] : u;
    float g = gr[j];
    if (mr) g *= mr[j] * scale;
    if (silu) {
      const float sg = 1.0f / (1.0f + expf(-y0));
      g *= sg * (1.0f + y0 * (1.0f - sg));
    }
    if (lw) {
      if (dlw) atomicAdd(dlw + j, g * u);
      if (dlb) atomicAdd(dlb + j, g);
      const float du = g * lw[j];
      s1 += du;
      s2 = fmaf(du, u, s2);
    }
  }
  float m1 = 0.f, m2 = 0.f;
  if (lw) {
    block_sum2(s1, s2, m1, m2);
    m1 /= N; m2 /= N;
  }
  for (int j = threadIdx.x; j < N; j += 256) {
    const float hv = hr[j];
    const float cv = cr ? cr[j] : 0.f;
    const float v = hv * (1.0f + cv);
    const float u = lw ? (v - mean) * rstd : v;
    const float y0 = lw ? u * lw[j] + lb[j] : u;
    float g = gr[j];
    if (mr) g *= mr[j] * scale;
    if (silu) {
      const float sg = 1.0f / (1.0f + expf(-y0));
      g *= sg * (1.0f + y0 * (1.0f - sg));
    }
    float dv = g;
    if (lw) dv = rstd * (g * lw[j] - m1 - u * m2);
    const float dhv = dv * (1.0f + cv);
    dh[(long long)b * N + j] = dhv;
    if (BF16) dh_bf[(long long)b * N + j] = __float2bfloat16_rn(dhv);
    if (dcond) {
      const float dcv = dv * hv;
      dcond[(long long)b * cond_ld + j] = dcv;
      if (BF16) dcond_bf[(long long)b * cond_ld + j] = __float2bfloat16_rn(dcv);
    }
  }
}

// a[b][j] *= mask[b][j] * scale for the first N columns of a row-major [B][ld] matrix (dropout on a concat buffer)
__global__ void mul_mask_cols_kernel(float* __restrict__ a, int ld, const float* __restrict__ mask, float scale, int B, int N) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * N) return;
  const int b = (int)(i / N), j = (int)(i % N);
  a[(long long)b * ld + j] *= mask[i] * scale;
}


// dgrad of a wide Linear (H = W = 1, k = 1, Cout = N large): dx[b][e] = sum_n dy[b][n] * w[n][e].  The generic kernel gives one
// thread a serial reduction over all N; here each CTA owns a 64-row chunk of w (split-K) and adds its partial sums.
// DET: chunk x stores its partial sums into slot x of dx ([chunks][B][E]), summed in order by slot_sum_kernel.
template <bool DET>
__global__ void __launch_bounds__(256) linear_dgrad_splitk_kernel(const float* __restrict__ dy, const float* __restrict__ w,
                                                                  float* __restrict__ dx, int B, int N, int E) {
  __shared__ float ds[32][65];
  const int n0 = blockIdx.x * 64, e = blockIdx.y * 256 + threadIdx.x;
  const int nn = min(64, N - n0);
  for (int b0 = 0; b0 < B; b0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 64; i += 256) {
      const int bi = i >> 6, j = i & 63;
      ds[bi][j] = (b0 + bi < B && j < nn) ? dy[(long long)(b0 + bi) * N + n0 + j] : 0.f;
    }
    __syncthreads();
    if (e >= E) continue;
#pragma unroll 1
    for (int bb = 0; bb < 32 && b0 + bb < B; bb += 8) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < nn; ++j) {
        const float wv = w[(long long)(n0 + j) * E + e];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(ds[bb + i][j], wv, acc[i]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (b0 + bb + i < B) {
          if constexpr (DET) dx[((long long)blockIdx.x * B + b0 + bb + i) * E + e] = acc[i];
          else atomicAdd(dx + (long long)(b0 + bb + i) * E + e, acc[i]);
        }
    }
  }
}

// dgrad of a 3x3 stride-1 conv onto <= 4 output channels (the image heads: C -> 3): dx[b,y,x,ci] = sum_{tap,co} dy[b,y+1-ky,
// x+1-kx,co] * w[tap][co][ci].  One thread = one pixel x 4 input channels; the (<= 36 x Cin) weights sit in shared memory.
__global__ void __launch_bounds__(256) conv3x3_dgrad_smalln_kernel(const float* __restrict__ dy, const float* __restrict__ w,
                                                                   float* __restrict__ dx, int B, int H, int W, int Cin, int Cout,
                                                                   int accumulate) {
  extern __shared__ float ws[];   // [9][Cout][Cin]
  for (int i = threadIdx.x; i < 9 * Cout * Cin; i += 256) ws[i] = w[i];
  __syncthreads();
  const int L = Cin >> 2;
  const long long total = (long long)B * H * W * L;
  for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (long long)gridDim.x * 256) {
    const int cq = (int)(idx % L);
    long long pix = idx / L;
    const int x = (int)(pix % W); pix /= W;
    const int y = (int)(pix % H);
    const int b = (int)(pix / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y + 1 - ky;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = x + 1 - kx;
        if (xx < 0 || xx >= W) continue;
        const float* g = dy + (((long long)b * H + yy) * W + xx) * Cout;
        for (int co = 0; co < Cout; ++co) {
          const float gv = g[co];
          const float4 wv = *reinterpret_cast<const float4*>(ws + ((ky * 3 + kx) * Cout + co) * Cin + 4 * cq);
          acc.x = fmaf(gv, wv.x, acc.x); acc.y = fmaf(gv, wv.y, acc.y); acc.z = fmaf(gv, wv.z, acc.z); acc.w = fmaf(gv, wv.w, acc.w);
        }
      }
    }
    float4* o = reinterpret_cast<float4*>(dx + ((((long long)b * H + y) * W + x) * Cin + 4 * cq));
    if (accumulate) { const float4 t = *o; acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w; }
    *o = acc;
  }
}

}  // namespace pdae

using namespace pdae;

extern "C" int pdae_conv2d_dgrad_simt(const float* dy, const float* w_tco, float* dx, int B, int H, int W, int Cin, int Cout,
                                      int ksize, int stride, int pad, int accumulate, pdae_stream_t stream) {
  PDAE_REQUIRE(dy && w_tco && dx, "conv2d_dgrad: null pointer");
  if (H == 1 && W == 1 && ksize == 1 && stride == 1 && pad == 0 && Cout >= 1024 && !accumulate) {   // wide Linear: split-K
    PDAE_CUDA(cudaMemsetAsync(dx, 0, (size_t)B * Cin * sizeof(float), (cudaStream_t)stream));
    linear_dgrad_splitk_kernel<false><<<dim3(cdiv(Cout, 64), cdiv(Cin, 256)), 256, 0, (cudaStream_t)stream>>>(dy, w_tco, dx, B, Cout, Cin);
    PDAE_LAUNCH_CHECK("linear_dgrad_splitk_kernel");
    return PDAE_OK;
  }
  if (ksize == 3 && stride == 1 && pad == 1 && Cout <= 4 && Cin % 4 == 0 && (size_t)9 * Cout * Cin * 4 <= 48 * 1024 &&
      !((uintptr_t)dx & 15)) {                                                                       // image heads
    const long long items = (long long)B * H * W * (Cin / 4);
    long long gx = (items + 255) / 256;
    if (gx > 148 * 16) gx = 148 * 16;
    conv3x3_dgrad_smalln_kernel<<<(unsigned)gx, 256, (size_t)9 * Cout * Cin * 4, (cudaStream_t)stream>>>(dy, w_tco, dx, B, H, W, Cin,
                                                                                                       Cout, accumulate);
    PDAE_LAUNCH_CHECK("conv3x3_dgrad_smalln_kernel");
    return PDAE_OK;
  }
  DgradArgs p;
  p.dy = dy; p.w = w_tco; p.dx = dx; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
  p.ksize = ksize; p.stride = stride; p.pad = pad; p.accumulate = accumulate;
  p.Ho = (H + 2 * pad - ksize) / stride + 1; p.Wo = (W + 2 * pad - ksize) / stride + 1;
  p.M = (long long)B * H * W; p.K = ksize * ksize * Cout;
  dim3 grid(cdiv(p.M, DBM), cdiv(Cin, DBN));
  conv_dgrad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  PDAE_LAUNCH_CHECK("conv_dgrad_kernel");
  return PDAE_OK;
}

extern "C" int pdae_conv2d_wgrad_simt(const float* x, int in_nchw, int a_silu, const float* dy, float* dw_tcico, int B, int H,
                                      int W, int Cin, int Cout, int ksize, int stride, int pad, pdae_stream_t stream) {
  PDAE_REQUIRE(x && dy && dw_tcico, "conv2d_wgrad: null pointer");
  WgradArgs p;
  p.x = x; p.dy = dy; p.dw = dw_tcico; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
  p.ksize = ksize; p.stride = stride; p.pad = pad; p.in_nchw = in_nchw; p.a_silu = a_silu;
  p.Ho = (H + 2 * pad - ksize) / stride + 1; p.Wo = (W + 2 * pad - ksize) / stride + 1;
  p.P = (long long)B * p.Ho * p.Wo; p.MK = ksize * ksize * Cin;
  const int gx = cdiv(p.MK, DBM), gy = cdiv(Cout, DBN);
  long long splits = (148LL * 4 + (long long)gx * gy - 1) / ((long long)gx * gy);  // enough CTAs to fill the GPU
  long long maxs = (p.P + 255) / 256;
  if (splits > maxs) splits = maxs;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  p.chunk = (int)(((p.P + splits - 1) / splits + DBK - 1) / DBK * DBK);
  const int gz = (int)((p.P + p.chunk - 1) / p.chunk);
  dim3 grid(gx, gy, gz);
  conv_wgrad_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  PDAE_LAUNCH_CHECK("conv_wgrad_kernel");
  return PDAE_OK;
}

extern "C" int pdae_colsum(const float* dy, int64_t M, int N, float* out, pdae_stream_t stream) {
  PDAE_REQUIRE(dy && out && N > 0, "colsum: bad args");
  if (N % 4 == 0 && !((uintptr_t)dy & 15)) {
    long long rows = (M / 592 + 7) / 8 * 8;      // about four CTAs per SM, eight-row granules
    rows = rows < 32 ? 32 : (rows > 512 ? 512 : rows);
    colsum_v4_kernel<false><<<(unsigned)cdiv(M, rows), 256, 0, (cudaStream_t)stream>>>(dy, M, N, out, (int)rows);
    PDAE_LAUNCH_CHECK("colsum_v4_kernel");
    return PDAE_OK;
  }
  const int rows = 256;
  colsum_kernel<false><<<cdiv(M, rows), N < 256 ? (N < 32 ? 32 : N) : 256, 0, (cudaStream_t)stream>>>(dy, M, N, out, rows);
  PDAE_LAUNCH_CHECK("colsum_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_bwd_sums(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* dy, int silu,
                                int resample, int B, int H, int W, float* S, pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && ab && dy && S, "gn_bwd_sums: null pointer");
  if (!src2) C2 = 0;
  const int C = C1 + C2;
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C % 32 == 0 && (size_t)2 * C * 4 <= 48 * 1024, "gn_bwd_sums: bad channels");
  PDAE_REQUIRE(resample >= 0 && resample <= 2, "gn_bwd_sums: bad resample mode");
  PDAE_REQUIRE(resample != PDAE_RESAMPLE_DOWN2 || (H % 2 == 0 && W % 2 == 0), "gn_bwd_sums: odd dims for DOWN2");
  cudaStream_t s = (cudaStream_t)stream;
  PDAE_CUDA(cudaMemsetAsync(S, 0, (size_t)B * C * 2 * sizeof(float), s));
  int ppc = 256;                                   // low-resolution layers: fewer pixels per CTA so that >= ~4 CTAs/SM exist
  while (ppc > 8 && (long long)B * cdiv((long long)H * W, ppc) < 592) ppc >>= 1;
  dim3 grid(cdiv((long long)H * W, ppc), B);
  const size_t sm = 2 * C * sizeof(float);
  if (resample == PDAE_RESAMPLE_NONE) gn_bwd_sums_kernel<PDAE_RESAMPLE_NONE, false><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, S, ppc);
  else if (resample == PDAE_RESAMPLE_UP2) gn_bwd_sums_kernel<PDAE_RESAMPLE_UP2, false><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, S, ppc);
  else gn_bwd_sums_kernel<PDAE_RESAMPLE_DOWN2, false><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, S, ppc);
  PDAE_LAUNCH_CHECK("gn_bwd_sums_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_bwd_coef(const float* S, const double* sums, const float* gamma, const float* beta, const float* emb,
                                int emb_ld, const float* embz, int embz_ld, int B, int C, int HW, float eps, float* kk,
                                float* dgamma, float* dbeta, float* demb, int demb_ld, float* dembz, int dembz_ld,
                                pdae_stream_t stream) {
  PDAE_REQUIRE(S && sums && gamma && beta && kk, "gn_bwd_coef: null pointer");
  gn_bwd_coef_kernel<false><<<B, C < 1024 ? (C < 32 ? 32 : C) : 1024, 0, (cudaStream_t)stream>>>(
      S, sums, gamma, beta, emb, emb_ld, embz, embz_ld, C, HW, eps, kk, dgamma, dbeta, demb, demb_ld, dembz, dembz_ld);
  PDAE_LAUNCH_CHECK("gn_bwd_coef_kernel");
  return PDAE_OK;
}

extern "C" int pdae_gn_bwd_apply(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* kk,
                                 const float* dy, int silu, int resample, int B, int H, int W, const float* add, int add_ld,
                                 float* dx1, float* dx2, pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && ab && kk && dy && dx1, "gn_bwd_apply: null pointer");
  if (!src2) C2 = 0;
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && !(dx2 && !src2), "gn_bwd_apply: bad channels");
  PDAE_REQUIRE(resample >= 0 && resample <= 2, "gn_bwd_apply: bad resample mode");
  PDAE_REQUIRE(resample != PDAE_RESAMPLE_DOWN2 || (H % 2 == 0 && W % 2 == 0), "gn_bwd_apply: odd dims for DOWN2");
  const long long items = (long long)H * W * ((dx2 ? C1 + C2 : C1) / 4);
  int gx = cdiv(items, 256);
  if (gx > 148 * 16) gx = 148 * 16;
  dim3 grid(gx, B);
  cudaStream_t s = (cudaStream_t)stream;
  if (resample == PDAE_RESAMPLE_NONE) gn_bwd_apply_kernel<PDAE_RESAMPLE_NONE><<<grid, 256, 0, s>>>(src1, C1, src2, C2, ab, kk, dy, silu, H, W, add, add_ld, dx1, dx2);
  else if (resample == PDAE_RESAMPLE_UP2) gn_bwd_apply_kernel<PDAE_RESAMPLE_UP2><<<grid, 256, 0, s>>>(src1, C1, src2, C2, ab, kk, dy, silu, H, W, add, add_ld, dx1, dx2);
  else gn_bwd_apply_kernel<PDAE_RESAMPLE_DOWN2><<<grid, 256, 0, s>>>(src1, C1, src2, C2, ab, kk, dy, silu, H, W, add, add_ld, dx1, dx2);
  PDAE_LAUNCH_CHECK("gn_bwd_apply_kernel");
  return PDAE_OK;
}

extern "C" int pdae_embedding_bwd(const float* d_emb, const int64_t* idx, float* dw, int B, int E, pdae_stream_t stream) {
  PDAE_REQUIRE(d_emb && idx && dw, "embedding_bwd: null pointer");
  embedding_bwd_kernel<<<cdiv((long long)B * E, 256), 256, 0, (cudaStream_t)stream>>>(d_emb, idx, dw, B, E);
  PDAE_LAUNCH_CHECK("embedding_bwd_kernel");
  return PDAE_OK;
}

extern "C" int pdae_softmax_bwd(const float* P, float* dP, int64_t rows, int cols, float alpha, pdae_stream_t stream) {
  PDAE_REQUIRE(P && dP, "softmax_bwd: null pointer");
  softmax_bwd_kernel<<<cdiv(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(P, dP, rows, cols, alpha);
  PDAE_LAUNCH_CHECK("softmax_bwd_kernel");
  return PDAE_OK;
}

extern "C" int pdae_dsilu_mul(const float* g, const float* x, float* out, int64_t n, pdae_stream_t stream) {
  PDAE_REQUIRE(g && x && out, "dsilu_mul: null pointer");
  dsilu_mul_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(g, x, out, n);
  PDAE_LAUNCH_CHECK("dsilu_mul_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mul_mask(float* a, const float* mask, float scale, int64_t n, pdae_stream_t stream) {
  PDAE_REQUIRE(a && mask, "mul_mask: null pointer");
  mul_mask_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(a, mask, scale, n);
  PDAE_LAUNCH_CHECK("mul_mask_kernel");
  return PDAE_OK;
}

extern "C" int pdae_add_inplace(float* a, const float* b, int64_t n, pdae_stream_t stream) {
  PDAE_REQUIRE(a && b, "add_inplace: null pointer");
  add_inplace_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, n);
  PDAE_LAUNCH_CHECK("add_inplace_kernel");
  return PDAE_OK;
}

extern "C" int pdae_nchw_to_nhwc(const float* src, float* dst, int B, int C, int HW, pdae_stream_t stream) {
  PDAE_REQUIRE(src && dst, "nchw_to_nhwc: null pointer");
  nchw_to_nhwc_kernel<<<cdiv((long long)B * C * HW, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, B, C, HW);
  PDAE_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mlp_mod_ln_act_bwd(const float* h, const float* cond, const float* ln_w, const float* ln_b, float eps, int silu,
                                       const float* dy, int dy_ld, float* dh, float* dcond, float* d_ln_w, float* d_ln_b, int B,
                                       int N, pdae_stream_t stream) {
  PDAE_REQUIRE(h && dy && dh && B > 0 && N > 0 && dy_ld >= N, "mlp_mod_ln_act_bwd: bad args");
  PDAE_REQUIRE(!ln_w || ln_b, "mlp_mod_ln_act_bwd: LayerNorm weight without bias");
  PDAE_REQUIRE(!dcond || cond, "mlp_mod_ln_act_bwd: dcond without cond");
  mlp_mod_ln_act_bwd_kernel<false><<<B, 256, 0, (cudaStream_t)stream>>>(h, cond, N, ln_w, ln_b, eps, silu, dy, dy_ld, nullptr,
                                                                        1.0f, dh, nullptr, dcond, nullptr, d_ln_w, d_ln_b, N);
  PDAE_LAUNCH_CHECK("mlp_mod_ln_act_bwd_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mlp_mod_ln_act_bwd_bf16(const float* h, const float* cond, int cond_ld, const float* ln_w, const float* ln_b,
                                            float eps, int silu, const float* dy, int dy_ld, const float* mask, float mask_scale,
                                            float* dh, void* dh_bf16, float* dcond, void* dcond_bf16, float* d_ln_w, float* d_ln_b,
                                            int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(h && dy && dh && dh_bf16 && B > 0 && N > 0 && dy_ld >= N, "mlp_mod_ln_act_bwd_bf16: bad args");
  PDAE_REQUIRE(!ln_w || ln_b, "mlp_mod_ln_act_bwd_bf16: LayerNorm weight without bias");
  PDAE_REQUIRE(!dcond || (cond && dcond_bf16), "mlp_mod_ln_act_bwd_bf16: dcond without cond or its bf16 copy");
  PDAE_REQUIRE(!cond || cond_ld >= N, "mlp_mod_ln_act_bwd_bf16: cond_ld=%d < N=%d", cond_ld, N);
  mlp_mod_ln_act_bwd_kernel<true><<<B, 256, 0, (cudaStream_t)stream>>>(
      h, cond, cond_ld, ln_w, ln_b, eps, silu, dy, dy_ld, mask, mask_scale, dh, (__nv_bfloat16*)dh_bf16, dcond,
      (__nv_bfloat16*)dcond_bf16, d_ln_w, d_ln_b, N);
  PDAE_LAUNCH_CHECK("mlp_mod_ln_act_bwd_kernel<bf16>");
  return PDAE_OK;
}

extern "C" int pdae_mul_mask_cols(float* a, int ld, const float* mask, float scale, int B, int N, pdae_stream_t stream) {
  PDAE_REQUIRE(a && mask && B > 0 && N > 0 && ld >= N, "mul_mask_cols: bad args");
  mul_mask_cols_kernel<<<cdiv((long long)B * N, 256), 256, 0, (cudaStream_t)stream>>>(a, ld, mask, scale, B, N);
  PDAE_LAUNCH_CHECK("mul_mask_cols_kernel");
  return PDAE_OK;
}

// ---- deterministic forms (torch.use_deterministic_algorithms): no float atomics -------------------------------------------
// Every partial result has its own slot in a caller-owned workspace (no initialisation needed) and the slots are summed in a
// fixed order.  Split and chunk counts follow the shapes only, never the GPU.  Arguments and the workspace size are checked
// before any launch; the outputs are written, not added to, so they need no zeroing.
namespace pdae {
constexpr int DET_WGRAD_CTAS = 132 * 4;   // conv_wgrad_kernel: about four CTAs per SM of a 132-SM H100, a constant

static void wgrad_simt_args(WgradArgs& p, int B, int H, int W, int Cin, int Cout, int ksize, int stride, int pad) {
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.ksize = ksize; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - ksize) / stride + 1; p.Wo = (W + 2 * pad - ksize) / stride + 1;
  p.P = (long long)B * p.Ho * p.Wo; p.MK = ksize * ksize * Cin;
  const long long tiles = (long long)cdiv(p.MK, DBM) * cdiv(Cout, DBN);
  long long splits = (DET_WGRAD_CTAS + tiles - 1) / tiles, maxs = (p.P + 255) / 256;
  if (splits > maxs) splits = maxs;
  if (splits < 1) splits = 1;
  p.chunk = (int)(((p.P + splits - 1) / splits + DBK - 1) / DBK * DBK);
}
static bool wgrad_simt_shape_ok(int B, int H, int W, int Cin, int Cout, int ksize, int stride, int pad) {
  return B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && ksize > 0 && stride > 0 && pad >= 0 && H + 2 * pad >= ksize &&
         W + 2 * pad >= ksize;
}
static long long colsum_det_rows(long long M) {   // pdae_colsum's row chunk, used by both deterministic paths
  long long rows = (M / 592 + 7) / 8 * 8;
  return rows < 32 ? 32 : (rows > 512 ? 512 : rows);
}
static int gn_bwd_ppc(int B, int HW) {            // pdae_gn_bwd_sums' pixels per CTA (a function of B and HW)
  int ppc = 256;
  while (ppc > 8 && (long long)B * cdiv((long long)HW, ppc) < 592) ppc >>= 1;
  return ppc;
}
static bool dgrad_wide_linear(int H, int W, int ksize, int stride, int pad, int Cout, int accumulate) {
  return H == 1 && W == 1 && ksize == 1 && stride == 1 && pad == 0 && Cout >= 1024 && !accumulate;
}
}  // namespace pdae

#define PDAE_DET_WS(fn, need, ws, ws_bytes)                                                                               \
  PDAE_REQUIRE((need) == 0 || ((ws) && (ws_bytes) >= (need)), fn ": workspace of %lld bytes, %lld needed", (long long)(ws_bytes), \
               (long long)(need))

extern "C" int64_t pdae_conv2d_wgrad_simt_det_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride,
                                                             int pad) {
  if (!wgrad_simt_shape_ok(B, H, W, Cin, Cout, ksize, stride, pad)) {
    set_error("conv2d_wgrad_simt_det_workspace_bytes: bad shape");
    return PDAE_EINVAL;
  }
  WgradArgs p;
  wgrad_simt_args(p, B, H, W, Cin, Cout, ksize, stride, pad);
  const long long chunks = (p.P + p.chunk - 1) / p.chunk;
  return chunks > 1 ? chunks * p.MK * Cout * (int64_t)sizeof(float) : 0;
}

extern "C" int pdae_conv2d_wgrad_simt_det(const float* x, int in_nchw, int a_silu, const float* dy, float* dw_tcico, int B, int H,
                                          int W, int Cin, int Cout, int ksize, int stride, int pad, float* workspace,
                                          int64_t workspace_bytes, pdae_stream_t stream) {
  PDAE_REQUIRE(x && dy && dw_tcico, "conv2d_wgrad_simt_det: null pointer");
  const int64_t need = pdae_conv2d_wgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, ksize, stride, pad);
  if (need < 0) return PDAE_EINVAL;
  PDAE_DET_WS("conv2d_wgrad_simt_det", need, workspace, workspace_bytes);
  WgradArgs p;
  wgrad_simt_args(p, B, H, W, Cin, Cout, ksize, stride, pad);
  p.x = x; p.dy = dy; p.in_nchw = in_nchw; p.a_silu = a_silu;
  p.dw = need ? workspace : dw_tcico;
  const int gz = (int)((p.P + p.chunk - 1) / p.chunk);
  cudaStream_t s = (cudaStream_t)stream;
  conv_wgrad_kernel<true><<<dim3(cdiv(p.MK, DBM), cdiv(Cout, DBN), gz), 256, 0, s>>>(p);
  PDAE_LAUNCH_CHECK("conv_wgrad_kernel<det>");
  if (need) PDAE_CUDA(launch_slot_sum(workspace, gz, (long long)p.MK * Cout, dw_tcico, s));
  return PDAE_OK;
}

extern "C" int64_t pdae_conv2d_dgrad_simt_det_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride,
                                                             int pad, int accumulate) {
  if (!wgrad_simt_shape_ok(B, H, W, Cin, Cout, ksize, stride, pad)) {
    set_error("conv2d_dgrad_simt_det_workspace_bytes: bad shape");
    return PDAE_EINVAL;
  }
  return dgrad_wide_linear(H, W, ksize, stride, pad, Cout, accumulate) ? (int64_t)cdiv(Cout, 64) * B * Cin * sizeof(float) : 0;
}

// as pdae_conv2d_dgrad_simt; the wide-Linear split-K form stores each 64-row chunk's partial sums in its slot
extern "C" int pdae_conv2d_dgrad_simt_det(const float* dy, const float* w_tco, float* dx, int B, int H, int W, int Cin, int Cout,
                                          int ksize, int stride, int pad, int accumulate, float* workspace, int64_t workspace_bytes,
                                          pdae_stream_t stream) {
  PDAE_REQUIRE(dy && w_tco && dx, "conv2d_dgrad_simt_det: null pointer");
  const int64_t need = pdae_conv2d_dgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, ksize, stride, pad, accumulate);
  if (need < 0) return PDAE_EINVAL;
  PDAE_DET_WS("conv2d_dgrad_simt_det", need, workspace, workspace_bytes);
  if (!need) return pdae_conv2d_dgrad_simt(dy, w_tco, dx, B, H, W, Cin, Cout, ksize, stride, pad, accumulate, stream);
  cudaStream_t s = (cudaStream_t)stream;
  linear_dgrad_splitk_kernel<true><<<dim3(cdiv(Cout, 64), cdiv(Cin, 256)), 256, 0, s>>>(dy, w_tco, workspace, B, Cout, Cin);
  PDAE_LAUNCH_CHECK("linear_dgrad_splitk_kernel<det>");
  PDAE_CUDA(launch_slot_sum(workspace, cdiv(Cout, 64), (long long)B * Cin, dx, s));
  return PDAE_OK;
}

extern "C" int64_t pdae_colsum_det_workspace_bytes(int64_t M, int N) {
  if (M <= 0 || N <= 0) {
    set_error("colsum_det_workspace_bytes: M=%lld N=%d must be > 0", (long long)M, N);
    return PDAE_EINVAL;
  }
  const long long chunks = (M + colsum_det_rows(M) - 1) / colsum_det_rows(M);
  return chunks > 1 ? chunks * N * (int64_t)sizeof(float) : 0;
}

extern "C" int pdae_colsum_det(const float* dy, int64_t M, int N, float* out, float* workspace, int64_t workspace_bytes,
                               pdae_stream_t stream) {
  PDAE_REQUIRE(dy && out, "colsum_det: null pointer");
  const int64_t need = pdae_colsum_det_workspace_bytes(M, N);
  if (need < 0) return PDAE_EINVAL;
  PDAE_DET_WS("colsum_det", need, workspace, workspace_bytes);
  const long long rows = colsum_det_rows(M);
  const int chunks = cdiv(M, rows);
  float* slots = need ? workspace : out;
  cudaStream_t s = (cudaStream_t)stream;
  if (N % 4 == 0 && !((uintptr_t)dy & 15)) {
    colsum_v4_kernel<true><<<chunks, 256, 0, s>>>(dy, M, N, slots, (int)rows);
    PDAE_LAUNCH_CHECK("colsum_v4_kernel<det>");
  } else {
    colsum_kernel<true><<<chunks, N < 256 ? (N < 32 ? 32 : N) : 256, 0, s>>>(dy, M, N, slots, (int)rows);
    PDAE_LAUNCH_CHECK("colsum_kernel<det>");
  }
  if (need) PDAE_CUDA(launch_slot_sum(workspace, chunks, N, out, s));
  return PDAE_OK;
}

extern "C" int64_t pdae_gn_bwd_sums_det_workspace_bytes(int B, int H, int W, int C) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) {
    set_error("gn_bwd_sums_det_workspace_bytes: B=%d H=%d W=%d C=%d must be > 0", B, H, W, C);
    return PDAE_EINVAL;
  }
  return (int64_t)B * cdiv((long long)H * W, gn_bwd_ppc(B, H * W)) * C * 2 * (int64_t)sizeof(float);
}

extern "C" int pdae_gn_bwd_sums_det(const float* src1, int C1, const float* src2, int C2, const float* ab, const float* dy,
                                    int silu, int resample, int B, int H, int W, float* S, float* workspace, int64_t workspace_bytes,
                                    pdae_stream_t stream) {
  PDAE_REQUIRE(src1 && ab && dy && S && workspace, "gn_bwd_sums_det: null pointer");
  if (!src2) C2 = 0;
  const int C = C1 + C2;
  PDAE_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && C % 32 == 0 && C > 0 && C <= 6144, "gn_bwd_sums_det: bad channels C1=%d C2=%d", C1, C2);
  PDAE_REQUIRE(resample >= 0 && resample <= 2, "gn_bwd_sums_det: bad resample mode");
  PDAE_REQUIRE(resample != PDAE_RESAMPLE_DOWN2 || (H % 2 == 0 && W % 2 == 0), "gn_bwd_sums_det: odd dims for DOWN2");
  const int64_t need = pdae_gn_bwd_sums_det_workspace_bytes(B, H, W, C);
  if (need < 0) return PDAE_EINVAL;
  PDAE_DET_WS("gn_bwd_sums_det", need, workspace, workspace_bytes);
  cudaStream_t s = (cudaStream_t)stream;
  const int ppc = gn_bwd_ppc(B, H * W), P = cdiv((long long)H * W, ppc);
  const int L = C / 4, Lb = L < 256 ? L : 256;
  const size_t sm = (size_t)(256 / Lb) * 2 * C * sizeof(float);
  dim3 grid(P, B);
  if (resample == PDAE_RESAMPLE_NONE) gn_bwd_sums_kernel<PDAE_RESAMPLE_NONE, true><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, workspace, ppc);
  else if (resample == PDAE_RESAMPLE_UP2) gn_bwd_sums_kernel<PDAE_RESAMPLE_UP2, true><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, workspace, ppc);
  else gn_bwd_sums_kernel<PDAE_RESAMPLE_DOWN2, true><<<grid, 256, sm, s>>>(src1, C1, src2, C2, ab, dy, silu, H, W, workspace, ppc);
  PDAE_LAUNCH_CHECK("gn_bwd_sums_kernel<det>");
  PDAE_CUDA(launch_stat_parts_reduce(workspace, B, P, C, S, s));
  return PDAE_OK;
}

extern "C" int64_t pdae_gn_bwd_coef_det_workspace_bytes(int B, int C) {
  if (B <= 0 || C <= 0) {
    set_error("gn_bwd_coef_det_workspace_bytes: B=%d C=%d must be > 0", B, C);
    return PDAE_EINVAL;
  }
  return (int64_t)2 * B * C * sizeof(float);
}

extern "C" int pdae_gn_bwd_coef_det(const float* S, const double* sums, const float* gamma, const float* beta, const float* emb,
                                    int emb_ld, const float* embz, int embz_ld, int B, int C, int HW, float eps, float* kk,
                                    float* dgamma, float* dbeta, float* demb, int demb_ld, float* dembz, int dembz_ld,
                                    float* workspace, int64_t workspace_bytes, pdae_stream_t stream) {
  PDAE_REQUIRE(S && sums && gamma && beta && kk, "gn_bwd_coef_det: null pointer");
  PDAE_REQUIRE(C % 32 == 0 && C <= 2048, "gn_bwd_coef_det: C=%d (a multiple of 32, <= 2048)", C);
  const int64_t need = (dgamma || dbeta) ? pdae_gn_bwd_coef_det_workspace_bytes(B, C) : 0;
  if (need < 0) return PDAE_EINVAL;
  PDAE_DET_WS("gn_bwd_coef_det", need, workspace, workspace_bytes);
  cudaStream_t s = (cudaStream_t)stream;
  gn_bwd_coef_kernel<true><<<B, C < 1024 ? (C < 32 ? 32 : C) : 1024, (size_t)2 * C * sizeof(double), s>>>(
      S, sums, gamma, beta, emb, emb_ld, embz, embz_ld, C, HW, eps, kk, dgamma ? workspace : nullptr,
      dbeta ? workspace + (long long)B * C : nullptr, demb, demb_ld, dembz, dembz_ld);
  PDAE_LAUNCH_CHECK("gn_bwd_coef_kernel<det>");
  if (need) {
    gn_param_reduce_kernel<<<cdiv(C, 256), 256, 0, s>>>(workspace, B, C, dgamma, dbeta);
    PDAE_LAUNCH_CHECK("gn_param_reduce_kernel");
  }
  return PDAE_OK;
}

extern "C" int pdae_embedding_bwd_det(const float* d_emb, const int64_t* idx, float* dw, int B, int E, int rows,
                                      pdae_stream_t stream) {
  PDAE_REQUIRE(d_emb && idx && dw && B > 0 && E > 0 && rows > 0, "embedding_bwd_det: bad args");
  embedding_bwd_det_kernel<<<cdiv((long long)rows * E, 256), 256, 0, (cudaStream_t)stream>>>(d_emb, idx, dw, B, E, rows);
  PDAE_LAUNCH_CHECK("embedding_bwd_det_kernel");
  return PDAE_OK;
}
