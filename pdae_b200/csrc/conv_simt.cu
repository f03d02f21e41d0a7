// fp32 CUDA-core implicit-GEMM convolution / linear ("parity mode") and the Cout<=4 head conv.
//
// GEMM view: M = B*Ho*Wo output pixels, N = Cout, K = k*k*Cin (tap-major, channel-minor so that
// consecutive k are consecutive NHWC channels).  64x64x16 CTA tile, 256 threads, 4x4 micro-tile.
// This is the exact-fp32 path used (a) to hold rtol 1e-3 / atol 1e-4 against the CPU oracle and
// (b) for the shapes the tensor-core kernels do not take (Cin=3 stem, stride-2 encoder convs, Linear).
#include "common.cuh"

namespace pdae {

constexpr int BM = 64, BN = 64, BK = 16, APAD = 4;

struct ConvArgs {
  const void* in;
  const float* w;
  const float* bias;
  const float* residual;
  float* out;
  int B, H, W, Cin, Cout, Ho, Wo, ksize, stride, pad;
  int in_nchw, out_nchw, a_silu;
  long long M;
  int K;
};

// VEC4: Cin % 4 == 0, NHWC input -> 16-byte (fp32) / 8-byte (bf16) loads along channels.
template <typename TIn, bool VEC4>
__global__ void __launch_bounds__(256) conv_simt_kernel(ConvArgs p) {
  __shared__ __align__(16) float As[BK][BM + APAD];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const TIn* __restrict__ in = reinterpret_cast<const TIn*>(p.in);

  // A-load role: VEC4 -> row = tid/4, k-quad = tid%4 ; scalar -> row = tid%64, k = tid/64 + 4*i
  const int a_row = VEC4 ? (tid >> 2) : (tid & 63);
  const int a_k = VEC4 ? ((tid & 3) * 4) : (tid >> 6);
  const long long am = m0 + a_row;
  const bool a_valid = am < p.M;
  int ab = 0, aoy = 0, aox = 0;
  if (a_valid) {
    long long r = am;
    aox = (int)(r % p.Wo);
    r /= p.Wo;
    aoy = (int)(r % p.Ho);
    ab = (int)(r / p.Ho);
  }
  const int iy0 = aoy * p.stride - p.pad, ix0 = aox * p.stride - p.pad;

  // B-load role: k = tid/16, n-quad = tid%16
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  const bool b_vec = (p.Cout & 3) == 0;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < p.K; k0 += BK) {
    // ---- A tile ----
    if (VEC4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int kk = k0 + a_k;
      if (a_valid && kk < p.K) {
        const int tap = kk / p.Cin, ci = kk - tap * p.Cin;
        const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
        const int iy = iy0 + ky, ix = ix0 + kx;
        if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
          v = load4<TIn>(in + (((long long)ab * p.H + iy) * p.W + ix) * p.Cin + ci);
          if (p.a_silu) {
            v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w);
          }
        }
      }
      As[a_k + 0][a_row] = v.x;
      As[a_k + 1][a_row] = v.y;
      As[a_k + 2][a_row] = v.z;
      As[a_k + 3][a_row] = v.w;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kl = a_k + 4 * i;
        const int kk = k0 + kl;
        float v = 0.f;
        if (a_valid && kk < p.K) {
          const int tap = kk / p.Cin, ci = kk - tap * p.Cin;
          const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
          const int iy = iy0 + ky, ix = ix0 + kx;
          if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
            const long long off = p.in_nchw ? ((((long long)ab * p.Cin + ci) * p.H + iy) * p.W + ix)
                                            : ((((long long)ab * p.H + iy) * p.W + ix) * p.Cin + ci);
            v = load1<TIn>(in + off);
            if (p.a_silu) v = silu_f(v);
          }
        }
        As[kl][a_row] = v;
      }
    }
    // ---- B tile ----
    {
      const int kk = k0 + b_k;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kk < p.K) {
        const float* wp = p.w + (long long)kk * p.Cout + n0 + b_n;
        if (b_vec && n0 + b_n + 3 < p.Cout) {
          v = *reinterpret_cast<const float4*>(wp);
        } else {
          if (n0 + b_n + 0 < p.Cout) v.x = wp[0];
          if (n0 + b_n + 1 < p.Cout) v.y = wp[1];
          if (n0 + b_n + 2 < p.Cout) v.z = wp[2];
          if (n0 + b_n + 3 < p.Cout) v.w = wp[3];
        }
      }
      *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
    const int n = n0 + tx * 4;
    if (n >= p.Cout) continue;
    float v[4] = {acc[i][0], acc[i][1], acc[i][2], acc[i][3]};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (p.bias && n + j < p.Cout) v[j] += p.bias[n + j];
    if (!p.out_nchw) {
      const long long off = m * p.Cout + n;
      if (b_vec && n + 3 < p.Cout) {
        if (p.residual) {
          const float4 r = *reinterpret_cast<const float4*>(p.residual + off);
          v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
        }
        *reinterpret_cast<float4*>(p.out + off) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
        for (int j = 0; j < 4 && n + j < p.Cout; ++j) {
          float o = v[j];
          if (p.residual) o += p.residual[off + j];
          p.out[off + j] = o;
        }
      }
    } else {
      long long r = m;
      const int ox = (int)(r % p.Wo);
      r /= p.Wo;
      const int oy = (int)(r % p.Ho);
      const int b = (int)(r / p.Ho);
      for (int j = 0; j < 4 && n + j < p.Cout; ++j) {
        float o = v[j];
        if (p.residual) o += p.residual[m * p.Cout + n + j];
        p.out[(((long long)b * p.Cout + n + j) * p.Ho + oy) * p.Wo + ox] = o;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 3x3 / pad 1 / stride 1 conv with Cout <= 4 : one warp per output pixel, lanes over channels.
// Weights [9][Cin][4] live in shared memory; activations stream through L1/L2 (each input element
// is touched by 9 neighbouring pixels).  Output NCHW fp32.
template <typename TIn>
__global__ void __launch_bounds__(256) conv3x3_smalln_kernel(const TIn* __restrict__ in, const float* __restrict__ w4,
                                                            const float* __restrict__ bias, float* __restrict__ out,
                                                            int B, int H, int W, int Cin, int Cout) {
  extern __shared__ __align__(16) float sw[];  // [9*Cin][4]
  for (int i = threadIdx.x; i < 9 * Cin; i += blockDim.x)
    reinterpret_cast<float4*>(sw)[i] = reinterpret_cast<const float4*>(w4)[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long npix = (long long)B * H * W;
  for (long long pix = warp; pix < npix; pix += nwarps) {
    long long r = pix;
    const int x = (int)(r % W);
    r /= W;
    const int y = (int)(r % H);
    const int b = (int)(r / H);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int iy = y + tap / 3 - 1, ix = x + tap % 3 - 1;
      if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
      const TIn* src = in + (((long long)b * H + iy) * W + ix) * Cin;
      const float4* wt = reinterpret_cast<const float4*>(sw) + tap * Cin;
      for (int c = lane * 4; c < Cin; c += 128) {
        const float4 v = load4<TIn>(src + c);
        const float4 w0 = wt[c], w1 = wt[c + 1], w2 = wt[c + 2], w3 = wt[c + 3];
        a0 = fmaf(v.x, w0.x, a0); a1 = fmaf(v.x, w0.y, a1); a2 = fmaf(v.x, w0.z, a2); a3 = fmaf(v.x, w0.w, a3);
        a0 = fmaf(v.y, w1.x, a0); a1 = fmaf(v.y, w1.y, a1); a2 = fmaf(v.y, w1.z, a2); a3 = fmaf(v.y, w1.w, a3);
        a0 = fmaf(v.z, w2.x, a0); a1 = fmaf(v.z, w2.y, a1); a2 = fmaf(v.z, w2.z, a2); a3 = fmaf(v.z, w2.w, a3);
        a0 = fmaf(v.w, w3.x, a0); a1 = fmaf(v.w, w3.y, a1); a2 = fmaf(v.w, w3.z, a2); a3 = fmaf(v.w, w3.w, a3);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
      a2 += __shfl_xor_sync(0xffffffffu, a2, o);
      a3 += __shfl_xor_sync(0xffffffffu, a3, o);
    }
    if (lane < Cout) {
      const float v = (lane == 0 ? a0 : lane == 1 ? a1 : lane == 2 ? a2 : a3) + (bias ? bias[lane] : 0.f);
      out[(((long long)b * Cout + lane) * H + y) * W + x] = v;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Stem: 3x3 conv, pad 1, of the NCHW fp32 image (Cin <= 4) straight into the bf16 NHWC residual stream, with the
// per-channel (sum, sum^2) of the STORED (rounded) values accumulated for the first GroupNorms (unet.py:62-64, 195).
// HBM-bound on the output write (2 B x Cout per pixel); the image itself is tiny.  One CTA = pixels of ONE image;
// thread -> (pixel slot, channel octet); weights [27][Cout] in shared memory.
// S = 2: the semantic encoder's stride-2 stem (encoder/ffhq.py: nn.Conv2d(3, 64, 3, 2, 1)); H, W stay the INPUT size and the
// output is [B][H/2][W/2][Cout].  A thread's 4 output pixels read input columns 2 x0 - 1 .. 2 x0 + 7 of each row.
// DET: deterministic statistics -- no atomics: the thread partials meet in shared memory and are added in slot order, and the
// CTA's sums go to its own slot stats[b][blockIdx.x][Cout][2] (summed over the CTAs in order by stat_parts_reduce).
template <int CIN, int S = 1, bool DET = false>
__global__ void __launch_bounds__(256) stem_conv_bf16_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ bias, __nv_bfloat16* __restrict__ out,
                                                             float* __restrict__ stats, int H, int W, int Cout) {
  extern __shared__ float sm[];
  float* ws = sm;                          // [9*CIN][Cout]
  float* acc = sm + 9 * CIN * Cout;        // [2][Cout] per-CTA statistics
  const int b = blockIdx.y, HW = H * W;
  const int Ho = H / S, Wo = W / S, HWo = Ho * Wo;
  for (int i = threadIdx.x; i < 9 * CIN * Cout; i += 256) ws[i] = w[i];
  for (int i = threadIdx.x; i < 2 * Cout; i += 256) acc[i] = 0.f;
  __syncthreads();
  const int L = Cout >> 3, ppc = 256 / L;  // channel octets, pixel QUADS per CTA pass
  const int oct = threadIdx.x % L, slot = threadIdx.x / L;
  const int c = oct * 8;
  float bv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bv[j] = bias ? bias[c + j] : 0.f;
  float s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s1[j] = s2[j] = 0.f;
  const float* xb = x + (long long)b * CIN * HW;
  const int W4 = Wo >> 2, nquad = Ho * W4;   // Wo % 4 == 0 (host checks): a thread owns 4 horizontally adjacent pixels,
  if (slot < ppc) {                          // so every weight vector read from shared memory feeds 4 x 8 FMAs
    for (int qd = blockIdx.x * ppc + slot; qd < nquad; qd += gridDim.x * ppc) {
      const int y = qd / W4, x0 = (qd - y * W4) * 4;
      float a[4][8];
#pragma unroll
      for (int pp = 0; pp < 4; ++pp)
#pragma unroll
        for (int j = 0; j < 8; ++j) a[pp][j] = bv[j];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int iy = S * y + ky - 1;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
          const float* row = xb + (long long)ci * HW + (long long)iy * W + S * x0;
          float v[S == 1 ? 6 : 9];           // input columns S x0 - 1 .. S x0 + 3 S + 1
          if constexpr (S == 1) {
            const float4 mid = __ldg(reinterpret_cast<const float4*>(row));
            v[0] = x0 > 0 ? __ldg(row - 1) : 0.f;
            v[1] = mid.x; v[2] = mid.y; v[3] = mid.z; v[4] = mid.w;
            v[5] = x0 + 4 < W ? __ldg(row + 4) : 0.f;
          } else {                           // (the right pad column is never read: 2 (x0 + 3) + 1 <= W - 1)
            const float4 m0 = __ldg(reinterpret_cast<const float4*>(row));
            const float4 m1 = __ldg(reinterpret_cast<const float4*>(row + 4));
            v[0] = x0 > 0 ? __ldg(row - 1) : 0.f;
            v[1] = m0.x; v[2] = m0.y; v[3] = m0.z; v[4] = m0.w;
            v[5] = m1.x; v[6] = m1.y; v[7] = m1.z; v[8] = m1.w;
          }
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const float4 w0 = *reinterpret_cast<const float4*>(ws + ((ky * 3 + kx) * CIN + ci) * Cout + c);
            const float4 w1 = *reinterpret_cast<const float4*>(ws + ((ky * 3 + kx) * CIN + ci) * Cout + c + 4);
#pragma unroll
            for (int pp = 0; pp < 4; ++pp) {
              const float vv = v[S * pp + kx];
              a[pp][0] = fmaf(vv, w0.x, a[pp][0]); a[pp][1] = fmaf(vv, w0.y, a[pp][1]);
              a[pp][2] = fmaf(vv, w0.z, a[pp][2]); a[pp][3] = fmaf(vv, w0.w, a[pp][3]);
              a[pp][4] = fmaf(vv, w1.x, a[pp][4]); a[pp][5] = fmaf(vv, w1.y, a[pp][5]);
              a[pp][6] = fmaf(vv, w1.z, a[pp][6]); a[pp][7] = fmaf(vv, w1.w, a[pp][7]);
            }
          }
        }
      }
#pragma unroll
      for (int pp = 0; pp < 4; ++pp) {
        __nv_bfloat162 h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          h[j] = __floats2bfloat162_rn(a[pp][2 * j], a[pp][2 * j + 1]);
          const float2 r = __bfloat1622float2(h[j]);
          s1[2 * j] += r.x; s2[2 * j] = fmaf(r.x, r.x, s2[2 * j]);
          s1[2 * j + 1] += r.y; s2[2 * j + 1] = fmaf(r.y, r.y, s2[2 * j + 1]);
        }
        *reinterpret_cast<uint4*>(out + ((long long)b * HWo + (long long)y * Wo + x0 + pp) * Cout + c) = *reinterpret_cast<uint4*>(h);
      }
    }
    if (stats) {
      if constexpr (DET) {
        float* sp = acc + 2 * Cout + (size_t)slot * 2 * Cout;   // [ppc][2][Cout]
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sp[c + j] = s1[j];
          sp[Cout + c + j] = s2[j];
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          atomicAdd(acc + c + j, s1[j]);
          atomicAdd(acc + Cout + c + j, s2[j]);
        }
      }
    }
  }
  if constexpr (DET) {
    if (stats) {
      __syncthreads();
      for (int i = threadIdx.x; i < Cout; i += 256) {
        float a = 0.f, q = 0.f;
        for (int k = 0; k < ppc; ++k) {
          a += acc[2 * Cout + (size_t)k * 2 * Cout + i];
          q += acc[2 * Cout + (size_t)k * 2 * Cout + Cout + i];
        }
        *reinterpret_cast<float2*>(stats + (((long long)b * gridDim.x + blockIdx.x) * Cout + i) * 2) = make_float2(a, q);
      }
    }
  } else if (stats) {
    __syncthreads();
    for (int i = threadIdx.x; i < Cout; i += 256) {
      atomicAdd(stats + ((long long)b * Cout + i) * 2, acc[i]);
      atomicAdd(stats + ((long long)b * Cout + i) * 2 + 1, acc[Cout + i]);
    }
  }
}

}  // namespace pdae

using namespace pdae;

extern "C" int pdae_conv2d_simt(const void* in, int in_dtype, int in_nchw, const float* w_packed, const float* bias,
                                const float* residual, float* out, int out_nchw, int B, int H, int W, int Cin,
                                int Cout, int ksize, int stride, int pad, int a_silu, pdae_stream_t stream) {
  PDAE_REQUIRE(in && w_packed && out, "conv2d_simt: null pointer");
  PDAE_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv2d_simt: bad dims");
  PDAE_REQUIRE(ksize >= 1 && stride >= 1 && pad >= 0, "conv2d_simt: bad window");
  PDAE_REQUIRE(in_dtype == PDAE_F32 || in_dtype == PDAE_BF16, "conv2d_simt: bad dtype");
  PDAE_REQUIRE(!(in_nchw && in_dtype != PDAE_F32), "conv2d_simt: NCHW input must be fp32");
  ConvArgs p;
  p.in = in; p.w = w_packed; p.bias = bias; p.residual = residual; p.out = out;
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
  p.ksize = ksize; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - ksize) / stride + 1;
  p.Wo = (W + 2 * pad - ksize) / stride + 1;
  PDAE_REQUIRE(p.Ho > 0 && p.Wo > 0, "conv2d_simt: empty output");
  p.in_nchw = in_nchw; p.out_nchw = out_nchw; p.a_silu = a_silu;
  p.M = (long long)B * p.Ho * p.Wo;
  p.K = ksize * ksize * Cin;
  dim3 grid(cdiv(p.M, BM), cdiv(Cout, BN));
  PDAE_REQUIRE(grid.y <= 65535, "conv2d_simt: Cout too large");
  cudaStream_t s = (cudaStream_t)stream;
  const bool vec = (Cin % 4 == 0) && !in_nchw;
  if (in_dtype == PDAE_F32) {
    if (vec) conv_simt_kernel<float, true><<<grid, 256, 0, s>>>(p);
    else conv_simt_kernel<float, false><<<grid, 256, 0, s>>>(p);
  } else {
    if (vec) conv_simt_kernel<__nv_bfloat16, true><<<grid, 256, 0, s>>>(p);
    else conv_simt_kernel<__nv_bfloat16, false><<<grid, 256, 0, s>>>(p);
  }
  PDAE_LAUNCH_CHECK("conv_simt_kernel");
  return PDAE_OK;
}

extern "C" int pdae_conv3x3_smalln(const void* in, int in_dtype, const float* w_packed4, const float* bias,
                                   float* out_nchw, int B, int H, int W, int Cin, int Cout, pdae_stream_t stream) {
  PDAE_REQUIRE(in && w_packed4 && out_nchw, "conv3x3_smalln: null pointer");
  PDAE_REQUIRE(Cout >= 1 && Cout <= 4, "conv3x3_smalln: Cout must be <= 4 (got %d)", Cout);
  PDAE_REQUIRE(Cin % 4 == 0, "conv3x3_smalln: Cin %% 4 != 0");
  const size_t smem = (size_t)9 * Cin * 4 * sizeof(float);
  PDAE_REQUIRE(smem <= 200 * 1024, "conv3x3_smalln: Cin too large for shared weights");
  cudaStream_t s = (cudaStream_t)stream;
  const long long npix = (long long)B * H * W;
  int grid = (int)((npix + 7) / 8);
  if (grid > 148 * 32) grid = 148 * 32;
  if (in_dtype == PDAE_F32) {
    if (smem > 48 * 1024)
      PDAE_CUDA(cudaFuncSetAttribute(conv3x3_smalln_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv3x3_smalln_kernel<float><<<grid, 256, smem, s>>>((const float*)in, w_packed4, bias, out_nchw, B, H, W, Cin, Cout);
  } else if (in_dtype == PDAE_BF16) {
    if (smem > 48 * 1024)
      PDAE_CUDA(cudaFuncSetAttribute(conv3x3_smalln_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv3x3_smalln_kernel<__nv_bfloat16><<<grid, 256, smem, s>>>((const __nv_bfloat16*)in, w_packed4, bias, out_nchw, B, H, W, Cin, Cout);
  } else {
    PDAE_REQUIRE(false, "conv3x3_smalln: bad dtype");
  }
  PDAE_LAUNCH_CHECK("conv3x3_smalln_kernel");
  return PDAE_OK;
}

extern "C" int pdae_stem_conv_bf16(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc,
                                   float* ch_stats, int B, int H, int W, int Cin, int Cout, pdae_stream_t stream) {
  PDAE_REQUIRE(x_nchw && w_packed && out_bf16_nhwc && B > 0 && H > 0 && W > 0, "stem_conv_bf16: bad args");
  PDAE_REQUIRE(Cin >= 1 && Cin <= 4, "stem_conv_bf16: Cin=%d (image channels) must be 1..4", Cin);
  PDAE_REQUIRE(Cout % 8 == 0 && Cout >= 8 && Cout <= 256, "stem_conv_bf16: Cout=%d must be a multiple of 8 in [8, 256]", Cout);
  PDAE_REQUIRE(B <= 65535, "stem_conv_bf16: B too large for grid.y");
  PDAE_REQUIRE(W % 4 == 0 && ((uintptr_t)x_nchw & 15) == 0, "stem_conv_bf16: W=%d must be a multiple of 4 (16-byte aligned rows)", W);
  const int ppc = 256 / (Cout / 8);
  int gx = cdiv((long long)H * (W / 4), (long long)ppc * 2);   // ~2 pixel quads per thread: amortises the weight load and the flush
  if (gx > 148 * 8) gx = 148 * 8;
  if (gx < 1) gx = 1;
  const size_t smem = (size_t)(9 * Cin + 2) * Cout * sizeof(float);
  dim3 grid(gx, B);
  cudaStream_t s = (cudaStream_t)stream;
  __nv_bfloat16* o = (__nv_bfloat16*)out_bf16_nhwc;
  switch (Cin) {
    case 1: stem_conv_bf16_kernel<1><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    case 2: stem_conv_bf16_kernel<2><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    case 3: stem_conv_bf16_kernel<3><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    default: stem_conv_bf16_kernel<4><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
  }
  PDAE_LAUNCH_CHECK("stem_conv_bf16_kernel");
  return PDAE_OK;
}

extern "C" int pdae_stem_conv_s2_bf16(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc,
                                      float* ch_stats, int B, int H, int W, int Cin, int Cout, pdae_stream_t stream) {
  PDAE_REQUIRE(x_nchw && w_packed && out_bf16_nhwc, "stem_conv_s2_bf16: null pointer");
  PDAE_REQUIRE(B > 0 && B <= 65535, "stem_conv_s2_bf16: B=%d must be in [1, 65535]", B);
  PDAE_REQUIRE(Cin >= 1 && Cin <= 4, "stem_conv_s2_bf16: Cin=%d (image channels) must be 1..4", Cin);
  PDAE_REQUIRE(Cout % 8 == 0 && Cout >= 8 && Cout <= 256, "stem_conv_s2_bf16: Cout=%d must be a multiple of 8 in [8, 256]", Cout);
  PDAE_REQUIRE(H >= 2 && W >= 8 && H % 2 == 0 && W % 8 == 0,
               "stem_conv_s2_bf16: H=%d W=%d: H must be even and W a multiple of 8 (4-pixel output quads)", H, W);
  PDAE_REQUIRE(!(((uintptr_t)x_nchw | (uintptr_t)out_bf16_nhwc) & 15), "stem_conv_s2_bf16: x and out must be 16-byte aligned");
  PDAE_REQUIRE(!((uintptr_t)ch_stats & 3), "stem_conv_s2_bf16: ch_stats must be 4-byte aligned");
  const int Ho = H / 2, Wo = W / 2;
  const int ppc = 256 / (Cout / 8);
  int gx = cdiv((long long)Ho * (Wo / 4), (long long)ppc * 2);
  if (gx > 148 * 8) gx = 148 * 8;
  if (gx < 1) gx = 1;
  const size_t smem = (size_t)(9 * Cin + 2) * Cout * sizeof(float);
  dim3 grid(gx, B);
  cudaStream_t s = (cudaStream_t)stream;
  __nv_bfloat16* o = (__nv_bfloat16*)out_bf16_nhwc;
  switch (Cin) {
    case 1: stem_conv_bf16_kernel<1, 2><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    case 2: stem_conv_bf16_kernel<2, 2><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    case 3: stem_conv_bf16_kernel<3, 2><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
    default: stem_conv_bf16_kernel<4, 2><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, ch_stats, H, W, Cout); break;
  }
  PDAE_LAUNCH_CHECK("stem_conv_bf16_kernel<stride 2>");
  return PDAE_OK;
}

// Deterministic stems: the same convs, with the statistics in fixed slots (one per CTA) summed in a fixed order.  The CTA count
// follows (H, W, Cout, stride) only.
static int stem_grid_x(int H, int W, int Cout, int stride) {
  const int Ho = H / stride, Wo = W / stride, ppc = 256 / (Cout / 8);
  int gx = cdiv((long long)Ho * (Wo / 4), (long long)ppc * 2);
  if (gx > 148 * 8) gx = 148 * 8;
  return gx < 1 ? 1 : gx;
}

extern "C" int64_t pdae_stem_conv_det_workspace_bytes(int B, int H, int W, int Cout, int stride) {
  if (B <= 0 || H <= 0 || W <= 0 || Cout % 8 != 0 || Cout < 8 || Cout > 256 || (stride != 1 && stride != 2)) {
    ::pdae::set_error("stem_conv_det_workspace_bytes: B=%d H=%d W=%d Cout=%d stride=%d unsupported", B, H, W, Cout, stride);
    return PDAE_EINVAL;
  }
  return (int64_t)B * stem_grid_x(H, W, Cout, stride) * Cout * 2 * (int64_t)sizeof(float);
}

extern "C" int pdae_stem_conv_bf16_det(const float* x_nchw, const float* w_packed, const float* bias, void* out_bf16_nhwc,
                                       float* ch_stats, int B, int H, int W, int Cin, int Cout, int stride, float* workspace,
                                       int64_t workspace_bytes, pdae_stream_t stream) {
  PDAE_REQUIRE(x_nchw && w_packed && out_bf16_nhwc && ch_stats && workspace, "stem_conv_bf16_det: null pointer");
  PDAE_REQUIRE(stride == 1 || stride == 2, "stem_conv_bf16_det: stride=%d must be 1 or 2", stride);
  PDAE_REQUIRE(B > 0 && B <= 65535, "stem_conv_bf16_det: B=%d must be in [1, 65535]", B);
  PDAE_REQUIRE(Cin >= 1 && Cin <= 4, "stem_conv_bf16_det: Cin=%d (image channels) must be 1..4", Cin);
  PDAE_REQUIRE(Cout % 8 == 0 && Cout >= 8 && Cout <= 256, "stem_conv_bf16_det: Cout=%d must be a multiple of 8 in [8, 256]", Cout);
  PDAE_REQUIRE(stride == 1 ? (H > 0 && W > 0 && W % 4 == 0) : (H >= 2 && W >= 8 && H % 2 == 0 && W % 8 == 0),
               "stem_conv_bf16_det: H=%d W=%d unsupported at stride %d", H, W, stride);
  PDAE_REQUIRE(!(((uintptr_t)x_nchw | (uintptr_t)out_bf16_nhwc) & 15) && !(((uintptr_t)ch_stats | (uintptr_t)workspace) & 7),
               "stem_conv_bf16_det: x and out must be 16-byte, ch_stats and workspace 8-byte aligned");
  const int gx = stem_grid_x(H, W, Cout, stride);
  const long long need = (long long)B * gx * Cout * 2 * (long long)sizeof(float);
  PDAE_REQUIRE(workspace_bytes >= need, "stem_conv_bf16_det: workspace of %lld bytes, %lld needed (pdae_stem_conv_det_workspace_bytes)",
               (long long)workspace_bytes, need);
  const int ppc = 256 / (Cout / 8);
  const size_t smem = (size_t)(9 * Cin + 2 + 2 * ppc) * Cout * sizeof(float);
  PDAE_REQUIRE(smem <= 48 * 1024, "stem_conv_bf16_det: Cin=%d Cout=%d need %zu bytes of shared memory (at most 48 KiB)", Cin, Cout,
               smem);
  dim3 grid(gx, B);
  cudaStream_t s = (cudaStream_t)stream;
  __nv_bfloat16* o = (__nv_bfloat16*)out_bf16_nhwc;
#define PDAE_STEM_DET(S)                                                                                                     \
  switch (Cin) {                                                                                                             \
    case 1: stem_conv_bf16_kernel<1, S, true><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, workspace, H, W, Cout); break; \
    case 2: stem_conv_bf16_kernel<2, S, true><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, workspace, H, W, Cout); break; \
    case 3: stem_conv_bf16_kernel<3, S, true><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, workspace, H, W, Cout); break; \
    default: stem_conv_bf16_kernel<4, S, true><<<grid, 256, smem, s>>>(x_nchw, w_packed, bias, o, workspace, H, W, Cout); break; \
  }
  if (stride == 1) PDAE_STEM_DET(1) else PDAE_STEM_DET(2)
#undef PDAE_STEM_DET
  PDAE_LAUNCH_CHECK("stem_conv_bf16_kernel<det>");
  PDAE_CUDA(launch_stat_parts_reduce(workspace, B, gx, Cout, ch_stats, s));
  return PDAE_OK;
}
